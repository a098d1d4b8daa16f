"""Ansatz hyper-parameter record shared by the CUDA engine, the host shims and the tests.

The fields restate the knobs of the reference's hydra ansatz YAMLs that fix kernel shapes
(reference: src/deepqmc/conf/ansatz/psiformer.yaml, ferminet.yaml; SURVEY.md 8(a0)).
Pure data: no arithmetic.
"""
from __future__ import annotations

import dataclasses

__all__ = ['AnsatzSpec', 'psiformer_spec', 'ferminet_spec', 'transpsiformer_spec', 'paulinet_spec', 'paulinet_default_spec',
           'deeperwin_spec', 'log_dims']


@dataclasses.dataclass(frozen=True)
class AnsatzSpec:
    kind: str  # 'psiformer' | 'ferminet' | 'transpsiformer' | 'paulinet' | 'deeperwin'
    n_up: int
    n_down: int
    n_nuc: int
    embedding_dim: int = 256
    n_layers: int = 4
    n_heads: int = 4
    n_determinants: int = 16
    edge_dim: int = 32  # two_particle_stream_dim (FermiNet)
    # e-e cusp (reference: conf/ansatz/psiformer.yaml:18-26); 'none' for FermiNet
    cusp: str = 'psiformer'
    cusp_same_scale: float = 0.25
    cusp_anti_scale: float = 0.5
    # nuclear cusp factor (reference wf/cusp.py:81-101; `cusp_nuclei: false` in every shipped ansatz yaml)
    cusp_nuclei: str = 'none'  # 'none' | 'psiformer' | 'deepqmc'
    cusp_nuclei_alpha: float = 1.0
    cusp_nuclei_trainable: bool = True
    # TransPsiformer (reference: conf/ansatz/transpsiformer.yaml): nuclei are extra attention tokens
    # (elec_to_nuc = false) and the envelope exponents are read out of the nuclear embeddings
    n_env_per_nuc: int = 1  # SimplifiedNucleusDependentEnvelopes.n_envelope_per_nucleus (3)
    nuc_edge_dim: int = 32  # NucleiEmbedding edge_mlp width (gnn/electron_gnn.py:476-484)
    charges: tuple = ()     # nuclear charges (atom-type one-hot of the nuclear embedding)
    # conv-GNN family ("PauliNet" of the reference's tests, tests/conf/ansatz.yaml = BASELINE configs[0]):
    full_determinant: bool = True   # False: det_up(n_up x n_up) * det_down(n_down x n_down)
    conf_coeff: str = 'sum'         # 'sum' = SumPool | 'linear' = hk.Linear(1, no bias, init ones)
    cusp_alpha: float = 10.0        # fixed alpha of the DeepQMCCusp (wf/cusp.py:5-14)
    mult_act: str = 'identity'      # 'identity' | 'default' = 1 + 2 tanh(x / 4) (wf/nn_wave_function.py:17)
    jastrow_layers: int = 0         # hidden_layers ['log', n] of the Jastrow MLP on sum_i x_i; 0 = no Jastrow
    backflow_layers: int = 1        # hidden_layers ['log', n] of the per-spin backflow MLPs
    env_centers: tuple = ()         # per_shell envelopes: nucleus index of every envelope (wf/env.py:26-33)
    env_zeta_init: tuple = ()       # their initial exponents z / (k + 1)
    # conv-GNN variants (tests/conf/ansatz.yaml vs conf/ansatz/default.yaml):
    gnn_embedding: str = 'embed'    # 'embed': hk.Embed lookup | 'features': raw [|r_iI|, d_iI] for all nuclei (4 M wide)
    gnn_update: str = 'featurewise' # 'featurewise': sum_t g_t(conv_t) | 'concatenate': g([h, mean_up h, mean_down h, conv_same, conv_anti])
    gnn_conv_ne: bool = True        # nucleus -> electron convolution (needs the nuclear hk.Embed table)
    gnn_subnet_layers: int = 1      # layers of the w / h (and u) MLPs (hidden_layers ['log', n])
    gnn_deep_edges: bool = False    # deep_features 'shared': edge MLP u + normalised residual between layers
    gnn_residual_normalize: bool = False  # electron ResidualConnection(normalize=...)
    gnn_g_bias: bool = True
    backflow_bias: bool = True
    env_per_shell: bool = True      # False: one per-orbital exponent per nucleus, spin-unrestricted (as Psiformer)
    # BackflowOp branches (wf/nn_wave_function.py:14-33,111-125): 'mult' in every shipped config; 'add' / 'both' add
    # cutoff(r_i) * |envelope_i| * 0.1 tanh(f_add / 4) (Psiformer / FermiNet kinds)
    backflow_transform: str = 'mult'
    # DeepErwin (kind 'deeperwin'): width of the nuclear hk.Embed table that feeds h_ne (gnn/electron_gnn.py:513-514)
    nuc_embedding_dim: int = 32

    @property
    def n_elec(self):
        return self.n_up + self.n_down

    @property
    def head_dim(self):
        return self.embedding_dim // self.n_heads

    @property
    def n_feat_in(self):
        # Psiformer: [log1p|r_iI|, d_iI log1p/r] for all I (+) spin; FermiNet: [|r_iI|, d_iI]
        return 4 * self.n_nuc + (1 if self.kind in ('psiformer', 'transpsiformer') else 0)


def psiformer_spec(hamil, **kw):
    """reference: src/deepqmc/conf/ansatz/psiformer.yaml"""
    kw.setdefault('charges', tuple(float(z) for z in hamil.mol.charges))
    return AnsatzSpec('psiformer', hamil.n_up, hamil.n_down, hamil.n_nuc, **kw)


def ferminet_spec(hamil, **kw):
    """reference: src/deepqmc/conf/ansatz/ferminet.yaml"""
    kw.setdefault('cusp', 'none')
    kw.setdefault('charges', tuple(float(z) for z in hamil.mol.charges))
    return AnsatzSpec('ferminet', hamil.n_up, hamil.n_down, hamil.n_nuc, **kw)


def transpsiformer_spec(hamil, **kw):
    """reference: src/deepqmc/conf/ansatz/transpsiformer.yaml"""
    kw.setdefault('n_env_per_nuc', 3)
    kw.setdefault('charges', tuple(float(z) for z in hamil.mol.charges))
    return AnsatzSpec('transpsiformer', hamil.n_up, hamil.n_down, hamil.n_nuc, **kw)


def log_dims(d_in, d_out, n):
    """hidden_layers ['log', n] of the reference's MLP (hkext.py:95-99): n layer widths ending in d_out."""
    return [round(d_in ** (1 - k / n) * d_out ** (k / n)) for k in range(1, n + 1)]


def paulinet_spec(hamil, **kw):
    """reference: tests/conf/ansatz.yaml (the conv-GNN 'PauliNet' ansatz of the reference's own CPU tests,
    BASELINE configs[0]): embedding lookup, one featurewise convolution layer over same / anti / ne edges,
    ssp Jastrow and backflow MLPs, per-shell spin-restricted envelopes, spin-factorised determinants,
    hk.Linear determinant combination, DeepQMCCusp."""
    shells = []
    for i, (z, n_shell, n_ecp) in enumerate(zip(hamil.mol.charges, hamil.mol_shells, hamil.mol_ecp_shells)):
        for k in range(n_ecp, n_shell):  # per_shell = true (wf/env.py:26-33)
            shells.append((i, float(z) / (k + 1)))
    kw.setdefault('embedding_dim', 8)
    kw.setdefault('n_layers', 1)
    kw.setdefault('n_determinants', 2)
    kw.setdefault('edge_dim', 8)
    kw.setdefault('cusp', 'deepqmc')
    kw.setdefault('full_determinant', False)
    kw.setdefault('conf_coeff', 'linear')
    kw.setdefault('mult_act', 'default')
    kw.setdefault('jastrow_layers', 3)
    kw.setdefault('backflow_layers', 3)
    kw.setdefault('env_centers', tuple(c for c, _ in shells))
    kw.setdefault('env_zeta_init', tuple(z for _, z in shells))
    kw.setdefault('charges', tuple(float(z) for z in hamil.mol.charges))
    return AnsatzSpec('paulinet', hamil.n_up, hamil.n_down, hamil.n_nuc, **kw)


def paulinet_default_spec(hamil, **kw):
    """reference: src/deepqmc/conf/ansatz/default.yaml (the "PauliNet" column of SURVEY.md 8(a0)): raw
    nucleus-electron features, 3 layers of [h, mean_up, mean_down, conv_same, conv_anti] -> Linear+tanh with
    normalised residuals, two-layer tanh w / h MLPs, shared deep edge MLP, linear Jastrow and backflow,
    full determinants, per-orbital envelopes, hk.Linear conf_coeff, DeepQMCCusp."""
    d = dict(embedding_dim=128, n_layers=3, n_determinants=16, edge_dim=32, cusp='deepqmc', full_determinant=True,
             conf_coeff='linear', mult_act='identity', jastrow_layers=1, backflow_layers=1, backflow_bias=False,
             gnn_embedding='features', gnn_update='concatenate', gnn_conv_ne=False, gnn_subnet_layers=2,
             gnn_deep_edges=True, gnn_residual_normalize=True, gnn_g_bias=False, env_per_shell=False)
    d.update(kw)
    d.setdefault('charges', tuple(float(z) for z in hamil.mol.charges))
    return AnsatzSpec('paulinet', hamil.n_up, hamil.n_down, hamil.n_nuc, **d)


def deeperwin_spec(hamil, **kw):
    """reference: src/deepqmc/conf/ansatz/deeperwin.yaml -- the conv-GNN family with raw nucleus-electron features
    ([|d|, d] for every nucleus, no projection), |d| on same / anti edges and [|d|, d] on ne edges, same-spin edges with
    self-interaction, 4 layers of x <- tanh(g([x, mean_up x, mean_down x, conv_ee, conv_ne])) without residual, where
    conv_ee = conv_same + conv_anti and the ne convolution uses the ne edge stream itself as filter (w_for_ne: false) on
    h_ne of a 32-wide nuclear hk.Embed over atom types; separate deep edge MLPs u_same / u_anti / u_ne with normalised
    residual; one-layer tanh w / h / u / g MLPs with bias; linear bias-free backflow; 32 full determinants, SumPool, no
    cusp, no Jastrow; isotropic per-orbital spin-unrestricted envelopes exp(-softplus(zeta) |d|)."""
    d = dict(embedding_dim=256, n_layers=4, n_determinants=32, edge_dim=32, cusp='none', full_determinant=True,
             conf_coeff='sum', mult_act='identity', jastrow_layers=0, backflow_layers=1, backflow_bias=False,
             gnn_embedding='features', gnn_update='concatenate', gnn_conv_ne=True, gnn_subnet_layers=1,
             gnn_deep_edges=True, gnn_residual_normalize=False, gnn_g_bias=True, env_per_shell=False)
    d.update(kw)
    d.setdefault('charges', tuple(float(z) for z in hamil.mol.charges))
    return AnsatzSpec('deeperwin', hamil.n_up, hamil.n_down, hamil.n_nuc, **d)
