"""Parameter trees of the supported ansatzes: names, shapes, initialisation, packing.

Names follow the Haiku module paths the reference produces (visible for the test ansatz in
the reference's tests/test_wf/test_grad_psi.npz) so that parameters dumped from a reference
run with ``tests/conftest.py:39-52 flatten_pytree`` (':'-joined) load unchanged:
``<module path>:<param>``.  Initialisers restate the reference's choices
(src/deepqmc/hkext.py:66-80 'ferminet' init = VarianceScaling(1, fan_in, normal) weights and
VarianceScaling(1, fan_out, normal) biases; conf/ansatz/psiformer.yaml:10 envelopes to ones;
gnn/update_features.py:276 attention weights VarianceScaling(1, fan_in, normal)).
JAX's threefry stream cannot be reproduced, so values differ from a reference run with the
same seed; distributions match.
"""
from __future__ import annotations

import numpy as np

from .spec import AnsatzSpec, log_dims

P = 'neural_network_wave_function/~/'
ENV = P + 'exponential_envelopes'
CUSP = P + 'electronic_cusp_asymptotic'
NUC_CUSP = P + 'nuclear_cusp_asymptotic'
GNN = P + 'omni_net/~/electron_gnn/~/'
BF_UP = P + 'omni_net/~/Backflow/~/mlp/linear_0'
BF_DN = P + 'omni_net/~/Backflow_1/~/mlp/linear_0'
# second net of Backflow(multi_head=True, n_backflows=2) with backflow_transform = 'both' (wf/omni.py:69-73)
BF_UP_ADD = P + 'omni_net/~/Backflow/~/mlp_1/linear_0'
BF_DN_ADD = P + 'omni_net/~/Backflow_1/~/mlp_1/linear_0'


NUC_EMB = GNN + 'nuclei_embedding/'
HEAD = P + 'omni_net/~/nuclear_gnn_head/'


JASTROW = P + 'omni_net/~/Jastrow/~/mlp/'
CONF = P + 'conf_coeff'
EDGE_TYPES = ('same', 'anti', 'ne')


def conv_prefix(l):
    return layer_prefix(l) + 'convolution_electron_update_feature/~single_edge_type_update/'


def backflow_dims(spec, n_spin):
    n_orb = spec.n_elec if spec.full_determinant else n_spin
    return log_dims(spec.embedding_dim, spec.n_determinants * n_orb, spec.backflow_layers)


def comb_prefix(l):
    return layer_prefix(l) + 'combined_node_attention_update_feature/'


def layer_prefix(l):
    return GNN + ('electron_gnn_layer' if l == 0 else f'electron_gnn_layer_{l}') + '/~/'


def attn_prefix(l):
    return layer_prefix(l) + 'node_attention_electron_update_feature/'


def param_shapes(spec: AnsatzSpec) -> dict[str, tuple[int, ...]]:
    N, M, d, K = spec.n_elec, spec.n_nuc, spec.embedding_dim, spec.n_determinants
    s: dict[str, tuple[int, ...]] = {}
    if spec.kind == 'paulinet':
        # reference: tests/conf/ansatz.yaml / conf/ansatz/default.yaml; wf/env.py:10-75
        n_env, e = len(spec.env_centers), spec.edge_dim
        if spec.env_per_shell:  # per_shell, shared zetas, spin-restricted
            s[f'{ENV}:pi'] = (K * N, n_env)
            s[f'{ENV}:zetas'] = (n_env,)
        else:
            for nm in ('pi_up', 'pi_down', 'zetas_up', 'zetas_down'):
                s[f'{ENV}:{nm}'] = (K * N, M)
        if spec.gnn_embedding == 'embed':
            s[GNN + 'electron_embedding/ElectronicEmbedding:embeddings'] = (1 if spec.n_up == spec.n_down else 2, d)
        if spec.gnn_conv_ne:
            s[GNN + 'nuclei_embedding/~/embed:embeddings'] = (M, d)
        types = EDGE_TYPES if spec.gnn_conv_ne else EDGE_TYPES[:2]
        d_in, e_in = (d if spec.gnn_embedding == 'embed' else 4 * M), 4
        for l in range(spec.n_layers):
            c, lp = conv_prefix(l), layer_prefix(l)
            for t in types:
                dw = [e_in] + log_dims(e_in, e, spec.gnn_subnet_layers)   # w: edges -> two_particle_stream_dim
                dh = [d_in if t != 'ne' else d] + log_dims(d_in if t != 'ne' else d, e, spec.gnn_subnet_layers)
                for i in range(spec.gnn_subnet_layers):
                    s[c + f'w_{t}/linear_{i}:w'] = (dw[i], dw[i + 1])
                    if spec.gnn_update == 'concatenate':  # default.yaml: w_factory bias true; test ansatz: false
                        s[c + f'w_{t}/linear_{i}:b'] = (dw[i + 1],)
                    s[c + f'h_{t}/linear_{i}:w'] = (dh[i], dh[i + 1])
                    s[c + f'h_{t}/linear_{i}:b'] = (dh[i + 1],)
                if spec.gnn_update == 'featurewise':
                    s[lp + f'g_conv_{t}/linear_0:w'] = (e, d)
                    s[lp + f'g_conv_{t}/linear_0:b'] = (d,)
            if spec.gnn_update == 'concatenate':
                s[lp + 'g/linear_0:w'] = (3 * d_in + len(types) * e, d)
                if spec.gnn_g_bias:
                    s[lp + 'g/linear_0:b'] = (d,)
            if spec.gnn_deep_edges and l < spec.n_layers - 1:
                du = [e_in] + log_dims(e_in, e, spec.gnn_subnet_layers)
                for i in range(spec.gnn_subnet_layers):
                    s[lp + f'u/linear_{i}:w'] = (du[i], du[i + 1])
                    s[lp + f'u/linear_{i}:b'] = (du[i + 1],)
                e_in = e
            d_in = d
        dj = [d] + log_dims(d, 1, spec.jastrow_layers) if spec.jastrow_layers else []
        for i in range(len(dj) - 1):
            s[JASTROW + f'linear_{i}:w'] = (dj[i], dj[i + 1])
            if i < len(dj) - 2:  # bias: 'not_last'
                s[JASTROW + f'linear_{i}:b'] = (dj[i + 1],)
        for pre, n_spin in ((BF_UP, spec.n_up), (BF_DN, spec.n_down)):
            db = [d] + backflow_dims(spec, n_spin)
            base = pre.rsplit('linear_0', 1)[0]
            for i in range(len(db) - 1):
                s[base + f'linear_{i}:w'] = (db[i], db[i + 1])
                if spec.backflow_bias:
                    s[base + f'linear_{i}:b'] = (db[i + 1],)
        if spec.conf_coeff == 'linear':
            s[CONF + ':w'] = (K, 1)
        return s
    if spec.kind == 'deeperwin':
        return deeperwin_shapes(spec)
    if spec.kind != 'transpsiformer':
        for nm in ('pi_up', 'pi_down', 'zetas_up', 'zetas_down'):
            s[f'{ENV}:{nm}'] = (K * N, M)
    if spec.cusp == 'psiformer':
        s[f'{CUSP}:same_alpha'] = ()
        s[f'{CUSP}:anti_alpha'] = ()
    if spec.cusp_nuclei != 'none' and spec.cusp_nuclei_trainable:
        s[f'{NUC_CUSP}:nuc_alpha'] = ()
    if spec.kind == 'psiformer':
        s[GNN + 'electron_embedding/linear:w'] = (spec.n_feat_in, d)
        for l in range(spec.n_layers):
            a = attn_prefix(l)
            for nm in ('query', 'key', 'value', 'linear'):
                s[a + f'multi_head_attention/{nm}:w'] = (d, d)
            for i in range(2):
                s[a + f'mlp/linear_{i}:w'] = (d, d)
                s[a + f'mlp/linear_{i}:b'] = (d,)
    elif spec.kind == 'ferminet':
        de = spec.edge_dim
        d_in, e_in = spec.n_feat_in, 4
        for l in range(spec.n_layers):
            lp = layer_prefix(l)
            s[lp + 'g/linear_0:w'] = (3 * d_in + 2 * e_in, d)
            s[lp + 'g/linear_0:b'] = (d,)
            if l < spec.n_layers - 1:
                s[lp + 'u/linear_0:w'] = (e_in, de)
                s[lp + 'u/linear_0:b'] = (de,)
            d_in, e_in = d, de
    elif spec.kind == 'transpsiformer':
        # reference: conf/ansatz/transpsiformer.yaml; gnn/electron_gnn.py:435-537 NucleiEmbedding,
        # gnn/update_features.py:385-451 CombinedNodeAttentionUpdateFeature, wf/omni.py:181-211 head
        de, E = spec.nuc_edge_dim, spec.n_env_per_nuc
        s[GNN + 'electron_embedding/linear:w'] = (spec.n_feat_in, d)
        for nm, (i, o) in (('edge_mlp/linear_0', (4 + M, de)), ('edge_mlp/linear_1', (de, de)),
                           ('embed_mlp/linear_0', (de, d)), ('embed_mlp/linear_1', (d, d))):
            s[NUC_EMB + nm + ':w'] = (i, o)
            s[NUC_EMB + nm + ':b'] = (o,)
        for l in range(spec.n_layers):
            a = comb_prefix(l)
            for nm in ('query', 'key', 'value', 'linear'):
                s[a + f'multi_head_attention/{nm}:w'] = (d, d)
            for i in range(2):
                s[a + f'mlp/linear_{i}:w'] = (d, d)
                s[a + f'mlp/linear_{i}:b'] = (d,)
        for glu, spin in (('zetas_readout_glu', 'up'), ('zetas_readout_glu_1', 'down')):
            for lin in ('W', 'V'):
                s[HEAD + f'{glu}/{lin}:w'] = (d, K * E)
                s[HEAD + f'{glu}/{lin}:b'] = (K * E,)
            s[HEAD + f':zetas_bias_{spin}'] = (M, K, E)
    else:
        raise ValueError(spec.kind)
    s[BF_UP + ':w'] = (d, K * N)
    s[BF_DN + ':w'] = (d, K * N)
    if spec.backflow_transform == 'both':
        s[BF_UP_ADD + ':w'] = (d, K * N)
        s[BF_DN_ADD + ':w'] = (d, K * N)
    return s


DEEPERWIN_EDGE_IN = {'same': 1, 'anti': 1, 'ne': 4}  # DistancePowerEdgeFeature([1]) | + DifferenceEdgeFeature


def deeperwin_edge_width(spec, t, l):
    """Width of the type-t edge stream entering layer l: the raw features, then two_particle_stream_dim after the
    first deep update (electron_gnn.py:160-192)."""
    return DEEPERWIN_EDGE_IN[t] if l == 0 else spec.edge_dim


def n_atom_types(spec):
    return len(set(spec.charges))


def deeperwin_shapes(spec: AnsatzSpec) -> dict[str, tuple[int, ...]]:
    """reference: conf/ansatz/deeperwin.yaml; gnn/electron_gnn.py:72-158 (u<type> per edge type), :435-537
    (NucleiEmbedding: hk.Embed over atom types), gnn/update_features.py:162-238 (w_same / w_anti, no w_ne, h_<type> with
    the width of the filter), hkext.py:22-113 (MLP ['log', 1] = one Linear), wf/env.py:10-75 (one shell per nucleus)."""
    N, M, d, K, e = spec.n_elec, spec.n_nuc, spec.embedding_dim, spec.n_determinants, spec.edge_dim
    s: dict[str, tuple[int, ...]] = {}
    for nm in ('pi_up', 'pi_down', 'zetas_up', 'zetas_down'):
        s[f'{ENV}:{nm}'] = (K * N, M)
    s[GNN + 'nuclei_embedding/~/embed:embeddings'] = (n_atom_types(spec), spec.nuc_embedding_dim)
    d_in = 4 * M
    for l in range(spec.n_layers):
        c, lp = conv_prefix(l), layer_prefix(l)
        for t in ('same', 'anti'):
            s[c + f'w_{t}/linear_0:w'] = (deeperwin_edge_width(spec, t, l), e)
            s[c + f'w_{t}/linear_0:b'] = (e,)
            s[c + f'h_{t}/linear_0:w'] = (d_in, e)
            s[c + f'h_{t}/linear_0:b'] = (e,)
        ene = deeperwin_edge_width(spec, 'ne', l)
        s[c + 'h_ne/linear_0:w'] = (spec.nuc_embedding_dim, ene)
        s[c + 'h_ne/linear_0:b'] = (ene,)
        s[lp + 'g/linear_0:w'] = (3 * d_in + e + ene, d)
        s[lp + 'g/linear_0:b'] = (d,)
        if l < spec.n_layers - 1:
            for t in ('ne', 'same', 'anti'):
                s[lp + f'u{t}/linear_0:w'] = (deeperwin_edge_width(spec, t, l), e)
                s[lp + f'u{t}/linear_0:b'] = (e,)
        d_in = d
    s[BF_UP + ':w'] = (d, K * N)
    s[BF_DN + ':w'] = (d, K * N)
    return s


def init_params(spec: AnsatzSpec, seed: int = 0) -> dict[str, np.ndarray]:
    """Ansatz.init equivalent (reference: src/deepqmc/types.py:119-131)."""
    rng = np.random.default_rng(seed)
    out = {}
    for name, shape in param_shapes(spec).items():
        leaf = name.rsplit(':', 1)[1]
        if spec.kind == 'deeperwin' and leaf in ('w', 'b') and not name.startswith(ENV):
            # init 'deeperwin' (hkext.py:66-80): VarianceScaling(1, fan_avg, uniform) weights, zero biases
            lim = np.sqrt(3.0 / ((shape[0] + shape[1]) / 2)) if leaf == 'w' else 0.0
            v = rng.uniform(-lim, lim, size=shape)
        elif name == f'{ENV}:zetas' and spec.kind == 'paulinet':
            v = np.asarray(spec.env_zeta_init, dtype=np.float64)  # init_to_ones = false: z / (k + 1)
        elif name == f'{ENV}:pi' and spec.kind == 'paulinet':
            v = 1.0 + rng.standard_normal(shape) / np.sqrt(shape[0])
        elif name == CONF + ':w':
            v = np.ones(shape)  # w_init = jnp.ones
        elif leaf == 'embeddings':
            v = rng.standard_normal(shape)  # hk.Embed default: truncated normal
        elif name.startswith(ENV):
            v = np.ones(shape)
        elif name.startswith(NUC_CUSP):
            v = spec.cusp_nuclei_alpha * np.ones(shape)
        elif name.startswith(CUSP):
            v = np.ones(shape)
        elif leaf.startswith('zetas_bias'):
            v = 2 * np.ones(shape)  # wf/omni.py:199-203
        elif leaf == 'w':
            v = rng.standard_normal(shape) / np.sqrt(shape[0])
        elif leaf == 'b':
            v = rng.standard_normal(shape) / np.sqrt(shape[0])
        else:
            raise AssertionError(name)
        out[name] = np.asarray(v, dtype=np.float64)
    return out


def perturb_params(params, seed=1, scale=0.2):
    """Randomise the parameters that initialise to constants (envelopes, cusp alphas) so
    parity tests exercise them; used by tests and the benchmark's synthetic weights."""
    rng = np.random.default_rng(seed)
    out = dict(params)
    for k, v in params.items():
        if k.startswith(ENV) or k.startswith(CUSP) or k.startswith(NUC_CUSP) or 'zetas_bias' in k or k == CONF + ':w':
            out[k] = v * (1 + scale * rng.uniform(-1, 1, size=v.shape))
    return out


def n_params(spec):
    return int(sum(int(np.prod(s)) for s in param_shapes(spec).values()))


# ---- exchange with a reference run ------------------------------------------------------------------------------------
def flatten_haiku_tree(tree: dict, sep: str = ':') -> dict:
    """{'<module path>': {'<name>': array}} (the nested dict Haiku returns from init) -> {'<module path>:<name>': array},
    the key layout of this module and of the reference's own test helper (tests/conftest.py:39-52 flatten_pytree)."""
    out = {}
    for mod, leaves in tree.items():
        if isinstance(leaves, dict):
            for name, v in leaves.items():
                out[f'{mod}{sep}{name}'] = np.asarray(v)
        else:  # already flat
            out[mod] = np.asarray(leaves)
    return out


def unflatten_haiku_tree(flat: dict, sep: str = ':') -> dict:
    out: dict = {}
    for k, v in flat.items():
        mod, name = k.rsplit(sep, 1)
        out.setdefault(mod, {})[name] = np.asarray(v)
    return out


def save_params(path: str, params: dict) -> None:
    """np.savez of a flat or nested parameter tree with the ':'-flattened Haiku names (what
    ``np.savez(path, **flatten_pytree(params))`` writes on the reference side)."""
    flat = flatten_haiku_tree(params) if any(isinstance(v, dict) for v in params.values()) else params
    np.savez(path, **{k: np.asarray(v) for k, v in flat.items()})


def load_params(path: str, spec: AnsatzSpec | None = None) -> dict:
    """Read such a file; with ``spec`` the names and shapes are checked against the ansatz (a missing, extra or misshapen
    leaf raises instead of silently evaluating a different wave function)."""
    with np.load(path) as f:
        flat = {k: np.asarray(f[k], dtype=np.float64) for k in f.files}
    if spec is not None:
        want = param_shapes(spec)
        if set(flat) != set(want):
            raise ValueError(f'parameter names differ: missing {sorted(set(want) - set(flat))[:3]}, unexpected {sorted(set(flat) - set(want))[:3]}')
        for k, shp in want.items():
            if tuple(flat[k].shape) != tuple(shp):
                raise ValueError(f'{k}: shape {flat[k].shape}, expected {tuple(shp)}')
    return flat
