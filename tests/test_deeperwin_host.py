"""CPU: the DeepErwin ansatz (reference conf/ansatz/deeperwin.yaml) -- its parameter table, the fp64 oracle of
tests/deeperwin_oracle.py, the walker-independent upload (h_ne tables, softplus exponents) and the workspace plan."""
import numpy as np
import pytest
import torch

import deeperwin_oracle as DO
from deepqmc_b200 import params as PN
from deepqmc_b200.engine import (MODE_FORWARD, MODE_LANGEVIN, MODE_LOCAL_ENERGY, MODE_MCMC, MODE_VJP, Engine,
                                 _pack_haiku_params)
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from deepqmc_b200.spec import deeperwin_spec
from oracle import names as ON
from oracle import wf as owf
from oracle.laplacian import laplacian_hessian, laplacian_jvp_loop

SMALL = dict(embedding_dim=16, n_determinants=2, edge_dim=8, nuc_embedding_dim=6)


def _reference_table(n_up, n_down, charges, L=4, d=256, e=32, K=32, dn=32):
    """The DeepErwin parameter tree written out from the reference modules, independently of deepqmc_b200.params:
    ExponentialEnvelopes(per_shell=false, spin_restricted=false, per_orbital_exponent) -> pi/zetas_{up,down}[K N, M]
    (wf/env.py:26-55); NucleiEmbedding(subnet_type='embed', atom_type_embedding) -> hk.Embed 'embed'[n_types, 32]
    (gnn/electron_gnn.py:503-514); per layer ConvolutionElectronUpdateFeature edge_types [ee, ne], w_for_ne false ->
    w_same / w_anti ([|d|] -> e), h_same / h_anti (x -> e), h_ne (32 -> width of the ne edge stream) (update_features.py:
    199-211); g (concatenate; 3 x_dim + e + ne width -> d); u<type> for ne / same / anti on all but the last layer
    (electron_gnn.py:117-128); Backflow MLP(['log', 1], bias false) -> one 'linear_0' without bias (wf/omni.py:43-88)."""
    N, M = n_up + n_down, len(charges)
    root = 'neural_network_wave_function/~/'
    gnn = root + 'omni_net/~/electron_gnn/~/'
    t = {}
    for nm in ('pi_up', 'pi_down', 'zetas_up', 'zetas_down'):
        t[root + 'exponential_envelopes:' + nm] = (K * N, M)
    t[gnn + 'nuclei_embedding/~/embed:embeddings'] = (len(set(charges)), dn)
    x_dim, ee_in, ne_in = 4 * M, 1, 4
    for l in range(L):
        layer = gnn + ('electron_gnn_layer' if l == 0 else f'electron_gnn_layer_{l}') + '/~/'
        conv = layer + 'convolution_electron_update_feature/~single_edge_type_update/'
        for typ in ('same', 'anti'):
            t[conv + f'w_{typ}/linear_0:w'], t[conv + f'w_{typ}/linear_0:b'] = (ee_in, e), (e,)
            t[conv + f'h_{typ}/linear_0:w'], t[conv + f'h_{typ}/linear_0:b'] = (x_dim, e), (e,)
        t[conv + 'h_ne/linear_0:w'], t[conv + 'h_ne/linear_0:b'] = (dn, ne_in), (ne_in,)
        t[layer + 'g/linear_0:w'], t[layer + 'g/linear_0:b'] = (3 * x_dim + e + ne_in, d), (d,)
        if l < L - 1:
            for typ, w_in in (('ne', ne_in), ('same', ee_in), ('anti', ee_in)):
                t[layer + f'u{typ}/linear_0:w'], t[layer + f'u{typ}/linear_0:b'] = (w_in, e), (e,)
            ee_in = ne_in = e
        x_dim = d
    t[root + 'omni_net/~/Backflow/~/mlp/linear_0:w'] = (d, K * N)
    t[root + 'omni_net/~/Backflow_1/~/mlp/linear_0:w'] = (d, K * N)
    return t


@pytest.mark.parametrize('mol', ['LiH', 'N2'])
def test_parameter_table_matches_reference_modules(mol):
    m = Molecule.from_name(mol)
    h = MolecularHamiltonian(mol=m)
    spec = deeperwin_spec(h)
    want = _reference_table(h.n_up, h.n_down, [float(z) for z in m.charges])
    assert PN.param_shapes(spec) == want
    p = PN.init_params(spec, 0)
    assert {k: v.shape for k, v in p.items()} == want
    # init 'deeperwin' (hkext.py:66-80): zero biases, fan_avg uniform weights; envelopes to ones
    assert all(not np.any(v) for k, v in p.items() if k.endswith(':b'))
    w = p[PN.layer_prefix(1) + 'g/linear_0:w']
    assert np.abs(w).max() <= np.sqrt(3 / ((w.shape[0] + w.shape[1]) / 2))
    assert all(np.all(v == 1) for k, v in p.items() if k.startswith(PN.ENV))


def test_edge_builder_with_self_interaction_matches_golden(goldens):
    # reference: tests/test_gnn.py:7-32, MolecularGraphEdgeBuilder without the diagonal filter
    nodes = torch.tensor([[0.0, 0.0, 0.0], [0.0, 0.0, 2.0], [0.0, 0.0, 6.0]], dtype=torch.float64)
    full = DO.graph_edges(nodes, nodes)
    np.testing.assert_allclose(full.numpy(), np.asarray(goldens['graph_edge_builder_mask_self_False']['graph_edges']))


def _setup(mol, seed=0, **kw):
    m = Molecule.from_name(mol)
    h = MolecularHamiltonian(mol=m)
    spec = deeperwin_spec(h, **kw)
    rng = np.random.default_rng(seed + 11)
    p = {k: v + 0.3 * rng.standard_normal(v.shape) for k, v in PN.init_params(spec, seed).items()}  # nothing at its init value
    r = torch.as_tensor(m.coords[rng.integers(0, len(m.coords), size=spec.n_elec)] + rng.normal(size=(spec.n_elec, 3)))
    return m, spec, owf.to_torch(p), p, r, torch.as_tensor(m.coords)


def test_oracle_antisymmetry_and_nuclear_swap():
    m, spec, pt, _, r, R = _setup('N2', **SMALL)
    s0, l0 = DO.log_psi(spec, pt, r, R)
    for i, j in ((0, 1), (spec.n_up, spec.n_up + 2)):  # same-spin swaps
        rs = r.clone()
        rs[[i, j]] = rs[[j, i]]
        s1, l1 = DO.log_psi(spec, pt, rs, R)
        assert s1 == -s0 and abs(l1 - l0) < 1e-11
    # the two N nuclei exchanged: the raw features [|r - R_I|, r - R_I] are laid out nucleus by nucleus and the envelopes
    # are per nucleus, so the parameters that read them follow the permutation; the ne convolution (a sum over nuclei
    # with h_ne of the atom type) and everything else is invariant
    M = spec.n_nuc
    cols = torch.arange(4 * M).reshape(M, 4).flip(0).reshape(-1)
    ps = dict(pt)
    for t in ('same', 'anti'):
        k = ON.conv_prefix(0) + f'h_{t}/linear_0:w'
        ps[k] = pt[k][cols]
    k = ON.layer_prefix(0) + 'g/linear_0:w'
    ps[k] = pt[k][torch.cat([cols, cols + 4 * M, cols + 8 * M, torch.arange(12 * M, pt[k].shape[0])])]
    for nm in ('pi_up', 'pi_down', 'zetas_up', 'zetas_down'):
        ps[f'{ON.ENV}:{nm}'] = pt[f'{ON.ENV}:{nm}'].flip(1)
    s2, l2 = DO.log_psi(spec, ps, r, R.flip(0))
    assert s2 == s0 and abs(l2 - l0) < 1e-11
    assert abs(DO.log_psi(spec, pt, r, R.flip(0))[1] - l0) > 1e-6  # without the parameter permutation it differs


def test_oracle_laplacian_hessian_equals_jvp_loop():
    m, spec, pt, _, r, R = _setup('LiH', **SMALL)
    f = lambda x: DO.log_psi(spec, pt, x.reshape(-1, 3), R)[1]
    (la, ga), (lb, gb) = laplacian_hessian(f, r.reshape(-1)), laplacian_jvp_loop(f, r.reshape(-1))
    assert abs(la - lb) <= 1e-10 * max(1, abs(la)) and torch.allclose(ga, gb, rtol=1e-12, atol=1e-12)


def test_upload_softplus_exponents_and_hne_tables():
    """The engine receives softplus(zeta) (wf/env.py:62-66): the oracle in the reference's form equals the |zeta| form on the
    uploaded exponents, and d/dzeta of log|psi| is the uploaded exponent's gradient times sigmoid(zeta).  The h_ne tables
    are h_ne of the nuclear embedding rows of each nucleus' atom type."""
    m, spec, pt, p, r, R = _setup('LiH', **SMALL)
    packed = _pack_haiku_params(spec, p)
    for s, t in (('up', 'up'), ('down', 'dn')):
        z = p[f'{PN.ENV}:zetas_{s}']
        np.testing.assert_allclose(packed[f'env.zeta_{t}'], np.log1p(np.exp(z)), rtol=1e-14)
    zk = [f'{ON.ENV}:zetas_{s}' for s in ('up', 'down')]
    zeta = {k: pt[k].clone().requires_grad_() for k in zk}
    _, l_ref = DO.log_psi(spec, dict(pt, **zeta), r, R)
    g_ref = torch.autograd.grad(l_ref, [zeta[k] for k in zk])
    up = {k: torch.nn.functional.softplus(pt[k]).detach().requires_grad_() for k in zk}
    x = DO.deeperwin_embeddings(spec, pt, r, R)
    A = owf.orbitals(spec, dict(pt, **up), x, r, R)
    sg, ld = torch.linalg.slogdet(A)
    l_up = torch.log(torch.abs((sg * torch.exp(ld - ld.max().detach())).sum())) + ld.max().detach()
    assert abs(l_up.item() - l_ref.item()) < 1e-12
    g_up = torch.autograd.grad(l_up, [up[k] for k in zk])
    for k, a, b in zip(zk, g_ref, g_up):
        assert torch.allclose(a, b * torch.sigmoid(pt[k]), rtol=1e-10, atol=1e-13)
    xn = p[PN.GNN + 'nuclei_embedding/~/embed:embeddings']
    types = DO.atom_types(spec.charges).numpy()
    assert list(types) == [1, 0]  # Li (z = 3) sorts after H (z = 1)
    for l in range(spec.n_layers):
        c = PN.conv_prefix(l)
        want = np.tanh(xn[types] @ p[c + 'h_ne/linear_0:w'] + p[c + 'h_ne/linear_0:b'])
        np.testing.assert_allclose(packed[f'G{l}.hne'], want, rtol=1e-14)
        assert want.shape[1] == (4 if l == 0 else spec.edge_dim)


MODES = {'forward': MODE_FORWARD, 'local_energy': MODE_LOCAL_ENERGY, 'vjp': MODE_VJP, 'mcmc': MODE_MCMC, 'langevin': MODE_LANGEVIN}


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('mol,ecp', [('LiH', None), ('LiH', 'ccECP'), ('N2', None)])
def test_carved_never_exceeds_planned(built_lib, mol, ecp, dtype):
    h = MolecularHamiltonian(mol=Molecule.from_name(mol), ecp_type=ecp)
    eng = Engine(deeperwin_spec(h), h, dtype=dtype, plan_only=True, gemm_backend=1 if dtype == 'float32' else 0)
    for mname, mode in MODES.items():
        for B in (1, 257, 4096):
            planned, carved = eng.debug_plan(B, mode)
            assert planned == eng.workspace_bytes(B, mode)
            assert 0 < carved <= planned, (mname, B, dtype, planned, carved)
            floor = eng.workspace_bytes_min(B, mode)
            assert floor <= planned
            for cap in {max(floor, planned // 3), max(floor, planned // 50), floor}:
                _, c2 = eng.debug_plan(B, mode, cap)
                assert 0 < c2 <= cap, (mname, B, dtype, cap, c2)
    eng.close()
