"""GPU: the Hellmann-Feynman force with effective core potentials (dqmc_ecp_force) and the estimators of deepqmc_b200/force.py
that use it, against the fp64 oracle of tests/ecp_force_oracle.py (torch autograd of oracle/wf.py) with the same injected
quadrature twists; chunking, repeatability, NaN isolation, the cutoff radius and the refusals.

Bounds: fp64 1e-9, fp32 2e-3, relative to max(1e-3, |F|_inf).
"""
import gc
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import ecp_force_oracle as EO
from deepqmc_b200 import force as FO
from deepqmc_b200 import params as PN
from deepqmc_b200.ansatz import B200Ansatz
from deepqmc_b200.engine import MODE_ECP_FORCE
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from deepqmc_b200.types import PhysicalConfiguration
from oracle import force as OF
from oracle import wf as W
from oracle.hamil import OracleHamiltonian
from spin_fixture import walkers

DEV = 'cuda:0'
SMALL = dict(embedding_dim=32, n_layers=2, n_heads=4, n_determinants=4)
HYPER = {'psiformer': SMALL, 'ferminet': dict(embedding_dim=32, n_layers=2, n_determinants=4, edge_dim=8),
         'transpsiformer': SMALL, 'paulinet': {}}
TOL = {'float64': 1e-9, 'float32': 2e-3}


@pytest.fixture(autouse=True, scope='module')
def _return_cached_workspaces():
    """This file's engines size their workspaces at up to 60 % of the free HBM (full-size benzene: 16 GiB).  Once the engines
    are gone, torch's caching allocator would keep those blocks reserved, while engines created later in the same process
    allocate their device buffers with cudaMalloc outside that cache: hand the blocks back to the driver."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _mol(name):
    if name == 'CH4_c_last':  # carbon is nucleus 4: its non-local force must land in row 4 (the reference would write row 0)
        m = Molecule.from_name('CH4')
        return Molecule(coords=np.asarray(m.coords)[[1, 2, 3, 4, 0]].tolist(), charges=[1, 1, 1, 1, 6], charge=0, spin=0)
    return Molecule.from_name(name)


def _setup(name, ecp, kind, dtype, B, seed=0):
    mol = _mol(name)
    h = MolecularHamiltonian(mol=mol, ecp_type=ecp)
    a = B200Ansatz(h, kind, dtype=dtype, **HYPER[kind])
    a.gemm_backend = 1 if dtype == 'float32' and a.spec.embedding_dim % 32 == 0 else 0
    params = PN.perturb_params(a.init(seed))
    r = torch.as_tensor(walkers(h, B, seed=seed + 1), device=DEV)
    R = torch.as_tensor(mol.coords, device=DEV)
    pt = W.to_torch(params)
    return h, OracleHamiltonian(mol, ecp_type=ecp), a, params, r, R, (lambda x, y: W.log_psi(a.spec, pt, x, y))


def _twists(h, B, mode, seed=5):
    J, N = len(h.pot.nuc_with_nl_pot), h.n_up + h.n_down
    g = np.random.default_rng(seed)
    if mode == 'pair':
        return torch.as_tensor(g.uniform(0, math.pi / 5, size=(B, J, N)), device=DEV)
    return torch.as_tensor(g.uniform(0, math.pi / 5, size=(B, 1, 1)), device=DEV).expand(B, J, N).contiguous()


def _close(got, ref, dtype):
    scale = max(1e-3, float(ref.abs().max()))
    err = float((got.cpu().double() - ref).abs().max())
    assert err <= TOL[dtype] * scale, (err, scale)
    return err / scale


# (molecule, ECP): LiH, the carbon atom with two ECP families, C2 with an ECP on both nuclei, CH4 with carbon last
MOLS = [('LiH', 'ccECP'), ('C', 'ccECP'), ('C', 'bfd'), ('C2', 'ccECP'), ('CH4_c_last', 'ccECP')]


@pytest.mark.parametrize('twist', ['pair', 'walker'])
@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('kind', ['psiformer', 'ferminet'])
@pytest.mark.parametrize('name,ecp', MOLS)
def test_ecp_force_matches_oracle(name, ecp, kind, dtype, twist):
    h, oh, a, params, r, R, lp = _setup(name, ecp, kind, dtype, B=2)
    eng = a.engine_for(h, params)
    tw = _twists(h, 2, twist)
    bare, nl = eng.ecp_force(r.to(eng.dtype), R.to(eng.dtype), ecp_twist=tw.to(eng.dtype))
    Rc = R.cpu().double()
    for b in range(2):
        rb = r[b].cpu().double()
        _close(bare[b], EO.force_bare_local(oh, rb, Rc), dtype)
        ref = -EO.grad_nonloc_potential(oh, lp, rb, Rc, tw[b].cpu())
        _close(nl[b], ref, dtype)
        if name == 'CH4_c_last':
            assert float(nl[b, :4].abs().max()) == 0.0 and float(ref[4].abs().max()) > 0


@pytest.mark.parametrize('kind', ['psiformer', 'ferminet'])
@pytest.mark.parametrize('name', ['LiH', 'C2'])
def test_estimators_with_ecp_match_oracle(name, kind):
    """evaluate_hf_force_bare, evaluate_hf_force_ac_zb and antithetic_wrapper(bare) with an ECP (fp64): one twist per walker
    from rng, the mirrored copies from rng + 1."""
    h, oh, a, params, r, R, lp = _setup(name, 'ccECP', kind, 'float64', B=3)
    pc = PhysicalConfiguration(R, r, torch.zeros(3, device=DEV))
    e_loc = torch.tensor([-1.0, -0.5, -2.0], dtype=torch.float64, device=DEV)
    energy = -1.2
    rng = 7
    bare = FO.evaluate_hf_force_bare(h, a.apply)(rng, params, pc)
    zb = FO.evaluate_hf_force_ac_zb(h, a.apply)(rng, params, pc, e_loc, energy)
    anti = FO.antithetic_wrapper(FO.evaluate_hf_force_bare(h, a.apply), a.apply, 0.8)(rng, params, pc)
    N = h.n_up + h.n_down
    tw0, tw1 = FO.ecp_force_twist(h, rng, 3, N), FO.ecp_force_twist(h, rng + 1, 3, N)
    Rc = R.cpu().double()
    lp1 = lambda x, y: lp(x, y)[1]
    for b in range(3):
        rb = r[b].cpu().double()
        ref = EO.force_bare(oh, lp, rb, Rc, tw0[b])
        _close(bare[b], ref, 'float64')
        _close(zb[b], ref - 2 * (float(e_loc[b]) - energy) * OF.grad_R(lp1, rb, Rc), 'float64')
        rm = OF.antithetic_mirror(rb, Rc, 0.8)
        lw = 2 * (lp1(rm, Rc) - lp1(rb, Rc))
        w = torch.softmax(torch.stack([torch.zeros_like(lw), lw]), 0)
        _close(anti[b], w[0] * ref + w[1] * EO.force_bare(oh, lp, rm, Rc, tw1[b]), 'float64')
    with pytest.raises(RuntimeError, match='all-electron'):
        FO.evaluate_hf_force_ac_zvq(h, a.apply)(params, pc)


def test_all_electron_bare_equals_force_terms():
    h, oh, a, params, r, R, lp = _setup('LiH', None, 'psiformer', 'float64', B=4)
    eng = a.engine_for(h, params)
    bare, nl = eng.ecp_force(r, R)
    assert float((bare - eng.force_terms(r, R)[0]).abs().max()) <= 1e-13 * max(1.0, float(bare.abs().max()))
    assert float(nl.abs().max()) == 0.0


def _engine_with_env(h, kind, dtype, params, **env):
    mp = pytest.MonkeyPatch()
    for k, v in env.items():
        mp.setenv(k, v)
    try:
        a2 = B200Ansatz(h, kind, dtype=dtype, **HYPER[kind])
        a2.gemm_backend = 1 if dtype == 'float32' and a2.spec.embedding_dim % 32 == 0 else 0
        return a2.engine_for(h, params)
    finally:
        mp.undo()


def test_cutoff_against_no_cutoff():
    """The force's cutoff radius drops only pairs whose share is below 2^-100: relative 1e-12 against DQMC_ECP_CUTOFF=0, with
    some electrons far from the nuclei (fewer quadrature walkers run)."""
    h, oh, a, params, r, R, lp = _setup('C2', 'ccECP', 'psiformer', 'float64', B=4)
    r = r.clone()
    r[:2, :3] += 6.0  # well outside every radius
    eng = a.engine_for(h, params)
    n0 = eng.lib.dqmc_ecp_forward_count(eng.h)
    bare, nl = eng.ecp_force(r, R, seed=3)
    n_cut = eng.lib.dqmc_ecp_forward_count(eng.h) - n0
    e0 = _engine_with_env(h, 'psiformer', 'float64', params, DQMC_ECP_CUTOFF='0')
    m0 = e0.lib.dqmc_ecp_forward_count(e0.h)
    bare0, nl0 = e0.ecp_force(r, R, seed=3)
    n_all = e0.lib.dqmc_ecp_forward_count(e0.h) - m0
    assert n_all == 4 * 2 * (h.n_up + h.n_down) * 12 and n_cut < n_all
    assert torch.equal(bare, bare0)
    assert float((nl - nl0).abs().max()) <= 1e-12 * max(1.0, float(nl0.abs().max()))


@pytest.mark.parametrize('kind', ['psiformer', 'ferminet'])
@pytest.mark.parametrize('dtype', ['float64', 'float32'])
def test_chunking_repeat_and_nan(kind, dtype):
    """A workspace of the least size (one base walker per group, one virtual walker per reverse chunk) and DQMC_NSMS=2 give the
    bitwise outputs of the full plan; a repeated call is bitwise identical; a NaN walker leaves the others bitwise unchanged."""
    h, oh, a, params, r, R, lp = _setup('C2', 'ccECP', kind, dtype, B=5)
    eng = a.engine_for(h, params)
    r, R = r.to(eng.dtype), R.to(eng.dtype)
    ref = eng.ecp_force(r, R, seed=11)
    again = eng.ecp_force(r, R, seed=11)
    small = eng.ecp_force(r, R, seed=11, max_ws_bytes=eng.workspace_bytes_min(5, MODE_ECP_FORCE))
    for x, y, z in zip(ref, again, small):
        assert torch.equal(x, y) and torch.equal(x, z)
    assert float(ref[1].abs().max()) > 0
    rn = r.clone()
    rn[2, 1, 0] = float('nan')
    nan = eng.ecp_force(rn, R, seed=11)
    keep = [0, 1, 3, 4]
    for x, y in zip(ref, nan):
        assert torch.equal(x[keep], y[keep])
    e2 = _engine_with_env(h, kind, dtype, params, DQMC_NSMS='2')
    for x, y in zip(ref, e2.ecp_force(r, R, seed=11)):
        assert torch.equal(x, y)


def test_benzene_fp32_against_fp64_engine():
    """Full-size benzene ccECP Psiformer, 2 walkers: the fp32 engine (tensor-core backend) against the fp64 engine.  On an H100
    the bare force agrees to 6.7e-7 and the non-local part to 4.9e-3 of max(1e-3, |F|_inf): 720 quadrature ratios per walker,
    each with fp32 log|psi| differences and reverse-pass gradients of the full-size network, are summed.  The non-local bound
    is therefore 1e-2 here, not the 2e-3 of the small networks above."""
    mol = Molecule.from_name('benzene')
    h = MolecularHamiltonian(mol=mol, ecp_type='ccECP')
    a64 = B200Ansatz(h, 'psiformer', dtype='float64')
    params = PN.perturb_params(a64.init(0))
    a32 = B200Ansatz(h, 'psiformer', dtype='float32', gemm_backend=1)
    # both engines see the same fp32-representable walkers, nuclei and twists: the 1 / rho^2 terms of the bare force turn the
    # rounding of an electron close to a nucleus into force differences far above the engine's own fp32 error
    r = torch.as_tensor(walkers(h, 2, seed=1), device=DEV).float().double()
    R = torch.as_tensor(mol.coords, device=DEV).float().double()
    tw = _twists(h, 2, 'pair').float().double()
    b64, n64 = a64.engine_for(h, params).ecp_force(r, R, ecp_twist=tw)
    b32, n32 = a32.engine_for(h, params).ecp_force(r.float(), R.float(), ecp_twist=tw.float())
    rel = lambda x, y: float((x.double() - y).abs().max()) / max(1e-3, float(y.abs().max()))
    print(f'benzene ccECP fp32 vs fp64 engine: bare {rel(b32, b64):.2e}, nl {rel(n32, n64):.2e} (relative to max(1e-3, |F|_inf))')
    _close(b32, b64.cpu(), 'float32')
    assert rel(n32, n64) <= 1e-2


def test_refusals(tmp_path):
    """Status 2 for out_nl on the TransPsiformer and conv-GNN kinds, for R_batched with out_nl, and for pseudo-Hamiltonians;
    out_bare alone works on those kinds and with R_batched."""
    for kind in ('transpsiformer', 'paulinet'):
        h, oh, a, params, r, R, lp = _setup('LiH', 'ccECP', kind, 'float64', B=2)
        eng = a.engine_for(h, params)
        with pytest.raises(RuntimeError, match=r'\(2\)'):
            eng.ecp_force(r, R)
        bare, nl = eng.ecp_force(r, R, want_nl=False)
        assert nl is None
        for b in range(2):
            _close(bare[b], EO.force_bare_local(oh, r[b].cpu().double(), R.cpu().double()), 'float64')
    h, oh, a, params, r, R, lp = _setup('LiH', 'ccECP', 'psiformer', 'float64', B=2)
    eng = a.engine_for(h, params)
    R2 = torch.stack([R, R + 0.1])
    with pytest.raises(RuntimeError, match='per-walker nuclei'):
        eng.ecp_force(r, R2)
    bare2, _ = eng.ecp_force(r, R2, want_nl=False)
    assert torch.equal(bare2[1], eng.ecp_force(r[1:], R + 0.1, want_nl=False)[0][0])
    from ph_fixture import write_synthetic_ph

    mol = Molecule(coords=[[0.0, 0.0, 0.0], [2.4, 0.0, 0.0]], charges=[15, 1], charge=0, spin=0)
    hh = MolecularHamiltonian(mol=mol, ecp_type='PH', ph_data_dir=write_synthetic_ph(str(tmp_path)))
    aa = B200Ansatz(hh, 'psiformer', dtype='float64', **SMALL)
    pp = PN.perturb_params(aa.init(0))
    rr = torch.as_tensor(walkers(hh, 2, seed=1), device=DEV)
    with pytest.raises(RuntimeError, match='pseudo-Hamiltonian'):
        aa.engine_for(hh, pp).ecp_force(rr, torch.as_tensor(mol.coords, device=DEV), want_nl=False)
