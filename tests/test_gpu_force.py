"""GPU: position gradients (dqmc_wf_grad_positions), closed-form force terms (dqmc_force_terms) and the force estimators of
deepqmc_b200/force.py against the fp64 oracle (oracle/force.py, torch autograd of oracle/wf.py).

Bounds: fp64 1e-9 max(1, |grad|_inf); fp32 2e-3 max(1e-3, |grad|_inf), the bound of the fp32 parameter-gradient test.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from deepqmc_b200 import force as FO
from deepqmc_b200 import params as PN
from deepqmc_b200.ansatz import B200Ansatz
from deepqmc_b200.engine import MODE_GRAD_POS
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from deepqmc_b200.types import PhysicalConfiguration
from oracle import force as OF
from oracle import wf as W
from oracle.hamil import OracleHamiltonian
from spin_fixture import walkers

DEV = 'cuda:0'
SMALL = dict(embedding_dim=32, n_layers=2, n_heads=4, n_determinants=4)
NUC_CUSP = dict(cusp_nuclei='psiformer', cusp_nuclei_trainable=False, cusp_nuclei_alpha=1.3)
HYPER = {
    'psiformer': SMALL,
    'psiformer_nuc': dict(SMALL, **NUC_CUSP),
    'ferminet': dict(embedding_dim=32, n_layers=2, n_determinants=4, edge_dim=8),
    'ferminet_nuc': dict(embedding_dim=32, n_layers=3, n_determinants=2, edge_dim=8, cusp='psiformer', **NUC_CUSP),
    'transpsiformer': SMALL,
    'paulinet': {},
    'paulinet_default': {},
}
TOL = {'float64': 1e-9, 'float32': 2e-3}


def _molecule(name):
    if name == 'M7':  # 7 electrons, odd spin
        return Molecule(coords=[[0.0, 0.0, 0.0], [2.5, 0.3, 0.0]], charges=[4, 3], charge=0, spin=1)
    if name == 'C5':  # 30 electrons, all-electron
        return Molecule(coords=[[2.4 * i, 0.3 * (i % 2), 0.0] for i in range(5)], charges=[6] * 5, charge=0, spin=0)
    return Molecule.from_name(name)


def _setup(mol, kind, dtype, B, seed=0, ecp=None):
    h = MolecularHamiltonian(mol=_molecule(mol), ecp_type=ecp)
    a = B200Ansatz(h, kind.replace('_nuc', ''), dtype=dtype, **HYPER[kind])
    a.gemm_backend = 1 if dtype == 'float32' and a.spec.embedding_dim % 32 == 0 else 0  # the tensor-core backend where it serves
    params = PN.perturb_params(a.init(seed))
    r = torch.as_tensor(walkers(h, B, seed=seed + 1), device=DEV)
    R = torch.as_tensor(h.mol.coords, device=DEV)
    return h, a, params, r, R


def _log_psi(a, params):
    pt = W.to_torch(params)
    return lambda x, y: W.log_psi(a.spec, pt, x, y)[1]


def _close(got, ref, dtype, floor=0.0):
    """|got - ref|_inf within the bound of the module docstring, or within 1.5x ``floor``: the fp32 error of the engine's
    forward-Laplacian grad_r on the same walker.  A walker close to a node of psi (|grad| in the thousands) loses relative
    accuracy in fp32 on every path; there the reverse pass must be as accurate as the forward-Laplacian pass."""
    scale = max(1e-3 if dtype == 'float32' else 1.0, float(ref.abs().max()))
    err = float((got.cpu().double() - ref).abs().max())
    assert err <= max(TOL[dtype] * scale, 1.5 * floor), (err, scale, floor)


CASES = [('psiformer', 'LiH'), ('psiformer', 'N2'), ('psiformer', 'M7'), ('psiformer', 'C5'), ('psiformer_nuc', 'LiH'),
         ('ferminet', 'LiH'), ('ferminet', 'N2'), ('ferminet', 'M7'), ('ferminet', 'C5'), ('ferminet_nuc', 'N2'),
         ('transpsiformer', 'LiH'), ('transpsiformer', 'N2'), ('transpsiformer', 'M7'), ('transpsiformer', 'C5')]


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('kind,mol', CASES)
def test_grad_positions_match_oracle(kind, mol, dtype):
    h, a, params, r, R = _setup(mol, kind, dtype, B=2)
    eng = a.engine_for(h, params)
    trans = kind == 'transpsiformer'
    sign, log, gr, gR = eng.grad_positions(r.to(eng.dtype), R.to(eng.dtype), want_R=not trans)
    fl = eng.local_energy(r.to(eng.dtype), R.to(eng.dtype), want_grad=True)[4].reshape(gr.shape) if dtype == 'float32' else None
    lp = _log_psi(a, params)
    Rc = R.cpu().double()
    for b in range(r.shape[0]):
        rb = r[b].cpu().double()
        assert abs(log[b].item() - lp(rb, Rc).item()) <= TOL[dtype] * max(1, abs(log[b].item())) * 10
        ref_r = OF.grad_r(lp, rb, Rc)
        floor = 0.0 if fl is None else float((fl[b].cpu().double() - ref_r).abs().max())
        _close(gr[b], ref_r, dtype, floor)
        if not trans:
            _close(gR[b], OF.grad_R(lp, rb, Rc), dtype, floor)
    if trans:
        with pytest.raises(RuntimeError, match='nuclear stream'):
            eng.grad_positions(r.to(eng.dtype), R.to(eng.dtype), want_R=True)


@pytest.mark.parametrize('kind', ['psiformer_nuc', 'ferminet_nuc', 'transpsiformer'])
def test_reverse_and_forward_laplacian_gradients_agree(kind):
    """The reverse grad_r and dqmc_local_energy's forward-Laplacian out_grad agree; sum_m grad_R + sum_i grad_r = 0."""
    h, a, params, r, R = _setup('N2', kind, 'float64', B=5)
    eng = a.engine_for(h, params)
    trans = kind == 'transpsiformer'
    _, _, gr, gR = eng.grad_positions(r, R, want_R=not trans)
    g2 = eng.local_energy(r, R, want_grad=True)[4].reshape(gr.shape)
    assert float((gr - g2).abs().max()) <= 1e-10 * max(1.0, float(g2.abs().max()))
    if not trans:
        tot = gr.sum(1) + gR.sum(1)
        assert float(tot.abs().max()) <= 1e-10 * max(1.0, float(gr.abs().max()))


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('kind', ['psiformer', 'ferminet', 'transpsiformer', 'paulinet', 'paulinet_default'])
def test_force_terms_match_oracle(kind, dtype):
    h, a, params, r, R = _setup('LiH', kind, dtype, B=3)
    eng = a.engine_for(h, params)
    g = torch.randn(r.shape, generator=torch.Generator().manual_seed(1), dtype=torch.float64).to(DEV)
    bare, zvq, Q = eng.force_terms(r.to(eng.dtype), R.to(eng.dtype), grad_r=g.to(eng.dtype))
    Z = h.mol.charges
    Rc = R.cpu().double()
    for b in range(r.shape[0]):
        rb = r[b].cpu().double()
        _close(bare[b], OF.force_bare(rb, Rc, Z), dtype)
        _close(zvq[b], OF.force_ac_zvq(rb, Rc, Z, g[b].cpu()), dtype)
        _close(Q[b], OF.Q(rb, Rc, Z), dtype)


def _rel(got, ref, tol=1e-9):
    ref = ref.double()
    err = float((got.cpu().double() - ref).abs().max())
    assert err <= tol * max(1.0, float(ref.abs().max())), err


@pytest.mark.parametrize('kind', ['psiformer', 'ferminet', 'paulinet'])
def test_estimators_match_oracle(kind):
    """Every built estimator through the deepqmc_b200.force mirrors against oracle/force.py (fp64)."""
    h, a, params, r, R = _setup('LiH', kind, 'float64', B=3)
    pc = PhysicalConfiguration(R, r, torch.zeros(3, device=DEV))
    lp = _log_psi(a, params)
    Z, Rc = h.mol.charges, R.cpu().double()
    e_loc = h.local_energy(a.apply)(None, params, pc)[0]
    energy = float(e_loc.mean())
    bare = FO.evaluate_hf_force_bare(h, a.apply)(0, params, pc)
    zvq = FO.evaluate_hf_force_ac_zvq(h, a.apply)(params, pc)
    zvzbq = FO.evaluate_hf_force_ac_zvzbq(h, a.apply)(params, pc, e_loc, energy)
    anti_bare = FO.antithetic_wrapper(FO.evaluate_hf_force_bare(h, a.apply), a.apply, 0.8)(0, params, pc)
    anti_zvq = FO.antithetic_wrapper(lambda rng, p, c: FO.evaluate_hf_force_ac_zvq(h, a.apply)(p, c), a.apply, 0.8)(0, params, pc)
    zb_ok = kind != 'paulinet'
    if zb_ok:
        zb = FO.evaluate_hf_force_ac_zb(h, a.apply)(0, params, pc, e_loc, energy)
        zvqzb = FO.evaluate_hf_force_ac_zvqzb(h, a.apply)(params, pc, e_loc, energy)
    else:
        with pytest.raises(ValueError, match='paulinet'):
            FO.evaluate_hf_force_ac_zb(h, a.apply)(0, params, pc, e_loc, energy)
    for b in range(3):
        rb, el = r[b].cpu().double(), float(e_loc[b])
        g_r = OF.grad_r(lp, rb, Rc)
        _rel(bare[b], OF.force_bare(rb, Rc, Z))
        _rel(zvq[b], OF.force_ac_zvq(rb, Rc, Z, g_r))
        _rel(zvzbq[b], OF.force_ac_zvzbq(rb, Rc, Z, g_r, el, energy))
        _rel(anti_bare[b], OF.antithetic(lambda x, y: OF.force_bare(x, y, Z), lp, rb, Rc, 0.8))
        _rel(anti_zvq[b], OF.antithetic(lambda x, y: OF.force_ac_zvq(x, y, Z, OF.grad_r(lp, x, y)), lp, rb, Rc, 0.8))
        if zb_ok:
            g_R = OF.grad_R(lp, rb, Rc)
            _rel(zb[b], OF.force_ac_zb(rb, Rc, Z, g_R, el, energy))
            _rel(zvqzb[b], OF.force_ac_zvqzb(rb, Rc, Z, g_r, g_R, el, energy))


@pytest.mark.parametrize('ecp', [None, 'ccECP'])
def test_finite_difference_estimator_matches_oracle(ecp):
    h, a, params, r, R = _setup('LiH', 'psiformer', 'float64', B=2, ecp=ecp)
    pc = PhysicalConfiguration(R, r, torch.zeros(2, device=DEV))
    N = h.n_up + h.n_down
    n_nl = 0 if h.nl_params is None else len(h.pot.nuc_with_nl_pot)
    tw = torch.as_tensor(np.random.default_rng(5).uniform(0, np.pi / 5, size=(2, n_nl, N)), device=DEV) if n_nl else None
    e_loc = h.local_energy(a.apply)(None, params, pc, ecp_twist=tw)[0]
    step = 1e-3
    got = FO.evaluate_finite_difference_force(h, a.apply, step)(0, params, pc, e_loc, None, ecp_twist=tw)
    oh = OracleHamiltonian(h.mol, ecp_type=ecp)
    pt = W.to_torch(params)
    Rc = R.cpu().double()
    for b in range(2):
        phi = None if tw is None else tw[b].cpu()
        el = lambda x, y: oh.local_energy(lambda z: W.log_psi(a.spec, pt, z, y), x, y, phi_random=phi)[0]
        lp = lambda x, y: W.log_psi(a.spec, pt, x, y)[1]
        ref = OF.force_finite_difference(el, lp, r[b].cpu().double(), Rc, step, float(e_loc[b]))
        # E' - E_loc is O(h): a relative bound on the difference quotient
        assert float((got[b].cpu() - ref).abs().max()) <= 1e-7 / step * max(1.0, float(e_loc.abs().max())), (got[b], ref)


@pytest.mark.parametrize('kind', ['psiformer', 'ferminet'])
@pytest.mark.parametrize('dtype', ['float64', 'float32'])
def test_chunking_repeat_nan_and_batched_R(kind, dtype):
    """A one-walker workspace and DQMC_NSMS=2 give the bitwise outputs of the full plan; repeated calls are bitwise
    identical; a NaN walker leaves the others untouched; R_batched with two geometries equals two unbatched calls;
    n_walkers = 0 is a no-op."""
    h, a, params, r, R = _setup('N2', kind, dtype, B=6)
    eng = a.engine_for(h, params)
    r, R = r.to(eng.dtype), R.to(eng.dtype)
    ref = eng.grad_positions(r, R)
    again = eng.grad_positions(r, R)
    one = eng.grad_positions(r, R, max_ws_bytes=eng.workspace_bytes_min(6, MODE_GRAD_POS))
    for x, y, z in zip(ref, again, one):
        assert torch.equal(x, y) and torch.equal(x, z)
    rn = r.clone()
    rn[2, 1, 0] = float('nan')
    nan = eng.grad_positions(rn, R)
    keep = [0, 1, 3, 4, 5]
    for x, y in zip(ref, nan):
        assert torch.equal(x[keep], y[keep])
    R2 = torch.stack([R] * 3 + [R + 0.1] * 3)
    bat = eng.grad_positions(r, R2)
    lo, hi = eng.grad_positions(r[:3], R), eng.grad_positions(r[3:], R + 0.1)
    for x, y, z in zip(bat, lo, hi):
        assert torch.equal(x, torch.cat([y, z]))
    empty = eng.grad_positions(r[:0], R)
    assert empty[2].shape == (0, h.n_up + h.n_down, 3)
    mp = pytest.MonkeyPatch()
    mp.setenv('DQMC_NSMS', '2')
    try:
        a2 = B200Ansatz(h, kind, dtype=dtype, gemm_backend=a.gemm_backend, **HYPER[kind])
        e2 = a2.engine_for(h, params)
        for x, y in zip(ref, e2.grad_positions(r, R)):
            assert torch.equal(x, y)
    finally:
        mp.undo()


def test_refusals(tmp_path):
    """Status 2: conv-GNN kinds, the additive backflow branch, ECP and pseudo-Hamiltonian engines in dqmc_force_terms, and
    out_zvq without grad_r."""
    for kind in ('paulinet', 'paulinet_default'):
        h, a, params, r, R = _setup('LiH', kind, 'float64', B=2)
        with pytest.raises(RuntimeError, match=r'\(2\)'):
            a.engine_for(h, params).grad_positions(r, R)
    h = MolecularHamiltonian(mol=Molecule.from_name('LiH'))
    a = B200Ansatz(h, 'psiformer', dtype='float64', backflow_transform='add', **SMALL)
    params = PN.perturb_params(a.init(0))
    r = torch.as_tensor(walkers(h, 2, seed=1), device=DEV)
    R = torch.as_tensor(h.mol.coords, device=DEV)
    with pytest.raises(RuntimeError, match='additive backflow'):
        a.engine_for(h, params).grad_positions(r, R)
    from ph_fixture import write_synthetic_ph

    hh, aa, pp, rr, RR = _setup('LiH', 'psiformer', 'float64', B=2, ecp='ccECP')
    with pytest.raises(RuntimeError, match='all-electron'):
        aa.engine_for(hh, pp).force_terms(rr, RR)
    mol = Molecule(coords=[[0.0, 0.0, 0.0], [2.4, 0.0, 0.0]], charges=[15, 1], charge=0, spin=0)
    hh = MolecularHamiltonian(mol=mol, ecp_type='PH', ph_data_dir=write_synthetic_ph(str(tmp_path)))
    aa = B200Ansatz(hh, 'psiformer', dtype='float64', **SMALL)
    pp = PN.perturb_params(aa.init(0))
    rr = torch.as_tensor(walkers(hh, 2, seed=1), device=DEV)
    with pytest.raises(RuntimeError, match='all-electron'):
        aa.engine_for(hh, pp).force_terms(rr, torch.as_tensor(mol.coords, device=DEV))
    h, a, params, r, R = _setup('LiH', 'psiformer', 'float64', B=2)
    eng = a.engine_for(h, params)
    assert eng.lib.dqmc_force_terms(eng.h, r.data_ptr(), R.data_ptr(), 0, 2, None, None, r.data_ptr(), None,
                                    eng._stream()) == 2
