"""GPU: the zero-variance term of the AC-ZV / AC-ZVZB force estimators (dqmc_zv_force, -dT/dR at fixed electron positions by
a nuclear-coordinate companion of the forward-Laplacian pass) against the fp64 oracle (tests/zv_force_oracle.py), against central
differences of the engine's own kinetic energy, and through the estimators of deepqmc_b200/force.py.

Bounds: fp64 1e-9 max(1, |f|_inf); fp32 2e-3 max(1e-3, |f|_inf), the bounds of tests/test_gpu_force.py.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from deepqmc_b200 import force as FO
from deepqmc_b200 import params as PN
from deepqmc_b200.ansatz import B200Ansatz
from deepqmc_b200.engine import MODE_ZV_FORCE
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from deepqmc_b200.types import PhysicalConfiguration
from oracle import force as OF
from oracle.hamil import OracleHamiltonian
from spin_fixture import walkers
import zv_force_oracle as ZO
from test_gpu_force import HYPER, SMALL, TOL, _log_psi, _setup

DEV = 'cuda:0'


def _parts(lp, r, R):
    """The two parts of f = 1/2 d_R Lap log|psi| + 1/2 d_R |grad log|psi||^2 by autograd of the oracle, each [M, 3]."""
    R = R.detach().clone().requires_grad_(True)
    x = r.detach().clone().reshape(-1).requires_grad_(True)
    (g,) = torch.autograd.grad(lp(x.reshape(r.shape), R), x, create_graph=True)
    lap = sum(torch.autograd.grad(g[k], x, create_graph=True)[0][k] for k in range(x.numel()))
    return torch.autograd.grad(0.5 * lap, R, retain_graph=True)[0], torch.autograd.grad(0.5 * (g * g).sum(), R)[0]


CASES = [('psiformer', 'LiH'), ('psiformer', 'N2'), ('psiformer', 'M7'), ('psiformer_nuc', 'LiH'), ('psiformer_nuc', 'N2'),
         ('ferminet', 'LiH'), ('ferminet', 'N2'), ('ferminet', 'M7'), ('ferminet_nuc', 'N2')]


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('kind,mol', CASES)
def test_zv_matches_oracle(kind, mol, dtype):
    """out_zv against -dT/dR by autograd of the oracle's kinetic energy; out_grad_R against the reverse pass.

    The bound is relative to the larger of |f|_inf and the two parts of f (1/2 d_R Lap log|psi| and 1/2 d_R |grad log|psi||^2),
    which cancel to f: rounding errors scale with the parts.  On these walkers the parts reach 37x |f| (M7, FermiNet:
    parts of 300 for |f| = 8), and near a node of psi 3e5x (N2, FermiNet: |grad log|psi|| = 2.2e3, parts of 9.2e10)."""
    h, a, params, r, R = _setup(mol, kind, dtype, B=2)
    eng = a.engine_for(h, params)
    rr, RR = r.to(eng.dtype), R.to(eng.dtype)
    zv, gR = eng.zv_force(rr, RR, want_grad_R=True)
    assert zv.shape == (2, h.n_nuc, 3)
    lp = _log_psi(a, params)
    Rc = R.cpu().double()
    for b in range(r.shape[0]):
        rb = r[b].cpu().double()
        p1, p2 = _parts(lp, rb, Rc)
        ref = p1 + p2
        assert float((ref - ZO.kinetic_nuclear_gradient(lp, rb, Rc)).abs().max()) <= 1e-12 * float(p1.abs().max() + 1)
        scale = max(1e-3 if dtype == 'float32' else 1.0, float(ref.abs().max()), float(p1.abs().max()), float(p2.abs().max()))
        err = float((zv[b].cpu().double() - ref).abs().max())
        assert err <= TOL[dtype] * scale, (err, scale)
    if dtype == 'float64':
        ref = eng.grad_positions(rr, RR, want_r=False)[3]
        assert float((gR - ref).abs().max()) <= 1e-10 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize('kind', ['psiformer', 'ferminet'])
def test_zv_central_differences_30_electrons(kind):
    """Oracle-free: -dT/dR against central differences (h = 1e-4, r fixed) of the engine's own fp64 hamil/E_kin on a
    30-electron all-electron system."""
    h, a, params, r, R = _setup('C5', kind, 'float64', B=2)
    eng = a.engine_for(h, params)
    zv, _ = eng.zv_force(r, R)
    step = 1e-4
    fd = torch.empty_like(zv)
    for k in range(R.numel()):
        dR = torch.zeros_like(R).reshape(-1)
        dR[k] = step
        dR = dR.reshape(R.shape)
        tp = eng.local_energy(r, R + dR)[1][1]
        tm = eng.local_energy(r, R - dR)[1][1]
        fd.reshape(2, -1)[:, k] = -(tp - tm) / (2 * step)
    scale = max(1.0, float(zv.abs().max()))
    assert float((zv - fd).abs().max()) <= 1e-6 * scale, (zv, fd)


@pytest.mark.parametrize('kind', ['psiformer', 'ferminet'])
def test_zv_estimators_match_oracle(kind):
    """AC-ZV and AC-ZVZB through the deepqmc_b200.force mirrors against tests/zv_force_oracle.py, whose zero-variance term is the
    reference's formulation (local energy of d psi / dR_k with the walker's exact local energy), fp64."""
    h, a, params, r, R = _setup('LiH', kind, 'float64', B=2)
    pc = PhysicalConfiguration(R, r, torch.zeros(2, device=DEV))
    lp = _log_psi(a, params)
    Z, Rc = h.mol.charges, R.cpu().double()
    e_loc = h.local_energy(a.apply)(None, params, pc)[0]
    energy = float(e_loc.mean())
    zv = FO.evaluate_hf_force_ac_zv(h, a.apply)(0, params, pc)
    zv_el = FO.evaluate_hf_force_ac_zv(h, a.apply)(0, params, pc, e_loc, energy)
    zvzb = FO.evaluate_hf_force_ac_zvzb(h, a.apply)(0, params, pc, e_loc, energy)
    assert torch.equal(zv, zv_el)
    oh = OracleHamiltonian(h.mol)
    for b in range(2):
        rb, el = r[b].cpu().double(), float(e_loc[b])
        f_zv = ZO.zv_term(oh, lp, rb, Rc, el)
        g_R = OF.grad_R(lp, rb, Rc)
        for got, ref in ((zv[b], ZO.force_ac_zv(rb, Rc, Z, f_zv)), (zvzb[b], ZO.force_ac_zvzb(rb, Rc, Z, f_zv, g_R, el, energy))):
            err = float((got.cpu() - ref.detach()).abs().max())
            assert err <= 1e-9 * max(1.0, float(ref.detach().abs().max())), err


@pytest.mark.parametrize('kind', ['psiformer', 'ferminet'])
@pytest.mark.parametrize('dtype', ['float64', 'float32'])
def test_zv_chunking_repeat_nan_and_batched_R(kind, dtype):
    """A one-walker workspace and DQMC_NSMS=2 give the bitwise outputs of the full plan; repeated calls are bitwise
    identical; a NaN walker leaves the others untouched; R_batched with two geometries equals two unbatched calls;
    n_walkers = 0 is a no-op."""
    h, a, params, r, R = _setup('N2', kind, dtype, B=6)
    eng = a.engine_for(h, params)
    r, R = r.to(eng.dtype), R.to(eng.dtype)
    ref = eng.zv_force(r, R, want_grad_R=True)
    again = eng.zv_force(r, R, want_grad_R=True)
    one = eng.zv_force(r, R, want_grad_R=True, max_ws_bytes=eng.workspace_bytes_min(6, MODE_ZV_FORCE))
    for x, y, z in zip(ref, again, one):
        assert torch.equal(x, y) and torch.equal(x, z)
    assert torch.isfinite(ref[0]).all()
    rn = r.clone()
    rn[2, 1, 0] = float('nan')
    nan = eng.zv_force(rn, R, want_grad_R=True)
    keep = [0, 1, 3, 4, 5]
    for x, y in zip(ref, nan):
        assert torch.equal(x[keep], y[keep])
    R2 = torch.stack([R] * 3 + [R + 0.1] * 3)
    bat = eng.zv_force(r, R2, want_grad_R=True)
    lo, hi = eng.zv_force(r[:3], R, want_grad_R=True), eng.zv_force(r[3:], R + 0.1, want_grad_R=True)
    for x, y, z in zip(bat, lo, hi):
        assert torch.equal(x, torch.cat([y, z]))
    empty = eng.zv_force(r[:0], R)
    assert empty[0].shape == (0, h.n_nuc, 3)
    mp = pytest.MonkeyPatch()
    mp.setenv('DQMC_NSMS', '2')
    try:
        a2 = B200Ansatz(h, kind, dtype=dtype, gemm_backend=a.gemm_backend, **HYPER[kind])
        e2 = a2.engine_for(h, params)
        for x, y in zip(ref, e2.zv_force(r, R, want_grad_R=True)):
            assert torch.equal(x, y)
    finally:
        mp.undo()


def test_zv_refusals(tmp_path):
    """Status 2 with a message for the TransPsiformer, the conv-GNN kinds, the additive backflow branch, ECP engines and
    pseudo-Hamiltonians; the estimators raise a ValueError that names the kind or the ECP."""
    for kind, what in (('transpsiformer', 'nuclear stream'), ('paulinet', 'conv-GNN'), ('paulinet_default', 'conv-GNN')):
        h, a, params, r, R = _setup('LiH', kind, 'float64', B=2)
        with pytest.raises(RuntimeError, match=what):
            a.engine_for(h, params).zv_force(r, R)
        pc = PhysicalConfiguration(R, r, torch.zeros(2, device=DEV))
        with pytest.raises(ValueError, match=a.spec.kind):
            FO.evaluate_hf_force_ac_zv(h, a.apply)(0, params, pc)
    h = MolecularHamiltonian(mol=Molecule.from_name('LiH'))
    a = B200Ansatz(h, 'psiformer', dtype='float64', backflow_transform='add', **SMALL)
    params = PN.perturb_params(a.init(0))
    r = torch.as_tensor(walkers(h, 2, seed=1), device=DEV)
    R = torch.as_tensor(h.mol.coords, device=DEV)
    with pytest.raises(RuntimeError, match='additive backflow'):
        a.engine_for(h, params).zv_force(r, R)
    hh, aa, pp, rr, RR = _setup('LiH', 'psiformer', 'float64', B=2, ecp='ccECP')
    with pytest.raises(RuntimeError, match='all-electron'):
        aa.engine_for(hh, pp).zv_force(rr, RR)
    pc = PhysicalConfiguration(RR, rr, torch.zeros(2, device=DEV))
    with pytest.raises(ValueError, match='ccECP'):
        FO.evaluate_hf_force_ac_zvzb(hh, aa.apply)(0, pp, pc, torch.zeros(2, device=DEV), 0.0)
    from ph_fixture import write_synthetic_ph

    mol = Molecule(coords=[[0.0, 0.0, 0.0], [2.4, 0.0, 0.0]], charges=[15, 1], charge=0, spin=0)
    hh = MolecularHamiltonian(mol=mol, ecp_type='PH', ph_data_dir=write_synthetic_ph(str(tmp_path)))
    aa = B200Ansatz(hh, 'psiformer', dtype='float64', **SMALL)
    pp = PN.perturb_params(aa.init(0))
    rr = torch.as_tensor(walkers(hh, 2, seed=1), device=DEV)
    with pytest.raises(RuntimeError, match='all-electron'):
        aa.engine_for(hh, pp).zv_force(rr, torch.as_tensor(mol.coords, device=DEV))
