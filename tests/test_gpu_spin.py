"""GPU: the spin pass (dqmc_spin, Engine.spin, deepqmc_b200/spin.py) against the fp64 oracle (oracle/spin.py) and against
dqmc_wf_forward on explicitly swapped walkers.

Bounds: |ds2| <= 1e-9 max(1, sum|rho|) in fp64 and 2e-4 max(1, sum|rho|) in fp32 (the reference's fp32 tolerance,
tests/test_hamil.py:37-40), sum|rho| from the oracle: s2 is a sum of P ratios, each as accurate as a forward.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from deepqmc_b200 import params as PN
from deepqmc_b200 import spin as SP
from deepqmc_b200.ansatz import B200Ansatz
from deepqmc_b200.engine import MODE_FORWARD, MODE_SPIN
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from deepqmc_b200.types import PhysicalConfiguration
from oracle import spin as OS
from oracle import wf as W
from spin_fixture import known_answer_params, walkers

DEV = 'cuda:0'
SMALL = dict(embedding_dim=32, n_layers=2, n_heads=4, n_determinants=4)
KINDS = {
    'psiformer': SMALL,
    'ferminet': dict(embedding_dim=32, n_layers=2, n_determinants=4, edge_dim=8),
    'transpsiformer': SMALL,
    'paulinet': {},
    'paulinet_default': {},
}
TOL = {'float64': 1e-9, 'float32': 2e-4}
# one ratio is as accurate as two forwards: fp32 bound of the least accurate kind's forward (the FermiNet's, 1e-3 in
# test_gpu_parity.py::test_ferminet_n2_full_fp32_tensor_core_vs_fp64), relative to max(1, |rho|)
RATIO_TOL = {'float64': 1e-9, 'float32': 2e-3}


def _hamil(mol, ecp=None):
    return MolecularHamiltonian(mol=mol if isinstance(mol, Molecule) else Molecule.from_name(mol), ecp_type=ecp)


def _setup(mol, kind, dtype, B, seed=0, **hyper):
    h = _hamil(mol)
    a = B200Ansatz(h, kind, dtype=dtype, **hyper)
    params = PN.perturb_params(a.init(seed))
    r = torch.as_tensor(walkers(h, B, seed=seed + 1), device=DEV)
    R = torch.as_tensor(h.mol.coords, device=DEV)
    return h, a, params, r, R


def _oracle_wf(a, params, R):
    return OS.wave_function(a.spec, W.to_torch(params), R.cpu().double())


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('mol', ['LiH', 'C', 'B'])
@pytest.mark.parametrize('kind', sorted(KINDS))
def test_spin_matches_oracle(kind, mol, dtype):
    """Exact estimator and the raising estimator for every down electron against the fp64 oracle; C and B have n_up != n_down."""
    h, a, params, r, R = _setup(mol, kind, dtype, B=2, **KINDS[kind])
    eng = a.engine_for(h, params)
    wf = _oracle_wf(a, params, R)
    s2, rho = eng.spin(r.to(eng.dtype), R, want_ratios=True)
    N = h.n_up + h.n_down
    for b in range(r.shape[0]):
        rb = r[b].cpu().double()
        ref_rho = OS.spin_ratios(wf, rb, h.n_up, h.n_down)  # [n_up, n_down]
        ref = float(OS.evaluate_spin(wf, rb, h.n_up, h.n_down))
        scale = max(1.0, float(ref_rho.abs().sum()))
        assert abs(s2[b].item() - ref) <= TOL[dtype] * scale, (b, s2[b].item(), ref)
        assert torch.allclose(rho[b].cpu().double(), ref_rho.reshape(-1), rtol=RATIO_TOL[dtype], atol=RATIO_TOL[dtype])
    for beta in range(h.n_up, N):
        c, _ = eng.spin(r.to(eng.dtype), R, down_idx=beta)
        for b in range(r.shape[0]):
            rb = r[b].cpu().double()
            ref_rho = OS.ratios(wf, rb, h.n_up, beta)
            ref = float(OS.spin_raising(wf, rb, h.n_up, beta))
            assert abs(c[b].item() - ref) <= TOL[dtype] * max(1.0, float(ref_rho.abs().sum())), (beta, b, c[b].item(), ref)


def _molecule(n_elec):
    n_nuc = -(-n_elec // 6)
    charges = [n_elec // n_nuc + (i < n_elec % n_nuc) for i in range(n_nuc)]
    coords = [[2.5 * i, 0.3 * (i % 2), 0.0] for i in range(n_nuc)]
    return Molecule(coords=coords, charges=charges, charge=0, spin=n_elec % 2)


def _swapped_walkers_forward(eng, h, r, R, down_idx):
    """dqmc_wf_forward on walkers built in torch with the pair p swapped -> sign, log [B, P]."""
    n_up, n_down = h.n_up, h.n_down
    pairs = ([(a, n_up + j) for a in range(n_up) for j in range(n_down)] if down_idx < 0
             else [(a, down_idx) for a in range(n_up)])
    sw = torch.stack([SP.swap_electrons(r, a, b) for a, b in pairs], 1).reshape(-1, *r.shape[1:])  # [B P, N, 3]
    s, l = eng.wf_forward(sw, R)
    return s.reshape(r.shape[0], -1), l.reshape(r.shape[0], -1)


def _swapped_forward(eng, h, r, R, down_idx):
    """ratio[b, p] from dqmc_wf_forward on walkers built in torch with the pair p swapped."""
    s0, l0 = eng.wf_forward(r, R)
    s, l = _swapped_walkers_forward(eng, h, r, R, down_idx)
    return s.double() * s0.double()[:, None] * torch.exp(l.double() - l0.double()[:, None])


@pytest.mark.parametrize('nsms', [None, 2])
@pytest.mark.parametrize('mol', ['LiH', 'M7', 'N2', 'benzene'])
def test_ratios_match_swapped_forwards(mol, nsms):
    """out_ratio of the production fp32 engine (whole-trunk kernel; slot sizes 4, 8, 16 and 32: LiH, a 7-electron
    molecule, N2 and benzene with its 30 ccECP valence electrons, 4 walkers per 128-row tile and slater_fwd2_kernel<30>)
    against dqmc_wf_forward on explicitly swapped walkers, per pair, both measured against the fp64 engine: a batch that is
    not a multiple of the walkers per tile, with DQMC_NSMS=2, and with a workspace that splits one walker's pairs across
    forward chunks.  The launch count shows that the compact forwards ran: the base walkers' envelope and embedding tables
    (two launches) and no embedding launch per forward chunk.  The compact forwards (two rows formed in the trunk's tile
    load from the base walkers' embedding table as emb(r, +-1) = emb(r, -+1) +- 2 w_spin, two envelope rows afresh in
    slater_fwd2_kernel) differ from the plain forward of the materialised walkers by the rounding of those rows, which
    unequilibrated walkers near a node amplify; they must be as accurate as the plain forward: the largest and the mean
    error against fp64 within 1.5x / 1.2x of the plain forward's."""
    h = _hamil(_molecule(7) if mol == 'M7' else mol, 'ccECP' if mol == 'benzene' else None)
    assert h.n_up + h.n_down <= 32  # the whole-trunk kernel and slater_fwd2_kernel serve at most 32 electrons
    mp = pytest.MonkeyPatch()
    if nsms:
        mp.setenv('DQMC_NSMS', str(nsms))
    try:
        a = B200Ansatz(h, 'psiformer', dtype='float32', gemm_backend=1)
        params = PN.perturb_params(a.init(0))
        eng = a.engine_for(h, params)
    finally:
        mp.undo()
    e64 = B200Ansatz(h, 'psiformer', dtype='float64').engine_for(h, params)
    B = 37 if mol != 'benzene' else 5
    r = torch.as_tensor(walkers(h, B, seed=3), device=DEV, dtype=torch.float32)
    R = torch.as_tensor(h.mol.coords, device=DEV, dtype=torch.float32)
    P = h.n_up * h.n_down
    # one walker's pairs in chunks of about a third: the spin prefix of one walker + a forward chunk of P // 3 + 1 walkers
    small = eng.workspace_bytes_min(B, MODE_SPIN) - eng.workspace_bytes(1, MODE_FORWARD) + eng.workspace_bytes(P // 3 + 1,
                                                                                                              MODE_FORWARD)
    sg, lg = eng.wf_forward(r, R)
    for down_idx in (-1, h.n_up + h.n_down - 1):
        ref = _swapped_forward(eng, h, r, R, down_idx)
        _, r64 = e64.spin(r.double(), R.double(), down_idx=down_idx, want_ratios=True)
        sc = r64.abs().clamp(min=1.0)
        err_copy = (ref - r64).abs() / sc
        # launches of one plain forward over all swapped walkers (one chunk) vs the spin pass given sign / log: pair kernel +
        # envelope table + embedding table + that forward without its embedding launch + accumulate
        n0 = eng.launch_count
        _swapped_walkers_forward(eng, h, r, R, down_idx)
        n_fwd = eng.launch_count - n0
        n0 = eng.launch_count
        s2, rho = eng.spin(r, R, sign=sg, log=lg, down_idx=down_idx, want_ratios=True)
        assert eng.launch_count - n0 == n_fwd + 3, (eng.launch_count - n0, n_fwd)
        err = (rho.double() - r64).abs() / sc
        assert float(err.max()) <= 1.5 * float(err_copy.max()), (down_idx, float(err.max()), float(err_copy.max()))
        assert float(err.mean()) <= 1.2 * float(err_copy.mean()), (down_idx, float(err.mean()), float(err_copy.mean()))
        c0 = (h.n_up - h.n_down) / 2 * ((h.n_up - h.n_down) / 2 + 1) + h.n_down if down_idx < 0 else 1.0
        assert torch.allclose(s2.double(), c0 - rho.double().sum(1), rtol=0, atol=1e-6 * (abs(c0) + float(rho.abs().sum(1).max())))
        # splitting one walker's pairs across forward chunks does not change a bit
        s2c, rhoc = eng.spin(r, R, down_idx=down_idx, want_ratios=True, max_ws_bytes=small)
        assert torch.equal(s2c, s2) and torch.equal(rhoc, rho)


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('mol', ['LiH', 'C', 'N2'])
def test_known_answer_on_the_engine(mol, dtype):
    """Orbitals with no spin or inter-electron dependence in one full determinant: s2 = N/2 (N/2 + 1) at every walker."""
    h = _hamil(mol)
    a = B200Ansatz(h, 'psiformer', dtype=dtype, gemm_backend=1 if dtype == 'float32' else 0, cusp='none')
    params = known_answer_params(a.spec, PN.perturb_params(a.init(2)))
    r = torch.as_tensor(walkers(h, 64, seed=4), device=DEV)
    R = torch.as_tensor(h.mol.coords, device=DEV)
    pc = PhysicalConfiguration(R, r, torch.zeros(64, device=DEV))
    s2 = SP.evaluate_spin(h, a.apply)(params, pc)
    N = h.n_up + h.n_down
    P = h.n_up * h.n_down
    assert torch.allclose(s2.double().cpu(), torch.full((64,), N / 2 * (N / 2 + 1), dtype=torch.float64), rtol=0,
                          atol=TOL[dtype] * P)


def test_repeatable_and_walker_independent():
    h = _hamil('N2')
    a = B200Ansatz(h, 'psiformer', dtype='float32', gemm_backend=1)
    eng = a.engine_for(h, PN.perturb_params(a.init(0)))
    r = torch.as_tensor(walkers(h, 300, seed=5), device=DEV, dtype=torch.float32)
    R = torch.as_tensor(h.mol.coords, device=DEV, dtype=torch.float32)
    s1, p1 = eng.spin(r, R, want_ratios=True)
    s2, p2 = eng.spin(r, R, want_ratios=True)
    assert torch.equal(s1, s2) and torch.equal(p1, p2)
    r2 = r.clone()
    r2[7] += 0.3
    s3, _ = eng.spin(r2, R)
    keep = torch.arange(300, device=DEV) != 7
    assert torch.equal(s3[keep], s1[keep]) and not torch.equal(s3[7], s1[7])
    # caller-supplied sign / log give the same result as the forward inside the call
    sg, lg = eng.wf_forward(r, R)
    s4, _ = eng.spin(r, R, sign=sg, log=lg)
    assert torch.equal(s4, s1)


def test_status_codes():
    h = _hamil('LiH')
    a = B200Ansatz(h, 'psiformer', dtype='float64', **SMALL)
    eng = a.engine_for(h, PN.perturb_params(a.init(0)))
    R = torch.as_tensor(h.mol.coords, device=DEV)
    r = torch.as_tensor(walkers(h, 3), device=DEV)
    s2, _ = eng.spin(r[:0], R)
    assert s2.shape == (0,)
    for bad in (0, 1, 4, -2):  # down electrons of LiH are 2 and 3
        with pytest.raises(RuntimeError, match='down_idx'):
            eng.spin(r, R, down_idx=bad)
    rc = eng.lib.dqmc_spin(eng.h, r.data_ptr(), R.data_ptr(), 1, 3, None, None, -1, r.data_ptr(), None, None, 0, None)
    assert rc == 2
    sg, lg = eng.wf_forward(r, R)
    for half in (dict(sign=sg), dict(log=lg)):  # sign and log of the walkers come together or not at all
        with pytest.raises(RuntimeError, match='sign and log'):
            eng.spin(r, R, **half)
    # no down electrons: the constant D/2 (D/2 + 1), no forwards; the raising estimator is refused
    hl = MolecularHamiltonian(mol=Molecule(coords=[[0.0, 0.0, 0.0]], charges=[3], charge=0, spin=3))
    al = B200Ansatz(hl, 'psiformer', dtype='float64', **SMALL)
    el = al.engine_for(hl, PN.perturb_params(al.init(0)))
    rl = torch.as_tensor(walkers(hl, 5), device=DEV)
    Rl = torch.as_tensor(hl.mol.coords, device=DEV)
    assert el.workspace_bytes(5, MODE_SPIN) == 0 and el.workspace_bytes_min(5, MODE_SPIN) == 0
    n0 = el.launch_count
    s2, _ = el.spin(rl, Rl)
    assert torch.equal(s2.cpu(), torch.full((5,), 1.5 * 2.5, dtype=torch.float64)) and el.launch_count - n0 == 1
    with pytest.raises(RuntimeError, match='down_idx'):
        el.spin(rl, Rl, down_idx=3)


def _grads_close(got, ref, tol):
    # every parameter autograd reaches must come back from the engine, and nothing else
    ref = {k: v for k, v in ref.items() if v is not None}
    assert set(got) == set(ref), sorted(set(got) ^ set(ref))
    for k, v in ref.items():
        g = got[k].detach().cpu().double().reshape(v.shape)
        assert torch.allclose(g, v, rtol=tol, atol=tol * max(1.0, float(v.abs().max()))), (k, float((g - v).abs().max()))


def test_spin_penalty_gradients_match_autograd():
    """Squared and raising penalty gradients (compute_mean_spin_tangent, compute_mean_spin_raising_tangent) against torch
    autograd through the fp64 oracle of surrogate losses whose gradient is the reference's tangent (loss/spin.py:74-229)."""
    h, a, params, r, R = _setup('LiH', 'psiformer', 'float64', B=4, **SMALL)
    B = r.shape[0]
    pc = PhysicalConfiguration(R[None, None], r[None, None], torch.zeros(1, 1, B, device=DEV))
    w = torch.tensor([[[1.0, 0.5, 2.0, 1.5]]], device=DEV, dtype=torch.float64)
    mask = torch.tensor([[[True, True, False, True]]], device=DEV)
    pt = {k: v.clone().requires_grad_(True) for k, v in W.to_torch(params).items()}
    Rc = R.cpu()
    wf = lambda x: W.log_psi(a.spec, pt, x, Rc)
    wc, mc = w[0, 0].cpu(), mask[0, 0].cpu().double()
    n_mask = mc.sum()
    # squared penalty
    sc = SP.compute_spin_contributions(h, a, [params], pc)
    grads = SP.compute_mean_spin_tangent(sc, w, mask, a, [params], pc)[0]
    mean = (sc[0, 0].cpu() * wc).mean()
    loss = sum((sc[0, 0, b].cpu() - mean) * wc[b] * mc[b] / n_mask * wf(r[b].cpu())[1] for b in range(B))
    ref = dict(zip(pt, torch.autograd.grad(loss, list(pt.values()), allow_unused=True)))
    _grads_close(grads, ref, 1e-8)
    # raising penalty
    c, rho, beta = SP.compute_spin_raising_contributions(0, h, a, pc, [params], return_ratios=True)
    grads = SP.compute_mean_spin_raising_tangent(c, rho, beta, w, mask, a, [params], pc)[0]
    cm = (c[0, 0].cpu() * wc).mean()
    loss = 0.0
    for b in range(B):
        rb = r[b].cpu()
        cb = OS.spin_raising(wf, rb, h.n_up, beta)  # differentiable in the parameters
        loss = loss + cm * wc[b] * mc[b] / n_mask * (2 * (c[0, 0, b].cpu() - cm) * wf(rb)[1] + cb)
    ref = dict(zip(pt, torch.autograd.grad(loss, list(pt.values()), allow_unused=True)))
    _grads_close(grads, ref, 1e-8)
