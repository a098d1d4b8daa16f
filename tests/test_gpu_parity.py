"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on the same seeded
inputs, plus size-independent properties at the benchmark's full walker count.

Tolerances (SURVEY.md 8d): fp64 mode |dE_loc| <= 1e-8 max(1,|E_loc|), |dlog|psi|| <= 1e-10;
fp32 mode <= 2e-4 relative (the reference's own E_loc regression tolerance, tests/test_hamil.py:37-40).
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from deepqmc_b200 import params as PN
from deepqmc_b200.ansatz import B200Ansatz
from deepqmc_b200.hamil import STAT_KEYS, MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from deepqmc_b200.types import PhysicalConfiguration

DEV = 'cuda:0'


def make(mol_name, ecp=None, dtype='float64', seed=0, B=4, kind='psiformer', **hyper):
    from oracle.hamil import OracleHamiltonian

    mol = Molecule.from_name(mol_name)
    hamil = MolecularHamiltonian(mol=mol, ecp_type=ecp)
    ansatz = B200Ansatz(hamil, kind, dtype=dtype, **hyper)
    params = PN.perturb_params(ansatz.init(seed))
    rng = np.random.default_rng(seed)
    N = hamil.n_up + hamil.n_down
    r = mol.coords[rng.integers(0, len(mol.coords), size=(B, N))] + rng.normal(size=(B, N, 3))
    r = torch.as_tensor(r, device=DEV)
    R = torch.as_tensor(mol.coords, device=DEV)
    return mol, hamil, OracleHamiltonian(mol, ecp_type=ecp), ansatz, params, r, R


def oracle_eval(ansatz, ohamil, params, r, R, twist=None):
    from oracle import wf

    pt = wf.to_torch(params)
    Rc = R.cpu()
    out = []
    for b in range(r.shape[0]):
        f = lambda x: wf.log_psi(ansatz.spec, pt, x, Rc)
        s, l = f(r[b].cpu())
        e, st = ohamil.local_energy(f, r[b].cpu(), Rc, phi_random=None if twist is None else twist[b].cpu())
        out.append((s.item(), l.item(), e.item(), {k: v.item() for k, v in st.items()}))
    return out


SMALL = dict(embedding_dim=32, n_layers=2, n_heads=4, n_determinants=4)


@pytest.mark.parametrize('mol_name,hyper,B', [
    ('LiH', SMALL, 4),
    ('LiH', dict(), 2),  # full Psiformer: d=256, L=4, H=4, K=16 (BASELINE configs[1])
    ('N2', dict(embedding_dim=32, n_layers=2, n_heads=2, n_determinants=3), 2),
    ('H2O', dict(embedding_dim=64, n_layers=1, n_heads=4, n_determinants=2), 3),
])
def test_local_energy_fp64(mol_name, hyper, B):
    mol, hamil, oh, ansatz, params, r, R = make(mol_name, B=B, **hyper)
    pc = PhysicalConfiguration(R, r, torch.zeros(B, device=DEV))
    psi = ansatz.apply(params, pc)
    E, stats, grad = hamil.local_energy(ansatz.apply)(None, params, pc, return_grad=True)
    assert set(stats) == set(STAT_KEYS)
    ref = oracle_eval(ansatz, oh, params, r, R)
    for b, (s, l, e, st) in enumerate(ref):
        assert psi.sign[b].item() == s
        assert abs(psi.log[b].item() - l) <= 1e-10 * max(1, abs(l))
        assert abs(E[b].item() - e) <= 1e-8 * max(1, abs(e)), (b, E[b].item(), e)
        for k in STAT_KEYS:
            assert abs(stats[k][b].item() - st[k]) <= 1e-8 * max(1, abs(st[k])), (k, stats[k][b].item(), st[k])
    # quantum force = grad log|psi| against autograd
    from oracle import wf

    pt = wf.to_torch(params)
    g = torch.func.grad(lambda x: wf.log_psi(ansatz.spec, pt, x.reshape(-1, 3), R.cpu())[1])(r[0].cpu().reshape(-1))
    assert torch.allclose(grad[0].cpu(), g, rtol=1e-8, atol=1e-9)


def test_single_sample_signature():
    """The reference's Ansatz/Hamiltonian act on one sample (types.py:107-150); the mirror accepts that too."""
    mol, hamil, oh, ansatz, params, r, R = make('LiH', B=2, **SMALL)
    pc1 = PhysicalConfiguration(R, r[0], torch.zeros((), device=DEV))
    psi = ansatz.apply(params, pc1)
    assert psi.log.dim() == 0
    E, stats = hamil.local_energy(ansatz.apply)(None, params, pc1)
    Eb, _ = hamil.local_energy(ansatz.apply)(None, params, PhysicalConfiguration(R, r, torch.zeros(2, device=DEV)))
    assert E.dim() == 0 and abs(E.item() - Eb[0].item()) < 1e-12


def test_ecp_local_and_nonlocal_fp64():
    """ccECP carbon atom: local + non-local (12-point quadrature, injected twists) parity."""
    mol, hamil, oh, ansatz, params, r, R = make('C', ecp='ccECP', B=3, **SMALL)
    assert (hamil.n_up, hamil.n_down) == (3, 1)
    N = 4
    tw = torch.as_tensor(np.random.default_rng(5).uniform(0, np.pi / 5, size=(3, 1, N)), device=DEV)
    pc = PhysicalConfiguration(R, r, torch.zeros(3, device=DEV))
    E, stats = hamil.local_energy(ansatz.apply)(None, params, pc, ecp_twist=tw)
    ref = oracle_eval(ansatz, oh, params, r, R, twist=tw)
    for b, (s, l, e, st) in enumerate(ref):
        assert abs(stats['hamil/V_nl'][b].item() - st['hamil/V_nl']) <= 1e-8 * max(1, abs(st['hamil/V_nl']))
        assert abs(stats['hamil/V_loc'][b].item() - st['hamil/V_loc']) <= 1e-9 * max(1, abs(st['hamil/V_loc']))
        assert abs(E[b].item() - e) <= 1e-8 * max(1, abs(e))
    with pytest.raises(AssertionError):  # rng is mandatory with a non-local ECP (gaussian_type_ecp.py:176)
        hamil.local_energy(ansatz.apply)(None, params, pc)
    # Philox twists: valid, deterministic per seed, different across seeds
    E1, s1 = hamil.local_energy(ansatz.apply)(7, params, pc)
    E2, s2 = hamil.local_energy(ansatz.apply)(7, params, pc)
    E3, s3 = hamil.local_energy(ansatz.apply)(8, params, pc)
    assert torch.equal(E1, E2) and not torch.equal(E1, E3)
    assert torch.all(torch.isfinite(E1))


def test_determinism_rng_independence_and_chunking():
    """reference tests/test_energy.py:38-92: determinism, rng-independence without ECP,
    batch_size chunking == unbatched."""
    mol, hamil, oh, ansatz, params, r, R = make('LiH', B=7, **SMALL)
    pc = PhysicalConfiguration(R, r, torch.zeros(7, device=DEV))
    f = hamil.local_energy(ansatz.apply)
    E1, _ = f(1, params, pc)
    E2, _ = f(1, params, pc)
    E3, _ = f(2, params, pc)
    assert torch.equal(E1, E2) and torch.equal(E1, E3)
    eng = ansatz.engine_for(hamil, params)
    one = eng.lib.dqmc_workspace_bytes(eng.h, 1, 1)
    eng._ws = None
    Ec, *_ = eng.local_energy(r, R, max_ws_bytes=3 * one)  # chunks of <= 3 walkers
    eng._ws = None
    assert torch.allclose(Ec, E1, rtol=0, atol=1e-12)


def test_batched_nuclei_equals_shared():
    mol, hamil, oh, ansatz, params, r, R = make('LiH', B=3, **SMALL)
    eng = ansatz.engine_for(hamil, params)
    E0, *_ = eng.local_energy(r, R)
    E1, *_ = eng.local_energy(r, R[None].expand(3, -1, -1).contiguous())
    assert torch.equal(E0, E1)
    # translation invariance: shift electrons and nuclei of walker 1 together
    Rb = R[None].repeat(3, 1, 1)
    shift = torch.tensor([0.3, -1.1, 0.7], device=DEV, dtype=torch.float64)
    Rb[1] += shift
    rs = r.clone()
    rs[1] += shift
    E2, *_ = eng.local_energy(rs, Rb)
    assert torch.allclose(E2, E0, rtol=1e-9, atol=1e-9)


def test_fp32_mode_within_reference_tolerance():
    mol, hamil, oh, ansatz, params, r, R = make('LiH', B=4, dtype='float32')
    pc = PhysicalConfiguration(R.float(), r.float(), torch.zeros(4, device=DEV))
    E, stats = hamil.local_energy(ansatz.apply)(None, params, pc)
    ref = oracle_eval(ansatz, oh, params, r.double(), R.double())
    for b, (s, l, e, st) in enumerate(ref):
        scale_b = max(1, abs(e), 0.5 * abs(st['hamil/lap']), 0.5 * st['hamil/quantum_force'])
        assert abs(E[b].item() - e) <= 2e-4 * scale_b, (E[b].item(), e)


def test_metropolis_injected_noise_matches_oracle():
    """reference electron_samplers.py:102-163 with identical (injected) random numbers."""
    from oracle import wf
    from oracle.sampling import metropolis_step

    mol, hamil, oh, ansatz, params, r, R = make('LiH', B=6, **SMALL)
    eng = ansatz.engine_for(hamil, params)
    sign, log = eng.wf_forward(r, R)
    rng = np.random.default_rng(3)
    nsub, B, N = 5, 6, 4
    nn = torch.as_tensor(rng.normal(size=(nsub, B, N, 3)), device=DEV)
    nu = torch.as_tensor(rng.uniform(size=(nsub, B)), device=DEV)
    state = dict(r=r.clone(), sign=sign.clone(), log=log.clone(), age=torch.zeros(B, dtype=torch.int32, device=DEV),
                 tau=torch.tensor([0.4], dtype=torch.float64, device=DEV))
    stats = eng.mcmc_sweep(state, R, nsub, target_acceptance=0.57, max_age=2, noise_normal=nn, noise_uniform=nu)
    pt = wf.to_torch(params)
    Rc = R.cpu()
    wfb = lambda rr: tuple(torch.stack(x) for x in zip(*[wf.log_psi(ansatz.spec, pt, rr[b], Rc) for b in range(B)]))
    ost = dict(r=r.cpu().clone(), sign=sign.cpu().clone(), log=log.cpu().clone(), age=torch.zeros(B, dtype=torch.int32),
               tau=torch.tensor(0.4, dtype=torch.float64))
    for s in range(nsub):
        ost, acc = metropolis_step(wfb, ost, nn[s].cpu(), nu[s].cpu(), 0.57, 2)
    assert torch.allclose(state['r'].cpu(), ost['r'], atol=1e-12)
    assert torch.allclose(state['log'].cpu(), ost['log'], atol=1e-10)
    assert torch.equal(state['age'].cpu(), ost['age'])
    assert abs(state['tau'].item() - ost['tau'].item()) < 1e-12
    assert abs(stats[0].item() - acc.item()) < 1e-12
    assert abs(stats[4].item() - ost['log'].mean().item()) < 1e-10
    assert abs(stats[5].item() - ost['log'].std(unbiased=False).item()) < 1e-10


def test_metropolis_philox_statistics():
    """In-kernel Philox stream: acceptance in (0,1), tau adapts toward the target, walkers move,
    sampled log|psi| rises from the initial guess (equilibration)."""
    mol, hamil, oh, ansatz, params, r, R = make('LiH', B=512, **SMALL)
    eng = ansatz.engine_for(hamil, params)
    sign, log = eng.wf_forward(r, R)
    state = dict(r=r.clone(), sign=sign.clone(), log=log.clone(), age=torch.zeros(512, dtype=torch.int32, device=DEV),
                 tau=torch.tensor([1.0], dtype=torch.float64, device=DEV))
    accs = []
    for it in range(10):
        st = eng.mcmc_sweep(state, R, 10, seed=11, step0=10 * it)
        accs.append(st[0].item())
    assert 0.35 < accs[-1] < 0.8, accs
    assert state['log'].mean().item() > log.mean().item()
    s2, l2 = eng.wf_forward(state['r'], R)
    assert torch.allclose(l2, state['log'], atol=1e-9)  # state psi consistent with state r
    # different seeds -> different chains; same seed/step -> identical
    a = dict((k, v.clone()) for k, v in state.items())
    b = dict((k, v.clone()) for k, v in state.items())
    eng.mcmc_sweep(a, R, 2, seed=1, step0=0)
    eng.mcmc_sweep(b, R, 2, seed=1, step0=0)
    assert torch.equal(a['r'], b['r'])
    c = dict((k, v.clone()) for k, v in state.items())
    eng.mcmc_sweep(c, R, 2, seed=2, step0=0)
    assert not torch.equal(a['r'], c['r'])


def test_full_size_properties_4096_walkers():
    """BASELINE configs[1] size (LiH Psiformer d=256 L=4 K=16, 4096 walkers), fp32 production mode:
    size-independent properties instead of an oracle run.
      * exchange of two same-spin electrons: sign flips, log|psi| and E_loc unchanged
      * E_loc finite, E_kin + V_loc + V_el + E_nuc == E_loc (assembly identity, hamil.py:165-172)
      * fp32 result agrees with the fp64 engine on the same walkers to 2e-4
    """
    mol, hamil, oh, ansatz, params, r, R = make('LiH', B=4096, dtype='float32')
    r = (torch.as_tensor(mol.coords, device=DEV)[torch.randint(0, 2, (4096, 4), device=DEV)]
         + 0.8 * torch.randn(4096, 4, 3, device=DEV, dtype=torch.float64))
    pc = PhysicalConfiguration(R.float(), r.float(), torch.zeros(4096, device=DEV))
    f = hamil.local_energy(ansatz.apply)
    E, st = f(None, params, pc)
    psi = ansatz.apply(params, pc)
    assert torch.isfinite(E).all()
    perm = torch.tensor([1, 0, 2, 3], device=DEV)
    pcx = PhysicalConfiguration(R.float(), r.float()[:, perm], torch.zeros(4096, device=DEV))
    Ex, _ = f(None, params, pcx)
    psix = ansatz.apply(params, pcx)
    assert torch.equal(psix.sign, -psi.sign)
    dl = (psix.log - psi.log).abs()
    assert dl.median().item() < 2e-5 and dl.quantile(0.99).item() < 2e-3, (dl.median().item(), dl.max().item())
    scale = torch.maximum(E.abs(), st['hamil/E_kin'].abs()).clamp(min=1)
    dE = (Ex - E).abs() / scale
    assert dE.median().item() < 1e-4 and dE.quantile(0.99).item() < 5e-3, (dE.median().item(), dE.max().item())
    e_nuc = 3.0 * 1.0 / np.linalg.norm(mol.coords[0] - mol.coords[1])
    asm = st['hamil/E_kin'] + st['hamil/V_loc'] + st['hamil/V_el'] + st['hamil/V_nl'] + e_nuc
    assert ((asm - E).abs() / scale).max().item() < 1e-5
    a64 = B200Ansatz(hamil, 'psiformer', dtype='float64')
    E64, st64 = hamil.local_energy(a64.apply)(None, params, PhysicalConfiguration(R, r, torch.zeros(4096, device=DEV)))
    rel = ((E.double() - E64).abs() / torch.maximum(E64.abs(), st64['hamil/E_kin'].abs()).clamp(min=1))
    # median at fp32 round-off; the tail are walkers next to a node / nucleus where E_kin cancels badly
    assert rel.median().item() < 2e-5 and rel.quantile(0.9).item() < 2e-4 and rel.quantile(0.99).item() < 2e-3, (
        rel.median().item(), rel.quantile(0.99).item(), rel.max().item())


def test_benzene_ccecp_small_hyper_vs_oracle():
    """BASELINE configs[3] geometry (benzene, ccECP, N = 30 valence electrons, M = 12, 6 non-local
    centres): full E_loc including the 12-point non-local quadrature, reduced widths so the oracle's
    autograd Hessian (90 coordinates) and 2160 forwards stay in seconds."""
    hyper = dict(embedding_dim=32, n_layers=1, n_heads=2, n_determinants=2)
    mol, hamil, oh, ansatz, params, r, R = make('benzene', ecp='ccECP', B=1, **hyper)
    assert (hamil.n_up, hamil.n_down) == (15, 15)
    tw = torch.as_tensor(np.random.default_rng(2).uniform(0, np.pi / 5, size=(1, 6, 30)), device=DEV)
    pc = PhysicalConfiguration(R, r, torch.zeros(1, device=DEV))
    E, stats = hamil.local_energy(ansatz.apply)(None, params, pc, ecp_twist=tw)
    (s, l, e, st), = oracle_eval(ansatz, oh, params, r, R, twist=tw)
    for k in STAT_KEYS:
        assert abs(stats[k][0].item() - st[k]) <= 1e-7 * max(1, abs(st[k])), (k, stats[k][0].item(), st[k])
    assert abs(E[0].item() - e) <= 1e-7 * max(1, abs(e))


def test_benzene_full_size_one_walker_vs_oracle():
    """BASELINE configs[3] at FULL size (benzene, ccECP, Psiformer d = 256, L = 4, H = 4, K = 16): ONE walker against the
    ORACLE (autograd Hessian over the 90 coordinates, all 2160 quadrature forwards; about a minute of host time):
      * fp64 engine: log|psi| to 1e-10, E_loc and all six statistics to 1e-8 (relative to max(1, |value|));
      * fp32 production engine (tensor-core backend: whole-trunk kernel for the quadrature forwards, 3xTF32 forward-Laplacian
        rows): E_loc to 2e-4 of its natural scale max(1, |E|, |lap| / 2, |grad|^2 / 2) -- E_kin = -(lap + |grad|^2) / 2 is a
        difference of those two terms, fp32 round-off is relative to them, not to their difference -- and V_nl to 2e-4 of
        max(1, |V_nl|)."""
    mol, hamil, oh, a64, params, r, R = make('benzene', ecp='ccECP', B=1)
    # a typical walker, not a freshly drawn one (whose Laplacian next to a nucleus is ~1e6): 40 Metropolis sub-steps first
    eng = a64.engine_for(hamil, params)
    sg, lg = eng.wf_forward(r, R)
    state = dict(r=r.clone(), sign=sg, log=lg, age=torch.zeros(1, dtype=torch.int32, device=DEV),
                 tau=torch.tensor([0.3], dtype=torch.float64, device=DEV))
    for it in range(4):
        eng.mcmc_sweep(state, R, 10, seed=3, step0=10 * it)
    r = state['r'].clone()
    tw = torch.as_tensor(np.random.default_rng(5).uniform(0, np.pi / 5, size=(1, 6, 30)), device=DEV)
    pc = PhysicalConfiguration(R, r, torch.zeros(1, device=DEV))
    psi = a64.apply(params, pc)
    E64, s64 = hamil.local_energy(a64.apply)(None, params, pc, ecp_twist=tw)
    (s, l, e, st), = oracle_eval(a64, oh, params, r, R, twist=tw)
    assert psi.sign[0].item() == s
    assert abs(psi.log[0].item() - l) <= 1e-10 * max(1, abs(l)), (psi.log[0].item(), l)
    assert abs(E64[0].item() - e) <= 1e-8 * max(1, abs(e)), (E64[0].item(), e)
    for k in STAT_KEYS:
        assert abs(s64[k][0].item() - st[k]) <= 1e-8 * max(1, abs(st[k])), (k, s64[k][0].item(), st[k])
    a32 = B200Ansatz(hamil, 'psiformer', dtype='float32', gemm_backend=1)
    pc32 = PhysicalConfiguration(R.float(), r.float(), torch.zeros(1, device=DEV))
    E32, s32 = hamil.local_energy(a32.apply)(None, params, pc32, ecp_twist=tw.float())
    psi32 = a32.apply(params, pc32)
    assert psi32.sign[0].item() == s
    assert abs(psi32.log[0].item() - l) <= 2e-4 * max(1, abs(l))
    scale = max(1.0, abs(e), 0.5 * abs(st['hamil/lap']), 0.5 * st['hamil/quantum_force'])
    assert abs(E32[0].item() - e) <= 2e-4 * scale, (E32[0].item(), e, scale)
    assert abs(s32['hamil/V_nl'][0].item() - st['hamil/V_nl']) <= 2e-4 * max(1, abs(st['hamil/V_nl'])), (
        s32['hamil/V_nl'][0].item(), st['hamil/V_nl'])
    assert abs(s32['hamil/V_loc'][0].item() - st['hamil/V_loc']) <= 1e-5 * max(1, abs(st['hamil/V_loc']))


def test_benzene_full_psiformer_fp32_tensor_core_vs_fp64():
    """Full-width benzene Psiformer (d=256, L=4, K=16): fp32 tensor-core engine against the fp64
    CUDA-core engine on the same walkers and quadrature twists (the oracle is too slow here)."""
    mol, hamil, oh, a64, params, r, R = make('benzene', ecp='ccECP', B=3)
    a32 = B200Ansatz(hamil, 'psiformer', dtype='float32', gemm_backend=1)
    tw = torch.as_tensor(np.random.default_rng(2).uniform(0, np.pi / 5, size=(3, 6, 30)), device=DEV)
    f64 = hamil.local_energy(a64.apply)
    f32 = hamil.local_energy(a32.apply)
    E64, s64 = f64(None, params, PhysicalConfiguration(R, r, torch.zeros(3, device=DEV)), ecp_twist=tw)
    E32, s32 = f32(None, params, PhysicalConfiguration(R.float(), r.float(), torch.zeros(3, device=DEV)), ecp_twist=tw.float())
    psi64 = a64.apply(params, PhysicalConfiguration(R, r, torch.zeros(3, device=DEV)))
    psi32 = a32.apply(params, PhysicalConfiguration(R.float(), r.float(), torch.zeros(3, device=DEV)))
    assert torch.equal(psi64.sign.float(), psi32.sign)
    assert (psi64.log - psi32.log.double()).abs().max().item() < 2e-3
    for b in range(3):
        scale = max(1.0, abs(E64[b].item()), 0.5 * abs(s64['hamil/lap'][b].item()), 0.5 * s64['hamil/quantum_force'][b].item())
        assert abs(E32[b].item() - E64[b].item()) <= 1e-3 * scale, (b, E32[b].item(), E64[b].item())
        assert abs(s32['hamil/V_nl'][b].item() - s64['hamil/V_nl'][b].item()) <= 2e-3 * max(1, abs(s64['hamil/V_nl'][b].item()))


@pytest.mark.parametrize('mol_name,hyper,B', [
    ('LiH', dict(embedding_dim=32, n_layers=3, n_determinants=4), 3),
    ('N2', dict(embedding_dim=32, n_layers=2, n_determinants=2), 2),  # BASELINE configs[2] geometry
])
def test_ferminet_local_energy_fp64(mol_name, hyper, B):
    """FermiNet trunk (reference conf/ansatz/ferminet.yaml: one- and two-electron streams, shared edge
    MLP, residual/sqrt2, no cusp) through the same engine: psi, E_loc, stats against the oracle."""
    mol, hamil, oh, ansatz, params, r, R = make(mol_name, B=B, kind='ferminet', **hyper)
    pc = PhysicalConfiguration(R, r, torch.zeros(B, device=DEV))
    psi = ansatz.apply(params, pc)
    E, stats = hamil.local_energy(ansatz.apply)(None, params, pc)
    for b, (s, l, e, st) in enumerate(oracle_eval(ansatz, oh, params, r, R)):
        assert psi.sign[b].item() == s and abs(psi.log[b].item() - l) <= 1e-10 * max(1, abs(l))
        assert abs(E[b].item() - e) <= 1e-8 * max(1, abs(e))
        for k in STAT_KEYS:
            assert abs(stats[k][b].item() - st[k]) <= 1e-8 * max(1, abs(st[k])), (k, stats[k][b].item(), st[k])


def test_ferminet_n2_full_fp32_tensor_core_vs_fp64():
    """N2 FermiNet at full width (d=256, L=4, K=16, 32-wide edge stream): fp32 tensor-core engine vs fp64."""
    mol, hamil, oh, a64, params, r, R = make('N2', B=4, kind='ferminet')
    a32 = B200Ansatz(hamil, 'ferminet', dtype='float32', gemm_backend=1)
    E64, s64 = hamil.local_energy(a64.apply)(None, params, PhysicalConfiguration(R, r, torch.zeros(4, device=DEV)))
    E32, s32 = hamil.local_energy(a32.apply)(None, params, PhysicalConfiguration(R.float(), r.float(), torch.zeros(4, device=DEV)))
    for b in range(4):
        scale = max(1.0, abs(E64[b].item()), 0.5 * abs(s64['hamil/lap'][b].item()), 0.5 * s64['hamil/quantum_force'][b].item())
        assert abs(E32[b].item() - E64[b].item()) <= 1e-3 * scale, (b, E32[b].item(), E64[b].item())


@pytest.mark.parametrize('mol_name,hyper,B', [
    ('LiH', SMALL, 3),
    ('H2O', dict(embedding_dim=32, n_layers=2, n_heads=2, n_determinants=3), 2),
    ('cyclobutadiene_square', dict(embedding_dim=32, n_layers=1, n_heads=2, n_determinants=2), 1),  # BASELINE configs[4] geometry
])
def test_transpsiformer_local_energy_fp64(mol_name, hyper, B):
    """TransPsiformer (reference conf/ansatz/transpsiformer.yaml): nuclear attention tokens, envelope
    exponents from the NuclearGNNHead (SURVEY.md 8a row a7) -- wave function, E_loc and the 6 stats
    against the oracle; fp32 engine within the reference's 2e-4 tolerance."""
    mol, hamil, oh, ansatz, params, r, R = make(mol_name, B=B, kind='transpsiformer', **hyper)
    pc = PhysicalConfiguration(R, r, torch.zeros(B, device=DEV))
    psi = ansatz.apply(params, pc)
    E, stats = hamil.local_energy(ansatz.apply)(None, params, pc)
    ref = oracle_eval(ansatz, oh, params, r, R)
    for b, (s, l, e, st) in enumerate(ref):
        assert psi.sign[b].item() == s
        assert abs(psi.log[b].item() - l) <= 1e-10 * max(1, abs(l))
        assert abs(E[b].item() - e) <= 1e-8 * max(1, abs(e)), (b, E[b].item(), e)
        for k in STAT_KEYS:
            assert abs(stats[k][b].item() - st[k]) <= 1e-8 * max(1, abs(st[k])), (k, stats[k][b].item(), st[k])
    a32 = B200Ansatz(hamil, 'transpsiformer', dtype='float32', **hyper)
    E32, _ = hamil.local_energy(a32.apply)(None, params, PhysicalConfiguration(R.float(), r.float(), torch.zeros(B, device=DEV)))
    for b, (_, _, e, st) in enumerate(ref):  # same scale as test_fp32_mode_within_reference_tolerance
        scale_b = max(1, abs(e), 0.5 * abs(st['hamil/lap']), 0.5 * st['hamil/quantum_force'])
        assert abs(E32[b].item() - e) <= 2e-4 * scale_b, (b, E32[b].item(), e)


def test_transpsiformer_geometry_change_refreshes_nuclear_stream():
    """The nuclear stream (keys/values of the nuclear tokens, envelope exponents) is a function of R:
    a call with another geometry must not reuse the uploaded one."""
    mol, hamil, oh, ansatz, params, r, R = make('LiH', B=2, kind='transpsiformer', **SMALL)
    from oracle import wf

    pt = wf.to_torch(params)
    R2 = R.clone()
    R2[1, 0] += 0.3
    for Rx in (R, R2, R):
        psi = ansatz.apply(params, PhysicalConfiguration(Rx, r, torch.zeros(2, device=DEV)))
        for b in range(2):
            _, l = wf.log_psi(ansatz.spec, pt, r[b].cpu(), Rx.cpu())
            assert abs(psi.log[b].item() - l.item()) <= 1e-10 * max(1, abs(l.item()))


@pytest.mark.parametrize('mol_name,hyper,B', [
    ('LiH', dict(), 4),               # the reference's own test ansatz on LiH (BASELINE configs[0])
    ('LiH', dict(n_layers=2), 2),     # second layer: dense tangents through the convolution
    ('C', dict(), 2),                 # n_up != n_down: two electron types, per-spin backflow widths differ
    ('H2O', dict(n_layers=2, n_determinants=3), 2),
])
def test_paulinet_test_ansatz_local_energy_fp64(mol_name, hyper, B):
    """conv-GNN 'PauliNet' ansatz of the reference's CPU tests (tests/conf/ansatz.yaml; SURVEY.md 8a rows
    a9, a10, a12-a14): embedding lookup, same/anti/ne convolutions, ssp Jastrow + backflow, default mult_act,
    per-shell envelopes, spin-factorised determinants, hk.Linear conf_coeff, DeepQMCCusp."""
    mol, hamil, oh, ansatz, params, r, R = make(mol_name, B=B, kind='paulinet', **hyper)
    pc = PhysicalConfiguration(R, r, torch.zeros(B, device=DEV))
    psi = ansatz.apply(params, pc)
    E, stats = hamil.local_energy(ansatz.apply)(None, params, pc)
    ref = oracle_eval(ansatz, oh, params, r, R)
    for b, (s, l, e, st) in enumerate(ref):
        assert psi.sign[b].item() == s
        assert abs(psi.log[b].item() - l) <= 1e-10 * max(1, abs(l))
        assert abs(E[b].item() - e) <= 1e-8 * max(1, abs(e)), (b, E[b].item(), e)
        for k in STAT_KEYS:
            assert abs(stats[k][b].item() - st[k]) <= 1e-8 * max(1, abs(st[k])), (k, stats[k][b].item(), st[k])


def test_paulinet_256_walkers_fp32_and_sampler():
    """BASELINE configs[0]: LiH, PauliNet test ansatz, 256 walkers -- fp32 engine against fp64 engine on
    Metropolis-equilibrated walkers, plus one decorrelated sampling step through the sampler mirror."""
    from deepqmc_b200.sampling import DecorrSampler

    mol = Molecule.from_name('LiH')
    hamil = MolecularHamiltonian(mol=mol)
    a64 = B200Ansatz(hamil, 'paulinet', dtype='float64')
    a32 = B200Ansatz(hamil, 'paulinet', dtype='float32')
    params = PN.perturb_params(a64.init(0))
    R = torch.as_tensor(mol.coords, device=DEV)
    smp = DecorrSampler(hamil, a64.apply, length=20, tau=0.1, max_age=20)
    state = smp.init(3, params, 256, R)
    for it in range(3):
        state, pc, stats = smp.sample(it, state, params, R)
    assert 0.05 < stats['sampling/acceptance'].item() <= 1.0
    E64, s64 = hamil.local_energy(a64.apply)(None, params, pc)
    E32, _ = hamil.local_energy(a32.apply)(None, params, PhysicalConfiguration(R.float(), pc.r.float(), torch.zeros(256, device=DEV)))
    scale = torch.maximum(torch.maximum(E64.abs(), 0.5 * s64['hamil/lap'].abs()), 0.5 * s64['hamil/quantum_force']).clamp(min=1)
    assert torch.isfinite(E64).all()
    assert ((E32.double() - E64).abs() <= 2e-4 * scale).float().mean().item() > 0.99


@pytest.mark.parametrize('mol_name,nb', [('LiH', 6), ('cyclobutadiene_square', 2)])
def test_excited_state_overlap_two_states_vs_oracle(mol_name, nb):
    """BASELINE configs[4] (two electronic states, TransPsiformer; LiH and the cyclobutadiene geometry of
    conf/hamil/mol/cyclobutadiene_square.yaml, reduced widths): Psi_i(r ~ Psi_j^2) blocks, sample-wise ratios and the
    symmetrised mean overlap (reference loss/overlap.py:19-150) against the oracle, plus every state's E_loc on its own
    walkers (what the excited-state loss sums, loss/loss_function.py)."""
    from deepqmc_b200.overlap import compute_mean_overlap, compute_psi_ratio
    from deepqmc_b200.sampling import MetropolisSampler, MultiElectronicStateSampler
    from oracle import wf
    from oracle.hamil import OracleHamiltonian

    hyper = dict(embedding_dim=32, n_layers=1, n_heads=2, n_determinants=2)
    mol = Molecule.from_name(mol_name)
    hamil = MolecularHamiltonian(mol=mol)
    ansatz = B200Ansatz(hamil, 'transpsiformer', dtype='float64', **hyper)
    params = [PN.perturb_params(ansatz.init(s), seed=10 + s) for s in range(2)]
    R = torch.as_tensor(mol.coords, device=DEV)
    smp = MultiElectronicStateSampler(MetropolisSampler(hamil, ansatz.apply, tau=0.3), 2)
    state = smp.init(5, params, nb, R)
    state, pc, stats = smp.sample(6, state, params, R)
    Nel = hamil.n_up + hamil.n_down
    assert pc.r.shape == (2, nb, Nel, 3) and stats['sampling/acceptance'].shape == (2,)
    if mol_name != 'LiH':  # E_loc of each state on its own walkers against the oracle
        oh = OracleHamiltonian(mol)
        for st_i in range(2):
            pcs = PhysicalConfiguration(R, pc.r[st_i], torch.zeros(nb, device=DEV))
            E, _ = hamil.local_energy(ansatz.apply)(None, params[st_i], pcs)
            (s_, l_, e_, _), = oracle_eval(ansatz, oh, params[st_i], pc.r[st_i][:1], R)
            assert abs(E[0].item() - e_) <= 1e-8 * max(1, abs(e_)), (st_i, E[0].item(), e_)
    ratio, _ = compute_psi_ratio(ansatz, params, pc)
    pts = [wf.to_torch(p) for p in params]
    Rc = R.cpu()
    ref = torch.zeros(2, 2, nb, dtype=torch.float64)
    logs = torch.zeros(2, 2, nb, dtype=torch.float64)
    signs = torch.zeros(2, 2, nb, dtype=torch.float64)
    for i in range(2):
        for j in range(2):
            for b in range(nb):
                s, l = wf.log_psi(ansatz.spec, pts[i], pc.r[j, b].cpu(), Rc)
                signs[i, j, b], logs[i, j, b] = s, l
    mean_log = logs.mean(dim=(-1, -2))  # per wave function over the samples of all states (loss/overlap.py:93-95)
    for i in range(2):
        for j in range(2):
            ref[i, j] = signs[i, j] * signs[j, j] * torch.exp((logs[i, j] - mean_log[i]) - (logs[j, j] - mean_log[j]))
    assert torch.allclose(ratio.cpu(), ref, rtol=1e-8, atol=1e-10)
    assert torch.allclose(ratio[0, 0].cpu(), torch.ones(nb, dtype=torch.float64)) and torch.allclose(ratio[1, 1].cpu(), torch.ones(nb, dtype=torch.float64))
    loss, ostats = compute_mean_overlap(ratio)
    S = ostats['overlap/pairwise/mean'].cpu()
    x = ref.mean(-1)
    expect = torch.sign(x) * torch.sqrt(torch.clamp(x * x.T, min=0))
    assert torch.allclose(S, expect, rtol=1e-8, atol=1e-10) and abs(loss.item() - expect[0, 1].item() ** 2) < 1e-10


@pytest.mark.parametrize('mol_name,hyper,B', [
    ('LiH', dict(embedding_dim=32, n_determinants=4, edge_dim=8), 3),
    ('H2O', dict(embedding_dim=16, n_determinants=3, edge_dim=8, n_layers=2), 2),
    ('C', dict(embedding_dim=16, n_determinants=2, edge_dim=16), 2),   # n_up != n_down
])
def test_paulinet_default_yaml_local_energy_fp64(mol_name, hyper, B):
    """'PauliNet' of conf/ansatz/default.yaml (SURVEY.md 8(a0) column 3): raw nucleus-electron features, concatenate
    update of [h, mean_up, mean_down, conv_same, conv_anti], two-layer tanh w / h MLPs, shared deep edge MLP with
    normalised residuals, linear Jastrow / backflow, full determinants, hk.Linear conf_coeff, DeepQMCCusp."""
    mol, hamil, oh, ansatz, params, r, R = make(mol_name, B=B, kind='paulinet_default', **hyper)
    pc = PhysicalConfiguration(R, r, torch.zeros(B, device=DEV))
    psi = ansatz.apply(params, pc)
    E, stats = hamil.local_energy(ansatz.apply)(None, params, pc)
    ref = oracle_eval(ansatz, oh, params, r, R)
    for b, (s, l, e, st) in enumerate(ref):
        assert psi.sign[b].item() == s
        assert abs(psi.log[b].item() - l) <= 1e-10 * max(1, abs(l))
        assert abs(E[b].item() - e) <= 1e-8 * max(1, abs(e)), (b, E[b].item(), e)
        for k in STAT_KEYS:
            assert abs(stats[k][b].item() - st[k]) <= 1e-8 * max(1, abs(st[k])), (k, stats[k][b].item(), st[k])


@pytest.mark.parametrize('form', ['psiformer', 'deepqmc'])
def test_nuclear_cusp_factor_fp64(form):
    """NuclearCuspAsymptotic (reference wf/cusp.py:81-101; off in the shipped yamls): value, gradient and Laplacian
    contributions on the plain electron-nucleus distances."""
    hyper = dict(SMALL, cusp_nuclei=form, cusp_nuclei_alpha=0.7)
    mol, hamil, oh, ansatz, params, r, R = make('H2O', B=2, **hyper)
    pc = PhysicalConfiguration(R, r, torch.zeros(2, device=DEV))
    psi = ansatz.apply(params, pc)
    E, stats = hamil.local_energy(ansatz.apply)(None, params, pc)
    for b, (s, l, e, st) in enumerate(oracle_eval(ansatz, oh, params, r, R)):
        assert abs(psi.log[b].item() - l) <= 1e-10 * max(1, abs(l))
        assert abs(E[b].item() - e) <= 1e-8 * max(1, abs(e)), (b, E[b].item(), e)
        assert abs(stats['hamil/lap'][b].item() - st['hamil/lap']) <= 1e-8 * max(1, abs(st['hamil/lap']))


def test_parameter_vjp_matches_autograd_fp64():
    """dqmc_wf_vjp_params (SURVEY.md 8(f) N1): d/dparams sum_b w_b log|psi(r_b)| for the Psiformer against torch
    autograd through the oracle, every parameter group (envelopes, cusp exponents, embedding, attention, MLP,
    backflow heads)."""
    from oracle import wf

    mol, hamil, oh, ansatz, params, r, R = make('H2O', B=3, embedding_dim=32, n_layers=2, n_heads=2, n_determinants=3)
    w = torch.as_tensor(np.random.default_rng(3).normal(size=3), device=DEV)
    psi, grads = ansatz.log_psi_vjp(params, PhysicalConfiguration(R, r, torch.zeros(3, device=DEV)), w)
    pt = {k: torch.as_tensor(v, dtype=torch.float64).requires_grad_(True) for k, v in params.items()}
    tot = 0
    for b in range(3):
        s, l = wf.log_psi(ansatz.spec, pt, r[b].cpu(), R.cpu())
        assert psi.sign[b].item() == s.item() and abs(psi.log[b].item() - l.item()) <= 1e-10 * max(1, abs(l.item()))
        tot = tot + w[b].cpu() * l
    tot.backward()
    assert set(grads) == set(pt)
    for k, v in pt.items():
        ref = v.grad
        assert torch.allclose(grads[k].cpu().reshape(ref.shape), ref, rtol=1e-8, atol=1e-9 * max(1.0, ref.abs().max().item())), k


def test_energy_gradient_fp32_close_to_fp64():
    """Energy gradient = one local-energy pass + one reverse pass with cotangent (E_loc - <E>) / B
    (reference loss/energy.py:77-102): the fp32 engine (tensor-core forward GEMMs) agrees with the fp64 engine."""
    from deepqmc_b200.energy import compute_mean_energy_tangent, median_clip_and_mask

    mol = Molecule.from_name('LiH')
    hamil = MolecularHamiltonian(mol=mol)
    hyper = dict(embedding_dim=64, n_layers=2, n_heads=2, n_determinants=4)
    a64 = B200Ansatz(hamil, 'psiformer', dtype='float64', **hyper)
    a32 = B200Ansatz(hamil, 'psiformer', dtype='float32', gemm_backend=1, **hyper)
    params = PN.perturb_params(a64.init(0))
    rng = np.random.default_rng(0)
    r = torch.as_tensor(mol.coords[rng.integers(0, 2, size=(64, 4))] + 0.7 * rng.normal(size=(64, 4, 3)), device=DEV)
    R = torch.as_tensor(mol.coords, device=DEV)
    out = {}
    for name, a, dt in (('f64', a64, torch.float64), ('f32', a32, torch.float32)):
        pc = PhysicalConfiguration(R.to(dt), r.to(dt), torch.zeros(64, device=DEV))
        E, _ = hamil.local_energy(a.apply)(None, params, pc)
        Ec, mask = median_clip_and_mask(E, 5.0)
        out[name] = compute_mean_energy_tangent(Ec, None, mask, a, params, pc)
    for k in out['f64']:
        g64, g32 = out['f64'][k].double(), out['f32'][k].double()
        assert (g64 - g32).abs().max().item() <= 2e-3 * max(1e-3, g64.abs().max().item()), k
