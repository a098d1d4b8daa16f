"""CPU: the spin estimators' oracle (oracle/spin.py) on known answers, the mean / std / tangent algebra of deepqmc_b200/spin.py
against the reference's tests/test_spin.py cases restated in numpy, its all-rank reductions in a gloo world of two, and the
workspace plan of the spin pass (DQMC_MODE_SPIN)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from deepqmc_b200 import params as PN
from deepqmc_b200 import spin as SP
from deepqmc_b200.engine import MODE_SPIN, Engine
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from deepqmc_b200.spec import ferminet_spec, paulinet_default_spec, paulinet_spec, psiformer_spec, transpsiformer_spec
from oracle import spin as OS
from oracle import wf as W
from spin_fixture import known_answer_params, walkers

SMALL = dict(embedding_dim=32, n_layers=2, n_heads=2, n_determinants=3)


@pytest.mark.parametrize('mol', ['LiH', 'C', 'B', 'N2'])
def test_oracle_spin_independent_orbitals_give_maximal_spin(mol):
    """Orbitals without spin or inter-electron dependence in one full determinant: every swap ratio is -1, so
    s2 = D/2 (D/2 + 1) + n_down + n_up n_down = N/2 (N/2 + 1) at every walker."""
    h = MolecularHamiltonian(mol=Molecule.from_name(mol))
    spec = psiformer_spec(h, cusp='none', **SMALL)
    p = W.to_torch(known_answer_params(spec, PN.perturb_params(PN.init_params(spec, 3))))
    R = torch.as_tensor(h.mol.coords)
    wf = OS.wave_function(spec, p, R)
    N = h.n_up + h.n_down
    for r in torch.as_tensor(walkers(h, 3, seed=1)):
        rho = OS.spin_ratios(wf, r, h.n_up, h.n_down)
        assert torch.allclose(rho, -torch.ones_like(rho), rtol=0, atol=1e-12)
        # the sum of n_up n_down ratios: 1e-12 per ratio
        assert abs(float(OS.evaluate_spin(wf, r, h.n_up, h.n_down)) - N / 2 * (N / 2 + 1)) < 1e-12 * max(1, rho.numel())
        for beta in range(h.n_up, N):
            assert abs(float(OS.spin_raising(wf, r, h.n_up, beta)) - (1 + h.n_up)) < 1e-12 * h.n_up


def _gaussian_orbitals(n, seed):
    g = torch.Generator().manual_seed(seed)
    centers = torch.randn(n, 3, generator=g, dtype=torch.float64)
    poly = torch.randn(n, 4, generator=g, dtype=torch.float64)

    def phi(x):  # [m, 3] -> [m, n]
        d = x[:, None, :] - centers[None]
        return (poly[None, :, 0] + (d * poly[None, :, 1:]).sum(-1)) * torch.exp(-0.5 * (d**2).sum(-1))

    return phi


def test_oracle_spin_closed_shell_singlet_is_zero():
    """det(phi(r_up)) det(phi(r_down)) with the same spatial orbitals is a singlet: s2 = 0 at every walker."""
    n = 3
    phi = _gaussian_orbitals(n, 0)

    def wf(r):
        s1, l1 = torch.linalg.slogdet(phi(r[:n]))
        s2, l2 = torch.linalg.slogdet(phi(r[n:]))
        return s1 * s2, l1 + l2

    g = torch.Generator().manual_seed(1)
    for _ in range(4):
        r = torch.randn(2 * n, 3, generator=g, dtype=torch.float64)
        assert abs(float(OS.evaluate_spin(wf, r, n, n))) < 1e-12


def test_oracle_spin_without_down_electrons_is_the_constant():
    phi = _gaussian_orbitals(3, 2)
    wf = lambda r: torch.linalg.slogdet(phi(r))
    r = torch.randn(3, 3, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    assert float(OS.evaluate_spin(wf, r, 3, 0)) == 1.5 * 2.5


def test_mean_and_std_match_reference_cases():
    """reference tests/test_spin.py::TestComputeMeanSpin, restated in numpy."""
    sc = np.array([[[1.0, 2.0, 3.0], [4.0, 5.0, 6.0]]])
    w = np.array([[[1.0, 2.0, 1.0], [0.5, 1.0, 1.5]]])
    mean, stats = SP.compute_mean_spin(torch.as_tensor(sc), torch.as_tensor(w))
    assert abs(float(mean) - np.mean(sc * w)) < 1e-14
    wm = (sc * w).sum(-1) / w.sum(-1)
    ws = np.sqrt((w * (sc - wm[..., None]) ** 2).sum(-1) / w.sum(-1))
    assert np.allclose(stats['spin/mean'].numpy(), wm, rtol=0, atol=1e-14)
    assert np.allclose(stats['spin/std'].numpy(), ws, rtol=0, atol=1e-14)
    # a subset of the states selects the matching weight column
    mean1, stats1 = SP.compute_mean_spin(torch.as_tensor(sc[:, 1:2]), torch.as_tensor(w), states=[1])
    assert abs(float(mean1) - np.mean(sc[:, 1:2] * w[:, 1:2])) < 1e-14
    assert abs(float(stats1['spin/mean'][0, 0]) - (sc[0, 1] * w[0, 1]).sum() / w[0, 1].sum()) < 1e-14


def test_squared_penalty_cotangent_matches_reference_tangent():
    """reference tests/test_spin.py::TestComputeMeanSpinTangent: sum_b cot_b t_b equals the reference's forward-mode
    masked_mean((s2 - <s2 w>) t w, mask) for any log-psi tangent t."""
    sc = np.array([[[1.0, 3.0], [2.0, 4.0]]])
    w = np.array([[[1.0, 1.0], [2.0, 1.0]]])
    lpt = np.array([[[0.5, -0.5], [1.0, 0.0]]])
    mask = np.array([[[True, True], [True, False]]])
    cot = SP.spin_tangent_cotangents(torch.as_tensor(sc), torch.as_tensor(w), torch.as_tensor(mask)).numpy()
    mean = np.mean(sc * w, axis=-1, keepdims=True)
    expected = np.where(mask, (sc - mean) * lpt * w, 0.0).sum() / mask.sum()
    assert abs((cot * lpt).sum() - expected) < 1e-14


def test_raising_penalty_cotangents_match_reference_tangent():
    """The reverse-pass form of the raising penalty's tangent: base cotangents a_b (2 (c_b - <c w>) + sum_a rho_ba) and
    swapped cotangents -a_b rho_ba contracted with the log-psi tangents of the base walkers (t_b) and of the swapped ones
    (t_ba) equal the reference's masked_mean(<c w> w (2 (c - <c w>) t + dc), mask) with dc_b = -sum_a rho_ba (t_ba - t_b)
    (loss/spin.py:177-229)."""
    rng = np.random.default_rng(0)
    Mb, S, B, nu = 2, 2, 5, 3
    rho = rng.normal(size=(Mb, S, B, nu))
    c = 1 - rho.sum(-1)
    w = rng.uniform(0.5, 1.5, size=(Mb, S, B))
    mask = rng.uniform(size=(Mb, S, B)) > 0.2
    t, tsw = rng.normal(size=(Mb, S, B)), rng.normal(size=(Mb, S, B, nu))
    base, sw = SP.spin_raising_cotangents(*(torch.as_tensor(x) for x in (c, rho, w, mask)))
    got = (base.numpy() * t).sum() + (sw.numpy() * tsw).sum()
    mean = np.mean(c * w, axis=-1, keepdims=True)
    dc = -(rho * (tsw - t[..., None])).sum(-1)
    expected = np.where(mask, mean * w * (2 * (c - mean) * t + dc), 0.0).sum() / mask.sum()
    assert abs(got - expected) < 1e-12


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    from deepqmc_b200 import parallel
    from deepqmc_b200 import spin as SPw

    parallel.init_from_env('gloo')
    g = torch.Generator().manual_seed(0)
    sc = torch.randn(2, 3, 8, generator=g, dtype=torch.float64)
    w = torch.rand(2, 3, 8, generator=g, dtype=torch.float64) + 0.5
    mask = torch.rand(2, 3, 8, generator=g) > 0.3
    rho = torch.randn(2, 3, 8, 4, generator=g, dtype=torch.float64)
    lo, hi = parallel.shard_bounds(8)
    res = {}
    for name, x, ww, m, rr in (('all', sc, w, mask, rho), ('shard', sc[..., lo:hi], w[..., lo:hi], mask[..., lo:hi],
                                                           rho[..., lo:hi, :])):
        if name == 'all':  # single-rank reference on the concatenated batch: no collective
            saved = parallel.world
            parallel.world = lambda: (0, 1)
        mean, stats = SPw.compute_mean_spin(x, ww)
        cot = SPw.spin_tangent_cotangents(x, ww, m)
        base, swp = SPw.spin_raising_cotangents(1 - rr.sum(-1), rr, ww, m)
        if name == 'all':
            parallel.world = saved
            cot, base, swp = cot[..., lo:hi], base[..., lo:hi], swp[..., lo:hi, :]
        res[name] = (mean, stats['spin/mean'], stats['spin/std'], cot, base, swp)
    ok = all(torch.allclose(a, b, rtol=1e-13, atol=1e-14) for a, b in zip(res['all'], res['shard']))
    q.put((rank, bool(ok)))
    torch.distributed.destroy_process_group()


def test_mean_spin_gloo_world2_equals_single_rank():
    """compute_mean_spin and the penalty cotangents on two ranks holding half the walkers each equal one rank holding all."""
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(60)
    assert res == [(0, True), (1, True)]


def _specs(h):
    yield psiformer_spec(h, **SMALL)
    yield transpsiformer_spec(h, **SMALL)
    yield ferminet_spec(h, **dict(SMALL, edge_dim=8))
    yield paulinet_spec(h)
    yield paulinet_default_spec(h)


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('mol', ['LiH', 'C', 'N2'])
def test_spin_plan_carved_never_exceeds_planned(built_lib, mol, dtype):
    h = MolecularHamiltonian(mol=Molecule.from_name(mol))
    for spec in _specs(h):
        eng = Engine(spec, h, dtype=dtype, plan_only=True,
                     gemm_backend=1 if dtype == 'float32' and spec.embedding_dim % 32 == 0 else 0)
        for B in (1, 257, 4096):
            planned, carved = eng.debug_plan(B, MODE_SPIN)
            assert planned == eng.workspace_bytes(B, MODE_SPIN)
            assert 0 < carved <= planned, (spec.kind, B, dtype, planned, carved)
            floor = eng.workspace_bytes_min(B, MODE_SPIN)
            assert floor <= planned
            for cap in {max(floor, planned // 3), max(floor, planned // 50), floor}:
                _, c2 = eng.debug_plan(B, MODE_SPIN, cap)
                assert 0 < c2 <= cap, (spec.kind, B, dtype, cap, c2)
            with pytest.raises(RuntimeError, match='workspace'):
                eng.debug_plan(B, MODE_SPIN, floor // 2)
        eng.close()


def test_spin_plan_without_down_electrons_is_empty(built_lib):
    """No down electrons: the exact estimator is the constant D/2 (D/2 + 1) without forwards, so the spin pass plans and
    carves no workspace."""
    h = MolecularHamiltonian(mol=Molecule(coords=[[0.0, 0.0, 0.0]], charges=[3], charge=0, spin=3))
    assert (h.n_up, h.n_down) == (3, 0)
    eng = Engine(psiformer_spec(h, **SMALL), h, dtype='float64', plan_only=True)
    for B in (1, 4096):
        assert eng.debug_plan(B, MODE_SPIN) == (0, 0)
        assert eng.workspace_bytes_min(B, MODE_SPIN) == 0
    eng.close()
