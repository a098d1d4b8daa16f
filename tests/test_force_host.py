"""CPU: the force oracle (oracle/force.py) on known answers, the estimator algebra of deepqmc_b200/force.py against the
reference's formulas restated in numpy, compute_mean_and_std in a gloo world of two, and the workspace plan of
dqmc_wf_grad_positions (DQMC_MODE_GRAD_POS) on plan-only engines."""
import dataclasses
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from deepqmc_b200 import force as FO
from deepqmc_b200 import params as PN
from deepqmc_b200.engine import MODE_GRAD_POS, Engine
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from deepqmc_b200.spec import ferminet_spec, paulinet_default_spec, paulinet_spec, psiformer_spec, transpsiformer_spec
from deepqmc_b200.types import PhysicalConfiguration
from oracle import force as OF
from oracle import wf as W
from spin_fixture import walkers

SMALL = dict(embedding_dim=32, n_layers=2, n_heads=4, n_determinants=4)
F64 = torch.float64


def _np_Q(r, R, c):
    d = r[None] - R[:, None]
    return c[:, None] * (d / np.linalg.norm(d, axis=-1, keepdims=True)).sum(1)


def _np_dQ(r, R, c):
    d = r[None] - R[:, None]  # [M, N, 3]
    n = np.linalg.norm(d, axis=-1)
    eye = np.eye(3)
    J = eye[None, None] / n[..., None, None] - d[..., :, None] * d[..., None, :] / n[..., None, None] ** 3  # [M, N, a, b]
    return c[:, None, None, None] * J


def _np_nuclear_force(R, Z):
    eps = np.finfo(np.float64).eps
    F = np.zeros_like(R)
    for m in range(len(R)):
        for n in range(len(R)):
            if n != m:
                d = R[m] - R[n]
                F[m] += Z[m] * Z[n] * d / np.sqrt(eps + d @ d) ** 3
    return F


def test_h2_nuclear_force():
    """H2 at 1.4 bohr: the nuclear repulsion pushes the protons apart with 1 / 1.4^2."""
    R = torch.tensor([[0.0, 0.0, 0.0], [0.0, 0.0, 1.4]], dtype=F64)
    f = OF.nuclear_force(R, [1.0, 1.0])
    ref = torch.tensor([[0, 0, -1 / 1.4**2], [0, 0, 1 / 1.4**2]], dtype=F64)
    assert torch.allclose(f, ref, rtol=1e-14, atol=1e-15)
    assert torch.allclose(FO.nuclear_force(R, None, [1.0, 1.0]), ref, rtol=1e-14, atol=1e-15)


def test_hydrogen_exact_wave_function_zvq_has_zero_variance():
    """Hydrogen atom, psi = exp(-|r - R|): every AC-ZVQ sample vanishes to round-off, the bare samples do not."""
    R = torch.zeros(1, 3, dtype=F64)
    log_psi = lambda r, R_: -torch.linalg.norm(r[0] - R_[0])
    g = torch.Generator().manual_seed(0)
    zvq, bare = [], []
    for _ in range(16):
        r = torch.randn(1, 3, generator=g, dtype=F64)
        zvq.append(OF.force_ac_zvq(r, R, [1.0], OF.grad_r(log_psi, r, R)))
        bare.append(OF.force_bare(r, R, [1.0]))
    assert torch.stack(zvq).abs().max() < 1e-14
    assert torch.stack(bare).abs().max() > 0.1


@pytest.mark.parametrize('kind', ['psiformer', 'ferminet'])
@pytest.mark.parametrize('mol', ['LiH', 'N2', 'H2O'])
def test_oracle_translation_identity(kind, mol):
    """Moving every electron and nucleus together leaves psi unchanged: sum_m grad_R + sum_i grad_r = 0."""
    h = MolecularHamiltonian(mol=Molecule.from_name(mol))
    spec = (psiformer_spec if kind == 'psiformer' else ferminet_spec)(h, **(SMALL if kind == 'psiformer' else dict(SMALL, edge_dim=8)))
    spec = dataclasses.replace(spec, cusp_nuclei='psiformer', cusp_nuclei_trainable=False, cusp_nuclei_alpha=1.3)
    params = W.to_torch(PN.perturb_params(PN.init_params(spec, 0)))
    R = torch.as_tensor(h.mol.coords, dtype=F64)
    r = torch.as_tensor(walkers(h, 1, seed=2)[0])
    lp = lambda x, y: W.log_psi(spec, params, x, y)[1]
    gr, gR = OF.grad_r(lp, r, R), OF.grad_R(lp, r, R)
    scale = max(1.0, float(gr.abs().max()), float(gR.abs().max()))
    assert float((gr.sum(0) + gR.sum(0)).abs().max()) < 1e-11 * scale


def test_Q_and_its_jacobian_match_numpy():
    rng = np.random.default_rng(0)
    r, R, c = rng.normal(size=(5, 3)), rng.normal(size=(3, 3)), np.array([1.0, 3.0, 7.0])
    q = OF.Q(torch.as_tensor(r), torch.as_tensor(R), c).numpy()
    assert np.allclose(q, _np_Q(r, R, c), rtol=1e-13, atol=1e-14)
    assert np.allclose(FO.Q(torch.as_tensor(r), torch.as_tensor(R), c).numpy(), q, rtol=1e-13, atol=1e-14)
    J = OF.dQ_dr(torch.as_tensor(r), torch.as_tensor(R), c).numpy()  # [M, a, N, b]
    assert np.allclose(J.transpose(0, 2, 1, 3), _np_dQ(r, R, c), rtol=1e-12, atol=1e-13)
    assert np.allclose(OF.nuclear_force(torch.as_tensor(R), c).numpy(), _np_nuclear_force(R, c), rtol=1e-12)


def test_antithetic_mirror_geometry_and_weights():
    """A mirrored electron lands at 2 R_nn - r; electrons beyond r_cut stay; the weights are softmax(0, 2 dlog|psi|)."""
    R = torch.tensor([[0.0, 0.0, 0.0], [0.0, 0.0, 2.0], [0.0, 0.0, 4.0]], dtype=F64)
    r = torch.tensor([[[0.1, 0.2, 0.3], [0.0, 0.3, 2.2], [3.0, 3.0, 3.0], [0.0, 0.0, 1.0]]], dtype=F64)
    pc = PhysicalConfiguration(R, r, torch.zeros(1))
    _, m = FO.antithetic_sampler(pc, 0.5)
    exp = r.clone()
    exp[0, 0] = -r[0, 0]
    exp[0, 1] = 2 * R[1] - r[0, 1]
    # electron 3 is equidistant from nuclei 0 and 1 and beyond r_cut: unchanged; electron 2 far away: unchanged
    assert torch.equal(m.r, exp)
    _, m2 = FO.antithetic_sampler(pc, 1.5)
    assert torch.allclose(m2.r[0, 3], 2 * R[0] - r[0, 3])  # tie -> the first nucleus
    for b in range(1):
        assert torch.allclose(OF.antithetic_mirror(r[b], R, 0.5), exp[b])

    class _Psi:
        def __init__(self, log):
            self.log = log

    log_psi = lambda rr: -(rr**2).sum((-1, -2))
    wf = lambda params, pc_: _Psi(log_psi(pc_.r))
    force = lambda rng, params, pc_: pc_.r[..., :3, :] * (1.0 if rng == 5 else 2.0)
    got = FO.antithetic_wrapper(force, wf, 0.5)(5, None, pc)
    lw = 2 * (log_psi(exp) - log_psi(r))
    w1 = torch.exp(lw) / (1 + torch.exp(lw))
    ref = (1 - w1)[:, None, None] * r[..., :3, :] + w1[:, None, None] * 2.0 * exp[..., :3, :]
    assert torch.allclose(got, ref, rtol=1e-14, atol=1e-15)


def test_estimator_algebra_matches_reference_formulas():
    """(E_loc - energy) algebra of ZVZBQ / ZB / ZVQZB and the oracle's ZVQ against numpy."""
    rng = np.random.default_rng(3)
    r, R, Z = rng.normal(size=(4, 3)), rng.normal(size=(2, 3)) * 2, np.array([3.0, 1.0])
    g_r, g_R = rng.normal(size=(4, 3)), rng.normal(size=(2, 3))
    e_loc, energy = -7.9, -8.05
    t = lambda x: torch.as_tensor(x)
    Fn = _np_nuclear_force(R, Z)
    d = r[None] - R[:, None]
    bare = Fn + Z[:, None] * (d / np.linalg.norm(d, axis=-1, keepdims=True) ** 3).sum(1)
    zvq = Fn + np.einsum('mnab,nb->ma', _np_dQ(r, R, Z), g_r)
    q = _np_Q(r, R, Z)
    assert np.allclose(OF.force_bare(t(r), t(R), Z).numpy(), bare, rtol=1e-12)
    assert np.allclose(OF.force_ac_zvq(t(r), t(R), Z, t(g_r)).numpy(), zvq, rtol=1e-12)
    assert np.allclose(OF.force_ac_zvzbq(t(r), t(R), Z, t(g_r), e_loc, energy).numpy(), zvq - 2 * (e_loc - energy) * q, rtol=1e-12)
    assert np.allclose(OF.force_ac_zb(t(r), t(R), Z, t(g_R), e_loc, energy).numpy(), bare - 2 * (e_loc - energy) * g_R, rtol=1e-12)
    assert np.allclose(OF.force_ac_zvqzb(t(r), t(R), Z, t(g_r), t(g_R), e_loc, energy).numpy(),
                       zvq - 2 * (e_loc - energy) * g_R, rtol=1e-12)


def test_finite_difference_displacement_matches_reference():
    """R - h e_k and r + sum_m softmax_m(-|R_m - r_i|) (h e_k)_m, batched (force.py) and per walker (oracle)."""
    rng = np.random.default_rng(4)
    B, N, M, h = 3, 5, 2, 1e-3
    r, R = rng.normal(size=(B, N, 3)), rng.normal(size=(M, 3))
    Rs, rs = FO.finite_difference_displacements(torch.as_tensor(r), torch.as_tensor(R), h)
    assert Rs.shape == (3 * M, M, 3) and rs.shape == (3 * M, B, N, 3)
    for b in range(B):
        dist = np.linalg.norm(R[:, None] - r[b][None], axis=-1)
        w = np.exp(-dist) / np.exp(-dist).sum(0, keepdims=True)
        for k, (Rk, rk) in enumerate(OF.fd_displacements(torch.as_tensor(r[b]), torch.as_tensor(R), h)):
            dR = np.zeros(3 * M)
            dR[k] = h
            dR = dR.reshape(M, 3)
            assert np.allclose(Rs[k].numpy(), R - dR, rtol=0, atol=1e-15)
            assert np.allclose(Rk.numpy(), R - dR, rtol=0, atol=1e-15)
            assert np.allclose(rs[k, b].numpy(), r[b] + np.einsum('nj,ne->ej', dR, w), rtol=0, atol=1e-15)
            assert np.allclose(rk.numpy(), rs[k, b].numpy(), rtol=0, atol=1e-15)


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    from deepqmc_b200 import force as FOw
    from deepqmc_b200 import parallel

    parallel.init_from_env('gloo')
    x = torch.randn(2, 3, 10, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    lo, hi = parallel.shard_bounds(10)
    got = FOw.compute_mean_and_std('force', x[..., lo:hi])
    ok = (torch.allclose(got['force/mean'], x.mean(-1), rtol=1e-13, atol=1e-14)
          and torch.allclose(got['force/std'], x.std(-1, unbiased=False), rtol=1e-13, atol=1e-14))
    q.put((rank, bool(ok)))
    torch.distributed.destroy_process_group()


def test_mean_and_std_gloo_world2_equals_single_rank():
    """compute_mean_and_std on two ranks holding half the samples each equals numpy's mean / population std of all."""
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


def _engine(spec, h, dtype):
    return Engine(spec, h, dtype=dtype, plan_only=True, gemm_backend=1 if dtype == 'float32' and spec.embedding_dim % 32 == 0 else 0)


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('mol', ['LiH', 'N2'])
def test_grad_pos_plan_carved_never_exceeds_planned(built_lib, mol, dtype):
    h = MolecularHamiltonian(mol=Molecule.from_name(mol))
    for spec in (psiformer_spec(h, **SMALL), transpsiformer_spec(h, **SMALL), ferminet_spec(h, **dict(SMALL, edge_dim=8))):
        eng = _engine(spec, h, dtype)
        for B in (1, 257, 4096):
            planned, carved = eng.debug_plan(B, MODE_GRAD_POS)
            assert planned == eng.workspace_bytes(B, MODE_GRAD_POS)
            assert 0 < carved <= planned, (spec.kind, B, dtype, planned, carved)
            floor = eng.workspace_bytes_min(B, MODE_GRAD_POS)
            assert 0 < floor <= planned
            for cap in {max(floor, planned // 3), floor}:
                _, c2 = eng.debug_plan(B, MODE_GRAD_POS, cap)
                assert 0 < c2 <= cap, (spec.kind, B, dtype, cap, c2)
            with pytest.raises(RuntimeError, match='workspace'):
                eng.debug_plan(B, MODE_GRAD_POS, floor // 2)
        eng.close()


def test_grad_pos_refused_for_conv_gnn_and_additive_backflow(built_lib):
    h = MolecularHamiltonian(mol=Molecule.from_name('LiH'))
    bf = dataclasses.replace(psiformer_spec(h, **SMALL), backflow_transform='add')
    for spec in (paulinet_spec(h), paulinet_default_spec(h), bf):
        eng = _engine(spec, h, 'float64')
        assert eng.workspace_bytes(8, MODE_GRAD_POS) == 0
        with pytest.raises(RuntimeError, match=r'\(2\)'):
            eng.debug_plan(8, MODE_GRAD_POS)
        eng.close()
