"""GPU: the reverse passes against fp64 autograd.

- the softmax attention backward (Engine::attention_bwd, attn_bwd_kernel) through dqmc_debug_attention_bwd: N = 2 ... 43 (an
  engine needs two electrons; at N = 71, the largest count whose fp64 backward tiling fits the shared memory at dh = 64, engine
  creation already refuses the configuration); heads of 64 and 16; N(0, 1) rows,
  scores spanning +-60 (near one-hot softmax rows), output cotangents scaled by 1e3 and 1e-3; the TransPsiformer's nuclear
  tokens (LiH, cyclobutadiene) with their cotangents summed atomically over 64 walkers;
- the weight- and bias-gradient reductions every reverse pass runs (Engine::wgrad / Engine::bgrad) through dqmc_debug_wgrad: row
  counts from 1 to 4096 * 256 + 77 (one row; a partial 32-row tile; one weight block; the first weight split; the bias split
  past its 128-block cap; the weight split at its 256-block cap, with block boundaries inside a walker of the odd electron count
  N = 5), K and Nc not multiples of 32, every per-spin electron range, the empty one included (a spin block without electrons:
  nothing is added), data of mixed sign and all positive;
- the parameter reverse pass dqmc_wf_vjp_params end to end against autograd through oracle.wf, every ansatz kind, on fully
  polarised, odd-spin and larger systems, with mixed-sign, one-hot, all-zero and training cotangents, and the full-width
  Psiformer; the fp32 engine at FermiNet batch sizes whose edge rows pass 1M, in one chunk and in several uneven ones.

Bounds (H100, measured worst case beside each constant):
- attention backward: per output array (dQ, dK, dV, dKn, dVn) max |err| <= max(C (u / 2^-24) err32, F u max|ref|), err32 the
  error of the same autograd evaluated in fp32 on the CPU (the conditioning of the case), u the unit roundoff of the engine;
- wgrad / bgrad: |dW - ref| <= c u (|A|^T |dY|) elementwise, u = 2^-24 (fp32) or 2^-53 (fp64); rows outside the range and
  the empty range add exactly nothing;
- fp64 end to end: per parameter array |g - ref| <= 1e-9 max|ref| + 1e-12 max over all arrays of max|ref|;
- fp32 end to end: per parameter array the error is at most a multiple of the error of the same autograd evaluated in fp32 on
  the CPU, or a floor of a few u max|ref| of the array, and never more than a cap times max|ref|;
- arrays log|psi| never reads (the down-spin heads of a polarised system) are exactly zero, as jax.grad gives them.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from deepqmc_b200.ansatz import B200Ansatz
from deepqmc_b200.engine import MODE_VJP
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from deepqmc_b200 import params as PN
from reverse_reference import attention_bwd_ref, log_psi_grads, wgrad_ref

DEV = 'cuda:0'
U = {'float64': 2.0 ** -53, 'float32': 2.0 ** -24}


def _chain(n, spin, z=1, step=1.6):
    return Molecule(coords=[[step * i, 0.2 * (i % 2), 0.0] for i in range(n)], charges=[z] * n, charge=0, spin=spin)


SYSTEMS = {
    'H2_triplet': lambda: _chain(2, 2, step=1.4),
    'H4_polarised': lambda: _chain(4, 4),
    'H7_polarised': lambda: _chain(7, 7),
    'H7_doublet': lambda: _chain(7, 1),  # odd spin: n_up = n_down + 1
    'N2': lambda: Molecule.from_name('N2'),
    'C5': lambda: _chain(5, 0, z=6, step=2.4),  # 30 electrons
}
HYPER = {
    'psiformer': dict(embedding_dim=32, n_layers=2, n_heads=4, n_determinants=4),
    'transpsiformer': dict(embedding_dim=32, n_layers=2, n_heads=4, n_determinants=4),
    'ferminet': dict(embedding_dim=32, n_layers=2, n_determinants=4, edge_dim=8),
    'paulinet': dict(),
    'paulinet_default': dict(embedding_dim=16, n_determinants=3, edge_dim=8),
}
POLARISED = ('H2_triplet', 'H4_polarised', 'H7_polarised')
# the reference's spin means over an empty spin block are NaN: these kinds have no gradient to compare against there
MEAN_KINDS = ('ferminet', 'paulinet_default')


def _cases(systems, kinds=tuple(HYPER)):
    return [(k, s) for k in kinds for s in systems if not (k in MEAN_KINDS and s in POLARISED)]


def _setup(system, kind, dtype, B, seed=0, **hyper):
    mol = SYSTEMS[system]()
    hamil = MolecularHamiltonian(mol=mol)
    ansatz = B200Ansatz(hamil, kind, dtype=dtype, **{**HYPER[kind], **hyper})
    if dtype == 'float32' and ansatz.spec.embedding_dim % 32 == 0:
        ansatz.gemm_backend = 1  # the tensor cores where production uses them
    params = PN.perturb_params(ansatz.init(seed))
    rng = np.random.default_rng(seed)
    N = hamil.n_up + hamil.n_down
    r = torch.as_tensor(mol.coords[rng.integers(0, len(mol.coords), size=(B, N))] + rng.normal(size=(B, N, 3)))
    R = torch.as_tensor(mol.coords)
    eng = ansatz.engine_for(hamil, params)
    return eng, ansatz.spec, params, r, R


def _vjp(eng, r, R, w, **kw):
    s, l, g = eng.vjp_params(r.to(DEV), R.to(DEV), w.to(DEV), **kw)
    return s.cpu().double(), l.cpu().double(), {k: v.detach().cpu().double() for k, v in g.items()}


def _errors(g, ref):
    """per array: (max |g - ref|, max |ref|)"""
    assert set(g) == set(ref)
    return {k: (float((g[k].reshape(ref[k].shape) - ref[k]).abs().max()) if ref[k].numel() else 0.0,
                float(ref[k].abs().max()) if ref[k].numel() else 0.0) for k in ref}


def _assert_unread_zero(g, ref):
    for k, v in ref.items():
        if v.numel() and not v.any():
            assert not g[k].any(), f'{k}: log|psi| does not read this array, its gradient must be exactly zero'


# ---- 0. attention backward through dqmc_debug_attention_bwd ------------------------------------------------------------------
ATT_N = [2, 3, 8, 17, 30, 32, 43]
ATT_C, ATT_F = 16.0, 256.0  # measured worst (H100): 0.10 of the bound (fp64, cyclobutadiene), 0.078 (fp32, N = 3 spread)
_ATT_ENGINES = {}


def _att_engine(mol_key, kind, dtype, **hyper):
    key = (mol_key, kind, dtype, tuple(sorted(hyper.items())))
    if key not in _ATT_ENGINES:
        if isinstance(mol_key, int):  # a neutral chain of ceil(N / 9) nuclei carrying N electrons
            n_nuc = -(-mol_key // 9)
            charges = [mol_key // n_nuc + (i < mol_key % n_nuc) for i in range(n_nuc)]
            mol = Molecule(coords=[[2.5 * i, 0.3 * (i % 2), 0.0] for i in range(n_nuc)], charges=charges, charge=0,
                           spin=mol_key % 2)
        else:
            mol = Molecule.from_name(mol_key)
        hamil = MolecularHamiltonian(mol=mol)
        a = B200Ansatz(hamil, kind, dtype=dtype, **hyper)
        _ATT_ENGINES[key] = a.engine_for(hamil, PN.perturb_params(a.init(0)))
    return _ATT_ENGINES[key]


def _att_inputs(B, N, d, g, case):
    Q, K, V, dO = (torch.randn(B * N, d, generator=g, dtype=torch.float64) for _ in range(4))
    if case == 'spread':  # q.k / sqrt(dh) with standard deviation ~25: rows span about +-60, near one-hot softmax
        Q, K = Q * 5.0, K * 5.0
    dO = dO * {'dO_1e3': 1e3, 'dO_1e-3': 1e-3}.get(case, 1.0)
    return torch.cat([Q, K, V], dim=1), dO


def _check_attention_bwd(eng, layer, QKV, dO, N, H, label):
    from tc_reference import weight

    dt = eng.dtype
    QKV, dO = QKV.to(dt), dO.to(dt)  # the values the kernel sees
    kn = vn = None
    if eng.spec.kind == 'transpsiformer':
        kn, vn = weight(eng, f'L{layer}.kn').cpu(), weight(eng, f'L{layer}.vn').cpu()
    got = eng.debug_attention_bwd(layer, QKV.to(DEV), dO.to(DEV))
    ref = attention_bwd_ref(QKV, dO, N, H, kn, vn)
    r32 = attention_bwd_ref(QKV, dO, N, H, kn, vn, dtype=torch.float32)
    d = QKV.shape[1] // 3
    split = lambda t: [] if t is None else [t] if t.shape[1] == d else list(t.split(d, dim=1))
    names = ['dQ', 'dK', 'dV', 'dKn', 'dVn']
    u = U['float64' if dt == torch.float64 else 'float32']
    worst = 0.0
    for name, gv, rv, cv in zip(names, sum((split(t) for t in got), []), sum((split(t) for t in ref), []),
                                sum((split(t) for t in r32), [])):
        assert torch.isfinite(gv).all(), name
        err = float((gv.cpu().double() - rv).abs().max())
        err32 = float((cv.double() - rv).abs().max())
        bound = max(ATT_C * (u / U['float32']) * err32, ATT_F * u * float(rv.abs().max()))
        worst = max(worst, err / bound if bound else (0.0 if err == 0 else float('inf')))
        assert err <= bound, (name, err, err32, float(rv.abs().max()))
    print(f'attention_bwd {label}: worst err / bound = {worst:.3g}')


@pytest.mark.parametrize('case', ['unit', 'spread', 'dO_1e3', 'dO_1e-3'])
@pytest.mark.parametrize('dh', [64, 16])
@pytest.mark.parametrize('N', ATT_N)
@pytest.mark.parametrize('dtype', ['float64', 'float32'])
def test_attention_bwd_against_fp64(dtype, N, dh, case):
    H = 2 if dh == 64 else 4
    eng = _att_engine(N, 'psiformer', dtype, embedding_dim=H * dh, n_layers=1, n_heads=H, n_determinants=1)
    B = 5
    g = torch.Generator().manual_seed(1000 * N + dh + len(case))
    QKV, dO = _att_inputs(B, N, H * dh, g, case)
    _check_attention_bwd(eng, 0, QKV, dO, N, H, f'{dtype} N={N} dh={dh} {case}')


@pytest.mark.parametrize('case', ['unit', 'spread'])
@pytest.mark.parametrize('mol', ['LiH', 'cyclobutadiene_square'])
@pytest.mark.parametrize('dtype', ['float64', 'float32'])
def test_attention_bwd_nuclear_tokens_against_fp64(dtype, mol, case):
    """TransPsiformer, d = 128, 2 heads of 64, both layers: the nuclear tokens' key / value cotangents are sums over 64
    walkers, accumulated atomically by 64 x 2 blocks."""
    eng = _att_engine(mol, 'transpsiformer', dtype, embedding_dim=128, n_layers=2, n_heads=2, n_determinants=2)
    N = eng.spec.n_elec
    g = torch.Generator().manual_seed(N + len(case))
    QKV, dO = _att_inputs(64, N, 128, g, case)
    for layer in range(2):
        _check_attention_bwd(eng, layer, QKV, dO, N, 2, f'{dtype} {mol} layer {layer} {case}')


# ---- 1. weight / bias gradients through dqmc_debug_wgrad ----------------------------------------------------------------------
WG_ROWS = [1, 31, 4095, 4097, 2048 * 128 + 1, 4096 * 256 + 77]
WG_K, WG_NC = 33, 45
# B: 5 electrons, n_up = 3 -> electron ranges of every walker
WG_RANGES = {'all': (0, -1), 'up': (0, 3), 'down': (3, 5), 'empty': (5, 5)}
# c of |dW - ref| <= c u |A|^T |dY| and of |db - ref| <= c u sum |dY|; measured worst on an H100: 2.98 (fp64), 3.54 (fp32)
WG_C = {'float64': 8.0, 'float32': 8.0}
# all-positive data, where every partial sum of a block's serial run grows with the rows: measured 17.3 (fp64), 17.2 (fp32) at
# 4096 * 256 + 77 rows (18.9 in another run: the atomic order varies), far below the rows-per-block (4128) a worst-case serial sum allows
WG_C_POS = {'float64': 48.0, 'float32': 48.0}


_WG_ENGINES = {}


def _wg_engine(dtype):
    if dtype not in _WG_ENGINES:
        hamil = MolecularHamiltonian(mol=Molecule.from_name('B'))
        assert (hamil.n_up, hamil.n_down) == (3, 2)
        a = B200Ansatz(hamil, 'psiformer', dtype=dtype, embedding_dim=16, n_layers=1, n_heads=2, n_determinants=2)
        _WG_ENGINES[dtype] = a.engine_for(hamil, a.init(0))
    return _WG_ENGINES[dtype]


@pytest.mark.parametrize('rng_name', list(WG_RANGES))
@pytest.mark.parametrize('rows,data', [(n, 'mixed') for n in WG_ROWS] + [(WG_ROWS[-1], 'positive')])
@pytest.mark.parametrize('dtype', ['float64', 'float32'])
def test_wgrad_bgrad_against_fp64(dtype, rows, data, rng_name):
    eng = _wg_engine(dtype)
    lo, hi = WG_RANGES[rng_name]
    g = torch.Generator().manual_seed(rows)
    A = torch.randn(rows, WG_K, generator=g, dtype=torch.float64)
    dY = torch.randn(rows, WG_NC, generator=g, dtype=torch.float64)
    if data == 'positive':
        A, dY = A.abs(), dY.abs()
    A, dY = A.to(eng.dtype), dY.to(eng.dtype)  # the values the kernel sees
    dW, db = eng.debug_wgrad(A.to(DEV), dY.to(DEV), lo, hi)
    dW, db = dW.cpu().double(), db.cpu().double()
    rW, rb, mW, mb = wgrad_ref(A, dY, 5, lo, hi)
    if rng_name == 'empty':
        assert not dW.any() and not db.any(), 'an empty electron range must add nothing'
        return
    u = U[dtype]
    worst = 0.0
    for got, ref, mag in ((dW, rW, mW), (db, rb, mb)):
        err = (got - ref).abs()
        assert not err[mag == 0].any()
        worst = max(worst, float((err / (u * mag.clamp_min(1e-300))).max()))
    c = (WG_C_POS if data == 'positive' else WG_C)[dtype]
    print(f'wgrad {dtype} rows={rows} {rng_name} {data}: worst |err| / (u |A|^T|dY|) = {worst:.3g} (bound {c})')
    assert worst <= c


# ---- 2. dqmc_wf_vjp_params end to end ----------------------------------------------------------------------------------------
E2E_TOL64 = 1e-9
E2E_ATOL64 = 1e-12
# fp64: measured worst (H100) 0.017 of the bound (PauliNet, C5); fp32: 0.43 of the bound (Psiformer, H7 doublet).
# fp32: per array err <= max(E2E_C32 * err of the fp32 CPU autograd, E2E_FLOOR32 u max|ref|) and err <= E2E_CAP32 max|ref|.  The
# floor carries the arrays the fp32 CPU evaluation happens to get nearly exact: PauliNet's Jastrow output layer on the H7
# doublet was measured at 138 u max|ref| with a CPU error of 3 u.
E2E_C32, E2E_FLOOR32, E2E_CAP32 = 16.0, 512.0, 2e-3


@pytest.mark.parametrize('kind,system', _cases(SYSTEMS))
def test_vjp_params_fp64_against_autograd(kind, system):
    B = 2 if system == 'C5' else 3
    eng, spec, params, r, R = _setup(system, kind, 'float64', B)
    w = torch.as_tensor(np.random.default_rng(3).normal(size=B))
    s, l, g = _vjp(eng, r, R, w)
    rs, rl, ref = log_psi_grads(spec, params, r, R, w)
    assert torch.equal(s, rs)
    assert (l - rl).abs().max() <= 1e-10 * max(1.0, float(rl.abs().max()))
    _assert_unread_zero(g, ref)
    errs = _errors(g, ref)
    top = max(m for _, m in errs.values())
    worst = max(e / (E2E_TOL64 * m + E2E_ATOL64 * top) for e, m in errs.values())
    print(f'vjp fp64 {kind} {system}: worst err / bound = {worst:.3g}')
    for k, (e, m) in errs.items():
        assert e <= E2E_TOL64 * m + E2E_ATOL64 * top, (k, e, m)


@pytest.mark.parametrize('kind,system', _cases(('H4_polarised', 'H7_doublet', 'N2')))
def test_vjp_params_fp32_against_autograd(kind, system):
    B = 3
    eng, spec, params, r, R = _setup(system, kind, 'float32', B)
    w = torch.as_tensor(np.random.default_rng(3).normal(size=B))
    r32, R32, w32 = r.float(), R.float(), w.float()
    s, l, g = _vjp(eng, r32, R32, w32)
    p32 = {k: np.asarray(v, dtype=np.float32) for k, v in params.items()}  # the parameters the fp32 engine holds
    rs, rl, ref = log_psi_grads(spec, p32, r32.double(), R32.double(), w32.double())
    _, _, cpu32 = log_psi_grads(spec, p32, r32, R32, w32, dtype=torch.float32)
    _assert_unread_zero(g, ref)
    floor = _errors(cpu32, ref)
    worst = 0.0
    for k, (e, m) in _errors(g, ref).items():
        bound = min(max(E2E_C32 * floor[k][0], E2E_FLOOR32 * U['float32'] * m), E2E_CAP32 * m)
        worst = max(worst, e / bound if bound else (0.0 if e == 0 else float('inf')))
        assert e <= bound, (k, e, floor[k][0], m)
    print(f'vjp fp32 {kind} {system}: worst err / bound = {worst:.3g}')


def test_vjp_params_full_width_psiformer_n2_fp64():
    """d = 256, L = 4, H = 4, K = 16 (the shipped Psiformer) on N2."""
    eng, spec, params, r, R = _setup('N2', 'psiformer', 'float64', 2, embedding_dim=256, n_layers=4, n_heads=4,
                                     n_determinants=16)
    w = torch.tensor([0.7, -1.3], dtype=torch.float64)
    s, l, g = _vjp(eng, r, R, w)
    rs, rl, ref = log_psi_grads(spec, params, r, R, w)
    assert torch.equal(s, rs)
    errs = _errors(g, ref)
    top = max(m for _, m in errs.values())
    for k, (e, m) in errs.items():
        assert e <= E2E_TOL64 * m + E2E_ATOL64 * top, (k, e, m)


# ---- 3. cotangent properties -------------------------------------------------------------------------------------------------
PROP_CASES = [('psiformer', 'H7_polarised'), ('psiformer', 'N2'), ('transpsiformer', 'H4_polarised'),
              ('ferminet', 'H7_doublet'), ('paulinet', 'H4_polarised')]


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('kind,system', PROP_CASES)
def test_vjp_params_cotangent_properties(kind, system, dtype):
    """All-zero weights give exactly zero; twice the weights give twice the gradient; a one-hot weight over B walkers gives the
    gradient of that walker alone (the B = 1 run); sign and log agree with the plain forward.  The parameter gradients are
    atomic sums over walkers and determinants, whose order varies from run to run, so 'twice' and 'one-hot' hold to the
    round-off of that order: 1e-12 (fp64) / 1e-5 (fp32) of each array's largest entry, the bound of the chunking test."""
    tol = {'float64': 1e-12, 'float32': 1e-5}[dtype]
    B = 5
    eng, spec, params, r, R = _setup(system, kind, dtype, B)
    dt = eng.dtype
    r, R = r.to(dt), R.to(dt)
    w = torch.as_tensor(np.random.default_rng(5).normal(size=B)).to(dt)
    s, l, g = _vjp(eng, r, R, w)
    s0, l0, g0 = _vjp(eng, r, R, torch.zeros(B, dtype=dt))
    assert torch.equal(s, s0) and torch.equal(l, l0)
    for k, v in g0.items():
        assert not v.any(), f'{k}: zero cotangent, nonzero gradient'
    amax = lambda t: float(t.abs().max()) if t.numel() else 0.0
    _, _, g2 = _vjp(eng, r, R, 2 * w)
    for k, v in g.items():
        assert amax(g2[k] - 2 * v) <= 2 * tol * amax(v), k
    fs, fl = eng.wf_forward(r.to(DEV), R.to(DEV))
    fs, fl = fs.cpu().double(), fl.cpu().double()
    if dtype == 'float64':
        assert torch.equal(s, fs)
        assert float((l - fl).abs().max()) <= 1e-10 * max(1.0, float(l.abs().max()))
    # fp32: not compared.  On these unequilibrated walkers the fp32 plain forward disagrees with the fp64 engine by more than
    # 2e-3 in log|psi| (or in sign) on every walker of the Psiformer H7-polarised / N2 and TransPsiformer H4 cases, so there is
    # no well-conditioned walker to hold the reverse pass to; that forward disagreement is left for the forward pins.
    b = 3
    oh = torch.zeros(B, dtype=dt)
    oh[b] = 1
    _, _, gb = _vjp(eng, r, R, oh)
    _, _, g1 = _vjp(eng, r[b:b + 1], R, torch.ones(1, dtype=dt))
    for k, v in g1.items():
        assert amax(gb[k] - v) <= tol * amax(v), k


def test_grad_positions_walker_isolation():
    """grad_positions of finite walkers does not change when their neighbours hold nan or inf positions."""
    eng, spec, params, r, R = _setup('H7_polarised', 'psiformer', 'float64', 6)
    r = r.to(DEV)
    s, l, gr, gR = eng.grad_positions(r, R.to(DEV))
    bad = r.clone()
    bad[1, 0, 0] = float('nan')
    bad[4, 2, 1] = float('inf')
    s2, l2, gr2, gR2 = eng.grad_positions(bad, R.to(DEV))
    for b in (0, 2, 3, 5):
        assert torch.equal(gr[b], gr2[b]) and torch.equal(gR[b], gR2[b]) and s[b] == s2[b] and l[b] == l2[b], b


# ---- 4. FermiNet at batch sizes whose edge rows pass 1M, fp32 against the fp64 engine ------------------------------------------
# Unequilibrated random walkers include some near a node or with near-singular orbital matrices, where fp32 log|psi| and its
# derivatives are off by orders more than elsewhere; with all-positive weights those few walkers dominate the sum.  The
# cotangent is therefore zero on walkers whose fp32 log|psi| differs from fp64 by more than 1e-4 (or in sign), so that what is
# compared is the reduction over the >1M edge rows.  Per array max |g32 - g64| <= LB_C max|g64|; measured worst on an H100
# beside it.
LB_C = {'positive': 1e-3, 'training': 1e-3}  # measured worst 2.6e-4 (C5, training cotangent)


@pytest.mark.parametrize('weights', ['positive', 'training'])
@pytest.mark.parametrize('system,B', [('N2', 7600), ('C5', 2400)])
def test_vjp_params_ferminet_large_batch_fp32(system, B, weights):
    mol = SYSTEMS[system]()
    hamil = MolecularHamiltonian(mol=mol)
    N = hamil.n_up + hamil.n_down
    assert B * N * N > 1 << 20
    a64 = B200Ansatz(hamil, 'ferminet', dtype='float64')
    a32 = B200Ansatz(hamil, 'ferminet', dtype='float32', gemm_backend=1)
    params = PN.perturb_params(a64.init(0))
    rng = np.random.default_rng(7)
    r = torch.as_tensor(mol.coords[rng.integers(0, len(mol.coords), size=(B, N))] + rng.normal(size=(B, N, 3)))
    R = torch.as_tensor(mol.coords)
    e64, e32 = a64.engine_for(hamil, params), a32.engine_for(hamil, params)
    if weights == 'positive':
        w = torch.full((B,), 1.0 / B, dtype=torch.float64)
    else:  # (E_loc - <E>) / B with E_loc of the fp64 engine
        from deepqmc_b200.types import PhysicalConfiguration

        E, _ = hamil.local_energy(a64.apply)(None, params, PhysicalConfiguration(R.to(DEV), r.to(DEV), torch.zeros(B, device=DEV)))
        E = E.cpu().double()
        w = (E - E.mean()) / B
    s64, l64, _ = _vjp(e64, r, R, torch.zeros(B, dtype=torch.float64))
    s32, l32, _ = _vjp(e32, r.float(), R.float(), torch.zeros(B, dtype=torch.float32))
    good = (s64 == s32) & ((l64 - l32).abs() <= 1e-4)
    assert int(good.sum()) * N * N > 1 << 20, int(good.sum())  # the rows that carry a cotangent still pass 1M
    w = torch.where(good, w, torch.zeros_like(w))
    _, _, g64 = _vjp(e64, r, R, w)
    _, _, g32 = _vjp(e32, r.float(), R.float(), w.float())
    # several uneven chunks: a workspace for a third of the batch plus a few walkers
    _, _, g32c = _vjp(e32, r.float(), R.float(), w.float(), max_ws_bytes=e32.workspace_bytes(B // 3 + 7, MODE_VJP))
    worst = 0.0
    for k, v in g64.items():
        m = float(v.abs().max())
        for gg in (g32, g32c):
            e = float((gg[k] - v).abs().max())
            worst = max(worst, e / m if m else (0.0 if e == 0 else float('inf')))
            assert e <= LB_C[weights] * m, (k, e, m)
    print(f'ferminet large batch {system} B={B} {weights} ({int(good.sum())} walkers): worst max|g32 - g64| / max|g64| = {worst:.3g}')
