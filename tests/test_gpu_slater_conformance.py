"""GPU: the determinant tail kernel by kernel, against the fp64 restatement of tests/slater_reference.py (itself checked against
autograd by tests/test_slater_reference.py):
- the Slater determinants through dqmc_debug_slater (the engine's own backflow activation and dispatch): slater_small_kernel
  at every NS, slater_fwd2_kernel at every NM instance (exact and padded), slater_fwd_reg_kernel (naturally and through
  DQMC_SLATER_FWD1) and slater_kernel (past 32 electrons, through DQMC_SLATER_GENERIC, the forward-Laplacian pass, the
  additive backflow branch); fp32 and fp64; K = 1, 3, 16, 32; n_up = n_down, n_down + 1 and n_down = 0; one envelope term
  per nucleus (Psiformer), three (TransPsiformer) and PauliNet's per-shell, spin-factorised tables with the default mult_act;
  one walker, a few, and many walkers per persistent block;
- input classes: walkers near the nuclei; orbital matrices of prescribed condition number; electron rows scaled by 2^k,
  k in [-100, 100] (pivots either side of LogProd's 1e+-30 range); odd and even row orders and tied pivot candidates (the
  parity of each variant); exactly singular matrices (slogdet's sign 0, log -inf); forward-Laplacian tangents dense,
  electron-structured and scaled by 1e+-3;
- the determinant sum through dqmc_debug_det_sum: logs spread over +-80, designed cancellation |sum| / sum |.| down to 1e-6,
  hk.Linear weights with negative entries, singular determinants among finite ones and all of them singular;
- bitwise: repeated runs, and walker isolation (a walker with nan / inf positions or backflow rows leaves the others' outputs
  unchanged).

Errors are taken per walker and determinant, relative to the rms of the fp64 reference over the case; they are bounded as
multiples of what the same reference evaluated in fp32 on the CPU gets wrong, plus a small floor, and by an absolute cap per
kernel.  The factors were measured on an H100 80GB HBM3 at 700 W power limit; each constant's comment gives the worst measured
value and the margin."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from deepqmc_b200 import params as PN
from deepqmc_b200.ansatz import B200Ansatz
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from slater_reference import TailParams, det_sum_ref, orbitals, slater_ref
from test_gpu_tc_conformance import _molecule

DEV = 'cuda:0'
SWITCHES = ('DQMC_SLATER_GENERIC', 'DQMC_SLATER_FWD1', 'DQMC_NSMS')

# (rms factor, max factor, absolute cap on the max relative error) per kernel: measured worst values in the comments.
FACTORS = {
    # thread-per-determinant registers, fp32: measured worst 20.3 (rms) / 25.2 (max), both the Laplacian of tangents scaled by
    # 1e3 (the fp32 restatement rounds the same products in another order); largest relative error 4.3e-4; margin about 2x
    'slater_small_kernel': (40.0, 50.0, 1e-3),
    # ex2.approx envelopes, rcp.approx pivots, LogProd: measured worst 4.05 / 7.41, 4.5e-4 (N = 30, 64 walkers); margin 2x
    'slater_fwd2_kernel': (8.0, 15.0, 1e-3),
    # measured worst 2.84 / 4.44 (PauliNet N = 10 through DQMC_SLATER_FWD1), 1.4e-5; margin about 2x
    'slater_fwd_reg_kernel': (6.0, 9.0, 5e-5),
    # warp Gauss-Jordan: measured worst 4.53 / 4.86 (PauliNet N = 8 Laplacian), 2.4e-4; margin about 2x
    'slater_kernel': (9.0, 10.0, 5e-4),
    # determinant sum: measured worst 1.54 / 2.57 above the floor; margin about 2x.  The cap is scaled by max(1, 1e-2 / cancel)
    # (fp32's rounding of the terms over |sum| / sum |.|): measured 1.6e-5 down to cancellation 1e-2, 1.4e-3 at 1e-4, 0.25 at 1e-6
    'finalize_kernel': (3.5, 5.5, 5e-5),
}
FLOOR = 1e-6  # relative; far below any fp32 error of these cases
# fp64 engines: max relative error <= FP64_FACTOR * kappa * 2^-52 + FP64_FLOOR, kappa the largest condition number of the case;
# measured worst 0.57 kappa eps (small kernel gradient), largest relative error 4.1e-8 (kappa 1e10); margin about 2x
FP64_FACTOR, FP64_FLOOR = 1.2, 1e-13

_ENGINES = {}


def _mol(N, n_down=None):
    """A chain with N electrons: n_up = n_down (even N) or n_down + 1 (odd N); n_down = 0: N hydrogens, fully polarised."""
    if n_down == 0:
        return Molecule(coords=[[1.6 * i, 0.2 * (i % 2), 0.0] for i in range(N)], charges=[1] * N, charge=0, spin=N)
    return _molecule(N)


def _engine(N, dtype='float32', kind='psiformer', n_down=None, env=(), conf_w=None, **hyper):
    """Engine per configuration (cached); env: switches set only around its creation (every other switch unset)."""
    key = (N, dtype, kind, n_down, tuple(env), conf_w, tuple(sorted(hyper.items())))
    if key not in _ENGINES:
        m = Molecule.from_name(N) if isinstance(N, str) else _mol(N, n_down)
        hamil = MolecularHamiltonian(mol=m)
        if kind in ('psiformer', 'transpsiformer'):
            hyper = dict(dict(embedding_dim=32, n_layers=1, n_heads=2), **hyper)
        mp = pytest.MonkeyPatch()
        for k in SWITCHES:
            mp.delenv(k, raising=False)
        for k, v in env:
            mp.setenv(k, str(v))
        try:
            a = B200Ansatz(hamil, kind, dtype=dtype, gemm_backend=0, **hyper)
            params = PN.perturb_params(a.init(0))
            if conf_w is not None:
                import numpy as np
                params[PN.CONF + ':w'] = np.asarray(conf_w, dtype=np.float64).reshape(-1, 1)
            eng = a.engine_for(hamil, params)
        finally:
            mp.undo()
        _ENGINES[key] = eng
    return _ENGINES[key]


def _expect(eng, S, env=()):
    """The kernel (and template instance) the engine's dispatch must pick, restated from its rules."""
    sp, env = eng.spec, dict(env)
    N, K, M = sp.n_elec, sp.n_determinants, sp.n_nuc
    f32 = eng.dtype == torch.float32
    add = sp.backflow_transform != 'mult'
    generic = 'DQMC_SLATER_GENERIC' in env
    if (N <= 4 or (N <= 6 and f32)) and not add and not generic:
        return f'slater_small_kernel<{min(N, 6)}>'
    size = 4 if f32 else 8
    smem = size * (((K * N * (N | 1) + 3) & ~3) + 2 * M * ((N + 7) & ~7))
    if S == 1 and N <= 32 and not add and not generic:
        if smem <= 110 * 1024 and 'DQMC_SLATER_FWD1' not in env:
            nm = 14 if N == 14 else 16 if N <= 16 else 28 if N == 28 else 30 if N == 30 else 32
            return f'slater_fwd2_kernel<{nm}>'
        return 'slater_fwd_reg_kernel'
    return 'slater_kernel'


# ---- inputs ----------------------------------------------------------------------------------------------------------------

def _walkers(eng, B, g):
    """Electrons near the nuclei: a random nucleus plus N(0, 0.7^2) per coordinate."""
    R = torch.as_tensor(eng.hamil.mol.coords, dtype=torch.float64)
    N = eng.spec.n_elec
    idx = torch.randint(0, R.shape[0], (B, N), generator=g)
    return (R[idx] + 0.7 * torch.randn(B, N, 3, generator=g, dtype=torch.float64)).to(eng.dtype)


def _bfw(eng):
    sp = eng.spec
    return sp.n_determinants * sp.n_elec * (2 if sp.backflow_transform == 'both' else 1)


def _conditioned(eng, r, kappa, g):
    """Backflow rows (S = 1) for which A = env (x) bf is U diag(sigma) V^T per walker and determinant, sigma log-spaced from 1 to
    1 / kappa (identity mult_act, multiplicative branch, full determinants)."""
    sp = eng.spec
    B, N, K = r.shape[0], sp.n_elec, sp.n_determinants
    P = TailParams.of_engine(eng).to(torch.float64)
    from slater_reference import envelopes

    env = envelopes(r.double().cpu(), P)                                     # [B, K, N, N]
    U = torch.linalg.qr(torch.randn(B, K, N, N, generator=g, dtype=torch.float64))[0]
    V = torch.linalg.qr(torch.randn(B, K, N, N, generator=g, dtype=torch.float64))[0]
    sig = torch.logspace(0, -math.log10(kappa), N, dtype=torch.float64)
    A = U @ torch.diag_embed(sig.expand(B, K, N)) @ V.transpose(-1, -2)
    A = A * (N ** 0.5)  # O(1) entries
    bf = (A / env).permute(0, 2, 1, 3).reshape(B * N, K * N)
    return bf.to(eng.dtype)


def _bf_rows(eng, r, S, inp, g):
    """Backflow slot rows [B N S][BFW] of class `inp` (N(0, 1) values; tangents dense, electron-structured or scaled)."""
    sp = eng.spec
    B, N = r.shape[0], sp.n_elec
    x = torch.randn(B, N, S, _bfw(eng), generator=g, dtype=torch.float64)
    if S > 1:
        if inp == 'electron':
            x[:, :, 1:S - 1] *= (torch.arange(N)[:, None] == torch.arange(S - 2)[None, :] // 3)[None, :, :, None]
        elif inp in ('big', 'small'):
            sc = 1e3 if inp == 'big' else 1e-3
            x[:, :, 1:S - 1] *= sc
            x[:, :, S - 1] *= sc ** 2
        elif inp.startswith('kappa'):
            x[:, :, 0] = _conditioned(eng, r, float(inp[5:]), g).double().reshape(B, N, -1)
    elif inp.startswith('kappa'):
        return _conditioned(eng, r, float(inp[5:]), g)
    return x.reshape(B * N * S, -1).to(eng.dtype)


# ---- comparison ------------------------------------------------------------------------------------------------------------

def _run(eng, r, BF, S):
    """Two runs of the hook: bitwise equal, and the caller's rows untouched."""
    r, BF = r.to(DEV), BF.to(DEV)
    keep = BF.clone()
    out = eng.debug_slater(r, BF, S)
    out2 = eng.debug_slater(r, BF, S)
    torch.cuda.synchronize()
    bits = torch.int64 if BF.dtype == torch.float64 else torch.int32
    assert torch.equal(BF.view(bits), keep.view(bits))
    for a, b in zip(out[:4], out2[:4]):
        assert a is None or torch.equal(a.nan_to_num(), b.nan_to_num())
    return out


def _rel_errors(out, ref, ref32):
    """(rms, max, rms32, max32) of |out - ref| and |ref32 - ref| over the rms of ref."""
    o, r, r32 = out.double().cpu(), ref.double().cpu(), ref32.double().cpu()
    scale = r.pow(2).mean().sqrt().clamp_min(1e-300)
    e, e32 = (o - r).abs() / scale, (r32 - r).abs() / scale
    return e.pow(2).mean().sqrt().item(), e.max().item(), e32.pow(2).mean().sqrt().item(), e32.max().item()


def _assert_close(tag, kernel, res, cap_scale=1.0):
    print(f'measured {tag} {kernel}: ' + '; '.join(
        f'{c} rms {r:.2e} ({r / max(r32, 1e-300):.2f}x fp32) max {m:.2e} ({m / max(m32, 1e-300):.2f}x fp32)'
        for c, (r, m, r32, m32) in res.items()))
    f_rms, f_max, cap = FACTORS[kernel.split('<')[0]]
    cap *= cap_scale
    for c, (r, m, r32, m32) in res.items():
        assert r <= f_rms * r32 + FLOOR and m <= f_max * m32 + FLOOR and m <= cap, (tag, kernel, c, r, m, r32, m32)


def _assert_fp64(tag, kernel, res, kappa):
    bound = FP64_FACTOR * kappa * 2.0 ** -52 + FP64_FLOOR
    print(f'measured {tag} {kernel} (fp64, kappa {kappa:.1e}): ' + '; '.join(
        f'{c} max {m:.2e} ({m / (kappa * 2.0 ** -52):.2f}x kappa eps)' for c, (_, m, _, _) in res.items()))
    for c, (_, m, _, _) in res.items():
        assert m <= bound, (tag, kernel, c, m, bound)


def _check(eng, r, BF, S, tag, env=(), expect=None):
    """Run the hook, assert the kernel, and compare sign / log (/ grad / lap) with fp64 and the fp32 CPU yardstick."""
    sign, log, grad, lap, kernel = _run(eng, r, BF, S)
    assert kernel == (expect or _expect(eng, S, env)), (kernel, expect or _expect(eng, S, env))
    P = TailParams.of_engine(eng)
    ref = slater_ref(r.cpu(), BF.cpu(), P, S)
    A = orbitals(r.cpu().double(), BF.cpu().double().reshape(r.shape[0], r.shape[1], S, -1)[:, :, 0], P.to(torch.float64))
    kappa = torch.linalg.cond(A)
    # the sign is fixed wherever fp32 rounding of A cannot move the determinant through zero
    ok = kappa * 2.0 ** -24 < 0.1 if eng.dtype == torch.float32 else kappa * 2.0 ** -52 < 0.1
    assert torch.equal(sign.cpu()[ok], ref[0].to(sign.dtype)[ok]), (tag, kernel)
    assert torch.isfinite(log).all()
    pairs = [('log', log, ref[1])] + ([('grad', grad, ref[2]), ('lap', lap, ref[3])] if S > 1 else [])
    if eng.dtype == torch.float64:
        _assert_fp64(tag, kernel, {c: _rel_errors(o, rf, rf) for c, o, rf in pairs}, kappa.max().item())
        return kernel
    ref32 = slater_ref(r.cpu(), BF.cpu(), P.to(torch.float32), S, dtype=torch.float32)
    r32 = [ref32[1]] + ([ref32[2], ref32[3]] if S > 1 else [])
    _assert_close(tag, kernel, {c: _rel_errors(o, rf, x) for (c, o, rf), x in zip(pairs, r32)})
    return kernel


def _case(N, dtype='float32', S1=True, inp='walker', B=4, env=(), seed=0, expect=None, **eng_kw):
    eng = _engine(N, dtype, env=env, **eng_kw)
    n = eng.spec.n_elec
    S = 1 if S1 else 3 * n + 2
    g = torch.Generator().manual_seed(1000 * n + 17 * B + seed)
    r = _walkers(eng, B, g)
    BF = _bf_rows(eng, r, S, 'dense' if inp == 'walker' else inp, g)
    return _check(eng, r, BF, S, f'N={n} {dtype} S={S} {inp} B={B} {dict(env)} {eng_kw}', env, expect)


# ---- plain forward (S = 1) -------------------------------------------------------------------------------------------------

N_F32 = [2, 3, 4, 5, 6, 7, 8, 13, 14, 15, 16, 17, 24, 27, 28, 29, 30, 31, 32, 33, 40, 43]
N_F64 = [2, 3, 4, 5, 14, 16, 28, 29, 30, 31, 33]


@pytest.mark.parametrize('inp', ['walker', 'kappa10', 'kappa1e3', 'kappa1e5'])
@pytest.mark.parametrize('N', N_F32)
def test_slater_forward_fp32_matches_fp64(N, inp):
    """fp32, K = 16: slater_small_kernel<NS> (N <= 6), slater_fwd2_kernel at every instance, exact (14, 28, 30, 32) and padded
    (7, 8, 13, 15, 16 -> <16>; 17, 24, 27, 29, 31 -> <32>), slater_kernel past 32 electrons; walkers near the nuclei and
    orbital matrices of condition number 10, 1e3 and 1e5."""
    _case(N, inp=inp)


@pytest.mark.parametrize('inp', ['walker', 'kappa1e5', 'kappa1e10'])
@pytest.mark.parametrize('N', N_F64)
def test_slater_forward_fp64_matches_fp64(N, inp):
    """fp64, K = 16: small at N <= 4; fwd2 up to N = 29 (its shared memory fits); slater_fwd_reg_kernel at N = 30, 31 where it
    does not; slater_kernel past 32; condition numbers up to 1e10."""
    _case(N, 'float64', inp=inp)


@pytest.mark.parametrize('env,N,dtype', [
    ((('DQMC_SLATER_FWD1', 1),), 9, 'float32'), ((('DQMC_SLATER_FWD1', 1),), 32, 'float32'),
    ((('DQMC_SLATER_FWD1', 1),), 13, 'float64'),
    ((('DQMC_SLATER_GENERIC', 1),), 3, 'float32'), ((('DQMC_SLATER_GENERIC', 1),), 6, 'float32'),
    ((('DQMC_SLATER_GENERIC', 1),), 12, 'float32'), ((('DQMC_SLATER_GENERIC', 1),), 4, 'float64'),
])
def test_slater_forward_switches_match_fp64(env, N, dtype):
    """slater_fwd_reg_kernel through DQMC_SLATER_FWD1 and slater_kernel at small N through DQMC_SLATER_GENERIC."""
    _case(N, dtype, env=env)
    _case(N, dtype, env=env, inp='kappa1e3', seed=1)


@pytest.mark.parametrize('case', [
    dict(N=4, n_down=0), dict(N=6, n_down=0), dict(N=7, n_down=0), dict(N=4, n_down=0, dtype='float64'),
    dict(N=7, n_down=0, env=(('DQMC_SLATER_FWD1', 1),)), dict(N=7, n_down=0, env=(('DQMC_SLATER_GENERIC', 1),)),
    dict(N=5, n_determinants=1), dict(N=17, n_determinants=1), dict(N=30, n_determinants=3), dict(N=9, n_determinants=3),
    dict(N=40, n_determinants=3), dict(N=32, n_determinants=32), dict(N=12, n_determinants=32),
    dict(N='LiH', kind='transpsiformer'), dict(N=17, kind='transpsiformer'), dict(N=5, kind='transpsiformer', dtype='float64'),
    dict(N='LiH', kind='paulinet'), dict(N=10, kind='paulinet'), dict(N=9, kind='paulinet', dtype='float64'),
    dict(N=10, kind='paulinet', env=(('DQMC_SLATER_FWD1', 1),)), dict(N=10, kind='paulinet', env=(('DQMC_SLATER_GENERIC', 1),)),
], ids=lambda c: '-'.join(f'{k}={v}' for k, v in c.items() if k != 'env') + ('-' + c['env'][0][0][12:] if 'env' in c else ''))
def test_slater_forward_spins_kinds_match_fp64(case):
    """n_down = 0 (fully polarised hydrogen chains: the fwd2 distance panel of an empty spin block), K = 1, 3 and 32 (K not a
    multiple of the warps per block; K = 32 at N = 32 no longer fits fwd2), three envelope terms per nucleus (TransPsiformer),
    PauliNet's per-shell spin-factorised tables with the default mult_act (fwd2, fwd_reg and slater_kernel zero the
    spin-off-diagonal blocks)."""
    case = dict(case)
    N, dtype = case.pop('N'), case.pop('dtype', 'float32')
    env = case.pop('env', ())
    _case(N, dtype, env=env, **case)


@pytest.mark.parametrize('B', [1, 3, 64])
@pytest.mark.parametrize('N', [8, 30])
def test_slater_fwd2_persistent_walker_loop(N, B):
    """slater_fwd2_kernel on an engine created with DQMC_NSMS=2 (a grid of 6 blocks): one walker, a few, and ten or more walkers
    per persistent block."""
    _case(N, B=B, env=(('DQMC_NSMS', 2),))


# ---- edges: scaled rows, row orders and ties, exact singularity ------------------------------------------------------------

VARIANTS = {  # (N, dtype, env) reaching each kernel
    'small': (5, 'float32', ()), 'small64': (3, 'float64', ()),
    'fwd2': (9, 'float32', ()), 'fwd2_30': (30, 'float32', ()),
    'fwd_reg': (30, 'float64', ()), 'fwd_reg1': (11, 'float32', (('DQMC_SLATER_FWD1', 1),)),
    'generic': (8, 'float32', (('DQMC_SLATER_GENERIC', 1),)), 'generic40': (40, 'float32', ()),
}


def _variant(name):
    N, dtype, env = VARIANTS[name]
    return _engine(N, dtype, env=env), env


@pytest.mark.parametrize('variant', list(VARIANTS))
def test_slater_scaled_rows_match_fp64(variant):
    """Electron rows multiplied by 2^k, k spread over [-100, 100] (N distinct values per walker, in random order): pivots far
    outside (1e-30, 1e30), every value of the elimination still normal (LogProd<float>'s mantissa / exponent split and its
    plain-log path).  The
    unscaled matrix is N I + N(0, 1) with its rows ordered like the scales, so partial pivoting on the scaled rows eliminates in a
    stable order: the comparison sees the log of the pivot product, not the growth of an unstable elimination order."""
    eng, env = _variant(variant)
    sp = eng.spec
    N, K, B = sp.n_elec, sp.n_determinants, 3
    g = torch.Generator().manual_seed(N + 5)
    r = _walkers(eng, B, g)
    # walker b: 2^(o_b + j), o_b = -70, 0, 70 and j over [-30, 30]: pivots from 2^-100 to 2^100, while the multipliers of the
    # elimination (ratios of row scales, down to 2^-60 / N) stay normal in fp32
    k = torch.stack([o + torch.linspace(-30, 30, N)[torch.randperm(N, generator=g)].round() for o in (-70, 0, 70)])  # [B, N]
    A = N * torch.eye(N, dtype=torch.float64) + torch.randn(B, K, N, N, generator=g, dtype=torch.float64)
    order = torch.argsort(-k, dim=1)  # order[b, j]: the row with the j-th largest scale pivots column j
    A = torch.zeros_like(A).scatter_(2, order[:, None, :, None].expand(B, K, N, N), A)
    from slater_reference import envelopes

    e = envelopes(r.double(), TailParams.of_engine(eng).to(torch.float64))
    BF = (A / e * torch.exp2(k.double())[:, None, :, None]).permute(0, 2, 1, 3).reshape(B * N, K * N).to(eng.dtype)
    _check(eng, r, BF, 1, f'{variant} scaled rows', env)


@pytest.mark.parametrize('variant', list(VARIANTS))
def test_slater_row_orders_and_ties(variant):
    """Walkers whose electrons are permuted within a spin block (odd and even permutations: the determinant's sign follows the
    parity) and walkers with several electrons at one position whose first orbital column holds +-1 (pivot candidates of
    equal magnitude): the sign of every variant's pivot-order parity (inversion count, cycle count, explicit swaps)."""
    eng, env = _variant(variant)
    sp = eng.spec
    N, n_up, W = sp.n_elec, sp.n_up, _bfw(eng)
    g = torch.Generator().manual_seed(N + 9)
    r0 = _walkers(eng, 1, g)
    bf0 = torch.randn(N, W, generator=g, dtype=torch.float64).to(eng.dtype)
    rs, bfs = [r0[0]], [bf0]
    for swaps in ([(0, 1)], [(0, 1), (1, 2)], [(n_up - 1, 0)], [(N - 1, n_up)], [(0, 2), (1, n_up - 1), (n_up, N - 1)]):
        perm = list(range(N))
        for a, b in swaps:
            if a != b and (a < n_up) == (b < n_up) and max(a, b) < N:
                perm[a], perm[b] = perm[b], perm[a]
        rs.append(r0[0][perm])
        bfs.append(bf0[perm])
    # ties: the up electrons 0 .. 2 at one position, orbital 0 of every determinant +-1 in their rows
    rt, bt = r0[0].clone(), bf0.clone()
    m = min(3, n_up)
    rt[:m] = rt[0]
    bt[:m, ::N] = torch.tensor([1.0, -1.0, 1.0][:m], dtype=bt.dtype)[:, None]
    rs.append(rt)
    bfs.append(bt)
    r, BF = torch.stack(rs), torch.cat(bfs)
    _check(eng, r, BF, 1, f'{variant} row orders / ties', env)
    sign, log = _run(eng, r, BF, 1)[:2]
    assert (sign[1:6].abs() == 1).all()


@pytest.mark.parametrize('where', ['col0', 'col_mid', 'col_last', 'row'])
@pytest.mark.parametrize('variant', list(VARIANTS))
def test_slater_singular_is_slogdet_convention(variant, where):
    """An exactly zero orbital column (mu = 0, N // 2, N - 1) or electron row in the odd determinants: sign 0 and log -inf for
    those (torch.linalg.slogdet's convention), the even ones unchanged and finite."""
    eng, env = _variant(variant)
    sp = eng.spec
    N, K = sp.n_elec, sp.n_determinants
    B = 2
    g = torch.Generator().manual_seed(N + 13)
    r = _walkers(eng, B, g)
    BF = _bf_rows(eng, r, 1, 'dense', g).reshape(B, N, K, N)
    base_sign, base_log = _run(eng, r, BF.reshape(B * N, -1), 1)[:2]
    odd = torch.arange(K) % 2 == 1
    if where == 'row':
        BF[:, N // 2, odd] = 0
    else:
        BF[:, :, odd, {'col0': 0, 'col_mid': N // 2, 'col_last': N - 1}[where]] = 0
    sign, log, _, _, kernel = _run(eng, r, BF.reshape(B * N, -1), 1)
    assert kernel == _expect(eng, 1, env)
    ref = torch.linalg.slogdet(orbitals(r.cpu().double(), BF.reshape(B, N, -1).cpu().double(),
                                        TailParams.of_engine(eng).to(torch.float64)))
    assert (ref[0][:, odd] == 0).all() and (ref[1][:, odd] == -math.inf).all()
    assert (sign[:, odd] == 0).all(), (kernel, sign)
    assert (log[:, odd] == -math.inf).all(), (kernel, log)
    assert torch.equal(sign[:, ~odd], base_sign[:, ~odd]) and torch.equal(log[:, ~odd], base_log[:, ~odd])


# ---- forward-Laplacian pass (S = 3N + 2) -----------------------------------------------------------------------------------

@pytest.mark.parametrize('N,dtype', [(2, 'float32'), (3, 'float32'), (4, 'float32'), (5, 'float32'), (6, 'float32'),
                                     (2, 'float64'), (3, 'float64'), (4, 'float64'), (5, 'float64'), (8, 'float32'),
                                     (17, 'float32'), (30, 'float32'), (33, 'float32'), (43, 'float32')])
def test_slater_fl_matches_fp64(N, dtype):
    """Forward-Laplacian pass, K = 3: slater_small_kernel at every NS (fp32 2 .. 6, fp64 2 .. 4) and slater_kernel (fp64 N = 5;
    fp32 N = 8, 17, 30, 33, 43), dense tangents."""
    _case(N, dtype, S1=False, B=2 if N < 30 else 1, n_determinants=3)


@pytest.mark.parametrize('inp', ['electron', 'big', 'small', 'kappa1e2', 'kappa1e4'])
@pytest.mark.parametrize('N', [4, 8])
def test_slater_fl_input_classes_match_fp64(N, inp):
    """Electron-structured tangents (tangent t non-zero only in electron t // 3's rows), tangents scaled by 1e3 / 1e-3, and
    orbital matrices of condition number up to 1e4 (small kernel at N = 4, slater_kernel at N = 8)."""
    _case(N, S1=False, inp=inp, B=2, n_determinants=3)


@pytest.mark.parametrize('case', [
    dict(N=4, backflow_transform='add'), dict(N=4, backflow_transform='both'), dict(N=9, backflow_transform='both'),
    dict(N=4, backflow_transform='both', dtype='float64'), dict(N='LiH', kind='paulinet'), dict(N=8, kind='paulinet'),
    dict(N=5, n_down=0), dict(N=3, kind='transpsiformer'),
], ids=lambda c: '-'.join(f'{k}={v}' for k, v in c.items()))
def test_slater_fl_branches_match_fp64(case):
    """The additive backflow branch ('add' and 'both', Psiformer: slater_kernel with the electron factor of
    bf_add_factor_kernel), PauliNet's spin-factorised determinants with the default mult_act (small kernel for LiH,
    slater_kernel at N = 8), n_down = 0, and three envelope terms per nucleus."""
    case = dict(case)
    N, dtype = case.pop('N'), case.pop('dtype', 'float32')
    if case.get('kind') != 'paulinet':
        case.setdefault('n_determinants', 3)
    _case(N, dtype, S1=False, B=2, **case)


# ---- determinant sum -------------------------------------------------------------------------------------------------------

def _det_inputs(eng, B, cancel, g):
    """det_sign / det_log / det_grad / det_lap [B, K(, 3N)] with logs spread over +-80 and, for K > 1, the last determinant set so
    that |sum_k c_k s_k e^l_k| / sum_k |c_k e^l_k| = cancel (computed in fp64 from the rounded values)."""
    sp = eng.spec
    K, T3 = sp.n_determinants, 3 * sp.n_elec
    dt = eng.dtype
    # a cancellation below fp32's resolution of e^l at |l| ~ 80 (ulp 7.6e-6) needs the cancelling terms at small |l|: there the
    # largest log sits in [-1, 1] and the others spread over [-80, -2]
    fine = cancel < 1e-4
    l = torch.rand(B, K, generator=g, dtype=torch.float64) * (78 if fine else 160) - 80
    if fine:
        l[:, 0] = torch.rand(B, generator=g, dtype=torch.float64) * 2 - 1
    s = torch.where(torch.rand(B, K, generator=g) < 0.5, -1.0, 1.0).double()
    c = TailParams.of_engine(eng).conf_w
    c = torch.ones(K, dtype=torch.float64) if c is None else c.cpu().double()
    l = l.to(dt).double()
    if K > 1 and cancel < 1:
        t = c[:-1] * s[:, :-1] * torch.exp(l[:, :-1])
        rest = t.sum(-1)
        # |rest + x| = cancel (|t|.sum() + |x|) with x = c_K s_K e^{l_K} of sign opposite to rest
        x = -(rest + torch.sign(rest) * cancel * t.abs().sum(-1)) / (1 - cancel)
        s[:, -1] = torch.sign(x / c[-1])
        l[:, -1] = torch.log((x / c[-1]).abs()).to(dt).double()
        terms = c * s * torch.exp(l)
        ratio = terms.sum(-1).abs() / terms.abs().sum(-1)
        assert ((ratio > cancel / 3) & (ratio < cancel * 3)).all(), ratio  # the rounded inputs still cancel as designed
    grad = torch.randn(B, K, T3, generator=g, dtype=torch.float64)
    lap = torch.randn(B, K, generator=g, dtype=torch.float64) * 3
    return s.to(dt), l.to(dt), grad.to(dt), lap.to(dt)


def _check_det_sum(eng, r, s, l, gr, lp, tag):
    outs = [eng.debug_det_sum(r.to(DEV), s.to(DEV), l.to(DEV), gr.to(DEV), lp.to(DEV)) for _ in range(2)]
    torch.cuda.synchronize()
    for a, b in zip(*outs):
        assert torch.equal(a.nan_to_num(), b.nan_to_num())
    sign, log, grad, stats = outs[0]
    conf_w = TailParams.of_engine(eng).conf_w
    ref = det_sum_ref(s, l, gr, lp, conf_w=conf_w)
    kw = dict(conf_w=conf_w.cpu().float() if conf_w is not None else None, dtype=torch.float32)
    ref32 = det_sum_ref(s.float(), l.float(), gr.float(), lp.float(), **kw)
    return (sign, log, grad, stats[4], stats[5]), ref, ref32


@pytest.mark.parametrize('cancel', [1.0, 1e-2, 1e-4, 1e-6])
@pytest.mark.parametrize('K,kind', [(1, 'psiformer'), (2, 'psiformer'), (16, 'psiformer'), (2, 'paulinet'), (16, 'paulinet')])
def test_det_sum_matches_fp64(K, kind, cancel):
    """finalize_kernel (cusp 'none'): SumPool (Psiformer) and hk.Linear weights with negative entries (PauliNet); logs over
    +-80, the sum cancelling to |sum| / sum |.| = cancel."""
    if K == 1 and cancel < 1:
        pytest.skip('one determinant cannot cancel')
    conf_w = None if kind == 'psiformer' else tuple([0.8, -1.3, 0.5, -0.2] * 4)[:K]
    eng = _engine(8, kind=kind, cusp='none', n_determinants=K, conf_w=conf_w)
    B = 32
    g = torch.Generator().manual_seed(K + int(-math.log10(cancel)))
    r = _walkers(eng, B, g)
    s, l, gr, lp = _det_inputs(eng, B, cancel, g)
    out, ref, ref32 = _check_det_sum(eng, r, s, l, gr, lp, f'K={K} {kind} cancel={cancel}')
    sign, log, grad, lap, g2 = out
    if cancel >= 1e-4:  # far from fp32's 2^-24 relative rounding of the terms
        assert torch.equal(sign.cpu(), ref[0].float())
    res = {'log': _rel_errors(log, ref[1], ref32[1]), 'grad': _rel_errors(grad, ref[2], ref32[2]),
           'lap': _rel_errors(lap, ref[3], ref32[3]),
           'g2': _rel_errors(g2, (ref[2] ** 2).sum(-1), (ref32[2] ** 2).sum(-1))}
    _assert_close(f'K={K} {kind} cancel={cancel}', 'finalize_kernel', res, max(1.0, 1e-2 / cancel))


def test_det_sum_singular_determinants():
    """A determinant at (sign 0, log -inf) among finite ones drops out of the sum and its jets; all of them at (0, -inf) give
    log psi = -inf and sign 0."""
    eng = _engine(8, cusp='none', n_determinants=4)
    B = 4
    g = torch.Generator().manual_seed(3)
    r = _walkers(eng, B, g)
    s, l, gr, lp = _det_inputs(eng, B, 1.0, g)
    s[:2, 1], l[:2, 1] = 0, -math.inf
    s[2:], l[2:] = 0, -math.inf
    out, ref, ref32 = _check_det_sum(eng, r, s, l, gr, lp, 'singular')
    sign, log, grad, lap, _ = (t.cpu().double() for t in out)
    assert torch.equal(sign[2:], torch.zeros(2, dtype=torch.float64)) and (log[2:] == -math.inf).all()
    assert torch.equal(sign[:2], ref[0][:2])
    res = {c: _rel_errors(o[:2], rf[:2], x[:2]) for c, o, rf, x in
           (('log', log, ref[1], ref32[1]), ('grad', grad, ref[2], ref32[2]), ('lap', lap, ref[3], ref32[3]))}
    _assert_close('singular among finite', 'finalize_kernel', res)


# ---- walker isolation ------------------------------------------------------------------------------------------------------

ISO_VARIANTS = ['small', 'fwd2', 'fwd2_30', 'fwd_reg', 'fwd_reg1', 'generic', 'generic40', 'fl_small', 'fl_generic', 'fl_add']


@pytest.mark.parametrize('what', ['r', 'bf'])
@pytest.mark.parametrize('case', ['nan', 'inf'])
@pytest.mark.parametrize('variant', ISO_VARIANTS)
def test_slater_walker_isolation_bitwise(variant, case, what):
    """Every other walker's positions or backflow rows set to nan / inf: the kept walkers' outputs are bit for bit those of a
    run without the bad walkers, and every bad walker's log-determinants are non-finite."""
    if variant.startswith('fl_'):
        eng = {'fl_small': lambda: _engine(4, n_determinants=3), 'fl_generic': lambda: _engine(8, n_determinants=3),
               'fl_add': lambda: _engine(4, n_determinants=3, backflow_transform='both')}[variant]()
        S = 3 * eng.spec.n_elec + 2
    else:
        eng, _ = _variant(variant)
        S = 1
    N, walkers = eng.spec.n_elec, 5
    g = torch.Generator().manual_seed(N + 21)
    r = _walkers(eng, walkers, g)
    BF = _bf_rows(eng, r, S, 'dense', g)
    base = _run(eng, r, BF, S)
    bad = torch.arange(walkers) % 2 == 1
    r1, BF1 = r.clone(), BF.clone().reshape(walkers, -1)
    if what == 'r':
        r1[bad] = float(case)
    else:
        BF1[bad] = float(case)
    out = _run(eng, r1, BF1.reshape(BF.shape), S)
    for a, b in zip(base[:4], out[:4]):
        if a is not None:
            assert torch.isfinite(a).all()
            assert torch.equal(b[~bad.to(b.device)], a[~bad.to(a.device)])
    assert not torch.isfinite(out[1][bad.to(DEV)]).any()


@pytest.mark.parametrize('case', ['nan', 'inf'])
def test_det_sum_walker_isolation_bitwise(case):
    """The determinant sum with every other walker's determinant logs and jets set to nan / inf."""
    eng = _engine(8, cusp='none', n_determinants=4)
    B = 6
    g = torch.Generator().manual_seed(5)
    r = _walkers(eng, B, g)
    s, l, gr, lp = _det_inputs(eng, B, 1.0, g)
    base = eng.debug_det_sum(r.to(DEV), s.to(DEV), l.to(DEV), gr.to(DEV), lp.to(DEV))
    bad = torch.arange(B) % 2 == 1
    l1, gr1, lp1 = l.clone(), gr.clone(), lp.clone()
    l1[bad], gr1[bad], lp1[bad] = float(case), float(case), float(case)
    out = eng.debug_det_sum(r.to(DEV), s.to(DEV), l1.to(DEV), gr1.to(DEV), lp1.to(DEV))
    torch.cuda.synchronize()
    keep = ~bad.to(DEV)
    assert torch.equal(out[0][keep], base[0][keep]) and torch.equal(out[1][keep], base[1][keep])
    assert torch.equal(out[2][keep], base[2][keep]) and torch.equal(out[3][:, keep], base[3][:, keep])
    assert not torch.isfinite(out[1][bad.to(DEV)]).any()
