"""GPU: the forward-Laplacian pass (S = 3N + 2 slots per electron: value, 3N tangents, Laplacian) kernel by kernel, against fp64
jets from nested forward-mode AD (tests/tc_reference.py, itself checked against autograd by tests/test_fl_reference.py):
- the forward-Laplacian attention through dqmc_debug_attention with S = 3N + 2: attn_fl_f32_kernel (SIMT and 3xTF32 mma.sync
  variants, every <N, dh> instance, exact and partial 16-row tiles, every tangent-chunk size class), the generic attn_fl_kernel
  with the TransPsiformer's nuclear tokens (SIMT and tensor cores), and its fp64 instance;
- the MLP that follows it through dqmc_debug_mlp: 3xTF32 row GEMMs with the fused tanh-Laplacian epilogue (tiles of whole slot
  groups), row GEMMs + tanh_fl_kernel, and the CUDA-core path of fp64 engines;
- bitwise: repeated runs, and walker isolation (one walker's rows never change another walker's outputs).

Errors are taken per slot class (value, tangents, Laplacian), per walker and head, relative to the rms of the fp64 reference
over that class; they are bounded as multiples of what the same reference evaluated in fp32 on the CPU gets wrong, plus a
small floor, and by an absolute cap per kernel.  The factors were measured on an H100 80GB HBM3 at 700 W power limit; each
constant's comment gives the worst measured value and the margin."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from deepqmc_b200 import params as PN
from deepqmc_b200.ansatz import B200Ansatz
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from tc_reference import attention_fl_ref, mlp_fl_ref, weight
from test_gpu_tc_conformance import _molecule, _qkv

DEV = 'cuda:0'
AB_SWITCHES = ('DQMC_ATTN_FL_MMA', 'DQMC_ATTN_TB', 'DQMC_ATTN_NT', 'DQMC_ATTN_GENERIC', 'DQMC_NO_FUSE_TANH')

# (rms factor, max factor, absolute cap on the max relative error) per kernel / path: measured worst values in the comments.
FACTORS = {
    # SIMT: measured worst 1.48 (rms) / 1.55 (max), largest relative error 1.1e-3 (tangents of near one-hot rows, where the
    # fp32 restatement shows the same); margin about 2x
    'attn_fl_f32_kernel': (3.0, 3.0, 3e-3),
    # 3xTF32 mma.sync tangent chunks (2^-22 representation error per operand against fp32's 2^-24): measured worst 12.7 (rms,
    # Laplacian) / 11.4 (max), 1.1e-3; margin about 2x.  Plain TF32 (a dropped low product) is far beyond.
    'attn_fl_f32_kernel_mma': (25.0, 25.0, 3e-3),
    # generic kernel with nuclear tokens, SIMT: measured worst 1.67 / 1.87, 2.4e-3 (LiH, near one-hot rows); margin about 2x
    'attn_fl_kernel': (3.5, 4.0, 5e-3),
    # ... tensor cores: measured worst 5.27 / 4.59, 2.5e-4; margin about 2.3x
    'attn_fl_kernel_mma': (12.0, 12.0, 1e-3),
    # 3xTF32 row GEMMs with the tanh-Laplacian epilogue: measured worst 9.10 / 9.91, 4.6e-5; margin about 2x
    'gemm_fused_tanh': (18.0, 20.0, 1e-4),
    # ... with tanh_fl_kernel: measured worst 9.02 / 10.2, 4.1e-5; margin about 2x
    'gemm_tanh_fl_kernel': (18.0, 20.0, 1e-4),
}
FLOOR = 1e-6  # relative; far below any fp32 error of these contractions
# fp64 engines (attn_fl_kernel<double>, gemm_kernel + tanh_fl_kernel): cap on the max relative error; measured worst 2.5e-14
FP64_CAP = 1e-12

SLOT_CLASSES = (('value', lambda S: slice(0, 1)), ('tangents', lambda S: slice(1, S - 1)),
                ('laplacian', lambda S: slice(S - 1, S)))
SCALES = {'big': 1e3, 'small': 1e-3}

_ENGINES = {}


def _engine(mol, kind='psiformer', dtype='float32', env=(), **hyper):
    """Engine per configuration (cached); env: A/B switches set only around its creation (every other switch unset)."""
    key = (mol if isinstance(mol, str) else (tuple(mol.charges), tuple(mol.coords.ravel())), kind, dtype, tuple(env),
           tuple(sorted(hyper.items())))
    if key not in _ENGINES:
        m = Molecule.from_name(mol) if isinstance(mol, str) else mol
        hamil = MolecularHamiltonian(mol=m)
        mp = pytest.MonkeyPatch()
        for k in AB_SWITCHES:
            mp.delenv(k, raising=False)
        for k, v in env:
            mp.setenv(k, str(v))
        try:
            a = B200Ansatz(hamil, kind, dtype=dtype, gemm_backend=1 if dtype == 'float32' else 0, **hyper)
            eng = a.engine_for(hamil, PN.perturb_params(a.init(0)))
        finally:
            mp.undo()
        _ENGINES[key] = (hamil, eng)
    return _ENGINES[key]


def _rows(B, N, S, c, g, inp):
    """Slot rows [B N S][c] (row (b N + i) S + s).  dense: N(0, 1) everywhere; electron: tangent t non-zero only in the rows of
    electron t // 3 (first-layer structure); big / small: tangents scaled by 1e3 / 1e-3 and Laplacians by its square relative
    to the values (coordinates rescaled); spread (attention): values as _qkv(spread=True) -- scores up to +-60, |V| up to 2e3."""
    x = torch.randn(B, N, S, c, generator=g)
    if inp == 'electron':
        x[:, :, 1:S - 1] *= (torch.arange(N)[:, None] == torch.arange(S - 2)[None, :] // 3)[None, :, :, None]
    elif inp in SCALES:
        x[:, :, 1:S - 1] *= SCALES[inp]
        x[:, :, S - 1] *= SCALES[inp] ** 2
    elif inp == 'spread':
        x[:, :, 0] = _qkv(B, N, c // 3, g, True).reshape(B, N, c)
    return x.reshape(B * N * S, c)


def _errors(out, ref, ref32, N, S, H):
    """{class: (rms, max, rms32, max32)} of |out - ref| and |ref32 - ref| over the rms of ref per (walker, head, class)."""
    B = out.shape[0] // (N * S)
    o, r, r32 = (t.to(DEV).double().reshape(B, N, S, H, -1) for t in (out, ref, ref32))
    res = {}
    for name, sl in SLOT_CLASSES:
        rc = r[:, :, sl(S)]
        scale = rc.pow(2).mean(dim=(1, 2, 4), keepdim=True).sqrt().clamp_min(1e-300)
        e, e32 = (o[:, :, sl(S)] - rc).abs() / scale, (r32[:, :, sl(S)] - rc).abs() / scale
        res[name] = (e.pow(2).mean().sqrt().item(), e.max().item(), e32.pow(2).mean().sqrt().item(), e32.max().item())
    return res


def _assert_close(tag, kernel, res):
    print(f'measured {tag} {kernel}: ' + '; '.join(
        f'{c} rms {r:.2e} ({r / max(r32, 1e-300):.2f}x fp32) max {m:.2e} ({m / max(m32, 1e-300):.2f}x fp32)'
        for c, (r, m, r32, m32) in res.items()))
    f_rms, f_max, cap = FACTORS[kernel]
    for c, (r, m, r32, m32) in res.items():
        assert r <= f_rms * r32 + FLOOR and m <= f_max * m32 + FLOOR and m <= cap, (tag, kernel, c, r, m, r32, m32)


def _assert_fp64(tag, kernel, res):
    print(f'measured {tag} {kernel} (fp64): ' + '; '.join(f'{c} max {m:.2e}' for c, (_, m, _, _) in res.items()))
    for c, (_, m, _, _) in res.items():
        assert m <= FP64_CAP, (tag, kernel, c, m)


# ---- forward-Laplacian attention ------------------------------------------------------------------------------------------

def _tokens(eng, layer):
    if eng.spec.kind != 'transpsiformer':
        return None, None
    return weight(eng, f'L{layer}.kn'), weight(eng, f'L{layer}.vn')


def _check_attention(eng, QKV, layer, expect, tag):
    N, H = eng.spec.n_elec, eng.spec.n_heads
    S = 3 * N + 2
    O, kernel = eng.debug_attention(layer, QKV, S=S)
    O2, _ = eng.debug_attention(layer, QKV, S=S)
    torch.cuda.synchronize()
    assert kernel == expect, (kernel, expect)
    assert torch.equal(O, O2)  # single writer of every running sum: bitwise reproducible
    assert torch.isfinite(O).all()
    kn, vn = _tokens(eng, layer)
    ref = attention_fl_ref(QKV, N, H, S, kn, vn)
    if eng.dtype == torch.float64:
        _assert_fp64(tag, kernel, _errors(O, ref, ref, N, S, H))
        return
    cpu = lambda t: None if t is None else t.cpu()
    ref32 = attention_fl_ref(QKV.cpu(), N, H, S, cpu(kn), cpu(vn), dtype=torch.float32)
    _assert_close(tag, kernel, _errors(O, ref, ref32, N, S, H))


def _psiformer_attention(N, env, expect, inp='dense', B=2, d=256, H=4, seed=0):
    _, eng = _engine(_molecule(N), env=env, n_layers=1, embedding_dim=d, n_heads=H)
    S = 3 * N + 2
    g = torch.Generator(device='cpu').manual_seed(1000 * N + seed)
    _check_attention(eng, _rows(B, N, S, 3 * d, g, inp).to(DEV), 0, expect, f'N={N} {inp} {dict(env)}')


ATTN_N = [2, 3, 4, 5, 9, 10, 14, 16, 17, 19, 20, 24, 28, 30, 31, 32]
SIMT, MMA = 'attn_fl_f32_kernel', 'attn_fl_f32_kernel_mma'


@pytest.mark.parametrize('mma', [0, 1])
@pytest.mark.parametrize('N', ATTN_N)
def test_fl_attention_every_instance_matches_fp64(N, mma):
    """Psiformer, d = 256, 4 heads of 64: the <N, 64> instances (N = 4, 10, 14, 28, 30) and the runtime-N one, exact and partial
    16-row tiles of the tensor-core variant, either side of its default switch at 20 electrons; both variants forced."""
    _psiformer_attention(N, (('DQMC_ATTN_FL_MMA', mma),), MMA if mma else SIMT)


@pytest.mark.parametrize('inp', ['dense', 'electron'])
def test_fl_attention_past_the_mma_limit_matches_fp64(inp):
    """N = 40 is past the 32 rows of the tensor-core variant: SIMT even when the tensor cores are asked for."""
    _psiformer_attention(40, (('DQMC_ATTN_FL_MMA', 1),), SIMT, inp)


@pytest.mark.parametrize('inp', ['electron', 'big', 'small', 'spread'])
@pytest.mark.parametrize('mma', [0, 1])
@pytest.mark.parametrize('N', [4, 17, 30])
def test_fl_attention_input_ranges_match_fp64(N, mma, inp):
    """First-layer structure (tangent t non-zero only in the rows of electron t // 3), tangent rows 1e3 and 1e-3 times the values (the 3xTF32 split keeps the 8-bit exponent: no range assumption), and near
    one-hot softmax rows (scores up to +-60, |V| up to 2e3)."""
    _psiformer_attention(N, (('DQMC_ATTN_FL_MMA', mma),), MMA if mma else SIMT, inp)


def _chunk_cases():
    cases = []
    for N in (4, 17, 30):
        for mma in (0, 1):
            # 7 divides neither 12 nor 51 (N = 30: the chunk of 7 does not fit the shared memory, 4 leaves a last chunk of 2);
            # all 3N tangents in one chunk fit at N = 4 only
            for tb in {4: (1, 7, 12), 17: (1, 7), 30: (1, 4)}[N]:
                cases.append(pytest.param(N, (('DQMC_ATTN_FL_MMA', mma), ('DQMC_ATTN_TB', tb)), MMA if mma else SIMT,
                                          id=f'{N}-{"mma" if mma else "simt"}-tb{tb}'))
        for nt in (32, 512):
            cases.append(pytest.param(N, (('DQMC_ATTN_FL_MMA', 0), ('DQMC_ATTN_NT', nt)), SIMT, id=f'{N}-simt-nt{nt}'))
    return cases


@pytest.mark.parametrize('N,env,expect', _chunk_cases())
def test_fl_attention_tangent_chunks_match_fp64(N, env, expect):
    """Tangent chunks of one tangent, chunks that leave a short last chunk, and all 3N tangents at once; the SIMT variant with
    32 and 512 threads per block."""
    _psiformer_attention(N, env, expect, 'dense')


@pytest.mark.parametrize('mma', [0, 1])
@pytest.mark.parametrize('d', [128, 192])
def test_fl_attention_runtime_head_dim_matches_fp64(d, mma):
    """The runtime-dh instance attn_fl_f32_kernel<0, 0>: 4 heads of 32 (d = 128) and of 48 (d = 192: three 16-column groups of
    the tensor-core outputs)."""
    _psiformer_attention(10, (('DQMC_ATTN_FL_MMA', mma),), MMA if mma else SIMT, 'dense', d=d, H=4)


TRANS = dict(embedding_dim=128, n_layers=2, n_heads=2, n_determinants=2)


def _trans_mol(name):
    return {'chain20': lambda: _molecule(20, 4), 'N40+8': lambda: _molecule(40, 8)}.get(name, lambda: name)()


@pytest.mark.parametrize('inp', ['dense', 'spread'])
@pytest.mark.parametrize('mol,expect', [('LiH', 'attn_fl_kernel'), ('chain20', 'attn_fl_kernel_mma'),
                                        ('cyclobutadiene_square', 'attn_fl_kernel_mma'), ('N40+8', 'attn_fl_kernel_mma')])
def test_fl_attention_generic_nuclear_tokens_match_fp64(mol, expect, inp):
    """Generic attn_fl_kernel with the TransPsiformer's nuclear key / value tokens (d = 128, 2 heads), both layers: LiH (4 + 2
    keys, SIMT), 20 electrons on 4 nuclei (the default switch to the tensor cores), cyclobutadiene (28 + 8), 40 electrons on 8
    nuclei (tensor cores past 32 electrons)."""
    hamil, eng = _engine(_trans_mol(mol), 'transpsiformer', **TRANS)
    N = eng.spec.n_elec
    S = 3 * N + 2
    g = torch.Generator(device='cpu').manual_seed(N + 7)
    QKV = _rows(2, N, S, 384, g, inp).to(DEV)
    for layer in range(2):
        _check_attention(eng, QKV, layer, expect, f'{mol} L{layer} {inp}')


@pytest.mark.parametrize('mma', [0, 1])
def test_fl_attention_generic_psiformer_matches_fp64(mma):
    """Psiformer with DQMC_ATTN_GENERIC=1 at N = 30: the generic kernel without tokens, SIMT and tensor cores."""
    _psiformer_attention(30, (('DQMC_ATTN_FL_MMA', mma), ('DQMC_ATTN_GENERIC', 1)),
                         'attn_fl_kernel_mma' if mma else 'attn_fl_kernel', 'dense')


@pytest.mark.parametrize('mol', [4, 17, 30, 'LiH', 'cyclobutadiene_square'])
def test_fl_attention_fp64_matches_fp64(mol):
    """fp64 engines (attn_fl_kernel<double>): Psiformer N = 4, 17, 30 (d = 256) and the TransPsiformer with tokens."""
    if isinstance(mol, int):
        _, eng = _engine(_molecule(mol), dtype='float64', n_layers=1)
        layers = (0,)
    else:
        _, eng = _engine(mol, 'transpsiformer', dtype='float64', **TRANS)
        layers = (0, 1)
    N, d = eng.spec.n_elec, eng.spec.embedding_dim
    g = torch.Generator(device='cpu').manual_seed(N + 64)
    QKV = _rows(2, N, 3 * N + 2, 3 * d, g, 'dense').double().to(DEV)
    for layer in layers:
        _check_attention(eng, QKV, layer, 'attn_fl_kernel', f'{mol} L{layer}')


# ---- the MLP after the attention -------------------------------------------------------------------------------------------

def _fused(S):
    return (128 // S) * S >= 112


def _walker_count(N, S, count):
    """one: 1 walker; partial: the last tile is partial (fused epilogue: tiles of G = 128 // S slot groups, one per electron;
    otherwise tiles of 128 rows); many: far more tiles than the H100's 132 SMs."""
    if count == 'one':
        return 1
    if count == 'partial':
        G = 128 // S
        return next(B for B in range(3, 3 + 128) if ((B * N) % G if _fused(S) else (B * N * S) % 128))
    return -(-150 * 128 // (N * S)) + 1


def _check_mlp(eng, O, X, expect, tag, layer=0):
    N, d = eng.spec.n_elec, eng.spec.embedding_dim
    S = 3 * N + 2
    out, path = eng.debug_mlp(layer, O, X, S=S)
    out2, _ = eng.debug_mlp(layer, O, X, S=S)
    torch.cuda.synchronize()
    assert path == expect, (path, expect)
    assert torch.equal(out, out2)
    assert torch.isfinite(out).all()
    ref = mlp_fl_ref(eng, layer, O, X, N, S)
    if eng.dtype == torch.float64:
        _assert_fp64(tag, path, _errors(out, ref, ref, N, S, 1))
        return
    W = {f'L{layer}.{n}': weight(eng, f'L{layer}.{n}', torch.float32).cpu() for n in ('wo', 'w1', 'w2', 'b1', 'b2')}
    ref32 = mlp_fl_ref(W, layer, O.cpu(), X.cpu(), N, S, dtype=torch.float32)
    _assert_close(tag, path, _errors(out, ref, ref32, N, S, 1))


def _mlp_case(N, count, inp='dense', env=(), expect=None, dtype='float32'):
    _, eng = _engine(_molecule(N), env=env, dtype=dtype, n_layers=1)
    S = 3 * N + 2
    B = _walker_count(N, S, count)
    g = torch.Generator(device='cpu').manual_seed(31 * N + B)
    O, X = (_rows(B, N, S, 256, g, inp).to(DEV, getattr(torch, dtype)) for _ in range(2))
    expect = expect or ('gemm_fused_tanh' if _fused(S) else 'gemm_tanh_fl_kernel')
    _check_mlp(eng, O, X, expect, f'MLP N={N} S={S} walkers={B} {inp} {dict(env)}')


@pytest.mark.parametrize('count', ['one', 'partial', 'many'])
@pytest.mark.parametrize('N', [2, 3, 4, 5, 8, 9, 10, 14, 28, 30])
def test_fl_mlp_matches_fp64(N, count):
    """fp32 tensor-core engines, d = 256: S = 8, 11, 14, 17, 29, 32 take the fused tanh-Laplacian epilogue of the row GEMM
    (tiles of whole slot groups, rpt = (128 / S) S), S = 26, 44, 86, 92 the separate tanh_fl_kernel; one walker, a partial last
    tile, and more tiles than SMs."""
    _mlp_case(N, count)


@pytest.mark.parametrize('inp', ['electron', 'big', 'small'])
@pytest.mark.parametrize('N', [4, 8])
def test_fl_mlp_input_ranges_match_fp64(N, inp):
    """First-layer tangent structure and tangents 1e3 / 1e-3 times the values, fused (N = 4) and separate (N = 8) tanh."""
    _mlp_case(N, 'partial', inp)


def test_fl_mlp_engine_created_without_fused_tanh_matches_fp64():
    """N = 4 on an engine created with DQMC_NO_FUSE_TANH=1: row GEMMs + tanh_fl_kernel where the fused epilogue would
    otherwise run."""
    _mlp_case(4, 'partial', env=(('DQMC_NO_FUSE_TANH', 1),), expect='gemm_tanh_fl_kernel')


@pytest.mark.parametrize('N', [4, 8])
def test_fl_mlp_fp64_matches_fp64(N):
    """fp64 engine: CUDA-core gemm_kernel + tanh_fl_kernel."""
    _mlp_case(N, 'partial', dtype='float64', expect='simt_gemm_tanh_fl_kernel')


# ---- walker isolation ------------------------------------------------------------------------------------------------------

def _poison(X, rows_per_walker, walkers, case, g):
    """X [walkers rows_per_walker][c] with every odd walker's rows replaced -> (X', mask of the replaced rows)."""
    bad = (torch.arange(walkers * rows_per_walker) // rows_per_walker) % 2 == 1
    Y = X.clone()
    if case == 'finite':
        Y[bad] = torch.randn(int(bad.sum()), X.shape[1], generator=g).to(X.device, X.dtype)
    else:
        Y[bad] = float(case)
    return Y, bad.to(X.device)


ISO_CASES = ['finite', 'inf', 'nan']


def _assert_isolated(base, out, bad, case):
    assert torch.isfinite(base).all()
    assert torch.equal(out[~bad], base[~bad])
    if case != 'finite':
        assert not torch.isfinite(out[bad]).all(dim=1).any()


@pytest.mark.parametrize('case', ISO_CASES)
@pytest.mark.parametrize('variant', ['simt', 'mma', 'generic'])
def test_fl_attention_walker_isolation_bitwise(variant, case):
    """Forward-Laplacian attention (SIMT at N = 4, tensor cores at N = 17, generic with nuclear tokens for LiH): every other
    walker's slot rows replaced by other finite rows, inf or nan; the kept walkers are bit for bit unchanged and every replaced
    row comes out non-finite."""
    if variant == 'generic':
        _, eng = _engine('LiH', 'transpsiformer', **TRANS)
    else:
        _, eng = _engine(_molecule(4 if variant == 'simt' else 17), env=(('DQMC_ATTN_FL_MMA', int(variant == 'mma')),),
                         n_layers=1)
    N, d = eng.spec.n_elec, eng.spec.embedding_dim
    S, walkers = 3 * N + 2, 5
    g = torch.Generator(device='cpu').manual_seed(N)
    QKV = _rows(walkers, N, S, 3 * d, g, 'dense').to(DEV)
    base, _ = eng.debug_attention(0, QKV, S=S)
    Q1, bad = _poison(QKV, N * S, walkers, case, g)
    out, _ = eng.debug_attention(0, Q1, S=S)
    torch.cuda.synchronize()
    _assert_isolated(base, out, bad, case)


@pytest.mark.parametrize('case', ISO_CASES)
@pytest.mark.parametrize('N', [4, 8])
def test_fl_mlp_walker_isolation_bitwise(N, case):
    """The MLP with the fused epilogue (N = 4, S = 14: a tile holds the slot groups of 9 electrons, i.e. of three walkers) and
    with tanh_fl_kernel (N = 8): every other walker's O and X rows replaced."""
    _, eng = _engine(_molecule(N), n_layers=1)
    S, walkers = 3 * N + 2, 11
    g = torch.Generator(device='cpu').manual_seed(N + 1)
    O, X = (_rows(walkers, N, S, 256, g, 'dense').to(DEV) for _ in range(2))
    base, path = eng.debug_mlp(0, O, X, S=S)
    assert path == ('gemm_fused_tanh' if N == 4 else 'gemm_tanh_fl_kernel')
    O1, bad = _poison(O, N * S, walkers, case, g)
    X1, _ = _poison(X, N * S, walkers, case, g)
    out, _ = eng.debug_mlp(0, O1, X1, S=S)
    torch.cuda.synchronize()
    _assert_isolated(base, out, bad, case)
