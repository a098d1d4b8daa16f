"""GPU: the whole-trunk kernel (trunk_tc.cuh) and the plain-forward tensor-core attention (attn_mma.cuh) across their shape
space, against fp64 restatements of the same operations; walker isolation (one walker's rows never change another walker's
outputs, bit for bit); the non-local ECP's gathering quadrature forwards under every workspace chunking.

Tolerances are multiples of what a plain-fp32 restatement of the same layers gets wrong against fp64.  The factors were
measured on an H100 80GB HBM3 at 700 W power limit; each constant's comment gives the worst measured value and the margin."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from deepqmc_b200 import params as PN
from deepqmc_b200.ansatz import B200Ansatz
from deepqmc_b200.engine import MODE_FORWARD, MODE_LOCAL_ENERGY
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from tc_reference import attention_ref, trunk_ref, weight

DEV = 'cuda:0'
HALF_RANGE = 65504 / 16  # largest |x| of an activation / Q / K / V the scaled half split represents (kActScale = 16)

# whole-trunk kernel against fp64, as multiples of the plain-fp32 restatement's error (rms, max) + an absolute floor.
# Launches of several walkers: measured worst 11.5 (rms) and 16.6 (max), 11.3 / 12.4 with activations near the top of the
# half range; margin about 1.6x / 1.5x.
TRUNK_RMS_FACTOR = 18.0
TRUNK_MAX_FACTOR = 25.0
# One walker (at most 32 rows, where the fp32 restatement happens to be most accurate): measured worst 18.4 (rms) and 19.7
# (max); margin about 1.6x / 2x.  Dropping the padding-key mask gives errors of O(1), the lost low product of P V about 230x
# the fp32 restatement's rms.
TRUNK_RMS_FACTOR_ONE = 30.0
TRUNK_MAX_FACTOR_ONE = 40.0
# plain-forward attention: max |O - O_fp64| / sum_j p_j |v_j| per element.  Measured worst 2.3e-5 (near one-hot rows: the fp32
# restatement itself shows 2.7e-5 there), 3.2e-6 with N(0, 1) rows; margin 4x.  Half-precision P V (lost low product): 2e-4 - 4e-4.
ATTN_REL_MAX = 1e-4
# ... and the rms of that relative error as a multiple of the same rms of the plain-fp32 restatement (evaluated on the CPU, so
# the yardstick does not depend on which GPU GEMM algorithm runs): measured worst 1.73, the same in three runs; margin 2.3x
ATTN_FACTOR = 4.0


def _molecule(n_elec, n_nuc=None):
    """A neutral chain of nuclei with n_elec electrons: charges as equal as possible (n_nuc nuclei, default: ceil(n / 6))."""
    n_nuc = n_nuc or -(-n_elec // 6)
    charges = [n_elec // n_nuc + (i < n_elec % n_nuc) for i in range(n_nuc)]
    coords = [[2.5 * i, 0.3 * (i % 2), 0.0] for i in range(n_nuc)]
    return Molecule(coords=coords, charges=charges, charge=0, spin=n_elec % 2)


_ENGINES = {}


def _engine(mol, kind='psiformer', ecp=None, nsms=None, env=(), **hyper):
    """fp32 engine with the tensor-core backend (one per configuration, cached); nsms: DQMC_NSMS at creation (SM count the
    persistent kernels size their grids by); env: further switches set around its creation."""
    key = (mol if isinstance(mol, str) else (tuple(mol.charges), tuple(mol.coords.ravel())), kind, ecp, nsms, tuple(env),
           tuple(sorted(hyper.items())))
    if key not in _ENGINES:
        m = Molecule.from_name(mol) if isinstance(mol, str) else mol
        hamil = MolecularHamiltonian(mol=m, ecp_type=ecp)
        mp = pytest.MonkeyPatch()
        if nsms:
            mp.setenv('DQMC_NSMS', str(nsms))
        for k, v in env:
            mp.setenv(k, str(v))
        try:
            a = B200Ansatz(hamil, kind, dtype='float32', gemm_backend=1, **hyper)
            params = PN.perturb_params(a.init(0))
            eng = a.engine_for(hamil, params)
        finally:
            mp.undo()
        _ENGINES[key] = (hamil, a, params, eng)
    return _ENGINES[key]


def _heavy(shape, g, clip):
    """Heavy-tailed rows: randn * exp(2 randn), clipped to +-clip."""
    return (torch.randn(*shape, generator=g) * torch.exp(2 * torch.randn(*shape, generator=g))).clamp(-clip, clip)


# ---- 1. whole-trunk kernel across its shape space -------------------------------------------------------------------------

def _np(N):
    return 1 << (N - 1).bit_length()


def _check_trunk(eng, X0, N, L, near_top=False):
    out = eng.debug_trunk(X0)
    torch.cuda.synchronize()
    peaks = {}
    ref = trunk_ref(eng, X0, N, L, peaks=peaks)
    ref32 = trunk_ref(eng, X0, N, L, dtype=torch.float32)
    # inside the half operands' range; near_top: within a factor 2 of its top
    assert peaks['act'] < HALF_RANGE and peaks['qkv'] < HALF_RANGE, peaks
    assert not near_top or max(peaks.values()) > HALF_RANGE / 2, peaks
    assert torch.isfinite(out).all()
    err, err32 = (out.double() - ref).abs().max().item(), (ref32.double() - ref).abs().max().item()
    rms, rms32 = (out.double() - ref).pow(2).mean().sqrt().item(), (ref32.double() - ref).pow(2).mean().sqrt().item()
    print(f'measured trunk N={N} L={L} rows={X0.shape[0]}: rms/rms32 {rms / rms32:.2f} max/max32 {err / err32:.2f} '
          f'peaks {peaks}')
    f_rms, f_max = (TRUNK_RMS_FACTOR_ONE, TRUNK_MAX_FACTOR_ONE) if X0.shape[0] == N else (TRUNK_RMS_FACTOR, TRUNK_MAX_FACTOR)
    assert rms < f_rms * rms32 + 1e-6 and err < f_max * err32 + 1e-5, (err, err32, rms, rms32)


@pytest.mark.parametrize('dist', ['normal', 'heavy'])
@pytest.mark.parametrize('count', ['one', 'partial_tile', 'persistent'])
@pytest.mark.parametrize('N', [2, 3, 5, 8, 9, 16, 17, 32])
def test_trunk_matches_fp64_every_slot_size(N, count, dist):
    """Every walker slot size NP = 2 .. 32 (both attention paths: keys = the 16-row window masked to the slot for NP <= 16, the
    slot itself for NP = 32), full slots (N = NP) and mostly padded ones (N = 9, 17); one walker, a single partial tile
    (G - 1 walkers, G = 128 / NP per tile), and several tiles per CTA with a ragged last tile on a 2-SM grid (the persistent
    loop and the barrier phases wrap); N(0, 1) and heavy-tailed embedding rows (|x| up to 30: independent rows much larger than
    that make Q K^T so large that near-tied scores flip the softmax under any fp32 rounding, and the comparison would measure
    that instead of the kernel; the top of the range is the next test's)."""
    G = 128 // _np(N)
    walkers = {'one': 1, 'partial_tile': G - 1 if G > 1 else 1, 'persistent': 5 * G + 1}[count]
    _, _, _, eng = _engine(_molecule(N), nsms=2 if count == 'persistent' else None)
    g = torch.Generator(device='cpu').manual_seed(1000 * N + walkers)
    X0 = torch.randn(walkers * N, 256, generator=g) if dist == 'normal' else _heavy((walkers * N, 256), g, 30.0)
    _check_trunk(eng, X0.to(DEV), N, 4)


@pytest.mark.parametrize('L', [1, 2, 3, 8])
@pytest.mark.parametrize('N', [9, 16])
def test_trunk_matches_fp64_layer_counts(N, L):
    """1, 2, 3 and kTrMaxLayers = 8 layers (the weight stream of every layer count) at a padded and a full slot."""
    _, _, _, eng = _engine(_molecule(N), n_layers=L)
    G = 128 // _np(N)
    walkers = 3 * G + 1
    g = torch.Generator(device='cpu').manual_seed(77 * L + N)
    _check_trunk(eng, torch.randn(walkers * N, 256, generator=g).to(DEV), N, L)


@pytest.mark.parametrize('N', [5, 17, 32])
def test_trunk_matches_fp64_near_the_half_range(N):
    """Activations or Q / K / V within a factor 2 of the largest magnitude the scaled half split represents (16 |x| < 65504),
    through all four layers.  The electrons of a walker share one heavy-tailed embedding row, scaled so that the largest
    magnitude met on the way is 0.8 of the range: every score of a query is then the same number in any arithmetic (a uniform
    softmax: no near-tied scores to flip), while the half operands of every dense layer run near the top of their range."""
    _, _, _, eng = _engine(_molecule(N))
    walkers = 2 * (128 // _np(N)) + 1
    g = torch.Generator(device='cpu').manual_seed(4094 + N)
    X0 = _heavy((walkers, 256), g, 30.0).repeat_interleave(N, dim=0).to(DEV)
    peaks = {}
    trunk_ref(eng, X0, N, 4, peaks=peaks)
    _check_trunk(eng, X0 * (0.8 * HALF_RANGE / max(peaks.values())), N, 4, near_top=True)


# ---- 2. plain-forward attention through dqmc_debug_attention ---------------------------------------------------------------

def _qkv(B, N, d, g, spread):
    """Q | K | V rows.  spread: Q, K scaled so that the scores q.k / sqrt(dh) span about +-60 (near one-hot softmax rows) and
    |V| up to 2e3; otherwise N(0, 1)."""
    Q, K, V = (torch.randn(B * N, d, generator=g) for _ in range(3))
    if spread:
        s = 5.0  # q.k / 8 ~ N(0, s^4): standard deviation 25, |scores| up to ~60 over a row
        Q, K = Q * s, K * s
        V = (V * torch.exp(torch.randn(B * N, d, generator=g))).clamp(-4, 4) * 500
    return torch.cat([Q, K, V], dim=1)


def _nuclear_tokens(eng, layer):
    if eng.spec.kind != 'transpsiformer':
        return None, None
    return weight(eng, f'L{layer}.kn'), weight(eng, f'L{layer}.vn')


def _check_attention(eng, N, H, QKV, layer=0, expect_mma=True):
    d = QKV.shape[1] // 3
    kn, vn = _nuclear_tokens(eng, layer)
    O, kernel = eng.debug_attention(layer, QKV)
    O2, _ = eng.debug_attention(layer, QKV)
    torch.cuda.synchronize()
    assert (kernel == 'attn_fwd_mma_kernel') == expect_mma, kernel
    assert torch.equal(O, O2)  # every output element is written, from the inputs alone
    ref, mag = attention_ref(QKV, N, H, kn, vn)
    cpu = lambda t: None if t is None else t.cpu()
    ref32, _ = attention_ref(QKV.cpu(), N, H, cpu(kn), cpu(vn), dtype=torch.float32)
    assert O.shape == (QKV.shape[0], d) and torch.isfinite(O).all()
    rel = (O.double() - ref).abs() / mag
    rel32 = (ref32.to(DEV).double() - ref).abs() / mag
    rms, rms32 = rel.pow(2).mean().sqrt().item(), rel32.pow(2).mean().sqrt().item()
    print(f'measured attention N={N} H={H} rows={QKV.shape[0]} Mn={0 if kn is None else kn.shape[0]} {kernel}: '
          f'max {rel.max().item():.2e} (fp32 {rel32.max().item():.2e}) rms ratio {rms / rms32:.2f}')
    assert rel.max().item() < ATTN_REL_MAX and rms < ATTN_FACTOR * rms32, (rel.max().item(), rms, rms32)


@pytest.mark.parametrize('spread', [False, True])
@pytest.mark.parametrize('N', [2, 4, 9, 16, 17, 24, 31, 32, 33, 40, 41, 48])
def test_attention_psiformer_matches_fp64(N, spread):
    """Psiformer, d = 256, 4 heads of 64: key tiles NK8 = 1 .. 6, exact and partial 16-query tiles, up to the N = 48 limit of
    attn_fwd_mma_kernel; N(0, 1) rows and near one-hot scores (+-60) with |V| up to 2e3."""
    _, _, _, eng = _engine(_molecule(N), n_layers=1)
    g = torch.Generator(device='cpu').manual_seed(N + 100 * spread)
    _check_attention(eng, N, 4, _qkv(7, N, 256, g, spread).to(DEV))


@pytest.mark.parametrize('spread', [False, True])
def test_attention_past_the_mma_limit_matches_fp64(spread):
    """N = 49 electrons is past the 48 keys of attn_fwd_mma_kernel: the engine picks another kernel, which matches fp64 too."""
    N = 49
    _, _, _, eng = _engine(_molecule(N), n_layers=1)
    g = torch.Generator(device='cpu').manual_seed(49 + 100 * spread)
    _check_attention(eng, N, 4, _qkv(3, N, 256, g, spread).to(DEV), expect_mma=False)


def _trans_mol(name):
    # N + Mn = 48: 40 electrons on 8 nuclei
    return _molecule(40, 8) if name == 'N+Mn=48' else name


@pytest.mark.parametrize('spread', [False, True])
@pytest.mark.parametrize('mol', ['LiH', 'cyclobutadiene_square', 'N+Mn=48'])
def test_attention_transpsiformer_nuclear_tokens_match_fp64(mol, spread):
    """TransPsiformer, d = 128, 2 heads of 64: the keys and values carry the layer's nuclear tokens (LiH 4 + 2, NK8 = 1;
    cyclobutadiene 28 + 8, NK8 = 5; 40 + 8 = 48, NK8 = 6), in both layers."""
    hamil, _, _, eng = _engine(_trans_mol(mol), 'transpsiformer', embedding_dim=128, n_layers=2, n_heads=2, n_determinants=2)
    N = hamil.n_up + hamil.n_down
    g = torch.Generator(device='cpu').manual_seed(N + 100 * spread)
    QKV = _qkv(6, N, 128, g, spread).to(DEV)
    for layer in range(2):
        _check_attention(eng, N, 2, QKV, layer=layer)


# ---- 3. walker isolation ---------------------------------------------------------------------------------------------------

def _poison(X, N, walkers, case, g):
    """X [walkers N][c] with every odd walker's rows replaced; -> (X', mask of the replaced rows)."""
    bad = (torch.arange(walkers * N) // N) % 2 == 1
    Y = X.clone()
    n = int(bad.sum())
    if case == 'finite':
        Y[bad] = torch.randn(n, X.shape[1], generator=g).to(X.device)
    elif case == 'inf':
        Y[bad] = float('inf')
    elif case == 'nan':
        Y[bad] = float('nan')
    else:
        Y[bad] = case(n, X.shape[1]).to(X.device)
    return Y, bad.to(X.device)


ISO_CASES = ['finite', 'past_half_range', 'inf', 'nan']


@pytest.mark.parametrize('case', ISO_CASES)
@pytest.mark.parametrize('N', [2, 3, 5, 16, 17])
def test_trunk_walker_isolation_bitwise(N, case):
    """Walker slots NP = 2, 4, 8, 16, 32: replacing every other walker's embedding rows (other finite rows; rows whose V is past
    the range of the half split; inf; nan) leaves the other walkers' trunk outputs bit for bit unchanged, and a walker with
    non-finite or out-of-range inputs comes out non-finite (nothing hides a bad walker)."""
    _, _, _, eng = _engine(_molecule(N))
    G = 128 // _np(N)
    walkers = 2 * G + 3
    g = torch.Generator(device='cpu').manual_seed(N)
    X0 = torch.randn(walkers * N, 256, generator=g).to(DEV)
    base = eng.debug_trunk(X0)
    # |x| = 3000 is inside the half range of the activations (16 |x| < 65504), its Q / K / V rows are far outside it
    big = lambda n, c: 3000.0 * torch.sign(torch.randn(n, c, generator=g))
    X1, bad = _poison(X0, N, walkers, big if case == 'past_half_range' else case, g)
    out = eng.debug_trunk(X1)
    torch.cuda.synchronize()
    assert torch.isfinite(base).all()
    assert torch.equal(out[~bad], base[~bad])
    if case != 'finite':
        assert not torch.isfinite(out[bad]).all(dim=1).any()


@pytest.mark.parametrize('case', ISO_CASES)
@pytest.mark.parametrize('mol', [4, 17, 'LiH-trans'])
def test_attention_walker_isolation_bitwise(mol, case):
    """The same for the plain-forward attention (dqmc_debug_attention), with nuclear tokens for the TransPsiformer: Q | K | V rows
    of every other walker replaced (finite rows; V past the half range; inf; nan)."""
    if mol == 'LiH-trans':
        hamil, _, _, eng = _engine('LiH', 'transpsiformer', embedding_dim=128, n_layers=2, n_heads=2, n_determinants=2)
        H = 2
    else:
        hamil, _, _, eng = _engine(_molecule(mol), n_layers=1)
        H = 4
    N = hamil.n_up + hamil.n_down
    d = 64 * H
    walkers = 9
    g = torch.Generator(device='cpu').manual_seed(N)
    QKV = _qkv(walkers, N, d, g, False).to(DEV)
    base, _ = eng.debug_attention(0, QKV)

    def past_range(n, c):
        rows = torch.randn(n, c, generator=g)
        rows[:, 2 * d:] = 1e5 * torch.sign(rows[:, 2 * d:])
        return rows

    Q1, bad = _poison(QKV, N, walkers, past_range if case == 'past_half_range' else case, g)
    out, _ = eng.debug_attention(0, Q1)
    torch.cuda.synchronize()
    assert torch.isfinite(base).all()
    assert torch.equal(out[~bad], base[~bad])
    if case != 'finite':
        assert not torch.isfinite(out[bad]).all(dim=1).any()


def _walkers(hamil, B, seed):
    mol = hamil.mol
    rng = np.random.default_rng(seed)
    N = hamil.n_up + hamil.n_down
    pr = hamil.ns_valence / hamil.ns_valence.sum()
    r = mol.coords[rng.choice(len(mol.coords), size=(B, N), p=pr)] + rng.normal(size=(B, N, 3)) * 0.7
    return torch.as_tensor(r, device=DEV).float(), torch.as_tensor(mol.coords, device=DEV).float()


@pytest.mark.parametrize('mol', ['LiH', 'C', 'benzene'])
def test_wf_forward_walker_isolation_bitwise(mol):
    """End to end, finite walkers only: the plain forward (whole-trunk kernel) of a batch, then the same batch with every other
    walker replaced by a different random walker; the kept walkers' sign and log|psi| are bit for bit unchanged.  Walker slots
    NP = 4 (LiH), 8 (C, 6 electrons), 32 (benzene, ccECP: 30 valence electrons)."""
    hamil, _, _, eng = _engine(mol, ecp='ccECP' if mol == 'benzene' else None)
    B = 77
    r, R = _walkers(hamil, B, 1)
    r2, _ = _walkers(hamil, B, 2)
    keep = torch.arange(B, device=DEV) % 2 == 0
    r2[keep] = r[keep]
    s1, l1 = eng.wf_forward(r, R)
    s2, l2 = eng.wf_forward(r2, R)
    torch.cuda.synchronize()
    assert torch.isfinite(l1).all()
    assert torch.equal(s1[keep], s2[keep]) and torch.equal(l1[keep], l2[keep])
    assert not torch.equal(l1[~keep], l2[~keep])  # the replaced walkers did change


# ---- 4. ECP gather path and chunking --------------------------------------------------------------------------------------

@pytest.mark.parametrize('emb_table', [True, False])
def test_ecp_quadrature_chunking_bitwise(emb_table):
    """Benzene ccECP, 2 walkers, fixed quadrature twists: V_nl and E_loc with the default workspace (both walkers' virtual
    walkers in one plain-forward chunk) and with workspaces that cut each walker's quadrature group into chunks whose
    boundaries (virtual-walker indices) are multiples of neither 12 nor the group size -- the gathering tile load of the
    whole-trunk kernel (moved electron ((v0 + w) / 12) % N, base walker (v0 + w) / group) and the envelope table see every
    chunk offset.  Without the embedding table (an engine created under DQMC_ECP_EMB_TABLE_OFF=1, envelope table on) as
    well: for the same walkers and workspace it launches one embed_fwd_kernel per ECP group fewer than the default engine."""
    hamil, _, _, eng = _engine('benzene', ecp='ccECP', env=() if emb_table else (('DQMC_ECP_EMB_TABLE_OFF', 1),))
    table_on = None if emb_table else _engine('benzene', ecp='ccECP')[3]
    N = hamil.n_up + hamil.n_down
    J = len(hamil.pot.nuc_with_nl_pot)
    vper = 12 * J * N  # virtual walkers (quadrature forwards) per walker
    r, R = _walkers(hamil, 2, 4)
    g = torch.Generator(device='cpu').manual_seed(5)
    tw = (torch.rand(2, J, N, generator=g, dtype=torch.float64) * math.pi / 5).to(DEV).float()

    def run(e, **kw):
        n0 = e.launch_count
        E, st, _, _, _ = e.local_energy(r, R, ecp_twist=tw, **kw)
        return E, st, e.launch_count - n0

    E0, st0, n_default = run(eng)
    if table_on is not None:
        assert n_default == run(table_on)[2] - 1  # one ECP group (both walkers)
    # workspace of the ECP pass with one walker per group: its fixed part + a plain-forward chunk of `chunk` virtual walkers
    prefix = eng.workspace_bytes(1, MODE_LOCAL_ENERGY) - eng.workspace_bytes(vper, MODE_FORWARD)
    for chunk in (1001, vper - 1, 517):
        assert chunk % 12 and vper % chunk
        wsb = prefix + eng.workspace_bytes(chunk, MODE_FORWARD)
        assert eng.workspace_bytes_min(2, MODE_LOCAL_ENERGY) <= wsb < eng.workspace_bytes(2, MODE_LOCAL_ENERGY)
        # the chunk the engine takes: a dry pass of the call carves exactly the fixed part + `chunk` virtual walkers' rows,
        # and one more virtual walker would not fit
        assert eng.debug_plan(2, MODE_LOCAL_ENERGY, wsb)[1] == wsb
        assert prefix + eng.workspace_bytes(chunk + 1, MODE_FORWARD) > wsb
        E1, st1, n1 = run(eng, max_ws_bytes=wsb)
        torch.cuda.synchronize()
        assert n1 > n_default  # the quadrature forwards did run in several chunks
        if table_on is not None:
            assert n1 == run(table_on, max_ws_bytes=wsb)[2] - 2  # two ECP groups (one walker each)
        assert torch.isfinite(E1).all()
        assert torch.equal(st1[3], st0[3]), (chunk, st1[3], st0[3])
        assert torch.equal(E1, E0), (chunk, E1, E0)
