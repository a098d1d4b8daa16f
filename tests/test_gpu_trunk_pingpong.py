"""GPU: the two warpgroups of the whole-trunk kernel and of the fused MLP block run their halves of a tile independently (own
weight ring, own barriers, MMA token handed back and forth).  Bit-for-bit invariants that only a correct schedule keeps: the
output does not depend on how many tiles a CTA runs, nor on which warpgroup a walker lands in; a tile whose second warpgroup
has no walker (and a single walker) still matches fp64; the MLP block is deterministic run to run."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from deepqmc_b200 import params as PN
from deepqmc_b200.ansatz import B200Ansatz
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from tc_reference import trunk_ref, weight

DEV = 'cuda:0'
NS = [2, 4, 5, 9, 16, 17, 30, 32]
LS = [1, 4, 8]
# the bounds of tests/test_gpu_tc_conformance.py (multiples of the plain-fp32 restatement's error against fp64)
TRUNK_RMS_FACTOR, TRUNK_MAX_FACTOR = 18.0, 25.0
TRUNK_RMS_FACTOR_ONE, TRUNK_MAX_FACTOR_ONE = 30.0, 40.0
MLP_MAX_ERR = 3e-5  # tests/test_gpu_tcgen05.py: fused MLP block against fp64


def _molecule(n_elec):
    n_nuc = -(-n_elec // 6)
    charges = [n_elec // n_nuc + (i < n_elec % n_nuc) for i in range(n_nuc)]
    coords = [[2.5 * i, 0.3 * (i % 2), 0.0] for i in range(n_nuc)]
    return Molecule(coords=coords, charges=charges, charge=0, spin=n_elec % 2)


def _slot(N):
    return 1 << (N - 1).bit_length()


def _make(hamil, kind, params, env, **hyper):
    mp = pytest.MonkeyPatch()
    for k, v in env.items():
        mp.setenv(k, v)
    try:
        a = B200Ansatz(hamil, kind, dtype='float32', gemm_backend=1, **hyper)
        return a.engine_for(hamil, params if params is not None else PN.perturb_params(a.init(0)))
    finally:
        mp.undo()


_TRUNK = {}


def _trunk_engine(N, L, nsms=None):
    """Psiformer engine with N electrons and L layers (the same parameters for every nsms); nsms: DQMC_NSMS at creation."""
    key = (N, L)
    if key not in _TRUNK:
        hamil = MolecularHamiltonian(mol=_molecule(N))
        a = B200Ansatz(hamil, 'psiformer', dtype='float32', gemm_backend=1, n_layers=L)
        params = PN.perturb_params(a.init(0))
        _TRUNK[key] = (hamil, params, a.engine_for(hamil, params))
    hamil, params, eng = _TRUNK[key]
    if nsms is None:
        return eng
    return _make(hamil, 'psiformer', params, {'DQMC_NSMS': str(nsms)}, n_layers=L)


def _rows(walkers, N, seed):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return torch.randn(walkers * N, 256, generator=g).to(DEV)


@pytest.mark.parametrize('L', LS)
@pytest.mark.parametrize('N', NS)
def test_trunk_bitwise_equal_across_grids(N, L):
    """1, 2 and 3 CTAs (up to 8 tiles per CTA: ring and token phases carried across tiles and layers) and the full grid
    give the same bits; the last tile's second warpgroup has no walker."""
    G = 128 // _slot(N)
    walkers = 7 * G + G // 2 - 1
    X0 = _rows(walkers, N, 100 * N + L)
    base = _trunk_engine(N, L).debug_trunk(X0)
    torch.cuda.synchronize()
    assert torch.isfinite(base).all()
    for nsms in (1, 2, 3):
        eng = _trunk_engine(N, L, nsms)
        out = eng.debug_trunk(X0)
        torch.cuda.synchronize()
        assert torch.equal(out, base), nsms
        del eng


@pytest.mark.parametrize('L', LS)
@pytest.mark.parametrize('N', NS)
def test_trunk_bitwise_equal_in_either_warpgroup(N, L):
    """Moving every walker by half a tile (G / 2 walkers in front) puts it in the other warpgroup: its rows come out bit for
    bit the same."""
    G = 128 // _slot(N)
    walkers = 3 * G + 1
    X0 = _rows(walkers, N, 200 * N + L)
    pad = _rows(G // 2, N, 300 * N + L)
    eng = _trunk_engine(N, L)
    base = eng.debug_trunk(X0)
    out = eng.debug_trunk(torch.cat([pad, X0]))
    torch.cuda.synchronize()
    assert torch.equal(out[(G // 2) * N:], base)


@pytest.mark.parametrize('count', ['one', 'half_tile', 'tiles_and_a_half'])
@pytest.mark.parametrize('L', LS)
@pytest.mark.parametrize('N', NS)
def test_trunk_empty_second_warpgroup_matches_fp64(N, L, count):
    """Walker counts that leave warpgroup 1 of the last tile empty (G / 2 walkers: one tile; 2 G + G / 2: three tiles) and a
    single walker, against the fp64 restatement with the bounds of the conformance tests."""
    G = 128 // _slot(N)
    walkers = {'one': 1, 'half_tile': G // 2, 'tiles_and_a_half': 2 * G + G // 2}[count]
    eng = _trunk_engine(N, L)
    X0 = _rows(walkers, N, 400 * N + 10 * L + walkers)
    out = eng.debug_trunk(X0)
    torch.cuda.synchronize()
    ref = trunk_ref(eng, X0, N, L)
    ref32 = trunk_ref(eng, X0, N, L, dtype=torch.float32)
    assert torch.isfinite(out).all()
    err, err32 = (out.double() - ref).abs().max().item(), (ref32.double() - ref).abs().max().item()
    rms, rms32 = (out.double() - ref).pow(2).mean().sqrt().item(), (ref32.double() - ref).pow(2).mean().sqrt().item()
    print(f'measured trunk N={N} L={L} walkers={walkers}: rms/rms32 {rms / rms32:.2f} max/max32 {err / err32:.2f}')
    f_rms, f_max = (TRUNK_RMS_FACTOR_ONE, TRUNK_MAX_FACTOR_ONE) if walkers == 1 else (TRUNK_RMS_FACTOR, TRUNK_MAX_FACTOR)
    assert rms < f_rms * rms32 + 1e-6 and err < f_max * err32 + 1e-5, (err, err32, rms, rms32)


@pytest.mark.parametrize('rows', [1, 50, 128 * 5 + 40, 148 * 128 + 77])
@pytest.mark.parametrize('kind', ['psiformer', 'transpsiformer'])
def test_mlp_block_deterministic_and_matches_fp64(kind, rows):
    """The fused MLP block of the DQMC_TC_TRUNK=0 path (d = 256 Psiformer, d = 128 TransPsiformer): bitwise equal run to run,
    on a 2-SM grid and on the full grid; rows that leave the second warpgroup of the last tile empty; against fp64."""
    hamil = MolecularHamiltonian(mol=Molecule.from_name('LiH'))
    hyper = dict(embedding_dim=128, n_layers=2, n_heads=2, n_determinants=2) if kind == 'transpsiformer' else {}
    d = hyper.get('embedding_dim', 256)
    eng = _make(hamil, kind, None, {'DQMC_TC_TRUNK': '0'}, **hyper)
    eng2 = _make(hamil, kind, None, {'DQMC_TC_TRUNK': '0', 'DQMC_NSMS': '2'}, **hyper)
    g = torch.Generator(device='cpu').manual_seed(rows + d)
    O = torch.randn(rows, d, generator=g).to(DEV)
    X = (3 * torch.randn(rows, d, generator=g)).to(DEV)
    out = eng.debug_mlp_block(1, O, X)
    again = eng.debug_mlp_block(1, O, X)
    out2 = eng2.debug_mlp_block(1, O, X)
    torch.cuda.synchronize()
    assert torch.equal(out, again) and torch.equal(out, out2)
    W = lambda name: weight(eng, name)
    A = X.double() + O.double() @ W('L1.wo')
    M1 = torch.tanh(A @ W('L1.w1') + W('L1.b1')[0])
    ref = A + torch.tanh(M1 @ W('L1.w2') + W('L1.b2')[0])
    err = (out.double() - ref).abs().max().item()
    assert err < MLP_MAX_ERR, err
