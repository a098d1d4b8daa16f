"""GPU: the tensor-core lock and the continuous weight stream of the whole-trunk kernel and of the fused MLP block.

The two warpgroups of a CTA take the lock in whatever order they reach it, so which GEMM runs when depends on timing; each
warpgroup's weight ring runs along one stream of slots across GEMM, layer and tile boundaries.  Neither may change a bit of
the output: the phase timers (which change the timing and so the lock order) on or off, one CTA running every tile, two
CTAs, or the full grid (the stream crosses every layer boundary and, on few SMs, many tiles), walker counts that end inside
a tile's first or second warpgroup.  The kernels' error word (set when a lock wait passes its bound) stays clear.  A
correctness check: every configuration runs once."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from deepqmc_b200 import params as PN
from deepqmc_b200.ansatz import B200Ansatz
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule

DEV = 'cuda:0'


def _molecule(n_elec):
    n_nuc = -(-n_elec // 6)
    charges = [n_elec // n_nuc + (i < n_elec % n_nuc) for i in range(n_nuc)]
    coords = [[2.5 * i, 0.3 * (i % 2), 0.0] for i in range(n_nuc)]
    return Molecule(coords=coords, charges=charges, charge=0, spin=n_elec % 2)


def _engine(hamil, kind, params, env, **hyper):
    mp = pytest.MonkeyPatch()
    for k, v in env.items():
        mp.setenv(k, v)
    try:
        a = B200Ansatz(hamil, kind, dtype='float32', gemm_backend=1, **hyper)
        return a.engine_for(hamil, params if params is not None else PN.perturb_params(a.init(0)))
    finally:
        mp.undo()


def _rows(n, d, seed, scale=1.0):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (scale * torch.randn(n, d, generator=g)).to(DEV)


# (DQMC_NSMS, DQMC_TRUNK_PHASES) of the engines compared with the full grid without timers
TRUNK_RUNS = [(None, '1'), (1, None), (2, None), (1, '1')]


@pytest.mark.parametrize('end', ['first_warpgroup', 'second_warpgroup'])
@pytest.mark.parametrize('L', [1, 4])
@pytest.mark.parametrize('N', [4, 30])
def test_trunk_bitwise_equal_under_any_lock_order(N, L, end):
    """140 full tiles and a last one whose walkers end a quarter of the way into its first or its second warpgroup: more
    tiles than the H100 has SMs, so on the full grid some CTAs run two; one CTA runs all 141 tiles."""
    hamil = MolecularHamiltonian(mol=_molecule(N))
    a = B200Ansatz(hamil, 'psiformer', dtype='float32', gemm_backend=1, n_layers=L)
    params = PN.perturb_params(a.init(0))
    G = 128 // (1 << (N - 1).bit_length())
    walkers = 140 * G + (G // 4 if end == 'first_warpgroup' else G // 2 + G // 4)
    X0 = _rows(walkers * N, 256, 10 * N + L)
    eng = _engine(hamil, 'psiformer', params, {}, n_layers=L)
    base = eng.debug_trunk(X0)
    torch.cuda.synchronize()
    assert torch.isfinite(base).all()
    assert eng.debug_tc_error() == 0
    for nsms, phases in TRUNK_RUNS:
        env = {k: v for k, v in (('DQMC_NSMS', nsms and str(nsms)), ('DQMC_TRUNK_PHASES', phases)) if v}
        e = _engine(hamil, 'psiformer', params, env, n_layers=L)
        out = e.debug_trunk(X0)
        torch.cuda.synchronize()
        assert torch.equal(out, base), env
        assert e.debug_tc_error() == 0, env
        if phases:
            ph = e.debug_trunk_phases()
            assert ph['tile_layer_pairs'] == 141 * L, ph
        del e


@pytest.mark.parametrize('end', ['first_warpgroup', 'second_warpgroup'])
@pytest.mark.parametrize('kind', ['psiformer', 'transpsiformer'])
def test_mlp_block_bitwise_equal_under_any_lock_order(kind, end):
    """The fused MLP block (d = 256 Psiformer, d = 128 TransPsiformer) twice on the same input, on 1 and 2 SMs and on the full
    grid (140 full tiles and one ending inside its first or second warpgroup): the same bits, the error word clear."""
    hamil = MolecularHamiltonian(mol=Molecule.from_name('LiH'))
    hyper = dict(embedding_dim=128, n_layers=2, n_heads=2, n_determinants=2) if kind == 'transpsiformer' else {}
    d = hyper.get('embedding_dim', 256)
    rows = 140 * 128 + (32 if end == 'first_warpgroup' else 96)
    O, X = _rows(rows, d, rows + d), _rows(rows, d, rows + d + 1, 3.0)
    a = B200Ansatz(hamil, kind, dtype='float32', gemm_backend=1, **hyper)
    params = PN.perturb_params(a.init(0))
    engines = [_engine(hamil, kind, params, {'DQMC_TC_TRUNK': '0', **({'DQMC_NSMS': str(n)} if n else {})}, **hyper)
               for n in (None, 1, 2)]
    base = engines[0].debug_mlp_block(1, O, X)
    again = engines[0].debug_mlp_block(1, O, X)
    torch.cuda.synchronize()
    assert torch.isfinite(base).all()
    assert torch.equal(again, base)
    for e in engines[1:]:
        out = e.debug_mlp_block(1, O, X)
        torch.cuda.synchronize()
        assert torch.equal(out, base)
    for e in engines:
        assert e.debug_tc_error() == 0
