"""GPU: the non-local ECP's cutoff radius.  A (nucleus, electron) pair runs its 12 quadrature forwards only when its squared
distance is at most rc2, the largest d2 with sum_l (2l+1) sum_t |beta_lt| exp(-alpha_lt d2) >= 2^-100 (engine.cu
ecp_cutoff_rc2); a pair beyond it would add less than 2^-100 times its largest psi ratio to V_nl.  DQMC_ECP_CUTOFF=0 keeps every
pair and is the reference here: E_loc and V_nl with and without the cutoff, the forward counter against a plain restatement of
rc2, designed walkers at and beyond the radius, walker isolation, and the quadrature forwards split across workspace chunks."""
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

DEV = 'cuda:0'
EPS = 2.0 ** -100
SMALL = dict(embedding_dim=32, n_layers=2, n_heads=4, n_determinants=4)

_ENGINES = {}


def _engine(mol, dtype, cutoff, env=(), **hyper):
    """(hamil, engine) with the ccECP; cutoff False: created under DQMC_ECP_CUTOFF=0 (every pair active); env: further
    switches set around its creation.  fp32 engines take the tensor-core backend.  Same parameters for all settings."""
    key = (mol, dtype, cutoff, tuple(env), tuple(sorted(hyper.items())))
    if key not in _ENGINES:
        hamil = MolecularHamiltonian(mol=Molecule.from_name(mol), ecp_type='ccECP')
        mp = pytest.MonkeyPatch()
        if not cutoff:
            mp.setenv('DQMC_ECP_CUTOFF', '0')
        for k, v in env:
            mp.setenv(k, str(v))
        try:
            kw = dict(gemm_backend=1) if dtype == 'float32' else {}
            a = B200Ansatz(hamil, 'psiformer', dtype=dtype, **kw, **hyper)
            eng = a.engine_for(hamil, PN.perturb_params(a.init(0)))
        finally:
            mp.undo()
        _ENGINES[key] = (hamil, eng)
    return _ENGINES[key]


def _rc2(hamil, dtype):
    """Squared cutoff radius per non-local nucleus slot, restated: bisection of the weight bound to adjacent doubles, on the
    parameters rounded to the engine's dtype as the engine holds them."""
    out = []
    for I in hamil.pot.nuc_with_nl_pot:
        nl = hamil.pot.nl_params[I].astype(dtype).astype(np.float64)  # [L][alpha | beta][T]
        terms = [(2 * l + 1, a, abs(b)) for l in range(nl.shape[0]) for a, b in zip(nl[l, 0], nl[l, 1]) if b != 0]

        def w(d2):
            return sum(c * b * math.exp(-a * d2) for c, a, b in terms)

        lo, hi = 0.0, 1.0
        while w(hi) >= EPS:
            lo, hi = hi, 2 * hi
        while True:
            mid = lo + 0.5 * (hi - lo)
            if mid <= lo or mid >= hi:
                break
            if w(mid) >= EPS:
                lo = mid
            else:
                hi = mid
        out.append(lo)
    return torch.tensor(out, dtype=torch.float64)


def _active(hamil, dtype, r, R):
    """[B][J][N] pair inside the cutoff radius (d2 in double, as the engine decides)."""
    nuc = torch.as_tensor(hamil.pot.nuc_with_nl_pot)
    d = r.double().cpu()[:, None, :, :] - R.double().cpu()[nuc][None, :, None, :]
    d2 = (d * d).sum(-1)
    return ~(d2 > _rc2(hamil, dtype)[None, :, None])


def _walkers(hamil, B, seed, spread, dtype):
    mol = hamil.mol
    rng = np.random.default_rng(seed)
    N = hamil.n_up + hamil.n_down
    pr = hamil.ns_valence / hamil.ns_valence.sum()
    r = mol.coords[rng.choice(len(mol.coords), size=(B, N), p=pr)] + rng.normal(size=(B, N, 3)) * spread
    tdt = torch.float32 if dtype == 'float32' else torch.float64
    return torch.as_tensor(r, device=DEV, dtype=tdt), torch.as_tensor(mol.coords, device=DEV, dtype=tdt)


def _twists(B, J, N, seed, like):
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.rand(B, J, N, generator=g, dtype=torch.float64) * math.pi / 5).to(DEV, like.dtype)


def _eloc(eng, r, R, tw, **kw):
    n0 = eng.ecp_forward_count
    E, st, _, _, _ = eng.local_energy(r, R, ecp_twist=tw, **kw)
    torch.cuda.synchronize()
    return E, st[3].clone(), eng.ecp_forward_count - n0


def test_benzene_fp32_cutoff_equals_all_pairs():
    """Benzene ccECP, fp32 tensor-core engine, 256 seeded walkers, fixed twists: E_loc and V_nl with the cutoff are those of
    every pair, bit for bit (a skipped pair would need a psi ratio near 1e22 to move an fp32 E_loc); the forward counter is
    12 x the restated active-pair count with the cutoff and 12 B J N without."""
    hamil, on = _engine('benzene', 'float32', True)
    _, off = _engine('benzene', 'float32', False)
    N, J, B = hamil.n_up + hamil.n_down, len(hamil.pot.nuc_with_nl_pot), 256
    r, R = _walkers(hamil, B, 11, 0.7, 'float32')
    tw = _twists(B, J, N, 3, r)
    E1, V1, n1 = _eloc(on, r, R, tw)
    E0, V0, n0 = _eloc(off, r, R, tw)
    act = _active(hamil, np.float32, r, R)
    assert n0 == 12 * B * J * N
    assert n1 == 12 * int(act.sum())
    assert 0 < n1 < n0
    assert torch.isfinite(E1).all()
    assert torch.equal(V1, V0), (V1 - V0).abs().max()
    assert torch.equal(E1, E0), (E1 - E0).abs().max()


@pytest.mark.parametrize('mol,spread', [('C', 2.0), ('LiH', 4.0)])
def test_fp64_cutoff_matches_all_pairs(mol, spread):
    """fp64 engine, small ccECP systems (carbon atom: r_c 3.07 bohr; LiH: the Li channel reaches 7.3 bohr), walkers spread
    wide enough that part of the pairs fall outside: with and without the cutoff within 1e-13 relative."""
    hamil, on = _engine(mol, 'float64', True, **SMALL)
    _, off = _engine(mol, 'float64', False, **SMALL)
    N, J, B = hamil.n_up + hamil.n_down, len(hamil.pot.nuc_with_nl_pot), 64
    r, R = _walkers(hamil, B, 5, spread, 'float64')
    tw = _twists(B, J, N, 7, r)
    E1, V1, n1 = _eloc(on, r, R, tw)
    E0, V0, n0 = _eloc(off, r, R, tw)
    act = _active(hamil, np.float64, r, R)
    assert n1 == 12 * int(act.sum()) and n0 == 12 * B * J * N
    assert 0 < n1 < n0
    assert torch.isfinite(E1).all()
    assert ((E1 - E0).abs() <= 1e-13 * E0.abs().clamp(min=1)).all(), (E1 - E0).abs().max()
    assert ((V1 - V0).abs() <= 1e-13 * V0.abs().clamp(min=1)).all(), (V1 - V0).abs().max()


def test_designed_walkers_at_and_beyond_the_radius():
    """Carbon atom, fp64: every electron beyond r_c (no forwards, V_nl exactly 0, finite E_loc); every electron inside (12 N
    forwards); one electron at d2 just below rc2 (12 forwards) and just above (none) with the others beyond."""
    hamil, on = _engine('C', 'float64', True, **SMALL)
    _, off = _engine('C', 'float64', False, **SMALL)
    N = hamil.n_up + hamil.n_down
    rc = math.sqrt(float(_rc2(hamil, np.float64)[0]))
    R = torch.as_tensor(hamil.mol.coords, device=DEV, dtype=torch.float64)
    dirs = torch.tensor([[1.0, 0, 0], [0, 1.0, 0], [0, 0, 1.0], [-0.6, -0.64, 0.48]], dtype=torch.float64)[:N]
    dirs = dirs / dirs.norm(dim=-1, keepdim=True)
    far = R.cpu()[0] + dirs * (rc + 0.8)
    near = R.cpu()[0] + dirs * 0.9
    below, above = far.clone(), far.clone()
    below[0] = R.cpu()[0] + torch.tensor([1.0, 0, 0], dtype=torch.float64) * rc * math.sqrt(1 - 1e-12)
    above[0] = R.cpu()[0] + torch.tensor([1.0, 0, 0], dtype=torch.float64) * rc * math.sqrt(1 + 1e-12)
    tw1 = _twists(1, 1, N, 1, R)
    for walker, want in ((far, 0), (near, 12 * N), (below, 12), (above, 0)):
        r = walker[None].to(DEV)
        E, V, n = _eloc(on, r, R, tw1)
        assert n == want, (n, want)
        assert int(_active(hamil, np.float64, r, R).sum()) * 12 == want
        assert torch.isfinite(E).all()
        if want == 0:
            assert V.item() == 0.0
        E0, V0, _ = _eloc(off, r, R, tw1)
        assert abs(E.item() - E0.item()) <= 1e-13 * max(1.0, abs(E0.item()))


def test_benzene_walker_isolation_mixed_active_counts():
    """The kept walkers' E_loc and V_nl are bit for bit unchanged when every other walker of the batch is replaced by one with a
    different number of active pairs (compressed onto the ring: nearly all pairs; blown up: few): offsets into the group's
    pair list never mix walkers."""
    hamil, eng = _engine('benzene', 'float32', True)
    N, J, B = hamil.n_up + hamil.n_down, len(hamil.pot.nuc_with_nl_pot), 16
    r, R = _walkers(hamil, B, 21, 0.7, 'float32')
    tw = _twists(B, J, N, 9, r)
    E1, V1, _ = _eloc(eng, r, R, tw)
    r2 = r.clone()
    tight, _ = _walkers(hamil, B, 22, 0.3, 'float32')
    loose, _ = _walkers(hamil, B, 23, 1.6, 'float32')
    r2[1::4], r2[3::4] = tight[1::4], loose[3::4]
    counts = _active(hamil, np.float32, r2, R).sum((1, 2))
    assert len(set(counts.tolist())) > B // 2  # mixed active counts
    E2, V2, n2 = _eloc(eng, r2, R, tw)
    assert n2 == 12 * int(counts.sum())
    assert torch.equal(E2[0::2], E1[0::2]) and torch.equal(V2[0::2], V1[0::2])


# engines without the base walkers' tables: their switches, and the table launches per ECP group they leave out
# (env_table_kernel, embed_fwd_kernel of the embedding table)
TABLES_OFF = {'envelope_only': ((('DQMC_ECP_EMB_TABLE_OFF', 1),), 1),
              'none': ((('DQMC_ECP_EMB_TABLE_OFF', 1), ('DQMC_ECP_ENV_TABLE_OFF', 1)), 2)}


@pytest.mark.parametrize('tables', ['both', 'envelope_only', 'none'])
def test_cutoff_quadrature_chunking_bitwise(tables):
    """Benzene ccECP, 2 walkers: workspaces whose plain-forward chunks cut the active-pair list at offsets that are not
    multiples of 12 (mid-pair, mid-walker) give V_nl and E_loc bit for bit equal to the default workspace.  With the base
    walkers' embedding and envelope tables, with the envelope table only, and with neither; the engines created without a
    table launch its kernel fewer times per ECP group than the default engine, for the same walkers and workspace."""
    env, per_group = TABLES_OFF.get(tables, ((), 0))
    hamil, eng = _engine('benzene', 'float32', True, env=env)
    _, tables_on = _engine('benzene', 'float32', True)
    N, J = hamil.n_up + hamil.n_down, len(hamil.pot.nuc_with_nl_pot)
    vper = 12 * J * N
    r, R = _walkers(hamil, 2, 4, 0.7, 'float32')
    tw = _twists(2, J, N, 5, r)

    def launches(e, **kw):
        n0 = e.launch_count
        out = _eloc(e, r, R, tw, **kw)
        return out, e.launch_count - n0

    (E0, V0, n_def), n_launch = launches(eng)
    assert n_launch == launches(tables_on)[1] - per_group  # one ECP group (both walkers)
    per_walker = 12 * _active(hamil, np.float32, r, R).sum((1, 2))
    assert n_def == int(per_walker.sum()) and (per_walker < vper).all()
    prefix = eng.workspace_bytes(1, MODE_LOCAL_ENERGY) - eng.workspace_bytes(vper, MODE_FORWARD)
    for chunk in (89, 517, int(per_walker.min()) - 1):
        assert chunk % 12
        wsb = prefix + eng.workspace_bytes(chunk, MODE_FORWARD)
        assert eng.debug_plan(2, MODE_LOCAL_ENERGY, wsb)[1] == wsb
        (E1, V1, n1), n_launch = launches(eng, max_ws_bytes=wsb)
        assert n_launch == launches(tables_on, max_ws_bytes=wsb)[1] - 2 * per_group  # two ECP groups (one walker each)
        assert n1 == n_def
        assert torch.isfinite(E1).all()
        assert torch.equal(V1, V0), (chunk, V1, V0)
        assert torch.equal(E1, E0), (chunk, E1, E0)
