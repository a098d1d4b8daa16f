"""CPU: the two oracle formulations of the AC-ZV zero-variance term (zv_force_oracle.zv_term, the reference's local energy of
d psi / dR_k, and kinetic_nuclear_gradient, -dT/dR by autograd) against each other and against central differences of the
oracle's kinetic energy; the algebra of the AC-ZV / AC-ZVZB mirrors of deepqmc_b200/force.py on a stub engine; the workspace
plan of dqmc_zv_force (DQMC_MODE_ZV_FORCE) on plan-only engines."""
import dataclasses
import types

import pytest
import torch

from deepqmc_b200 import force as FO
from deepqmc_b200 import params as PN
from deepqmc_b200.ansatz import B200Ansatz
from deepqmc_b200.engine import MODE_ZV_FORCE, Engine
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from deepqmc_b200.spec import ferminet_spec, paulinet_spec, psiformer_spec, transpsiformer_spec
from deepqmc_b200.types import PhysicalConfiguration
from oracle import wf as W
from oracle.hamil import OracleHamiltonian
from spin_fixture import walkers
import zv_force_oracle as ZO

SMALL = dict(embedding_dim=32, n_layers=2, n_heads=4, n_determinants=4)
HYPER = {'psiformer': SMALL, 'ferminet': dict(embedding_dim=32, n_layers=2, n_determinants=4, edge_dim=8)}


def _problem(mol, kind):
    h = MolecularHamiltonian(mol=Molecule.from_name(mol))
    a = B200Ansatz(h, kind, dtype='float64', **HYPER[kind])
    pt = W.to_torch(PN.perturb_params(a.init(0)))
    lp = lambda x, y: W.log_psi(a.spec, pt, x, y)[1]
    r = torch.as_tensor(walkers(h, 1, seed=1))[0]
    return h, lp, r, torch.as_tensor(h.mol.coords)


@pytest.mark.parametrize('kind', ['psiformer', 'ferminet'])
@pytest.mark.parametrize('mol', ['LiH', 'N2'])
def test_oracle_zv_formulations_agree(mol, kind):
    """The reference's formulation -(E'_k - e_loc) g_k with the walker's exact local energy equals -dT/dR (1e-9), and both
    equal central differences of the oracle's kinetic energy in R at fixed r."""
    h, lp, r, R = _problem(mol, kind)
    oh = OracleHamiltonian(h.mol)
    e_loc = oh.local_energy(lambda x: (None, lp(x, R)), r, R)[0].detach()
    zv = ZO.zv_term(oh, lp, r, R, e_loc).detach()
    kg = ZO.kinetic_nuclear_gradient(lp, r, R)
    scale = max(1.0, float(kg.abs().max()))
    assert float((zv - kg).abs().max()) <= 1e-9 * scale
    step, fd = 1e-4, torch.empty_like(R)
    for k in range(R.numel()):
        dR = torch.zeros(R.numel(), dtype=R.dtype)
        dR[k] = step
        dR = dR.reshape(R.shape)
        fd.reshape(-1)[k] = -(ZO.kinetic_energy(lp, r, R + dR) - ZO.kinetic_energy(lp, r, R - dR)).detach() / (2 * step)
    # central differences: O(h^2) truncation (measured below 1e-6 of the scale on these walkers)
    assert float((fd - kg).abs().max()) <= 1e-5 * scale


def test_zv_mirror_algebra():
    """AC-ZV = bare + f_zv and AC-ZVZB = bare + f_zv - 2 (E_loc - energy) grad_R log|psi| on a stub engine, single walker
    and batch; the ValueError of the kinds and Hamiltonians without the companion pass."""
    g = torch.Generator().manual_seed(0)
    B, M, N = 3, 2, 4
    bare, zv, gR = (torch.randn(B, M, 3, generator=g, dtype=torch.float64) for _ in range(3))
    spec = types.SimpleNamespace(kind='ferminet', backflow_transform='mult')
    calls = []

    class Eng:
        def __init__(self):
            self.spec = spec

        def force_terms(self, r, R):
            return bare[: r.shape[0]], None, None

        def zv_force(self, r, R, want_grad_R=False):
            calls.append(want_grad_R)
            return zv[: r.shape[0]], gR[: r.shape[0]] if want_grad_R else None

    hamil = types.SimpleNamespace(loc_params=None, ph=None, ecp_type=None)
    mp = pytest.MonkeyPatch()
    mp.setattr(FO, '_engine', lambda h, wf, p: Eng())
    try:
        r = torch.randn(B, N, 3, generator=g, dtype=torch.float64)
        R = torch.randn(M, 3, generator=g, dtype=torch.float64)
        pc = PhysicalConfiguration(R, r, torch.zeros(B))
        e_loc, energy = torch.tensor([-1.0, -1.5, -0.7], dtype=torch.float64), -1.1
        got = FO.evaluate_hf_force_ac_zv(hamil, None)(0, None, pc)
        assert torch.equal(got, bare + zv) and calls == [False]
        got = FO.evaluate_hf_force_ac_zvzb(hamil, None)(0, None, pc, e_loc, energy)
        assert torch.allclose(got, bare + zv - 2 * (e_loc - energy)[:, None, None] * gR, rtol=1e-15, atol=1e-15)
        one = FO.evaluate_hf_force_ac_zvzb(hamil, None)(0, None, PhysicalConfiguration(R, r[0], torch.zeros(())), e_loc[:1],
                                                        energy)
        assert one.shape == (M, 3) and torch.allclose(one, got[0], rtol=1e-15, atol=1e-15)
        spec.kind = 'paulinet'
        with pytest.raises(ValueError, match='paulinet'):
            FO.evaluate_hf_force_ac_zv(hamil, None)(0, None, pc)
        spec.kind = 'psiformer'
        hamil.loc_params, hamil.ecp_type = object(), 'ccECP'
        with pytest.raises(ValueError, match='ccECP'):
            FO.evaluate_hf_force_ac_zvzb(hamil, None)(0, None, pc, e_loc, energy)
    finally:
        mp.undo()


def _engine(spec, h, dtype):
    return Engine(spec, h, dtype=dtype, plan_only=True, gemm_backend=1 if dtype == 'float32' and spec.embedding_dim % 32 == 0 else 0)


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('mol', ['LiH', 'N2'])
def test_zv_plan_carved_never_exceeds_planned(built_lib, mol, dtype):
    h = MolecularHamiltonian(mol=Molecule.from_name(mol))
    for spec in (psiformer_spec(h, **SMALL), ferminet_spec(h, **dict(SMALL, edge_dim=8))):
        eng = _engine(spec, h, dtype)
        for B in (1, 257, 4096):
            planned, carved = eng.debug_plan(B, MODE_ZV_FORCE)
            assert planned == eng.workspace_bytes(B, MODE_ZV_FORCE)
            assert 0 < carved <= planned, (spec.kind, B, dtype, planned, carved)
            floor = eng.workspace_bytes_min(B, MODE_ZV_FORCE)
            assert 0 < floor <= planned
            for cap in {max(floor, planned // 3), floor}:
                _, c2 = eng.debug_plan(B, MODE_ZV_FORCE, cap)
                assert 0 < c2 <= cap, (spec.kind, B, dtype, cap, c2)
            with pytest.raises(RuntimeError, match='workspace'):
                eng.debug_plan(B, MODE_ZV_FORCE, floor // 2)
        eng.close()


def test_zv_plan_refused_kinds(built_lib):
    """No workspace and status 2 for the TransPsiformer, the conv-GNN kinds, the additive backflow branch and ECP engines."""
    h = MolecularHamiltonian(mol=Molecule.from_name('LiH'))
    he = MolecularHamiltonian(mol=Molecule.from_name('LiH'), ecp_type='ccECP')
    bf = dataclasses.replace(psiformer_spec(h, **SMALL), backflow_transform='add')
    for spec, hh in ((transpsiformer_spec(h, **SMALL), h), (paulinet_spec(h), h), (bf, h), (psiformer_spec(he, **SMALL), he)):
        eng = _engine(spec, hh, 'float64')
        assert eng.workspace_bytes(8, MODE_ZV_FORCE) == 0
        with pytest.raises(RuntimeError, match=r'\(2\)'):
            eng.debug_plan(8, MODE_ZV_FORCE)
        eng.close()
