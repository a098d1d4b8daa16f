"""CPU: the ECP force oracle (tests/ecp_force_oracle.py) -- differentiable quadrature points, the closed-form Jacobian of the
quadrature point that the engine evaluates, the non-local gradient against finite differences, the local ECP force -- and the
workspace plan of dqmc_ecp_force (DQMC_MODE_ECP_FORCE) on plan-only engines."""
import math

import numpy as np
import pytest
import torch

import ecp_force_oracle as EO
from deepqmc_b200 import params as PN
from deepqmc_b200.ansatz import B200Ansatz
from deepqmc_b200.engine import MODE_ECP_FORCE, Engine
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from deepqmc_b200.spec import ferminet_spec, psiformer_spec
from oracle import wf as W
from oracle.hamil import OracleHamiltonian
from spin_fixture import walkers

F64 = torch.float64
SMALL = dict(embedding_dim=32, n_layers=2, n_heads=4, n_determinants=4)


def test_quadrature_points_match_the_oracle_hamiltonian():
    oh = OracleHamiltonian(Molecule.from_name('C'), ecp_type='ccECP')
    g = np.random.default_rng(0)
    for _ in range(20):
        ri, RI = torch.as_tensor(g.normal(size=3)), torch.as_tensor(g.normal(size=3))
        tw = float(g.uniform(0, math.pi / 5))
        ref = oh.quadrature_points(ri, RI, tw)
        assert float((EO.quadrature_points(ri, RI, tw) - ref).abs().max()) <= 1e-15 * max(1.0, float(ref.abs().max()))


def test_closed_form_jacobian_matches_autograd():
    g = np.random.default_rng(1)
    for _ in range(20):
        d = g.normal(size=3)
        tw = float(g.uniform(0, math.pi / 5))
        ref = torch.autograd.functional.jacobian(lambda x: EO.quadrature_points(x, torch.zeros(3, dtype=F64), tw),
                                                 torch.as_tensor(d))
        got = EO.jacobian_closed_form(d, tw)
        assert np.abs(got - ref.numpy()).max() <= 1e-12
        # u_q = +-e_z (vertices 0 and 1): f_q = +-d, so df_q/dd = +-1 (to rounding)
        assert np.abs(got[0] - np.eye(3)).max() <= 1e-14 and np.abs(got[1] + np.eye(3)).max() <= 1e-14


def _psiformer(mol, ecp='ccECP'):
    h = MolecularHamiltonian(mol=mol, ecp_type=ecp)
    a = B200Ansatz(h, 'psiformer', dtype='float64', **SMALL)
    params = PN.perturb_params(a.init(0))
    pt = W.to_torch(params)
    return h, OracleHamiltonian(mol, ecp_type=ecp), (lambda x, y: W.log_psi(a.spec, pt, x, y))


@pytest.mark.parametrize('name', ['LiH', 'CH4_c_last'])
def test_nonlocal_gradient_matches_central_differences(name):
    """Row I of grad_nonloc_potential = the central difference of nucleus I's share of V_nl in R_I (fixed twists, fp64)."""
    mol = _mol(name)
    h, oh, lp = _psiformer(mol)
    r = torch.as_tensor(walkers(h, 1, seed=3)[0])
    R = torch.as_tensor(mol.coords)
    nl_nuc = np.unique(np.nonzero(oh.nl_params)[0])
    tw = torch.as_tensor(np.random.default_rng(2).uniform(0, math.pi / 5, size=(len(nl_nuc), r.shape[0])))
    got = EO.grad_nonloc_potential(oh, lp, r, R, tw)
    h_ = 1e-5
    for j, I in enumerate(nl_nuc):
        for c in range(3):
            Rp, Rm = R.clone(), R.clone()
            Rp[I, c] += h_
            Rm[I, c] -= h_
            fd = (EO.nonloc_share(oh, lp, r, Rp, tw, I, j) - EO.nonloc_share(oh, lp, r, Rm, tw, I, j)) / (2 * h_)
            assert abs(float(got[I, c] - fd)) <= 1e-6 * max(1.0, abs(float(fd))), (I, c, float(got[I, c]), float(fd))
    others = [m for m in range(len(R)) if m not in nl_nuc]
    assert float(got[others].abs().max()) == 0.0 if others else True


def _np_local_force(r, R, Zv, loc):
    """F_nuc(Z_eff) + Z_m sum_i d / |d|^3 + V_ecp'(rho) d / rho: the closed form of force_terms_kernel, restated."""
    eps = np.finfo(np.float64).eps
    F = np.zeros_like(R)
    for m in range(len(R)):
        for n in range(len(R)):
            if n != m:
                d = R[m] - R[n]
                F[m] += Zv[m] * Zv[n] * d / np.sqrt(eps + d @ d) ** 3
        for ri in r:
            d = ri - R[m]
            rho = np.linalg.norm(d)
            F[m] += Zv[m] * d / rho**3
            if loc is not None:
                a, b = loc[m, :, 0], loc[m, :, 1]  # [3, T]
                dv = (b[0] * np.exp(-a[0] * rho**2) * (-1 / rho**2 - 2 * a[0])).sum()
                dv += (-2 * a[1] * rho * b[1] * np.exp(-a[1] * rho**2)).sum()
                dv += (b[2] * np.exp(-a[2] * rho**2) * (1 - 2 * a[2] * rho**2)).sum()
                F[m] += dv * d / rho
    return F


@pytest.mark.parametrize('name,ecp', [('LiH', 'ccECP'), ('C', 'bfd'), ('CH4_c_last', 'ccECP'), ('LiH', None)])
def test_local_ecp_force_matches_autograd(name, ecp):
    mol = _mol(name)
    oh = OracleHamiltonian(mol, ecp_type=ecp)
    R = np.asarray(mol.coords)
    for s in range(3):
        r = walkers(MolecularHamiltonian(mol=mol, ecp_type=ecp), 1, seed=s)[0]
        got = EO.force_bare_local(oh, torch.as_tensor(r), torch.as_tensor(R)).numpy()
        ref = _np_local_force(r, R, oh.ns_valence, oh.loc_params)
        assert np.abs(got - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())


def _mol(name):
    if name == 'CH4_c_last':  # carbon is not nucleus 0: its non-local force belongs in row 4, not row 0
        m = Molecule.from_name('CH4')
        return Molecule(coords=np.asarray(m.coords)[[1, 2, 3, 4, 0]].tolist(), charges=[1, 1, 1, 1, 6], charge=0, spin=0,
                        unit='bohr')
    return Molecule.from_name(name)


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('name', ['LiH', 'CH4_c_last'])
def test_ecp_force_plan_carved_never_exceeds_planned(built_lib, name, dtype):
    h = MolecularHamiltonian(mol=_mol(name), ecp_type='ccECP')
    for spec in (psiformer_spec(h, **SMALL), ferminet_spec(h, **dict(SMALL, edge_dim=8))):
        eng = Engine(spec, h, dtype=dtype, plan_only=True, gemm_backend=1 if dtype == 'float32' else 0)
        for B in (1, 257, 4096):
            planned, carved = eng.debug_plan(B, MODE_ECP_FORCE)
            assert planned == eng.workspace_bytes(B, MODE_ECP_FORCE)
            assert 0 < carved <= planned, (spec.kind, B, dtype, planned, carved)
            floor = eng.workspace_bytes_min(B, MODE_ECP_FORCE)
            assert 0 < floor <= planned
            for cap in {max(floor, planned // 3), floor}:
                _, c2 = eng.debug_plan(B, MODE_ECP_FORCE, cap)
                assert 0 < c2 <= cap, (spec.kind, B, dtype, cap, c2)
            with pytest.raises(RuntimeError, match='workspace'):
                eng.debug_plan(B, MODE_ECP_FORCE, floor // 2)
        eng.close()
