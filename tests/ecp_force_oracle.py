"""fp64 oracle of the ECP parts of the bare Hellmann-Feynman force (reference force.py:252-301,
ecp/gaussian_type_ecp.py:127-159 local_potential, :257-328 grad_nonloc_potential, ecp/ecp_force_utils.py), single walker, torch
autograd.  Shared by test_ecp_force_host.py and test_gpu_ecp_force.py.

The quadrature points are restated from oracle/hamil.py's ``OracleHamiltonian.quadrature_points`` (reference ecp_utils.py:34-60)
in differentiable torch, so that autograd carries the points' motion with R_I.  ``log_psi(r[N, 3], R[M, 3]) -> (sign, log)``
(e.g. ``lambda r, R: oracle.wf.log_psi(spec, params, r, R)``).  Nucleus I's non-local force is written into row I.
"""
import math

import numpy as np
import torch

from oracle import force as OF
from oracle.hamil import icosahedron, legendre_values

F64 = torch.float64


def _rot_y(t):
    c, s, o, z = torch.cos(t), torch.sin(t), torch.ones_like(t), torch.zeros_like(t)
    return torch.stack([torch.stack([c, z, s]), torch.stack([z, o, z]), torch.stack([-s, z, c])])


def _rot_z(p):
    c, s, o, z = torch.cos(p), torch.sin(p), torch.ones_like(p), torch.zeros_like(p)
    return torch.stack([torch.stack([c, -s, z]), torch.stack([s, c, z]), torch.stack([z, z, o])])


def quadrature_points(r_i, R_I, phi_random):
    """[12, 3] quadrature points of electron i around nucleus I, differentiable in r_i and R_I."""
    _, ico = icosahedron()
    diff = r_i - R_I
    radius = torch.linalg.norm(diff)
    theta = torch.acos(torch.clamp(diff[2] / radius, -1.0, 1.0))
    phi = torch.atan2(diff[1], diff[0])
    rot = _rot_z(phi) @ _rot_y(theta) @ _rot_z(torch.as_tensor(float(phi_random), dtype=F64))
    return radius * (torch.as_tensor(ico) @ rot.T) + R_I


def jacobian_closed_form(d, phi_random):
    """df_q/dd [12, 3, 3] of f_q(d) = rho Rz(phi) Ry(theta) Rz(phi_random) u_q, restated in numpy from the closed form the engine
    evaluates (kernels_mcmc.cuh ecp_force_accumulate_kernel)."""
    d = np.asarray(d, dtype=np.float64)
    rho = np.linalg.norm(d)
    s = math.hypot(d[0], d[1])
    th, ph = math.acos(np.clip(d[2] / rho, -1, 1)), math.atan2(d[1], d[0])
    _, ico = icosahedron()
    c, sn = math.cos(phi_random), math.sin(phi_random)
    w = ico @ np.array([[c, -sn, 0], [sn, c, 0], [0, 0, 1]]).T
    ct, st, cp, sp = math.cos(th), math.sin(th), math.cos(ph), math.sin(ph)
    Ry = np.array([[ct, 0, st], [0, 1, 0], [-st, 0, ct]])
    dRy = np.array([[-st, 0, ct], [0, 0, 0], [-ct, 0, -st]])
    Rz = np.array([[cp, -sp, 0], [sp, cp, 0], [0, 0, 1]])
    dRz = np.array([[-sp, -cp, 0], [cp, -sp, 0], [0, 0, 0]])
    dth = (d[2] * d / rho**2 - np.array([0, 0, 1.0])) / s
    dph = np.array([-d[1], d[0], 0.0]) / s**2
    f = rho * w @ (Rz @ Ry).T
    t1 = rho * w @ (Rz @ dRy).T
    t2 = rho * w @ (dRz @ Ry).T
    return f[:, :, None] * (d / rho**2)[None, None] + t1[:, :, None] * dth[None, None] + t2[:, :, None] * dph[None, None]


def nonloc_share(oh, log_psi, r, R, phi_random, I, j):
    """Nucleus I's share of V_nl, sum_i sum_l (2l+1)/12 v_l(|r_i - R_I|) sum_q P_l(cos th_q) psi(r_q) / psi(r), with every
    quadrature point and psi itself depending on R (reference gaussian_type_ecp.py:161-255); phi_random[j, i]."""
    nlp = oh.nl_params
    thetas, _ = icosahedron()
    L = nlp.shape[1]
    leg = torch.as_tensor(legendre_values(L, np.cos(thetas)))  # [12, L]
    coefs = torch.as_tensor((np.arange(L) * 2 + 1) / 12.0)
    a, b = torch.as_tensor(nlp[I, :, 0, :]), torch.as_tensor(nlp[I, :, 1, :])
    s0, l0 = log_psi(r, R)
    total = torch.zeros((), dtype=F64)
    for i in range(r.shape[0]):
        dist = torch.linalg.norm(r[i] - R[I])
        v_l = (b * torch.exp(-a * dist**2)).sum(-1)
        pts = quadrature_points(r[i], R[I], phi_random[j, i])
        ratios = []
        for q in range(12):
            rq = torch.cat([r[:i], pts[q][None], r[i + 1:]])
            sq, lq = log_psi(rq, R)
            ratios.append(torch.exp(lq - l0) * sq * s0)
        total = total + (v_l * coefs * (torch.stack(ratios)[:, None] * leg).sum(0)).sum()
    return total


def grad_nonloc_potential(oh, log_psi, r, R, phi_random):
    """[M, 3]: row I = d/dR_I of nucleus I's share of V_nl (autograd with respect to all of R, row I kept; reference
    gaussian_type_ecp.py:257-328, ecp_force_utils.py:37-68).  The force is its negative."""
    out = torch.zeros(R.shape, dtype=F64)
    if oh.nl_params is None:
        return out
    for j, I in enumerate(np.unique(np.nonzero(oh.nl_params)[0])):
        Rv = R.detach().clone().requires_grad_(True)
        (g,) = torch.autograd.grad(nonloc_share(oh, log_psi, r.detach(), Rv, phi_random, I, j), Rv)
        out[I] = g[I]
    return out


def force_bare_local(oh, r, R):
    """F_nuc(Z_eff) - grad_R V_loc [M, 3], V_loc = OracleHamiltonian.local_potential (Coulomb on Z_eff + the local ECP)."""
    Rv = R.detach().clone().requires_grad_(True)
    (g,) = torch.autograd.grad(oh.local_potential(r.detach(), Rv), Rv)
    return OF.nuclear_force(R, oh.ns_valence) - g


def force_bare(oh, log_psi, r, R, phi_random):
    """The bare force with an ECP [M, 3]: force_bare_local - grad_nonloc_potential."""
    return force_bare_local(oh, r, R) - grad_nonloc_potential(oh, log_psi, r, R, phi_random)
