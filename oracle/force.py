"""fp64 oracle of the Hellmann-Feynman force estimators (reference src/deepqmc/force.py), single walker, torch autograd.

Every derivative here is taken by autograd of a closure ``log_psi(r[N, 3], R[M, 3]) -> log|psi|`` (e.g.
``lambda r, R: oracle.wf.log_psi(spec, params, r, R)``), so the oracle shares no derivative code with the engine.  The
estimators are restated from the cited lines of the reference for Cartesian nuclear coordinates, all-electron.
"""
import torch

F64 = torch.float64


def _eps():
    return torch.finfo(F64).eps


def nuclear_energy(R, Z):
    # reference physics.py:112-116 (eps-safe pairwise distances)
    Z = torch.as_tensor(Z, dtype=F64)
    n = len(Z)
    if n < 2:
        return torch.zeros((), dtype=F64)
    i, j = torch.triu_indices(n, n, 1)
    d = R[i] - R[j]
    return (Z[i] * Z[j] / torch.sqrt(_eps() + (d * d).sum(-1))).sum()


def nuclear_force(R, Z):
    """-grad_R E_nuc [M, 3] (reference force.py:30-38)."""
    if R.shape[0] < 2:
        return torch.zeros_like(R)
    R = R.detach().clone().requires_grad_(True)
    (g,) = torch.autograd.grad(nuclear_energy(R, Z), R)
    return -g


def local_potential(r, R, Z):
    # electron-nucleus Coulomb attraction on the plain norm (reference physics.py:124-140)
    Z = torch.as_tensor(Z, dtype=F64)
    return -(Z / torch.linalg.norm(r[:, None] - R[None], dim=-1)).sum()


def grad_r(log_psi, r, R):
    """grad_r log|psi| [N, 3] (reference force.py:109-118)."""
    r = r.detach().clone().requires_grad_(True)
    (g,) = torch.autograd.grad(log_psi(r, R.detach()), r)
    return g


def grad_R(log_psi, r, R):
    """grad_R log|psi| [M, 3] (reference force.py:96-106)."""
    R = R.detach().clone().requires_grad_(True)
    (g,) = torch.autograd.grad(log_psi(r.detach(), R), R)
    return g


def Q(r, R, c):
    """Q_m = c_m sum_i d_im / |d_im| [M, 3] (reference force.py:122-132)."""
    c = torch.as_tensor(c, dtype=F64)
    d = r[None] - R[:, None]
    return (c[:, None, None] * d / torch.linalg.norm(d, dim=-1, keepdim=True)).sum(-2)


def dQ_dr(r, R, c):
    """jacfwd(Q) with respect to r: [M, 3, N, 3]."""
    return torch.autograd.functional.jacobian(lambda x: Q(x, R, c), r.detach())


def force_bare(r, R, Z):
    """F_nuc - grad_R V_loc [M, 3] (reference force.py:250-301, all-electron)."""
    R_ = R.detach().clone().requires_grad_(True)
    (g,) = torch.autograd.grad(local_potential(r.detach(), R_, Z), R_)
    return nuclear_force(R, Z) - g


def force_ac_zvq(r, R, Z, g_r):
    """sum_{i,b} g_r[i, b] dQ[m, a, i, b] + F_nuc (reference force.py:172-194)."""
    return (g_r[None, None] * dQ_dr(r, R, Z)).sum((-1, -2)) + nuclear_force(R, Z)


def force_ac_zvzbq(r, R, Z, g_r, e_loc, energy):
    """ZVQ - 2 (E_loc - energy) Q (reference force.py:536-546)."""
    return force_ac_zvq(r, R, Z, g_r) - 2 * (e_loc - energy) * Q(r, R, Z)


def force_ac_zb(r, R, Z, g_R, e_loc, energy):
    """bare - 2 (E_loc - energy) grad_R log|psi| (reference force.py:437-447)."""
    return force_bare(r, R, Z) - 2 * (e_loc - energy) * g_R


def force_ac_zvqzb(r, R, Z, g_r, g_R, e_loc, energy):
    """ZVQ - 2 (E_loc - energy) grad_R log|psi| (reference force.py:643-654)."""
    return force_ac_zvq(r, R, Z, g_r) - 2 * (e_loc - energy) * g_R


def antithetic_mirror(r, R, r_cut):
    """r - 2 (r - R_nn) for electrons with |r - R_nn|^2 < r_cut^2 (reference force.py:197-203, sampling_utils.py:72-75)."""
    d = r[:, None] - R[None]
    d2 = (d * d).sum(-1)
    idx = torch.argmin(d2, -1)
    dn = d[torch.arange(len(r)), idx]
    return r - 2 * dn * (d2[torch.arange(len(r)), idx] < r_cut**2)[:, None]


def antithetic(force_fn, log_psi, r, R, r_cut):
    """softmax(0, 2 dlog|psi|)-weighted average of force_fn(r, R) and force_fn(mirrored r, R) (reference force.py:237-247)."""
    r_ = antithetic_mirror(r, R, r_cut)
    lw = 2 * (log_psi(r_, R) - log_psi(r, R))
    w = torch.softmax(torch.stack([torch.zeros_like(lw), lw]), 0)
    return w[0] * force_fn(r, R) + w[1] * force_fn(r_, R)


def fd_displacements(r, R, h):
    """-> [(R_k, r_k)] for the 3M nuclear coordinates (reference force.py:579-590)."""
    out = []
    M = R.shape[0]
    dists = torch.linalg.norm(R[:, None] - r[None], dim=-1)  # [M, N]
    w = torch.exp(-dists) / torch.exp(-dists).sum(-2, keepdim=True)
    for k in range(3 * M):
        dR = torch.zeros(M * 3, dtype=F64)
        dR[k] = h
        dR = dR.reshape(M, 3)
        out.append((R - dR, r + torch.einsum('nj,ne->ej', dR, w)))
    return out


def force_finite_difference(local_energy, log_psi, r, R, h, e_loc):
    """exp(2 (log psi' - log psi)) (E' - E_loc) / h [M, 3] (reference force.py:576-604); local_energy(r, R) -> E."""
    lp0 = log_psi(r, R)
    vals = [torch.exp(2 * (log_psi(rk, Rk) - lp0)) * (local_energy(rk, Rk) - e_loc) / h for Rk, rk in fd_displacements(r, R, h)]
    return torch.stack(vals).reshape(R.shape)
