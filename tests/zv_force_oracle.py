"""fp64 oracle of the AC-ZV / AC-ZVZB force estimators (reference force.py:135-169 make_zv_term_via_jvp, :41-57
make_general_jvp_nuc_wf, :304-411 evaluate_hf_force_ac_zv / evaluate_hf_force_ac_zvzb), single walker, torch autograd of a
closure ``log_psi(r[N, 3], R[M, 3]) -> log|psi|`` (e.g. ``lambda r, R: oracle.wf.log_psi(spec, params, r, R)[1]``), Cartesian
nuclear coordinates, all-electron.  Shared by test_zv_force_host.py and test_gpu_zv_force.py; imports nothing from the product.

Two formulations of the zero-variance term: ``zv_term`` restates the reference literally (the local energy of
d psi / dR_k minus e_loc, times d_k log|psi|), ``kinetic_nuclear_gradient`` is -dT/dR at fixed r.  They agree when e_loc is
the walker's exact local energy.
"""
import torch

from oracle import force as OF


def _lap_grad(f, x):
    """(Hessian trace, gradient) of scalar f at x[3N] by reverse-mode autograd with create_graph, so that both stay
    differentiable in whatever else f depends on.  (Nesting torch.func transforms to third order through slogdet gives wrong
    values in the torch this was written against; plain autograd agrees with central differences.)"""
    x = x.detach().clone().requires_grad_(True)
    (g,) = torch.autograd.grad(f(x), x, create_graph=True)
    lap = sum(torch.autograd.grad(g[k], x, create_graph=True)[0][k] for k in range(x.numel()))
    return lap, g


def kinetic_energy(log_psi, r, R):
    """T = -1/2 (Lap_r log|psi| + |grad_r log|psi||^2) (the hamil/E_kin statistic), differentiable in R."""
    lap, g = _lap_grad(lambda x: log_psi(x.reshape(r.shape), R), r.reshape(-1))
    return -0.5 * (lap + (g * g).sum())


def kinetic_nuclear_gradient(log_psi, r, R):
    """-dT/dR [M, 3] at fixed r by autograd of the kinetic energy: the closed form of zv_term for an all-electron
    Hamiltonian when e_loc is the walker's exact local energy."""
    R = R.detach().clone().requires_grad_(True)
    (g,) = torch.autograd.grad(kinetic_energy(log_psi, r.detach(), R), R)
    return -g


def zv_term(hamil, log_psi, r, R, e_loc):
    """-(E'_k - e_loc) g_k [M, 3] for the 3M Cartesian nuclear coordinates k (reference force.py:135-169, 41-57): E'_k is the
    local energy of psi'_k = d psi / dR_k, i.e. of log|psi| + log|d_k log psi|, with its Hessian-trace Laplacian and the
    potentials of ``hamil`` (an all-electron ``oracle.hamil.OracleHamiltonian``); g_k = d_k log|psi|."""
    r, R = r.detach(), R.detach()
    g = OF.grad_R(log_psi, r, R)
    pot = hamil.local_potential(r, R) + hamil.electronic_potential(r) + hamil.nuclear_energy(R)
    out = []
    for k in range(R.numel()):
        def log_psi_k(x, k=k):
            x = x.reshape(r.shape)
            y = R.clone().requires_grad_(True)
            lp = log_psi(x, y)
            (dlp,) = torch.autograd.grad(lp, y, create_graph=True)
            return lp + torch.log(torch.abs(dlp.reshape(-1)[k]))
        lap, gr = _lap_grad(log_psi_k, r.reshape(-1))
        out.append(-0.5 * (lap + (gr * gr).sum()) + pot)
    return -(torch.stack(out).reshape(R.shape) - e_loc) * g


def force_ac_zv(r, R, Z, f_zv):
    """bare + f_zv (reference force.py:343-355)."""
    return OF.force_bare(r, R, Z) + f_zv


def force_ac_zvzb(r, R, Z, f_zv, g_R, e_loc, energy):
    """bare + f_zv - 2 (E_loc - energy) grad_R log|psi| (reference force.py:394-411)."""
    return OF.force_bare(r, R, Z) + f_zv - 2 * (e_loc - energy) * g_R
