"""Hellmann-Feynman force estimators on top of the engine's position gradients (``dqmc_wf_grad_positions``) and closed-form
force terms (``dqmc_force_terms``, and ``dqmc_ecp_force`` with an effective core potential).

Mirror of the reference's ``force.py`` (Cartesian nuclear coordinates) with its names and argument order.  Every estimator
factory takes ``(hamil, ansatz.apply)`` and returns a batched callable: ``phys_conf`` carries r [B, N, 3] and R [M, 3] or
[B, M, 3], the forces come back as [B, M, 3].  The ``(E_loc - energy)`` algebra is elementwise torch, as in ``spin.py``.

grad_r log|psi| comes from the reverse pass where the ansatz kind has one and from the forward-Laplacian pass of
``dqmc_local_energy`` otherwise, so the ZVQ family runs on every kind; grad_R log|psi| (the zero-bias estimators) needs the
reverse pass into the nuclear coordinates: Psiformer and FermiNet.

With a Gaussian-type ECP the bare force (and so AC-ZB and the antithetic wrapper around bare) adds -grad_R of the local ECP
and the non-local part -grad_nonloc_potential (``dqmc_ecp_force``; Psiformer and FermiNet).  As in the reference, every
(nucleus, electron) pair of a walker shares one quadrature twist, drawn per walker from ``rng`` (the energy pass draws one per
pair); unlike the reference, nucleus I's non-local force lands in row I, not in row j (its index among the non-local nuclei):
the two agree when the ECP nuclei come first, as in every molecule the reference ships.  The ZVQ family refuses ECP engines,
which the reference documents as incompatible.

AC-ZV and AC-ZVZB take their zero-variance term from the wave function itself: the reference evaluates the local energy
E'_kappa of psi'_kappa = d psi / dR_kappa and forms -(E'_kappa - E_loc) d_kappa log|psi|.  With an all-electron Hamiltonian
the potential cancels there, and the term equals -dT/dR_kappa at fixed electron positions (T the local kinetic energy)
whenever E_loc is the walker's exact local energy, as the reference's monitors pass it.  ``dqmc_zv_force`` computes that
closed form by a nuclear-coordinate companion of the forward-Laplacian pass (Psiformer and FermiNet with multiplicative
backflow); it neither divides by d_kappa log|psi| nor reads ``e_loc``.  ECP engines are refused (the reference's E'_kappa
then contains the non-local operator acting on psi').
"""
from __future__ import annotations

import torch

from .spin import _ansatz_of, weighted_std
from .types import PhysicalConfiguration


def _batched(phys_conf):
    r, R = phys_conf.r, phys_conf.R
    single = r.dim() == 2
    return (r[None] if single else r), R, single


def _unbatch(x, single):
    return x[0] if single and x is not None else x


def nuclear_force(R, phys_conf: PhysicalConfiguration, nuclear_charges):
    """-grad_R of the nuclear repulsion sum_{I<J} Z_I Z_J / |R_I - R_J| (eps-safe norm) -> [..., M, 3]
    (reference force.py:30-38; ``phys_conf`` is accepted for the reference's signature)."""
    Z = torch.as_tensor(nuclear_charges, dtype=R.dtype, device=R.device)
    d = R[..., :, None, :] - R[..., None, :, :]
    rho = torch.sqrt(torch.finfo(R.dtype).eps + (d * d).sum(-1))
    w = Z[:, None] * Z[None, :] / rho**3
    w = w * (1 - torch.eye(len(Z), dtype=R.dtype, device=R.device))
    return (w[..., None] * d).sum(-2)


def Q(r, R, c):
    """Q_m = c_m sum_i (r_i - R_m) / |r_i - R_m| -> [..., M, 3] (reference force.py:122-132, plain norm)."""
    c = torch.as_tensor(c, dtype=r.dtype, device=r.device)
    d = r[..., None, :, :] - R[..., :, None, :]
    return c[:, None] * (d / torch.linalg.norm(d, dim=-1, keepdim=True)).sum(-2)


def diffs_to_nearest_nuc(r, R):
    """-> (z [..., N, 4] = (r_i - R_nn, |r_i - R_nn|^2), idx [..., N]): the nearest nucleus by the squared distance, the first
    index on ties (reference sampling_utils.py:72-75)."""
    d = r[..., :, None, :] - R[..., None, :, :]
    z = torch.cat([d, (d * d).sum(-1, keepdim=True)], -1)
    idx = torch.argmin(z[..., -1], dim=-1)
    return torch.gather(z, -2, idx[..., None, None].expand(*idx.shape, 1, 4)).squeeze(-2), idx


def antithetic_sampler(phys_conf: PhysicalConfiguration, r_cut: float):
    """-> (phys_conf, mirrored): electrons within ``r_cut`` of their nearest nucleus mirrored through it, r -> 2 R_nn - r
    (reference force.py:197-203)."""
    z, _ = diffs_to_nearest_nuc(phys_conf.r, phys_conf.R)
    r_ = phys_conf.r - 2 * z[..., :3] * (z[..., -1] < r_cut**2)[..., None]
    return phys_conf, phys_conf.replace(r=r_)


def antithetic_wrapper(evaluate_force, wf, r_cut: float):
    """Antithetic-sampling variance reduction of an estimator ``(rng, params, phys_conf) -> [B, M, 3]``: the importance-
    weighted average of the force on the walkers and on their mirrored copies, weights softmax over (0, 2 dlog|psi|) in fp64
    (reference force.py:206-247).  The mirrored copies get the rng ``rng + 1``."""

    def evaluate_force_antithetic(rng, params, phys_conf: PhysicalConfiguration):
        phys_conf, phys_conf_ = antithetic_sampler(phys_conf, r_cut)
        log_weight_ = 2 * (wf(params, phys_conf_).log.double() - wf(params, phys_conf).log.double())
        weights = torch.softmax(torch.stack((torch.zeros_like(log_weight_), log_weight_), 0), 0)
        rng_ = None if rng is None else rng + 1
        force = evaluate_force(rng, params, phys_conf)
        force_ = evaluate_force(rng_, params, phys_conf_)
        w = weights.to(force.dtype)[..., None, None]
        return w[0] * force + w[1] * force_

    return evaluate_force_antithetic


def _engine(hamil, wf, params):
    return _ansatz_of(wf).engine_for(hamil, params)


def _grad_r(eng, r, R):
    """grad_r log|psi| [B, N, 3]: reverse pass where the kind has one, forward-Laplacian pass otherwise."""
    spec = eng.spec
    if spec.kind in ('psiformer', 'ferminet', 'transpsiformer') and spec.backflow_transform == 'mult':
        return eng.grad_positions(r, R, want_r=True, want_R=False)[2]
    grad = eng.local_energy(r, R, want_grad=True)[4]
    return grad.reshape(r.shape)


def _grad_R(eng, r, R):
    spec = eng.spec
    if spec.kind not in ('psiformer', 'ferminet') or spec.backflow_transform != 'mult':
        raise ValueError(f'grad_R log|psi| (zero-bias force estimators) is not available for the {spec.kind!r} ansatz kind '
                         f'(backflow {spec.backflow_transform!r}): Psiformer and FermiNet with multiplicative backflow only')
    return eng.grad_positions(r, R, want_r=False, want_R=True)[3]


def make_grad_log_wf(hamil, wf):
    """-> f(params, phys_conf) -> grad_r log|psi| [B, N, 3] (reference force.py:109-118)."""

    def grad_log_wf(params, phys_conf: PhysicalConfiguration):
        r, R, single = _batched(phys_conf)
        return _unbatch(_grad_r(_engine(hamil, wf, params), r, R), single)

    return grad_log_wf


def make_grad_nuc_log_wf(hamil, wf):
    """-> f(params, phys_conf) -> grad_R log|psi| [B, M, 3] (reference force.py:96-106)."""

    def grad_nuc_log_wf(params, phys_conf: PhysicalConfiguration):
        r, R, single = _batched(phys_conf)
        return _unbatch(_grad_R(_engine(hamil, wf, params), r, R), single)

    return grad_nuc_log_wf


def _has_ecp(hamil):
    return getattr(hamil, 'loc_params', None) is not None


def ecp_force_twist(hamil, rng, B, N):
    """-> [B, J, N] quadrature twists of the ECP force: one per walker, uniform in [0, pi/5) from a generator seeded with
    ``rng`` as ``evaluate_finite_difference_force`` seeds its twists, shared by every (nucleus, electron) pair of the walker
    (reference ecp_force_utils.py:55-57 passes the un-folded rng to every pair); None without non-local nuclei."""
    n_nl = 0 if hamil.nl_params is None else len(hamil.pot.nuc_with_nl_pot)
    if not n_nl:
        return None
    g = torch.Generator(device='cpu').manual_seed(0 if rng is None else int(rng))
    return (torch.rand(B, generator=g, dtype=torch.float64) * (torch.pi / 5))[:, None, None].expand(B, n_nl, N)


def _bare(hamil, eng, rng, r, R):
    """F_nuc - grad_R V_loc (- grad_R V_nl with an ECP) [B, M, 3]."""
    if not _has_ecp(hamil):
        return eng.force_terms(r, R)[0]
    tw = ecp_force_twist(hamil, rng, r.shape[0], r.shape[1])
    bare, nl = eng.ecp_force(r, R, seed=0 if rng is None else int(rng), ecp_twist=tw, want_nl=tw is not None)
    return bare if nl is None else bare + nl


def evaluate_hf_force_bare(hamil, wf):
    """-> f(rng, params, phys_conf) -> F_nuc - grad_R V_loc - grad_R V_nl [B, M, 3] (reference force.py:250-301): all-electron
    F_nuc + Z_m sum_i d_im / |d_im|^3; with a Gaussian-type ECP the local ECP terms and -grad_nonloc_potential added
    (dqmc_ecp_force, twists drawn from ``rng``: see the module docstring)."""

    def evaluate_hf_force_bare_(rng, params, phys_conf: PhysicalConfiguration):
        r, R, single = _batched(phys_conf)
        return _unbatch(_bare(hamil, _engine(hamil, wf, params), rng, r, R), single)

    return evaluate_hf_force_bare_


def _bare_plus_zvq(eng, r, R):
    return eng.force_terms(r, R, grad_r=_grad_r(eng, r, R))[1]


def evaluate_hf_force_ac_zvq(hamil, wf):
    """-> f(params, phys_conf) -> F_nuc + sum_i (dQ/dr_i)^T grad_i log|psi| [B, M, 3] (reference force.py:172-194, 450-487)."""

    def evaluate_hf_force_ac_zvq_(params, phys_conf: PhysicalConfiguration):
        r, R, single = _batched(phys_conf)
        return _unbatch(_bare_plus_zvq(_engine(hamil, wf, params), r, R), single)

    return evaluate_hf_force_ac_zvq_


def _zb_factor(e_loc, energy, like):
    f64 = lambda x: torch.as_tensor(x, dtype=torch.float64, device=like.device)  # a Python float energy must not become fp32
    return (-2 * (f64(e_loc) - f64(energy))).to(like.dtype)


def evaluate_hf_force_ac_zvzbq(hamil, wf):
    """-> f(params, phys_conf, e_loc, energy) -> ZVQ - 2 (E_loc - energy) Q [B, M, 3] (reference force.py:490-546)."""

    def evaluate_hf_force_ac_zvzbq_(params, phys_conf: PhysicalConfiguration, e_loc, energy):
        r, R, single = _batched(phys_conf)
        eng = _engine(hamil, wf, params)
        _, zvq, q = eng.force_terms(r, R, grad_r=_grad_r(eng, r, R))
        f = zvq + _zb_factor(e_loc, energy, q).reshape(-1, 1, 1) * q
        return _unbatch(f, single)

    return evaluate_hf_force_ac_zvzbq_


def evaluate_hf_force_ac_zb(hamil, wf):
    """-> f(rng, params, phys_conf, e_loc, energy) -> bare - 2 (E_loc - energy) grad_R log|psi| [B, M, 3]
    (reference force.py:412-447; with an ECP, bare as in ``evaluate_hf_force_bare``)."""

    def evaluate_hf_force_ac_zb_(rng, params, phys_conf: PhysicalConfiguration, e_loc, energy):
        r, R, single = _batched(phys_conf)
        eng = _engine(hamil, wf, params)
        gR = _grad_R(eng, r, R)
        f = _bare(hamil, eng, rng, r, R) + _zb_factor(e_loc, energy, gR).reshape(-1, 1, 1) * gR
        return _unbatch(f, single)

    return evaluate_hf_force_ac_zb_


def evaluate_hf_force_ac_zvqzb(hamil, wf):
    """-> f(params, phys_conf, e_loc, energy) -> ZVQ - 2 (E_loc - energy) grad_R log|psi| [B, M, 3]
    (reference force.py:609-654)."""

    def evaluate_hf_force_ac_zvqzb_(params, phys_conf: PhysicalConfiguration, e_loc, energy):
        r, R, single = _batched(phys_conf)
        eng = _engine(hamil, wf, params)
        gR = _grad_R(eng, r, R)
        f = _bare_plus_zvq(eng, r, R) + _zb_factor(e_loc, energy, gR).reshape(-1, 1, 1) * gR
        return _unbatch(f, single)

    return evaluate_hf_force_ac_zvqzb_


def _zv(hamil, eng, r, R, want_grad_R):
    """(-dT/dR [B, M, 3], grad_R log|psi| or None) of dqmc_zv_force, with the refusals of the AC-ZV family."""
    spec = eng.spec
    if spec.kind not in ('psiformer', 'ferminet') or spec.backflow_transform != 'mult':
        raise ValueError(f'the AC-ZV / AC-ZVZB force estimators are not available for the {spec.kind!r} ansatz kind '
                         f'(backflow {spec.backflow_transform!r}): Psiformer and FermiNet with multiplicative backflow only')
    if _has_ecp(hamil) or getattr(hamil, 'ph', None) is not None:
        raise ValueError(f'the AC-ZV / AC-ZVZB force estimators need an all-electron Hamiltonian (ecp_type '
                         f'{hamil.ecp_type!r})')
    return eng.zv_force(r, R, want_grad_R=want_grad_R)


def evaluate_hf_force_ac_zv(hamil, wf):
    """-> f(rng, params, phys_conf, e_loc=None, energy=None) -> bare + f_zv [B, M, 3] (reference force.py:304-355), with
    f_zv = -dT/dR at fixed r (see the module docstring).  ``e_loc`` and ``energy`` are accepted for the reference's
    signature; the closed form uses neither."""

    def evaluate_hf_force_ac_zv_(rng, params, phys_conf: PhysicalConfiguration, e_loc=None, energy=None):
        r, R, single = _batched(phys_conf)
        eng = _engine(hamil, wf, params)
        zv, _ = _zv(hamil, eng, r, R, False)
        return _unbatch(_bare(hamil, eng, rng, r, R) + zv, single)

    return evaluate_hf_force_ac_zv_


def evaluate_hf_force_ac_zvzb(hamil, wf):
    """-> f(rng, params, phys_conf, e_loc, energy) -> bare + f_zv - 2 (E_loc - energy) grad_R log|psi| [B, M, 3]
    (reference force.py:358-411); grad_R log|psi| comes from the same companion pass as f_zv."""

    def evaluate_hf_force_ac_zvzb_(rng, params, phys_conf: PhysicalConfiguration, e_loc, energy):
        r, R, single = _batched(phys_conf)
        eng = _engine(hamil, wf, params)
        zv, gR = _zv(hamil, eng, r, R, True)
        f = _bare(hamil, eng, rng, r, R) + zv + _zb_factor(e_loc, energy, gR).reshape(-1, 1, 1) * gR
        return _unbatch(f, single)

    return evaluate_hf_force_ac_zvzb_


def finite_difference_displacements(r, R, step_size):
    """-> (Rs [3M, ..., M, 3], rs [3M, ..., N, 3]): the reference's displaced geometries (force.py:579-590): nuclear
    coordinate k moved by -h, every electron by sum_m softmax_m(-|R_m - r_i|) (h e_k)_m."""
    M = R.shape[-2]
    dR = (torch.eye(3 * M, dtype=R.dtype, device=R.device) * step_size).reshape(3 * M, M, 3)
    dists = torch.linalg.norm(R[..., :, None, :] - r[..., None, :, :], dim=-1)  # [..., M, N]
    w = torch.softmax(-dists, dim=-2)
    dr = torch.einsum('kmc,...mn->k...nc', dR, w)
    Rs = R - dR.reshape(3 * M, *([1] * (R.dim() - 2)), M, 3)
    return Rs, r + dr


def evaluate_finite_difference_force(hamil, wf, step_size: float):
    """-> f(rng, params, phys_conf, e_loc, energy) -> exp(2 (log psi' - log psi)) (E' - E_loc) / h [B, M, 3]
    (reference force.py:549-606): 3M displaced local energies per walker, one dqmc_local_energy call per nuclear coordinate.
    With a non-local ECP every displaced copy of walker b reuses walker b's quadrature twists (the reference shares one rng
    over the copies): drawn once per call from ``rng`` unless ``ecp_twist`` [B, J, N] is given.  ``energy`` is accepted for
    the reference's signature and not used."""

    def evaluate_finite_difference_force_(rng, params, phys_conf: PhysicalConfiguration, e_loc, energy, ecp_twist=None):
        r, R, single = _batched(phys_conf)
        eng = _engine(hamil, wf, params)
        B, N, M = r.shape[0], r.shape[1], R.shape[-2]
        n_nl = 0 if hamil.nl_params is None else len(hamil.pot.nuc_with_nl_pot)
        if n_nl and ecp_twist is None:
            g = torch.Generator(device='cpu').manual_seed(0 if rng is None else int(rng))
            ecp_twist = torch.rand(B, n_nl, N, generator=g, dtype=torch.float64) * (torch.pi / 5)
        log0 = eng.wf_forward(r, R)[1]
        Rs, rs = finite_difference_displacements(r, R, step_size)
        e0 = torch.as_tensor(e_loc, device=r.device).to(log0.dtype).reshape(B)
        out = torch.empty(3 * M, B, dtype=log0.dtype, device=log0.device)
        seed = 0 if rng is None else int(rng)
        for k in range(3 * M):
            E, _, _, log, _ = eng.local_energy(rs[k], Rs[k], seed=seed, ecp_twist=ecp_twist)
            out[k] = torch.exp(2 * (log - log0)) * (E - e0) / step_size
        return _unbatch(out.T.reshape(B, M, 3), single)

    return evaluate_finite_difference_force_


def compute_mean_and_std(name: str, observable_samples, axis: int = -1):
    """{name/mean, name/std} over ``axis`` and over every rank's samples (reference observable.py:60-67)."""
    x = torch.as_tensor(observable_samples)
    mean, std = weighted_std(x, torch.ones_like(x), axis=axis)
    return {f'{name}/mean': mean, f'{name}/std': std}
