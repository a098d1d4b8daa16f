"""Total spin <S^2> of the electronic states and the spin penalty of the loss on top of the CUDA spin pass (``dqmc_spin``).

Mirror of the reference's ``physics.py:159-239`` (``evaluate_spin``, ``make_stochastic_spin_raising_operator``) and
``loss/spin.py`` (contributions, mean / std, penalty tangents), with the reference's names and conventions.  The swapped
forwards of every walker run inside the engine; the [mol, state, B] algebra that follows is elementwise torch.
``params`` is a sequence with one parameter tree per electronic state, ``phys_conf`` carries the batch shape
[mol, state, B].  The parameter tangents are reverse passes (``dqmc_wf_vjp_params``) per (molecule, state), all-reduced
over the ranks like ``overlap.compute_mean_overlap_tangent``.
"""
from __future__ import annotations

import numpy as np
import torch

from . import parallel
from .types import PhysicalConfiguration


def _ansatz_of(ansatz_apply):
    ansatz = getattr(ansatz_apply, '__self__', None)
    if ansatz is None or not hasattr(ansatz, 'engine_for'):
        raise TypeError('expected the bound .apply of a deepqmc_b200 B200Ansatz')
    return ansatz


def _spin_call(hamil, ansatz, params, phys_conf, down_idx, want_ratios=False):
    eng = ansatz.engine_for(hamil, params)
    r, R = phys_conf.r, phys_conf.R
    single = r.dim() == 2
    if R.dim() == 3:  # one geometry per call (the spin pass takes no per-walker nuclei)
        if not bool((R == R[:1]).all()):
            raise ValueError('spin: one nuclear geometry per call (all rows of a batched R must be equal)')
        R = R[0]
    s2, ratio = eng.spin(r[None] if single else r, R, down_idx=down_idx, want_ratios=want_ratios)
    if single:
        s2, ratio = s2[0], (ratio[0] if ratio is not None else None)
    return s2, ratio


def evaluate_spin(hamil, ansatz_apply):
    """-> f(params, phys_conf) -> s2[B]: D/2 (D/2 + 1) + n_down - sum_{a,b} psi(r with a, b swapped) / psi(r), D = n_up - n_down
    (reference physics.py:159-181)."""
    ansatz = _ansatz_of(ansatz_apply)

    def evaluate_spin_(params, phys_conf: PhysicalConfiguration):
        return _spin_call(hamil, ansatz, params, phys_conf, -1)[0]

    return evaluate_spin_


def make_stochastic_spin_raising_operator(hamil, ansatz_apply):
    """-> f(params, phys_conf, down_idx) -> 1 - sum_a psi(r with a, down_idx swapped) / psi(r) (reference physics.py:226-239).
    ``down_idx`` is one electron index in [n_up, N) shared by the batch."""
    ansatz = _ansatz_of(ansatz_apply)

    def evaluate_stochastic_spin_raising_operator(params, phys_conf: PhysicalConfiguration, down_idx):
        return _spin_call(hamil, ansatz, params, phys_conf, _one_index(down_idx))[0]

    return evaluate_stochastic_spin_raising_operator


def _one_index(down_idx) -> int:
    d = torch.as_tensor(down_idx).reshape(-1)
    if d.numel() == 0 or not bool((d == d[0]).all()):
        raise ValueError('down_idx must be one index shared by the whole batch')
    return int(d[0])


def _states(phys_conf, states):
    return list(range(phys_conf.r.shape[1])) if states is None else list(states)


def _mol_state_conf(phys_conf, m, s):
    R = phys_conf.R[m, s]
    return PhysicalConfiguration(R[0] if R.dim() == 3 else R, phys_conf.r[m, s], phys_conf.mol_idx[m, s])


def compute_spin_contributions(hamil, ansatz, params, phys_conf: PhysicalConfiguration, states=None):
    """-> s2[mol, len(states), B] with the parameter tree params[state] for every state (reference loss/spin.py:12-44)."""
    states = _states(phys_conf, states)
    Mb, B = phys_conf.r.shape[0], phys_conf.r.shape[2]
    out = torch.empty(Mb, len(states), B, dtype=phys_conf.r.dtype, device=phys_conf.r.device)
    f = evaluate_spin(hamil, ansatz.apply)
    for j, s in enumerate(states):
        for m in range(Mb):
            out[m, j] = f(params[s], _mol_state_conf(phys_conf, m, s))
    return out


def _state_weights(weight, states, like):
    if weight is None:
        return torch.ones_like(like)
    return torch.stack([weight[:, s] for s in states], 1).to(like.dtype)


def _all_reduce(t):
    if parallel.world()[1] > 1:
        torch.distributed.all_reduce(t)
    return t


def weighted_std(x, weights, axis=-1):
    """sqrt of the weighted average of (x - weighted mean)^2 (reference utils.py:191-196); the sums run over every rank."""
    wsum = _all_reduce(weights.double().sum(axis, keepdim=True))
    mean = _all_reduce((x * weights).double().sum(axis, keepdim=True)) / wsum
    var = _all_reduce((weights * (x - mean) ** 2).double().sum(axis, keepdim=True)) / wsum
    return mean.squeeze(axis), var.sqrt().squeeze(axis)


def _all_device_mean(x, axis=None):
    """Mean over ``axis`` (all axes if None) and over every rank's walkers (reference parallel.py:175-182)."""
    x = x.double()
    if axis is None:
        packed = torch.stack([x.sum(), torch.tensor(float(x.numel()), dtype=torch.float64, device=x.device)])
        _all_reduce(packed)
        return packed[0] / packed[1]
    s = _all_reduce(x.sum(axis, keepdim=True))
    n = _all_reduce(torch.full_like(s, float(x.shape[axis])))
    return s / n


def compute_mean_spin(spin_contributions, weight, states=None):
    """-> (all-device mean of s2 * w, {'spin/mean', 'spin/std'} [mol, state]): the weighted mean and std of every
    (molecule, state) row over all ranks' walkers (reference loss/spin.py:47-71)."""
    states = list(range(spin_contributions.shape[1])) if states is None else states
    w = _state_weights(weight, states, spin_contributions)
    mean, std = weighted_std(spin_contributions, w, axis=-1)
    return _all_device_mean(spin_contributions * w).to(spin_contributions.dtype), {'spin/mean': mean, 'spin/std': std}


def _sum_grads(acc, g):
    if acc is None:
        return dict(g)
    for k, v in g.items():
        acc[k] = acc[k] + v if k in acc else v
    return acc


def _all_reduce_grads(g):
    if parallel.world()[1] > 1:
        keys = sorted(g)
        flat = torch.cat([g[k].reshape(-1) for k in keys])
        torch.distributed.all_reduce(flat)
        o = 0
        for k in keys:
            n = g[k].numel()
            g[k] = flat[o:o + n].reshape(g[k].shape)
            o += n
    return g


def _mask_count(mask):
    return _all_reduce(mask.double().sum().reshape(1))[0]


def spin_tangent_cotangents(spin_contributions, weight, gradient_mask, states=None):
    """Per-walker cotangents of the squared spin penalty: (s2 - <s2 w>) w mask / n_mask, with the all-device mean of
    s2 * w per (molecule, state) row and n_mask the all-device count of the mask (reference loss/spin.py:74-115)."""
    states = list(range(spin_contributions.shape[1])) if states is None else states
    w = _state_weights(weight, states, spin_contributions)
    mask = torch.ones_like(spin_contributions, dtype=torch.bool) if gradient_mask is None else torch.stack(
        [gradient_mask[:, s] for s in states], 1)
    mean = _all_device_mean(spin_contributions * w, axis=-1).to(spin_contributions.dtype)
    n_mask = _mask_count(mask).to(spin_contributions.dtype)
    return (spin_contributions - mean) * w * mask.to(w.dtype) / n_mask


def compute_mean_spin_tangent(spin_contributions, weight, gradient_mask, ansatz, params, phys_conf, states=None):
    """Parameter gradient of the squared spin penalty <s2>: one reverse pass per (molecule, state) with the cotangents of
    ``spin_tangent_cotangents`` -> list of {haiku name: gradient}, one per entry of ``states``, summed over all ranks
    (reference loss/spin.py:74-115)."""
    states = _states(phys_conf, states)
    cot = spin_tangent_cotangents(spin_contributions, weight, gradient_mask, states)
    grads = []
    for j, s in enumerate(states):
        g = None
        for m in range(phys_conf.r.shape[0]):
            _, gm = ansatz.log_psi_vjp(params[s], _mol_state_conf(phys_conf, m, s), cot[m, j].contiguous())
            g = _sum_grads(g, gm)
        grads.append(_all_reduce_grads(g))
    return grads


def draw_down_idx(rng, hamil) -> int:
    """One spin-down electron index in [n_up, N) from the host RNG (``rng``: a numpy Generator or an int seed)."""
    gen = rng if isinstance(rng, np.random.Generator) else np.random.default_rng(rng)
    return int(hamil.n_up + gen.integers(hamil.n_down))


def compute_spin_raising_contributions(rng, hamil, ansatz, phys_conf: PhysicalConfiguration, params, batch_size=None,
                                       states=None, return_ratios=False):
    """-> c[mol, len(states), B] = 1 - sum_a psi(r with a, beta swapped) / psi(r), one beta for the whole batch drawn from
    the host RNG (reference loss/spin.py:118-174).  ``batch_size``: walkers per engine call (all at once if None).
    ``return_ratios``: also the ratios [mol, len(states), B, n_up] and beta, which the penalty tangent needs."""
    if hamil.n_down == 0:
        raise ValueError('the spin-raising estimator needs at least one spin-down electron')
    states = _states(phys_conf, states)
    beta = draw_down_idx(rng, hamil)
    Mb, B = phys_conf.r.shape[0], phys_conf.r.shape[2]
    like = dict(dtype=phys_conf.r.dtype, device=phys_conf.r.device)
    out = torch.empty(Mb, len(states), B, **like)
    ratios = torch.empty(Mb, len(states), B, hamil.n_up, **like) if return_ratios else None
    step = B if batch_size is None else max(1, int(batch_size) // parallel.world()[1])
    for j, s in enumerate(states):
        for m in range(Mb):
            pc = _mol_state_conf(phys_conf, m, s)
            for b0 in range(0, B, step):
                part = PhysicalConfiguration(pc.R, pc.r[b0:b0 + step], pc.mol_idx[b0:b0 + step])
                c, rho = _spin_call(hamil, ansatz, params[s], part, beta, return_ratios)
                out[m, j, b0:b0 + step] = c
                if return_ratios:
                    ratios[m, j, b0:b0 + step] = rho
    return (out, ratios, beta) if return_ratios else out


def swap_electrons(r, a, b):
    """r[..., N, 3] with the positions of electrons a and b exchanged (a, b: ints or index tensors broadcast over r[..., 0, 0])."""
    out = r.clone()
    out[..., a, :], out[..., b, :] = r[..., b, :], r[..., a, :]
    return out


def spin_raising_cotangents(spin_raising_contributions, spin_raising_ratios, weight, gradient_mask, states=None):
    """Per-walker cotangents of the spin-raising penalty (reference loss/spin.py:177-229 with the forward-mode tangent of
    the contributions written as a reverse pass): with a_b = <c w> w_b mask_b / n_mask,
    base walker b: a_b (2 (c_b - <c w>) + sum_a rho_ba); walker b with electrons a and beta swapped: -a_b rho_ba.
    -> (base [mol, state, B], swapped [mol, state, B, n_up])."""
    c = spin_raising_contributions
    states = list(range(c.shape[1])) if states is None else states
    w = _state_weights(weight, states, c)
    mask = torch.ones_like(c, dtype=torch.bool) if gradient_mask is None else torch.stack([gradient_mask[:, s] for s in states], 1)
    mean = _all_device_mean(c * w, axis=-1).to(c.dtype)
    n_mask = _mask_count(mask).to(c.dtype)
    a = mean * w * mask.to(c.dtype) / n_mask
    rho = spin_raising_ratios
    return a * (2 * (c - mean) + rho.sum(-1)), -a[..., None] * rho


def compute_mean_spin_raising_tangent(spin_raising_contributions, spin_raising_ratios, down_idx, weight, gradient_mask,
                                      ansatz, params, phys_conf, states=None):
    """Parameter gradient of the spin-raising penalty: one reverse pass per (molecule, state) over the B walkers and their
    n_up B swapped copies with the cotangents of ``spin_raising_cotangents`` -> list of {haiku name: gradient}, one per
    entry of ``states``, summed over all ranks (reference loss/spin.py:177-229, loss_function.py:250-297)."""
    states = _states(phys_conf, states)
    base, swapped = spin_raising_cotangents(spin_raising_contributions, spin_raising_ratios, weight, gradient_mask, states)
    beta = _one_index(down_idx)
    grads = []
    for j, s in enumerate(states):
        g = None
        for m in range(phys_conf.r.shape[0]):
            pc = _mol_state_conf(phys_conf, m, s)
            r = pc.r
            sw = torch.stack([swap_electrons(r, a, beta) for a in range(spin_raising_ratios.shape[-1])], 1)  # [B, n_up, N, 3]
            r_all = torch.cat([r, sw.reshape(-1, *r.shape[1:])])
            cot = torch.cat([base[m, j], swapped[m, j].reshape(-1)]).contiguous()
            mol_idx = torch.cat([pc.mol_idx, pc.mol_idx.repeat_interleave(sw.shape[1])])
            _, gm = ansatz.log_psi_vjp(params[s], PhysicalConfiguration(pc.R, r_all, mol_idx), cot)
            g = _sum_grads(g, gm)
        grads.append(_all_reduce_grads(g))
    return grads
