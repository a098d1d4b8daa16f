"""Restatement of the reference's spin estimators (TEST INFRASTRUCTURE, see oracle/__init__).

Follows src/deepqmc/physics.py:159-181 (evaluate_spin), :184-223 (make_permute_single_down_with_all_up: the position of
down electron beta exchanged with every up electron alpha, accumulator -= sign' sign exp(log' - log)) and :226-239
(make_stochastic_spin_raising_operator: the same loop for one beta, started at 1).  torch.float64, single walker.
``wf(r) -> (sign, log|psi|)``; ``wave_function(spec, params, R)`` builds it from oracle/wf.py.
"""
from __future__ import annotations

import torch

from . import wf as W


def wave_function(spec, params, R):
    return lambda r: W.log_psi(spec, params, r, R)


def swapped(r, a, b):
    """r with the positions of electrons a and b exchanged (physics.py:201-209)."""
    idx = torch.arange(r.shape[0])
    idx[a], idx[b] = b, a
    return r[idx]


def ratios(wf, r, n_up, down_idx):
    """rho[alpha] = psi(r with alpha, down_idx swapped) / psi(r) for every up electron alpha (physics.py:210-216)."""
    s0, l0 = wf(r)
    out = []
    for a in range(n_up):
        s, l = wf(swapped(r, a, down_idx))
        out.append(s0 * s * torch.exp(l - l0))
    return torch.stack(out) if out else torch.zeros(0, dtype=r.dtype)


def spin_ratios(wf, r, n_up, n_down):
    """rho[alpha, beta - n_up] for all (up, down) pairs."""
    if n_down == 0:
        return torch.zeros(n_up, 0, dtype=r.dtype)
    return torch.stack([ratios(wf, r, n_up, n_up + j) for j in range(n_down)], 1)


def evaluate_spin(wf, r, n_up, n_down):
    """s2 = D/2 (D/2 + 1) + n_down - sum_{alpha, beta} rho (physics.py:166-179)."""
    D = n_up - n_down
    return D / 2 * (D / 2 + 1) + n_down - spin_ratios(wf, r, n_up, n_down).sum()


def spin_raising(wf, r, n_up, down_idx):
    """1 - sum_alpha rho[alpha, down_idx] (physics.py:230-237)."""
    return 1.0 - ratios(wf, r, n_up, down_idx).sum()
