"""Shared inputs of the spin tests (test_spin_host.py, test_gpu_spin.py)."""
import numpy as np

from deepqmc_b200 import params as PN


def known_answer_params(spec, params):
    """Psiformer parameters whose orbitals depend neither on the electron's spin nor on the other electrons: trunk weights
    zero (every layer is the identity), the spin row of the embedding zero, equal up / down envelopes and backflow heads.
    With a full determinant and no e-e cusp every up / down swap then negates psi, so <S^2> = N/2 (N/2 + 1) everywhere."""
    assert spec.kind == 'psiformer' and spec.cusp == 'none' and spec.full_determinant
    out = {k: np.asarray(v, dtype=np.float64).copy() for k, v in params.items()}
    for k in out:
        if k.startswith(PN.GNN) and ('multi_head_attention' in k or '/mlp/' in k):
            out[k][...] = 0.0
    emb = PN.GNN + 'electron_embedding/linear:w'
    out[emb][-1] = 0.0  # the +-1 spin feature is the last input column
    out[f'{PN.ENV}:pi_down'] = out[f'{PN.ENV}:pi_up'].copy()
    out[f'{PN.ENV}:zetas_down'] = out[f'{PN.ENV}:zetas_up'].copy()
    out[PN.BF_DN + ':w'] = out[PN.BF_UP + ':w'].copy()
    return out


def walkers(hamil, B, seed=0, dtype=np.float64):
    """B walkers with every electron near a random nucleus."""
    rng = np.random.default_rng(seed)
    N = hamil.n_up + hamil.n_down
    R = np.asarray(hamil.mol.coords)
    return (R[rng.integers(0, len(R), size=(B, N))] + 0.8 * rng.normal(size=(B, N, 3))).astype(dtype)
