"""CPU: the fp64 references of the reverse-pass tests (tests/reverse_reference.py) checked against a plain row loop and against
finite differences, so that the GPU tests compare the kernels with something known to be right."""
import numpy as np
import pytest
import torch

from deepqmc_b200 import params as PN
from deepqmc_b200.ansatz import B200Ansatz
from deepqmc_b200.hamil import MolecularHamiltonian
from deepqmc_b200.molecule import Molecule
from reverse_reference import attention_bwd_ref, log_psi_grads, wgrad_ref


@pytest.mark.parametrize('lo,hi', [(0, -1), (0, 3), (3, 5), (5, 5)])
def test_wgrad_ref_is_the_masked_row_sum(lo, hi):
    rng = np.random.default_rng(0)
    rows, N = 23, 5
    A, dY = rng.normal(size=(rows, 7)), rng.normal(size=(rows, 4))
    dW, db = np.zeros((7, 4)), np.zeros(4)
    for row in range(rows):
        if hi == -1 or lo <= row % N < hi:
            dW += np.outer(A[row], dY[row])
            db += dY[row]
    rW, rb, mW, mb = wgrad_ref(torch.as_tensor(A), torch.as_tensor(dY), N, lo, hi)
    assert np.allclose(rW.numpy(), dW, rtol=0, atol=1e-13) and np.allclose(rb.numpy(), db, rtol=0, atol=1e-13)
    assert (mW.numpy() >= np.abs(dW) - 1e-13).all() and (mb.numpy() >= np.abs(db) - 1e-13).all()
    if lo == hi:
        assert not rW.any() and not rb.any()


def _richardson(f, x, h=1e-4):
    d = lambda s: (f(x + s) - f(x - s)) / (2 * s)
    return (4 * d(h / 2) - d(h)) / 3


@pytest.mark.parametrize('kind,spin', [('psiformer', 2), ('psiformer', 0), ('transpsiformer', 2), ('paulinet', 2)])
def test_log_psi_grads_against_finite_differences(kind, spin):
    """d/dparams sum_b w_b log|psi(r_b)| of the reference against Richardson-extrapolated central differences, at 1e-8, for
    the largest entry of every parameter array; with both spins up (spin = 2) no down-spin head is read, and the difference
    quotient and the reference both give exact zeros there."""
    mol = Molecule(coords=[[0.0, 0.0, 0.0], [1.4, 0.1, 0.0]], charges=[1, 1], charge=0, spin=spin)
    hamil = MolecularHamiltonian(mol=mol)
    hyper = {} if kind == 'paulinet' else dict(embedding_dim=8, n_layers=1, n_heads=2, n_determinants=2)
    ansatz = B200Ansatz(hamil, kind, dtype='float64', **hyper)
    params = {k: np.asarray(v, dtype=np.float64) for k, v in PN.perturb_params(ansatz.init(0)).items()}
    rng = np.random.default_rng(1)
    r = torch.as_tensor(mol.coords[rng.integers(0, 2, size=(2, 2))] + 0.7 * rng.normal(size=(2, 2, 3)))
    R = torch.as_tensor(mol.coords)
    w = torch.tensor([0.8, -1.1], dtype=torch.float64)
    _, _, g = log_psi_grads(ansatz.spec, params, r, R, w)
    for name, v in params.items():
        if v.size == 0:
            continue
        i = int(np.argmax(np.abs(g[name].numpy()).ravel()))

        def f(x):
            p = dict(params)
            q = v.copy().ravel()
            q[i] = x
            p[name] = q.reshape(v.shape)
            return float((w * log_psi_grads(ansatz.spec, p, r, R, torch.zeros(2, dtype=torch.float64))[1]).sum())

        fd = _richardson(f, float(v.ravel()[i]))
        got = float(g[name].reshape(-1)[i])
        assert abs(got - fd) <= 1e-8 * max(1.0, abs(fd)), (name, got, fd)


@pytest.mark.parametrize('Mn', [0, 2])
def test_attention_bwd_ref_against_finite_differences(Mn):
    """Every cotangent of the attention reference (dQ | dK | dV and the shared nuclear tokens' dKn / dVn) against
    Richardson-extrapolated central differences of sum(dO * O), at 1e-8."""
    from tc_reference import attention_value

    g = torch.Generator().manual_seed(Mn)
    B, N, H, d = 2, 3, 2, 8
    QKV = torch.randn(B * N, 3 * d, generator=g, dtype=torch.float64)
    dO = torch.randn(B * N, d, generator=g, dtype=torch.float64)
    kn, vn = (torch.randn(Mn, d, generator=g, dtype=torch.float64) for _ in range(2)) if Mn else (None, None)
    got = attention_bwd_ref(QKV, dO, N, H, kn, vn)

    def loss(q, k, v):
        return float((attention_value(q.reshape(B, N, 3 * d), H, k, v).reshape(B * N, d) * dO).sum())

    for which, t, gt in ((0, QKV, got[0]), (1, kn, got[1]), (2, vn, got[2])):
        if t is None:
            assert gt is None
            continue
        for idx in range(t.numel()):
            def f(x):
                ts = [QKV, kn, vn]
                u = ts[which].clone().reshape(-1)
                u[idx] = x
                ts[which] = u.reshape(t.shape)
                return loss(*ts)

            fd = _richardson(f, float(t.reshape(-1)[idx]))
            assert abs(float(gt.reshape(-1)[idx]) - fd) <= 1e-8 * max(1.0, abs(fd)), (which, idx)
