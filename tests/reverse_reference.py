"""Plain torch references of the engine's reverse passes, by autograd in fp64 (the reference) or fp32 (the yardstick for what
fp32 arithmetic gets wrong anyway): the softmax attention backward, the weight- and bias-gradient reductions of the dense
layers, and the parameter gradient d/dparams sum_b w_b log|psi(r_b)| through oracle.wf; shared by the reverse-pass
conformance tests."""
import numpy as np
import torch


def attention_bwd_ref(QKV, dO, N, H, kn=None, vn=None, dtype=torch.float64):
    """Cotangents of tc_reference.attention_value (softmax(q [K; Kn]^T / sqrt(dh)) [V; Vn] per walker and head) for the output
    cotangent dO [B N][d], by autograd -> (dQKV [B N][3d], dKn [Mn][d] or None, dVn [Mn][d] or None): the nuclear tokens
    kn / vn [Mn][d] are shared by every walker, so their cotangents are sums over walkers."""
    from tc_reference import attention_value

    rows, d3 = QKV.shape
    x = QKV.detach().to(dtype).reshape(rows // N, N, d3).requires_grad_(True)
    leaf = lambda t: None if t is None else t.detach().to(dtype).requires_grad_(True)
    kn, vn = leaf(kn), leaf(vn)
    out = attention_value(x, H, kn, vn)
    (out * dO.detach().to(dtype).reshape(out.shape)).sum().backward()
    return x.grad.reshape(rows, d3), None if kn is None else kn.grad, None if vn is None else vn.grad


def row_mask(rows, N, lo, hi):
    """Rows b N + i of electrons lo <= i < hi (hi = -1: every row) -> bool [rows]."""
    i = torch.arange(rows) % N
    return torch.ones(rows, dtype=torch.bool) if hi == -1 else (i >= lo) & (i < hi)


def wgrad_ref(A, dY, N, lo, hi, dtype=torch.float64):
    """The parameter cotangents of Y = A W + b over the selected rows, by autograd of sum(dY * Y):  dW = A^T dY, db = column
    sums of dY -> (dW [K, Nc], db [Nc], |A|^T |dY|, sum |dY|: the magnitudes a rounded sum accumulates)."""
    m = row_mask(A.shape[0], N, lo, hi).to(A.device)
    A, dY = A.to(dtype) * m[:, None], dY.to(dtype) * m[:, None]
    W = torch.zeros(A.shape[1], dY.shape[1], dtype=dtype, device=A.device, requires_grad=True)
    b = torch.zeros(dY.shape[1], dtype=dtype, device=A.device, requires_grad=True)
    (dY * (A @ W + b * m[:, None])).sum().backward()
    return W.grad, b.grad, A.abs().T @ dY.abs(), dY.abs().sum(0)


def log_psi_grads(spec, params, r, R, w, dtype=torch.float64):
    """d/dparams sum_b w_b log|psi(r_b)| by autograd through oracle.wf, one walker at a time, in `dtype` -> (sign [B], log [B],
    {name: gradient in fp64}).  A parameter that log|psi| never reads (the down-spin heads of a fully polarised system) gets
    an exact zero, as jax.grad gives it."""
    from oracle import wf

    pt = {k: torch.as_tensor(np.asarray(v), dtype=dtype).requires_grad_(True) for k, v in params.items()}
    r, R, w = r.detach().cpu().to(dtype), R.detach().cpu().to(dtype), w.detach().cpu().to(dtype)
    signs, logs, tot = [], [], 0
    for b in range(r.shape[0]):
        s, l = wf.log_psi(spec, pt, r[b], R)
        signs.append(float(s))
        logs.append(float(l.detach()))
        tot = tot + w[b] * l
    tot.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)).double() for k, v in pt.items()}
    return torch.tensor(signs, dtype=torch.float64), torch.tensor(logs, dtype=torch.float64), grads
