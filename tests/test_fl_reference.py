"""CPU: the fp64 forward-Laplacian jet references of tests/tc_reference.py (attention_fl_ref, mlp_fl_ref), which the GPU tests
of the forward-Laplacian attention and MLP kernels compare against, checked against plain calculus: a small composite
x in R^{3N} -> nonlinear per-electron features -> Q | K | V (or O, X) -> attention (or MLP) -> outputs, whose tangents and
Laplacian are the Jacobian and the Hessian trace of the composite (torch.autograd.functional).  Also against the kernels'
closed-form derivative rules restated in fp64 (kernels_trunk.cuh, attn_fl_kernel header; gemm_wgmma.cuh, tanh epilogue), so
that a rule and a reference that agree with each other but not with calculus are caught."""
import pytest
import torch
from torch.autograd.functional import jacobian

from tc_reference import attention_fl_ref, attention_value, mlp_fl_ref, mlp_value

F64 = torch.float64
N, H, DH = 3, 2, 4
D = H * DH
S = 3 * N + 2
SLOT_CLASSES = (slice(0, 1), slice(1, S - 1), slice(S - 1, S))  # value, tangents, Laplacian


def _randn(g, *shape):
    return torch.randn(*shape, generator=g, dtype=F64)


def _features(g, width):
    """x [3N] -> [N, width]: every electron's row depends nonlinearly on every coordinate (dense tangents, non-zero second
    derivatives)."""
    A, B, c = _randn(g, 3, width), _randn(g, 3, width) * 0.5, _randn(g, width) * 0.3

    def f(x):
        r = x.reshape(N, 3)
        return torch.tanh(r @ A + (r * r).sum(0, keepdim=True).sqrt() @ B * torch.sin(r[:, :1]) + c) * 2.0
    return f


def _jets(f, x):
    """Value, tangents and Laplacian of f at x as slot rows [N S][c] (row i S + s), from the autograd Jacobian and Hessian."""
    val = f(x)
    J = jacobian(f, x)                                                    # [N, c, 3N]
    Hs = jacobian(lambda y: jacobian(f, y, create_graph=True), x)         # [N, c, 3N, 3N]
    lap = Hs.diagonal(dim1=-2, dim2=-1).sum(-1)
    return torch.cat([val[:, None], J.permute(0, 2, 1), lap[:, None]], dim=1).reshape(N * S, -1)


def _check(out, exact):
    """Every slot class on its own, relative to that class's largest exact magnitude."""
    for sl in SLOT_CLASSES:
        o, e = out.reshape(N, S, -1)[:, sl], exact.reshape(N, S, -1)[:, sl]
        assert ((o - e).abs().max() / e.abs().max()).item() < 1e-10, sl


def attention_fl_closed_form(QKV, kn, vn):
    """The rules of the attn_fl_kernel header comment (kernels_trunk.cuh) in fp64, one walker, Mn = kn.shape[0] tokens:
    s^t = c (q^t k + q k^t); p^t = p (s^t - m^t), m^t = sum_j p s^t; s^L = c (q^L k + q k^L + 2 sum_t q^t k^t);
    lap p = p (u - V + s^L - sum_j p s^L), u = sum_t (s^t - m^t)^2, V = sum_j p u; o^t = p^t v + p v^t;
    o^L = (lap p) v + 2 sum_t p^t v^t + p v^L; the nuclear keys / values carry no tangents and no Laplacian."""
    y = QKV.reshape(N, S, 3 * D)
    out = torch.zeros(N, S, D, dtype=F64)
    c = DH ** -0.5
    for h in range(H):
        cols = slice(h * DH, (h + 1) * DH)
        q, k, v = (y[:, :, i * D:(i + 1) * D][:, :, cols] for i in range(3))  # [N, S, dh]
        tok = lambda t: torch.cat([t[:, None, cols], torch.zeros(t.shape[0], S - 1, DH, dtype=F64)], dim=1)
        k, v = torch.cat([k, tok(kn)]), torch.cat([v, tok(vn)])               # [N + Mn, S, dh]
        p = torch.softmax(c * q[:, 0] @ k[:, 0].T, dim=-1)
        st = c * (torch.einsum('ite,je->tij', q[:, 1:-1], k[:, 0]) + torch.einsum('ie,jte->tij', q[:, 0], k[:, 1:-1]))
        m = (p * st).sum(-1, keepdim=True)
        pt = p * (st - m)
        u = ((st - m) ** 2).sum(0)
        sL = c * (q[:, -1] @ k[:, 0].T + q[:, 0] @ k[:, -1].T + 2 * torch.einsum('ite,jte->ij', q[:, 1:-1], k[:, 1:-1]))
        lapp = p * (u - (p * u).sum(-1, keepdim=True) + sL - (p * sL).sum(-1, keepdim=True))
        out[:, 0, cols] = p @ v[:, 0]
        out[:, 1:-1, cols] = (pt @ v[:, 0] + torch.einsum('ij,jte->tie', p, v[:, 1:-1])).permute(1, 0, 2)
        out[:, -1, cols] = lapp @ v[:, 0] + 2 * torch.einsum('tij,jte->ie', pt, v[:, 1:-1]) + p @ v[:, -1]
    return out.reshape(N * S, D)


def tanh_fl_closed_form(Z, bias):
    """The tanh rule of the row-GEMM epilogue (gemm_wgmma.cuh) and tanh_fl_kernel: y = tanh(z + b), y_t = y' z_t,
    y_L = y' z_L + y'' sum_t z_t^2 (the bias on value rows only)."""
    z = Z.reshape(-1, S, Z.shape[-1])
    y = torch.tanh(z[:, 0] + bias)
    y1, y2 = 1 - y * y, -2 * y * (1 - y * y)
    lap = y1 * z[:, -1] + y2 * (z[:, 1:-1] ** 2).sum(1)
    return torch.cat([y[:, None], y1[:, None] * z[:, 1:-1], lap[:, None]], dim=1).reshape(Z.shape)


def mlp_fl_closed_form(Wd, O, X):
    """The engine's row-GEMM sequence (linear layers act slot by slot) with the tanh rule after W1 and W2."""
    A = X + O @ Wd['L0.wo']
    M1 = tanh_fl_closed_form(A @ Wd['L0.w1'], Wd['L0.b1'][0])
    return A + tanh_fl_closed_form(M1 @ Wd['L0.w2'], Wd['L0.b2'][0])


@pytest.mark.parametrize('Mn', [0, 2])
@pytest.mark.parametrize('seed', [0, 1])
def test_attention_fl_ref_matches_autograd(seed, Mn):
    """attention_fl_ref fed with the autograd jets of the features = the composite's Jacobian and Hessian trace; so does the
    kernels' closed form; with and without nuclear tokens (constants behind the electron keys)."""
    g = torch.Generator().manual_seed(seed)
    feat, Wqkv = _features(g, 6), _randn(g, 6, 3 * D)
    kn, vn = _randn(g, Mn, D), _randn(g, Mn, D)
    x = _randn(g, 3 * N)
    qkv = lambda y: feat(y) @ Wqkv
    tokens = (kn, vn) if Mn else (None, None)
    exact = _jets(lambda y: attention_value(qkv(y)[None], H, *tokens)[0], x)
    QKV = _jets(qkv, x)
    ref = attention_fl_ref(QKV, N, H, S, *tokens)
    assert ref.shape == (N * S, D) and ref.dtype == F64
    _check(ref, exact)
    _check(attention_fl_closed_form(QKV, kn, vn), exact)


@pytest.mark.parametrize('seed', [0, 1])
def test_mlp_fl_ref_matches_autograd(seed):
    """mlp_fl_ref (O and X both carry jets) = the composite's Jacobian and Hessian trace; so does the tanh rule."""
    g = torch.Generator().manual_seed(seed)
    feat_o, feat_x = _features(g, 5), _features(g, 5)
    Po, Px = _randn(g, 5, D), _randn(g, 5, D)
    Wd = {'L0.wo': _randn(g, D, D) / D ** 0.5, 'L0.w1': _randn(g, D, D) / D ** 0.5, 'L0.w2': _randn(g, D, D) / D ** 0.5,
          'L0.b1': _randn(g, 1, D), 'L0.b2': _randn(g, 1, D)}
    x = _randn(g, 3 * N)
    o_of, x_of = (lambda y: feat_o(y) @ Po), (lambda y: feat_x(y) @ Px)
    exact = _jets(lambda y: mlp_value(torch.cat([o_of(y), x_of(y)], dim=-1), lambda n: Wd['L0.' + n]), x)
    O, X = _jets(o_of, x), _jets(x_of, x)
    ref = mlp_fl_ref(Wd, 0, O, X, N, S)
    assert ref.shape == (N * S, D) and ref.dtype == F64
    _check(ref, exact)
    _check(mlp_fl_closed_form(Wd, O, X), exact)


def test_the_comparison_sees_a_lost_term():
    """The bound has teeth: the tanh rule with the last tangent missing from sum_t z_t^2, or the attention rule without the
    factor 2 of 2 sum_t q^t k^t, misses the Laplacian far beyond 1e-10."""
    g = torch.Generator().manual_seed(3)
    Z, b = _randn(g, 2 * S, D), _randn(g, D)
    z = Z.reshape(-1, S, D)
    y = torch.tanh(z[:, 0] + b)
    lossy = (1 - y * y) * z[:, -1] - 2 * y * (1 - y * y) * (z[:, 1:-2] ** 2).sum(1)
    good = tanh_fl_closed_form(Z, b).reshape(-1, S, D)[:, -1]
    assert ((lossy - good).abs().max() / good.abs().max()).item() > 1e-3
    QKV = _randn(g, N * S, 3 * D)
    q = QKV.reshape(N, S, 3 * D)
    half = q.clone()
    half[:, 1:-1, :D] /= 2 ** 0.5  # q^t k^t halved (and the tangent slots' q^t k / q k^t with it)
    ref = attention_fl_ref(QKV, N, H, S).reshape(N, S, D)[:, -1]
    assert ((attention_fl_ref(half.reshape(N * S, -1), N, H, S).reshape(N, S, D)[:, -1] - ref).abs().max() /
            ref.abs().max()).item() > 1e-3
