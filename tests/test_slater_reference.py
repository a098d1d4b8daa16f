"""CPU: the fp64 references of the determinant tail in tests/slater_reference.py (slater_ref, det_sum_ref), which the GPU tests of
the Slater kernels and of the determinant sum compare against, checked against plain calculus: a small composite
x in R^{3N} -> backflow rows BF(x) -> log|det A(x, BF(x))| (and the sum of K such determinants), whose tangents and Laplacian
are the autograd Jacobian and Hessian trace of the composite; full and spin-factorised determinants, per-orbital and three
envelope terms per nucleus, the default mult_act and the additive backflow branch."""
import pytest
import torch
from torch.autograd.functional import jacobian

from slater_reference import TailParams, det_sum_ref, logabsdet_lu, orbitals, slater_ref, slater_value

F64 = torch.float64
N, NUP, M, K = 4, 2, 2, 3
S = 3 * N + 2


def _params(g, rep=1, **kw):
    R = torch.randn(M, 3, generator=g, dtype=F64)
    t = lambda: torch.rand(K * N, M * rep, generator=g, dtype=F64) + 0.5
    return TailParams(R, t(), t(), t(), t(), NUP, K, **kw)


def _bf_of(g, width):
    """x [3N] -> [N, width] backflow rows, nonlinear in every coordinate (dense tangents, non-zero second derivatives)."""
    A, c = torch.randn(3 * N, N * width, generator=g, dtype=F64) / 3, torch.randn(N * width, generator=g, dtype=F64)
    return lambda x: torch.tanh(x @ A + c).reshape(N, width) * 1.5 + torch.sin(x[:N, None])


def _jets(f, x):
    """(value, d f / dx_t [.., 3N], sum_t d^2 f / dx_t^2) of f at x by autograd."""
    J = jacobian(f, x)
    Hs = jacobian(lambda y: jacobian(f, y, create_graph=True), x)
    return f(x), J, Hs.diagonal(dim1=-2, dim2=-1).sum(-1)


def _slot_rows(f, x):
    """The backflow rows with their autograd jets as slot rows [N S][width] (row i S + s)."""
    val, J, lap = _jets(f, x)
    return torch.cat([val[:, None], J.permute(0, 2, 1), lap[:, None]], dim=1).reshape(N * S, -1)


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max()).item()


CASES = [dict(), dict(full_det=False), dict(rep=3), dict(mult_act='default', full_det=False), dict(transform='add'),
         dict(transform='both')]


@pytest.mark.parametrize('case', range(len(CASES)))
def test_slater_ref_matches_autograd(case):
    """slater_ref fed with the autograd jets of BF(x) = the Jacobian and Hessian trace of log|det A(x, BF(x))|."""
    kw = dict(CASES[case])
    g = torch.Generator().manual_seed(case)
    P = _params(g, kw.pop('rep', 1), **kw)
    width = K * N * (2 if P.transform == 'both' else 1)
    bf = _bf_of(g, width)
    x = torch.randn(3 * N, generator=g, dtype=F64) * 0.8
    logdet = lambda y: slater_value(y.reshape(1, N, 3), bf(y)[None], P)[1][0]
    val, J, lap = _jets(logdet, x)
    sign, lg, grad, lp = slater_ref(x.reshape(1, N, 3), _slot_rows(bf, x), P, S)
    assert lg.dtype == F64 and grad.shape == (1, K, 3 * N) and lp.shape == (1, K)
    assert torch.all(sign.abs() == 1)
    assert _rel(lg[0], val) < 1e-12
    assert _rel(grad[0], J) < 1e-10
    assert _rel(lp[0], lap) < 1e-10
    if not P.full_det:  # spin-factorised: det A = det(up block) det(down block)
        A = orbitals(x.reshape(1, N, 3), bf(x)[None], P)[0]
        blocks = torch.linalg.slogdet(A[:, :NUP, :NUP])[1] + torch.linalg.slogdet(A[:, NUP:, NUP:])[1]
        assert _rel(lg[0], blocks) < 1e-12


@pytest.mark.parametrize('conf', [False, True])
def test_det_sum_ref_matches_autograd(conf):
    """det_sum_ref on K = 3 determinants of mixed sign (and hk.Linear weights with a negative one) whose logs and jets come
    from x = the Jacobian and Hessian trace of log|sum_k c_k s_k exp(l_k(x))|."""
    g = torch.Generator().manual_seed(7 + conf)
    Wl = torch.randn(3 * N, K, generator=g, dtype=F64)
    l_of = lambda x: torch.tanh(x @ Wl) * 3 + (x ** 2).sum() * torch.tensor([0.1, -0.2, 0.3], dtype=F64)
    s = torch.tensor([1.0, -1.0, 1.0], dtype=F64)
    w = torch.tensor([0.7, 1.3, -0.4], dtype=F64) if conf else None
    c = s * (w if conf else 1)
    x = torch.randn(3 * N, generator=g, dtype=F64)
    val, J, lap = _jets(lambda y: torch.log((c * torch.exp(l_of(y))).sum().abs()), x)
    lv, lJ, llap = _jets(l_of, x)
    sign, lg, grad, lp = det_sum_ref(s[None], lv[None], lJ[None], llap[None], conf_w=w)
    assert sign.item() == torch.sign((c * torch.exp(lv)).sum()).item()
    assert _rel(lg[0], val) < 1e-12
    assert _rel(grad[0], J) < 1e-10
    assert _rel(lp[0], lap) < 1e-10


def test_det_sum_ref_singular_determinants():
    """A determinant at (0, -inf) drops out of the sum and of its jets; all of them at (0, -inf) give sign 0, log -inf."""
    g = torch.Generator().manual_seed(11)
    l, gr, lp = torch.randn(1, 3, generator=g, dtype=F64), torch.randn(1, 3, 6, generator=g, dtype=F64), torch.randn(1, 3, generator=g, dtype=F64)
    s = torch.tensor([[1.0, -1.0, 1.0]], dtype=F64)
    full = det_sum_ref(s[:, :2], l[:, :2], gr[:, :2], lp[:, :2])
    s0, l0 = s.clone(), l.clone()
    s0[0, 2], l0[0, 2] = 0.0, -float('inf')
    part = det_sum_ref(s0, l0, gr, lp)
    for a, b in zip(full, part):
        assert torch.allclose(a, b, rtol=1e-14, atol=0)
    z = det_sum_ref(torch.zeros(1, 3, dtype=F64), torch.full((1, 3), -float('inf'), dtype=F64))
    assert z[0].item() == 0 and z[1].item() == -float('inf')


def test_logabsdet_lu_matches_slogdet():
    """The LU restatement gives slogdet's value on matrices that need row exchanges, in fp64 and in fp32."""
    g = torch.Generator().manual_seed(13)
    A = torch.randn(5, 3, 9, 9, generator=g, dtype=F64)
    A[..., 0, :] *= 1e-6  # the first row is never the first pivot
    assert _rel(logabsdet_lu(A), torch.linalg.slogdet(A)[1]) < 1e-13
    assert _rel(logabsdet_lu(A.float()).double(), torch.linalg.slogdet(A)[1]) < 1e-5


def test_slater_ref_runs_in_fp32():
    """The fp32 restatement (the yardstick of the GPU bounds) runs in fp32 end to end and agrees with fp64 to fp32 accuracy."""
    g = torch.Generator().manual_seed(5)
    P = _params(g)
    bf = _bf_of(g, K * N)
    x = torch.randn(3 * N, generator=g, dtype=F64)
    rows = _slot_rows(bf, x)
    r = x.reshape(1, N, 3)
    ref = slater_ref(r, rows, P, S)
    r32 = slater_ref(r.float(), rows.float(), P, S, dtype=torch.float32)
    assert all(t.dtype == torch.float32 for t in r32)
    for a, b in zip(ref[1:], r32[1:]):
        assert _rel(b.double(), a) < 1e-3
