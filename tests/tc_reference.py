"""Plain torch restatements of the Psiformer trunk layers and of the softmax attention, in fp64 (the reference) or fp32 (the
yardstick for what fp32 arithmetic gets wrong anyway), and of the forward-Laplacian jets of the attention and of the MLP after
it; shared by the tensor-core kernel tests."""
import torch


def weight(eng, name, dtype=torch.float64):
    """Parameter `name` of the engine's table as the device sees it (rounded to fp32 for an fp32 engine), as a [K, N] tensor."""
    flat = torch.as_tensor(eng._flat, device=eng.device)
    off, K, Nc = eng.entries[name]
    w = flat[off:off + K * Nc].reshape(K, Nc)
    return (w.float() if eng.dtype == torch.float32 else w).to(dtype)


def trunk_ref(eng, X0, N, L, H=4, dtype=torch.float64, peaks=None):
    """The layers of gnn/update_features.py:241-286 (hk.MultiHeadAttention + hkext.py MLP / residuals) in torch.  `peaks`: a
    dict that receives the largest |activation| and |Q|, |K|, |V| met on the way (the half operands' range check)."""
    W = lambda name: weight(eng, name, dtype)
    X = X0.to(dtype)
    rows, d = X.shape
    B, dh = rows // N, d // H
    act, qkv_peak = X.abs().max().item(), 0.0
    for l in range(L):
        p = f'L{l}.'
        QKV = X @ W(p + 'wqkv')
        qkv_peak = max(qkv_peak, QKV.abs().max().item())
        q, k, v = ((t.reshape(B, N, H, dh).permute(0, 2, 1, 3)) for t in QKV.split(d, dim=1))
        att = torch.softmax(q @ k.transpose(-1, -2) / dh ** 0.5, dim=-1)
        O = (att @ v).permute(0, 2, 1, 3).reshape(rows, d)
        A = X + O @ W(p + 'wo')
        M1 = torch.tanh(A @ W(p + 'w1') + W(p + 'b1')[0])
        X = A + torch.tanh(M1 @ W(p + 'w2') + W(p + 'b2')[0])
        act = max(act, A.abs().max().item(), X.abs().max().item())
    if peaks is not None:
        peaks.update(act=act, qkv=qkv_peak)
    return X


def attention_ref(QKV, N, H, kn=None, vn=None, dtype=torch.float64):
    """softmax(q [K; Kn]^T / sqrt(dh)) [V; Vn] per (walker, head) on Q | K | V rows [B N][3d] (nuclear tokens kn / vn [Mn][d]
    shared by every walker) -> (O [B N][d], sum_j p_j |v_j| [B N][d], the magnitude the weighted sum accumulates)."""
    rows, d3 = QKV.shape
    d = d3 // 3
    B, dh = rows // N, d // H
    q, k, v = ((t.to(dtype).reshape(B, N, H, dh).permute(0, 2, 1, 3)) for t in QKV.split(d, dim=1))
    if kn is not None:
        tok = lambda t: t.to(dtype).reshape(1, -1, H, dh).permute(0, 2, 1, 3).expand(B, H, -1, dh)
        k, v = torch.cat([k, tok(kn)], dim=2), torch.cat([v, tok(vn)], dim=2)
    p = torch.softmax(q @ k.transpose(-1, -2) / dh ** 0.5, dim=-1)
    back = lambda t: t.permute(0, 2, 1, 3).reshape(rows, d)
    return back(p @ v), back(p @ v.abs())


# ---- forward-Laplacian jets by nested forward-mode AD ----------------------------------------------------------------------
# A forward-Laplacian pass carries per electron S = 3N + 2 slots: the value x, the tangents x^t = dx / dr_t (t = 1 .. 3N) and the
# Laplacian x^L = sum_t d^2 x / dr_t^2.  For out = f(x):  out^t = Df[x^t],  out^L = Df[x^L] + sum_t D^2f[x^t, x^t].  The
# references below get both terms from torch.func.jvp of the plain value function (nested for the second derivative), not
# from the kernels' closed-form rules.

def jet(f, x, xt, xL):
    """(f(x), Df[x^t] for each t, Df[x^L] + sum_t D^2f[x^t, x^t]); xt stacks the tangents along dim 0."""
    from torch.func import jvp, vmap

    val, dL = jvp(f, (x,), (xL,))

    def along(v):
        return jvp(lambda y: jvp(f, (y,), (v,))[1], (x,), (v,))

    d1, d2 = vmap(along)(xt)
    return val, d1, dL + d2.sum(0)


def _slots(Y, N, S):
    """slot rows [B N S][c] (row (b N + i) S + s) -> (values [B, N, c], tangents [S - 2, B, N, c], Laplacians [B, N, c])."""
    y = Y.reshape(-1, N, S, Y.shape[-1])
    return y[:, :, 0], y[:, :, 1:S - 1].movedim(2, 0), y[:, :, S - 1]


def _unslots(val, d1, lap):
    return torch.cat([val[:, :, None], d1.movedim(0, 2), lap[:, :, None]], dim=2).reshape(-1, val.shape[-1])


def attention_value(qkv, H, kn=None, vn=None):
    """softmax(q [K; Kn]^T / sqrt(dh)) [V; Vn] per (walker, head) on Q | K | V [B, N, 3d] -> [B, N, d]; nuclear tokens
    kn / vn [Mn][d] are walker-independent constants."""
    B, N, d3 = qkv.shape
    d = d3 // 3
    dh = d // H
    q, k, v = (t.reshape(B, N, H, dh).transpose(1, 2) for t in qkv.split(d, dim=-1))
    if kn is not None:
        tok = lambda t: t.reshape(1, -1, H, dh).transpose(1, 2).expand(B, H, -1, dh)
        k, v = torch.cat([k, tok(kn)], dim=2), torch.cat([v, tok(vn)], dim=2)
    p = torch.softmax(q @ k.transpose(-1, -2) / dh ** 0.5, dim=-1)
    return (p @ v).transpose(1, 2).reshape(B, N, d)


def attention_fl_ref(QKV, N, H, S, kn=None, vn=None, dtype=torch.float64):
    """Forward-Laplacian softmax attention on slot rows QKV [B N S][3d] -> O [B N S][d] (same slot layout), by nested
    forward-mode AD of attention_value."""
    c = lambda t: None if t is None else t.to(dtype)
    kn, vn = c(kn), c(vn)
    x, xt, xL = _slots(QKV.to(dtype), N, S)
    return _unslots(*jet(lambda y: attention_value(y, H, kn, vn), x, xt, xL))


def mlp_value(ox, W):
    """O | X [..., 2d] -> A + tanh(tanh(A W1 + b1) W2 + b2), A = X + O Wo; W: name -> [K, N] tensor (biases [1, N])."""
    d = ox.shape[-1] // 2
    O, X = ox[..., :d], ox[..., d:]
    A = X + O @ W('wo')
    return A + torch.tanh(torch.tanh(A @ W('w1') + W('b1')[0]) @ W('w2') + W('b2')[0])


def mlp_fl_ref(eng, layer, O, X, N, S, dtype=torch.float64):
    """The engine's post-attention sequence of `layer` (mlp_value) with forward-Laplacian jets on slot rows O, X [B N S][d]
    -> [B N S][d].  eng: an engine (weights from its parameter table, as the device sees them) or a dict name -> tensor."""
    if isinstance(eng, dict):
        W = lambda n: eng[f'L{layer}.{n}'].to(O.device, dtype)
    else:
        W = lambda n: weight(eng, f'L{layer}.{n}', dtype).to(O.device)
    x, xt, xL = _slots(torch.cat([O, X], dim=1).to(dtype), N, S)
    return _unslots(*jet(lambda y: mlp_value(y, W), x, xt, xL))
