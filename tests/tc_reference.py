"""Plain torch restatements of the Psiformer trunk layers and of the softmax attention, in fp64 (the reference) or fp32 (the
yardstick for what fp32 arithmetic gets wrong anyway); shared by the tensor-core kernel tests."""
import torch


def weight(eng, name, dtype=torch.float64):
    """Parameter `name` of the engine's table as the device sees it (rounded to fp32), as a [K, N] tensor."""
    flat = torch.as_tensor(eng._flat, device='cuda:0')
    off, K, Nc = eng.entries[name]
    return flat[off:off + K * Nc].reshape(K, Nc).float().to(dtype)


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
