"""Thin Python owner of one ``dqmc_handle``: config marshalling, parameter packing, workspace.

Everything numerical happens inside libdqmc_b200.so; this module only moves pointers.  torch is
used for device memory and streams (plumbing).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from . import params as PN
from .spec import AnsatzSpec

MODE_FORWARD, MODE_LOCAL_ENERGY, MODE_VJP, MODE_MCMC, MODE_LANGEVIN, MODE_SPIN, MODE_GRAD_POS, MODE_ECP_FORCE = 0, 1, 2, 3, 4, 5, 6, 7
MODE_ZV_FORCE = 8
_TORCH_DTYPE = {0: torch.float64, 1: torch.float32}


def paulinet_backflow_hidden(spec: AnsatzSpec) -> list[int]:
    """Hidden widths of the per-spin backflow MLPs, padded to the wider spin."""
    du, dd = PN.backflow_dims(spec, spec.n_up)[:-1], PN.backflow_dims(spec, spec.n_down)[:-1]
    return [max(a, b) for a, b in zip(du, dd)]


def paulinet_env_rep(spec: AnsatzSpec) -> int:
    """Envelope terms per nucleus in the engine layout = the largest number of shells on one nucleus."""
    return max(max((spec.env_centers.count(c) for c in set(spec.env_centers)), default=1), 1)


def softplus(x):
    return np.logaddexp(0.0, x)


def nuclear_types(spec: AnsatzSpec) -> np.ndarray:
    """Atom type of every nucleus: the index of its charge among the sorted distinct charges (the hk.Embed input of
    NucleiEmbedding with atom_type_embedding, gnn/electron_gnn.py:516-524)."""
    return np.unique(np.asarray(spec.charges), return_inverse=True)[1]


def _pack_deeperwin(spec: AnsatzSpec, params: dict) -> dict[str, np.ndarray]:
    """DeepErwin tree -> engine entries.  Walker-independent preparation only: h_ne of the nuclear embeddings per layer
    (the sender data of the ne convolution, as the test ansatz's hne table) and the envelope exponents softplus(zeta)
    (wf/env.py:55-70; the Slater kernels take |exponent|, and softplus > 0)."""
    g = lambda k: np.asarray(params[k], dtype=np.float64)
    K, N = spec.n_determinants, spec.n_elec
    xn = g(PN.GNN + 'nuclei_embedding/~/embed:embeddings')[nuclear_types(spec)]  # [M, 32]
    out = {}
    for l in range(spec.n_layers):
        c, lp = PN.conv_prefix(l), PN.layer_prefix(l)
        for t in ('same', 'anti'):
            for m in ('w', 'h'):
                out[f'G{l}.{m}_{t}.0.w'] = g(c + f'{m}_{t}/linear_0:w')
                out[f'G{l}.{m}_{t}.0.b'] = g(c + f'{m}_{t}/linear_0:b')[None]
        out[f'G{l}.hne'] = np.tanh(xn @ g(c + 'h_ne/linear_0:w') + g(c + 'h_ne/linear_0:b'))
        out[f'G{l}.g.w'], out[f'G{l}.g.b'] = g(lp + 'g/linear_0:w'), g(lp + 'g/linear_0:b')[None]
        if l < spec.n_layers - 1:
            for t in PN.EDGE_TYPES:
                out[f'G{l}.u_{t}.0.w'], out[f'G{l}.u_{t}.0.b'] = g(lp + f'u{t}/linear_0:w'), g(lp + f'u{t}/linear_0:b')[None]
    for s_, t in (('up', 'up'), ('down', 'dn')):
        out[f'bf.{t}'], out[f'bfb.{t}'] = g((PN.BF_UP if t == 'up' else PN.BF_DN) + ':w'), np.zeros((1, K * N))
        out[f'env.pi_{t}'] = g(f'{PN.ENV}:pi_{s_}')
        out[f'env.zeta_{t}'] = softplus(g(f'{PN.ENV}:zetas_{s_}'))
    out['cusp.alpha'] = np.zeros((1, 2))
    return out


def _pack_haiku_params(spec: AnsatzSpec, params: dict, R=None) -> dict[str, np.ndarray]:
    """Haiku-named tree (deepqmc_b200.params) -> the engine's packed entries."""
    g = lambda k: np.asarray(params[k], dtype=np.float64)
    out = {}
    if spec.kind == 'deeperwin':
        return _pack_deeperwin(spec, params)
    if spec.kind in ('psiformer', 'transpsiformer'):
        out['emb.w'] = g(PN.GNN + 'electron_embedding/linear:w')
        for l in range(spec.n_layers):
            a = PN.attn_prefix(l) if spec.kind == 'psiformer' else PN.comb_prefix(l)
            out[f'L{l}.wqkv'] = np.concatenate(
                [g(a + f'multi_head_attention/{n}:w') for n in ('query', 'key', 'value')], axis=1
            )
            out[f'L{l}.wo'] = g(a + 'multi_head_attention/linear:w')
            out[f'L{l}.w1'], out[f'L{l}.b1'] = g(a + 'mlp/linear_0:w'), g(a + 'mlp/linear_0:b')[None]
            out[f'L{l}.w2'], out[f'L{l}.b2'] = g(a + 'mlp/linear_1:w'), g(a + 'mlp/linear_1:b')[None]
    elif spec.kind == 'paulinet':
        N, K, M, d, n_up = spec.n_elec, spec.n_determinants, spec.n_nuc, spec.embedding_dim, spec.n_up
        nl = spec.gnn_subnet_layers
        if spec.gnn_embedding == 'embed':
            out['emb.table'] = g(PN.GNN + 'electron_embedding/ElectronicEmbedding:embeddings')
        types = PN.EDGE_TYPES if spec.gnn_conv_ne else PN.EDGE_TYPES[:2]
        xn = g(PN.GNN + 'nuclei_embedding/~/embed:embeddings') if spec.gnn_conv_ne else None
        w_bias = spec.gnn_update == 'concatenate'
        for l in range(spec.n_layers):
            c, lp = PN.conv_prefix(l), PN.layer_prefix(l)
            for t in types:
                for i in range(nl):
                    out[f'G{l}.w_{t}.{i}.w'] = g(c + f'w_{t}/linear_{i}:w')
                    if w_bias:
                        out[f'G{l}.w_{t}.{i}.b'] = g(c + f'w_{t}/linear_{i}:b')[None]
                if t != 'ne':
                    for i in range(nl):
                        out[f'G{l}.h_{t}.{i}.w'] = g(c + f'h_{t}/linear_{i}:w')
                        out[f'G{l}.h_{t}.{i}.b'] = g(c + f'h_{t}/linear_{i}:b')[None]
                else:
                    # nuclear embeddings are an hk.Embed lookup (gnn/electron_gnn.py:514): h_ne of them is walker-independent
                    hn = xn
                    for i in range(nl):
                        hn = np.tanh(hn @ g(c + f'h_ne/linear_{i}:w') + g(c + f'h_ne/linear_{i}:b'))
                    out[f'G{l}.hne'] = hn
                if spec.gnn_update == 'featurewise':
                    out[f'G{l}.g_{t}.w'] = g(lp + f'g_conv_{t}/linear_0:w')
                    out[f'G{l}.g_{t}.b'] = g(lp + f'g_conv_{t}/linear_0:b')[None]
            if spec.gnn_update == 'concatenate':
                out[f'G{l}.g.w'] = g(lp + 'g/linear_0:w')
                if spec.gnn_g_bias:
                    out[f'G{l}.g.b'] = g(lp + 'g/linear_0:b')[None]
            if spec.gnn_deep_edges and l < spec.n_layers - 1:
                for i in range(nl):
                    out[f'G{l}.u.{i}.w'] = g(lp + f'u/linear_{i}:w')
                    out[f'G{l}.u.{i}.b'] = g(lp + f'u/linear_{i}:b')[None]
        for i in range(spec.jastrow_layers):
            out[f'J{i}.w'] = g(PN.JASTROW + f'linear_{i}:w')
            if i < spec.jastrow_layers - 1:
                out[f'J{i}.b'] = g(PN.JASTROW + f'linear_{i}:b')[None]
        hid = paulinet_backflow_hidden(spec)
        dims_pad = [d] + hid
        for tag, pre, n_spin, off in (('up', PN.BF_UP, n_up, 0), ('dn', PN.BF_DN, spec.n_down, 0 if spec.full_determinant else n_up)):
            base = pre.rsplit('linear_0', 1)[0]
            nl = spec.backflow_layers
            zb = lambda k, n: g(k) if spec.backflow_bias else np.zeros(n)
            for i in range(nl - 1):  # hidden layers, zero-padded to the wider spin (ssp(0) = 0 keeps the padding inert)
                w = g(base + f'linear_{i}:w')
                b = zb(base + f'linear_{i}:b', w.shape[1])
                wp, bp = np.zeros((dims_pad[i], dims_pad[i + 1])), np.zeros((1, dims_pad[i + 1]))
                wp[:w.shape[0], :w.shape[1]], bp[0, :b.shape[0]] = w, b
                out[f'bfh{i}.{tag}'], out[f'bfb{i}.{tag}'] = wp, bp
            w = g(base + f'linear_{nl - 1}:w')
            b = zb(base + f'linear_{nl - 1}:b', w.shape[1])
            n_orb = N if spec.full_determinant else n_spin
            cols = (np.arange(K)[:, None] * N + off + np.arange(n_orb)[None, :]).ravel()  # (k, mu') -> k N + mu
            wp, bp = np.zeros((dims_pad[-1], K * N)), np.zeros((1, K * N))
            wp[:w.shape[0], cols], bp[0, cols] = w, b
            out[f'bf.{tag}'], out[f'bfb.{tag}'] = wp, bp
        if spec.env_per_shell:
            # per-shell spin-restricted envelopes (wf/env.py:26-75) -> engine layout [K N][M rep], unused terms pi = 0
            rep = paulinet_env_rep(spec)
            pi, zeta = g(f'{PN.ENV}:pi'), g(f'{PN.ENV}:zetas')
            pe, ze = np.zeros((K * N, M * rep)), np.ones((K * N, M * rep))
            seen = {}
            for j, c in enumerate(spec.env_centers):
                sh = seen.get(c, 0)
                seen[c] = sh + 1
                pe[:, c * rep + sh], ze[:, c * rep + sh] = pi[:, j], zeta[j]
            for t in ('up', 'dn'):
                out[f'env.pi_{t}'], out[f'env.zeta_{t}'] = pe, ze
        else:
            for s_, t in (('up', 'up'), ('down', 'dn')):
                out[f'env.pi_{t}'] = g(f'{PN.ENV}:pi_{s_}')
                out[f'env.zeta_{t}'] = g(f'{PN.ENV}:zetas_{s_}')
        out['cusp.alpha'] = np.array([[spec.cusp_alpha, spec.cusp_alpha]], dtype=np.float64)
        if spec.conf_coeff == 'linear':
            out['conf.w'] = g(PN.CONF + ':w').reshape(1, K)
        return out
    elif spec.kind == 'ferminet':
        for l in range(spec.n_layers):
            lp = PN.layer_prefix(l)
            out[f'F{l}.wg'], out[f'F{l}.bg'] = g(lp + 'g/linear_0:w'), g(lp + 'g/linear_0:b')[None]
            if l < spec.n_layers - 1:
                out[f'F{l}.wu'], out[f'F{l}.bu'] = g(lp + 'u/linear_0:w'), g(lp + 'u/linear_0:b')[None]
    else:
        raise NotImplementedError(spec.kind)
    out['bf.up'], out['bf.dn'] = g(PN.BF_UP + ':w'), g(PN.BF_DN + ':w')
    if spec.backflow_transform == 'both':  # [multiplicative head | additive head]
        out['bf.up'] = np.concatenate([out['bf.up'], g(PN.BF_UP_ADD + ':w')], axis=1)
        out['bf.dn'] = np.concatenate([out['bf.dn'], g(PN.BF_DN_ADD + ':w')], axis=1)
    if spec.kind == 'transpsiformer':
        # walker-independent nuclear stream (deepqmc_b200/nuclear.py): per-layer key/value rows of the
        # nuclear tokens and the envelope exponents zetas[M, K, E] -> engine layout [K N][M E], pi = 1
        from .nuclear import nuclear_stream

        ns = nuclear_stream(spec, params, R)
        N, K, M, E = spec.n_elec, spec.n_determinants, spec.n_nuc, spec.n_env_per_nuc
        for l in range(spec.n_layers):
            out[f'L{l}.kn'], out[f'L{l}.vn'] = ns['kn'][l], ns['vn'][l]
        for s, t in (('up', 'up'), ('down', 'dn')):
            z = np.transpose(ns[f'zetas_{s}'], (1, 0, 2)).reshape(K, 1, M * E)  # [K][m E + e]
            out[f'env.zeta_{t}'] = np.broadcast_to(z, (K, N, M * E)).reshape(K * N, M * E).copy()
            out[f'env.pi_{t}'] = np.ones((K * N, M * E))
    else:
        for s, t in (('up', 'up'), ('down', 'dn')):
            out[f'env.pi_{t}'] = g(f'{PN.ENV}:pi_{s}')
            out[f'env.zeta_{t}'] = g(f'{PN.ENV}:zetas_{s}')
    if spec.cusp == 'psiformer':
        out['cusp.alpha'] = np.array([[g(f'{PN.CUSP}:same_alpha'), g(f'{PN.CUSP}:anti_alpha')]], dtype=np.float64)
    elif spec.cusp == 'deepqmc':
        out['cusp.alpha'] = np.array([[spec.cusp_alpha, spec.cusp_alpha]], dtype=np.float64)
    else:
        out['cusp.alpha'] = np.ones((1, 2))
    return out


def _unpack_psiformer_grads(spec: AnsatzSpec, entries: dict, flat) -> dict:
    """Engine-layout gradient vector -> Haiku-named tree (inverse of _pack_haiku_params for the Psiformer)."""
    def e(name):
        off, rows, cols = entries[name]
        return flat[off:off + rows * cols].reshape(rows, cols)

    d = spec.embedding_dim
    out = {PN.GNN + 'electron_embedding/linear:w': e('emb.w')}
    for l in range(spec.n_layers):
        a = PN.attn_prefix(l) if spec.kind == 'psiformer' else PN.comb_prefix(l)
        qkv = e(f'L{l}.wqkv')
        for j, n in enumerate(('query', 'key', 'value')):
            out[a + f'multi_head_attention/{n}:w'] = qkv[:, j * d:(j + 1) * d]
        out[a + 'multi_head_attention/linear:w'] = e(f'L{l}.wo')
        out[a + 'mlp/linear_0:w'], out[a + 'mlp/linear_0:b'] = e(f'L{l}.w1'), e(f'L{l}.b1')[0]
        out[a + 'mlp/linear_1:w'], out[a + 'mlp/linear_1:b'] = e(f'L{l}.w2'), e(f'L{l}.b2')[0]
    out[PN.BF_UP + ':w'], out[PN.BF_DN + ':w'] = e('bf.up'), e('bf.dn')
    if spec.kind == 'psiformer':
        for s_, t in (('up', 'up'), ('down', 'dn')):
            out[f'{PN.ENV}:pi_{s_}'] = e(f'env.pi_{t}')
            out[f'{PN.ENV}:zetas_{s_}'] = e(f'env.zeta_{t}')
    if spec.cusp == 'psiformer':
        ca = e('cusp.alpha')
        out[f'{PN.CUSP}:same_alpha'], out[f'{PN.CUSP}:anti_alpha'] = ca[0, 0], ca[0, 1]
    return out


def _unpack_deeperwin_grads(spec: AnsatzSpec, entries: dict, flat, params: dict) -> dict:
    """Engine-layout gradient vector -> Haiku-named DeepErwin tree (inverse of _pack_deeperwin).  The walker-independent
    preparation is differentiated here: the cotangents of the h_ne tables G<l>.hne are pulled back through
    tanh(embed[type] W + b) to h_ne and the atom-type embedding table, and the uploaded exponent softplus(zeta) maps its
    gradient through sigmoid(zeta)."""
    def e(name):
        off, rows, cols = entries[name]
        return flat[off:off + rows * cols].reshape(rows, cols)

    dev, dt = flat.device, flat.dtype
    leaf = lambda k: torch.as_tensor(np.asarray(params[k], dtype=np.float64)).requires_grad_(True)
    emb_k = PN.GNN + 'nuclei_embedding/~/embed:embeddings'
    emb = leaf(emb_k)
    types = torch.as_tensor(nuclear_types(spec))
    out, loss = {}, 0.0
    for l in range(spec.n_layers):
        c, lp = PN.conv_prefix(l), PN.layer_prefix(l)
        for t in ('same', 'anti'):
            for m in ('w', 'h'):
                out[c + f'{m}_{t}/linear_0:w'] = e(f'G{l}.{m}_{t}.0.w')
                out[c + f'{m}_{t}/linear_0:b'] = e(f'G{l}.{m}_{t}.0.b')[0]
        out[lp + 'g/linear_0:w'], out[lp + 'g/linear_0:b'] = e(f'G{l}.g.w'), e(f'G{l}.g.b')[0]
        if l < spec.n_layers - 1:
            for t in PN.EDGE_TYPES:
                out[lp + f'u{t}/linear_0:w'], out[lp + f'u{t}/linear_0:b'] = e(f'G{l}.u_{t}.0.w'), e(f'G{l}.u_{t}.0.b')[0]
        w, b = leaf(c + 'h_ne/linear_0:w'), leaf(c + 'h_ne/linear_0:b')
        hn = torch.tanh(emb[types] @ w + b)
        loss = loss + (hn * e(f'G{l}.hne').detach().cpu().double()).sum()
        out[c + 'h_ne/linear_0:w'], out[c + 'h_ne/linear_0:b'] = w, b
    loss.backward()
    for k, v in list(out.items()):
        if isinstance(v, torch.Tensor) and v.requires_grad:
            out[k] = v.grad.to(device=dev, dtype=dt)
    out[emb_k] = emb.grad.to(device=dev, dtype=dt)
    for s_, t in (('up', 'up'), ('down', 'dn')):
        out[(PN.BF_UP if t == 'up' else PN.BF_DN) + ':w'] = e(f'bf.{t}')
        out[f'{PN.ENV}:pi_{s_}'] = e(f'env.pi_{t}')
        z = torch.as_tensor(np.asarray(params[f'{PN.ENV}:zetas_{s_}'], dtype=np.float64), device=dev, dtype=dt)
        out[f'{PN.ENV}:zetas_{s_}'] = e(f'env.zeta_{t}') * torch.sigmoid(z)
    return out


def _unpack_paulinet_grads(spec: AnsatzSpec, entries: dict, flat, params: dict) -> dict:
    """Engine-layout gradient vector -> Haiku-named tree for the conv-GNN test ansatz (inverse of _pack_haiku_params for
    spec.kind == 'paulinet', featurewise / hk.Embed variant).  The walker-independent h_ne(nuclear embedding) rows were
    evaluated on the host at upload; their cotangents G<l>.hne are pulled back through that small tanh MLP here."""
    def e(name):
        off, rows, cols = entries[name]
        return flat[off:off + rows * cols].reshape(rows, cols)

    N, K, M, d, n_up = spec.n_elec, spec.n_determinants, spec.n_nuc, spec.embedding_dim, spec.n_up
    nl = spec.gnn_subnet_layers
    out = {}
    if spec.gnn_embedding == 'embed':
        out[PN.GNN + 'electron_embedding/ElectronicEmbedding:embeddings'] = e('emb.table')
    types = PN.EDGE_TYPES if spec.gnn_conv_ne else PN.EDGE_TYPES[:2]
    dxn = None
    for l in range(spec.n_layers):
        c, lp = PN.conv_prefix(l), PN.layer_prefix(l)
        for t in types:
            for i in range(nl):
                out[c + f'w_{t}/linear_{i}:w'] = e(f'G{l}.w_{t}.{i}.w')
                if spec.gnn_update == 'concatenate':
                    out[c + f'w_{t}/linear_{i}:b'] = e(f'G{l}.w_{t}.{i}.b')[0]
                if t != 'ne':
                    out[c + f'h_{t}/linear_{i}:w'] = e(f'G{l}.h_{t}.{i}.w')
                    out[c + f'h_{t}/linear_{i}:b'] = e(f'G{l}.h_{t}.{i}.b')[0]
            if spec.gnn_update == 'featurewise':
                out[lp + f'g_conv_{t}/linear_0:w'] = e(f'G{l}.g_{t}.w')
                out[lp + f'g_conv_{t}/linear_0:b'] = e(f'G{l}.g_{t}.b')[0]
        if spec.gnn_update == 'concatenate':
            out[lp + 'g/linear_0:w'] = e(f'G{l}.g.w')
            if spec.gnn_g_bias:
                out[lp + 'g/linear_0:b'] = e(f'G{l}.g.b')[0]
        if spec.gnn_deep_edges and l < spec.n_layers - 1:
            for i in range(nl):
                out[lp + f'u/linear_{i}:w'] = e(f'G{l}.u.{i}.w')
                out[lp + f'u/linear_{i}:b'] = e(f'G{l}.u.{i}.b')[0]
        if spec.gnn_conv_ne:  # host: hne = tanh MLP(xn) -> gradients of the nuclear table and of h_ne
            leaves = {k: torch.as_tensor(np.asarray(params[k], dtype=np.float64)).requires_grad_(True)
                      for k in [PN.GNN + 'nuclei_embedding/~/embed:embeddings']
                      + [c + f'h_ne/linear_{i}:{wb}' for i in range(nl) for wb in 'wb']}
            hn = leaves[PN.GNN + 'nuclei_embedding/~/embed:embeddings']
            for i in range(nl):
                hn = torch.tanh(hn @ leaves[c + f'h_ne/linear_{i}:w'] + leaves[c + f'h_ne/linear_{i}:b'])
            (hn * e(f'G{l}.hne').detach().cpu().double()).sum().backward()
            for k, v in leaves.items():
                g = v.grad.to(device=flat.device, dtype=flat.dtype)
                if k.endswith('embed:embeddings'):
                    dxn = g if dxn is None else dxn + g
                else:
                    out[k] = g
    if dxn is not None:
        out[PN.GNN + 'nuclei_embedding/~/embed:embeddings'] = dxn
    for i in range(spec.jastrow_layers):
        out[PN.JASTROW + f'linear_{i}:w'] = e(f'J{i}.w')
        if i < spec.jastrow_layers - 1:
            out[PN.JASTROW + f'linear_{i}:b'] = e(f'J{i}.b')[0]
    for tag, pre, n_spin, off in (('up', PN.BF_UP, n_up, 0), ('dn', PN.BF_DN, spec.n_down, 0 if spec.full_determinant else n_up)):
        base = pre.rsplit('linear_0', 1)[0]
        nb = spec.backflow_layers
        for i in range(nb - 1):
            shp = np.asarray(params[base + f'linear_{i}:w']).shape
            out[base + f'linear_{i}:w'] = e(f'bfh{i}.{tag}')[:shp[0], :shp[1]]
            if spec.backflow_bias:
                out[base + f'linear_{i}:b'] = e(f'bfb{i}.{tag}')[0, :shp[1]]
        shp = np.asarray(params[base + f'linear_{nb - 1}:w']).shape
        n_orb = N if spec.full_determinant else n_spin
        cols = torch.as_tensor((np.arange(K)[:, None] * N + off + np.arange(n_orb)[None, :]).ravel(), device=flat.device)
        out[base + f'linear_{nb - 1}:w'] = e(f'bf.{tag}')[:shp[0]][:, cols]
        if spec.backflow_bias:
            out[base + f'linear_{nb - 1}:b'] = e(f'bfb.{tag}')[0, cols]
    if spec.env_per_shell:  # packed [K N][M rep] (both spins share the parameters) -> pi[K N, n_env], zetas[n_env]
        rep = paulinet_env_rep(spec)
        idx, seen = [], {}
        for c_ in spec.env_centers:
            sh = seen.get(c_, 0)
            seen[c_] = sh + 1
            idx.append(c_ * rep + sh)
        idx = torch.as_tensor(idx, device=flat.device)
        dpi = e('env.pi_up') + e('env.pi_dn')
        dze = e('env.zeta_up') + e('env.zeta_dn')
        out[f'{PN.ENV}:pi'] = dpi[:, idx]
        out[f'{PN.ENV}:zetas'] = dze[:, idx].sum(0)
    else:
        for s_, t in (('up', 'up'), ('down', 'dn')):
            out[f'{PN.ENV}:pi_{s_}'] = e(f'env.pi_{t}')
            out[f'{PN.ENV}:zetas_{s_}'] = e(f'env.zeta_{t}')
    if spec.conf_coeff == 'linear':
        out[PN.CONF + ':w'] = e('conf.w').reshape(spec.n_determinants, 1)
    return out


def _unpack_ferminet_grads(spec: AnsatzSpec, entries: dict, flat) -> dict:
    """Engine-layout gradient vector -> Haiku-named tree for the FermiNet (inverse of _pack_haiku_params)."""
    def e(name):
        off, rows, cols = entries[name]
        return flat[off:off + rows * cols].reshape(rows, cols)

    out = {}
    for l in range(spec.n_layers):
        lp = PN.layer_prefix(l)
        out[lp + 'g/linear_0:w'], out[lp + 'g/linear_0:b'] = e(f'F{l}.wg'), e(f'F{l}.bg')[0]
        if l < spec.n_layers - 1:
            out[lp + 'u/linear_0:w'], out[lp + 'u/linear_0:b'] = e(f'F{l}.wu'), e(f'F{l}.bu')[0]
    out[PN.BF_UP + ':w'], out[PN.BF_DN + ':w'] = e('bf.up'), e('bf.dn')
    for s_, t in (('up', 'up'), ('down', 'dn')):
        out[f'{PN.ENV}:pi_{s_}'] = e(f'env.pi_{t}')
        out[f'{PN.ENV}:zetas_{s_}'] = e(f'env.zeta_{t}')
    if spec.cusp == 'psiformer':
        ca = e('cusp.alpha')
        out[f'{PN.CUSP}:same_alpha'], out[f'{PN.CUSP}:anti_alpha'] = ca[0, 0], ca[0, 1]
    return out


class Engine:
    """One engine per (ansatz spec, Hamiltonian constants, dtype, device)."""

    def __init__(self, spec: AnsatzSpec, hamil, dtype: str = 'float64', device: int | None = None,
                 gemm_backend: int = 0, _lib_path: str | None = None, plan_only: bool = False):
        """``plan_only``: a handle created with device = -1 -- no CUDA context; only the parameter table, the workspace
        sizes and ``debug_plan`` work (tests/test_plan.py checks the workspace planner on the CPU with it)."""
        self._host = _lib_path is not None  # emulator build: "device" pointers are host pointers
        self.lib = _lib.load(_lib_path)
        self.plan_only = plan_only
        if not self._host and not plan_only and not torch.cuda.is_available():
            raise RuntimeError('deepqmc_b200 needs a CUDA device (H100, sm_90a); there is no CPU path')
        self.spec, self.hamil = spec, hamil
        self.dtype_code = {'float64': 0, 'float32': 1}[dtype]
        self.dtype = _TORCH_DTYPE[self.dtype_code]
        if plan_only:
            self.device_index, self.device = -1, torch.device('cpu')
        else:
            self.device_index = 0 if self._host else (torch.cuda.current_device() if device is None else device)
            self.device = torch.device('cpu') if self._host else torch.device('cuda', self.device_index)
        cfg = _lib.DqmcConfig()
        cfg.kind = {'psiformer': 0, 'ferminet': 1, 'transpsiformer': 2, 'paulinet': 3, 'deeperwin': 3}[spec.kind]
        cfg.dtype, cfg.gemm_backend = self.dtype_code, gemm_backend
        cfg.n_up, cfg.n_down, cfg.n_nuc = spec.n_up, spec.n_down, spec.n_nuc
        cfg.embedding_dim, cfg.n_layers, cfg.n_heads = spec.embedding_dim, spec.n_layers, spec.n_heads
        cfg.n_determinants, cfg.edge_dim = spec.n_determinants, spec.edge_dim
        cfg.n_env_per_nuc = spec.n_env_per_nuc
        cfg.n_nuc_tokens = spec.n_nuc if spec.kind == 'transpsiformer' else 0
        if spec.kind in ('paulinet', 'deeperwin'):
            cfg.n_env_per_nuc = paulinet_env_rep(spec) if spec.env_per_shell else 1
            cfg.gnn_features = 1 if spec.gnn_embedding == 'features' else 0
            cfg.gnn_concat = 1 if spec.gnn_update == 'concatenate' else 0
            cfg.gnn_conv_ne = 1 if spec.gnn_conv_ne else 0
            cfg.gnn_sub_n = spec.gnn_subnet_layers
            cfg.gnn_deep_edges = 1 if spec.gnn_deep_edges else 0
            cfg.gnn_res_norm = 1 if spec.gnn_residual_normalize else 0
            cfg.gnn_g_bias = 1 if spec.gnn_g_bias else 0
            cfg.gnn_w_bias = 1 if spec.gnn_update == 'concatenate' else 0
            assert spec.n_layers <= 8 and spec.gnn_subnet_layers <= 4
            if spec.kind == 'deeperwin':  # conf/ansatz/deeperwin.yaml (deepqmc_b200.spec.deeperwin_spec)
                cfg.gnn_sep_edges = cfg.gnn_self_edges = cfg.gnn_ne_identity = cfg.gnn_no_res = 1
                cfg.gnn_edge_in[:] = [PN.DEEPERWIN_EDGE_IN[t] for t in PN.EDGE_TYPES]
            d_in, e_in = (spec.embedding_dim if spec.gnn_embedding == 'embed' else 4 * spec.n_nuc), 4
            for l in range(spec.n_layers):
                for i, v in enumerate(PN.log_dims(e_in, spec.edge_dim, spec.gnn_subnet_layers)):
                    cfg.gnn_w_dims[l * 4 + i] = v
                    cfg.gnn_u_dims[l * 4 + i] = v
                for i, v in enumerate(PN.log_dims(d_in, spec.edge_dim, spec.gnn_subnet_layers)):
                    cfg.gnn_h_dims[l * 4 + i] = v
                if spec.gnn_deep_edges and l < spec.n_layers - 1:
                    e_in = spec.edge_dim
                d_in = spec.embedding_dim
            cfg.factorized_det = 0 if spec.full_determinant else 1
            cfg.conf_linear = 1 if spec.conf_coeff == 'linear' else 0
            cfg.mult_act = 1 if spec.mult_act == 'default' else 0
            cfg.n_elec_types = 1 if spec.n_up == spec.n_down else 2
            jd = PN.log_dims(spec.embedding_dim, 1, spec.jastrow_layers) if spec.jastrow_layers else []
            cfg.jastrow_n = len(jd)
            for i, v in enumerate(jd):
                cfg.jastrow_dims[i] = v
            hid = paulinet_backflow_hidden(spec)
            cfg.backflow_n = len(hid)
            for i, v in enumerate(hid):
                cfg.backflow_dims[i] = v
        cfg.cusp_kind = {'psiformer': 1, 'deepqmc': 2}.get(spec.cusp, 0)
        cfg.backflow_add = {'mult': 0, 'add': 1, 'both': 2}[spec.backflow_transform]
        if cfg.backflow_add and spec.kind not in ('psiformer', 'ferminet'):
            raise NotImplementedError('additive backflow branch: Psiformer / FermiNet kinds only')
        cfg.nuc_cusp_kind = {'psiformer': 1, 'deepqmc': 2}.get(spec.cusp_nuclei, 0)
        for m in range(spec.n_nuc):
            cfg.z_nuclear[m] = float(hamil.mol.charges[m])
        cfg.cusp_same_scale, cfg.cusp_anti_scale = spec.cusp_same_scale, spec.cusp_anti_scale
        M = spec.n_nuc
        assert M <= _lib.MAX_NUC
        for m in range(M):
            cfg.z_valence[m] = float(hamil.ns_valence[m])
            cfg.ecp_mask[m] = int(hamil.ecp_mask[m])
        lp, nl = getattr(hamil, 'loc_params', None), getattr(hamil, 'nl_params', None)
        if lp is not None and lp.shape[-1] > 0:
            Tm = lp.shape[-1]
            assert Tm <= _lib.MAX_T
            cfg.ecp_loc_terms = Tm
            arr = np.zeros((_lib.MAX_NUC, 3, 2, _lib.MAX_T))
            arr[:M, :, :, :Tm] = lp
            cfg.ecp_loc[:] = arr.ravel().tolist()
        if nl is not None and nl.size > 0:
            L, Tn = nl.shape[1], nl.shape[3]
            assert L <= _lib.MAX_L and Tn <= _lib.MAX_T
            cfg.ecp_nl_lmax_p1, cfg.ecp_nl_terms = L, Tn
            arr = np.zeros((_lib.MAX_NUC, _lib.MAX_L, 2, _lib.MAX_T))
            arr[:M, :L, :, :Tn] = nl
            cfg.ecp_nl[:] = arr.ravel().tolist()
        self._cfg = cfg
        h = C.c_void_p()
        rc = self.lib.dqmc_create(C.byref(cfg), self.device_index, C.byref(h))
        if rc != 0:
            raise RuntimeError(f'dqmc_create failed with status {rc}')
        self.h = h
        ph = getattr(hamil, 'ph', None)
        if ph is not None:  # pseudo-Hamiltonian tables (deepqmc_b200/ph.py) -> device
            n_tab, _, G = ph.tables.shape
            rc = self.lib.dqmc_set_pseudo_hamiltonian(h, n_tab, G, float(ph.r_max),
                                                      ph.tables.ctypes.data_as(C.POINTER(C.c_double)),
                                                      ph.tab_of_nuc.ctypes.data_as(C.POINTER(C.c_int32)))
            self._check(rc, 'dqmc_set_pseudo_hamiltonian')
        self.entries = {}
        name = C.create_string_buffer(64)
        off, rows, cols = C.c_int64(), C.c_int32(), C.c_int32()
        for i in range(self.lib.dqmc_param_count(h)):
            self.lib.dqmc_param_entry(h, i, name, 64, C.byref(off), C.byref(rows), C.byref(cols))
            self.entries[name.value.decode()] = (off.value, rows.value, cols.value)
        self.n_packed = self.lib.dqmc_param_total(h)
        self._ws = None
        self._ws_ok = {}  # (n_walkers, mode, cap) -> the workspace (view) that serves that request
        self._params_version = None
        self._nuc_R_dev = None

    # ------------------------------------------------------------------------------------
    def _check(self, rc, what):
        if rc != 0:
            raise RuntimeError(f'{what} failed ({rc}): {self.lib.dqmc_last_error(self.h).decode()}')

    def _stream(self):
        return C.c_void_p(0 if self._host else torch.cuda.current_stream(self.device).cuda_stream)

    def set_params(self, params: dict, R=None):
        """Upload a parameter tree.  TransPsiformer: ``R`` (default: the Hamiltonian's geometry) fixes
        the walker-independent nuclear stream that is uploaded with the parameters."""
        if self.spec.kind == 'transpsiformer':
            R = self.hamil.mol.coords if R is None else R
            R = np.asarray(R.detach().cpu() if torch.is_tensor(R) else R, dtype=np.float64)
            self._nuc_R, self._nuc_R_dev = R, None
        self._params = params
        packed = _pack_haiku_params(self.spec, params, R)
        if self.spec.cusp_nuclei != 'none':  # NuclearCuspAsymptotic: alpha (trainable or fixed) + the nuclear charges
            al = (float(np.asarray(params[f'{PN.NUC_CUSP}:nuc_alpha'])) if self.spec.cusp_nuclei_trainable
                  else self.spec.cusp_nuclei_alpha)
            packed['cusp.nuc'] = np.array([[al, *[float(z) for z in self.hamil.mol.charges]]], dtype=np.float64)
        flat = np.zeros(self.n_packed, dtype=np.float64)
        for k, (off, rows, cols) in self.entries.items():
            v = packed[k]
            assert v.shape == (rows, cols), (k, v.shape, rows, cols)
            flat[off:off + rows * cols] = v.ravel()
        self._flat = flat  # keep alive until the async copy is done
        rc = self.lib.dqmc_set_params(self.h, flat.ctypes.data_as(C.POINTER(C.c_double)), self.n_packed, self._stream())
        self._check(rc, 'dqmc_set_params')
        if not self._host:
            torch.cuda.current_stream(self.device).synchronize()

    def workspace(self, n_walkers: int, mode: int, max_bytes: int | None = None):
        """The engine's scratch buffer for one call of the entry point ``mode`` names: dqmc_workspace_bytes (a dry pass of the
        code that carves it), capped at ``max_bytes`` / 60 % of the free HBM -- the engine then chunks the walkers -- but
        never below dqmc_workspace_bytes_min.  An explicit ``max_bytes`` also caps the view handed to the call when a larger
        buffer is already held, so the engine chunks exactly as that size makes it."""
        key = (n_walkers, mode, max_bytes)
        if self._ws is not None and key in self._ws_ok:  # hot path: no driver queries per call
            return self._ws_ok[key]
        explicit = max_bytes is not None
        need = self.lib.dqmc_workspace_bytes(self.h, n_walkers, mode)
        if max_bytes is None and not self._host:
            free = torch.cuda.mem_get_info(self.device)[0] + (self._ws.numel() if self._ws is not None else 0)
            max_bytes = int(0.6 * free)
        if max_bytes is not None:
            need = min(need, max(max_bytes, self.lib.dqmc_workspace_bytes_min(self.h, n_walkers, mode)))
        if self._ws is None or self._ws.numel() < need:
            self._ws = None
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
            self._ws_ok = {}
        self._ws_ok[key] = self._ws[:need] if explicit else self._ws
        return self._ws_ok[key]

    def _prep(self, x):
        x = torch.as_tensor(x, dtype=self.dtype, device=self.device)
        return x.contiguous()

    def _R(self, R, B):
        R = self._prep(R)
        assert R.dim() in (2, 3) and tuple(R.shape[-2:]) == (self.spec.n_nuc, 3), f'R must be [M, 3] or [B, M, 3], got {tuple(R.shape)}'
        batched = 1 if R.dim() == 3 else 0
        if batched:
            assert R.shape[0] == B
        if self.spec.kind == 'transpsiformer':
            if batched:
                raise NotImplementedError('TransPsiformer engine: one geometry per call (unbatched R)')
            # the nuclear stream depends on the geometry: compare the CONTENTS with the geometry it was evaluated for (never a
            # pointer / version key: temporaries of different geometries reuse addresses in the caching allocator)
            if self._nuc_R_dev is None or self._nuc_R_dev.device != R.device or not torch.equal(R.double(), self._nuc_R_dev):
                Rh = R.detach().cpu().double().numpy()
                if not np.allclose(Rh, self._nuc_R, rtol=0, atol=1e-12):
                    self.set_params(self._params, Rh)
                self._nuc_R_dev = R.detach().double().clone()
        return R, batched

    # ------------------------------------------------------------------------------------
    def wf_forward(self, r, R, max_ws_bytes=None):
        r = self._prep(r)
        B = r.shape[0]
        R, Rb = self._R(R, B)
        sign = torch.empty(B, dtype=self.dtype, device=self.device)
        log = torch.empty(B, dtype=self.dtype, device=self.device)
        ws = self.workspace(B, MODE_FORWARD, max_ws_bytes)
        rc = self.lib.dqmc_wf_forward(self.h, r.data_ptr(), R.data_ptr(), Rb, B, sign.data_ptr(), log.data_ptr(),
                                      ws.data_ptr(), ws.numel(), self._stream())
        self._check(rc, 'dqmc_wf_forward')
        return sign, log

    def wf_orbitals(self, r, R, max_ws_bytes=None):
        """-> (orb_up[B, K, n_up, n_orb], orb_down[B, K, n_down, n_orb]): envelope * mult_act(backflow), the matrices whose
        determinants make up psi; n_orb = N for full determinants, the spin's electron count otherwise
        (reference: Ansatz.apply(..., return_mos=True), wf/nn_wave_function.py:131-142)."""
        r = self._prep(r)
        B, N = r.shape[0], r.shape[1]
        R, Rb = self._R(R, B)
        K, n_up = self.spec.n_determinants, self.spec.n_up
        out = torch.empty(B, K, N, N, dtype=self.dtype, device=self.device)
        ws = self.workspace(B, MODE_FORWARD, max_ws_bytes)
        rc = self.lib.dqmc_wf_orbitals(self.h, r.data_ptr(), R.data_ptr(), Rb, B, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                       self._stream())
        self._check(rc, 'dqmc_wf_orbitals')
        if self.spec.full_determinant:
            return out[:, :, :n_up, :], out[:, :, n_up:, :]
        return out[:, :, :n_up, :n_up], out[:, :, n_up:, n_up:]

    def local_energy(self, r, R, seed=0, ecp_twist=None, want_grad=False, max_ws_bytes=None):
        r = self._prep(r)
        B, N = r.shape[0], r.shape[1]
        R, Rb = self._R(R, B)
        mk = lambda *s: torch.empty(*s, dtype=self.dtype, device=self.device)
        E, stats, sign, log = mk(B), mk(6, B), mk(B), mk(B)
        grad = mk(B, 3 * N) if want_grad else None
        tw = self._prep(ecp_twist) if ecp_twist is not None else None
        ws = self.workspace(B, MODE_LOCAL_ENERGY, max_ws_bytes)
        rc = self.lib.dqmc_local_energy(
            self.h, r.data_ptr(), R.data_ptr(), Rb, B, seed, tw.data_ptr() if tw is not None else None,
            E.data_ptr(), stats.data_ptr(), sign.data_ptr(), log.data_ptr(),
            grad.data_ptr() if grad is not None else None, ws.data_ptr(), ws.numel(), self._stream())
        self._check(rc, 'dqmc_local_energy')
        return E, stats, sign, log, grad

    def vjp_params(self, r, R, weights, max_ws_bytes=None):
        """-> (sign[B], log[B], grads): grads = d/dparams sum_b weights[b] log|psi(r_b)| as a Haiku-named dict
        (reference: loss/loss_function.py:53-82; SURVEY.md 8(f) N1).  Every ansatz kind (the additive backflow branch excepted)."""
        r = self._prep(r)
        B = r.shape[0]
        R, Rb = self._R(R, B)
        w = self._prep(weights)
        assert w.shape == (B,)
        sign = torch.empty(B, dtype=self.dtype, device=self.device)
        log = torch.empty(B, dtype=self.dtype, device=self.device)
        flat = torch.empty(self.n_packed, dtype=self.dtype, device=self.device)
        ws = self.workspace(B, MODE_VJP, max_ws_bytes)
        rc = self.lib.dqmc_wf_vjp_params(self.h, r.data_ptr(), R.data_ptr(), Rb, B, w.data_ptr(), sign.data_ptr(), log.data_ptr(),
                                         flat.data_ptr(), ws.data_ptr(), ws.numel(), self._stream())
        self._check(rc, 'dqmc_wf_vjp_params')
        if self.spec.kind == 'deeperwin':
            grads = _unpack_deeperwin_grads(self.spec, self.entries, flat, self._params)
        elif self.spec.kind == 'paulinet':
            grads = _unpack_paulinet_grads(self.spec, self.entries, flat, self._params)
        else:
            unpack = _unpack_ferminet_grads if self.spec.kind == 'ferminet' else _unpack_psiformer_grads
            grads = unpack(self.spec, self.entries, flat)
        if self.spec.cusp_nuclei != 'none' and self.spec.cusp_nuclei_trainable:
            grads[f'{PN.NUC_CUSP}:nuc_alpha'] = flat[self.entries['cusp.nuc'][0]]
        if self.spec.kind == 'transpsiformer':
            # the walker-independent nuclear stream is differentiated on the host: the engine accumulated the
            # cotangents of its outputs (keys / values of the nuclear tokens, envelope exponents)
            from .nuclear import nuclear_stream_vjp

            def e(name):
                off, rows, cols = self.entries[name]
                return flat[off:off + rows * cols].reshape(rows, cols).detach().cpu().double().numpy()

            N, K, M, E = self.spec.n_elec, self.spec.n_determinants, self.spec.n_nuc, self.spec.n_env_per_nuc
            cot = {'kn': [e(f'L{l}.kn') for l in range(self.spec.n_layers)],
                   'vn': [e(f'L{l}.vn') for l in range(self.spec.n_layers)]}
            for s_, t in (('up', 'up'), ('down', 'dn')):  # engine [K N][M E] -> zetas[M, K, E] (shared by the orbitals)
                cot[f'zetas_{s_}'] = e(f'env.zeta_{t}').reshape(K, N, M, E).sum(1).transpose(1, 0, 2)
            host = nuclear_stream_vjp(self.spec, self._params, self._nuc_R, cot)
            for k, v in host.items():
                v = v.to(device=self.device, dtype=self.dtype)
                grads[k] = grads[k] + v.reshape(grads[k].shape) if k in grads else v
        return sign, log, grads

    def spin(self, r, R, sign=None, log=None, down_idx=-1, want_ratios=False, max_ws_bytes=None):
        """-> (s2[B], ratios[B, P] or None).  down_idx = -1: exact <S^2> per walker over all n_up n_down swaps (P = n_up n_down,
        p = a n_down + (b - n_up)); down_idx in [n_up, N): the spin-raising contribution of that down electron (P = n_up,
        p = a).  sign / log of the walkers are optional (computed inside the call when missing)
        (reference: physics.py:159-239; dqmc_spin)."""
        r = self._prep(r)
        B = r.shape[0]
        R, Rb = self._R(R, B)
        n_up, n_down = self.spec.n_up, self.spec.n_down
        P = n_up * n_down if down_idx < 0 else n_up
        s2 = torch.empty(B, dtype=self.dtype, device=self.device)
        ratio = torch.empty(B, P, dtype=self.dtype, device=self.device) if want_ratios else None
        sg = self._prep(sign) if sign is not None else None
        lg = self._prep(log) if log is not None else None
        ptr = lambda t: t.data_ptr() if t is not None else None
        ws = self.workspace(B, MODE_SPIN, max_ws_bytes)
        rc = self.lib.dqmc_spin(self.h, r.data_ptr(), R.data_ptr(), Rb, B, ptr(sg), ptr(lg), int(down_idx), s2.data_ptr(),
                                ptr(ratio), ws.data_ptr(), ws.numel(), self._stream())
        self._check(rc, 'dqmc_spin')
        return s2, ratio

    def grad_positions(self, r, R, want_r=True, want_R=True, max_ws_bytes=None):
        """-> (sign[B], log[B], grad_r[B, N, 3] or None, grad_R[B, M, 3] or None): gradients of log|psi| with respect to the
        electron and nuclear positions by the reverse pass (dqmc_wf_grad_positions; reference force.py:96-118).  Psiformer and
        FermiNet: both; TransPsiformer: grad_r only; conv-GNN kinds and the additive backflow branch: not available."""
        r = self._prep(r)
        B, N = r.shape[0], r.shape[1]
        R, Rb = self._R(R, B)
        mk = lambda *s: torch.empty(*s, dtype=self.dtype, device=self.device)
        sign, log = mk(B), mk(B)
        gr = mk(B, N, 3) if want_r else None
        gR = mk(B, self.spec.n_nuc, 3) if want_R else None
        ptr = lambda t: t.data_ptr() if t is not None else None
        ws = self.workspace(B, MODE_GRAD_POS, max_ws_bytes)
        rc = self.lib.dqmc_wf_grad_positions(self.h, r.data_ptr(), R.data_ptr(), Rb, B, sign.data_ptr(), log.data_ptr(), ptr(gr),
                                             ptr(gR), ws.data_ptr(), ws.numel(), self._stream())
        self._check(rc, 'dqmc_wf_grad_positions')
        return sign, log, gr, gR

    def force_terms(self, r, R, grad_r=None):
        """-> (bare[B, M, 3], zvq[B, M, 3] or None, Q[B, M, 3]): the closed-form per-walker force terms of dqmc_force_terms
        (all-electron Hamiltonians); zvq needs ``grad_r`` [B, N, 3] = grad_r log|psi|."""
        r = self._prep(r)
        B = r.shape[0]
        R, Rb = self._R(R, B)
        mk = lambda *s: torch.empty(*s, dtype=self.dtype, device=self.device)
        M = self.spec.n_nuc
        bare, Q = mk(B, M, 3), mk(B, M, 3)
        g = self._prep(grad_r).reshape(B, -1) if grad_r is not None else None
        zvq = mk(B, M, 3) if g is not None else None
        ptr = lambda t: t.data_ptr() if t is not None else None
        rc = self.lib.dqmc_force_terms(self.h, r.data_ptr(), R.data_ptr(), Rb, B, ptr(g), bare.data_ptr(), ptr(zvq), Q.data_ptr(),
                                       self._stream())
        self._check(rc, 'dqmc_force_terms')
        return bare, zvq, Q

    def ecp_force(self, r, R, seed=0, ecp_twist=None, want_nl=True, max_ws_bytes=None):
        """-> (bare[B, M, 3], nl[B, M, 3] or None): the Hellmann-Feynman force terms with an effective core potential
        (dqmc_ecp_force): bare = F_nuc(Z_eff) - grad_R V_loc, nl = -grad_R V_nl (reference force.py:295-297,
        gaussian_type_ecp.py:257-328), nl in the nucleus' own row.  ``seed`` / ``ecp_twist`` [B, J, N] choose the quadrature
        twists as in ``local_energy``.  nl: Psiformer and FermiNet with multiplicative backflow, unbatched R."""
        r = self._prep(r)
        B = r.shape[0]
        R, Rb = self._R(R, B)
        mk = lambda *s: torch.empty(*s, dtype=self.dtype, device=self.device)
        M = self.spec.n_nuc
        bare = mk(B, M, 3)
        nl = mk(B, M, 3) if want_nl else None
        tw = self._prep(ecp_twist) if ecp_twist is not None else None
        ptr = lambda t: t.data_ptr() if t is not None else None
        ws = self.workspace(B, MODE_ECP_FORCE, max_ws_bytes) if want_nl else None
        rc = self.lib.dqmc_ecp_force(self.h, r.data_ptr(), R.data_ptr(), Rb, B, seed, ptr(tw), bare.data_ptr(), ptr(nl), ptr(ws),
                                     ws.numel() if ws is not None else 0, self._stream())
        self._check(rc, 'dqmc_ecp_force')
        return bare, nl

    def zv_force(self, r, R, want_grad_R=False, max_ws_bytes=None):
        """-> (zv[B, M, 3], grad_R[B, M, 3] or None): the zero-variance term of the AC-ZV / AC-ZVZB force estimators,
        zv = -dT/dR_kappa at fixed r (T the local kinetic energy), by a nuclear-coordinate companion of the forward-Laplacian
        pass (dqmc_zv_force; reference force.py:135-169 for an all-electron Hamiltonian); grad_R = grad_R log|psi| from the
        same pass.  Psiformer and FermiNet with multiplicative backflow, all-electron."""
        r = self._prep(r)
        B = r.shape[0]
        R, Rb = self._R(R, B)
        mk = lambda *s: torch.empty(*s, dtype=self.dtype, device=self.device)
        M = self.spec.n_nuc
        zv = mk(B, M, 3)
        gR = mk(B, M, 3) if want_grad_R else None
        ws = self.workspace(B, MODE_ZV_FORCE, max_ws_bytes)
        rc = self.lib.dqmc_zv_force(self.h, r.data_ptr(), R.data_ptr(), Rb, B, zv.data_ptr(),
                                    gR.data_ptr() if gR is not None else None, ws.data_ptr(), ws.numel(), self._stream())
        self._check(rc, 'dqmc_zv_force')
        return zv, gR

    def mcmc_sweep(self, state, R, n_sub, target_acceptance=0.57, max_age=None, seed=0, step0=0, walker_offset=0,
                   noise_normal=None, noise_uniform=None, max_ws_bytes=None, exchange_probability=0.0, exchange_flags=None,
                   exchange_idx=None):
        """state: dict(r[B,N,3], sign[B], log[B], age[B] int32, tau[1]) -- updated IN PLACE.
        exchange_probability > 0 (or injected ``exchange_flags[n_sub]`` / ``exchange_idx[n_sub, B, 2]``): spin-exchange
        sub-steps mixed in (dqmc_mcmc_sweep_exchange; reference OppositeSpinExchangeSampler)."""
        r = state['r']
        B = r.shape[0]
        for k in ('r', 'sign', 'log', 'tau'):
            assert state[k].dtype == self.dtype and state[k].is_contiguous() and state[k].device == self.device, k
        assert state['age'].dtype == torch.int32
        R, Rb = self._R(R, B)
        nn = self._prep(noise_normal) if noise_normal is not None else None
        nu = self._prep(noise_uniform) if noise_uniform is not None else None
        stats = torch.zeros(7, dtype=self.dtype, device=self.device)
        ws = self.workspace(B, MODE_MCMC, max_ws_bytes)  # proposal buffers + the plain-forward chunk
        if exchange_probability > 0.0 or exchange_flags is not None:
            flags = None
            if exchange_flags is not None:
                flags = (C.c_int32 * n_sub)(*[int(f) for f in exchange_flags])
            xi = None
            if exchange_idx is not None:
                xi = exchange_idx.to(device=self.device, dtype=torch.int32).contiguous()
                assert xi.shape == (n_sub, B, 2)
            rc = self.lib.dqmc_mcmc_sweep_exchange(
                self.h, r.data_ptr(), state['sign'].data_ptr(), state['log'].data_ptr(), state['age'].data_ptr(),
                state['tau'].data_ptr(), R.data_ptr(), Rb, B, n_sub, float(target_acceptance if target_acceptance else 0.0),
                -1 if max_age is None else int(max_age), seed, step0, walker_offset,
                nn.data_ptr() if nn is not None else None, nu.data_ptr() if nu is not None else None,
                float(exchange_probability), flags, xi.data_ptr() if xi is not None else None,
                stats.data_ptr(), ws.data_ptr(), ws.numel(), self._stream())
            self._check(rc, 'dqmc_mcmc_sweep_exchange')
            return stats
        rc = self.lib.dqmc_mcmc_sweep(
            self.h, r.data_ptr(), state['sign'].data_ptr(), state['log'].data_ptr(), state['age'].data_ptr(),
            state['tau'].data_ptr(), R.data_ptr(), Rb, B, n_sub, float(target_acceptance if target_acceptance else 0.0),
            -1 if max_age is None else int(max_age), seed, step0, walker_offset,
            nn.data_ptr() if nn is not None else None, nu.data_ptr() if nu is not None else None,
            stats.data_ptr(), ws.data_ptr(), ws.numel(), self._stream())
        self._check(rc, 'dqmc_mcmc_sweep')
        return stats

    def langevin_sweep(self, state, R, n_sub, target_acceptance=0.57, max_age=None, seed=0, step0=0, walker_offset=0,
                       noise_normal=None, noise_uniform=None):
        """state: dict(r[B,N,3], sign[B], log[B], force[B,N,3], age[B] int32, tau[1]) -- updated IN PLACE.
        n_sub = 0: recompute sign / log / force of the current walkers (sampler update)."""
        r = state['r']
        B, N = r.shape[0], r.shape[1]
        for k in ('r', 'sign', 'log', 'force', 'tau'):
            assert state[k].dtype == self.dtype and state[k].is_contiguous() and state[k].device == self.device, k
        assert state['age'].dtype == torch.int32
        R, Rb = self._R(R, B)
        nn = self._prep(noise_normal) if noise_normal is not None else None
        nu = self._prep(noise_uniform) if noise_uniform is not None else None
        stats = torch.zeros(7, dtype=self.dtype, device=self.device)
        ws = self.workspace(B, MODE_LANGEVIN)  # proposal / force buffers + the forward-Laplacian chunk
        rc = self.lib.dqmc_langevin_sweep(
            self.h, r.data_ptr(), state['sign'].data_ptr(), state['log'].data_ptr(), state['force'].data_ptr(),
            state['age'].data_ptr(), state['tau'].data_ptr(), R.data_ptr(), Rb, B, n_sub,
            float(target_acceptance if target_acceptance else 0.0), -1 if max_age is None else int(max_age), seed, step0,
            walker_offset, nn.data_ptr() if nn is not None else None, nu.data_ptr() if nu is not None else None,
            stats.data_ptr(), ws.data_ptr(), ws.numel(), self._stream())
        self._check(rc, 'dqmc_langevin_sweep')
        return stats

    def debug_gemm(self, weight, A, bias=None, Res=None, S=1, sliced=False, backend=0):
        off, K, Nc = self.entries[weight]
        A = self._prep(A)
        rows = A.shape[0]
        out_rows = rows
        Cout = torch.zeros(out_rows, Nc, dtype=self.dtype, device=self.device)
        Res = self._prep(Res) if Res is not None else None
        rc = self.lib.dqmc_debug_gemm(self.h, weight.encode(), bias.encode() if bias else None, A.data_ptr(),
                                      Res.data_ptr() if Res is not None else None, Cout.data_ptr(),
                                      rows // self.spec.n_elec if sliced else rows, S, int(sliced),
                                      backend, self._stream())
        self._check(rc, 'dqmc_debug_gemm')
        return Cout

    def stats_pack(self, E, stats=None):
        """-> float64[11] on the device: sum E, sum E^2, B, sums of the six stats rows, max E, -min E (one launch)."""
        out = torch.empty(11, dtype=torch.float64, device=self.device)
        assert E.dtype == self.dtype and E.is_contiguous() and (stats is None or (stats.is_contiguous() and stats.shape == (6, E.shape[0])))
        rc = self.lib.dqmc_stats_pack(self.h, E.data_ptr(), stats.data_ptr() if stats is not None else None, E.shape[0],
                                      out.data_ptr(), self._stream())
        self._check(rc, 'dqmc_stats_pack')
        return out

    def debug_plan(self, n_walkers: int, mode: int, workspace_bytes: int = 0):
        """-> (planned, carved): dqmc_workspace_bytes and the highest offset the entry point of ``mode`` carves when given
        ``workspace_bytes`` (0: the planned size); host-only."""
        pl, cv = C.c_int64(), C.c_int64()
        rc = self.lib.dqmc_debug_plan(self.h, n_walkers, mode, workspace_bytes, C.byref(pl), C.byref(cv))
        self._check(rc, 'dqmc_debug_plan')
        return pl.value, cv.value

    def workspace_bytes(self, n_walkers: int, mode: int) -> int:
        return self.lib.dqmc_workspace_bytes(self.h, n_walkers, mode)

    def workspace_bytes_min(self, n_walkers: int, mode: int) -> int:
        return self.lib.dqmc_workspace_bytes_min(self.h, n_walkers, mode)

    def debug_mlp_block(self, layer, O, X):
        """One launch of the fused plain-forward MLP block of `layer` -> X' [rows, d] (self-test hook)."""
        O, X = self._prep(O), self._prep(X)
        out = torch.empty_like(O)
        rc = self.lib.dqmc_debug_mlp_block(self.h, layer, O.data_ptr(), X.data_ptr(), out.data_ptr(), O.shape[0], self._stream())
        self._check(rc, 'dqmc_debug_mlp_block')
        return out

    def debug_trunk(self, X0):
        """One launch of the whole-trunk kernel: all attention layers applied to the embedding rows -> [rows, d] (self-test hook)."""
        X0 = self._prep(X0)
        assert X0.dim() == 2 and X0.shape[1] == self.spec.embedding_dim and X0.shape[0] % self.spec.n_elec == 0, tuple(X0.shape)
        out = torch.empty_like(X0)
        rc = self.lib.dqmc_debug_trunk(self.h, X0.data_ptr(), out.data_ptr(), X0.shape[0], self._stream())
        self._check(rc, 'dqmc_debug_trunk')
        return out

    ATTN_KERNELS = ('attn_fwd_mma_kernel', 'attn_fl_f32_kernel', 'attn_fl_kernel', 'attn_fl_f32_kernel_mma', 'attn_fl_kernel_mma')

    def debug_attention(self, layer, QKV, S=1):
        """The softmax attention of `layer` (the kernel the engine picks) on Q | K | V rows [rows, 3d] with S slots per electron
        (1: plain forward; 3N + 2: value, 3N tangents, Laplacian; row (b N + i) S + s) -> (O [rows, d], name of the kernel that
        ran); the TransPsiformer's nuclear tokens come from the parameter table (self-test hook)."""
        QKV = self._prep(QKV)
        d = self.spec.embedding_dim
        assert QKV.dim() == 2 and QKV.shape[1] == 3 * d and QKV.shape[0] % (self.spec.n_elec * S) == 0, tuple(QKV.shape)
        out = torch.empty(QKV.shape[0], d, dtype=self.dtype, device=self.device)
        kernel = C.c_int32(-1)
        rc = self.lib.dqmc_debug_attention(self.h, layer, QKV.data_ptr(), out.data_ptr(), QKV.shape[0], S, C.byref(kernel),
                                           self._stream())
        self._check(rc, 'dqmc_debug_attention')
        return out, self.ATTN_KERNELS[kernel.value]

    MLP_PATHS = ('mlp_block', 'gemm_fused_tanh', 'gemm_tanh_fl_kernel', 'simt_gemm_tanh_fl_kernel')

    def debug_mlp(self, layer, O, X, S=1):
        """What follows the attention of `layer` on slot rows O, X [rows, d] (layout of debug_attention):
        Out = A + tanh(tanh(A W1 + b1) W2 + b2), A = X + O Wo, with forward-Laplacian propagation for S > 1
        -> (Out [rows, d], name of the path that ran) (self-test hook)."""
        O, X = self._prep(O), self._prep(X)
        d = self.spec.embedding_dim
        assert O.shape == X.shape and O.dim() == 2 and O.shape[1] == d and O.shape[0] % (self.spec.n_elec * S) == 0, tuple(O.shape)
        out = torch.empty_like(O)
        scratch = torch.empty(2 * O.shape[0], d, dtype=self.dtype, device=self.device)
        path = C.c_int32(-1)
        rc = self.lib.dqmc_debug_mlp(self.h, layer, S, O.data_ptr(), X.data_ptr(), out.data_ptr(), scratch.data_ptr(), O.shape[0],
                                     C.byref(path), self._stream())
        self._check(rc, 'dqmc_debug_mlp')
        return out, self.MLP_PATHS[path.value]

    SLATER_KERNELS = ('slater_small_kernel', 'slater_fwd2_kernel', 'slater_fwd_reg_kernel', 'slater_kernel')

    def _nuclei(self):
        return self._prep(self.hamil.mol.coords)

    def debug_slater(self, r, BF, S=1):
        """The engine's Slater determinants (backflow activation + the determinant kernel it picks) on walker positions
        r [B, N, 3] and pre-activation backflow head rows BF [B N S, BFW] (row (b N + i) S + s; BFW = K N, 2 K N for
        backflow_transform 'both'), the nuclei of the Hamiltonian -> (det_sign [B, K], det_log [B, K], det_grad [B, K, 3N] or
        None, det_lap [B, K] or None, kernel name with its template instance, e.g. 'slater_fwd2_kernel<30>').  BF is not
        changed (self-test hook)."""
        r, BF = self._prep(r), self._prep(BF)
        N, K = self.spec.n_elec, self.spec.n_determinants
        B = r.shape[0]
        assert r.shape == (B, N, 3) and BF.dim() == 2 and BF.shape[0] == B * N * S, (tuple(r.shape), tuple(BF.shape))
        mk = lambda *s: torch.empty(*s, dtype=self.dtype, device=self.device)
        sign, log = mk(B, K), mk(B, K)
        grad, lap = (mk(B, K, 3 * N), mk(B, K)) if S > 1 else (None, None)
        kernel = (C.c_int32 * 2)(-1, -1)
        ptr = lambda t: t.data_ptr() if t is not None else None
        R = self._nuclei()  # held until the call returns
        rc = self.lib.dqmc_debug_slater(self.h, r.data_ptr(), R.data_ptr(), BF.data_ptr(), BF.shape[0], S,
                                        sign.data_ptr(), log.data_ptr(), ptr(grad), ptr(lap), kernel, self._stream())
        self._check(rc, 'dqmc_debug_slater')
        name = self.SLATER_KERNELS[kernel[0]] + (f'<{kernel[1]}>' if kernel[1] else '')
        return sign, log, grad, lap, name

    def debug_det_sum(self, r, det_sign, det_log, det_grad=None, det_lap=None):
        """The engine's determinant sum (finalize_kernel; no Jastrow, no pseudo-Hamiltonian) on det_sign / det_log [B, K] and,
        for the forward-Laplacian pass, det_grad [B, K, 3N] / det_lap [B, K] -> (sign [B], log|psi| [B], grad log|psi|
        [B, 3N] or None, stats [6, B] or None: stats[4] = lap log|psi|, stats[5] = |grad log|psi||^2) (self-test hook)."""
        r, det_sign, det_log = self._prep(r), self._prep(det_sign), self._prep(det_log)
        N = self.spec.n_elec
        B = r.shape[0]
        S = 3 * N + 2 if det_grad is not None else 1
        mk = lambda *s: torch.empty(*s, dtype=self.dtype, device=self.device)
        sign, log = mk(B), mk(B)
        grad, stats = (mk(B, 3 * N), mk(6, B)) if S > 1 else (None, None)
        ptr = lambda t: t.data_ptr() if t is not None else None
        dg = self._prep(det_grad) if det_grad is not None else None
        dl = self._prep(det_lap) if det_lap is not None else None
        R = self._nuclei()
        rc = self.lib.dqmc_debug_det_sum(self.h, r.data_ptr(), R.data_ptr(), det_sign.data_ptr(),
                                         det_log.data_ptr(), ptr(dg), ptr(dl), B, S, sign.data_ptr(), log.data_ptr(),
                                         ptr(grad), ptr(stats), self._stream())
        self._check(rc, 'dqmc_debug_det_sum')
        return sign, log, grad, stats

    def debug_attention_bwd(self, layer, QKV, dO):
        """The softmax attention backward of `layer` (Engine::attention_bwd, the kernel the reverse passes run) on Q | K | V rows
        [rows, 3d] and output cotangents dO [rows, d] (row b N + i) -> (dQKV [rows, 3d], dKn [Mn, d], dVn [Mn, d]): the last two
        are the TransPsiformer nuclear tokens' cotangents summed over the walkers, None without nuclear tokens (self-test hook)."""
        QKV, dO = self._prep(QKV), self._prep(dO)
        d = self.spec.embedding_dim
        assert QKV.dim() == 2 and QKV.shape[1] == 3 * d and dO.shape == (QKV.shape[0], d), (tuple(QKV.shape), tuple(dO.shape))
        dQKV = torch.empty_like(QKV)
        Mn = self.spec.n_nuc if self.spec.kind == 'transpsiformer' else 0
        dKn = torch.zeros(Mn, d, dtype=self.dtype, device=self.device) if Mn else None
        dVn = torch.zeros(Mn, d, dtype=self.dtype, device=self.device) if Mn else None
        ptr = lambda t: t.data_ptr() if t is not None else None
        rc = self.lib.dqmc_debug_attention_bwd(self.h, layer, QKV.data_ptr(), dO.data_ptr(), dQKV.data_ptr(), ptr(dKn), ptr(dVn),
                                               QKV.shape[0], self._stream())
        self._check(rc, 'dqmc_debug_attention_bwd')
        return dQKV, dKn, dVn

    def debug_wgrad(self, A, dY, lo=0, hi=-1):
        """The reverse passes' weight- and bias-gradient reductions on A [rows, K] and dY [rows, Nc] -> (dW [K, Nc] = A^T dY,
        db [Nc] = column sums of dY), both over the rows b N + i with lo <= i < hi (hi = -1: every row) (self-test hook)."""
        A, dY = self._prep(A), self._prep(dY)
        assert A.dim() == 2 and dY.dim() == 2 and A.shape[0] == dY.shape[0], (tuple(A.shape), tuple(dY.shape))
        dW = torch.zeros(A.shape[1], dY.shape[1], dtype=self.dtype, device=self.device)
        db = torch.zeros(dY.shape[1], dtype=self.dtype, device=self.device)
        rc = self.lib.dqmc_debug_wgrad(self.h, A.data_ptr(), dY.data_ptr(), A.shape[0], A.shape[1], dY.shape[1], lo, hi,
                                       dW.data_ptr(), db.data_ptr(), self._stream())
        self._check(rc, 'dqmc_debug_wgrad')
        return dW, db

    TRUNK_PHASES = ('tile_load', 'qkv_mainloop', 'qkv_epilogue', 'attention', 'wo_mainloop', 'wo_epilogue', 'w1_mainloop',
                    'w1_epilogue', 'w2_mainloop', 'w2_epilogue', 'weight_wait', 'mma_turn', 'tile_layer_pairs')

    def debug_trunk_phases(self):
        """{phase: cycles} of the whole-trunk kernel's timers (engine created with DQMC_TRUNK_PHASES=1) since the last call;
        'tile_layer_pairs' is a count.  Resets the counters."""
        out = (C.c_uint64 * len(self.TRUNK_PHASES))()
        rc = self.lib.dqmc_debug_trunk_phases(self.h, out, len(out))
        self._check(rc, 'dqmc_debug_trunk_phases')
        return dict(zip(self.TRUNK_PHASES, out))

    def debug_tc_error(self):
        """The error word of the whole-trunk and fused MLP-block kernels since creation or the last call (0: none), then reset;
        synchronous."""
        flag = C.c_int32()
        self._check(self.lib.dqmc_debug_tc_error(self.h, C.byref(flag)), 'dqmc_debug_tc_error')
        return flag.value

    def profile_begin(self):
        self.lib.dqmc_profile_begin(self.h)

    def profile_end(self):
        ms, fl, n = C.c_double(), C.c_double(), C.c_int64()
        self.lib.dqmc_profile_end(self.h, C.byref(ms), C.byref(fl), C.byref(n))
        return ms.value, fl.value, n.value

    PROFILE_CLASSES = ('row_gemm', 'mlp_block', 'trunk')

    def profile_end_classes(self):
        """{class: (ms, algorithmic flops, launches)} for the three tensor-core kernel classes."""
        ms, fl, n = (C.c_double * 3)(), (C.c_double * 3)(), (C.c_int64 * 3)()
        self.lib.dqmc_profile_end_classes(self.h, ms, fl, n)
        return {k: (ms[i], fl[i], n[i]) for i, k in enumerate(self.PROFILE_CLASSES)}

    @property
    def launch_count(self):
        return self.lib.dqmc_launch_count(self.h)

    @property
    def ecp_forward_count(self):
        """Non-local ECP quadrature forwards run so far (12 per electron-nucleus pair inside the cutoff radius)."""
        return self.lib.dqmc_ecp_forward_count(self.h)

    def close(self):
        if getattr(self, 'h', None):
            self.lib.dqmc_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
