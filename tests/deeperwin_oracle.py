"""fp64 torch restatement of the reference's DeepErwin ansatz (src/deepqmc/conf/ansatz/deeperwin.yaml) for one walker.

Test infrastructure: functional and differentiable, independent of deepqmc_b200 (it reads the Haiku parameter names of
oracle/names.py and reuses the envelope x backflow orbitals of oracle/wf.py).  Follows
  gnn/electron_gnn.py:596-625   ElectronEmbedding: raw [|r_i - R_I|, r_i - R_I] for all nuclei, no spin, no projection
  gnn/electron_gnn.py:435-537   NucleiEmbedding: hk.Embed over atom types (jnp.unique(..., return_inverse=True))
  gnn/graph.py:226-335          edges receiver - sender; self_interaction keeps the (i, i) same-spin edge
  gnn/edge_features.py:21-78    |d| (eps-safe, utils.py:79-85) on same / anti, [|d|, d] on ne
  gnn/update_features.py:47-238 [x, mean_up x, mean_down x, conv_ee, conv_ne]; conv_ee = conv_same + conv_anti
                                (:218-224); w_for_ne = false: the ne edge stream is the filter and h_ne is as wide (:199-211)
  gnn/electron_gnn.py:160-259   deep_features 'separate' (u<type>), update 'concatenate', electron_residual false
  hkext.py:116-137              ResidualConnection(normalize=True): (e + u(e)) / sqrt 2 if the shapes match, else u(e)
  wf/env.py:55-70               exponent softplus(zeta) |d|
  wf/nn_wave_function.py:127-173 full determinants, identity mult_act, SumPool, no cusp
"""
from __future__ import annotations

import math

import torch

from oracle import names as P
from oracle import wf
from oracle.hamil import safe_norm

EDGE_TYPES = ('same', 'anti', 'ne')


def graph_edges(nodes_send, nodes_recv):
    """MolecularGraphEdgeBuilder's difference array [sender, receiver, 3] = receiver - sender (gnn/graph.py:23-31),
    self pairs included (self_interaction = true keeps the diagonal)."""
    return nodes_recv[None, :, :] - nodes_send[:, None, :]


def atom_types(charges):
    return torch.unique(torch.as_tensor(charges, dtype=torch.float64), return_inverse=True)[1]


def deeperwin_embeddings(spec, params, r, R, eps=None):
    """eps: the eps of the eps-safe edge norms, finfo(float64).eps by default.  The self edge's |d| is sqrt(eps) itself, so
    a comparison with a float32 evaluation passes finfo(float32).eps (what the reference computes in float32)."""
    N, n_up, L = spec.n_elec, spec.n_up, spec.n_layers
    x, _ = wf.ne_features(r, R, False)  # [N, 4M]
    xn = params[P.GNN + 'nuclei_embedding/~/embed:embeddings'][atom_types(spec.charges)]  # [M, 32]

    def lin(base, h):  # hkext.MLP, hidden_layers ['log', 1], bias, last_linear = false: one Linear + tanh
        return torch.tanh(h @ params[base + 'linear_0:w'] + params[base + 'linear_0:b'])

    up = torch.arange(N) < n_up
    mask = {'same': up[:, None] == up[None, :], 'anti': up[:, None] != up[None, :]}  # [sender j, receiver i]
    d_ee = graph_edges(r, r)
    d_ne = graph_edges(R, r)  # [I, i, 3]
    e = {'same': safe_norm(d_ee, eps)[..., None], 'anti': safe_norm(d_ee, eps)[..., None],
         'ne': torch.cat([safe_norm(d_ne, eps)[..., None], d_ne], -1)}
    sq2 = math.sqrt(2.0)
    for l in range(L):
        c, lp = P.conv_prefix(l), P.layer_prefix(l)
        conv_ee = 0
        for t in ('same', 'anti'):
            prod = lin(c + f'w_{t}/', e[t]) * lin(c + f'h_{t}/', x)[:, None, :]
            conv_ee = conv_ee + (prod * mask[t][:, :, None].to(prod.dtype)).sum(0)
        conv_ne = (e['ne'] * lin(c + 'h_ne/', xn)[:, None, :]).sum(0)
        f = torch.cat([x, x[:n_up].mean(0, keepdim=True).expand(N, -1), x[n_up:].mean(0, keepdim=True).expand(N, -1),
                       conv_ee, conv_ne], -1)
        x = lin(lp + 'g/', f)
        if l < L - 1:
            for t in EDGE_TYPES:
                u = lin(lp + f'u{t}/', e[t])
                e[t] = (e[t] + u) / sq2 if u.shape == e[t].shape else u
    return x


def softplus_envelope_params(params):
    """The reference's exponent softplus(zeta) (wf/env.py:62-66) in the |zeta| form of oracle.wf.orbitals."""
    out = dict(params)
    for s in ('up', 'down'):
        k = f'{P.ENV}:zetas_{s}'
        out[k] = torch.nn.functional.softplus(params[k])
    return out


def log_psi(spec, params, r, R, return_mos=False, eps=None):
    x = deeperwin_embeddings(spec, params, r, R, eps)
    A = wf.orbitals(spec, softplus_envelope_params(params), x, r, R)  # [K, N, N]
    if return_mos:
        return A[:, :spec.n_up], A[:, spec.n_up:]
    sign, ld = torch.linalg.slogdet(A)
    shift = ld.max().detach()
    psi = (sign * torch.exp(ld - shift)).sum()
    return torch.sign(psi).detach(), torch.log(torch.abs(psi)) + shift
