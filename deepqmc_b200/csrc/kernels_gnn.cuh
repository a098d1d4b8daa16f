// Convolution-GNN trunk of the reference's "PauliNet"-type ansatz (tests/conf/ansatz.yaml =
// BASELINE configs[0]; reference src/deepqmc/gnn/electron_gnn.py:160-259, gnn/update_features.py:
// 162-238, gnn/graph.py:226-335) with forward-Laplacian propagation on the augmented-row layout
// of kernels_trunk.cuh (slot 0 value, 1+t = d/dx_t, T+1 = Laplacian).
#pragma once
#include "common.cuh"

namespace dq {

// ------------------------------------------------------------------------------------------
// Embedding lookup: x_i = Embed[type(i)] (reference gnn/electron_gnn.py:620-624; one electron type
// when n_up == n_down, otherwise spin-down electrons are type 1, :337-343).  Constant in r: all
// derivative slots are zero.  One thread per (walker-electron, feature).
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void gnn_embed_kernel(const T* __restrict__ emb, int n_types, int N, int n_up, int S, int d,
                                 T* __restrict__ X, int total) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total * d) return;
  const int bi = idx / d, f = idx - bi * d;
  const int i = bi % N;
  const int type = (n_types > 1 && i >= n_up) ? 1 : 0;
  T* x = X + (size_t)bi * S * d + f;
  x[0] = emb[type * d + f];
  for (int s = 1; s < S; ++s) x[(size_t)s * d] = T(0);
}

// ------------------------------------------------------------------------------------------
// Raw edge features [|d|, d],  d = r_i - p_j (receiver - sender, graph.py:24; eps-safe norm,
// edge_features.py:42-78), sender = electron j != i (same / anti edges) or nucleus (ne edges).  An edge
// depends on r_i and r_j only, so its forward-Laplacian state is COMPACT:
//   slot 0 value | 1..3 d/dr_i | 4..6 d/dr_j (zero for nuclei) | 7 Laplacian over both particles.
// Layout E[b][i][jj][8][4], jj < N: electron sender, jj >= N: nucleus jj - N.  The (i, i) row is zero, or with
// self_edges (self_interaction, graph.py:226-335) the edge r_i - r_i: |d| = sqrt(eps) (eps-safe norm of a zero vector,
// utils.py:79-85), d = 0 and no derivative at all, since the difference vanishes identically.  The edge MLPs
// (w_t, u) run on these rows with the ordinary row GEMM and act_fl_kernel with S = 8 (slots 1..6 are the
// tangents, slot 7 the Laplacian).  One thread per (b, i, jj).
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void gnn_edge_feat_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M,
                                     int Mne, T* __restrict__ E, int total,
                                     const T* __restrict__ QA /*pseudo-Hamiltonian metric or null*/, int self_edges) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int NS = N + Mne;
  const int jj = idx % NS, i = (idx / NS) % N, b = idx / (NS * N);
  T* out = E + (size_t)idx * 32;
  for (int k = 0; k < 32; ++k) out[k] = T(0);
  if (jj == i) {
    if (self_edges) out[0] = m_sqrt(Num<T>::eps());
    return;
  }
  const T* ri = r + ((size_t)b * N + i) * 3;
  const bool nuc = jj >= N;
  const T* pj = nuc ? R + (R_batched ? (size_t)b * M * 3 : 0) + (size_t)(jj - N) * 3 : r + ((size_t)b * N + jj) * 3;
  const T d[3] = {ri[0] - pj[0], ri[1] - pj[1], ri[2] - pj[2]};
  const T dd = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
  const T rho2 = Num<T>::eps() + dd, rho = m_sqrt(rho2);
  const T sj = nuc ? T(0) : T(-1), np = nuc ? T(1) : T(2);
  out[0] = rho; out[1] = d[0]; out[2] = d[1]; out[3] = d[2];
  for (int c = 0; c < 3; ++c) {
    T* gi = out + (1 + c) * 4;  // d / d r_i,c
    gi[0] = d[c] / rho; gi[1 + c] = T(1);
    T* gj = out + (4 + c) * 4;  // d / d r_j,c
    gj[0] = sj * d[c] / rho; gj[1 + c] = sj;
  }
  out[7 * 4] = np * (T(3) / rho - dd / (rho2 * rho));
  if (QA) {
    // pseudo-Hamiltonian: tangents w.r.t. v_n = Q_n^-1 r_n (columns of Q_n), second derivatives weighted by A_n
    PhMetric<T> pm;
    const T u0 = d[0] / rho, u1 = d[1] / rho, u2 = d[2] / rho;
    T lap = T(0);
    for (int side = 0; side < (nuc ? 1 : 2); ++side) {
      pm.load(QA + ((size_t)b * N + (side == 0 ? i : jj)) * PH_STRIDE);
      const T sg = side == 0 ? T(1) : T(-1);
      const T qc[3][3] = {{pm.q[0], pm.q[1], pm.q[3]}, {T(0), pm.q[2], pm.q[4]}, {T(0), T(0), pm.q[5]}};  // column c of Q
      for (int c = 0; c < 3; ++c) {
        T* g = out + (1 + 3 * side + c) * 4;
        g[0] = sg * (u0 * qc[c][0] + u1 * qc[c][1] + u2 * qc[c][2]);
        g[1] = sg * qc[c][0]; g[2] = sg * qc[c][1]; g[3] = sg * qc[c][2];
      }
      T a0, a1, a2;
      pm.mul(u0, u1, u2, a0, a1, a2);
      lap += (pm.trace() - (u0 * a0 + u1 * a1 + u2 * a2)) / rho;
    }
    out[7 * 4] = lap;
  }
}

// Node-update input of the 'concatenate' rule (reference gnn/update_features.py:47-121 Residual / NodeSum with
// normalize = true, then the convolutions): F[b][i][s][:] = [x_i, mean_up x, mean_down x, conv_*(i)].  Linear, so it
// acts slot-wise.  grid = (B * S, N), block over features.
template <class T>
__global__ void gnn_concat_kernel(const T* __restrict__ X, int dx, const T* __restrict__ C, int dc, int N, int n_up,
                                  int S, T* __restrict__ F) {
  const int bs = blockIdx.x, b = bs / S, s = bs % S, i = blockIdx.y;
  const int ldf = 3 * dx + dc;
  T* f = F + ((size_t)(b * N + i) * S + s) * ldf;
  const int n_dn = N - n_up;
  for (int k = threadIdx.x; k < ldf; k += blockDim.x) {
    T v;
    if (k < dx) {
      v = X[((size_t)(b * N + i) * S + s) * dx + k];
    } else if (k < 3 * dx) {
      const bool up = k < 2 * dx;
      const int kk = up ? k - dx : k - 2 * dx;
      const int j0 = up ? 0 : n_up, j1 = up ? n_up : N;
      T acc = T(0);
      for (int j = j0; j < j1; ++j) acc += X[((size_t)(b * N + j) * S + s) * dx + kk];
      v = acc / (T)(up ? n_up : n_dn);
    } else {
      v = C[((size_t)(b * N + i) * S + s) * dc + (k - 3 * dx)];
    }
    f[k] = v;
  }
}

// ------------------------------------------------------------------------------------------
// Convolution  conv_t(i) = sum_{senders j of type t} w_t(e_ji) * h_t(x_j)  (update_features.py:
// 196-211; no normalisation) with the product rule on the augmented rows:
//   value   sum_j w h
//   d_t     sum_j (d_t w) h + w d_t h           (d_t w != 0 only for t in electron i or j)
//   Lap     sum_j (Lap w) h + w Lap h + 2 sum_{t in i, j} d_t w d_t h
// Hs / Ha: h_same(x_j) / h_anti(x_j) augmented rows [b][j][s][e]; Hne[M][ene]: h_ne of the (constant)
// nuclear embeddings.  Block per (b, i).
// Wsame / Wanti: the filters of the electron edge types evaluated on ALL (i, jj) pairs (compact layout, M = number of
// nuclear senders in it, 0 without 'ne' edges, row stride e); the kernel reads the one matching the pair.  Wne: the ne
// filter rows of the same layout with row stride ldne and width ene -- the w_ne output (ene = e), or with w_for_ne =
// false the ne edge stream itself (update_features.py:199-210).  self_edges: the same-spin sum includes j = i; that
// filter row carries no derivative (gnn_edge_feat_kernel), so the product rule counts the receiver's tangent once.
// C[b][i][s][:] = [conv_same | conv_anti | conv_ne], or with ee_sum [conv_same + conv_anti | conv_ne] (the 'ee' edge
// type, update_features.py:218-224).
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void gnn_conv_kernel(const T* __restrict__ Wsame, const T* __restrict__ Wanti, const T* __restrict__ Wne,
                                int ldne, int ene, const T* __restrict__ Hs, const T* __restrict__ Ha,
                                const T* __restrict__ Hne, int N, int M, int n_up, int S, int e, int ee_sum, int self_edges,
                                T* __restrict__ C) {
  const int bi = blockIdx.x, b = bi / N, i = bi - b * N;
  const int NS = N + M, T3 = S > 1 ? S - 2 : 0;
  const int ee_w = ee_sum ? e : 2 * e, dc = ee_w + (M > 0 ? ene : 0);
  const size_t wbase = (size_t)bi * NS * 8 * e;
  for (int idx = threadIdx.x; idx < S * dc; idx += blockDim.x) {
    const int s = idx / dc, k = idx - s * dc;
    const int t = s - 1;             // tangent index for 1 <= s <= T3
    const int te = t / 3, tc = t - 3 * te;
    T acc = T(0);
    if (k < ee_w) {
      const int grp = ee_sum ? -1 : (k >= e ? 1 : 0), f = k >= e ? k - e : k;  // grp 0: same only, 1: anti only
      for (int j = 0; j < N; ++j) {
        if (j == i && !self_edges) continue;
        const bool same = (i < n_up) == (j < n_up);
        if ((grp == 0 && !same) || (grp == 1 && same)) continue;
        const T* w = (same ? Wsame : Wanti) + wbase + (size_t)j * 8 * e + f;
        const T* h = (same ? Hs : Ha) + ((size_t)(b * N + j) * S) * e + f;
        T v;
        if (s == 0) {
          v = w[0] * h[0];
        } else if (s <= T3) {
          v = w[0] * h[(size_t)s * e];
          if (te == i) v += w[(1 + tc) * e] * h[0];
          else if (te == j) v += w[(4 + tc) * e] * h[0];
        } else {
          v = w[7 * e] * h[0] + w[0] * h[(size_t)s * e];
          T cr = T(0);
          for (int c = 0; c < 3; ++c)
            cr += w[(1 + c) * e] * h[(size_t)(1 + 3 * i + c) * e] + w[(4 + c) * e] * h[(size_t)(1 + 3 * j + c) * e];
          v += T(2) * cr;
        }
        acc += v;
      }
    } else {
      const int f = k - ee_w;
      for (int m = 0; m < M; ++m) {
        const T* w = Wne + ((size_t)bi * NS + N + m) * 8 * ldne + f;
        const T h0 = Hne[m * ene + f];
        if (s == 0) acc += w[0] * h0;
        else if (s <= T3) { if (te == i) acc += w[(1 + tc) * ldne] * h0; }
        else acc += w[7 * ldne] * h0;
      }
    }
    C[((size_t)bi * S + s) * dc + k] = acc;
  }
}

// Deep edge update with one u MLP per edge type (deep_features 'separate', electron_gnn.py:176-188): the MLPs ran on
// every pair into U0 / U1 / U2; each pair keeps its own type's output, with the normalised residual
// (e + u(e)) / sqrt 2 for the types whose width did not change (bit t of res_mask; hkext.py:116-137).  E / Eo: rows
// [pairs][slots][e] (slots = 8: compact forward-Laplacian rows, 1: values).  One thread per element.
template <class T>
__global__ void gnn_edge_select_kernel(const T* __restrict__ E, const T* __restrict__ U0, const T* __restrict__ U1,
                                       const T* __restrict__ U2, int slots, int N, int M, int n_up, int e, int res_mask,
                                       T scale, T* __restrict__ Eo, size_t n) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const int NS = N + M;
  const size_t pair = idx / ((size_t)slots * e);
  const int jj = (int)(pair % NS), i = (int)((pair / NS) % N);
  const int t = jj >= N ? 2 : (((i < n_up) == (jj < n_up)) ? 0 : 1);
  const T u = (t == 0 ? U0 : t == 1 ? U1 : U2)[idx];
  Eo[idx] = ((res_mask >> t) & 1) ? scale * (E[idx] + u) : u;
}

// ------------------------------------------------------------------------------------------
// Elementwise activation with forward-Laplacian propagation, in place on groups of S rows:
//   y = f(z); y_t = f'(z) z_t; y_L = f'(z) z_L + f''(z) sum_t z_t^2; out = out_scale (Res + y).
// act 0: tanh; 1: ssp = softplus + log(1/2) (reference hkext.py:11-19); 2: the default mult_act of the
// backflow 1 + 2 tanh(z / 4) (wf/nn_wave_function.py:17); 3: its default add_act 0.1 tanh(z / 4) (:18).
// grid = (groups, ceil(d / blockDim)).
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void act_fl_kernel(T* __restrict__ Z, int ldz, const T* __restrict__ Res, int ldr, int S, int d,
                              T out_scale, int act) {
  const int g = blockIdx.x;
  const int f = blockIdx.y * blockDim.x + threadIdx.x;
  if (f >= d) return;
  T* z = Z + (size_t)g * S * ldz + f;
  const T* rs = Res ? Res + (size_t)g * S * ldr + f : nullptr;
  const T z0 = z[0];
  T y, y1, y2;
  if (act == 0) {
    y = m_tanh(z0); y1 = T(1) - y * y; y2 = T(-2) * y * y1;
  } else if (act == 1) {
    const T sg = T(1) / (T(1) + m_exp(-z0));
    y = (z0 > T(0) ? z0 + m_log1p(m_exp(-z0)) : m_log1p(m_exp(z0))) - T(0.6931471805599453094);
    y1 = sg; y2 = sg * (T(1) - sg);
  } else if (act == 2) {
    const T th = m_tanh(z0 * T(0.25)), sc = T(1) - th * th;
    y = T(1) + T(2) * th; y1 = T(0.5) * sc; y2 = T(-0.25) * th * sc;
  } else {  // 3: the default add_act of the backflow 0.1 tanh(z / 4) (wf/nn_wave_function.py:18)
    const T th = m_tanh(z0 * T(0.25)), sc = T(1) - th * th;
    y = T(0.1) * th; y1 = T(0.025) * sc; y2 = T(-0.0125) * th * sc;
  }
  z[0] = out_scale * ((rs ? rs[0] : T(0)) + y);
  if (S > 1) {
    const int T3 = S - 2;
    T ss = T(0);
    for (int t = 1; t <= T3; ++t) {
      T zt = z[(size_t)t * ldz];
      ss += zt * zt;
      z[(size_t)t * ldz] = out_scale * ((rs ? rs[(size_t)t * ldr] : T(0)) + y1 * zt);
    }
    T zl = z[(size_t)(T3 + 1) * ldz];
    z[(size_t)(T3 + 1) * ldz] = out_scale * ((rs ? rs[(size_t)(T3 + 1) * ldr] : T(0)) + y1 * zl + y2 * ss);
  }
}

// out = scale * (a + b), elementwise (normalised residual of the edge stream)
template <class T>
__global__ void axpby_kernel(const T* __restrict__ a, const T* __restrict__ b, T scale, T* __restrict__ out, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = scale * (a[i] + b[i]);
}

// Sum over the electrons of a walker, slot-wise (Jastrow with sum_first, wf/omni.py:35-37):
// Y[b][s][f] = sum_i X[b][i][s][f].  One thread per (b, s, f).
template <class T>
__global__ void sum_electrons_kernel(const T* __restrict__ X, int N, int S, int d, T* __restrict__ Y, int total) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int f = idx % d, s = (idx / d) % S, b = idx / (d * S);
  T a = T(0);
  for (int i = 0; i < N; ++i) a += X[(((size_t)b * N + i) * S + s) * d + f];
  Y[idx] = a;
}

}  // namespace dq
