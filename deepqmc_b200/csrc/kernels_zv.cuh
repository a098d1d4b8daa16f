// Nuclear-coordinate companion of the forward-Laplacian pass (dqmc_zv_force): for one Cartesian nuclear coordinate
// kappa = (m, c), every activation X[b][i][s][f] of the forward-Laplacian state gets a companion Xd of the same layout holding
// dX/dR_kappa at fixed electron positions (forward mode in R on top of the forward Laplacian in r).  Linear maps (row GEMMs
// without bias, residual adds, FermiNet's spin means) act on Xd as on X; every nonlinear rule of the pass has its companion
// below: the product and chain rules applied once more to the existing rule.  The output is
//   f_zv = 1/2 (Lap log|psi| + |grad log|psi||^2)_dot = -dT/dR_kappa   (T = local kinetic energy, r fixed)
// and, from the companion of the value slot, g_kappa = d log|psi| / dR_kappa.
//
// Radial functions of d = r_i - R_m are written as functions of u = |d|^2 (rho = sqrt(eps + u)): for g(u),
//   d_c g = 2 d_c g',  d_c d_e g = 2 delta_ce g' + 4 d_c d_e g'',  Lap g = 6 g' + 4 u g'',  d_c Lap g = d_c (20 g'' + 8 u g'''),
// and for d_a s(u):
//   d_c (d_a s) = delta_ac s + 2 d_a d_c s',
//   d_c d_e (d_a s) = 2 s' (delta_ac d_e + delta_ae d_c + delta_ce d_a) + 4 d_a d_c d_e s'',
//   d_c Lap (d_a s) = delta_ac (10 s' + 4 u s'') + d_a d_c (28 s'' + 8 u s''').
// d/dR_m = -d/dr_i on a function of r_i - R_m.
#pragma once
#include "common.cuh"

namespace dq {

// u-derivatives (1st..3rd) of F(rho(u)), rho = sqrt(eps + u), from the rho-derivatives F1..F3
template <class T>
__device__ __forceinline__ void zv_chain_u(T rho, T F1, T F2, T F3, T& g1, T& g2, T& g3) {
  const T r1 = T(0.5) / rho, r2 = T(-0.25) / (rho * rho * rho), r3 = T(0.375) / (rho * rho * rho * rho * rho);
  g1 = F1 * r1;
  g2 = F2 * r1 * r1 + F1 * r2;
  g3 = F3 * r1 * r1 * r1 + T(3) * F2 * r1 * r2 + F1 * r3;
}

// companion of the jet (value, d/dr_i,e, Lap) of a radial function g(u) of d: -(d_c g, d_c d_e g, d_c Lap g)
template <class T>
__device__ __forceinline__ void zv_radial(const T (&dx)[3], T u, int c, T g1, T g2, T g3, T& v, T (&de)[3], T& l) {
  v = T(-2) * dx[c] * g1;
#pragma unroll
  for (int e = 0; e < 3; ++e) de[e] = -((c == e ? T(2) * g1 : T(0)) + T(4) * dx[c] * dx[e] * g2);
  l = -dx[c] * (T(20) * g2 + T(8) * u * g3);
}

// ------------------------------------------------------------------------------------------
// Seed: companion of the electron-nucleus features (embed_kernel: [log1p rho, d log1p(rho) / rho] (log_rescale) or
// FermiNet's raw [rho, d]; the spin column has no companion) and of their projection by W (null: identity, d == F).  Only
// the pairs (i, m) of nucleus m are nonzero.  grid = B N blocks (one electron each), block over the output features.
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void zv_embed_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M, int S,
                                int log_rescale, const T* __restrict__ W, int d, T* __restrict__ Xd, int total, int m, int c) {
  __shared__ T fv[4], fd[3][4], fl[4];
  const int bi = blockIdx.x;
  if (bi >= total) return;
  const int b = bi / N, i = bi % N;
  if (threadIdx.x == 0) {
    const T* ri = r + (size_t)bi * 3;
    const T* Rm = R + (R_batched ? (size_t)b * M * 3 : 0) + 3 * m;
    const T dx[3] = {ri[0] - Rm[0], ri[1] - Rm[1], ri[2] - Rm[2]};
    const T u = dx[0] * dx[0] + dx[1] * dx[1] + dx[2] * dx[2];
    const T rho = m_sqrt(Num<T>::eps() + u);
    T F1, F2, F3, s, S1, S2, S3;
    if (log_rescale) {
      const T F = m_log1p(rho);
      F1 = T(1) / (T(1) + rho); F2 = -F1 * F1; F3 = T(2) * F1 * F1 * F1;
      const T ir = T(1) / rho;
      s = F * ir;
      S1 = F1 * ir - F * ir * ir;
      S2 = F2 * ir - T(2) * F1 * ir * ir + T(2) * F * ir * ir * ir;
      S3 = F3 * ir - T(3) * F2 * ir * ir + T(6) * F1 * ir * ir * ir - T(6) * F * ir * ir * ir * ir;
    } else {
      F1 = T(1); F2 = T(0); F3 = T(0);
      s = T(1); S1 = T(0); S2 = T(0); S3 = T(0);
    }
    T g1, g2, g3, s1, s2, s3;
    zv_chain_u(rho, F1, F2, F3, g1, g2, g3);
    zv_chain_u(rho, S1, S2, S3, s1, s2, s3);
    T de[3];
    zv_radial(dx, u, c, g1, g2, g3, fv[0], de, fl[0]);
    for (int e = 0; e < 3; ++e) fd[e][0] = de[e];
    for (int a = 0; a < 3; ++a) {
      fv[1 + a] = -((a == c ? s : T(0)) + T(2) * dx[a] * dx[c] * s1);
      for (int e = 0; e < 3; ++e)
        fd[e][1 + a] = -(T(2) * s1 * ((a == c ? dx[e] : T(0)) + (a == e ? dx[c] : T(0)) + (c == e ? dx[a] : T(0))) +
                         T(4) * dx[a] * dx[c] * dx[e] * s2);
      fl[1 + a] = -((a == c ? T(10) * s1 + T(4) * u * s2 : T(0)) + dx[a] * dx[c] * (T(28) * s2 + T(8) * u * s3));
    }
  }
  __syncthreads();
  const int T3 = S - 2;
  T* Xg = Xd + (size_t)bi * S * d;
  for (int f = threadIdx.x; f < d; f += blockDim.x) {
    T y0 = 0, y1 = 0, y2 = 0, y3 = 0, yl = 0;
    if (W) {
      for (int a = 0; a < 4; ++a) {
        const T w = W[(size_t)(4 * m + a) * d + f];
        y0 += fv[a] * w; y1 += fd[0][a] * w; y2 += fd[1][a] * w; y3 += fd[2][a] * w; yl += fl[a] * w;
      }
    } else if (f >= 4 * m && f < 4 * m + 4) {
      const int a = f - 4 * m;
      y0 = fv[a]; y1 = fd[0][a]; y2 = fd[1][a]; y3 = fd[2][a]; yl = fl[a];
    }
    Xg[f] = y0;
    for (int t = 0; t < T3; ++t) {
      T v = T(0);
      if (t == 3 * i) v = y1;
      else if (t == 3 * i + 1) v = y2;
      else if (t == 3 * i + 2) v = y3;
      Xg[(size_t)(1 + t) * d + f] = v;
    }
    Xg[(size_t)(1 + T3) * d + f] = yl;
  }
}

// ------------------------------------------------------------------------------------------
// Companion of an elementwise activation y = out_scale (Res + phi(z)) with its forward-Laplacian rule (tanh_fl_kernel: act 0,
// tanh; act_fl_kernel act 2: the BackflowOp's 1 + 2 tanh(z / 4)):
//   yd   = s (Resd + phi' zd)
//   yd_t = s (Resd_t + phi'' zd z_t + phi' zd_t)
//   yd_L = s (Resd_L + phi' zd_L + phi'' (zd z_L + 2 sum_t z_t zd_t) + phi''' zd sum_t z_t^2)
// Z: the primal pre-activation rows (read only; run this before the primal rule overwrites them), Zd: the companion
// pre-activation, replaced by the companion of y.  grid = (groups, ceil(d / blockDim)).
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void zv_act_kernel(const T* __restrict__ Z, int ldz, T* __restrict__ Zd, int ldzd, const T* __restrict__ Resd,
                              int ldr, int S, int d, T out_scale, int act) {
  const int g = blockIdx.x;
  const int f = blockIdx.y * blockDim.x + threadIdx.x;
  if (f >= d) return;
  const T* z = Z + (size_t)g * S * ldz + f;
  T* zd = Zd + (size_t)g * S * ldzd + f;
  const T* rs = Resd ? Resd + (size_t)g * S * ldr + f : nullptr;
  T y1, y2, y3;
  if (act == 0) {
    const T y = m_tanh(z[0]);
    y1 = T(1) - y * y; y2 = T(-2) * y * y1; y3 = T(-2) * y1 * y1 + T(4) * y * y * y1;
  } else {
    const T th = m_tanh(z[0] * T(0.25)), sc = T(1) - th * th;
    y1 = T(0.5) * sc; y2 = T(-0.25) * th * sc; y3 = T(-0.0625) * sc * sc + T(0.125) * th * th * sc;
  }
  const T zd0 = zd[0];
  zd[0] = out_scale * ((rs ? rs[0] : T(0)) + y1 * zd0);
  const int T3 = S - 2;
  T ss = T(0), sx = T(0);
  for (int t = 1; t <= T3; ++t) {
    const T zt = z[(size_t)t * ldz], zdt = zd[(size_t)t * ldzd];
    ss += zt * zt;
    sx += zt * zdt;
    zd[(size_t)t * ldzd] = out_scale * ((rs ? rs[(size_t)t * ldr] : T(0)) + y2 * zd0 * zt + y1 * zdt);
  }
  const T zl = z[(size_t)(T3 + 1) * ldz], zdl = zd[(size_t)(T3 + 1) * ldzd];
  zd[(size_t)(T3 + 1) * ldzd] = out_scale * ((rs ? rs[(size_t)(T3 + 1) * ldr] : T(0)) + y1 * zdl +
                                             y2 * (zd0 * zl + T(2) * sx) + y3 * zd0 * ss);
}

// ------------------------------------------------------------------------------------------
// FermiNet node-update input of the companion: [hd_i, mean_up hd, mean_down hd, 0, 0] in fermi_agg_kernel's layout (the
// two-particle stream does not depend on R, so its companion is zero and is not computed).  grid = (B S, N).
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void zv_agg_kernel(const T* __restrict__ Hd, int dh, int de, int N, int n_up, int S, T* __restrict__ Fd) {
  const int bs = blockIdx.x, b = bs / S, s = bs % S, i = blockIdx.y;
  const int ldf = 3 * dh + 2 * de;
  T* f = Fd + ((size_t)(b * N + i) * S + s) * ldf;
  const int n_dn = N - n_up;
  for (int k = threadIdx.x; k < ldf; k += blockDim.x) {
    T v = T(0);
    if (k < dh) {
      v = Hd[((size_t)(b * N + i) * S + s) * dh + k];
    } else if (k < 3 * dh) {
      const bool up = k < 2 * dh;
      const int kk = up ? k - dh : k - 2 * dh;
      const int j0 = up ? 0 : n_up, j1 = up ? n_up : N;
      T acc = T(0);
      for (int j = j0; j < j1; ++j) acc += Hd[((size_t)(b * N + j) * S + s) * dh + kk];
      v = acc / (T)(up ? n_up : n_dn);
    }
    f[k] = v;
  }
}

// ------------------------------------------------------------------------------------------
// Companion of the forward-Laplacian attention (attn_fl_kernel's algebra, no extra tokens), one block per (walker, head),
// tangents one at a time.  With delta^t = s^t - m^t and a dot for the companion:
//   sd = c (qd k + q kd),  pd = p (sd - sum_j p sd),  od = pd v + p vd
//   sd^t = c (qd^t k + q^t kd + qd k^t + q kd^t),  md^t = sum_j (pd s^t + p sd^t),  pd^t = pd delta^t + p (sd^t - md^t)
//   od^t = pd^t v + p^t vd + pd v^t + p vd^t
//   sd^L = c (qd^L k + q^L kd + qd k^L + q kd^L + 2 sum_t (qd^t k^t + q^t kd^t))
//   pd^L = pd (u - V + s^L - M^L) + p (ud - Vd + sd^L - Md^L),  ud = 2 sum_t delta^t (sd^t - md^t)
//   od^L = pd^L v + p^L vd + 2 sum_t (pd^t v^t + p^t vd^t) + pd v^L + p vd^L
// QKV / QKVd: [rows][ldq] primal and companion rows; Od: companion output [rows][ldo].
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void zv_attn_kernel(const T* __restrict__ QKV, const T* __restrict__ QKVd, int ldq, T* __restrict__ Od, int ldo,
                               int N, int S, int dh, int dmodel, T scale) {
  DQMC_DYN_SMEM(smem_raw);
  const int dhp = dh + 1, NN = N * N, ND = N * dhp;
  T* q = reinterpret_cast<T*>(smem_raw);  // [N][dhp] each: q k v qd kd vd (value slot), then the same for tangent t
  T* k = q + ND; T* v = k + ND; T* qd = v + ND; T* kd = qd + ND; T* vd = kd + ND;
  T* qt = vd + ND; T* kt = qt + ND; T* vt = kt + ND; T* qtd = vt + ND; T* ktd = qtd + ND; T* vtd = ktd + ND;
  T* p = vtd + ND;   // [N][N]
  T* pd = p + NN;
  T* st = pd + NN;   // s^t, then p^t (s^L, then p^L)
  T* std_ = st + NN; // sd^t, then pd^t
  T* u = std_ + NN;
  T* ud = u + NN;
  T* qk = ud + NN;   // sum_t q^t k^t
  T* qkd = qk + NN;  // sum_t (qd^t k^t + q^t kd^t)
  T* olapd = qkd + NN;  // [N][dh]
  T* mrow = olapd + N * dh;  // [N] each
  T* mrowd = mrow + N;
  T* vrow = mrowd + N;
  T* vrowd = vrow + N;
  const int b = blockIdx.x, h = blockIdx.y;
  const int tid = threadIdx.x, nt = blockDim.x;
  const int T3 = S - 2;
  const size_t row0 = (size_t)b * N * S;
  auto load = [&](int slot, T* a, T* bb, T* cc, T* ad, T* bd, T* cd) {
    for (int idx = tid; idx < N * dh; idx += nt) {
      const int e = idx % dh, i = idx / dh;
      const size_t o = (row0 + (size_t)i * S + slot) * ldq + h * dh + e;
      const int w = i * dhp + e;
      a[w] = QKV[o]; bb[w] = QKV[o + dmodel]; cc[w] = QKV[o + 2 * dmodel];
      ad[w] = QKVd[o]; bd[w] = QKVd[o + dmodel]; cd[w] = QKVd[o + 2 * dmodel];
    }
  };
  auto dot = [&](const T* x, const T* y) {
    T a = T(0);
    for (int e = 0; e < dh; ++e) a += x[e] * y[e];
    return a;
  };
  // row reductions of one [N][N] pair: out[i] = sum_j a[i][j] x[i][j] (+ sum_j ad[i][j] xd[i][j])
  auto rowsum = [&](const T* a, const T* x, const T* a2, const T* x2, T* out) {
    for (int i = tid; i < N; i += nt) {
      T s = T(0);
      for (int j = 0; j < N; ++j) s += a[i * N + j] * x[i * N + j] + (a2 ? a2[i * N + j] * x2[i * N + j] : T(0));
      out[i] = s;
    }
  };
  load(0, q, k, v, qd, kd, vd);
  __syncthreads();
  for (int idx = tid; idx < NN; idx += nt) {
    const int i = idx / N, j = idx % N;
    p[idx] = scale * dot(q + i * dhp, k + j * dhp);
    pd[idx] = scale * (dot(qd + i * dhp, k + j * dhp) + dot(q + i * dhp, kd + j * dhp));
    u[idx] = ud[idx] = qk[idx] = qkd[idx] = T(0);
  }
  for (int idx = tid; idx < N * dh; idx += nt) olapd[idx] = T(0);
  __syncthreads();
  for (int i = tid; i < N; i += nt) {  // softmax row i and its companion
    T mx = p[i * N];
    for (int j = 1; j < N; ++j) mx = p[i * N + j] > mx ? p[i * N + j] : mx;
    T sum = T(0);
    for (int j = 0; j < N; ++j) {
      const T e = m_exp(p[i * N + j] - mx);
      p[i * N + j] = e;
      sum += e;
    }
    const T inv = T(1) / sum;
    T ms = T(0);
    for (int j = 0; j < N; ++j) {
      p[i * N + j] *= inv;
      ms += p[i * N + j] * pd[i * N + j];
    }
    for (int j = 0; j < N; ++j) pd[i * N + j] = p[i * N + j] * (pd[i * N + j] - ms);
  }
  __syncthreads();
  for (int idx = tid; idx < N * dh; idx += nt) {
    const int i = idx / dh, e = idx % dh;
    T a = T(0);
    for (int j = 0; j < N; ++j) a += pd[i * N + j] * v[j * dhp + e] + p[i * N + j] * vd[j * dhp + e];
    Od[(row0 + (size_t)i * S) * ldo + h * dh + e] = a;
  }
  for (int t = 0; t < T3; ++t) {
    __syncthreads();
    load(1 + t, qt, kt, vt, qtd, ktd, vtd);
    __syncthreads();
    for (int idx = tid; idx < NN; idx += nt) {
      const int i = idx / N, j = idx % N;
      const T *qi = q + i * dhp, *qdi = qd + i * dhp, *qti = qt + i * dhp, *qtdi = qtd + i * dhp;
      const T *kj = k + j * dhp, *kdj = kd + j * dhp, *ktj = kt + j * dhp, *ktdj = ktd + j * dhp;
      st[idx] = scale * (dot(qti, kj) + dot(qi, ktj));
      std_[idx] = scale * (dot(qtdi, kj) + dot(qti, kdj) + dot(qdi, ktj) + dot(qi, ktdj));
      qk[idx] += dot(qti, ktj);
      qkd[idx] += dot(qtdi, ktj) + dot(qti, ktdj);
    }
    __syncthreads();
    rowsum(p, st, nullptr, nullptr, mrow);
    rowsum(pd, st, p, std_, mrowd);
    __syncthreads();
    for (int idx = tid; idx < NN; idx += nt) {
      const int i = idx / N;
      const T dl = st[idx] - mrow[i], dld = std_[idx] - mrowd[i];
      u[idx] += dl * dl;
      ud[idx] += T(2) * dl * dld;
      st[idx] = p[idx] * dl;                     // p^t
      std_[idx] = pd[idx] * dl + p[idx] * dld;   // pd^t
    }
    __syncthreads();
    for (int idx = tid; idx < N * dh; idx += nt) {
      const int i = idx / dh, e = idx % dh;
      T a = T(0), c2 = T(0);
      for (int j = 0; j < N; ++j) {
        const T ptj = st[i * N + j], ptdj = std_[i * N + j];
        a += ptdj * v[j * dhp + e] + ptj * vd[j * dhp + e] + pd[i * N + j] * vt[j * dhp + e] + p[i * N + j] * vtd[j * dhp + e];
        c2 += ptdj * vt[j * dhp + e] + ptj * vtd[j * dhp + e];
      }
      Od[(row0 + (size_t)i * S + 1 + t) * ldo + h * dh + e] = a;
      olapd[idx] += T(2) * c2;
    }
  }
  __syncthreads();
  load(1 + T3, qt, kt, vt, qtd, ktd, vtd);
  __syncthreads();
  for (int idx = tid; idx < NN; idx += nt) {
    const int i = idx / N, j = idx % N;
    const T *qi = q + i * dhp, *qdi = qd + i * dhp, *qli = qt + i * dhp, *qldi = qtd + i * dhp;
    const T *kj = k + j * dhp, *kdj = kd + j * dhp, *klj = kt + j * dhp, *kldj = ktd + j * dhp;
    st[idx] = scale * (dot(qli, kj) + dot(qi, klj) + T(2) * qk[idx]);
    std_[idx] = scale * (dot(qldi, kj) + dot(qli, kdj) + dot(qdi, klj) + dot(qi, kldj) + T(2) * qkd[idx]);
  }
  __syncthreads();
  rowsum(p, st, nullptr, nullptr, mrow);     // M^L
  rowsum(pd, st, p, std_, mrowd);            // Md^L
  rowsum(p, u, nullptr, nullptr, vrow);      // V
  rowsum(pd, u, p, ud, vrowd);               // Vd
  __syncthreads();
  for (int idx = tid; idx < NN; idx += nt) {
    const int i = idx / N;
    const T w = u[idx] - vrow[i] + st[idx] - mrow[i];
    const T wd = ud[idx] - vrowd[i] + std_[idx] - mrowd[i];
    st[idx] = p[idx] * w;                  // p^L
    std_[idx] = pd[idx] * w + p[idx] * wd; // pd^L
  }
  __syncthreads();
  for (int idx = tid; idx < N * dh; idx += nt) {
    const int i = idx / dh, e = idx % dh;
    T a = olapd[idx];
    for (int j = 0; j < N; ++j)
      a += std_[i * N + j] * v[j * dhp + e] + st[i * N + j] * vd[j * dhp + e] + pd[i * N + j] * vt[j * dhp + e] +
           p[i * N + j] * vtd[j * dhp + e];
    Od[(row0 + (size_t)i * S + 1 + T3) * ldo + h * dh + e] = a;
  }
}

template <class T>
inline size_t zv_attn_smem_bytes(int N, int dh) {
  return sizeof(T) * ((size_t)12 * N * (dh + 1) + (size_t)10 * N * N + (size_t)N * dh + 4 * (size_t)N);
}

// ------------------------------------------------------------------------------------------
// Companion of the Slater determinants (slater_kernel's algebra, multiplicative backflow, no pseudo-Hamiltonian), one warp
// per (walker b, determinant k).  A = env (.) bf, Ad = envd (.) bf + env (.) bfd (envd: the companion of nucleus m's envelope
// terms), likewise for the tangent and Laplacian entries.  With B = A^-1, Gd = B Ad, G_t = B A_t, H_t = B Ad_t:
//   (log|det A|)d = tr Gd
//   (tr G_t)d     = tr H_t - tr(Gd G_t)
//   (Lap)d        = tr(B Ad_L) - tr(Gd B A_L) - 2 sum_t [tr(G_t H_t) - tr(G_t Gd G_t)]
// BF / BFd: the activated backflow rows [b][i][s][ldb] (orbital k N + mu); outputs zl[B K], zg[B K][T3], zlap[B K].
// An exactly singular A has no inverse: its outputs carry no meaning (the determinant sum weighs them by zero).
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void zv_slater_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M, int n_up,
                                 int K, int S, int total, const T* __restrict__ pi_up, const T* __restrict__ pi_dn,
                                 const T* __restrict__ zeta_up, const T* __restrict__ zeta_dn, const T* __restrict__ BF,
                                 const T* __restrict__ BFd, int ldb, T* __restrict__ zl, T* __restrict__ zg,
                                 T* __restrict__ zlap, int rep, int full_det, int m_k, int c_k) {
  DQMC_DYN_SMEM(smem_raw);
  const int NP = N + 1, N2 = 2 * N + 1, NQ = N * NP;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int gw = blockIdx.x * wpb + wib;
  T* env = reinterpret_cast<T*>(smem_raw) + ((size_t)20 * NQ + (size_t)N * N2 + N) * wib;
  T* denv = env + NQ;    // [3][N][NP]
  T* bfv = denv + 3 * NQ;
  T* envd = bfv + NQ;
  T* denvd = envd + NQ;  // [3][N][NP]
  T* bfd = denvd + 3 * NQ;
  T* Ad = bfd + NQ;      // A dot
  T* Gd = Ad + NQ;       // B A dot
  T* AL = Gd + NQ;
  T* ALd = AL + NQ;
  T* At = ALd + NQ;
  T* Atd = At + NQ;
  T* Gt = Atd + NQ;
  T* Ht = Gt + NQ;
  T* Wt = Ht + NQ;
  T* aug = Wt + NQ;      // [N][N2]
  T* fcol = aug + N * N2;
  if (gw >= total) return;
  const int b = gw / K, k = gw % K;
  const int T3 = S - 2;
  const T* rb = r + (size_t)b * N * 3;
  const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
  const size_t brow0 = (size_t)b * N * S;
  auto bfp = [&](const T* base, int i, int s, int mu) { return base[(brow0 + (size_t)i * S + s) * ldb + k * N + mu]; };

  for (LaneWalk w(lane, N); w.i < N; w.next()) {
    const int i = w.i, mu = w.j;
    const T* pi = (i < n_up ? pi_up : pi_dn) + (size_t)(k * N + mu) * M * rep;
    const T* ze = (i < n_up ? zeta_up : zeta_dn) + (size_t)(k * N + mu) * M * rep;
    T e = 0, de[3] = {0, 0, 0}, le = 0, ed = 0, ded[3] = {0, 0, 0}, led = 0;
    for (int m = 0; m < M; ++m) {
      const T dx[3] = {rb[3 * i] - Rb[3 * m], rb[3 * i + 1] - Rb[3 * m + 1], rb[3 * i + 2] - Rb[3 * m + 2]};
      const T u = dx[0] * dx[0] + dx[1] * dx[1] + dx[2] * dx[2];
      const T rho2 = Num<T>::eps() + u, rho = m_sqrt(rho2);
      const T gr2 = u / rho2, lr = T(3) / rho - u / (rho2 * rho);
      T F1 = T(0), F2 = T(0), F3 = T(0);
      for (int et = 0; et < rep; ++et) {
        const T a = m_abs(ze[m * rep + et]);
        const T ex = pi[m * rep + et] * m_exp(-a * rho);
        e += ex;
        const T cc = -a * ex / rho;
        de[0] += cc * dx[0]; de[1] += cc * dx[1]; de[2] += cc * dx[2];
        le += ex * (a * a * gr2 - a * lr);
        F1 -= a * ex; F2 += a * a * ex; F3 -= a * a * a * ex;
      }
      if (m == m_k) {
        T g1, g2, g3, v, dd[3], l;
        zv_chain_u(rho, F1, F2, F3, g1, g2, g3);
        zv_radial(dx, u, c_k, g1, g2, g3, v, dd, l);
        ed = v; ded[0] = dd[0]; ded[1] = dd[1]; ded[2] = dd[2]; led = l;
      }
    }
    if (!full_det && ((i < n_up) != (mu < n_up))) {
      e = le = ed = led = T(0);
      for (int c = 0; c < 3; ++c) de[c] = ded[c] = T(0);
    }
    const T bf0 = bfp(BF, i, 0, mu), bfd0 = bfp(BFd, i, 0, mu);
    const T bfl = bfp(BF, i, 1 + T3, mu), bfdl = bfp(BFd, i, 1 + T3, mu);
    const int o = i * NP + mu;
    env[o] = e; bfv[o] = bf0; envd[o] = ed; bfd[o] = bfd0;
    T al = le * bf0 + e * bfl, ald = led * bf0 + le * bfd0 + ed * bfl + e * bfdl;
    for (int c = 0; c < 3; ++c) {
      denv[c * NQ + o] = de[c];
      denvd[c * NQ + o] = ded[c];
      const T x = bfp(BF, i, 1 + 3 * i + c, mu), xd = bfp(BFd, i, 1 + 3 * i + c, mu);
      al += T(2) * de[c] * x;
      ald += T(2) * (ded[c] * x + de[c] * xd);
    }
    AL[o] = al; ALd[o] = ald;
    Ad[o] = ed * bf0 + e * bfd0;
    aug[i * N2 + mu] = e * bf0;
    aug[i * N2 + N + mu] = (i == mu) ? T(1) : T(0);
  }
  __syncwarp();

  // Gauss-Jordan with partial pivoting on [A | I] (slater_kernel's elimination; the inverse is all that is needed here)
  for (int c = 0; c < N; ++c) {
    T best = T(-1);
    int bi = c;
    for (int rr = c + lane; rr < N; rr += 32) {
      const T vv = m_abs(aug[rr * N2 + c]);
      if (vv > best) { best = vv; bi = rr; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const T ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (bi != c) {
      for (int j = lane; j < 2 * N; j += 32) {
        const T t0 = aug[c * N2 + j];
        aug[c * N2 + j] = aug[bi * N2 + j];
        aug[bi * N2 + j] = t0;
      }
    }
    __syncwarp();
    const T pv = aug[c * N2 + c];
    for (int rr = lane; rr < N; rr += 32) fcol[rr] = aug[rr * N2 + c];
    __syncwarp();
    const T ipv = pv != T(0) ? T(1) / pv : T(0);
    for (int j = lane; j < 2 * N; j += 32) aug[c * N2 + j] *= ipv;
    __syncwarp();
    for (LaneWalk w(lane, 2 * N); w.i < N; w.next()) {
      if (w.i != c) aug[w.i * N2 + w.j] -= fcol[w.i] * aug[c * N2 + w.j];
    }
    __syncwarp();
  }
  // B[mu][i] = aug[mu][N + i];  C = B X for X [N][NP]
  auto bmul = [&](const T* X, T* C) {
    for (LaneWalk w(lane, N); w.i < N; w.next()) {
      T a = T(0);
      for (int i = 0; i < N; ++i) a += aug[w.i * N2 + N + i] * X[i * NP + w.j];
      C[w.i * NP + w.j] = a;
    }
  };
  // sum_{mu nu} X[mu][nu] Y[nu][mu]
  auto trprod = [&](const T* X, const T* Y) {
    T a = T(0);
    for (LaneWalk w(lane, N); w.i < N; w.next()) a += X[w.i * NP + w.j] * Y[w.j * NP + w.i];
    return warp_sum(a);
  };
  bmul(Ad, Gd);
  bmul(AL, At);  // B A_L
  __syncwarp();
  T ld = T(0), lapd = T(0);
  for (LaneWalk w(lane, N); w.i < N; w.next()) {
    if (w.i == w.j) ld += Gd[w.i * NP + w.i];
    lapd += aug[w.j * N2 + N + w.i] * ALd[w.i * NP + w.j];  // B[mu][i] ALd[i][mu], (i, mu) = (w.i, w.j)
  }
  ld = warp_sum(ld);
  lapd = warp_sum(lapd) - trprod(Gd, At);
  const size_t bk = (size_t)b * K + k;
  for (int t = 0; t < T3; ++t) {
    const int it = t / 3, ct = t % 3;
    __syncwarp();
    for (LaneWalk w(lane, N); w.i < N; w.next()) {
      const int i = w.i, mu = w.j, o = i * NP + mu;
      const T x = bfp(BF, i, 1 + t, mu), xd = bfp(BFd, i, 1 + t, mu);
      T a = env[o] * x, ad = envd[o] * x + env[o] * xd;
      if (i == it) {
        a += denv[ct * NQ + o] * bfv[o];
        ad += denvd[ct * NQ + o] * bfv[o] + denv[ct * NQ + o] * bfd[o];
      }
      At[o] = a; Atd[o] = ad;
    }
    __syncwarp();
    bmul(At, Gt);
    bmul(Atd, Ht);
    __syncwarp();
    for (LaneWalk w(lane, N); w.i < N; w.next()) {  // Wt = Gd G_t
      T a = T(0);
      for (int j = 0; j < N; ++j) a += Gd[w.i * NP + j] * Gt[j * NP + w.j];
      Wt[w.i * NP + w.j] = a;
    }
    __syncwarp();
    T trh = T(0);
    for (int mu = lane; mu < N; mu += 32) trh += Ht[mu * NP + mu];
    trh = warp_sum(trh);
    const T gdt = trh - trprod(Gd, Gt);
    lapd -= T(2) * (trprod(Gt, Ht) - trprod(Gt, Wt));
    if (lane == 0) zg[bk * T3 + t] = gdt;
  }
  if (lane == 0) { zl[bk] = ld; zlap[bk] = lapd; }
}

template <class T>
inline size_t zv_slater_smem_per_warp(int N) {
  return sizeof(T) * ((size_t)20 * N * (N + 1) + (size_t)N * (2 * N + 1) + N);
}
template <class T>
inline int zv_slater_warps_per_block(int N) {
  const size_t pw = zv_slater_smem_per_warp<T>(N);
  const int w = (int)((96 * 1024) / pw);
  return w < 1 ? 1 : (w > 4 ? 4 : w);
}

// ------------------------------------------------------------------------------------------
// Companion of the determinant sum, the nuclear cusp and the kinetic assembly (finalize_kernel's algebra, all-electron,
// no Jastrow), one block per walker.  p_k = c_k s_k exp(l_k) / psi; with the det sum's companions
//   ld = sum_k p_k ld_k,  pd_k = p_k (ld_k - ld),  gd_t = sum_k (pd_k g_kt + p_k gd_kt)
//   Lap_dot = sum_k (pd_k lap_k + p_k lapd_k) + sum_t [sum_k (pd_k g_kt^2 + 2 p_k g_kt gd_kt) - 2 g_t gd_t] + the nuclear cusp's
// (the e-e cusp does not depend on R).  G [B][T3]: the primal grad log|psi| of finalize_kernel.  Writes
//   out_zv[b ld + kappa] = 1/2 Lap_dot + sum_t G_t Gd_t  (= -dT/dR_kappa),  out_gR[b ld + kappa] = d log|psi| / dR_kappa.
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void zv_finalize_kernel(int N, int M, int K, int S, int nuc_cusp_kind, const T* __restrict__ r,
                                   const T* __restrict__ R, int R_batched, const T* __restrict__ det_sign,
                                   const T* __restrict__ det_log, const T* __restrict__ det_grad, const T* __restrict__ det_lap,
                                   const T* __restrict__ zl, const T* __restrict__ zg, const T* __restrict__ zlap,
                                   const T* __restrict__ conf_w, const T* __restrict__ G, const T* __restrict__ nuc_cusp,
                                   int m_k, int c_k, int ld_out, int kappa, T* __restrict__ out_zv, T* __restrict__ out_gR) {
  DQMC_DYN_SMEM(smem_raw);
  T* pk = reinterpret_cast<T*>(smem_raw);  // [K]
  T* pkd = pk + K;                          // [K]
  T* scratch = pkd + K;                     // [66]
  T* misc = scratch + 66;                   // [2]
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const int T3 = S - 2;
  const T* ds = det_sign + (size_t)b * K;
  const T* dl = det_log + (size_t)b * K;
  const T* zlb = zl + (size_t)b * K;
  if (tid == 0) {
    T shift = dl[0];
    for (int k = 1; k < K; ++k) shift = dl[k] > shift ? dl[k] : shift;
    if ((shift - shift) != T(0)) shift = T(0);
    T psi = T(0);
    for (int k = 0; k < K; ++k) {
      pk[k] = (conf_w ? conf_w[k] : T(1)) * ds[k] * m_exp(dl[k] - shift);
      psi += pk[k];
    }
    T lbar = T(0);
    for (int k = 0; k < K; ++k) {
      pk[k] /= psi;
      if (pk[k] != T(0)) lbar += pk[k] * zlb[k];
    }
    for (int k = 0; k < K; ++k) pkd[k] = pk[k] != T(0) ? pk[k] * (zlb[k] - lbar) : T(0);
    misc[0] = lbar;
  }
  __syncthreads();
  const T* rb = r + (size_t)b * N * 3;
  const T* Rm = R + (R_batched ? (size_t)b * M * 3 : 0) + 3 * m_k;
  T al = T(0), sc = T(0), den0 = T(0);
  if (nuc_cusp_kind != 0) {
    al = nuc_cusp[0];
    const T zn = nuc_cusp[1 + m_k];
    sc = zn * (nuc_cusp_kind == 1 ? al * al : T(1) / (al * al));
    den0 = nuc_cusp_kind == 1 ? al : T(1) / al;
  }
  // companion of the nuclear cusp -sc / (den0 + |r_i - R_m|) (plain norm) for electron i: value, d/dr_i,e, Lap
  auto cusp = [&](int i, T& v, T (&de)[3], T& l) {
    const T dx[3] = {rb[3 * i] - Rm[0], rb[3 * i + 1] - Rm[1], rb[3 * i + 2] - Rm[2]};
    const T u = dx[0] * dx[0] + dx[1] * dx[1] + dx[2] * dx[2];
    const T rho = m_sqrt(u), den = den0 + rho;
    const T F1 = sc / (den * den), F2 = T(-2) * sc / (den * den * den), F3 = T(6) * sc / (den * den * den * den);
    T g1, g2, g3;
    zv_chain_u(rho, F1, F2, F3, g1, g2, g3);
    zv_radial(dx, u, c_k, g1, g2, g3, v, de, l);
  };
  const T* dg = det_grad + (size_t)b * K * T3;
  const T* zgb = zg + (size_t)b * K * T3;
  const T* Gb = G + (size_t)b * T3;
  T lap_d = T(0), gg_d = T(0);
  for (int t = tid; t < T3; t += nt) {
    T gd = T(0), gdd = T(0), a_d = T(0);
    for (int k = 0; k < K; ++k) {
      if (pk[k] == T(0)) continue;
      const T g = dg[(size_t)k * T3 + t], gz = zgb[(size_t)k * T3 + t];
      gd += pk[k] * g;
      gdd += pkd[k] * g + pk[k] * gz;
      a_d += pkd[k] * g * g + T(2) * pk[k] * g * gz;
    }
    lap_d += a_d - T(2) * gd * gdd;
    if (nuc_cusp_kind != 0) {
      T v, de[3], l;
      cusp(t / 3, v, de, l);
      gdd += de[t % 3];
    }
    gg_d += Gb[t] * gdd;
  }
  T val_d = T(0), dummy = T(0);
  if (nuc_cusp_kind != 0)
    for (int i = tid; i < N; i += nt) {
      T v, de[3], l;
      cusp(i, v, de, l);
      val_d += v;
      lap_d += l;
    }
  block_sum2(lap_d, gg_d, scratch);
  block_sum2(val_d, dummy, scratch);
  if (tid == 0) {
    for (int k = 0; k < K; ++k)
      if (pk[k] != T(0)) lap_d += pkd[k] * det_lap[(size_t)b * K + k] + pk[k] * zlap[(size_t)b * K + k];
    out_zv[(size_t)b * ld_out + kappa] = T(0.5) * lap_d + gg_d;
    if (out_gR) out_gR[(size_t)b * ld_out + kappa] = misc[0] + val_d;
  }
}

template <class T>
inline size_t zv_finalize_smem_bytes(int K) {
  return sizeof(T) * ((size_t)2 * K + 66 + 2);
}

}  // namespace dq
