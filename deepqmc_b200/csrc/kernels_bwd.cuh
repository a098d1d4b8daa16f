// Reverse pass of the plain forward (S = 1): d/dparams sum_b w_b log|psi(r_b)| for the Psiformer.
// This is the parameter VJP the reference's loss takes through `jvp`/`grad` of ansatz.apply
// (reference src/deepqmc/loss/loss_function.py:53-82 compute_log_psi_tangent, loss/energy.py:77-102:
// grad E = 2 < (E_loc - <E_loc>) d log|psi| / d theta >), SURVEY.md 8(f) row N1.
// Parameter gradients are ACCUMULATED (atomicAdd) into a caller-zeroed buffer with the engine's
// packed layout.  Kernels are SIMT and generic in T (fp64 parity / fp32).
#pragma once
#include "common.cuh"

namespace dq {

template <class T>
__device__ __forceinline__ void atomic_add(T* p, T v) { atomicAdd(p, v); }

// ------------------------------------------------------------------------------------------
// dW[k][n] += sum_rows A[row][k] * dY[row][n]  (weight gradient of Y = A W).  Tile 32 x 32 of dW per block,
// the row range is split over blockIdx.z; partial tiles are added atomically.
// Row selection for the per-spin backflow heads: rows are (b, i) with i = row % Nel; only i in [lo, hi) counts.
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void gemm_tn_kernel(const T* __restrict__ A, int lda, const T* __restrict__ dY, int ldy, int rows, int K,
                               int Nc, int rows_per_block, int Nel, int lo, int hi, T* __restrict__ dW, int ldw) {
  __shared__ T As[32][33];
  __shared__ T Ys[32][33];
  const int k0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8 threads, 4 k-rows each
  const int r_begin = blockIdx.z * rows_per_block;
  const int r_end = r_begin + rows_per_block < rows ? r_begin + rows_per_block : rows;
  T acc[4] = {T(0), T(0), T(0), T(0)};
  for (int r0 = r_begin; r0 < r_end; r0 += 32) {
    __syncthreads();
    for (int rr = ty; rr < 32; rr += 8) {
      const int row = r0 + rr;
      bool ok = row < r_end;
      if (ok && Nel > 0) { const int i = row % Nel; ok = i >= lo && i < hi; }
      As[rr][tx] = (ok && k0 + tx < K) ? A[(size_t)row * lda + k0 + tx] : T(0);
      Ys[rr][tx] = (ok && n0 + tx < Nc) ? dY[(size_t)row * ldy + n0 + tx] : T(0);
    }
    __syncthreads();
#pragma unroll 4
    for (int rr = 0; rr < 32; ++rr) {
      const T y = Ys[rr][tx];
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[q] += As[rr][ty * 4 + q] * y;
    }
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int k = k0 + ty * 4 + q, n = n0 + tx;
    if (k < K && n < Nc && acc[q] != T(0)) atomic_add(dW + (size_t)k * ldw + n, acc[q]);
  }
}

// db[n] += sum_rows dZ[row][n]
// (rows are (b, i) with i = row % Nel; Nel > 0: only electrons lo <= i < hi count -- per-spin biases)
template <class T>
__global__ void colsum_kernel(const T* __restrict__ dZ, int ld, int rows, int Nc, int rows_per_block, T* __restrict__ db,
                              int Nel, int lo, int hi) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= Nc) return;
  const int r_begin = blockIdx.y * rows_per_block;
  const int r_end = r_begin + rows_per_block < rows ? r_begin + rows_per_block : rows;
  T acc = T(0);
  for (int r = r_begin; r < r_end; ++r) {
    if (Nel > 0) { const int i = r % Nel; if (i < lo || i >= hi) continue; }
    acc += dZ[(size_t)r * ld + n];
  }
  atomic_add(db + n, acc);
}

// dZ = dY * (1 - y^2) with y = Y - Ysub (Ysub nullable): backward of y = tanh(z) given the stored outputs.
template <class T>
__global__ void tanh_bwd_kernel(const T* __restrict__ dY, const T* __restrict__ Y, const T* __restrict__ Ysub,
                                T* __restrict__ dZ, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const T y = Y[i] - (Ysub ? Ysub[i] : T(0));
  dZ[i] = dY[i] * (T(1) - y * y);
}

// Backward of y = scale * (res + tanh(z)) (FermiNet residual / sqrt(2), hkext.py:116-137) or y = tanh(z) (Res null,
// scale 1) from the stored outputs: dZ = dY scale (1 - t^2), t = Y / scale - res.
template <class T>
__global__ void tanh_res_bwd_kernel(const T* __restrict__ dY, const T* __restrict__ Y, const T* __restrict__ Res, T scale,
                                    T* __restrict__ dZ, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const T t = Y[i] / scale - (Res ? Res[i] : T(0));
  dZ[i] = dY[i] * scale * (T(1) - t * t);
}

// Backward of fermi_agg_kernel (kernels_trunk.cuh) for the plain forward: from dF[b][i][3 dh + 2 de]
//   dH[b][j][k]    = dF[b][j][k] + (1 / n_spin(j)) sum_i dF[b][i][dh (1 + down(j)) + k]  (+ res_scale * dRes[b][j][k])
//   dE[b][j][i][k] = dF[b][i][3 dh + de down(j) + k] / n_spin(j)
// One block per (walker, electron j).  dH / dE may be null (first layer: nothing upstream has parameters).
template <class T>
__global__ void fermi_agg_bwd_kernel(const T* __restrict__ dF, int dh, int de, int N, int n_up, const T* __restrict__ dRes,
                                     T res_scale, T* __restrict__ dH, T* __restrict__ dE, int ldf_ /*row stride, 0: 3 dh + 2 de*/) {
  const int b = blockIdx.x, j = blockIdx.y;
  const int ldf = ldf_ > 0 ? ldf_ : 3 * dh + 2 * de;
  const bool down = j >= n_up;
  const T inv = T(1) / (T)(down ? N - n_up : n_up);
  const T* dFb = dF + (size_t)b * N * ldf;
  if (dH)
    for (int k = threadIdx.x; k < dh; k += blockDim.x) {
      T acc = T(0);
      for (int i = 0; i < N; ++i) acc += dFb[(size_t)i * ldf + dh * (down ? 2 : 1) + k];
      T v = dFb[(size_t)j * ldf + k] + inv * acc;
      if (dRes) v += res_scale * dRes[((size_t)b * N + j) * dh + k];
      dH[((size_t)b * N + j) * dh + k] = v;
    }
  if (dE)
    for (int idx = threadIdx.x; idx < N * de; idx += blockDim.x) {
      const int i = idx / de, k = idx - i * de;
      dE[(((size_t)b * N + j) * N + i) * de + k] = inv * dFb[(size_t)i * ldf + 3 * dh + (down ? de : 0) + k];
    }
}

// y += a x
template <class T>
__global__ void axpy_kernel(const T* __restrict__ x, T a, T* __restrict__ y, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] += a * x[i];
}

// W[rows][cols] -> Wt[cols][rows]
template <class T>
__global__ void transpose_kernel(const T* __restrict__ W, int rows, int cols, T* __restrict__ Wt) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * cols) return;
  const int r = idx / cols, c = idx - r * cols;
  Wt[(size_t)c * rows + r] = W[idx];
}

// ------------------------------------------------------------------------------------------
// Attention backward (plain forward), one block per (walker, head):  P = softmax(c q k^T), o = P v;
//   dV = P^T dO;  dP = dO V^T;  dS = P (dP - rowsum(dP P));  dq = c dS k;  dk = c dS^T q.
// QKV / dQKV rows [b][i][3 dmodel]; dO rows [b][i][dmodel].
// dynamic smem = sizeof(T) * (4 N (dh + 1) + 2 N N).
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void attn_bwd_kernel(const T* __restrict__ QKV, int ldq, const T* __restrict__ dO, int ldo, int N, int dh,
                                int dmodel, T scale, T* __restrict__ dQKV, const T* __restrict__ Kn,
                                const T* __restrict__ Vn, int Mn, T* __restrict__ dKn, T* __restrict__ dVn) {
  // Kn / Vn [Mn][dmodel] (nullable): keys / values of Mn walker-independent extra tokens behind the N electron
  // keys (TransPsiformer nuclei); their cotangents are accumulated over walkers into dKn / dVn (atomicAdd).
  DQMC_DYN_SMEM(smem_raw);
  const int NK = N + Mn;
  const int dhp = dh + 1, NN = N * NK;
  T* q = reinterpret_cast<T*>(smem_raw);  // [N][dhp]
  T* go = q + N * dhp;                    // [N][dhp]  dO
  T* k = go + N * dhp;                    // [NK][dhp]
  T* v = k + NK * dhp;                    // [NK][dhp]
  T* p = v + NK * dhp;                    // [N][NK]
  T* ds = p + NN;                         // [N][NK]
  const int b = blockIdx.x, h = blockIdx.y, tid = threadIdx.x, nt = blockDim.x;
  const size_t row0 = (size_t)b * N;
  for (int idx = tid; idx < N * dh; idx += nt) {
    const int i = idx / dh, e = idx - i * dh;
    const T* src = QKV + (row0 + i) * ldq + h * dh + e;
    q[i * dhp + e] = src[0]; k[i * dhp + e] = src[dmodel]; v[i * dhp + e] = src[2 * dmodel];
    go[i * dhp + e] = dO[(row0 + i) * ldo + h * dh + e];
  }
  for (int idx = tid; idx < Mn * dh; idx += nt) {
    const int m = idx / dh, e = idx - m * dh;
    k[(N + m) * dhp + e] = Kn[(size_t)m * dmodel + h * dh + e];
    v[(N + m) * dhp + e] = Vn[(size_t)m * dmodel + h * dh + e];
  }
  __syncthreads();
  for (int idx = tid; idx < NN; idx += nt) {
    const int i = idx / NK, j = idx - i * NK;
    T a = T(0), c = T(0);
    for (int e = 0; e < dh; ++e) { a += q[i * dhp + e] * k[j * dhp + e]; c += go[i * dhp + e] * v[j * dhp + e]; }
    p[idx] = a * scale;
    ds[idx] = c;  // dP
  }
  __syncthreads();
  for (int i = tid; i < N; i += nt) {
    T mx = p[i * NK];
    for (int j = 1; j < NK; ++j) mx = p[i * NK + j] > mx ? p[i * NK + j] : mx;
    T sum = T(0);
    for (int j = 0; j < NK; ++j) { T ex = m_exp(p[i * NK + j] - mx); p[i * NK + j] = ex; sum += ex; }
    T inv = T(1) / sum, dot = T(0);
    for (int j = 0; j < NK; ++j) { p[i * NK + j] *= inv; dot += p[i * NK + j] * ds[i * NK + j]; }
    for (int j = 0; j < NK; ++j) ds[i * NK + j] = p[i * NK + j] * (ds[i * NK + j] - dot) * scale;  // c dS
  }
  __syncthreads();
  for (int idx = tid; idx < N * dh; idx += nt) {
    const int i = idx / dh, e = idx - i * dh;
    T dq = T(0), dk = T(0), dv = T(0);
    for (int j = 0; j < NK; ++j) dq += ds[i * NK + j] * k[j * dhp + e];
    for (int j = 0; j < N; ++j) {
      dk += ds[j * NK + i] * q[j * dhp + e];
      dv += p[j * NK + i] * go[j * dhp + e];
    }
    T* dst = dQKV + (row0 + i) * ldq + h * dh + e;
    dst[0] = dq; dst[dmodel] = dk; dst[2 * dmodel] = dv;
  }
  for (int idx = tid; dKn && idx < Mn * dh; idx += nt) {  // dKn / dVn null: parameter cotangents not wanted
    const int m = idx / dh, e = idx - m * dh;
    T dk = T(0), dv = T(0);
    for (int j = 0; j < N; ++j) {
      dk += ds[j * NK + N + m] * q[j * dhp + e];
      dv += p[j * NK + N + m] * go[j * dhp + e];
    }
    atomic_add(dKn + (size_t)m * dmodel + h * dh + e, dk);
    atomic_add(dVn + (size_t)m * dmodel + h * dh + e, dv);
  }
}

template <class T>
inline size_t attn_bwd_smem_bytes(int N, int dh, int Mn = 0) {
  return sizeof(T) * ((size_t)2 * N * (dh + 1) + (size_t)2 * (N + Mn) * (dh + 1) + (size_t)2 * N * (N + Mn));
}

// ------------------------------------------------------------------------------------------
// Determinant-sum backward: dlogdet[b][k] = w_b p_k,  p_k = c_k s_k e^{l_k - shift} / psi  (d log|psi| / d logdet_k),
// plus the trainable cusp exponents (PsiformerCusp: -s a^2 / (a + r)) accumulated into dalpha[2].
// One thread per walker.
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void finalize_bwd_kernel(const T* __restrict__ r, int N, int n_up, int K, int B,
                                    const T* __restrict__ det_sign, const T* __restrict__ det_log,
                                    const T* __restrict__ weights, int cusp_kind, T same_scale, T anti_scale,
                                    const T* __restrict__ cusp_alpha, T* __restrict__ dlogdet, T* __restrict__ dalpha,
                                    const T* __restrict__ R, int R_batched, int M, int nuc_cusp_kind,
                                    const T* __restrict__ nuc_cusp /*[1 + M]: alpha, charges*/, T* __restrict__ dnuc_alpha,
                                    const T* __restrict__ conf_w /*[K] hk.Linear determinant weights or null (SumPool)*/,
                                    T* __restrict__ dconf_w) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const T w = weights ? weights[b] : T(1);  // null: per-walker cotangent 1 (position gradients)
  const T* ds = det_sign + (size_t)b * K;
  const T* dl = det_log + (size_t)b * K;
  T shift = dl[0];
  for (int k = 1; k < K; ++k) shift = dl[k] > shift ? dl[k] : shift;
  if ((shift - shift) != T(0)) shift = T(0);
  T psi = T(0);
  for (int k = 0; k < K; ++k) psi += (conf_w ? conf_w[k] : T(1)) * ds[k] * m_exp(dl[k] - shift);
  for (int k = 0; k < K; ++k) {
    const T xk = ds[k] * m_exp(dl[k] - shift) / psi;  // d log|psi| / d c_k;  times c_k: d log|psi| / d logdet_k
    dlogdet[(size_t)b * K + k] = w * (conf_w ? conf_w[k] : T(1)) * xk;
    if (conf_w && dconf_w) atomic_add(dconf_w + k, w * xk);
  }
  if (cusp_kind == 1 && dalpha) {
    const T as_ = cusp_alpha[0], aa_ = cusp_alpha[1];
    T gs = T(0), ga = T(0);
    const T* rb = r + (size_t)b * N * 3;
    for (int i = 0; i < N; ++i)
      for (int j = i + 1; j < N; ++j) {
        const T dx0 = rb[3 * i] - rb[3 * j], dx1 = rb[3 * i + 1] - rb[3 * j + 1], dx2 = rb[3 * i + 2] - rb[3 * j + 2];
        const T rho = m_sqrt(Num<T>::eps() + dx0 * dx0 + dx1 * dx1 + dx2 * dx2);
        const bool same = (i < n_up) == (j < n_up);
        const T al = same ? as_ : aa_, sc = same ? same_scale : anti_scale;
        const T g = -sc * al * (al + T(2) * rho) / ((al + rho) * (al + rho));  // d/dalpha of -s a^2 / (a + rho)
        if (same) gs += g; else ga += g;
      }
    atomic_add(dalpha, w * gs);
    atomic_add(dalpha + 1, w * ga);
  }
  if (nuc_cusp_kind != 0 && dnuc_alpha) {
    // NuclearCuspAsymptotic exponent (wf/cusp.py:81-101) on the plain electron-nucleus distances:
    // psiformer form -Z a^2 / (a + d), deepqmc form -Z / (a (1 + a d))
    const T al = nuc_cusp[0];
    const T* rb = r + (size_t)b * N * 3;
    const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
    T g = T(0);
    for (int i = 0; i < N; ++i)
      for (int m = 0; m < M; ++m) {
        const T dx0 = rb[3 * i] - Rb[3 * m], dx1 = rb[3 * i + 1] - Rb[3 * m + 1], dx2 = rb[3 * i + 2] - Rb[3 * m + 2];
        const T dist = m_sqrt(dx0 * dx0 + dx1 * dx1 + dx2 * dx2), z = nuc_cusp[1 + m];
        if (nuc_cusp_kind == 1) g -= z * al * (al + T(2) * dist) / ((al + dist) * (al + dist));
        else g += z * (T(1) + T(2) * al * dist) / (al * al * (T(1) + al * dist) * (T(1) + al * dist));
      }
    atomic_add(dnuc_alpha, w * g);
  }
}

// ------------------------------------------------------------------------------------------
// Slater backward, one warp per (walker, determinant): rebuild A = env * bf, invert it (Gauss-Jordan with partial
// pivoting), G = dlogdet A^-T;  dBF[b][i][k N + mu] = G[i][mu] env[i][mu];  envelope parameters:
//   dpi[o][m] += G bf e^{-|zeta| rho},  dzeta[o][m] += G bf pi e^{-|zeta| rho} (-rho sign(zeta))   (o = k N + mu).
// dpi_up null: no envelope-parameter gradients.  cpart (nullable) [B K][N][M][3]: this determinant's share of the pair
// cotangent d log|psi| / d d_im (d_im = r_i - R_m) through the envelopes,
//   sum_mu G bf sum_t pi e^{-|zeta| rho} (-|zeta|) d_im / rho,
// summed over mu in a fixed order by one lane per (i, m) (no atomics: callers reduce over k in order).
// dynamic smem per warp: sizeof(T) * (N (2N + 1) + 2 N (N + 1)).
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void slater_bwd_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M,
                                  int n_up, int K, int total, const T* __restrict__ pi_up, const T* __restrict__ pi_dn,
                                  const T* __restrict__ zeta_up, const T* __restrict__ zeta_dn,
                                  const T* __restrict__ BF, int ldb, const T* __restrict__ dlogdet, T* __restrict__ dBF,
                                  T* __restrict__ dpi_up, T* __restrict__ dpi_dn, T* __restrict__ dzeta_up,
                                  T* __restrict__ dzeta_dn, int rep, int full_det, T* __restrict__ cpart) {
  // full_det == 0: spin-factorised determinants = block-diagonal A (off-diagonal spin blocks zero, as in slater_kernel)
  DQMC_DYN_SMEM(smem_raw);
  const int NP = N + 1, N2 = 2 * N + 1;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int gw = blockIdx.x * wpb + wib;
  const size_t per_warp = (size_t)N * N2 + (size_t)2 * N * NP;
  T* aug = reinterpret_cast<T*>(smem_raw) + per_warp * wib;  // [N][N2]
  T* env = aug + N * N2;                                      // [N][NP]
  T* bfv = env + N * NP;                                      // [N][NP]
  if (gw >= total) return;
  const int b = gw / K, k = gw % K;
  const T* rb = r + (size_t)b * N * 3;
  const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
  for (int idx = lane; idx < N * N; idx += 32) {
    const int i = idx / N, mu = idx - i * N;
    const T* pi = (i < n_up ? pi_up : pi_dn) + (size_t)(k * N + mu) * M * rep;
    const T* ze = (i < n_up ? zeta_up : zeta_dn) + (size_t)(k * N + mu) * M * rep;
    T e = T(0);
    for (int m = 0; m < M; ++m) {
      const T dx0 = rb[3 * i] - Rb[3 * m], dx1 = rb[3 * i + 1] - Rb[3 * m + 1], dx2 = rb[3 * i + 2] - Rb[3 * m + 2];
      const T rho = m_sqrt(Num<T>::eps() + dx0 * dx0 + dx1 * dx1 + dx2 * dx2);
      for (int et = 0; et < rep; ++et) e += pi[m * rep + et] * m_exp(-m_abs(ze[m * rep + et]) * rho);
    }
    if (!full_det && ((i < n_up) != (mu < n_up))) e = T(0);
    const T bf0 = BF[((size_t)b * N + i) * ldb + k * N + mu];
    env[i * NP + mu] = e;
    bfv[i * NP + mu] = bf0;
    aug[i * N2 + mu] = e * bf0;
    aug[i * N2 + N + mu] = (i == mu) ? T(1) : T(0);
  }
  __syncwarp();
  for (int c = 0; c < N; ++c) {
    T best = T(-1);
    int bi = c;
    for (int rr = c + lane; rr < N; rr += 32) {
      T vv = m_abs(aug[rr * N2 + c]);
      if (vv > best) { best = vv; bi = rr; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      T ob = __shfl_xor_sync(0xffffffffu, best, o);
      int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    const int prow = bi;
    if (prow != c) {
      for (int j = lane; j < 2 * N; j += 32) {
        T t0 = aug[c * N2 + j];
        aug[c * N2 + j] = aug[prow * N2 + j];
        aug[prow * N2 + j] = t0;
      }
    }
    __syncwarp();
    const T ipv = T(1) / aug[c * N2 + c];
    __syncwarp();
    for (int j = lane; j < 2 * N; j += 32) aug[c * N2 + j] *= ipv;
    __syncwarp();
    for (int rr = 0; rr < N; ++rr) {
      if (rr == c) continue;
      const T f = aug[rr * N2 + c];
      __syncwarp();
      for (int j = lane; j < 2 * N; j += 32) aug[rr * N2 + j] -= f * aug[c * N2 + j];
      __syncwarp();
    }
  }
  // A^-1[mu][i] = aug[mu][N + i];  G[i][mu] = dlogdet * A^-1[mu][i]
  const T dl = dlogdet[(size_t)b * K + k];
  for (int idx = lane; idx < N * N; idx += 32) {
    const int i = idx / N, mu = idx - i * N;
    const bool blocked = !full_det && ((i < n_up) != (mu < n_up));
    const T G = blocked ? T(0) : dl * aug[mu * N2 + N + i];
    dBF[((size_t)b * N + i) * ldb + k * N + mu] = G * env[i * NP + mu];
    if (blocked || !dpi_up) continue;
    const T gb = G * bfv[i * NP + mu];  // d / d env[i][mu]
    const bool up = i < n_up;
    const T* pi = (up ? pi_up : pi_dn) + (size_t)(k * N + mu) * M * rep;
    const T* ze = (up ? zeta_up : zeta_dn) + (size_t)(k * N + mu) * M * rep;
    T* dpi = (up ? dpi_up : dpi_dn) + (size_t)(k * N + mu) * M * rep;
    T* dze = (up ? dzeta_up : dzeta_dn) + (size_t)(k * N + mu) * M * rep;
    for (int m = 0; m < M; ++m) {
      const T dx0 = rb[3 * i] - Rb[3 * m], dx1 = rb[3 * i + 1] - Rb[3 * m + 1], dx2 = rb[3 * i + 2] - Rb[3 * m + 2];
      const T rho = m_sqrt(Num<T>::eps() + dx0 * dx0 + dx1 * dx1 + dx2 * dx2);
      for (int et = 0; et < rep; ++et) {
        const T z = ze[m * rep + et], ex = m_exp(-m_abs(z) * rho);
        atomic_add(dpi + m * rep + et, gb * ex);
        atomic_add(dze + m * rep + et, gb * pi[m * rep + et] * ex * (-rho) * (z > T(0) ? T(1) : (z < T(0) ? T(-1) : T(0))));
      }
    }
  }
  if (!cpart) return;
  for (int idx = lane; idx < N * M; idx += 32) {
    const int i = idx / M, m = idx - i * M;
    const bool up = i < n_up;
    const T dx0 = rb[3 * i] - Rb[3 * m], dx1 = rb[3 * i + 1] - Rb[3 * m + 1], dx2 = rb[3 * i + 2] - Rb[3 * m + 2];
    const T rho = m_sqrt(Num<T>::eps() + dx0 * dx0 + dx1 * dx1 + dx2 * dx2);
    T acc = T(0);
    for (int mu = 0; mu < N; ++mu) {
      if (!full_det && (up != (mu < n_up))) continue;
      const T gb = dl * aug[mu * N2 + N + i] * bfv[i * NP + mu];
      const T* pi = (up ? pi_up : pi_dn) + ((size_t)(k * N + mu) * M + m) * rep;
      const T* ze = (up ? zeta_up : zeta_dn) + ((size_t)(k * N + mu) * M + m) * rep;
      T de = T(0);  // d env[i][mu] / d rho_im
      for (int et = 0; et < rep; ++et) {
        const T az = m_abs(ze[et]);
        de -= pi[et] * az * m_exp(-az * rho);
      }
      acc += gb * de;
    }
    const T s = acc / rho;
    T* c = cpart + (((size_t)gw * N + i) * M + m) * 3;
    c[0] = s * dx0; c[1] = s * dx1; c[2] = s * dx2;
  }
}

template <class T>
inline size_t slater_bwd_smem_per_warp(int N) { return sizeof(T) * ((size_t)N * (2 * N + 1) + (size_t)2 * N * (N + 1)); }

// Electron-nucleus features of the plain forward as a row matrix Feat[rows][F] (for dW_emb = Feat^T dX0).
template <class T>
__global__ void embed_feat_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M, int n_up,
                                  T* __restrict__ Feat, int total) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total * M) return;
  const int bi = idx / M, m = idx - bi * M, b = bi / N, i = bi - b * N;
  const int F = 4 * M + 1;
  const T* ri = r + (size_t)bi * 3;
  const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
  const T dx0 = ri[0] - Rb[3 * m], dx1 = ri[1] - Rb[3 * m + 1], dx2 = ri[2] - Rb[3 * m + 2];
  const T rho = m_sqrt(Num<T>::eps() + dx0 * dx0 + dx1 * dx1 + dx2 * dx2);
  const T g = m_log1p(rho), s = g / rho;
  T* f = Feat + (size_t)bi * F;
  f[4 * m] = g; f[4 * m + 1] = dx0 * s; f[4 * m + 2] = dx1 * s; f[4 * m + 3] = dx2 * s;
  if (m == 0) f[F - 1] = i < n_up ? T(1) : T(-1);
}


// ------------------------------------------------------------------------------------------
// Position gradients of log|psi| from the reverse pass (reference: jax.grad of wf(...).log with respect to r and R,
// force.py:96-118 make_grad_nuc_log_wf / make_grad_log_wf).  One block per walker, every sum in a fixed order.
// Phase 1, thread per (i, m): the pair cotangent c_im = d log|psi| / d d_im (d_im = r_i - R_m) into cbuf[B][N][M][3]:
//   envelopes  sum_k cpart[b][k][i][m]  (slater_bwd_kernel),
//   features   dFeat[b i][4 m .. 4 m + 3] through the Jacobian of [f(rho), d s(rho)], rho = sqrt(eps + |d|^2):
//              log_rescale 1 (Psiformer, embed_feat_kernel) f = log1p rho, s = f / rho; 0 (FermiNet) f = rho, s = 1,
//   nuclear cusp (finalize_kernel, plain distance): -sc / (den0 + |d|).
// Phase 2: grad_r[b][i] = sum_m c_im + the e-e cusp + the e-e edge features dE[b][j][i][4] (FermiNet: sender j,
// receiver i, [rho, r_i - r_j]);  grad_R[b][m] = -sum_i c_im.  grad_r / grad_R nullable.
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void pos_grad_reduce_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M, int n_up,
                                       int K, const T* __restrict__ cpart, const T* __restrict__ dFeat, int ldf, int log_rescale,
                                       const T* __restrict__ dE, int cusp_kind, T same_scale, T anti_scale,
                                       const T* __restrict__ cusp_alpha, int nuc_cusp_kind, const T* __restrict__ nuc_cusp,
                                       T* __restrict__ cbuf, T* __restrict__ grad_r, T* __restrict__ grad_R) {
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const T* rb = r + (size_t)b * N * 3;
  const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
  T* cb = cbuf + (size_t)b * N * M * 3;
  for (int idx = tid; idx < N * M; idx += nt) {
    const int i = idx / M, m = idx - i * M;
    const T d[3] = {rb[3 * i] - Rb[3 * m], rb[3 * i + 1] - Rb[3 * m + 1], rb[3 * i + 2] - Rb[3 * m + 2]};
    const T d2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
    T c[3] = {T(0), T(0), T(0)};
    for (int k = 0; k < K; ++k) {
      const T* p = cpart + ((((size_t)b * K + k) * N + i) * M + m) * 3;
      c[0] += p[0]; c[1] += p[1]; c[2] += p[2];
    }
    if (dFeat) {
      const T rho = m_sqrt(Num<T>::eps() + d2);
      const T* f = dFeat + ((size_t)b * N + i) * ldf + 4 * m;
      T fp, s, sp;  // f'(rho), s(rho), s'(rho)
      if (log_rescale) {
        const T g = m_log1p(rho);
        fp = T(1) / (T(1) + rho); s = g / rho; sp = fp / rho - g / (rho * rho);
      } else {
        fp = T(1); s = T(1); sp = T(0);
      }
      const T fd = f[1] * d[0] + f[2] * d[1] + f[3] * d[2];
      const T rad = (f[0] * fp + fd * sp) / rho;
      for (int a = 0; a < 3; ++a) c[a] += rad * d[a] + f[1 + a] * s;
    }
    if (nuc_cusp_kind != 0) {
      const T dist = m_sqrt(d2), al = nuc_cusp[0];
      const T sc = nuc_cusp[1 + m] * (nuc_cusp_kind == 1 ? al * al : T(1) / (al * al));
      const T den = (nuc_cusp_kind == 1 ? al : T(1) / al) + dist;
      const T cc = sc / (den * den) / dist;
      for (int a = 0; a < 3; ++a) c[a] += cc * d[a];
    }
    T* o = cb + ((size_t)i * M + m) * 3;
    o[0] = c[0]; o[1] = c[1]; o[2] = c[2];
  }
  __syncthreads();
  T as_ = T(1), aa_ = T(1);
  if (cusp_kind != 0) { as_ = cusp_alpha[0]; aa_ = cusp_alpha[1]; }
  for (int i = tid; grad_r && i < N; i += nt) {
    T g[3] = {T(0), T(0), T(0)};
    for (int m = 0; m < M; ++m)
      for (int a = 0; a < 3; ++a) g[a] += cb[((size_t)i * M + m) * 3 + a];
    for (int j = 0; j < N; ++j) {
      if (j == i) continue;
      const T d[3] = {rb[3 * i] - rb[3 * j], rb[3 * i + 1] - rb[3 * j + 1], rb[3 * i + 2] - rb[3 * j + 2]};
      const T rho = m_sqrt(Num<T>::eps() + d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
      if (cusp_kind != 0) {  // both cusp forms are -sc / (den0 + rho), counted once per unordered pair
        const bool same = (i < n_up) == (j < n_up);
        const T al = same ? as_ : aa_;
        const T sc = (same ? same_scale : anti_scale) * (cusp_kind == 1 ? al * al : T(1) / (al * al));
        const T den = (cusp_kind == 1 ? al : T(1) / al) + rho;
        const T cc = sc / (den * den) / rho;
        for (int a = 0; a < 3; ++a) g[a] += cc * d[a];
      }
      if (dE) {  // edge (sender j -> receiver i) carries [rho, d], edge (i -> j) [rho, -d]: rho is shared
        const T* e1 = dE + (((size_t)b * N + j) * N + i) * 4;
        const T* e2 = dE + (((size_t)b * N + i) * N + j) * 4;
        const T rr = (e1[0] + e2[0]) / rho;
        for (int a = 0; a < 3; ++a) g[a] += rr * d[a] + e1[1 + a] - e2[1 + a];
      }
    }
    T* o = grad_r + ((size_t)b * N + i) * 3;
    o[0] = g[0]; o[1] = g[1]; o[2] = g[2];
  }
  for (int m = tid; grad_R && m < M; m += nt) {
    T g[3] = {T(0), T(0), T(0)};
    for (int i = 0; i < N; ++i)
      for (int a = 0; a < 3; ++a) g[a] -= cb[((size_t)i * M + m) * 3 + a];
    T* o = grad_R + ((size_t)b * M + m) * 3;
    o[0] = g[0]; o[1] = g[1]; o[2] = g[2];
  }
}

// ------------------------------------------------------------------------------------------
// Closed-form force terms per walker (reference force.py:30-38 nuclear_force, :122-132 Q, :172-194 bare + ZVQ,
// :252-301 bare, all-electron part), one block per walker, nucleus m per thread, sums in a fixed order:
//   F_nuc[m]  = sum_{n != m} Z_m Z_n (R_m - R_n) / rho_mn^3   (eps-safe norm, physics.py:112-116)
//   bare[m]   = F_nuc[m] + Z_m sum_i d_im / |d_im|^3          (-grad_R of the Coulomb attraction, plain norm)
//   Q[m]      = Z_m sum_i d_im / |d_im|
//   zvq[m]    = F_nuc[m] + Z_m sum_i (g_i / |d| - d (d . g_i) / |d|^3),  g_i = grad_{r_i} log|psi|
// d_im = r_i - R_m.  Every output nullable.  loc[M][3][2][Tm] (nullable; dqmc_ecp_force): bare also takes -grad_R of the
// local ECP, sum_t beta_0 e^{-alpha_0 rho^2} / rho + beta_1 e^{-alpha_1 rho^2} + beta_2 rho e^{-alpha_2 rho^2} per electron
// (gaussian_type_ecp.py:127-159): -grad_{R_m} = V'(rho) d_im / rho.
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void force_terms_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M,
                                   const T* __restrict__ Z, const T* __restrict__ grad_r, T* __restrict__ bare,
                                   T* __restrict__ zvq, T* __restrict__ Qo, const T* __restrict__ loc, int Tm) {
  const int b = blockIdx.x;
  const T* rb = r + (size_t)b * N * 3;
  const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
  const T* gb = grad_r ? grad_r + (size_t)b * N * 3 : nullptr;
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    const T zm = Z[m];
    T fn[3] = {T(0), T(0), T(0)};
    for (int n = 0; n < M; ++n) {
      if (n == m) continue;
      const T d[3] = {Rb[3 * m] - Rb[3 * n], Rb[3 * m + 1] - Rb[3 * n + 1], Rb[3 * m + 2] - Rb[3 * n + 2]};
      const T rho = m_sqrt(Num<T>::eps() + d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
      const T s = zm * Z[n] / (rho * rho * rho);
      for (int a = 0; a < 3; ++a) fn[a] += s * d[a];
    }
    T fb[3] = {T(0), T(0), T(0)}, q[3] = {T(0), T(0), T(0)}, fz[3] = {T(0), T(0), T(0)}, fl[3] = {T(0), T(0), T(0)};
    for (int i = 0; i < N; ++i) {
      const T d[3] = {rb[3 * i] - Rb[3 * m], rb[3 * i + 1] - Rb[3 * m + 1], rb[3 * i + 2] - Rb[3 * m + 2]};
      const T dist = m_sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), inv = T(1) / dist, inv3 = inv * inv * inv;
      T dg = T(0);
      if (gb) dg = d[0] * gb[3 * i] + d[1] * gb[3 * i + 1] + d[2] * gb[3 * i + 2];
      for (int a = 0; a < 3; ++a) {
        fb[a] += d[a] * inv3;
        q[a] += d[a] * inv;
        if (gb) fz[a] += gb[3 * i + a] * inv - d[a] * dg * inv3;
      }
      if (loc) {
        const T* lp = loc + (size_t)m * 6 * Tm;  // [r^-1, r^0, r^1][alpha, beta][t]
        T dv = T(0);
        for (int t = 0; t < Tm; ++t) {
          const T a0 = lp[t], b0 = lp[Tm + t], a1 = lp[2 * Tm + t], b1 = lp[3 * Tm + t], a2 = lp[4 * Tm + t], b2 = lp[5 * Tm + t];
          const T d2 = dist * dist;
          dv += b0 * m_exp(-a0 * d2) * (-inv * inv - T(2) * a0) - T(2) * a1 * dist * b1 * m_exp(-a1 * d2) +
                b2 * m_exp(-a2 * d2) * (T(1) - T(2) * a2 * d2);
        }
        for (int a = 0; a < 3; ++a) fl[a] += dv * inv * d[a];
      }
    }
    const size_t o = ((size_t)b * M + m) * 3;
    for (int a = 0; a < 3; ++a) {
      if (bare) bare[o + a] = loc ? fn[a] + zm * fb[a] + fl[a] : fn[a] + zm * fb[a];
      if (Qo) Qo[o + a] = zm * q[a];
      if (zvq) zvq[o + a] = fn[a] + zm * fz[a];
    }
  }
}

// ==========================================================================================
// conv-GNN ("PauliNet" test ansatz, tests/conf/ansatz.yaml) reverse pass, plain-forward VALUE layouts:
//   edge features E[b][i][jj][4] (receiver i, sender jj < N electron / jj >= N nucleus), filters W_t[b][i][jj][e],
//   node transforms H_t[b][j][e], convolutions C[b][i][t e + f] for t = same, anti, ne.
// ==========================================================================================
template <class T>
__global__ void gnn_edge_val_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M, int Mne,
                                    T* __restrict__ E, int total, int self_edges) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int NS = N + Mne;
  const int jj = idx % NS, i = (idx / NS) % N, b = idx / (NS * N);
  T* out = E + (size_t)idx * 4;
  out[0] = out[1] = out[2] = out[3] = T(0);
  if (jj == i) {
    if (self_edges) out[0] = m_sqrt(Num<T>::eps());  // self-interaction edge: |0| eps-safe (gnn_edge_feat_kernel)
    return;
  }
  const T* ri = r + ((size_t)b * N + i) * 3;
  const T* pj = jj >= N ? R + (R_batched ? (size_t)b * M * 3 : 0) + (size_t)(jj - N) * 3 : r + ((size_t)b * N + jj) * 3;
  const T d0 = ri[0] - pj[0], d1 = ri[1] - pj[1], d2 = ri[2] - pj[2];
  out[0] = m_sqrt(Num<T>::eps() + d0 * d0 + d1 * d1 + d2 * d2);
  out[1] = d0; out[2] = d1; out[3] = d2;
}

// C[b][i][t e + f] = sum_senders W_t[b][i][jj][f] * H_t(sender)[f]   (update_features.py:196-209, no normalisation)
template <class T>
__global__ void gnn_conv_val_kernel(const T* __restrict__ Wsame, const T* __restrict__ Wanti, const T* __restrict__ Wne,
                                    const T* __restrict__ Hs, const T* __restrict__ Ha, const T* __restrict__ Hne, int N,
                                    int M, int n_up, int e, T* __restrict__ C) {
  const int bi = blockIdx.x, b = bi / N, i = bi - b * N;
  const int NS = N + M, nt = M > 0 ? 3 : 2;
  for (int f = threadIdx.x; f < e; f += blockDim.x) {
    T as = T(0), aa = T(0), an = T(0);
    for (int j = 0; j < N; ++j) {
      if (j == i) continue;
      const bool same = (i < n_up) == (j < n_up);
      const size_t p = ((size_t)bi * NS + j) * e + f;
      const T v = (same ? Wsame : Wanti)[p] * (same ? Hs : Ha)[((size_t)b * N + j) * e + f];
      if (same) as += v; else aa += v;
    }
    for (int m = 0; m < M; ++m) an += Wne[((size_t)bi * NS + N + m) * e + f] * Hne[m * e + f];
    T* c = C + (size_t)bi * nt * e;
    c[f] = as; c[e + f] = aa;
    if (nt == 3) c[2 * e + f] = an;
  }
}

// Backward of gnn_conv_val_kernel.  dW_t is written for EVERY pair (zero where the pair is not of type t), dH_t / dHne
// are accumulated atomically (callers zero them).  Block per (walker, receiver).
template <class T>
__global__ void gnn_conv_bwd_kernel(const T* __restrict__ dC, const T* __restrict__ Wsame, const T* __restrict__ Wanti,
                                    const T* __restrict__ Wne, const T* __restrict__ Hs, const T* __restrict__ Ha,
                                    const T* __restrict__ Hne, int N, int M, int n_up, int e, T* __restrict__ dWsame,
                                    T* __restrict__ dWanti, T* __restrict__ dWne, T* __restrict__ dHs, T* __restrict__ dHa,
                                    T* __restrict__ dHne) {
  const int bi = blockIdx.x, b = bi / N, i = bi - b * N;
  const int NS = N + M, nt = M > 0 ? 3 : 2;
  for (int f = threadIdx.x; f < e; f += blockDim.x) {
    const T* dc = dC + (size_t)bi * nt * e;
    const T gs = dc[f], ga = dc[e + f], gn = nt == 3 ? dc[2 * e + f] : T(0);
    for (int jj = 0; jj < NS; ++jj) {
      const size_t p = ((size_t)bi * NS + jj) * e + f;
      T ws = T(0), wa = T(0), wn = T(0);
      if (jj < N && jj != i) {
        const size_t hj = ((size_t)b * N + jj) * e + f;
        if ((i < n_up) == (jj < n_up)) { ws = gs * Hs[hj]; atomic_add(dHs + hj, gs * Wsame[p]); }
        else { wa = ga * Ha[hj]; atomic_add(dHa + hj, ga * Wanti[p]); }
      } else if (jj >= N) {
        wn = gn * Hne[(jj - N) * e + f];
        atomic_add(dHne + (jj - N) * e + f, gn * Wne[p]);
      }
      dWsame[p] = ws; dWanti[p] = wa;
      if (nt == 3) dWne[p] = wn;
    }
  }
}

// DeepErwin convolutions on the value layouts (kernels_gnn.cuh gnn_conv_kernel with S = 1): C[b][i][:] =
// [conv_same + conv_anti (e) | conv_ne (ene)], the same-spin sum over j = i too with self_edges; the ne filter is the ne
// edge stream Ene (row stride ldne), Hne[M][ene].
template <class T>
__global__ void gnn_conv_val_dw_kernel(const T* __restrict__ Wsame, const T* __restrict__ Wanti, const T* __restrict__ Ene,
                                       int ldne, int ene, const T* __restrict__ Hs, const T* __restrict__ Ha,
                                       const T* __restrict__ Hne, int N, int M, int n_up, int e, int self_edges,
                                       T* __restrict__ C) {
  const int bi = blockIdx.x, b = bi / N, i = bi - b * N;
  const int NS = N + M, dc = e + ene;
  for (int k = threadIdx.x; k < dc; k += blockDim.x) {
    T acc = T(0);
    if (k < e) {
      for (int j = 0; j < N; ++j) {
        if (j == i && !self_edges) continue;
        const bool same = (i < n_up) == (j < n_up);
        acc += (same ? Wsame : Wanti)[((size_t)bi * NS + j) * e + k] * (same ? Hs : Ha)[((size_t)b * N + j) * e + k];
      }
    } else {
      const int f = k - e;
      for (int m = 0; m < M; ++m) acc += Ene[((size_t)bi * NS + N + m) * ldne + f] * Hne[m * ene + f];
    }
    C[(size_t)bi * dc + k] = acc;
  }
}

// Backward of gnn_conv_val_dw_kernel.  dW_same / dW_anti are written for every pair (zero where the pair is not of that
// type); dEne (nullable: nothing upstream) is INCREASED on the ne rows by dconv_ne * Hne -- the identity filter hands its
// cotangent to the ne edge stream; dH_* / dHne are accumulated atomically (callers zero them).  Block per (walker, receiver).
template <class T>
__global__ void gnn_conv_bwd_dw_kernel(const T* __restrict__ dC, const T* __restrict__ Wsame, const T* __restrict__ Wanti,
                                       const T* __restrict__ Ene, int ldne, int ene, const T* __restrict__ Hs,
                                       const T* __restrict__ Ha, const T* __restrict__ Hne, int N, int M, int n_up, int e,
                                       int self_edges, T* __restrict__ dWsame, T* __restrict__ dWanti, T* __restrict__ dEne,
                                       T* __restrict__ dHs, T* __restrict__ dHa, T* __restrict__ dHne) {
  const int bi = blockIdx.x, b = bi / N, i = bi - b * N;
  const int NS = N + M, dc = e + ene;
  const T* dc_ = dC + (size_t)bi * dc;
  for (int f = threadIdx.x; f < e; f += blockDim.x) {
    const T g = dc_[f];
    for (int jj = 0; jj < NS; ++jj) {
      const size_t p = ((size_t)bi * NS + jj) * e + f;
      T ws = T(0), wa = T(0);
      if (jj < N && (jj != i || self_edges)) {
        const size_t hj = ((size_t)b * N + jj) * e + f;
        if ((i < n_up) == (jj < n_up)) { ws = g * Hs[hj]; atomic_add(dHs + hj, g * Wsame[p]); }
        else { wa = g * Ha[hj]; atomic_add(dHa + hj, g * Wanti[p]); }
      }
      dWsame[p] = ws; dWanti[p] = wa;
    }
  }
  for (int f = threadIdx.x; f < ene; f += blockDim.x) {
    const T g = dc_[e + f];
    for (int m = 0; m < M; ++m) {
      const size_t p = ((size_t)bi * NS + N + m) * ldne + f;
      if (dEne) dEne[p] += g * Hne[m * ene + f];
      atomic_add(dHne + m * ene + f, g * Ene[p]);
    }
  }
}

// Backward of gnn_edge_select_kernel (kernels_gnn.cuh) on the value layout [pairs][e]: dU_t = s_t dE' on the pairs of type
// t (zero elsewhere), and dE += isq2 dE' on the pairs whose type kept the residual (dE nullable).
template <class T>
__global__ void gnn_edge_select_bwd_kernel(const T* __restrict__ dEn, int N, int M, int n_up, int e, int res_mask, T scale,
                                           T* __restrict__ dU0, T* __restrict__ dU1, T* __restrict__ dU2, T* __restrict__ dE,
                                           size_t n) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const int NS = N + M;
  const size_t pair = idx / e;
  const int jj = (int)(pair % NS), i = (int)((pair / NS) % N);
  const int t = jj >= N ? 2 : (((i < n_up) == (jj < n_up)) ? 0 : 1);
  const bool res = (res_mask >> t) & 1;
  const T g = dEn[idx], gu = res ? scale * g : g;
  dU0[idx] = t == 0 ? gu : T(0);
  dU1[idx] = t == 1 ? gu : T(0);
  if (dU2) dU2[idx] = t == 2 ? gu : T(0);
  if (dE && res) dE[idx] += scale * g;
}

// In-place backward of an activation from its stored OUTPUT y: dZ = dY f'(z).  kind 0 tanh (1 - y^2); 1 ssp = softplus + log(1/2)
// (sigmoid(z) = 1 - exp(-y) / 2); 2 the backflow's 1 + 2 tanh(z / 4) ((1 - t^2) / 2, t = (y - 1) / 2).
template <class T>
__global__ void act_bwd_kernel(T* __restrict__ dY, const T* __restrict__ Y, int kind, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const T y = Y[i];
  T d;
  if (kind == 0) d = T(1) - y * y;
  else if (kind == 1) d = T(1) - T(0.5) * m_exp(-y);
  else { const T t = T(0.5) * (y - T(1)); d = T(0.5) * (T(1) - t * t); }
  dY[i] *= d;
}

// hk.Embed lookup backward: dTable[type(i)][f] += sum_b dX[b][i][f]
template <class T>
__global__ void embed_table_bwd_kernel(const T* __restrict__ dX, int n_types, int N, int n_up, int d, int rows,
                                       T* __restrict__ dTable) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= d) return;
  T a0 = T(0), a1 = T(0);
  for (int row = blockIdx.y; row < rows; row += gridDim.y) {
    const int i = row % N;
    const T v = dX[(size_t)row * d + f];
    if (n_types > 1 && i >= n_up) a1 += v; else a0 += v;
  }
  atomic_add(dTable + f, a0);
  if (n_types > 1) atomic_add(dTable + d + f, a1);
}

// dX[b][i][f] += dJ[b][f]   (backward of the sum over electrons feeding the Jastrow, wf/omni.py:35-37)
template <class T>
__global__ void bcast_add_kernel(const T* __restrict__ dJ, int N, int d, T* __restrict__ dX, size_t total) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const size_t row = idx / d;
  dX[idx] += dJ[(row / N) * d + (idx - row * d)];
}

// dst[row][c] = src[row][off + c]   (column slice of a row-major matrix)
template <class T>
__global__ void slice_cols_kernel(const T* __restrict__ src, int lds, int off, int cols, T* __restrict__ dst, size_t total) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const size_t row = idx / cols;
  dst[idx] = src[row * lds + off + (idx - row * cols)];
}

}  // namespace dq

