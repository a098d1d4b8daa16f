// Determinant tail of the wave function with forward-Laplacian propagation:
// envelopes (x) backflow -> K signed log-determinants (+ gradient, Laplacian) -> exp-normalised
// determinant sum, e-e cusp, Coulomb / local-ECP potentials, local-energy assembly.
#pragma once
#include "common.cuh"

namespace dq {

// ------------------------------------------------------------------------------------------
// One block per (walker b, determinant k).
//   A[i][mu] = env_k[i][mu] * bf_k[i][mu]
//   reference: src/deepqmc/wf/env.py:57-75 (phi = sum_m pi exp(-|zeta| |r_i - R_m|), eps-safe
//   norm), wf/nn_wave_function.py:111-151 (multiplicative backflow with mult_act = identity,
//   full determinant, jnp.linalg.slogdet = partial-pivot LU sign/log convention).
//   d_t log|det A| = tr(A^-1 A^t);  lap log|det A| = tr(A^-1 A^L) - sum_t tr((A^-1 A^t)^2)
// BF: augmented rows [b][i][s][K*N] (orbital index k*N + mu, wf/omni.py:78-88).
// Every Slater kernel below follows slogdet's convention for an exactly singular A (a zero pivot: a zero orbital column or
// electron row, or an envelope flushed to zero): no division by the zero pivot, sign 0 and log -inf.  A^-1 does not exist
// there, so the gradient and Laplacian outputs of such a determinant carry no meaning (the determinant sum weighs them by
// exp(-inf) = 0).
// ------------------------------------------------------------------------------------------
// lane-strided walk over a rows x cols index space without per-item division
struct LaneWalk {
  int i, j, qi, qj, cols;
  __device__ __forceinline__ LaneWalk(int lane, int cols_) : cols(cols_) {
    i = lane / cols_; j = lane - i * cols_; qi = 32 / cols_; qj = 32 - qi * cols_;
  }
  __device__ __forceinline__ void next() {
    j += qj; i += qi;
    if (j >= cols) { j -= cols; ++i; }
  }
};

// ------------------------------------------------------------------------------------------
// Additive backflow branch of the BackflowOp (reference wf/nn_wave_function.py:14-33):
//   xs <- xs * mult_act(f_mult) + cutoff(r_i) * envel_i * add_act(f_add),
//   envel_i = sqrt(sum_{k, mu} xs[k, i, mu]^2) over the determinants and the orbitals of electron i's spin block,
//   cutoff = R^2 (6 - 8 R + 3 R^2) for R = min_I |r_i - R_I| / 0.5 < 1, else 1.
// This kernel evaluates the electron-local factor g_i = cutoff * envel with its gradient and Laplacian w.r.t. r_i:
// G[b][i][5] = (g, dg/dx, dg/dy, dg/dz, Lap g).  One thread per (walker, electron).
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void bf_add_factor_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M, int n_up,
                                     int K, const T* __restrict__ pi_up, const T* __restrict__ pi_dn,
                                     const T* __restrict__ zeta_up, const T* __restrict__ zeta_dn, int rep, int full_det,
                                     T* __restrict__ G, int total) {
  const int bi = blockIdx.x * blockDim.x + threadIdx.x;
  if (bi >= total) return;
  const int b = bi / N, i = bi - b * N;
  const T* ri = r + (size_t)bi * 3;
  const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
  const bool up = i < n_up;
  const int mu0 = full_det ? 0 : (up ? 0 : n_up), mu1 = full_det ? N : (up ? n_up : N);
  T S = T(0), gS0 = T(0), gS1 = T(0), gS2 = T(0), lS = T(0);
  for (int k = 0; k < K; ++k)
    for (int mu = mu0; mu < mu1; ++mu) {
      const T* pi = (up ? pi_up : pi_dn) + (size_t)(k * N + mu) * M * rep;
      const T* ze = (up ? zeta_up : zeta_dn) + (size_t)(k * N + mu) * M * rep;
      T e = T(0), d0 = T(0), d1 = T(0), d2 = T(0), le = T(0);
      for (int m = 0; m < M; ++m) {
        const T dx0 = ri[0] - Rb[3 * m], dx1 = ri[1] - Rb[3 * m + 1], dx2 = ri[2] - Rb[3 * m + 2];
        const T dd = dx0 * dx0 + dx1 * dx1 + dx2 * dx2;
        const T rho2 = Num<T>::eps() + dd, rho = m_sqrt(rho2);
        for (int et = 0; et < rep; ++et) {
          const T a = m_abs(ze[m * rep + et]);
          const T ex = pi[m * rep + et] * m_exp(-a * rho);
          const T c = -a * ex / rho;
          e += ex;
          d0 += c * dx0; d1 += c * dx1; d2 += c * dx2;
          le += ex * (a * a * dd / rho2 - a * (T(3) / rho - dd / (rho2 * rho)));
        }
      }
      S += e * e;
      gS0 += T(2) * e * d0; gS1 += T(2) * e * d1; gS2 += T(2) * e * d2;
      lS += T(2) * (d0 * d0 + d1 * d1 + d2 * d2 + e * le);
    }
  const T n = m_sqrt(S);
  const T n0 = gS0 / (T(2) * n), n1 = gS1 / (T(2) * n), n2 = gS2 / (T(2) * n);
  const T ln = lS / (T(2) * n) - (gS0 * gS0 + gS1 * gS1 + gS2 * gS2) / (T(4) * S * n);
  // cutoff on the plain distance to the nearest nucleus
  T best = T(-1), c0 = T(0), c1 = T(0), c2 = T(0);
  for (int m = 0; m < M; ++m) {
    const T dx0 = ri[0] - Rb[3 * m], dx1 = ri[1] - Rb[3 * m + 1], dx2 = ri[2] - Rb[3 * m + 2];
    const T dd = dx0 * dx0 + dx1 * dx1 + dx2 * dx2;
    if (best < T(0) || dd < best) { best = dd; c0 = dx0; c1 = dx1; c2 = dx2; }
  }
  const T rho = m_sqrt(best), Rr = rho * T(2);
  T c = T(1), cg0 = T(0), cg1 = T(0), cg2 = T(0), cl = T(0);
  if (Rr < T(1)) {
    c = Rr * Rr * (T(6) - T(8) * Rr + T(3) * Rr * Rr);
    const T cp = T(12) * Rr * (T(1) - Rr) * (T(1) - Rr) * T(2);            // dc/drho
    const T cpp = (T(12) - T(48) * Rr + T(36) * Rr * Rr) * T(4);           // d2c/drho2
    cg0 = cp * c0 / rho; cg1 = cp * c1 / rho; cg2 = cp * c2 / rho;
    cl = cpp + T(2) * cp / rho;
  }
  T* g = G + (size_t)bi * 5;
  g[0] = c * n;
  g[1] = c * n0 + n * cg0; g[2] = c * n1 + n * cg1; g[3] = c * n2 + n * cg2;
  g[4] = c * ln + T(2) * (cg0 * n0 + cg1 * n1 + cg2 * n2) + n * cl;
}

template <class T>
__global__ void slater_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M, int n_up,
                              int K, int S, int total, const T* __restrict__ pi_up, const T* __restrict__ pi_dn,
                              const T* __restrict__ zeta_up, const T* __restrict__ zeta_dn,
                              const T* __restrict__ BF, int ldb, T* __restrict__ det_sign, T* __restrict__ det_log,
                              T* __restrict__ det_grad, T* __restrict__ det_lap, int rep, int full_det,
                              const T* __restrict__ QA, const T* __restrict__ Gadd, int add_off, int mult_on) {
  // QA != null: pseudo-Hamiltonian metric per electron (common.cuh PhMetric; tangent slots are v-coordinates)
  // Gadd != null: additive backflow branch, A = env * bf_mult (mult_on) + g_i * bf_add with g from bf_add_factor_kernel and
  // the (already activated) additive head at column offset add_off of BF
  // full_det == 0: spin-factorised determinants det_up(n_up x n_up) det_down(n_down x n_down) (reference
  // wf/nn_wave_function.py:143-151) = determinant of the matrix with the spin-off-diagonal blocks zeroed.
  // rep = envelope terms per nucleus (1: ExponentialEnvelopes; 3: SimplifiedNucleusDependentEnvelopes,
  // reference wf/env.py:111-226): parameter rows are [K N][M rep], term m rep + e sits on nucleus m.
  // One WARP per (walker b, determinant k): all phases are lane-strided loops separated by
  // __syncwarp, reductions are warp shuffles (no block barriers: N <= ~40 electrons).
  DQMC_DYN_SMEM(smem_raw);
  const int NP = N + 1, N2 = 2 * N + 1;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int gw = blockIdx.x * wpb + wib;
  const size_t per_warp = (size_t)7 * N * NP + (size_t)N * N2 + N;
  T* env = reinterpret_cast<T*>(smem_raw) + per_warp * wib;  // [N][NP]
  T* denv = env + N * NP;                                     // [3][N][NP]
  T* bfv = denv + 3 * N * NP;                                 // [N][NP]
  T* AL = bfv + N * NP;                                       // [N][NP]  (reused as B^t)
  T* At = AL + N * NP;                                        // [N][NP]
  T* aug = At + N * NP;                                       // [N][N2]
  T* fcol = aug + N * N2;                                     // [N]
  if (gw >= total) return;
  const int b = gw / K, k = gw % K;
  const int T3 = S > 1 ? S - 2 : 0;
  const T* rb = r + (size_t)b * N * 3;
  const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
  const size_t brow0 = (size_t)b * N * S;

  for (LaneWalk w(lane, N); w.i < N; w.next()) {
    const int i = w.i, mu = w.j;
    const T* pi = (i < n_up ? pi_up : pi_dn) + (size_t)(k * N + mu) * M * rep;
    const T* ze = (i < n_up ? zeta_up : zeta_dn) + (size_t)(k * N + mu) * M * rep;
    T e = 0, de0 = 0, de1 = 0, de2 = 0, le = 0;
    PhMetric<T> pm;
    if (QA) pm.load(QA + ((size_t)b * N + i) * PH_STRIDE);
    for (int m = 0; m < M; ++m) {
      T dx0 = rb[3 * i] - Rb[3 * m], dx1 = rb[3 * i + 1] - Rb[3 * m + 1], dx2 = rb[3 * i + 2] - Rb[3 * m + 2];
      T d2 = dx0 * dx0 + dx1 * dx1 + dx2 * dx2;
      T rho2 = Num<T>::eps() + d2, rho = m_sqrt(rho2);
      T gr2 = d2 / rho2, lr = T(3) / rho - d2 / (rho2 * rho);  // |grad rho|^2, laplacian rho
      if (QA && S > 1) {
        T a0, a1, a2;
        pm.mul(dx0 / rho, dx1 / rho, dx2 / rho, a0, a1, a2);
        gr2 = (dx0 * a0 + dx1 * a1 + dx2 * a2) / rho;
        lr = (pm.trace() - gr2) / rho;
      }
      for (int et = 0; et < rep; ++et) {
        T a = m_abs(ze[m * rep + et]);
        T ex = pi[m * rep + et] * m_exp(-a * rho);
        e += ex;
        if (S > 1) {
          T c = -a * ex / rho;
          de0 += c * dx0; de1 += c * dx1; de2 += c * dx2;
          le += ex * (a * a * gr2 - a * lr);
        }
      }
    }
    if (QA && S > 1) pm.to_v(de0, de1, de2);
    if (!full_det && ((i < n_up) != (mu < n_up))) { e = T(0); de0 = T(0); de1 = T(0); de2 = T(0); le = T(0); }
    const T* bfrow = BF + (brow0 + (size_t)i * S) * ldb + k * N + mu;
    T bf0 = mult_on ? bfrow[0] : T(1);
    const bool blocked = !full_det && ((i < n_up) != (mu < n_up));
    const T* ga = Gadd ? Gadd + ((size_t)b * N + i) * 5 : nullptr;
    T a0 = e * bf0;
    if (ga && !blocked) a0 += ga[0] * bfrow[add_off];
    env[i * NP + mu] = e;
    bfv[i * NP + mu] = bf0;
    aug[i * N2 + mu] = a0;
    aug[i * N2 + N + mu] = (i == mu) ? T(1) : T(0);
    if (S > 1) {
      denv[(0 * N + i) * NP + mu] = de0;
      denv[(1 * N + i) * NP + mu] = de1;
      denv[(2 * N + i) * NP + mu] = de2;
      T al = le * bf0;
      if (mult_on) {
        T bfl = bfrow[(size_t)(1 + T3) * ldb];
        T x0 = bfrow[(size_t)(1 + 3 * i) * ldb], x1 = bfrow[(size_t)(2 + 3 * i) * ldb], x2 = bfrow[(size_t)(3 + 3 * i) * ldb];
        al += e * bfl + T(2) * (de0 * x0 + de1 * x1 + de2 * x2);
      }
      if (ga && !blocked) {
        const T* yr = bfrow + add_off;
        al += ga[4] * yr[0] + ga[0] * yr[(size_t)(1 + T3) * ldb] +
              T(2) * (ga[1] * yr[(size_t)(1 + 3 * i) * ldb] + ga[2] * yr[(size_t)(2 + 3 * i) * ldb] + ga[3] * yr[(size_t)(3 + 3 * i) * ldb]);
      }
      AL[i * NP + mu] = al;
    }
  }
  __syncwarp();

  // ---- Gauss-Jordan with partial pivoting on [A | I] (pivots == LU with partial pivoting) -----
  T logdet = T(0), sgn = T(1);
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
    const T pv = aug[c * N2 + c];
    logdet += m_log(m_abs(pv));
    T sg = pv > T(0) ? T(1) : (pv < T(0) ? T(-1) : T(0));
    sgn *= (prow != c ? -sg : sg);
    for (int rr = lane; rr < N; rr += 32) fcol[rr] = aug[rr * N2 + c];
    __syncwarp();
    // an exactly singular matrix (the whole remaining column is zero): no division by the zero pivot -- the pivot row is
    // scaled to zero, so the elimination below changes nothing -- and (sign 0, log -inf) as slogdet gives
    const T ipv = pv != T(0) ? T(1) / pv : T(0);
    for (int j = lane; j < 2 * N; j += 32) aug[c * N2 + j] *= ipv;
    __syncwarp();
    for (LaneWalk w(lane, 2 * N); w.i < N; w.next()) {
      const int rr = w.i, j = w.j;
      if (rr != c) aug[rr * N2 + j] -= fcol[rr] * aug[c * N2 + j];
    }
    __syncwarp();
  }
  const size_t bk = (size_t)b * K + k;
  if (lane == 0) { det_log[bk] = logdet; det_sign[bk] = sgn; }
  if (S == 1) return;

  // Ainv[mu][i] = aug[mu][N + i]
  T lap = T(0);
  for (LaneWalk w(lane, N); w.i < N; w.next()) {
    const int i = w.i, mu = w.j;
    lap += aug[mu * N2 + N + i] * AL[i * NP + mu];
  }
  lap = warp_sum(lap);
  T* Bt = AL;  // A^L no longer needed
  for (int t = 0; t < T3; ++t) {
    const int it = t / 3, ct = t % 3;
    __syncwarp();
    for (LaneWalk w(lane, N); w.i < N; w.next()) {
      const int i = w.i, mu = w.j;
      const T* bft_p = BF + (brow0 + (size_t)i * S + 1 + t) * ldb + k * N + mu;
      T a = mult_on ? env[i * NP + mu] * bft_p[0] : T(0);
      if (i == it) a += denv[(ct * N + i) * NP + mu] * bfv[i * NP + mu];
      if (Gadd && (full_det || ((i < n_up) == (mu < n_up)))) {
        const T* ga = Gadd + ((size_t)b * N + i) * 5;
        a += ga[0] * bft_p[add_off];
        if (i == it) a += ga[1 + ct] * BF[(brow0 + (size_t)i * S) * ldb + k * N + mu + add_off];
      }
      At[i * NP + mu] = a;
    }
    __syncwarp();
    for (LaneWalk w(lane, N); w.i < N; w.next()) {
      const int mu = w.i, nu = w.j;
      T a = T(0);
      for (int i = 0; i < N; ++i) a += aug[mu * N2 + N + i] * At[i * NP + nu];
      Bt[mu * NP + nu] = a;
    }
    __syncwarp();
    T tr2 = T(0), gt = T(0);
    for (LaneWalk w(lane, N); w.i < N; w.next()) {
      const int mu = w.i, nu = w.j;
      tr2 += Bt[mu * NP + nu] * Bt[nu * NP + mu];
      if (mu == nu) gt += Bt[mu * NP + mu];
    }
    tr2 = warp_sum(tr2);
    gt = warp_sum(gt);
    lap -= tr2;
    if (lane == 0) det_grad[bk * T3 + t] = gt;
  }
  if (lane == 0) det_lap[bk] = lap;
}

template <class T>
inline size_t slater_smem_per_warp(int N) {
  return sizeof(T) * ((size_t)7 * N * (N + 1) + (size_t)N * (2 * N + 1) + N);
}
// warps per block: as many as fit ~96 KB (two blocks per SM), at most 8
template <class T>
inline int slater_warps_per_block(int N) {
  size_t pw = slater_smem_per_warp<T>(N);
  int w = (int)((96 * 1024) / pw);
  return w < 1 ? 1 : (w > 8 ? 8 : w);
}
template <class T>
inline size_t slater_smem_bytes(int N) {
  return slater_smem_per_warp<T>(N) * slater_warps_per_block<T>(N);
}

// ------------------------------------------------------------------------------------------
// Small molecules (N = NS <= 6 electrons, compile time): ONE THREAD per (walker, determinant),
// the NS x NS matrix, its inverse and all per-tangent products live in registers (fully unrolled).
// Same algebra as slater_kernel (envelopes, Gauss-Jordan with partial pivoting, tr(A^-1 dA),
// tr((A^-1 dA)^2)); used for both S = 1 and the forward-Laplacian pass.
// ------------------------------------------------------------------------------------------
template <class T, int NS>
__global__ void slater_small_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int M, int n_up,
                                    int K, int S, int total, const T* __restrict__ pi_up, const T* __restrict__ pi_dn,
                                    const T* __restrict__ zeta_up, const T* __restrict__ zeta_dn,
                                    const T* __restrict__ BF, int ldb, T* __restrict__ det_sign,
                                    T* __restrict__ det_log, T* __restrict__ det_grad, T* __restrict__ det_lap,
                                    int rep, int full_det) {
  const int gid = blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= total) return;
  const int b = gid / K, k = gid % K;
  const int T3 = S > 1 ? S - 2 : 0;
  const T* rb = r + (size_t)b * NS * 3;
  const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
  const size_t brow0 = (size_t)b * NS * S;
  T env[NS][NS], de[3][NS][NS], bf0[NS][NS], A[NS][NS], Ai[NS][NS], AL[NS][NS];
#pragma unroll
  for (int i = 0; i < NS; ++i) {
    const T* pi_s = i < n_up ? pi_up : pi_dn;
    const T* ze_s = i < n_up ? zeta_up : zeta_dn;
#pragma unroll
    for (int mu = 0; mu < NS; ++mu) {
      const T* pi = pi_s + (size_t)(k * NS + mu) * M * rep;
      const T* ze = ze_s + (size_t)(k * NS + mu) * M * rep;
      T e = 0, d0 = 0, d1 = 0, d2_ = 0, le = 0;
      for (int m = 0; m < M; ++m) {
        T dx0 = rb[3 * i] - Rb[3 * m], dx1 = rb[3 * i + 1] - Rb[3 * m + 1], dx2 = rb[3 * i + 2] - Rb[3 * m + 2];
        T dd = dx0 * dx0 + dx1 * dx1 + dx2 * dx2;
        T rho2 = Num<T>::eps() + dd, rho = m_sqrt(rho2);
        for (int et = 0; et < rep; ++et) {
          T a = m_abs(ze[m * rep + et]);
          T ex = pi[m * rep + et] * m_exp(-a * rho);
          e += ex;
          if (S > 1) {
            T c = -a * ex / rho;
            d0 += c * dx0; d1 += c * dx1; d2_ += c * dx2;
            le += ex * (a * a * dd / rho2 - a * (T(3) / rho - dd / (rho2 * rho)));
          }
        }
      }
      if (!full_det && ((i < n_up) != (mu < n_up))) { e = T(0); d0 = T(0); d1 = T(0); d2_ = T(0); le = T(0); }
      const T* bfrow = BF + (brow0 + (size_t)i * S) * ldb + k * NS + mu;
      const T b0 = bfrow[0];
      env[i][mu] = e; bf0[i][mu] = b0;
      de[0][i][mu] = d0; de[1][i][mu] = d1; de[2][i][mu] = d2_;
      A[i][mu] = e * b0;
      Ai[i][mu] = (i == mu) ? T(1) : T(0);
      AL[i][mu] = T(0);
      if (S > 1) {
        const T bfl = bfrow[(size_t)(1 + T3) * ldb];
        const T x0 = bfrow[(size_t)(1 + 3 * i) * ldb], x1 = bfrow[(size_t)(2 + 3 * i) * ldb], x2 = bfrow[(size_t)(3 + 3 * i) * ldb];
        AL[i][mu] = le * b0 + e * bfl + T(2) * (d0 * x0 + d1 * x1 + d2_ * x2);
      }
    }
  }
  // Gauss-Jordan with partial pivoting on [A | I]
  T logdet = T(0), sgn = T(1);
#pragma unroll
  for (int c = 0; c < NS; ++c) {
    int prow = c;
    T best = m_abs(A[c][c]);
#pragma unroll
    for (int rr = c + 1; rr < NS; ++rr) {
      T v = m_abs(A[rr][c]);
      if (v > best) { best = v; prow = rr; }
    }
#pragma unroll
    for (int rr = c + 1; rr < NS; ++rr) {
      if (rr == prow) {
#pragma unroll
        for (int j = 0; j < NS; ++j) {
          T t0 = A[c][j]; A[c][j] = A[rr][j]; A[rr][j] = t0;
          T t1 = Ai[c][j]; Ai[c][j] = Ai[rr][j]; Ai[rr][j] = t1;
        }
      }
    }
    const T pv = A[c][c];
    logdet += m_log(m_abs(pv));
    const T sg = pv > T(0) ? T(1) : (pv < T(0) ? T(-1) : T(0));
    sgn *= (prow != c ? -sg : sg);
    if (pv == T(0)) continue;  // exactly singular: no division by zero, (sign 0, log -inf) like slogdet
    const T ipv = T(1) / pv;
#pragma unroll
    for (int j = 0; j < NS; ++j) { A[c][j] *= ipv; Ai[c][j] *= ipv; }
#pragma unroll
    for (int rr = 0; rr < NS; ++rr) {
      if (rr != c) {
        const T f = A[rr][c];
#pragma unroll
        for (int j = 0; j < NS; ++j) { A[rr][j] -= f * A[c][j]; Ai[rr][j] -= f * Ai[c][j]; }
      }
    }
  }
  const size_t bk = (size_t)b * K + k;
  det_log[bk] = logdet;
  det_sign[bk] = sgn;
  if (S == 1) return;
  T lap = T(0);
#pragma unroll
  for (int i = 0; i < NS; ++i)
#pragma unroll
    for (int mu = 0; mu < NS; ++mu) lap += Ai[mu][i] * AL[i][mu];
  for (int t = 0; t < T3; ++t) {
    const int it = t / 3, ct = t % 3;
    T At[NS][NS], Bt[NS][NS];
#pragma unroll
    for (int i = 0; i < NS; ++i)
#pragma unroll
      for (int mu = 0; mu < NS; ++mu) {
        T a = env[i][mu] * BF[(brow0 + (size_t)i * S + 1 + t) * ldb + k * NS + mu];
        if (i == it) a += (ct == 0 ? de[0][i][mu] : ct == 1 ? de[1][i][mu] : de[2][i][mu]) * bf0[i][mu];
        At[i][mu] = a;
      }
    T gt = T(0), tr2 = T(0);
#pragma unroll
    for (int mu = 0; mu < NS; ++mu)
#pragma unroll
      for (int nu = 0; nu < NS; ++nu) {
        T a = T(0);
#pragma unroll
        for (int i = 0; i < NS; ++i) a += Ai[mu][i] * At[i][nu];
        Bt[mu][nu] = a;
      }
#pragma unroll
    for (int mu = 0; mu < NS; ++mu) {
      gt += Bt[mu][mu];
#pragma unroll
      for (int nu = 0; nu < NS; ++nu) tr2 += Bt[mu][nu] * Bt[nu][mu];
    }
    lap -= tr2;
    det_grad[bk * T3 + t] = gt;
  }
  det_lap[bk] = lap;
}

// ------------------------------------------------------------------------------------------
// Forward-only (S = 1) Slater kernel for N <= 32: the hot kernel of the Metropolis sweep and of
// the non-local ECP quadrature (12 N N_ecp plain forwards per walker).  One block per walker,
// one warp per determinant (looping), lane r owns matrix ROW r entirely in registers:
//   * electron-nucleus distances are computed once per walker into shared memory,
//   * A[r][mu] = (sum_m pi exp(-|zeta| rho[r][m])) * bf[r][k N + mu]  built row-wise,
//   * LU with implicit partial pivoting: per column one warp arg-max, one broadcast per remaining
//     column (shuffle) and one FMA per lane -- no shared memory, no barriers;
//   * sign = parity(pivot order) * prod sign(pivot)  (== LAPACK getrf convention of slogdet).
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void slater_fwd_reg_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M,
                                      int n_up, int K, const T* __restrict__ pi_up, const T* __restrict__ pi_dn,
                                      const T* __restrict__ zeta_up, const T* __restrict__ zeta_dn,
                                      const T* __restrict__ BF, int ldb, T* __restrict__ det_sign,
                                      T* __restrict__ det_log, int rep, int full_det) {
  constexpr int NM = 32;
  DQMC_DYN_SMEM(smem_raw);
  T* rho = reinterpret_cast<T*>(smem_raw);  // [N][M]
  const int b = blockIdx.x;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const T* rb = r + (size_t)b * N * 3;
  const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
  for (int idx = threadIdx.x; idx < N * M; idx += blockDim.x) {
    const int i = idx / M, m = idx - i * M;
    T dx0 = rb[3 * i] - Rb[3 * m], dx1 = rb[3 * i + 1] - Rb[3 * m + 1], dx2 = rb[3 * i + 2] - Rb[3 * m + 2];
    rho[idx] = m_sqrt(Num<T>::eps() + dx0 * dx0 + dx1 * dx1 + dx2 * dx2);
  }
  __syncthreads();
  const bool rowok = lane < N;
  const T* pi = (lane < n_up ? pi_up : pi_dn);
  const T* ze = (lane < n_up ? zeta_up : zeta_dn);
  for (int k = wib; k < K; k += wpb) {
    T a[NM];
#pragma unroll
    for (int mu = 0; mu < NM; ++mu) {
      T v = (mu == lane) ? T(1) : T(0);  // padding rows/columns: identity
      if (rowok && mu < N) {
        const T* pk = pi + (size_t)(k * N + mu) * M * rep;
        const T* zk = ze + (size_t)(k * N + mu) * M * rep;
        T e = T(0);
        for (int m = 0; m < M; ++m)
          for (int et = 0; et < rep; ++et) e += pk[m * rep + et] * m_exp(-m_abs(zk[m * rep + et]) * rho[lane * M + m]);
        if (!full_det && ((lane < n_up) != (mu < n_up))) e = T(0);
        v = e * BF[((size_t)b * N + lane) * ldb + k * N + mu];
      }
      a[mu] = v;
    }
    T logdet = T(0), sgn = T(1);
    unsigned used = 0u;       // rows already chosen as pivots (same value in every lane)
    unsigned long long order0 = 0, order1 = 0, order2 = 0;  // pivot row of step c, 5 bits each, 12 steps per word
#pragma unroll
    for (int c = 0; c < NM; ++c) {
      const bool mine_used = (used >> lane) & 1u;
      T best = mine_used ? T(-1) : m_abs(a[c]);
      int bi = lane;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        T ob = __shfl_xor_sync(0xffffffffu, best, o);
        int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
      }
      const int prow = bi;
      used |= 1u << prow;
      if (c < 12) order0 |= (unsigned long long)prow << (5 * c);
      else if (c < 24) order1 |= (unsigned long long)prow << (5 * (c - 12));
      else order2 |= (unsigned long long)prow << (5 * (c - 24));
      const T pv = __shfl_sync(0xffffffffu, a[c], prow);
      logdet += m_log(m_abs(pv));
      sgn *= pv > T(0) ? T(1) : (pv < T(0) ? T(-1) : T(0));
      const bool elim = !((used >> lane) & 1u);  // rows not yet used (prow itself is used now)
      const T f = (elim && pv != T(0)) ? a[c] / pv : T(0);  // exactly singular: (sign 0, log -inf) like slogdet
#pragma unroll
      for (int j = c + 1; j < NM; ++j) {
        const T pj = __shfl_sync(0xffffffffu, a[j], prow);
        a[j] -= f * pj;
      }
    }
    if (lane == 0) {
      // parity of the permutation c -> pivot row(c) by cycle counting
      int perm[NM];
#pragma unroll
      for (int c = 0; c < NM; ++c)
        perm[c] = (int)((c < 12 ? (order0 >> (5 * c)) : c < 24 ? (order1 >> (5 * (c - 12))) : (order2 >> (5 * (c - 24)))) & 31ull);
      unsigned seen = 0u;
      int transp = 0;
      for (int c = 0; c < NM; ++c) {
        if ((seen >> c) & 1u) continue;
        int len = 0, x = c;
        while (!((seen >> x) & 1u)) { seen |= 1u << x; x = perm[x]; ++len; }
        transp += len - 1;
      }
      if (transp & 1) sgn = -sgn;
      det_log[(size_t)b * K + k] = logdet;
      det_sign[(size_t)b * K + k] = sgn;
    }
  }
}

// ------------------------------------------------------------------------------------------
// Forward-only (S = 1) Slater kernel, second generation (N <= 32): persistent blocks, one walker
// per iteration, two phases per walker.
//   phase 1, thread <-> orbital o = k N + mu (coalesced over the backflow row): envelopes
//     phi_o(r_i) = sum_m pi_o,m exp(-|zeta_o,m| rho_i,m) for 8 electrons at a time (parameters are
//     loaded once per 8 electrons, rho comes from shared memory as a broadcast), times the
//     backflow entry -> A[k][i][mu] in shared memory (odd row pitch: conflict-free row reads).
//   phase 2, warp <-> determinant k, lane <-> matrix row held in registers: LU with implicit
//     partial pivoting.  Pivot search is ONE redux.sync (max over the integer image of |a|, fp32)
//     plus a ballot; the pivot row reaches the other lanes by shuffles; the permutation parity
//     is accumulated as an inversion count (popc), so nothing leaves the register file.
// Same reference lines as slater_kernel; slogdet sign/log convention = LAPACK getrf.
// dynamic smem = sizeof(T) * (K N NP + N M), NP = N | 1.
// ------------------------------------------------------------------------------------------
// exp for the envelope sums of the plain-forward kernel: ex2.approx on a Cody-Waite reduced
// argument (the product x log2(e) is split into its rounded value and the exact FMA remainder),
// ~2 ulp like expf at a third of the instructions.
__device__ __forceinline__ float env_exp(float x) {
#ifndef DQMC_EMU
  const float t = x * 1.4426950216293335f;
  float e = fmaf(x, 1.4426950216293335f, -t);
  e = fmaf(x, 1.925963033500011e-8f, e);
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(t));
  return fmaf(y * e, 0.6931471805599453f, y);
#else
  return ::expf(x);
#endif
}
__device__ __forceinline__ double env_exp(double x) { return ::exp(x); }
// Envelope terms of the plain-forward kernel with the exponent pre-scaled ONCE per (orbital, nucleus): zs = -|zeta| log2(e)
// (fp32) and exp(-|zeta| rho) = ex2.approx(zs rho): one multiply + one MUFU per term instead of the 6-instruction
// Cody-Waite form above (the kernel is issue-bound: 173 k terms per benzene walker).  Error: the rounded product x = zs rho
// is off by <= 2^-23 |x| (scale and product rounding), i.e. the term by <= |x| 2^-23 e^{-|x|} ln 2 <= 3e-8 of a unit
// coefficient for every x -- large exponents only occur in terms that are themselves tiny -- plus the 2 ulp of ex2.approx.
__device__ __forceinline__ float env_scale(float z) { return z * 1.4426950408889634f; }
__device__ __forceinline__ double env_scale(double z) { return z; }
__device__ __forceinline__ float env_exp_scaled(float xs) {
#ifndef DQMC_EMU
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(xs));
  return y;
#else
  return ::exp2f(xs);
#endif
}
__device__ __forceinline__ double env_exp_scaled(double x) { return ::exp(x); }

// log|det| = sum of log|pivot|: fp32 keeps a running mantissa product and an integer exponent sum
// (one logf at the end instead of one per pivot); pivots outside the normal range take the plain path.
template <class T>
struct LogProd {
  T acc = T(0);
  __device__ __forceinline__ void mul(T apv) { acc += m_log(apv); }
  __device__ __forceinline__ T value() const { return acc; }
};
#ifndef DQMC_EMU
template <>
struct LogProd<float> {
  float mant = 1.f, extra = 0.f;
  int esum = 0;
  __device__ __forceinline__ void mul(float apv) {
    if (apv > 1e-30f && apv < 1e30f) {  // warp-uniform (the pivot is a broadcast value)
      mant *= apv;
      const int bits = __float_as_int(mant);
      esum += (bits >> 23) - 127;
      mant = __int_as_float((bits & 0x007fffff) | 0x3f800000);
    } else {
      extra += logf(apv);
    }
  }
  __device__ __forceinline__ float value() const { return fmaf((float)esum, 0.6931471805599453f, logf(mant)) + extra; }
};
#endif
__device__ __forceinline__ float pivot_rcp(float pv) {
#ifndef DQMC_EMU
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(pv));
  return y;
#else
  return 1.f / pv;
#endif
}
__device__ __forceinline__ double pivot_rcp(double pv) { return 1.0 / pv; }

__device__ __forceinline__ int warp_argmax_abs(float v, bool excluded, int lane) {
#ifndef DQMC_EMU
  const unsigned key = excluded ? 0u : __float_as_uint(fabsf(v)) + 1u;
  const unsigned kmax = __reduce_max_sync(0xffffffffu, key);
  const unsigned bal = __ballot_sync(0xffffffffu, key == kmax);
  return __ffs(bal) - 1;
#else
  float best = excluded ? -1.f : fabsf(v);
  int bi = lane;
  for (int o = 16; o > 0; o >>= 1) {
    float ob = __shfl_xor_sync(0xffffffffu, best, o);
    int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  return bi;
#endif
}
__device__ __forceinline__ int warp_argmax_abs(double v, bool excluded, int lane) {
  double best = excluded ? -1.0 : fabs(v);
  int bi = lane;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    double ob = __shfl_xor_sync(0xffffffffu, best, o);
    int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  return bi;
}

// 8 consecutive, 8-element-aligned values from shared memory with 16-byte vector loads
__device__ __forceinline__ void load8(const float* p, float* x) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
}
__device__ __forceinline__ void load8(const double* p, double* x) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const double2 a = *reinterpret_cast<const double2*>(p + 2 * i);
    x[2 * i] = a.x; x[2 * i + 1] = a.y;
  }
}

template <class T, int NM>
__global__ void __launch_bounds__(256, 3)
slater_fwd2_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M, int n_up, int K,
                   int B, const T* __restrict__ pi_up, const T* __restrict__ pi_dn, const T* __restrict__ zeta_up,
                   const T* __restrict__ zeta_dn, const T* __restrict__ BF, int ldb, T* __restrict__ det_sign,
                   T* __restrict__ det_log, int rep, int full_det, const T* __restrict__ env_base, long long v0, int vper,
                   int vlayout, const int* __restrict__ pairs) {
  DQMC_DYN_SMEM(smem_raw);
  const int NP = N | 1, KN = K * N;
  T* As = reinterpret_cast<T*>(smem_raw);  // [K][N][NP]
  // electron-nucleus distances, one panel per spin: rho[sb][m][il], il = electron index inside the spin block, padded to a
  // multiple of 8 (the padding repeats the block's last electron) -> the 8 electrons of an envelope step are ONE aligned
  // 32-byte (fp32) / 64-byte (fp64) segment, read with vector loads instead of 8 indexed scalar loads
  const int n_dn = N - n_up;
  const int NS = (((n_up > n_dn ? n_up : n_dn) + 7) >> 3) << 3;
  T* rho = As + (((size_t)KN * NP + 3) & ~(size_t)3);  // 16-byte aligned
  const int tid = threadIdx.x, nt = blockDim.x;
  const int lane = tid & 31, wib = tid >> 5, nw = nt >> 5;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    const T* rb = r + (size_t)b * N * 3;
    const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
    __syncthreads();  // previous walker's determinants are in registers / written
    if (env_base) {
      // Compact virtual-walker forward (virtual_move, common.cuh): walker v0 + b is a base walker with one electron moved
      // (non-local ECP quadrature) or an up / down pair swapped (spin pass).  The envelopes depend on the electron's own
      // position and spin only, so all rows but the moved ones come from the base walker's table env_base[w][i][k N + mu]
      // (env_table_kernel), the moved rows are evaluated afresh with the electron's own spin: 12 M (ECP) instead of N M
      // exponentials per orbital (the envelope sums were 3/4 of this kernel's MUFU-bound first phase).
      const VirtualMove mv = virtual_move((int)(v0 + b), vper, N, n_up, vlayout, pairs);
      const int bw = mv.base, nmv = mv.e1 < 0 ? 1 : 2;
      for (int idx = tid; idx < nmv * M; idx += nt) {
        const int t = idx / M, m = idx - t * M, imv = t ? mv.e1 : mv.e0;
        const T dx0 = rb[3 * imv] - Rb[3 * m], dx1 = rb[3 * imv + 1] - Rb[3 * m + 1], dx2 = rb[3 * imv + 2] - Rb[3 * m + 2];
        rho[idx] = m_sqrt(Num<T>::eps() + dx0 * dx0 + dx1 * dx1 + dx2 * dx2);
      }
      __syncthreads();
      for (int o = tid; o < KN; o += nt) {
        const int k = o / N, mu = o - k * N;
        auto env_new = [&](int im, const T* rj) {  // envelope of orbital o for electron im (own spin) at distances rj
          const int sbm = im >= n_up;
          const T* pi = (sbm ? pi_dn : pi_up) + (size_t)o * M * rep;
          const T* ze = (sbm ? zeta_dn : zeta_up) + (size_t)o * M * rep;
          T e = T(0);
          for (int m = 0; m < M; ++m)
            for (int t = 0; t < rep; ++t) e += pi[m * rep + t] * env_exp_scaled(env_scale(-m_abs(ze[m * rep + t])) * rj[m]);
          return e;
        };
        const T enew0 = env_new(mv.e0, rho);
        const T enew1 = nmv > 1 ? env_new(mv.e1, rho + M) : T(0);
        const T* eb = env_base + (size_t)bw * N * KN + o;
        const T* bfp = BF + (size_t)b * N * ldb + o;
        T* arow = As + (size_t)k * N * NP + mu;
        const bool mu_up = mu < n_up;
        // rows of the two spin blocks; a block that is structurally zero (spin-factorised determinants) is only cleared
        const T* ep = eb;
        const T* bp = bfp;
        T* ap = arow;
#pragma unroll 1
        for (int sb = 0; sb < 2; ++sb) {
          const int cnt = sb ? N - n_up : n_up;
          if (!full_det && ((sb == 0) != mu_up)) {
            for (int i = 0; i < cnt; ++i, ap += NP) *ap = T(0);
            ep += (size_t)cnt * KN; bp += (size_t)cnt * ldb;
          } else {
#pragma unroll 5
            for (int i = 0; i < cnt; ++i, ep += KN, bp += ldb, ap += NP) *ap = *ep * *bp;
          }
        }
        // the moved electrons' rows
        if (full_det || ((mv.e0 < n_up) == mu_up)) arow[mv.e0 * NP] = enew0 * bfp[(size_t)mv.e0 * ldb];
        if (nmv > 1 && (full_det || ((mv.e1 < n_up) == mu_up))) arow[mv.e1 * NP] = enew1 * bfp[(size_t)mv.e1 * ldb];
      }
    } else {
    for (int idx = tid; idx < 2 * M * NS; idx += nt) {
      const int sb = idx / (M * NS), rem = idx - sb * M * NS, m = rem / NS, il = rem - m * NS;
      const int nsp = sb ? n_dn : n_up;
      if (nsp == 0) continue;
      const int i = (sb ? n_up : 0) + (il < nsp ? il : nsp - 1);
      const T dx0 = rb[3 * i] - Rb[3 * m], dx1 = rb[3 * i + 1] - Rb[3 * m + 1], dx2 = rb[3 * i + 2] - Rb[3 * m + 2];
      rho[idx] = m_sqrt(Num<T>::eps() + dx0 * dx0 + dx1 * dx1 + dx2 * dx2);
    }
    __syncthreads();
    // ---- phase 1 ---------------------------------------------------------------------------
    for (int o = tid; o < KN; o += nt) {
      const int k = o / N, mu = o - k * N;
      const T* bfp = BF + (size_t)b * N * ldb + o;
      T* arow = As + (size_t)k * N * NP + mu;
#pragma unroll 1
      for (int sb = 0; sb < 2; ++sb) {
        const int ib = sb ? n_up : 0, nsp = sb ? n_dn : n_up;
        const T* pi = (sb ? pi_dn : pi_up) + (size_t)o * M * rep;
        const T* ze = (sb ? zeta_dn : zeta_up) + (size_t)o * M * rep;
        const T* rs = rho + (size_t)sb * M * NS;
        const bool off_block = !full_det && ((sb == 0) != (mu < n_up));  // spin-factorised determinants
#pragma unroll 1
        for (int il0 = 0; il0 < nsp; il0 += 8) {
          T e[8], bf[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            e[j] = T(0);
            bf[j] = il0 + j < nsp ? bfp[(size_t)(ib + il0 + j) * ldb] : T(0);
          }
          const T* rp = rs + il0;
          if (rep == 1) {
#pragma unroll 4
            for (int m = 0; m < M; ++m) {
              const T p = pi[m], z = env_scale(-m_abs(ze[m]));
              T r8[8];
              load8(rp + m * NS, r8);
#pragma unroll
              for (int j = 0; j < 8; ++j) e[j] += p * env_exp_scaled(z * r8[j]);
            }
          } else {
            for (int m = 0; m < M; ++m) {
              T r8[8];
              load8(rp + m * NS, r8);
              for (int t = 0; t < rep; ++t) {
                const T p = pi[m * rep + t], z = env_scale(-m_abs(ze[m * rep + t]));
#pragma unroll
                for (int j = 0; j < 8; ++j) e[j] += p * env_exp_scaled(z * r8[j]);
              }
            }
          }
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (il0 + j < nsp) arow[(ib + il0 + j) * NP] = off_block ? T(0) : e[j] * bf[j];
        }
      }
    }
    }  // full envelope evaluation
    __syncthreads();
    // ---- phase 2 ---------------------------------------------------------------------------
    for (int k = wib; k < K; k += nw) {
      T a[NM];
      const T* arow = As + ((size_t)k * N + (lane < N ? lane : 0)) * NP;
#pragma unroll
      for (int mu = 0; mu < NM; ++mu) {
        T v = (mu == lane) ? T(1) : T(0);  // padding rows / columns: identity
        if (lane < N && mu < N) v = arow[mu];
        a[mu] = v;
      }
      LogProd<T> logdet;
      bool neg = false, zero = false;  // sign of the pivot product / an exactly singular pivot (warp-uniform)
      unsigned used = N < 32 ? ~((1u << N) - 1u) : 0u;  // rows already chosen as pivots (warp-uniform); padding lanes never are
      int inv = 0;         // inversion count of the pivot order
#pragma unroll
      for (int c = 0; c < NM; ++c) {
        if (c < N) {
          const int prow = warp_argmax_abs(a[c], (used >> lane) & 1u, lane);
          inv += __popc(~used & ((1u << prow) - 1u));
          used |= 1u << prow;
          const T pv = __shfl_sync(0xffffffffu, a[c], prow);
          logdet.mul(m_abs(pv));
          neg ^= pv < T(0);
          zero |= pv == T(0);
          const bool elim = !((used >> lane) & 1u);
          const T f = (elim && pv != T(0)) ? a[c] * pivot_rcp(pv) : T(0);  // exactly singular: (sign 0, log -inf) like slogdet
#pragma unroll
          for (int j = c + 1; j < NM; ++j) {  // padding columns (j >= N) hold zeros in the live rows
            const T pj = __shfl_sync(0xffffffffu, a[j], prow);
            a[j] -= f * pj;
          }
        }
      }
      if (lane == 0) {
        det_log[(size_t)b * K + k] = logdet.value();
        det_sign[(size_t)b * K + k] = zero ? T(0) : ((neg != ((inv & 1) != 0)) ? T(-1) : T(1));
      }
    }
  }
}

// Envelope table of the base walkers of a non-local-ECP group: out[w][i][o] = sum_m pi_{o m} exp(-|zeta_{o m}| |r_i - R_m|),
// o = k N + mu (spin of electron i selects the parameter set).  One block per walker; thread <-> orbital, so the quadrature
// forwards read it coalesced.  reference: wf/env.py (ExponentialEnvelopes), used through ecp/gaussian_type_ecp.py:161-255.
template <class T>
__global__ void env_table_kernel(const T* __restrict__ r, const T* __restrict__ R, int N, int M, int n_up, int KN,
                                 const T* __restrict__ pi_up, const T* __restrict__ pi_dn, const T* __restrict__ zeta_up,
                                 const T* __restrict__ zeta_dn, int rep, T* __restrict__ out) {
  DQMC_DYN_SMEM(smem_raw);
  T* rho = reinterpret_cast<T*>(smem_raw);  // [N][M]
  const int w = blockIdx.x;
  const T* rb = r + (size_t)w * N * 3;
  for (int idx = threadIdx.x; idx < N * M; idx += blockDim.x) {
    const int i = idx / M, m = idx - i * M;
    const T dx0 = rb[3 * i] - R[3 * m], dx1 = rb[3 * i + 1] - R[3 * m + 1], dx2 = rb[3 * i + 2] - R[3 * m + 2];
    rho[idx] = m_sqrt(Num<T>::eps() + dx0 * dx0 + dx1 * dx1 + dx2 * dx2);
  }
  __syncthreads();
  for (int o = threadIdx.x; o < KN; o += blockDim.x)
    for (int i = 0; i < N; ++i) {
      const T* pi = (i < n_up ? pi_up : pi_dn) + (size_t)o * M * rep;
      const T* ze = (i < n_up ? zeta_up : zeta_dn) + (size_t)o * M * rep;
      T e = T(0);
      for (int m = 0; m < M; ++m)
        for (int t = 0; t < rep; ++t) e += pi[m * rep + t] * env_exp_scaled(env_scale(-m_abs(ze[m * rep + t])) * rho[i * M + m]);
      out[((size_t)w * N + i) * KN + o] = e;
    }
}

// ------------------------------------------------------------------------------------------
// Molecular orbitals  A[b][k][i][mu] = envelope_{k mu}(r_i) * backflow[b][i][k N + mu]  -- what Ansatz.apply returns
// with return_mos = True (reference wf/nn_wave_function.py:131-142; used by pretraining/pretraining.py:73-78).  BF already
// carries mult_act.  full_det == 0: the spin-off-diagonal blocks are written as zeros (the caller slices the
// n_up x n_up / n_down x n_down blocks).  One thread per (b, k, i, mu).
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void orbitals_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M, int n_up,
                                int K, const T* __restrict__ pi_up, const T* __restrict__ pi_dn,
                                const T* __restrict__ zeta_up, const T* __restrict__ zeta_dn, const T* __restrict__ BF,
                                int ldb, int rep, int full_det, T* __restrict__ out, size_t total,
                                const T* __restrict__ Gadd, int add_off, int mult_on) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int mu = (int)(idx % N), i = (int)((idx / N) % N), k = (int)((idx / ((size_t)N * N)) % K);
  const size_t b = idx / ((size_t)N * N * K);
  const T* ri = r + (b * N + i) * 3;
  const T* Rb = R + (R_batched ? b * M * 3 : 0);
  const T* pi = (i < n_up ? pi_up : pi_dn) + (size_t)(k * N + mu) * M * rep;
  const T* ze = (i < n_up ? zeta_up : zeta_dn) + (size_t)(k * N + mu) * M * rep;
  T e = T(0);
  for (int m = 0; m < M; ++m) {
    const T dx0 = ri[0] - Rb[3 * m], dx1 = ri[1] - Rb[3 * m + 1], dx2 = ri[2] - Rb[3 * m + 2];
    const T rho = m_sqrt(Num<T>::eps() + dx0 * dx0 + dx1 * dx1 + dx2 * dx2);
    for (int et = 0; et < rep; ++et) e += pi[m * rep + et] * m_exp(-m_abs(ze[m * rep + et]) * rho);
  }
  const bool blocked = !full_det && ((i < n_up) != (mu < n_up));
  if (blocked) e = T(0);
  const T* bfp = BF + (b * N + i) * ldb + k * N + mu;
  T a = mult_on ? e * bfp[0] : e;
  if (Gadd && !blocked) a += Gadd[(b * N + i) * 5] * bfp[add_off];
  out[idx] = a;
}

template <class T>
inline size_t slater_fwd2_smem_bytes(int N, int M, int K) {
  // A matrices (16-byte rounded) + the two per-spin distance panels [M][NS <= round8(N)]
  return sizeof(T) * ((((size_t)K * N * (N | 1) + 3) & ~(size_t)3) + 2 * (size_t)M * (((size_t)N + 7) & ~(size_t)7));
}

// ------------------------------------------------------------------------------------------
// Per-walker assembly.  reference: wf/nn_wave_function.py:152-171 (exp-normalised sum with
// stop-gradient shift, SumPool conf_coeff, cusp), wf/cusp.py:17-26 (PsiformerCusp),
// physics.py:79-141 (kinetic term, Coulomb terms, eps-safe e-e and n-n distances, plain e-n
// distance), ecp/gaussian_type_ecp.py:127-159 (local ECP), hamil.py:165-180 (sum + 6 stats).
// One block per walker.  stats layout: [6][B] in the order V_el, E_kin, V_loc, V_nl, lap, qf2.
// ------------------------------------------------------------------------------------------
struct FinalizeCfg {
  int N, M, n_up, K, S;
  int cusp_kind;  // 0 none, 1 psiformer -s a^2 / (a + r), 2 deepqmc -s / (a (1 + a r)) (wf/cusp.py:5-26)
  double cusp_same_scale, cusp_anti_scale;
  int ecp_terms;  // Tmax of loc params (0: plain Coulomb)
  int nuc_cusp_kind = 0;  // NuclearCuspAsymptotic (wf/cusp.py:81-101): 0 none, 1 psiformer, 2 deepqmc form, scale = Z_I
};

template <class T>
__global__ void finalize_kernel(FinalizeCfg c, const T* __restrict__ r, const T* __restrict__ R, int R_batched,
                                const T* __restrict__ det_sign, const T* __restrict__ det_log,
                                const T* __restrict__ det_grad, const T* __restrict__ det_lap,
                                const T* __restrict__ cusp_alpha /*[2] same, anti*/,
                                const T* __restrict__ z_val /*[M]*/, const T* __restrict__ ecp_loc /*[M][3][2][Tm]*/,
                                const int* __restrict__ ecp_mask, int B, T* __restrict__ out_sign,
                                T* __restrict__ out_log, T* __restrict__ out_E, T* __restrict__ out_stats,
                                T* __restrict__ out_grad, const T* __restrict__ conf_w /*[K] or null: SumPool*/,
                                const T* __restrict__ jastrow /*[B][S] augmented scalar rows or null*/,
                                const T* __restrict__ nuc_cusp /*[1 + M]: alpha, nuclear charges; or null*/,
                                PhArgs<T> ph /*pseudo-Hamiltonian (common.cuh); all null: none*/) {
  DQMC_DYN_SMEM(smem_raw);
  const int N = c.N, M = c.M, K = c.K, S = c.S;
  const T* QA = S > 1 ? ph.QA : nullptr;
  const int T3 = S > 1 ? S - 2 : 0;
  T* pk = reinterpret_cast<T*>(smem_raw);  // [K]
  T* grad = pk + K;                         // [3N]
  T* scratch = grad + 3 * N;                // [66]
  T* misc = scratch + 66;                   // [4]
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const T* rb = r + (size_t)b * N * 3;
  const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
  const T* ds = det_sign + (size_t)b * K;
  const T* dl = det_log + (size_t)b * K;
  if (tid == 0) {
    T shift = dl[0];
    for (int k = 1; k < K; ++k) shift = dl[k] > shift ? dl[k] : shift;
    if ((shift - shift) != T(0)) shift = T(0);  // +-inf shift -> 0 (nn_wave_function.py:154)
    T psi = T(0);
    for (int k = 0; k < K; ++k) {  // conf_coeff: SumPool or hk.Linear(1, no bias) (nn_wave_function.py:158)
      pk[k] = (conf_w ? conf_w[k] : T(1)) * ds[k] * m_exp(dl[k] - shift);
      psi += pk[k];
    }
    for (int k = 0; k < K; ++k) pk[k] /= psi;
    misc[0] = m_log(m_abs(psi)) + shift;
    misc[1] = psi > T(0) ? T(1) : (psi < T(0) ? T(-1) : T(0));
  }
  __syncthreads();
  // ---- cusp + e-e repulsion: thread i handles electron i ---------------------------------
  T cusp_v = T(0), cusp_l = T(0), vel = T(0), vloc = T(0), enuc = T(0);
  T as_ = T(1), aa_ = T(1);
  if (c.cusp_kind != 0) { as_ = cusp_alpha[0]; aa_ = cusp_alpha[1]; }
  for (int i = tid; i < N; i += nt) {
    T g0 = 0, g1 = 0, g2 = 0;
    PhMetric<T> pm;
    if (QA) pm.load(QA + ((size_t)b * N + i) * PH_STRIDE);
    for (int j = 0; j < N; ++j) {
      if (j == i) continue;
      T dx0 = rb[3 * i] - rb[3 * j], dx1 = rb[3 * i + 1] - rb[3 * j + 1], dx2 = rb[3 * i + 2] - rb[3 * j + 2];
      T d2 = dx0 * dx0 + dx1 * dx1 + dx2 * dx2;
      T rho2 = Num<T>::eps() + d2, rho = m_sqrt(rho2);
      vel += T(0.5) / rho;  // (dead for S == 1: only sign / log are written, the compiler drops it there)
      if (c.cusp_kind != 0) {
        bool same = (i < c.n_up) == (j < c.n_up);
        T al = same ? as_ : aa_;
        // both cusp functions are -sc / (den0 + r): psiformer sc = s a^2, den0 = a; deepqmc sc = s / a^2, den0 = 1 / a
        T sc = (T)(same ? c.cusp_same_scale : c.cusp_anti_scale) * (c.cusp_kind == 1 ? al * al : T(1) / (al * al));
        T den = (c.cusp_kind == 1 ? al : T(1) / al) + rho;
        T f = -sc / den, fp = sc / (den * den), fpp = T(-2) * sc / (den * den * den);
        cusp_v += T(0.5) * f;
        if (S > 1) {
          T cc = fp / rho;
          g0 += cc * dx0; g1 += cc * dx1; g2 += cc * dx2;
          if (QA) {  // tr(A_i Hess_i f): the pair (i, j) carries electron i's metric, (j, i) electron j's
            T a0, a1, a2;
            pm.mul(dx0 / rho, dx1 / rho, dx2 / rho, a0, a1, a2);
            const T uau = (dx0 * a0 + dx1 * a1 + dx2 * a2) / rho;
            cusp_l += fpp * uau + fp * (pm.trace() - uau) / rho;
          } else
          cusp_l += fpp * d2 / rho2 + fp * (T(3) / rho - d2 / (rho2 * rho));
        }
      }
    }
    // electron-nucleus attraction (plain norm) + local ECP (+ nuclear cusp factor on the plain distances,
    // reference wf/nn_wave_function.py:129,169-170).  Plain forwards (S == 1: Metropolis, ECP quadrature) write sign / log only:
    // the potentials are skipped there (N M (1 + 3 ecp_terms) exponentials per walker that nobody reads)
    for (int m = 0; m < M && (S > 1 || c.nuc_cusp_kind != 0); ++m) {
      T dx0 = rb[3 * i] - Rb[3 * m], dx1 = rb[3 * i + 1] - Rb[3 * m + 1], dx2 = rb[3 * i + 2] - Rb[3 * m + 2];
      T d2 = dx0 * dx0 + dx1 * dx1 + dx2 * dx2;
      T dist = m_sqrt(d2);
      if (S > 1) vloc -= z_val[m] / dist;
      if (c.nuc_cusp_kind != 0) {
        const T al = nuc_cusp[0], zn = nuc_cusp[1 + m];
        const T sc = zn * (c.nuc_cusp_kind == 1 ? al * al : T(1) / (al * al));
        const T den = (c.nuc_cusp_kind == 1 ? al : T(1) / al) + dist;
        const T f = -sc / den, fp = sc / (den * den), fpp = T(-2) * sc / (den * den * den);
        cusp_v += f;
        if (S > 1) {
          const T cc = fp / dist;
          g0 += cc * dx0; g1 += cc * dx1; g2 += cc * dx2;
          if (QA) {
            T a0, a1, a2;
            pm.mul(dx0 / dist, dx1 / dist, dx2 / dist, a0, a1, a2);
            const T uau = (dx0 * a0 + dx1 * a1 + dx2 * a2) / dist;
            cusp_l += fpp * uau + fp * (pm.trace() - uau) / dist;
          } else
          cusp_l += fpp + T(2) * fp / dist;
        }
      }
      if (S == 1) continue;
      if (ph.tabs && ph.tab_of_nuc[m] >= 0)  // local pseudo-Hamiltonian term r V_loc(r) / r (pseudo_hamiltonian.py:180-196)
        vloc += ph_interp(ph.tabs + (size_t)ph.tab_of_nuc[m] * 2 * ph.G, ph.G, ph.rmax, dist) / dist;
      if (c.ecp_terms > 0 && ecp_mask[m]) {
        const T* lp = ecp_loc + (size_t)m * 6 * c.ecp_terms;
        for (int tt = 0; tt < c.ecp_terms; ++tt) {
          vloc += lp[(0 * 2 + 1) * c.ecp_terms + tt] / dist * m_exp(-lp[(0 * 2 + 0) * c.ecp_terms + tt] * d2);
          vloc += lp[(1 * 2 + 1) * c.ecp_terms + tt] * m_exp(-lp[(1 * 2 + 0) * c.ecp_terms + tt] * d2);
          vloc += lp[(2 * 2 + 1) * c.ecp_terms + tt] * dist * m_exp(-lp[(2 * 2 + 0) * c.ecp_terms + tt] * d2);
        }
      }
    }
    if (S > 1) {
      if (QA) pm.to_v(g0, g1, g2);
      grad[3 * i] = g0; grad[3 * i + 1] = g1; grad[3 * i + 2] = g2;
    }
  }
  for (int idx = tid; idx < M * M && S > 1; idx += nt) {
    int I = idx / M, J = idx % M;
    if (I < J) {
      T dx0 = Rb[3 * I] - Rb[3 * J], dx1 = Rb[3 * I + 1] - Rb[3 * J + 1], dx2 = Rb[3 * I + 2] - Rb[3 * J + 2];
      enuc += z_val[I] * z_val[J] / m_sqrt(Num<T>::eps() + dx0 * dx0 + dx1 * dx1 + dx2 * dx2);
    }
  }
  block_sum2(cusp_v, cusp_l, scratch);
  if (S > 1) {  // block-uniform
    block_sum2(vel, vloc, scratch);
    T dummy = T(0);
    block_sum2(enuc, dummy, scratch);
  }
  const T* jr = jastrow ? jastrow + (size_t)b * S : nullptr;
  if (tid == 0) {
    out_sign[b] = misc[1];
    out_log[b] = misc[0] + cusp_v + (jr ? jr[0] : T(0));
  }
  if (S == 1) return;
  // ---- determinant sum: gradient and Laplacian -------------------------------------------
  const T* dg = det_grad + (size_t)b * K * T3;
  T sum_pg2 = T(0), sum_g2 = T(0);
  for (int t = tid; t < T3; t += nt) {
    T gd = T(0), pg2 = T(0);
    for (int k = 0; k < K; ++k) {
      T gk = dg[(size_t)k * T3 + t];
      gd += pk[k] * gk;
      pg2 += pk[k] * gk * gk;
    }
    sum_pg2 += pg2 - gd * gd;  // contributes sum_k p_k g_k^2 - (sum_k p_k g_k)^2
    T gtot = gd + grad[t] + (jr ? jr[1 + t] : T(0));
    grad[t] = gtot;
    sum_g2 += gtot * gtot;
    if (out_grad && !QA) out_grad[(size_t)b * T3 + t] = gtot;
  }
  block_sum2(sum_pg2, sum_g2, scratch);
  T first = T(0);
  if (QA) {  // first-order term sum_i b_i . grad_{r_i} log|psi|, grad_r = Q^-T grad_v (pseudo_hamiltonian.py:268-274)
    for (int i = tid; i < N; i += nt) {
      PhMetric<T> pm;
      const T* rec = QA + ((size_t)b * N + i) * PH_STRIDE;
      pm.load(rec);
      T g0 = grad[3 * i], g1 = grad[3 * i + 1], g2 = grad[3 * i + 2];
      pm.to_r(g0, g1, g2);
      first += rec[12] * g0 + rec[13] * g1 + rec[14] * g2;
      if (out_grad) {
        T* og = out_grad + (size_t)b * T3 + 3 * i;
        og[0] = g0; og[1] = g1; og[2] = g2;
      }
    }
    T dummy2 = T(0);
    block_sum2(first, dummy2, scratch);
  }
  if (tid == 0) {
    T lap = sum_pg2 + cusp_l + (jr ? jr[T3 + 1] : T(0));
    for (int k = 0; k < K; ++k) lap += pk[k] * det_lap[(size_t)b * K + k];
    // A already contains the 1/2 of the kinetic energy when a pseudo-Hamiltonian is active
    T ekin = QA ? first - (lap + sum_g2) : T(-0.5) * (lap + sum_g2);
    T e = ekin + vloc + vel + enuc;  // V_nl added by the non-local ECP pass
    out_E[b] = e;
    out_stats[0 * (size_t)B + b] = vel;
    out_stats[1 * (size_t)B + b] = ekin;
    out_stats[2 * (size_t)B + b] = vloc;
    out_stats[3 * (size_t)B + b] = T(0);
    out_stats[4 * (size_t)B + b] = lap;
    out_stats[5 * (size_t)B + b] = sum_g2;
  }
}

template <class T>
inline size_t finalize_smem_bytes(int N, int K) {
  return sizeof(T) * ((size_t)K + 3 * N + 66 + 4);
}

}  // namespace dq
