// Trunk kernels of the forward-Laplacian engine: electron embedding, row GEMM, tanh
// propagation, self-attention propagation.
//
// Activation layout ("augmented rows"): X[b][i][s][f], f fastest, for walker b, electron i and
// slot s in [0, S).  S == 1: plain forward (value only).  S == T+2, T = 3*N: slot 0 = value,
// slot 1+t = d/dx_t (t = 3*j + c, coordinate c of electron j), slot T+1 = Laplacian
// sum_t d^2/dx_t^2.  A dense layer acts on all slots alike (linearity), an elementwise
// nonlinearity mixes slot 0 with the others, attention mixes electrons -- the same propagation
// rules folx applies in the reference's CLI default (conf/hamil/qc_forward_laplacian.yaml).
#pragma once
#include "common.cuh"

namespace dq {

// ------------------------------------------------------------------------------------------
// Electron embedding: nucleus-electron features (+ spin) -> optional projection.
// reference: src/deepqmc/gnn/electron_gnn.py:596-619, gnn/edge_features.py:21-78,
//            conf/ansatz/psiformer.yaml:53-67, ferminet.yaml:45-56.
// grid = ceil(B*N / epb) blocks, each handling epb consecutive (walker, electron) pairs;
// dynamic smem = 5*F*sizeof(T), F = 4*M + use_spin.
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void embed_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M,
                             int n_up, int S, int log_rescale, int use_spin, const T* __restrict__ W, int d,
                             T* __restrict__ X, int total, int epb, const T* __restrict__ QA /*pseudo-Hamiltonian metric or null*/) {
  DQMC_DYN_SMEM(smem_raw);
  const int F = 4 * M + use_spin;
  T* feat = reinterpret_cast<T*>(smem_raw);  // [F]
  T* dfeat = feat + F;                        // [3][F]
  T* lfeat = dfeat + 3 * F;                   // [F]
  for (int bi = blockIdx.x * epb; bi < total && bi < (blockIdx.x + 1) * epb; ++bi) {
  __syncthreads();  // shared feature buffers are reused per electron
  const int b = bi / N, i = bi % N;
  const T* ri = r + (size_t)bi * 3;
  const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    T dx[3] = {ri[0] - Rb[3 * m], ri[1] - Rb[3 * m + 1], ri[2] - Rb[3 * m + 2]};
    T d2 = dx[0] * dx[0] + dx[1] * dx[1] + dx[2] * dx[2];
    T rho2 = Num<T>::eps() + d2, rho = m_sqrt(rho2);
    T gr2 = d2 / rho2;                     // |grad rho|^2
    T lr = T(3) / rho - d2 / (rho2 * rho);  // laplacian rho
    T au[3] = {dx[0] / rho, dx[1] / rho, dx[2] / rho};  // (A grad rho); A = 1 without a pseudo-Hamiltonian
    if (QA) {  // second derivatives weighted by A(r_i): u^T A u and tr(A Hess rho) (common.cuh, PhMetric)
      PhMetric<T> pm;
      pm.load(QA + (size_t)bi * PH_STRIDE);
      const T u0 = au[0], u1 = au[1], u2 = au[2];
      pm.mul(u0, u1, u2, au[0], au[1], au[2]);
      gr2 = u0 * au[0] + u1 * au[1] + u2 * au[2];
      lr = (pm.trace() - gr2) / rho;
    }
    T f0, f0p, f0pp, s, sp, spp;
    if (log_rescale) {
      T g = m_log1p(rho), gp = T(1) / (T(1) + rho), gpp = -gp * gp;
      f0 = g; f0p = gp; f0pp = gpp;
      s = g / rho;
      sp = gp / rho - g / rho2;
      spp = gpp / rho - T(2) * gp / rho2 + T(2) * g / (rho2 * rho);
    } else {
      f0 = rho; f0p = T(1); f0pp = T(0);
      s = T(1); sp = T(0); spp = T(0);
    }
    const int k0 = 4 * m;
    feat[k0] = f0;
    lfeat[k0] = f0pp * gr2 + f0p * lr;
    T ls = spp * gr2 + sp * lr;  // laplacian of s(rho)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      dfeat[c * F + k0] = f0p * dx[c] / rho;
      feat[k0 + 1 + c] = dx[c] * s;
      lfeat[k0 + 1 + c] = T(2) * sp * au[c] + dx[c] * ls;
#pragma unroll
      for (int e = 0; e < 3; ++e)
        dfeat[e * F + k0 + 1 + c] = (c == e ? s : T(0)) + dx[c] * sp * dx[e] / rho;
    }
  }
  if (use_spin && threadIdx.x == 0) {
    feat[F - 1] = i < n_up ? T(1) : T(-1);
    dfeat[F - 1] = dfeat[F + F - 1] = dfeat[2 * F + F - 1] = T(0);
    lfeat[F - 1] = T(0);
  }
  __syncthreads();
  const int T3 = S - 2;
  T* Xg = X + (size_t)bi * S * d;
  for (int f = threadIdx.x; f < d; f += blockDim.x) {
    T y0 = 0, y1 = 0, y2 = 0, y3 = 0, yl = 0;
    if (W) {
      for (int k = 0; k < F; ++k) {
        T w = W[(size_t)k * d + f];
        y0 += feat[k] * w;
        y1 += dfeat[k] * w;
        y2 += dfeat[F + k] * w;
        y3 += dfeat[2 * F + k] * w;
        yl += lfeat[k] * w;
      }
    } else {  // identity projection (d == F)
      y0 = feat[f]; y1 = dfeat[f]; y2 = dfeat[F + f]; y3 = dfeat[2 * F + f]; yl = lfeat[f];
    }
    Xg[f] = y0;
    if (S > 1) {
      if (QA) {  // tangent seeds = columns of Q_i
        PhMetric<T> pm;
        pm.load(QA + (size_t)bi * PH_STRIDE);
        pm.to_v(y1, y2, y3);
      }
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
  }
}

// ------------------------------------------------------------------------------------------
// Plain-forward (S == 1) electron embedding with projection: the first kernel of every Metropolis
// sub-step and of every non-local-ECP quadrature forward (12 N N_ecp per walker), so it is written
// as a small register-tiled GEMM  X[e, :] = feat[e, 0:F] @ W[F, d]  with the features computed in
// the block.  Same reference lines as embed_kernel (electron_gnn.py:596-619, edge_features.py:21-78).
// Block = 256 threads; W (F x d) is staged once per block in shared memory and reused for `epb`
// electrons (persistent over tiles of 32 electrons); thread tile = 8 electrons x 4 features.
// dynamic smem = sizeof(T) * (F * d + FP * 32), FP = F rounded up to a multiple of 4.
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void __launch_bounds__(256)
embed_fwd_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M, int n_up,
                 int log_rescale, const T* __restrict__ W, int d, T* __restrict__ X, int total, int epb,
                 long long v0 = 0, int vper = 0, const int* __restrict__ pairs = nullptr) {
  // vper > 0: compact mode of the non-local-ECP quadrature forwards -- row t is the MOVED electron of virtual walker v = v0 + t
  // (virtual_move, ECP layout over the active-pair list `pairs`); the other electrons' rows are those of the base walker (see
  // trunk_tc.cuh)
  DQMC_DYN_SMEM(smem_raw);
  const int F = 4 * M + 1;
  T* Ws = reinterpret_cast<T*>(smem_raw);  // [F][d]
  T* ft = Ws + (size_t)F * d;              // [F][32]  feature k of the tile's 32 electrons
  const int tid = threadIdx.x;
  for (int i = tid; i < F * d; i += 256) Ws[i] = W[i];
  const int e_begin = blockIdx.x * epb;
  const int e_end = e_begin + epb < total ? e_begin + epb : total;
  const int te = tid >> 6, tf = tid & 63;  // electron group (8 electrons), feature group (4 features)
  for (int e0 = e_begin; e0 < e_end; e0 += 32) {
    __syncthreads();  // previous tile done with ft (and Ws staged)
    for (int idx = tid; idx < 32 * M; idx += 256) {
      const int el = idx / M, m = idx - el * M;
      const int bi = e0 + el;
      T f0 = T(0), g0 = T(0), g1 = T(0), g2 = T(0);
      if (bi < e_end) {
        const int b = vper > 0 ? bi : bi / N;
        const T* ri = r + (vper > 0 ? ((size_t)bi * N + (size_t)virtual_move((int)(v0 + bi), vper, N, n_up, kVirtEcp, pairs).e0) : (size_t)bi) * 3;
        const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
        const T dx0 = ri[0] - Rb[3 * m], dx1 = ri[1] - Rb[3 * m + 1], dx2 = ri[2] - Rb[3 * m + 2];
        const T rho = m_sqrt(Num<T>::eps() + dx0 * dx0 + dx1 * dx1 + dx2 * dx2);
        T s = T(1);
        f0 = rho;
        if (log_rescale) { f0 = m_log1p(rho); s = f0 / rho; }
        g0 = dx0 * s; g1 = dx1 * s; g2 = dx2 * s;
      }
      ft[(4 * m) * 32 + el] = f0;
      ft[(4 * m + 1) * 32 + el] = g0;
      ft[(4 * m + 2) * 32 + el] = g1;
      ft[(4 * m + 3) * 32 + el] = g2;
    }
    if (tid < 32) {
      const int bi = e0 + tid;
      const int el_i = vper > 0 ? (bi < e_end ? virtual_move((int)(v0 + bi), vper, N, n_up, kVirtEcp, pairs).e0 : 0) : bi % N;
      ft[(F - 1) * 32 + tid] = (bi < e_end && el_i < n_up) ? T(1) : T(-1);
    }
    __syncthreads();
    for (int f0 = 4 * tf; f0 < d; f0 += 256) {
      T acc[8][4];
#pragma unroll
      for (int e = 0; e < 8; ++e)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[e][j] = T(0);
      const bool full = f0 + 3 < d;
      for (int k = 0; k < F; ++k) {
        T w[4], x[8];
        const T* wr = Ws + (size_t)k * d + f0;
        if (full) {
          ld4(wr, w);
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) w[j] = f0 + j < d ? wr[j] : T(0);
        }
        const T* xr = ft + k * 32 + te * 8;
        {
          T xa[4], xb[4];
          ld4(xr, xa);
          ld4(xr + 4, xb);
#pragma unroll
          for (int e = 0; e < 4; ++e) { x[e] = xa[e]; x[4 + e] = xb[e]; }
        }
#pragma unroll
        for (int e = 0; e < 8; ++e)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[e][j] += x[e] * w[j];
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int bi = e0 + te * 8 + e;
        if (bi >= e_end) continue;
        T* xo = X + (size_t)bi * d + f0;
        if (full) {
          st4(xo, acc[e]);
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (f0 + j < d) xo[j] = acc[e][j];
        }
      }
    }
  }
}

template <class T>
inline size_t embed_fwd_smem_bytes(int M, int d) {
  const int F = 4 * M + 1;
  return sizeof(T) * ((size_t)F * d + (size_t)F * 32);
}

// ------------------------------------------------------------------------------------------
// Row GEMM  C[row(m), :] = (Res[row(m), :]) + A[row(m), :] @ W + (bias on value rows)
// Plain SIMT tiling (CUDA cores), used for the fp64 parity mode and as the reference
// implementation the tensor-core fp32 path is validated against.
// sliced == 1: blockIdx.z = electron e, rows m = (b, s) -> physical row (b*Nel + e)*S + s,
//              weights W0 for e < z_split else W1 (per-spin backflow heads, wf/omni.py:43-88).
// ------------------------------------------------------------------------------------------
template <class T>
struct GemmArgs {
  const T* A; int lda;
  const T* W0; const T* W1; int z_split; int ldw;
  const T* bias;
  const T* Res; int ldr;
  T* C; int ldc;
  int M, N, K;
  int S;
  int sliced, Nel;
  const T* bias1 = nullptr;  // sliced: bias of the second weight (z >= z_split); null: `bias` for both
};

template <class T, int BM, int BN, int BK, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN)) gemm_kernel(GemmArgs<T> g) {
  constexpr int NT = (BM / TM) * (BN / TN);
  __shared__ T As[BK][BM + 1];
  __shared__ T Ws[BK][BN];
  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int z = blockIdx.z;
  const T* W = (g.sliced && z >= g.z_split) ? g.W1 : g.W0;
  const T* bias = (g.sliced && z >= g.z_split && g.bias1) ? g.bias1 : g.bias;
  auto phys_row = [&](int m) -> size_t {
    if (!g.sliced) return (size_t)m;
    int b = m / g.S, s = m % g.S;
    return ((size_t)b * g.Nel + z) * g.S + s;
  };
  T acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = T(0);

  for (int k0 = 0; k0 < g.K; k0 += BK) {
    for (int idx = tid; idx < BM * BK; idx += NT) {
      int mm = idx / BK, kk = idx % BK;
      int m = m0 + mm, k = k0 + kk;
      T v = T(0);
      if (m < g.M && k < g.K) v = g.A[phys_row(m) * g.lda + k];
      As[kk][mm] = v;
    }
    for (int idx = tid; idx < BK * BN; idx += NT) {
      int kk = idx / BN, nn = idx % BN;
      int k = k0 + kk, n = n0 + nn;
      T v = T(0);
      if (k < g.K && n < g.N) v = W[(size_t)k * g.ldw + n];
      Ws[kk][nn] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      T a[TM], w[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = As[kk][ty * TM + i];
#pragma unroll
      for (int j = 0; j < TN; ++j) w[j] = Ws[kk][tx * TN + j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] += a[i] * w[j];
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int m = m0 + ty * TM + i;
    if (m >= g.M) continue;
    size_t pr = phys_row(m);
    bool value_row = (pr % g.S) == 0;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int n = n0 + tx * TN + j;
      if (n >= g.N) continue;
      T v = acc[i][j];
      if (bias && value_row) v += bias[n];
      if (g.Res) v += g.Res[pr * g.ldr + n];
      g.C[pr * g.ldc + n] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------
// tanh propagation: y = tanh(z); y_t = y' z_t; y_lap = y' z_lap + y'' sum_t z_t^2
// optional residual (all slots): out = res_scale * (Res + y)
// grid = (G groups, ceil(d/blockDim)); in place on Z.
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void tanh_fl_kernel(T* __restrict__ Z, int ldz, const T* __restrict__ Res, int ldr, int S, int d,
                               T out_scale) {
  const int g = blockIdx.x;
  const int f = blockIdx.y * blockDim.x + threadIdx.x;
  if (f >= d) return;
  T* z = Z + (size_t)g * S * ldz + f;
  const T* rs = Res ? Res + (size_t)g * S * ldr + f : nullptr;
  T y = m_tanh(z[0]);
  T y1 = T(1) - y * y, y2 = T(-2) * y * y1;
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

// ---- warp-level tensor-core products for the tangent chunks (MMA variant below): mma.sync m16n8k8 on TF32 operands split
// hi + lo in registers ("3xTF32": a_lo b_hi + a_hi b_lo + a_hi b_hi accumulated in fp32, 2^-21-class products; the tangent
// rows have no bounded range, so the 8-bit exponent of TF32 is kept instead of scaled halves).  Fragment layouts (PTX ISA,
// m16n8k8 .tf32, g = lane / 4, t = lane % 4): A a0 (g, t) a1 (g + 8, t) a2 (g, t + 4) a3 (g + 8, t + 4); B b0 (k = t, n = g)
// b1 (k = t + 4, n = g); C c0 (g, 2 t) c1 (g, 2 t + 1) c2 (g + 8, 2 t) c3 (g + 8, 2 t + 1).
struct TfA { uint32_t hi[4], lo[4]; };
struct TfB { uint32_t hi[2], lo[2]; };
#ifdef DQMC_EMU
__device__ __forceinline__ uint32_t tf32_rna_bits(float x) {
  uint32_t u; std::memcpy(&u, &x, 4);
  if ((u & 0x7F800000u) != 0x7F800000u) u += 0x1000u;  // round to nearest, ties away
  return u & 0xFFFFE000u;
}
__device__ __forceinline__ void mma1688(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  float c[4] = {d[0], d[1], d[2], d[3]};
  emu::mma_m16n8k8_tf32(d, a, b, c);
}
#else
__device__ __forceinline__ uint32_t tf32_rna_bits(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void mma1688(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
#endif
__device__ __forceinline__ void tf32_split(float x, uint32_t& hi, uint32_t& lo) {
  hi = tf32_rna_bits(x);
  lo = tf32_rna_bits(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma3(float (&d)[4], const TfA& a, const TfB& b) {
  mma1688(d, a.lo, b.hi);
  mma1688(d, a.hi, b.lo);
  mma1688(d, a.hi, b.hi);
}

// Scores of a tangent chunk: st[t][i][j] = c (q^t_i . k_j + q_i . k^t_j), qk[i][j] += sum_t q^t_i . k^t_j for the N queries
// and NK >= N keys (keys j >= N are walker-independent extra tokens: k^t_j = 0).  Rows of q / k / qt / kt have pitch PQ
// floats (PQ % 32 == 4: conflict-free fragment loads), qt / kt are [tc][N][PQ], st is [tc][N][NK], qk [N][NK].
// A warp task owns one 16-query x 8-key tile for all tangents of the chunk (single writer of every running sum).
__device__ __forceinline__ void attn_fl_mma_scores(const float* q, const float* k, const float* qt, const float* kt, float* st,
                                                   float* qk, int N, int NK, int PQ, int dh, int tc, float scale, int tid, int nt) {
  const int wid = tid >> 5, nw = nt >> 5, lane = tid & 31, g = lane >> 2, tq = lane & 3;
  const int mtiles = (N + 15) >> 4, ntiles = (NK + 7) >> 3;
  for (int task = wid; task < mtiles * ntiles; task += nw) {
    const int mt = task / ntiles, nt8 = task - mt * ntiles;
    const int i0 = mt * 16 + g, i1 = i0 + 8, jn = nt8 * 8 + g;
    const int i0c = i0 < N ? i0 : N - 1, i1c = i1 < N ? i1 : N - 1, jc = jn < NK ? jn : NK - 1;
    const bool tang = nt8 * 8 < N;          // the tile holds electron keys (k^t != 0 for j < N)
    const bool jt = jn < N;                 // this lane's key carries tangents
    const int jtc = jt ? jn : N - 1;
    const float* q0 = q + i0c * PQ;
    const float* q1 = q + i1c * PQ;
    const float* kj = k + jc * PQ;
    float cacc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int t = 0; t < tc; ++t) {
      const float* qt0 = qt + (size_t)(t * N + i0c) * PQ;
      const float* qt1 = qt + (size_t)(t * N + i1c) * PQ;
      const float* ktj = kt + (size_t)(t * N + jtc) * PQ;
      float sacc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 2
      for (int e = tq; e < dh; e += 8) {
        TfA aqt;
        TfB bk;
        tf32_split(qt0[e], aqt.hi[0], aqt.lo[0]); tf32_split(qt1[e], aqt.hi[1], aqt.lo[1]);
        tf32_split(qt0[e + 4], aqt.hi[2], aqt.lo[2]); tf32_split(qt1[e + 4], aqt.hi[3], aqt.lo[3]);
        tf32_split(kj[e], bk.hi[0], bk.lo[0]); tf32_split(kj[e + 4], bk.hi[1], bk.lo[1]);
        mma3(sacc, aqt, bk);
        if (tang) {  // warp-uniform
          TfA aq;
          TfB bkt;
          tf32_split(q0[e], aq.hi[0], aq.lo[0]); tf32_split(q1[e], aq.hi[1], aq.lo[1]);
          tf32_split(q0[e + 4], aq.hi[2], aq.lo[2]); tf32_split(q1[e + 4], aq.hi[3], aq.lo[3]);
          tf32_split(jt ? ktj[e] : 0.f, bkt.hi[0], bkt.lo[0]); tf32_split(jt ? ktj[e + 4] : 0.f, bkt.hi[1], bkt.lo[1]);
          mma3(sacc, aq, bkt);
          mma3(cacc, aqt, bkt);
        }
      }
      const int j0 = nt8 * 8 + 2 * tq;
      float* s0 = st + ((size_t)t * N + i0) * NK;
      float* s1 = st + ((size_t)t * N + i1) * NK;
      if (i0 < N) {
        if (j0 < NK) s0[j0] = scale * sacc[0];
        if (j0 + 1 < NK) s0[j0 + 1] = scale * sacc[1];
      }
      if (i1 < N) {
        if (j0 < NK) s1[j0] = scale * sacc[2];
        if (j0 + 1 < NK) s1[j0 + 1] = scale * sacc[3];
      }
    }
    if (tang) {
      const int j0 = nt8 * 8 + 2 * tq;
      if (i0 < N) {
        if (j0 < N) qk[i0 * NK + j0] += cacc[0];
        if (j0 + 1 < N) qk[i0 * NK + j0 + 1] += cacc[1];
      }
      if (i1 < N) {
        if (j0 < N) qk[i1 * NK + j0] += cacc[2];
        if (j0 + 1 < N) qk[i1 * NK + j0 + 1] += cacc[3];
      }
    }
  }
}
// Outputs of a tangent chunk: o^t_i = sum_j p^t_ij v_j + p_ij v^t_j (written to Ot + t * ldt, row i at i * ldrow, dh columns),
// olap[i][:] += 2 sum_t sum_j p^t_ij v^t_j; pt is [tc][N][NK] (p^t, in the st buffer), p [N][NK], v [NK][PQ], vt [tc][N][PQ]
// (v^t_j = 0 for j >= N).  A warp task owns 16 queries x 16 columns for all tangents of the chunk.
__device__ __forceinline__ void attn_fl_mma_outputs(const float* pt, const float* p, const float* v, const float* vt, float* olap,
                                                    float* Ot, size_t ldt, size_t ldrow, int N, int NK, int PQ, int dh, int tc,
                                                    int tid, int nt) {
  const int wid = tid >> 5, nw = nt >> 5, lane = tid & 31, g = lane >> 2, tq = lane & 3;
  const int mtiles = (N + 15) >> 4, n_eg = dh >> 4;
  for (int task = wid; task < mtiles * n_eg; task += nw) {
    const int mt = task / n_eg, eg = task - mt * n_eg;
    const int i0 = mt * 16 + g, i1 = i0 + 8;
    const int i0c = i0 < N ? i0 : N - 1, i1c = i1 < N ? i1 : N - 1;
    float c2[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
    for (int t = 0; t < tc; ++t) {
      float oa[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
      const float* pt0 = pt + ((size_t)t * N + i0c) * NK;
      const float* pt1 = pt + ((size_t)t * N + i1c) * NK;
      const float* pr0 = p + i0c * NK;
      const float* pr1 = p + i1c * NK;
      for (int jb = 0; jb < NK; jb += 8) {
        const int j0 = jb + tq, j1 = j0 + 4;
        const bool v0 = j0 < NK, v1 = j1 < NK;  // keys beyond NK contribute nothing (A = 0, B read from a valid row)
        const int j0c = v0 ? j0 : NK - 1, j1c = v1 ? j1 : NK - 1;
        const bool tang = jb < N;               // warp-uniform: the k-step holds electron keys
        const bool t0v = j0 < N, t1v = j1 < N;
        const int j0t = t0v ? j0 : N - 1, j1t = t1v ? j1 : N - 1;
        TfA apt, ap;
        tf32_split(v0 ? pt0[j0c] : 0.f, apt.hi[0], apt.lo[0]); tf32_split(v0 ? pt1[j0c] : 0.f, apt.hi[1], apt.lo[1]);
        tf32_split(v1 ? pt0[j1c] : 0.f, apt.hi[2], apt.lo[2]); tf32_split(v1 ? pt1[j1c] : 0.f, apt.hi[3], apt.lo[3]);
        if (tang) {
          tf32_split(v0 ? pr0[j0c] : 0.f, ap.hi[0], ap.lo[0]); tf32_split(v0 ? pr1[j0c] : 0.f, ap.hi[1], ap.lo[1]);
          tf32_split(v1 ? pr0[j1c] : 0.f, ap.hi[2], ap.lo[2]); tf32_split(v1 ? pr1[j1c] : 0.f, ap.hi[3], ap.lo[3]);
        }
#pragma unroll
        for (int nn = 0; nn < 2; ++nn) {
          const int e = eg * 16 + nn * 8 + g;
          TfB bv;
          tf32_split(v[j0c * PQ + e], bv.hi[0], bv.lo[0]); tf32_split(v[j1c * PQ + e], bv.hi[1], bv.lo[1]);
          mma3(oa[nn], apt, bv);
          if (tang) {
            TfB bvt;
            tf32_split(t0v ? vt[(size_t)(t * N + j0t) * PQ + e] : 0.f, bvt.hi[0], bvt.lo[0]);
            tf32_split(t1v ? vt[(size_t)(t * N + j1t) * PQ + e] : 0.f, bvt.hi[1], bvt.lo[1]);
            mma3(oa[nn], ap, bvt);
            mma3(c2[nn], apt, bvt);
          }
        }
      }
#pragma unroll
      for (int nn = 0; nn < 2; ++nn) {
        const int e0 = eg * 16 + nn * 8 + 2 * tq;
        if (i0 < N) *(float2*)(Ot + (size_t)t * ldt + (size_t)i0 * ldrow + e0) = make_float2(oa[nn][0], oa[nn][1]);
        if (i1 < N) *(float2*)(Ot + (size_t)t * ldt + (size_t)i1 * ldrow + e0) = make_float2(oa[nn][2], oa[nn][3]);
      }
    }
#pragma unroll
    for (int nn = 0; nn < 2; ++nn) {
      const int e0 = eg * 16 + nn * 8 + 2 * tq;
      if (i0 < N) { olap[i0 * dh + e0] += 2.f * c2[nn][0]; olap[i0 * dh + e0 + 1] += 2.f * c2[nn][1]; }
      if (i1 < N) { olap[i1 * dh + e0] += 2.f * c2[nn][2]; olap[i1 * dh + e0 + 1] += 2.f * c2[nn][3]; }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Self-attention with forward-Laplacian propagation, one block per (walker, head).
// value algebra: hk.MultiHeadAttention (restated in reference src/deepqmc/hkext.py:215-253,
// folxext.py:7-17): logits = q k^T / sqrt(dh), softmax over keys, out = P v.
// derivative algebra: dense-Jacobian generalisation of reference src/deepqmc/folxext.py:70-171.
//   s^t  = c (q^t k + q k^t)            p^t  = p (s^t - m^t),  m^t = sum_j p s^t
//   s^L  = c (q^L k + q k^L + 2 sum_t q^t k^t)
//   lap p = p (u - V + s^L - sum_j p s^L),  u = sum_t (s^t - m^t)^2,  V = sum_j p u
//   o^t  = p^t v + p v^t ;  o^L = (lap p) v + 2 sum_t p^t v^t + p v^L
// QKV: [rows][ldq] with q at col h*dh, k at dmodel + h*dh, v at 2*dmodel + h*dh.
// ------------------------------------------------------------------------------------------
// MMA (float only, dh % 16 == 0): the tangent-chunk contractions as warp-level 3xTF32 tensor-core products
// (attn_fl_mma_scores / attn_fl_mma_outputs above); the shared-memory rows then have pitch dh + 4.
template <class T, bool MMA = false>
__global__ void attn_fl_kernel(const T* __restrict__ QKV, int ldq, T* __restrict__ O, int ldo, int N, int S, int dh,
                               int dmodel, T scale, int TB, const T* __restrict__ Kn, const T* __restrict__ Vn, int Mn) {
  // Tangent slots are processed in chunks of TB so that every phase has (TB x N x NK) or (N x dh)
  // independent work items (small molecules: all 3N tangents in one chunk).
  // Kn / Vn [Mn][dmodel] (nullable): key / value rows of Mn walker-independent extra tokens (the
  // nuclei of the TransPsiformer, reference gnn/update_features.py:385-451 with elec_to_nuc =
  // false); they sit behind the N electron keys (softmax is order-independent) and carry zero
  // tangents, so every derivative term with k^t_j, v^t_j, k^L_j, v^L_j vanishes for j >= N.
  DQMC_DYN_SMEM(smem_raw);
  const int NK = N + Mn;
  const int dhp = dh + (MMA ? 4 : 1), NN = N * NK;
  T* q = reinterpret_cast<T*>(smem_raw);   // [N][dhp]
  T* k = q + N * dhp;                      // [NK][dhp]
  T* v = k + NK * dhp;                     // [NK][dhp]
  T* qt = v + NK * dhp;                    // [TB][N][dhp]
  T* kt = qt + (size_t)TB * N * dhp;
  T* vt = kt + (size_t)TB * N * dhp;
  T* p = vt + (size_t)TB * N * dhp;  // [N][NK]
  T* st = p + NN;                 // [TB][N][NK]
  T* u = st + (size_t)TB * NN;    // [N][NK]
  T* qk = u + NN;                 // [N][NK]
  T* olap = qk + NN;              // [N][dh]
  T* mrow = olap + N * dh;        // [TB][N]
  T* vrow = mrow + TB * N;        // [N]
  const int b = blockIdx.x, h = blockIdx.y;
  const int tid = threadIdx.x, nt = blockDim.x;
  const int T3 = S > 1 ? S - 2 : 0;
  const size_t row0 = (size_t)b * N * S;
  auto load3 = [&](int slot0, int nslot, T* dq_, T* dk_, T* dv_) {
    for (int idx = tid; idx < nslot * N * dh; idx += nt) {
      int e = idx % dh, i = (idx / dh) % N, t = idx / (dh * N);
      const T* src = QKV + (row0 + (size_t)i * S + slot0 + t) * ldq + h * dh + e;
      int o = (t * N + i) * dhp + e;
      dq_[o] = src[0];
      dk_[o] = src[dmodel];
      dv_[o] = src[2 * dmodel];
    }
  };
  load3(0, 1, q, k, v);
  for (int idx = tid; idx < Mn * dh; idx += nt) {
    int e = idx % dh, m = idx / dh;
    k[(N + m) * dhp + e] = Kn[(size_t)m * dmodel + h * dh + e];
    v[(N + m) * dhp + e] = Vn[(size_t)m * dmodel + h * dh + e];
  }
  __syncthreads();
  for (int idx = tid; idx < NN; idx += nt) {
    int i = idx / NK, j = idx % NK;
    T a = T(0);
    for (int e = 0; e < dh; ++e) a += q[i * dhp + e] * k[j * dhp + e];
    p[idx] = a * scale;
    u[idx] = T(0);
    qk[idx] = T(0);
  }
  for (int idx = tid; idx < N * dh; idx += nt) olap[idx] = T(0);
  __syncthreads();
  for (int i = tid; i < N; i += nt) {  // softmax row i
    T mx = p[i * NK];
    for (int j = 1; j < NK; ++j) mx = p[i * NK + j] > mx ? p[i * NK + j] : mx;
    T sum = T(0);
    for (int j = 0; j < NK; ++j) {
      T e = m_exp(p[i * NK + j] - mx);
      p[i * NK + j] = e;
      sum += e;
    }
    T inv = T(1) / sum;
    for (int j = 0; j < NK; ++j) p[i * NK + j] *= inv;
  }
  __syncthreads();
  for (int idx = tid; idx < N * dh; idx += nt) {
    int i = idx / dh, e = idx % dh;
    T a = T(0);
    for (int j = 0; j < NK; ++j) a += p[i * NK + j] * v[j * dhp + e];
    O[(row0 + (size_t)i * S) * ldo + h * dh + e] = a;
  }
  if (S == 1) return;
  for (int t0 = 0; t0 < T3; t0 += TB) {
    const int tc = T3 - t0 < TB ? T3 - t0 : TB;
    __syncthreads();  // previous chunk done with qt/kt/vt/st
    load3(1 + t0, tc, qt, kt, vt);
    __syncthreads();
    if constexpr (MMA && std::is_same<T, float>::value) {
      attn_fl_mma_scores(q, k, qt, kt, st, qk, N, NK, dhp, dh, tc, scale, tid, nt);
    } else {
    for (int idx = tid; idx < tc * NN; idx += nt) {
      int j = idx % NK, i = (idx / NK) % N, t = idx / NN;
      const T* qti = qt + (t * N + i) * dhp;
      T a = T(0);
      if (j < N) {
        const T* ktj = kt + (t * N + j) * dhp;
        for (int e = 0; e < dh; ++e) a += qti[e] * k[j * dhp + e] + q[i * dhp + e] * ktj[e];
      } else {
        for (int e = 0; e < dh; ++e) a += qti[e] * k[j * dhp + e];
      }
      st[idx] = a * scale;
    }
    for (int idx = tid; idx < NN; idx += nt) {
      int i = idx / NK, j = idx % NK;
      if (j >= N) continue;
      T c = T(0);
      for (int t = 0; t < tc; ++t) {
        const T* qti = qt + (t * N + i) * dhp;
        const T* ktj = kt + (t * N + j) * dhp;
        for (int e = 0; e < dh; ++e) c += qti[e] * ktj[e];
      }
      qk[idx] += c;
    }
    }  // SIMT scores
    __syncthreads();
    for (int idx = tid; idx < tc * N; idx += nt) {  // (t, i)
      const T* pr = p + (idx % N) * NK;
      const T* sr = st + (size_t)idx * NK;
      T m = T(0);
      for (int j = 0; j < NK; ++j) m += pr[j] * sr[j];
      mrow[idx] = m;
    }
    __syncthreads();
    for (int idx = tid; idx < NN; idx += nt) {
      int i = idx / NK;
      T uu = T(0), pp = p[idx];
      for (int t = 0; t < tc; ++t) {
        T dv_ = st[t * NN + idx] - mrow[t * N + i];
        uu += dv_ * dv_;
        st[t * NN + idx] = pp * dv_;  // p^t
      }
      u[idx] += uu;
    }
    __syncthreads();
    if constexpr (MMA && std::is_same<T, float>::value) {
      attn_fl_mma_outputs(st, p, v, vt, olap, O + (row0 + 1 + t0) * ldo + h * dh, (size_t)ldo, (size_t)S * ldo, N, NK, dhp, dh, tc,
                          tid, nt);
    } else
    for (int idx = tid; idx < N * dh; idx += nt) {
      int i = idx / dh, e = idx % dh;
      T c2 = T(0);
      for (int t = 0; t < tc; ++t) {
        const T* sr = st + t * NN + i * NK;
        const T* vtt = vt + (size_t)t * N * dhp + e;
        T a = T(0), c = T(0);
        for (int j = 0; j < N; ++j) {
          T vtj = vtt[j * dhp];
          a += sr[j] * v[j * dhp + e] + p[i * NK + j] * vtj;
          c += sr[j] * vtj;
        }
        for (int j = N; j < NK; ++j) a += sr[j] * v[j * dhp + e];
        c2 += c;
        O[(row0 + (size_t)i * S + 1 + t0 + t) * ldo + h * dh + e] = a;
      }
      olap[idx] += T(2) * c2;
    }
  }
  __syncthreads();
  load3(1 + T3, 1, qt, kt, vt);
  __syncthreads();
  for (int idx = tid; idx < NN; idx += nt) {
    int i = idx / NK, j = idx % NK;
    T a = T(0);
    if (j < N) {
      for (int e = 0; e < dh; ++e) a += qt[i * dhp + e] * k[j * dhp + e] + q[i * dhp + e] * kt[j * dhp + e];
    } else {
      for (int e = 0; e < dh; ++e) a += qt[i * dhp + e] * k[j * dhp + e];
    }
    st[idx] = scale * (a + T(2) * qk[idx]);
  }
  __syncthreads();
  for (int i = tid; i < N; i += nt) {
    T m = T(0), V = T(0);
    for (int j = 0; j < NK; ++j) {
      m += p[i * NK + j] * st[i * NK + j];
      V += p[i * NK + j] * u[i * NK + j];
    }
    mrow[i] = m;
    vrow[i] = V;
  }
  __syncthreads();
  for (int idx = tid; idx < NN; idx += nt) {
    int i = idx / NK;
    st[idx] = p[idx] * (u[idx] - vrow[i] + st[idx] - mrow[i]);
  }
  __syncthreads();
  for (int idx = tid; idx < N * dh; idx += nt) {
    int i = idx / dh, e = idx % dh;
    T a = olap[idx];
    for (int j = 0; j < N; ++j) a += st[i * NK + j] * v[j * dhp + e] + p[i * NK + j] * vt[j * dhp + e];
    for (int j = N; j < NK; ++j) a += st[i * NK + j] * v[j * dhp + e];
    O[(row0 + (size_t)i * S + 1 + T3) * ldo + h * dh + e] = a;
  }
}

template <class T>
inline size_t attn_smem_bytes(int N, int dh, int TB, int Mn = 0, int pad = 1) {
  const size_t NK = N + Mn;
  return sizeof(T) * ((size_t)N * (dh + pad) + 2 * NK * (dh + pad) + (size_t)3 * TB * N * (dh + pad) +
                      (size_t)N * NK * (3 + TB) + (size_t)N * dh + (size_t)TB * N + N);
}
// largest tangent chunk whose working set fits `budget` bytes of shared memory
template <class T>
inline int attn_pick_tb(int N, int dh, int T3, size_t budget, int Mn = 0, int pad = 1) {
  int tb = T3 > 0 ? T3 : 1;
  while (tb > 1 && attn_smem_bytes<T>(N, dh, tb, Mn, pad) > budget) --tb;
  return tb;
}

// ------------------------------------------------------------------------------------------
// fp32 production variant of attn_fl_kernel: same algebra, but shared-memory rows are padded to
// dh+4 floats so that every operand is fetched with 128-bit LDS (own rows conflict-free, shared
// rows as broadcasts), the e-range of each dot product is split over 4 adjacent lanes and reduced
// with shuffles, and global traffic is float4.  Requires dh % 16 == 0.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float dot4(const float4& a, const float4& b) {
  return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
}
__device__ __forceinline__ void fma4(float4& acc, float s, const float4& v) {
  acc.x += s * v.x; acc.y += s * v.y; acc.z += s * v.z; acc.w += s * v.w;
}

// NE / DH: compile-time electron count / head dim (0 = use the runtime value): with constants the
// index arithmetic (div/mod by N, dh/4) folds away and the j-loops unroll.
// MMA (N <= 32, dh % 8 == 0): the three contractions that carry the tangent chunks -- s^t = c (q^t k + q k^t) with the
// running sum of q^t k^t, and o^t = p^t v + p v^t with the running sum of p^t v^t -- run as warp-level 3xTF32 tensor-core
// products straight from the shared-memory rows (pitch dh + 4: conflict-free fragment loads).  A warp task owns one
// 16-row x 8-key tile (scores) / 16-row x 16-column tile (outputs) for ALL tangents of the chunk, so every running sum has a
// single writer (bitwise reproducible).  The SIMT phases in between (softmax statistics, p^t) are shared with the other variant.
template <int NE, int DH, bool MMA>
__global__ void attn_fl_f32_kernel(const float* __restrict__ QKV, int ldq, float* __restrict__ O, int ldo, int N_rt,
                                   int S, int dh_rt, int dmodel, float scale, int TB) {
  DQMC_DYN_SMEM(smem_raw);
  const int N = NE ? NE : N_rt;
  const int dh = DH ? DH : dh_rt;
  const int PQ = dh + 4, NN = N * N, d4 = dh / 4;
  float* q = reinterpret_cast<float*>(smem_raw);
  float* k = q + N * PQ;
  float* v = k + N * PQ;
  float* qt = v + N * PQ;                    // [TB][N][PQ]
  float* kt = qt + (size_t)TB * N * PQ;
  float* vt = kt + (size_t)TB * N * PQ;
  float* olap = vt + (size_t)TB * N * PQ;    // [N][dh]   (16B aligned: all sizes above are multiples of 4 floats)
  float* p = olap + N * dh;                  // [N][N]
  float* st = p + NN;                        // [TB][N][N]
  float* ctp = st + (size_t)TB * NN;         // [TB][N][N]
  float* u = ctp + (size_t)TB * NN;          // [N][N]
  float* qk = u + NN;                        // [N][N]
  float* mrow = qk + NN;                     // [TB][N]
  float* vrow = mrow + TB * N;               // [N]
  const int b = blockIdx.x, h = blockIdx.y;
  const int tid = threadIdx.x, nt = blockDim.x;
  const int T3 = S > 1 ? S - 2 : 0;
  const size_t row0 = (size_t)b * N * S;
  // global -> shared with cp.async (16 B, L2 only): all copies of a chunk are in flight at once
  auto load3 = [&](int slot0, int nslot, float* dq_, float* dk_, float* dv_) {
    for (int idx = tid; idx < nslot * N * d4; idx += nt) {
      int e4 = idx % d4, i = (idx / d4) % N, t = idx / (d4 * N);
      const float4* src = (const float4*)(QKV + (row0 + (size_t)i * S + slot0 + t) * ldq + h * dh) + e4;
      int o = (t * N + i) * PQ + 4 * e4;
      cp_async16(dq_ + o, src);
      cp_async16(dk_ + o, src + dmodel / 4);
      cp_async16(dv_ + o, src + dmodel / 2);
    }
    cp_async_wait_all();
  };
  load3(0, 1, q, k, v);
  __syncthreads();
  for (int idx = tid; idx < NN; idx += nt) {
    int i = idx / N, j = idx % N;
    float a = 0.f;
    for (int e4 = 0; e4 < d4; ++e4) a += dot4(*(const float4*)(q + i * PQ + 4 * e4), *(const float4*)(k + j * PQ + 4 * e4));
    p[idx] = a * scale;
    u[idx] = 0.f;
    qk[idx] = 0.f;
  }
  for (int idx = tid; idx < N * dh; idx += nt) olap[idx] = 0.f;
  __syncthreads();
  for (int i = tid; i < N; i += nt) {  // softmax row i
    float mx = p[i * N];
    for (int j = 1; j < N; ++j) mx = fmaxf(mx, p[i * N + j]);
    float sum = 0.f;
    for (int j = 0; j < N; ++j) {
      float e = m_exp(p[i * N + j] - mx);
      p[i * N + j] = e;
      sum += e;
    }
    float inv = 1.f / sum;
    for (int j = 0; j < N; ++j) p[i * N + j] *= inv;
  }
  __syncthreads();
  for (int idx = tid; idx < N * d4; idx += nt) {
    int i = idx / d4, e4 = idx % d4;
    float4 a = make_float4(0, 0, 0, 0);
    for (int j = 0; j < N; ++j) fma4(a, p[i * N + j], *(const float4*)(v + j * PQ + 4 * e4));
    *(float4*)(O + (row0 + (size_t)i * S) * ldo + h * dh + 4 * e4) = a;
  }
  if (S == 1) return;
  const int e4_per = d4 / 4;  // each of the 4 cooperating lanes covers dh/4 floats = d4/4 float4
  for (int t0 = 0; t0 < T3; t0 += TB) {
    const int tc = T3 - t0 < TB ? T3 - t0 : TB;
    __syncthreads();  // previous chunk done with qt/kt/vt/st
    load3(1 + t0, tc, qt, kt, vt);
    __syncthreads();
    if constexpr (MMA) {
      attn_fl_mma_scores(q, k, qt, kt, st, qk, N, N, PQ, dh, tc, scale, tid, nt);
    } else {
    // ---- (t,i) x 4 lanes: a_j = q^t_i . k_j,  c_j = q^t_i . k^t_j ----------------------------
    {
      const int nitem = tc * N * 4;
      const int nround = (nitem + nt - 1) / nt;
      for (int rd = 0; rd < nround; ++rd) {
        const int idx = rd * nt + tid;
        const bool act = idx < nitem;
        const int eq = idx & 3, ti = act ? idx >> 2 : 0;  // ti = t*N + i
        const int t = ti / N;
        const float* own = qt + (size_t)ti * PQ + eq * (dh / 4);
        for (int j = 0; j < N; ++j) {
          const float* kj = k + j * PQ + eq * (dh / 4);
          const float* ktj = kt + (size_t)(t * N + j) * PQ + eq * (dh / 4);
          float a = 0.f, c = 0.f;
          if (act) {
            for (int e4 = 0; e4 < e4_per; ++e4) {
              float4 x = *(const float4*)(own + 4 * e4);
              a += dot4(x, *(const float4*)(kj + 4 * e4));
              c += dot4(x, *(const float4*)(ktj + 4 * e4));
            }
          }
          a += __shfl_xor_sync(0xffffffffu, a, 1); a += __shfl_xor_sync(0xffffffffu, a, 2);
          c += __shfl_xor_sync(0xffffffffu, c, 1); c += __shfl_xor_sync(0xffffffffu, c, 2);
          if (act && eq == 0) { st[(size_t)ti * N + j] = a; ctp[(size_t)ti * N + j] = c; }
        }
      }
    }
    __syncthreads();
    // ---- (t,j) x 4 lanes: b_i = k^t_j . q_i ; st = scale (a + b) -------------------------------
    {
      const int nitem = tc * N * 4;
      const int nround = (nitem + nt - 1) / nt;
      for (int rd = 0; rd < nround; ++rd) {
        const int idx = rd * nt + tid;
        const bool act = idx < nitem;
        const int eq = idx & 3, tj = act ? idx >> 2 : 0;
        const int t = tj / N, j = tj % N;
        const float* own = kt + (size_t)tj * PQ + eq * (dh / 4);
        for (int i = 0; i < N; ++i) {
          const float* qi = q + i * PQ + eq * (dh / 4);
          float bsum = 0.f;
          if (act)
            for (int e4 = 0; e4 < e4_per; ++e4) bsum += dot4(*(const float4*)(own + 4 * e4), *(const float4*)(qi + 4 * e4));
          bsum += __shfl_xor_sync(0xffffffffu, bsum, 1); bsum += __shfl_xor_sync(0xffffffffu, bsum, 2);
          if (act && eq == 0) {
            const size_t o = ((size_t)t * N + i) * N + j;
            st[o] = scale * (st[o] + bsum);
          }
        }
      }
    }
    }  // SIMT scores
    __syncthreads();
    for (int idx = tid; idx < tc * N; idx += nt) {  // (t, i)
      const float* pr = p + (idx % N) * N;
      const float* sr = st + (size_t)idx * N;
      float m = 0.f;
      for (int j = 0; j < N; ++j) m += pr[j] * sr[j];
      mrow[idx] = m;
    }
    __syncthreads();
    for (int idx = tid; idx < NN; idx += nt) {
      int i = idx / N;
      float uu = 0.f, cc = 0.f, pp = p[idx];
      for (int t = 0; t < tc; ++t) {
        float dv_ = st[t * NN + idx] - mrow[t * N + i];
        uu += dv_ * dv_;
        if constexpr (!MMA) cc += ctp[t * NN + idx];
        st[t * NN + idx] = pp * dv_;  // p^t
      }
      u[idx] += uu;
      if constexpr (!MMA) qk[idx] += cc;
    }
    __syncthreads();
    if constexpr (MMA) {
      attn_fl_mma_outputs(st, p, v, vt, olap, O + (row0 + 1 + t0) * ldo + h * dh, (size_t)ldo, (size_t)S * ldo, N, N, PQ, dh, tc, tid, nt);
    } else
    for (int idx = tid; idx < N * d4; idx += nt) {
      int i = idx / d4, e4 = idx % d4;
      float4 c2 = make_float4(0, 0, 0, 0);
      for (int t = 0; t < tc; ++t) {
        const float* sr = st + t * NN + i * N;
        float4 a = make_float4(0, 0, 0, 0);
        for (int j = 0; j < N; ++j) {
          float4 vtj = *(const float4*)(vt + (size_t)(t * N + j) * PQ + 4 * e4);
          float4 vj = *(const float4*)(v + j * PQ + 4 * e4);
          float sj = sr[j];
          fma4(a, sj, vj);
          fma4(a, p[i * N + j], vtj);
          fma4(c2, sj, vtj);
        }
        *(float4*)(O + (row0 + (size_t)i * S + 1 + t0 + t) * ldo + h * dh + 4 * e4) = a;
      }
      float4* ol = (float4*)(olap + i * dh + 4 * e4);
      float4 o = *ol;
      o.x += 2.f * c2.x; o.y += 2.f * c2.y; o.z += 2.f * c2.z; o.w += 2.f * c2.w;
      *ol = o;
    }
  }
  __syncthreads();
  load3(1 + T3, 1, qt, kt, vt);
  __syncthreads();
  for (int idx = tid; idx < NN; idx += nt) {
    int i = idx / N, j = idx % N;
    float a = 0.f;
    for (int e4 = 0; e4 < d4; ++e4)
      a += dot4(*(const float4*)(qt + i * PQ + 4 * e4), *(const float4*)(k + j * PQ + 4 * e4)) +
           dot4(*(const float4*)(q + i * PQ + 4 * e4), *(const float4*)(kt + j * PQ + 4 * e4));
    st[idx] = scale * (a + 2.f * qk[idx]);
  }
  __syncthreads();
  for (int i = tid; i < N; i += nt) {
    float m = 0.f, V = 0.f;
    for (int j = 0; j < N; ++j) {
      m += p[i * N + j] * st[i * N + j];
      V += p[i * N + j] * u[i * N + j];
    }
    mrow[i] = m;
    vrow[i] = V;
  }
  __syncthreads();
  for (int idx = tid; idx < NN; idx += nt) {
    int i = idx / N;
    st[idx] = p[idx] * (u[idx] - vrow[i] + st[idx] - mrow[i]);
  }
  __syncthreads();
  for (int idx = tid; idx < N * d4; idx += nt) {
    int i = idx / d4, e4 = idx % d4;
    float4 a = *(const float4*)(olap + i * dh + 4 * e4);
    for (int j = 0; j < N; ++j) {
      fma4(a, st[i * N + j], *(const float4*)(v + j * PQ + 4 * e4));
      fma4(a, p[i * N + j], *(const float4*)(vt + j * PQ + 4 * e4));
    }
    *(float4*)(O + (row0 + (size_t)i * S + 1 + T3) * ldo + h * dh + 4 * e4) = a;
  }
}

inline size_t attn_f32_smem_bytes(int N, int dh, int TB) {
  return sizeof(float) * ((size_t)3 * N * (dh + 4) + (size_t)3 * TB * N * (dh + 4) + (size_t)N * dh +
                          (size_t)N * N * (3 + 2 * TB) + (size_t)TB * N + N + 8);
}
inline int attn_f32_pick_tb(int N, int dh, int T3, size_t budget) {
  int tb = T3 > 0 ? T3 : 1;
  while (tb > 1 && attn_f32_smem_bytes(N, dh, tb) > budget) --tb;
  if (tb < 4 && T3 >= 4) {  // large molecules: allow up to ~200 KB for at least 4 tangents per chunk
    tb = 4;
    while (tb > 1 && attn_f32_smem_bytes(N, dh, tb) > (size_t)200 * 1024) --tb;
  }
  if (T3 > 0) {  // balance the chunks
    int nchunk = (T3 + tb - 1) / tb;
    tb = (T3 + nchunk - 1) / nchunk;
  }
  return tb;
}

}  // namespace dq

namespace dq {

// ------------------------------------------------------------------------------------------
// FermiNet two-electron stream, initial features.  reference: src/deepqmc/gnn/graph.py:23-31
// (edges = receiver - sender), :197-215 'up'/'down' builders (senders = spin-up / spin-down
// electrons, receivers = all electrons, self-interaction kept), gnn/edge_features.py:42-78
// ([|d| eps-safe, d]), conf/ansatz/ferminet.yaml:58-72.
// E[b][j][i][s][4]: sender j (0..N-1; j < n_up are the 'up' senders), receiver i, slot s.
// One thread per (b, j, i).
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void edge_feat_kernel(const T* __restrict__ r, int N, int S, T* __restrict__ E, int total,
                                 const T* __restrict__ QA /*pseudo-Hamiltonian metric or null*/) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int i = idx % N, j = (idx / N) % N, b = idx / (N * N);
  const T* rb = r + (size_t)b * N * 3;
  T* e = E + (size_t)idx * S * 4;
  T dx[3] = {rb[3 * i] - rb[3 * j], rb[3 * i + 1] - rb[3 * j + 1], rb[3 * i + 2] - rb[3 * j + 2]};
  T d2 = dx[0] * dx[0] + dx[1] * dx[1] + dx[2] * dx[2];
  T rho2 = Num<T>::eps() + d2, rho = m_sqrt(rho2);
  e[0] = rho; e[1] = dx[0]; e[2] = dx[1]; e[3] = dx[2];
  if (S == 1) return;
  const int T3 = S - 2;
  if (QA) {
    // pseudo-Hamiltonian: the tangent slots of electron n are the columns of Q_n, second derivatives carry A_n
    // (common.cuh PhMetric): d/dv_{n,c} d = +-Q_n[:, c], Lap rho = sum_{n in (i, j)} (tr A_n - u^T A_n u) / rho
    PhMetric<T> pi, pj;
    pi.load(QA + ((size_t)b * N + i) * PH_STRIDE);
    pj.load(QA + ((size_t)b * N + j) * PH_STRIDE);
    const T u0 = dx[0] / rho, u1 = dx[1] / rho, u2 = dx[2] / rho;
    for (int t = 0; t < T3; ++t) {
      const int el = t / 3, c = t % 3;
      T* et = e + (size_t)(1 + t) * 4;
      T q0 = T(0), q1 = T(0), q2 = T(0);  // +-column c of Q_el (lower triangular: q00 q10 q11 q20 q21 q22)
      if (i != j && (el == i || el == j)) {
        const PhMetric<T>& pm = el == i ? pi : pj;
        const T sg = el == i ? T(1) : T(-1);
        q0 = c == 0 ? sg * pm.q[0] : T(0);
        q1 = c == 0 ? sg * pm.q[1] : (c == 1 ? sg * pm.q[2] : T(0));
        q2 = c == 0 ? sg * pm.q[3] : (c == 1 ? sg * pm.q[4] : sg * pm.q[5]);
      }
      et[0] = u0 * q0 + u1 * q1 + u2 * q2;
      et[1] = q0; et[2] = q1; et[3] = q2;
    }
    T* el = e + (size_t)(1 + T3) * 4;
    T lap = T(0);
    if (i != j) {
      T a0, a1, a2;
      pi.mul(u0, u1, u2, a0, a1, a2);
      lap += (pi.trace() - (u0 * a0 + u1 * a1 + u2 * a2)) / rho;
      pj.mul(u0, u1, u2, a0, a1, a2);
      lap += (pj.trace() - (u0 * a0 + u1 * a1 + u2 * a2)) / rho;
    }
    el[0] = lap;
    el[1] = el[2] = el[3] = T(0);
    return;
  }
  for (int t = 0; t < T3; ++t) {
    const int el = t / 3, c = t % 3;
    T sgn = T(0);
    if (i != j) sgn = el == i ? T(1) : (el == j ? T(-1) : T(0));
    T* et = e + (size_t)(1 + t) * 4;
    et[0] = sgn * dx[c] / rho;
    et[1] = c == 0 ? sgn : T(0);
    et[2] = c == 1 ? sgn : T(0);
    et[3] = c == 2 ? sgn : T(0);
  }
  T* el = e + (size_t)(1 + T3) * 4;
  el[0] = i != j ? T(2) * (T(3) / rho - d2 / (rho2 * rho)) : T(0);
  el[1] = el[2] = el[3] = T(0);
}

// ------------------------------------------------------------------------------------------
// FermiNet node-update input: F[b][i][s][:] = [h_i, mean_up h, mean_down h, mean_{j in up} e_ji,
// mean_{j in down} e_ji]  (reference: gnn/update_features.py:47-159 Residual / NodeSum / EdgeSum
// features with normalize = true, electron_gnn.py:243-259 'concatenate').  All linear, so it acts
// slot-wise on the augmented rows.  grid = (B*S, N), block over features.
// ------------------------------------------------------------------------------------------
template <class T>
__global__ void fermi_agg_kernel(const T* __restrict__ H, int dh, const T* __restrict__ E, int de, int N, int n_up,
                                 int S, T* __restrict__ F) {
  const int bs = blockIdx.x, b = bs / S, s = bs % S, i = blockIdx.y;
  const int ldf = 3 * dh + 2 * de;
  T* f = F + ((size_t)(b * N + i) * S + s) * ldf;
  const int n_dn = N - n_up;
  for (int k = threadIdx.x; k < ldf; k += blockDim.x) {
    T v;
    if (k < dh) {
      v = H[((size_t)(b * N + i) * S + s) * dh + k];
    } else if (k < 3 * dh) {
      const bool up = k < 2 * dh;
      const int kk = up ? k - dh : k - 2 * dh;
      const int j0 = up ? 0 : n_up, j1 = up ? n_up : N;
      T acc = T(0);
      for (int j = j0; j < j1; ++j) acc += H[((size_t)(b * N + j) * S + s) * dh + kk];
      v = acc / (T)(up ? n_up : n_dn);
    } else {
      const bool up = k < 3 * dh + de;
      const int kk = up ? k - 3 * dh : k - 3 * dh - de;
      const int j0 = up ? 0 : n_up, j1 = up ? n_up : N;
      T acc = T(0);
      for (int j = j0; j < j1; ++j) acc += E[(((size_t)(b * N + j) * N + i) * S + s) * de + kk];
      v = acc / (T)(up ? n_up : n_dn);
    }
    f[k] = v;
  }
}

}  // namespace dq
