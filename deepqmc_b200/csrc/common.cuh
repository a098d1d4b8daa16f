// Shared device helpers for the local-energy engine (sm_90a).
// Compiles under nvcc (product) and, with -DDQMC_EMU, under g++ against
// tools/cuda_emu/cuda_emu.h (development-time logic checks only, never shipped).
#pragma once
#ifdef DQMC_EMU
#include "cuda_emu.h"
#else
#include <cuda_runtime.h>
#define DQMC_DYN_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
#define DQMC_LAUNCH(kern, grid, block, smem, stream, ...) kern<<<grid, block, smem, stream>>>(__VA_ARGS__)
#endif
#include <cmath>
#include <cstdint>

namespace dq {

template <class T> struct Num;
template <> struct Num<double> {
  // eps of the eps-safe norm: jnp.finfo(dtype).eps (reference: src/deepqmc/utils.py:79-85)
  static __host__ __device__ __forceinline__ double eps() { return 2.220446049250313e-16; }
};
template <> struct Num<float> {
  static __host__ __device__ __forceinline__ float eps() { return 1.1920928955078125e-07f; }
};

__host__ __device__ __forceinline__ double m_exp(double x) { return ::exp(x); }
__host__ __device__ __forceinline__ float m_exp(float x) { return ::expf(x); }
__host__ __device__ __forceinline__ double m_log(double x) { return ::log(x); }
__host__ __device__ __forceinline__ float m_log(float x) { return ::logf(x); }
__host__ __device__ __forceinline__ double m_log1p(double x) { return ::log1p(x); }
__host__ __device__ __forceinline__ float m_log1p(float x) { return ::log1pf(x); }
__host__ __device__ __forceinline__ double m_tanh(double x) { return ::tanh(x); }
__host__ __device__ __forceinline__ float m_tanh(float x) { return ::tanhf(x); }
__host__ __device__ __forceinline__ double m_sqrt(double x) { return ::sqrt(x); }
__host__ __device__ __forceinline__ float m_sqrt(float x) { return ::sqrtf(x); }
__host__ __device__ __forceinline__ double m_abs(double x) { return ::fabs(x); }
__host__ __device__ __forceinline__ float m_abs(float x) { return ::fabsf(x); }
__host__ __device__ __forceinline__ double m_cos(double x) { return ::cos(x); }
__host__ __device__ __forceinline__ float m_cos(float x) { return ::cosf(x); }
__host__ __device__ __forceinline__ double m_sin(double x) { return ::sin(x); }
__host__ __device__ __forceinline__ float m_sin(float x) { return ::sinf(x); }

// 16-byte asynchronous global -> shared copy (LDGSTS, bypasses L1 and registers)
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
#ifdef DQMC_EMU
  *reinterpret_cast<float4*>(smem_dst) = *reinterpret_cast<const float4*>(gmem_src);
#else
  unsigned sa = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gmem_src) : "memory");
#endif
}
__device__ __forceinline__ void cp_async_wait_all() {
#ifndef DQMC_EMU
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
#endif
}

// 4 consecutive elements with ONE memory instruction where the type allows it (float: 128-bit).
// The pointer must be 16-byte aligned for T = float.
template <class T>
__device__ __forceinline__ void ld4(const T* p, T (&v)[4]) {
  if constexpr (sizeof(T) == 4) {
    const float4 q = *reinterpret_cast<const float4*>(p);
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  } else {
    v[0] = p[0]; v[1] = p[1]; v[2] = p[2]; v[3] = p[3];
  }
}
template <class T>
__device__ __forceinline__ void st4(T* p, const T (&v)[4]) {
  if constexpr (sizeof(T) == 4) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
    p[0] = v[0]; p[1] = v[1]; p[2] = v[2]; p[3] = v[3];
  }
}

// The (up, down) pair that virtual walker p of the spin pass swaps (reference: physics.py:186-223).  down_idx < 0: exact
// estimator, all n_up n_down pairs, p = a n_down + (beta - n_up); otherwise spin-raising, beta = down_idx and p = a.
__host__ __device__ __forceinline__ void spin_pair(int p, int n_up, int N, int down_idx, int& a, int& beta) {
  if (down_idx < 0) {
    const int nd = N - n_up;
    a = p / nd;
    beta = n_up + (p - a * nd);
  } else {
    a = p;
    beta = down_idx;
  }
}

// Non-local ECP cutoff: the (electron, ECP nucleus) pair at squared distance d2 runs its 12 quadrature forwards unless d2 exceeds
// rc2, the nucleus' squared cutoff radius (engine.cu ecp_cutoff_rc2: beyond it sum_l (2l+1) sum_t |beta_lt| exp(-alpha_lt d2)
// < 2^-100).  d2 in double, as ecp_accumulate_kernel weights the pair; the pair list builder (ecp_pairs_kernel) and the
// accumulator both decide here.  A NaN distance keeps its pair, so rc2 = +inf (DQMC_ECP_CUTOFF=0) keeps every pair of every walker.
template <class T>
__host__ __device__ __forceinline__ bool ecp_pair_active(const T* ri, const T* RI, double rc2, double& d2) {
  const double dx = (double)ri[0] - (double)RI[0], dy = (double)ri[1] - (double)RI[1], dz = (double)ri[2] - (double)RI[2];
  d2 = dx * dx + dy * dy + dz * dz;
  return !(d2 > rc2);
}

// Compact virtual-walker forwards: virtual walker v is a base walker with one or two electrons moved; the consumers
// (embed_fwd_kernel, the whole-trunk kernel's tile load, slater_fwd2_kernel) take every other electron's rows from tables of
// the base walkers.  Two layouts:
//   layout == kVirtEcp: non-local ECP quadrature (ecp_points_kernel, v = 12 a + q): active pair a of the group's pair list
//     (ecp_pairs_kernel) is p = pairs[a] = (w J + j) N + i, vper = 12 J N; base walker w = p / (J N), electron e0 = p % N moved
//     to a quadrature point, e1 = -1;
//   layout >= -1: spin swaps (spin_pairs_kernel, v = w vper + p): base walker v / vper, up electron e0 and down electron e1 of
//     pair p exchange positions; layout is the down_idx of spin_pair (-1: all pairs); pairs is unused.
constexpr int kVirtEcp = -2;
// Virtual-walker indices are 32-bit: a group's virtual walkers are one plain-forward batch (int walker count).
struct VirtualMove {
  int base, e0, e1;
};
__host__ __device__ __forceinline__ VirtualMove virtual_move(int v, int vper, int N, int n_up, int layout, const int* pairs) {
  VirtualMove m;
  if (layout == kVirtEcp) {
    const int p = pairs[v / 12];
    m.base = p / (vper / 12);
    m.e0 = p % N;
    m.e1 = -1;
  } else {
    m.base = v / vper;
    spin_pair(v - m.base * vper, n_up, N, layout, m.e0, m.e1);
  }
  return m;
}

template <class T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Sum over the whole block; result valid in every thread. scratch: >= 33 T's of shared memory.
// Requires blockDim.x % 32 == 0 and all threads to call it.
template <class T>
__device__ __forceinline__ T block_sum(T v, T* scratch) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  v = warp_sum(v);
  __syncthreads();  // protect scratch from a previous use
  if (lane == 0) scratch[w] = v;
  __syncthreads();
  if (w == 0) {
    T x = lane < nw ? scratch[lane] : T(0);
    x = warp_sum(x);
    if (lane == 0) scratch[32] = x;
  }
  __syncthreads();
  return scratch[32];
}

template <class T>
__device__ __forceinline__ void block_sum2(T& a, T& b, T* scratch) {
  // scratch: >= 66 T's
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  a = warp_sum(a);
  b = warp_sum(b);
  __syncthreads();
  if (lane == 0) { scratch[w] = a; scratch[33 + w] = b; }
  __syncthreads();
  if (w == 0) {
    T x = lane < nw ? scratch[lane] : T(0);
    T y = lane < nw ? scratch[33 + lane] : T(0);
    x = warp_sum(x);
    y = warp_sum(y);
    if (lane == 0) { scratch[32] = x; scratch[65] = y; }
  }
  __syncthreads();
  a = scratch[32];
  b = scratch[65];
}


// ---- Pseudo-Hamiltonian helpers (reference ecp/pseudo_hamiltonian.py:165-278) -------------
// The PH replaces -1/2 Laplacian by  sum_i [ A(r_i) : Hess_i + b(r_i) . grad_i ]  with a symmetric positive
// 3x3 matrix A per electron.  The reference evaluates it as a plain Laplacian in coordinates v = Q^-1 r,
// A = Q Q^T; the forward-Laplacian engine does the same by seeding the tangent slots of electron i with the
// columns of Q_i and weighting the second derivatives of every function of r_i with A_i.
// Per (walker, electron) record of PH_STRIDE values: Q lower triangle (q00 q10 q11 q20 q21 q22),
// A (a00 a01 a02 a11 a12 a22), b (3).
constexpr int PH_STRIDE = 16;

template <class T>
struct PhMetric {  // second-derivative weights of a radial function of d = r_i - c, rho = |d| (or its eps-safe version)
  T q[6], a[6];
  __device__ __forceinline__ void load(const T* rec) {
#pragma unroll
    for (int k = 0; k < 6; ++k) { q[k] = rec[k]; a[k] = rec[6 + k]; }
  }
  __device__ __forceinline__ T trace() const { return a[0] + a[3] + a[5]; }
  // (A u)
  __device__ __forceinline__ void mul(T u0, T u1, T u2, T& o0, T& o1, T& o2) const {
    o0 = a[0] * u0 + a[1] * u1 + a[2] * u2;
    o1 = a[1] * u0 + a[3] * u1 + a[4] * u2;
    o2 = a[2] * u0 + a[4] * u1 + a[5] * u2;
  }
  // gradient w.r.t. r -> gradient w.r.t. v (Q^T g)
  __device__ __forceinline__ void to_v(T& g0, T& g1, T& g2) const {
    g0 = q[0] * g0 + q[1] * g1 + q[3] * g2;
    g1 = q[2] * g1 + q[4] * g2;
    g2 = q[5] * g2;
  }
  // gradient w.r.t. v -> gradient w.r.t. r (solve Q^T x = g)
  __device__ __forceinline__ void to_r(T& g0, T& g1, T& g2) const {
    g2 = g2 / q[5];
    g1 = (g1 - q[4] * g2) / q[2];
    g0 = (g0 - q[1] * g1 - q[3] * g2) / q[0];
  }
};

// linear interpolation on the uniform grid [0, rmax] with G points, 0 outside
// (jax.scipy.interpolate.RegularGridInterpolator(method='linear', fill_value=0), pseudo_hamiltonian.py:95-101)
template <class T>
__device__ __forceinline__ T ph_interp(const T* __restrict__ tab, int G, T rmax, T x) {
  if (!(x >= T(0) && x <= rmax)) return T(0);
  const T t = x * (T(G - 1) / rmax);
  int i0 = (int)t;
  if (i0 > G - 2) i0 = G - 2;
  const T w = t - T(i0);
  return tab[i0] + w * (tab[i0 + 1] - tab[i0]);
}

template <class T>
struct PhArgs {  // all null / 0: no pseudo-Hamiltonian
  const T* QA = nullptr;          // [walkers][N][PH_STRIDE]
  const T* tabs = nullptr;        // [n_tab][2][G]: r V_loc, r V_L2
  const int* tab_of_nuc = nullptr;  // [M] table index or -1
  int G = 0;
  T rmax = T(0);
};

// A, b, Q of every (walker, electron): compute_coefficients_of_differential_operators + Cholesky
// (pseudo_hamiltonian.py:198-233,254-259).  One thread per electron.
template <class T>
__global__ void ph_coeff_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M,
                                PhArgs<T> ph, T* __restrict__ QA, int total) {
  const int bi = blockIdx.x * blockDim.x + threadIdx.x;
  if (bi >= total) return;
  const int b = bi / N;
  const T* ri = r + (size_t)bi * 3;
  const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
  T a00 = T(0.5), a01 = T(0), a02 = T(0), a11 = T(0.5), a12 = T(0), a22 = T(0.5), b0 = T(0), b1 = T(0), b2 = T(0);
  for (int m = 0; m < M; ++m) {
    const int tb = ph.tab_of_nuc[m];
    if (tb < 0) continue;
    const T d0 = ri[0] - Rb[3 * m], d1 = ri[1] - Rb[3 * m + 1], d2 = ri[2] - Rb[3 * m + 2];
    const T dd = d0 * d0 + d1 * d1 + d2 * d2, dist = m_sqrt(dd);
    const T rv = ph_interp(ph.tabs + ((size_t)tb * 2 + 1) * ph.G, ph.G, ph.rmax, dist);
    const T v = rv / dist;  // V_L2
    b0 += T(2) * v * d0; b1 += T(2) * v * d1; b2 += T(2) * v * d2;
    const T dg = rv * dist;
    a00 += dg - v * d0 * d0; a11 += dg - v * d1 * d1; a22 += dg - v * d2 * d2;
    a01 -= v * d0 * d1; a02 -= v * d0 * d2; a12 -= v * d1 * d2;
  }
  T* o = QA + (size_t)bi * PH_STRIDE;
  const T q00 = m_sqrt(a00), q10 = a01 / q00, q20 = a02 / q00;
  const T q11 = m_sqrt(a11 - q10 * q10), q21 = (a12 - q20 * q10) / q11;
  const T q22 = m_sqrt(a22 - q20 * q20 - q21 * q21);
  o[0] = q00; o[1] = q10; o[2] = q11; o[3] = q20; o[4] = q21; o[5] = q22;
  o[6] = a00; o[7] = a01; o[8] = a02; o[9] = a11; o[10] = a12; o[11] = a22;
  o[12] = b0; o[13] = b1; o[14] = b2; o[15] = T(0);
}

// ---- Philox4x32-10 counter-based generator (Salmon et al. 2011), hand-written ---------
struct Philox {
  static __host__ __device__ __forceinline__ void mulhilo(uint32_t a, uint32_t b, uint32_t& hi, uint32_t& lo) {
    uint64_t p = (uint64_t)a * b;
    hi = (uint32_t)(p >> 32);
    lo = (uint32_t)p;
  }
  static __host__ __device__ __forceinline__ void gen(uint64_t key, uint64_t ctr_lo, uint64_t ctr_hi, uint32_t out[4]) {
    uint32_t c0 = (uint32_t)ctr_lo, c1 = (uint32_t)(ctr_lo >> 32), c2 = (uint32_t)ctr_hi, c3 = (uint32_t)(ctr_hi >> 32);
    uint32_t k0 = (uint32_t)key, k1 = (uint32_t)(key >> 32);
#pragma unroll
    for (int r = 0; r < 10; ++r) {
      uint32_t h0, l0, h1, l1;
      mulhilo(0xD2511F53u, c0, h0, l0);
      mulhilo(0xCD9E8D57u, c2, h1, l1);
      uint32_t n0 = h1 ^ c1 ^ k0, n1 = l1, n2 = h0 ^ c3 ^ k1, n3 = l0;
      c0 = n0; c1 = n1; c2 = n2; c3 = n3;
      k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
  }
  // uniform in (0,1)
  static __host__ __device__ __forceinline__ double u01(uint32_t a, uint32_t b) {
    uint64_t x = ((uint64_t)a << 21) ^ (uint64_t)(b >> 11);  // 53 bits
    x &= ((1ull << 53) - 1);
    return ((double)x + 0.5) * (1.0 / 9007199254740992.0);
  }
};

}  // namespace dq
