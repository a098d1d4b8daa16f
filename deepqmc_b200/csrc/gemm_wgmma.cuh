// fp32-accurate dense-layer GEMM on the Hopper tensor cores (sm_90a, wgmma): 3xTF32 split
//   C[row(m), :] = (Res) + A[row(m), :] @ W + (bias on value rows),  A, W, C fp32 in HBM.
//
//   a = a_hi + a_lo, w = w_hi + w_lo with *_hi = rna_tf32(.), *_lo = rna_tf32(. - *_hi) (both exactly representable in TF32);
//   acc(fp32, registers) = a_lo w_hi + a_hi w_hi + a_hi w_lo     -> ~2^-21 relative per product,
//   i.e. the accuracy class the reference demands (jax_default_matmul_precision='highest',
//   NVIDIA_TF32_OVERRIDE=0: src/deepqmc/__init__.py:9-34) at 1/3 of the TF32 tensor peak.
//
// F16 = true (plain forwards, S = 1): the same kernel with IEEE-half operands -- "3xFP16":
//   a 2^ea = a_hi + a_lo, w 2^ew = w_hi + w_lo with *_hi = rn_half(.), *_lo = rn_half(. - *_hi): 22 significant bits,
//   products exact in the fp32 accumulator, power-of-two scales undone in the epilogue (exact).  f16 wgmma runs at twice
//   the tf32 rate and a 128-byte swizzle row holds 64 k-values instead of 32, so a shared-memory stage covers twice
//   the K extent.  Halves below 2^-14 are subnormal (absolute spacing 2^-24): the scales keep O(1) activations and the
//   weights of a layer far above that, the absolute floor is ~2^-25 / 2^ea per activation.  Only plain forwards use it
//   (values bounded by construction: residual stream, tanh outputs, attention averages); the forward-Laplacian rows
//   (derivative slots of unbounded dynamic range) stay on 3xTF32.
//
// One CTA per tile of up to 128 rows x kBN columns, 256 threads = two warpgroups of 64 rows each:
//   all threads  : global fp32 rows of the next k-block -> split hi/lo -> 128B-swizzled K-major shared memory
//   thread 0     : TMA (cp.async.bulk.tensor) of the pre-split W^T hi/lo tiles of the next k-block (mbarrier)
//   warpgroups   : wgmma m64n128 on the current k-block, accumulators in registers
// two shared-memory stages: the loads / split of k-block i + 1 run under the MMAs of k-block i.  The epilogue (bias, residual,
// tanh with forward-Laplacian propagation) runs from a shared-memory copy of the accumulator tile that re-uses the stages.
// W^T (N x K, K contiguous) is split into hi/lo once per parameter upload (engine.cu).
#pragma once
#include <cstdint>

#include "tc_ptx.cuh"

namespace dq {
namespace tc {

constexpr int kBM = 128;          // rows per tile (two warpgroups x 64)
constexpr int kBN = 128;          // columns per tile (wgmma N)
constexpr int kBK = 32;           // fp32 per k-block = 128 bytes = one swizzle row
constexpr int kThreads = 256;

struct Params {
  const float* A; int lda;
  const float* bias;
  const float* Res; int ldr;
  float* C; int ldc;
  int M, N, K;
  int S;
  int sliced, Nel, z_split;
  int act;           // 0: none, 1: tanh with forward-Laplacian propagation fused into the epilogue
  int rpt;           // rows per tile (<= 128): G*S for act = 1 so that slot groups never straddle tiles
  int* err_flag;     // device int: set to non-zero if a barrier wait times out
  float a_scale;     // F16: activations are multiplied by this power of two before the split ...
  float unscale;     // ... and the accumulator by 2^-(ea + ew) in the epilogue
};

// tanh for the plain-forward epilogue: odd polynomial below |x| = 0.15, 1 - 2 / (1 + e^{2x})
// (ex2.approx + fast division) above; absolute error <= ~3e-7.  The forward-Laplacian epilogue
// keeps tanhf (derivative slots amplify the error); plain forwards only feed log|psi| ratios.
__device__ __forceinline__ float tanh_fwd(float x) {
  const float x2 = x * x;
  const float poly = x + x * x2 * (-0.33333333333f + x2 * (0.13333333333f + x2 * (-0.05396825397f)));
  const float e = ex2_approx(x * 2.8853900817779268f);
  const float big = 1.f - fast_div(2.f, 1.f + e);
  return fabsf(x) < 0.15f ? poly : big;
}

__device__ __forceinline__ size_t phys_row(const Params& p, int m, int z) {
  if (!p.sliced) return (size_t)m;
  int b = m / p.S, s = m % p.S;
  return ((size_t)b * p.Nel + z) * p.S + s;
}

struct SmemLayout {
  static constexpr int kStageBytes = 4 * kBM * 128;  // A hi, A lo, W hi, W lo: 128 rows x 128 B each
  static constexpr int kPitch = kBN + 4;             // fp32 accumulator tile of the epilogue (re-uses the stages)
  static __host__ __device__ int a_hi(int s) { return s * kStageBytes; }
  static __host__ __device__ int a_lo(int s) { return s * kStageBytes + kBM * 128; }
  static __host__ __device__ int w_hi(int s) { return s * kStageBytes + 2 * kBM * 128; }
  static __host__ __device__ int w_lo(int s) { return s * kStageBytes + 3 * kBM * 128; }
  static __host__ __device__ int bars() { return 2 * kStageBytes; }
  static __host__ __device__ int total() { return bars() + 64; }
};
static_assert(kBM * SmemLayout::kPitch * 4 <= 2 * SmemLayout::kStageBytes, "epilogue tile must fit the stages");

template <bool F16>
__global__ void __launch_bounds__(kThreads, 1)
gemm3x_kernel(const __grid_constant__ CUtensorMap map_hi0, const __grid_constant__ CUtensorMap map_lo0,
              const __grid_constant__ CUtensorMap map_hi1, const __grid_constant__ CUtensorMap map_lo1, Params p) {
  DQMC_TC_SMEM(smem);
  if ((smem_u32(smem) & 1023u) != 0u) tc_trap();
  uint64_t* full = (uint64_t*)(smem + SmemLayout::bars());  // [2] W tiles of a stage landed (TMA tx)
  const int tid = threadIdx.x, wg = tid >> 7;
  const int RPT = p.rpt;
  const int MT = (p.M + RPT - 1) / RPT, NT = (p.N + kBN - 1) / kBN;
  const int tile = blockIdx.x;
  const int nt = tile % NT, mt = (tile / NT) % MT, z = tile / (NT * MT);
  // k-blocks of 32 floats per stage; F16: two of them (64 halves = one 128-byte swizzle row)
  constexpr int kSub = F16 ? 2 : 1;
  const int KS = p.K / (kBK * kSub);
  const bool second = p.sliced && z >= p.z_split;
  const CUtensorMap* mh = second ? &map_hi1 : &map_hi0;
  const CUtensorMap* ml = second ? &map_lo1 : &map_lo0;

  if (tid == 0) {
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    fence_barrier_init();
    tma_prefetch_desc(mh);
    tma_prefetch_desc(ml);
  }
  __syncthreads();
  auto issue_w = [&](int ks) {
    const int s = ks & 1;
    mbar_expect_tx(&full[s], 2u * kBN * 128u);
    tma_load_2d(mh, &full[s], smem + SmemLayout::w_hi(s), ks * kBK * kSub, nt * kBN);
    tma_load_2d(ml, &full[s], smem + SmemLayout::w_lo(s), ks * kBK * kSub, nt * kBN);
  };
  if (tid == 0) issue_w(0);

  // A rows of this thread: 16-byte chunk `chunk` of tile rows r0 + kRowStep i.  A warp instruction covers 4 (F16: 2) complete
  // 128-byte row segments.
  constexpr int kChunks = F16 ? 16 : 8;  // float4 per row and stage
  constexpr int kRows = kBM * kChunks / kThreads;
  constexpr int kRowStep = kThreads / kChunks;
  const int chunk = tid % kChunks, r0 = tid / kChunks;
  const float* rowp[kRows];
#pragma unroll
  for (int i = 0; i < kRows; ++i) {
    const int lrow = r0 + kRowStep * i, m = mt * RPT + lrow;
    rowp[i] = (lrow < RPT && m < p.M) ? p.A + phys_row(p, m, z) * p.lda + chunk * 4 : nullptr;
  }
  float4 av[kRows];
  auto load_a = [&](int ks) {
#pragma unroll
    for (int i = 0; i < kRows; ++i)
      av[i] = rowp[i] ? __ldg((const float4*)(rowp[i] + ks * kBK * kSub)) : make_float4(0.f, 0.f, 0.f, 0.f);
  };
  auto store_a = [&](int s) {
    unsigned char* ah = smem + SmemLayout::a_hi(s);
    unsigned char* al = smem + SmemLayout::a_lo(s);
#pragma unroll
    for (int i = 0; i < kRows; ++i) {
      const int trow = r0 + kRowStep * i;
      if constexpr (F16) {
        const float sc = p.a_scale;
        const float x0 = av[i].x * sc, x1 = av[i].y * sc, x2 = av[i].z * sc, x3 = av[i].w * sc;
        const uint32_t h01 = pack_half2_rn(x0, x1), h23 = pack_half2_rn(x2, x3);
        const uint32_t l01 = pack_half2_rn(x0 - half_bits_to_float(h01 & 0xFFFFu), x1 - half_bits_to_float(h01 >> 16));
        const uint32_t l23 = pack_half2_rn(x2 - half_bits_to_float(h23 & 0xFFFFu), x3 - half_bits_to_float(h23 >> 16));
        const int c16 = chunk >> 1;
        const int off = trow * 128 + ((c16 ^ (trow & 7)) << 4) + (chunk & 1) * 8;
        *(uint2*)(ah + off) = make_uint2(h01, h23);
        *(uint2*)(al + off) = make_uint2(l01, l23);
      } else {
        float4 v = av[i], h, l;
        h.x = tf32_rna(v.x); l.x = tf32_rna(v.x - h.x);
        h.y = tf32_rna(v.y); l.y = tf32_rna(v.y - h.y);
        h.z = tf32_rna(v.z); l.z = tf32_rna(v.z - h.z);
        h.w = tf32_rna(v.w); l.w = tf32_rna(v.w - h.w);
        const int off = trow * 128 + ((chunk ^ (trow & 7)) << 4);
        *(float4*)(ah + off) = h;
        *(float4*)(al + off) = l;
      }
    }
  };
  load_a(0);
  store_a(0);

  float acc[kBN / 2];
#pragma unroll
  for (int i = 0; i < kBN / 2; ++i) acc[i] = 0.f;
  for (int ks = 0; ks < KS; ++ks) {
    const int s = ks & 1;
    fence_proxy_async();  // generic-proxy writes of the A stage -> visible to the tensor cores (async proxy)
    __syncthreads();      // ... by every thread; every warpgroup is done with stage s ^ 1 (waited below)
    if (tid == 0 && ks + 1 < KS) issue_w(ks + 1);
    if (ks + 1 < KS) load_a(ks + 1);  // global loads in flight under the MMAs
    mbar_wait(&full[s], (ks >> 1) & 1, p.err_flag);
    const uint32_t ah = smem_u32(smem + SmemLayout::a_hi(s)) + wg * 8192, al = smem_u32(smem + SmemLayout::a_lo(s)) + wg * 8192;
    const uint32_t wh = smem_u32(smem + SmemLayout::w_hi(s)), wl = smem_u32(smem + SmemLayout::w_lo(s));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t ko = k * 32;  // byte offset inside the 128B swizzle row (tf32: 8 k-values, f16: 16)
      const int first = (ks | k) ? 1 : 0;
      if constexpr (F16) {
        wgmma_f16_n128(acc, make_desc(al + ko), make_desc(wh + ko), first);
        wgmma_f16_n128(acc, make_desc(ah + ko), make_desc(wh + ko), 1);
        wgmma_f16_n128(acc, make_desc(ah + ko), make_desc(wl + ko), 1);
      } else {
        wgmma_tf32_n128(acc, make_desc(al + ko), make_desc(wh + ko), first);
        wgmma_tf32_n128(acc, make_desc(ah + ko), make_desc(wh + ko), 1);
        wgmma_tf32_n128(acc, make_desc(ah + ko), make_desc(wl + ko), 1);
      }
    }
    wgmma_commit();
    wgmma_wait0();
    fence_acc(acc);
    if (ks + 1 < KS) store_a(s ^ 1);
  }
  __syncthreads();  // every MMA has retired: the stages become the epilogue tile

  // ===================== epilogue =================================================================
  constexpr int P = SmemLayout::kPitch;
  float* st = (float*)smem;  // [128][P]
  {
    const int lane = tid & 31;
    const int fr = 64 * wg + 16 * ((tid >> 5) & 3) + (lane >> 2), fc = 2 * (lane & 3);
    const float us = F16 ? p.unscale : 1.f;
#pragma unroll
    for (int j = 0; j < kBN / 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        *(float2*)(st + (fr + 8 * h) * P + 8 * j + fc) = make_float2(acc[4 * j + 2 * h] * us, acc[4 * j + 2 * h + 1] * us);
  }
  __syncthreads();
  const int S = p.S;
  const int rows_here = (p.M - mt * RPT) < RPT ? (p.M - mt * RPT) : RPT;
  const int col0 = nt * kBN;
  if (p.act) {
    if (S == 1) {  // plain forward: every row is a value row
      for (int idx = tid; idx < rows_here * kBN; idx += kThreads) {
        const int r = idx / kBN, c = idx % kBN;
        const float b = (p.bias && col0 + c < p.N) ? __ldg(p.bias + col0 + c) : 0.f;
        st[r * P + c] = tanh_fwd(st[r * P + c] + b);
      }
    } else {
      // tanh + forward-Laplacian propagation (reference: hkext.py:104-113 MLP activation; rule
      // y_t = y' z_t, y_L = y' z_L + y'' sum_t z_t^2).  Tiles hold whole slot groups (rpt = G*S); one thread per
      // (group, column) rewrites the group's S rows of that column in place.
      const int ngrp = rows_here / S;
      for (int idx = tid; idx < ngrp * kBN; idx += kThreads) {
        const int g = idx / kBN, c = idx % kBN;
        float* zp = st + g * S * P + c;
        const float b = (p.bias && col0 + c < p.N) ? __ldg(p.bias + col0 + c) : 0.f;
        const float y = tanhf(zp[0] + b);
        const float y1 = 1.f - y * y, y2 = -2.f * y * y1;
        float s0 = 0.f, s1 = 0.f;
        int t = 1;
        for (; t + 1 <= S - 2; t += 2) {
          const float a0 = zp[t * P], a1 = zp[(t + 1) * P];
          s0 += a0 * a0; s1 += a1 * a1;
        }
        for (; t <= S - 2; ++t) {
          const float a = zp[t * P];
          s0 += a * a;
        }
        zp[0] = y;
        for (int u = 1; u < S - 1; ++u) zp[u * P] *= y1;
        zp[(S - 1) * P] = y1 * zp[(S - 1) * P] + y2 * (s0 + s1);
      }
    }
    __syncthreads();
  }
  const float* __restrict__ Resp = p.Res;
  float* __restrict__ Cp = p.C;
  const bool vec_ok = (p.N % 4) == 0 && (p.ldc % 4) == 0 && (!Resp || (p.ldr % 4) == 0);
  if (vec_ok) {
    for (int idx = tid; idx < rows_here * (kBN / 4); idx += kThreads) {
      const int r = idx / (kBN / 4), c = 4 * (idx % (kBN / 4)), col = col0 + c;
      if (col >= p.N) continue;
      const size_t pr = phys_row(p, mt * RPT + r, z);
      float4 o = *(const float4*)(st + r * P + c);
      if (Resp) {
        const float4 q = __ldg((const float4*)(Resp + pr * p.ldr + col));
        o.x += q.x; o.y += q.y; o.z += q.z; o.w += q.w;
      }
      if (p.bias && !p.act && pr % S == 0) {
        const float4 q = __ldg((const float4*)(p.bias + col));
        o.x += q.x; o.y += q.y; o.z += q.z; o.w += q.w;
      }
      *(float4*)(Cp + pr * p.ldc + col) = o;
    }
  } else {  // ragged N: scalar path
    for (int idx = tid; idx < rows_here * kBN; idx += kThreads) {
      const int r = idx / kBN, c = idx % kBN, col = col0 + c;
      if (col >= p.N) continue;
      const size_t pr = phys_row(p, mt * RPT + r, z);
      float o = st[r * P + c];
      if (Resp) o += Resp[pr * p.ldr + col];
      if (p.bias && !p.act && pr % S == 0) o += p.bias[col];
      Cp[pr * p.ldc + col] = o;
    }
  }
}

// ---- host side -----------------------------------------------------------------------------
// W^T split tensors: [Nrows][K] fp32, K contiguous.  Box = 32 fp32 (128 B) x BN rows, 128B swizzle.
inline int make_weight_map(CUtensorMap* map, const float* wt, int Nrows, int K, int BN) {
  return make_kmajor_map(map, wt, 4, Nrows, K, kBK, BN);
}

}  // namespace tc
}  // namespace dq
