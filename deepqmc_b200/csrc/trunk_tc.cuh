// Whole Psiformer trunk of a plain forward (S = 1) in ONE persistent launch on the Hopper tensor cores (wgmma).
//
//   for every layer l:   QKV = X Wqkv                                   (reference: gnn/update_features.py:241-286,
//                        O   = softmax(Q K^T / sqrt(dh)) V  per head      hk.MultiHeadAttention, algebra hkext.py:215-253;
//                        A   = X + O Wo                                   MLP hkext.py:22-113, residual rule :116-137;
//                        X   = A + tanh(tanh(A W1 + b1) W2 + b2)          conf/ansatz/psiformer.yaml:70-101)
//
// A CTA owns a tile of G = 128 / NP walkers (NP = electrons per walker rounded up to a power of two, tile row = walker slot x
// NP + electron) and carries it through ALL layers.  The operand of every dense GEMM is written by the previous stage straight
// into the 128-byte-swizzled K-major operand buffer in shared memory ("3xFP16" hi / lo halves, see gemm_wgmma.cuh); the
// dense GEMMs are those of the fused MLP block (fused_tc.cuh: wgmma m64 n256, accumulators in registers, weights streamed
// by TMA).  HBM sees the embedding rows once on the way in and the trunk output once on the way out; the residual stream
// (128 x 256 fp32) and Q / K / V (128 x 768 fp32) of the tile live in a per-CTA scratch buffer (512 KB, re-used for every
// tile and layer, i.e. L2 resident): the register file holds one accumulator, and shared memory (operand buffer + ring)
// cannot park them.
//
// Attention, one head at a time for the whole tile: K_h and V_h of the tile are staged in the (then idle) weight ring as
// fp32; two threads per tile row (32 head columns each) run an online softmax over the keys of the row's own walker and write
// O_h straight into k-block h of the Wo operand.
#pragma once
#include <cstdint>

#include "common.cuh"
#include "fused_tc.cuh"
#include "tc_ptx.cuh"

namespace dq {
namespace tc {

constexpr int kTrThreads = 256;
constexpr int kTrMaxLayers = 8;
constexpr int kTrQkvBytes = 128 * 768 * 4;                   // Q | K | V rows of the tile, fp32
constexpr int kTrScratchPerCta = kTrQkvBytes + 128 * 256 * 4;  // + residual stream rows
using TrSmem = MlpSmem;

struct TrunkParams {
  const float* X0; int ldx;      // embedding rows [rows][256]  (vper > 0: [walkers][256], the moved electron's row only)
  const float* Xbase;            // vper > 0 (non-local-ECP quadrature forwards): embedding rows of the group's base walkers
  long long v0; int vper;        //   [base][N][256]; walker w of this launch is virtual walker v0 + w = base (v0 + w) / vper
                                 //   with electron ((v0 + w) / 12) % N moved (ecp_points_kernel layout)
  float* Out; int ldout;         // trunk output rows [rows][256]
  const CUtensorMap* maps;       // device array [L][4][2]: (Wqkv, Wo, W1, W2) x (hi, lo); boxes of 64 halves x 256 rows
  const float* b1[kTrMaxLayers];
  const float* b2[kTrMaxLayers];
  float us[kTrMaxLayers][4];     // accumulator unscale of the four GEMMs of a layer: 1 / (a_scale * weight scale)
  unsigned char* scratch;        // gridDim.x * kTrScratchPerCta bytes
  int walkers, N, NP, L;         // walkers, electrons per walker, walker slot size (power of two >= N, <= 32), layers
  float a_scale;                 // power of two applied to activations before the hi / lo split
  float attn_scale;              // 1 / sqrt(dh)
  int* err_flag;
};

__global__ void __launch_bounds__(kTrThreads, 1)
trunk_f16_kernel(TrunkParams p) {
  DQMC_TC_SMEM(smem);
  if ((smem_u32(smem) & 1023u) != 0u) tc_trap();
  uint64_t* full = (uint64_t*)(smem + TrSmem::bars());
  float* sb1 = (float*)(smem + TrSmem::bias());
  float* sb2 = sb1 + 256;
  float* kst = (float*)(smem + TrSmem::wring(0));  // attention: K_h [128][64] fp32
  float* vst = (float*)(smem + TrSmem::wring(1));  //            V_h [128][64] fp32

  const int tid = threadIdx.x;
  const int N = p.N, NP = p.NP, L = p.L;
  const int lnp = 31 - __clz(NP);                // NP is a power of two
  const int G = 128 / NP;                        // walker slots per tile
  const int MT = (p.walkers + G - 1) / G;
  float* qkv = (float*)(p.scratch + (size_t)blockIdx.x * kTrScratchPerCta);  // [128][768]
  float* resid = qkv + 128 * 768;                                            // [128][256]

  if (tid == 0) {
    for (int i = 0; i < kMlpSlots; ++i) mbar_init(&full[i], 1);
    fence_barrier_init();
    for (int i = 0; i < 8 * L; ++i) tma_prefetch_desc(p.maps + i);
  }
  __syncthreads();
  const Frag f;
  uint32_t nslot = 0;
  float acc[128];
  // attention task of this thread: tile row ar, head columns 32 ah .. +31
  const int ar = tid >> 1, ah = tid & 1;
  const int a_slot = ar >> lnp;
  for (int tile = blockIdx.x; tile < MT; tile += gridDim.x) {
    // global row of tile row r (-1: padding row or walker past the end)
    auto grow_of = [&](int r) -> long long {
      const int walker = tile * G + (r >> lnp), el = r & (NP - 1);
      return (el < N && walker < p.walkers) ? (long long)walker * N + el : -1;
    };
    // ---- tile load: embedding rows -> residual stream and the operand buffer (loads in batches of 8 ahead of the stores)
    for (int i0 = 0; i0 < 128 * 64 / kTrThreads; i0 += 8) {
      float4 x[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int idx = tid + kTrThreads * (i0 + i), r = idx >> 6, c = 4 * (idx & 63);
        const long long row = grow_of(r);
        x[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row >= 0) {
          const float* xrow = p.X0 + (size_t)row * p.ldx;
          if (p.vper > 0) {
            const int walker = (int)(row / N), el = (int)(row % N);
            const long long v = p.v0 + walker;
            xrow = el == (int)((v / 12) % N) ? p.X0 + (size_t)walker * p.ldx : p.Xbase + ((size_t)(v / p.vper) * N + el) * p.ldx;
          }
          x[i] = __ldg((const float4*)(xrow + c));
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int idx = tid + kTrThreads * (i0 + i), r = idx >> 6, c = 4 * (idx & 63);
        *(float4*)(resid + r * 256 + c) = x[i];
        const float sc = p.a_scale;
        store_operand_quad(smem, r, c, make_float4(x[i].x * sc, x[i].y * sc, x[i].z * sc, x[i].w * sc));
      }
    }
    fence_proxy_async();
    __syncthreads();
    for (int l = 0; l < L; ++l) {
      const bool last = l == L - 1;
      const CUtensorMap* lm = p.maps + 8 * l;
      // ---- Q | K | V = X Wqkv, 256 columns at a time -> scratch (true values)
      for (int j = 0; j < 3; ++j) {
        gemm_abuf<256>(acc, smem, full, nslot, lm, lm + 1, 256 * j, p.err_flag);
        const float us = p.us[l][0];
#pragma unroll
        for (int jj = 0; jj < 32; ++jj)
#pragma unroll
          for (int h = 0; h < 2; ++h)
            *(float2*)(qkv + (f.fr + 8 * h) * 768 + 256 * j + 8 * jj + f.fc) =
                make_float2(acc[4 * jj + 2 * h] * us, acc[4 * jj + 2 * h + 1] * us);
      }
      sb1[tid] = __ldg(p.b1[l] + tid);
      sb2[tid] = __ldg(p.b2[l] + tid);
      __syncthreads();  // Q / K / V rows of the whole tile are in the scratch buffer
      // ---- attention, head by head
      for (int h = 0; h < 4; ++h) {
        {
          float4 kv[2 * 128 * 16 / kTrThreads];  // all loads of this thread first, then the stores
#pragma unroll
          for (int i = 0; i < 128 * 16 / kTrThreads; ++i) {
            const int idx = tid + kTrThreads * i, r = idx >> 4, c = 4 * (idx & 15);
            kv[2 * i] = *(const float4*)(qkv + r * 768 + 256 + 64 * h + c);
            kv[2 * i + 1] = *(const float4*)(qkv + r * 768 + 512 + 64 * h + c);
          }
#pragma unroll
          for (int i = 0; i < 128 * 16 / kTrThreads; ++i) {
            const int idx = tid + kTrThreads * i, r = idx >> 4, c = 4 * (idx & 15);
            *(float4*)(kst + r * 64 + c) = kv[2 * i];
            *(float4*)(vst + r * 64 + c) = kv[2 * i + 1];
          }
        }
        __syncthreads();
        float q[32], o[32];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 v = *(const float4*)(qkv + ar * 768 + 64 * h + 32 * ah + 4 * i);
          q[4 * i] = v.x; q[4 * i + 1] = v.y; q[4 * i + 2] = v.z; q[4 * i + 3] = v.w;
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) o[i] = 0.f;
        float mx = -3.0e38f, sum = 0.f;
        for (int e = 0; e < N; ++e) {  // keys of this row's walker
          const int kr = (a_slot << lnp) + e;
          const float* kp = kst + kr * 64 + 32 * ah;
          float sp[4] = {0.f, 0.f, 0.f, 0.f};  // four independent partial sums: the dot product is not one dependent chain
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 k4 = *(const float4*)(kp + 4 * i);
            sp[i & 3] += q[4 * i] * k4.x + q[4 * i + 1] * k4.y + q[4 * i + 2] * k4.z + q[4 * i + 3] * k4.w;
          }
          float s = (sp[0] + sp[1]) + (sp[2] + sp[3]);
          s = (s + __shfl_xor_sync(0xffffffffu, s, 1)) * p.attn_scale;
          const float mnew = fmaxf(mx, s);
          const float corr = __expf(mx - mnew), pe = __expf(s - mnew);
          sum = sum * corr + pe;
          mx = mnew;
          const float* vp = vst + kr * 64 + 32 * ah;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 v4 = *(const float4*)(vp + 4 * i);
            o[4 * i] = o[4 * i] * corr + pe * v4.x;
            o[4 * i + 1] = o[4 * i + 1] * corr + pe * v4.y;
            o[4 * i + 2] = o[4 * i + 2] * corr + pe * v4.z;
            o[4 * i + 3] = o[4 * i + 3] * corr + pe * v4.w;
          }
        }
        const float un = p.a_scale / sum;
#pragma unroll
        for (int i = 0; i < 8; ++i)
          store_operand_quad(smem, ar, 64 * h + 32 * ah + 4 * i,
                             make_float4(o[4 * i] * un, o[4 * i + 1] * un, o[4 * i + 2] * un, o[4 * i + 3] * un));
        __syncthreads();  // K_h / V_h staging is re-used by the next head (and the ring by the next GEMM)
      }
      fence_proxy_async();
      __syncthreads();
      // ---- A = X + O Wo, M1 = tanh(A W1 + b1), X = A + tanh(M1 W2 + b2)
      const float* xin[2];
      float* aout[2];
      float* xout[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = f.fr + 8 * h;
        xin[h] = resid + r * 256;
        aout[h] = resid + r * 256;
        const long long row = grow_of(r);
        xout[h] = !last ? resid + r * 256 : (row >= 0 ? p.Out + (size_t)row * p.ldout : nullptr);
      }
      mlp3<256>(acc, smem, full, nslot, lm + 2, lm + 3, lm + 4, lm + 5, lm + 6, lm + 7, p.us[l][1], p.us[l][2], p.us[l][3],
                p.a_scale, sb1, sb2, xin, aout, xout, !last, p.err_flag);
      fence_proxy_async();
      __syncthreads();  // next layer's operand complete / next tile's load may overwrite the residual rows
    }
  }
}

}  // namespace tc
}  // namespace dq
