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
// (128 x 256 fp32) and K / V of the tile (128 x 512, as split half pairs) live in a per-CTA scratch buffer (384 KB, re-used
// for every tile and layer, i.e. L2 resident): the register file holds one accumulator, and shared memory (operand buffer +
// ring) cannot park them.
//
// The QKV projection runs its column blocks in the order K, V, Q, and each epilogue splits its block into the hi / lo half
// pairs of the attention's operands (am_split2 of x kAmQS), once per element rather than once per reading warp:
//   K  -> scratch [128 rows][128 column pairs] of uint2 {hi, lo}: a score B fragment is one 8-byte load;
//   V  -> scratch [64 key pairs][256 columns] of uint2 {hi, lo} of keys (2 p, 2 p + 1): a P V B fragment is one 8-byte load
//         (the lanes of rows 2 p and 2 p + 1 swap one value to form the pairs);
//   Q  -> k-block h of the operand buffer for head h's 64 columns (hi / lo planes, the GEMM operand layout): once the Q
//         GEMM has retired, the warpgroup's X rows there are dead (X is in the residual rows).  Padding rows keep X.
// Attention on the tensor cores: warp w takes tile rows r0 = 16 w .. +15 and runs the 3xFP16 mma.sync task of attn_mma.cuh
// (shared with attn_fwd_mma_kernel) for each head, Q fragments by ldmatrix from the operand buffer, K / V fragments straight
// from the scratch (plain, coherent loads: this kernel wrote them), and writes O_h, scaled and split, over Q in k-block h
// (the rows of warp w's Q are read and overwritten by warp w only).  The keys of a task are its walker slot (NP = 32: 4 key tiles of 8) or, for slots of at most 16
// rows, the task's own 16 rows masked to the query's slot (2 key tiles; a walker whose V rows are non-finite cannot turn the
// other walkers of the window non-finite, see attn_task_mma's slot argument).  Padding rows (electron >= N) get no attention
// output: their operand rows keep the finite previous operand and are never stored.
#pragma once
#include <cstdint>

#include "attn_mma.cuh"
#include "common.cuh"
#include "fused_tc.cuh"
#include "tc_ptx.cuh"

namespace dq {
namespace tc {

constexpr int kTrThreads = 256;
constexpr int kTrMaxLayers = 8;
constexpr int kTrKvBytes = 128 * 512 * 4;                    // K | V of the tile, split half pairs (uint2 {hi, lo})
constexpr int kTrScratchPerCta = kTrKvBytes + 128 * 256 * 4;  // + residual stream rows
using TrSmem = MlpSmem;

struct TrunkParams {
  const float* X0; int ldx;      // embedding rows [rows][256]  (vper > 0, ECP layout: [walkers][256], the moved electron's row)
  const float* Xbase;            // vper > 0 (compact virtual-walker forwards): embedding rows of the group's base walkers
  long long v0; int vper;        //   [base][N][256]; walker w of this launch is virtual walker v0 + w, whose base walker and
  int n_up, vlayout;             //   moved electrons virtual_move(v0 + w, vper, N, n_up, vlayout, pairs) gives (common.cuh)
  const int* pairs;              //   ECP layout: the group's active-pair list
  const float* wspin;            // swap layout: embedding weights of the +-1 spin feature [256]
  float* Out; int ldout;         // trunk output rows [rows][256]
  const CUtensorMap* maps;       // device array [L][4][2]: (Wqkv, Wo, W1, W2) x (hi, lo); boxes of 32 halves x 256 rows
  const float* b1[kTrMaxLayers];
  const float* b2[kTrMaxLayers];
  float us[kTrMaxLayers][4];     // accumulator unscale of the four GEMMs of a layer: 1 / (a_scale * weight scale)
  unsigned char* scratch;        // gridDim.x * kTrScratchPerCta bytes
  int walkers, N, L;             // walkers, electrons per walker, layers
  float a_scale;                 // power of two applied to activations before the hi / lo split
  float attn_scale;              // 1 / sqrt(dh)
  int* err_flag;
  unsigned long long* phase;     // kPhases cycle / pair counters (fused_tc.cuh Phase), accumulated; nullptr: timers off
};

// The trunk's weight stream: per layer the K, V, Q column blocks of Wqkv (W^T rows 256, 512, 0), then Wo, W1, W2; maps
// [L][4][2] as TrunkParams::maps
struct TrunkMaps {
  static constexpr int G = 6;
  const CUtensorMap* maps;
  __device__ __forceinline__ WTile at(int l, int g) const {
    const CUtensorMap* m = maps + 8 * l + 2 * (g < 3 ? 0 : g - 2);
    return WTile{m, m + 1, g < 2 ? 256 * (g + 1) : 0};
  }
};

// NP: the walker slot (electrons rounded up to a power of two, <= 32), one instance each: an instance carries only the
// attention variant of its slot size.
template <int NP>
__global__ void __launch_bounds__(kTrThreads, 1)
trunk_f16_kernel(TrunkParams p) {
  static_assert(NP >= 1 && NP <= 32 && (NP & (NP - 1)) == 0, "walker slot: a power of two <= 32");
  DQMC_TC_SMEM(smem);
  if ((smem_u32(smem) & 1023u) != 0u) tc_trap();

  const int tid = threadIdx.x, wg = tid >> 7;
  const int N = p.N, L = p.L;
  constexpr int lnp = NP == 1 ? 0 : NP == 2 ? 1 : NP == 4 ? 2 : NP == 8 ? 3 : NP == 16 ? 4 : 5;
  constexpr int G = 128 / NP;                    // walker slots per tile
  const int MT = (p.walkers + G - 1) / G;
  uint2* kbuf = (uint2*)(p.scratch + (size_t)blockIdx.x * kTrScratchPerCta);  // [128 rows][128 column pairs]
  uint2* vbuf = kbuf + 128 * 128;                                              // [64 key pairs][256 columns]
  float* resid = (float*)(vbuf + 64 * 256);                                    // [128][256]

  if (tid == 0) {
    init_rings(smem);
    for (int i = 0; i < 8 * L; ++i) tma_prefetch_desc(p.maps + i);
  }
  unsigned long long* ph = (unsigned long long*)(smem + TrSmem::phases());
  if (tid < 32) ph[tid] = 0ull;
  const WeightStream<TrunkMaps> ws{TrunkMaps{p.maps}, L, MT};
  __syncthreads();
  stream_start<256>(smem, ws);
  PhaseClock pc(p.phase && (tid & 127) == 0 ? ph + 16 * wg : nullptr);
  const Frag f;
  Ring ring;
  float acc[128];
  // attention task of this warp: tile rows r0 .. r0 + 15 (lane: rows r0 + ag, r0 + ag + 8), keys from tile row k0 (inside
  // the warpgroup's 64 rows: a walker slot is at most 32 rows and aligned)
  const int lane = tid & 31, r0 = 16 * (tid >> 5), ag = lane >> 2;
  const int k0 = r0 & ~((NP > 16 ? NP : 16) - 1);
  // From here on the warpgroups only meet at the tensor-core lock: warpgroup w owns tile rows 64 w .. +63 (operand rows,
  // residual and Q / K / V scratch rows, attention keys, weight ring) and synchronises its own 128 threads.  Both run every
  // tile and layer of the CTA (a warpgroup without walkers computes on zero rows and stores nothing): each runs the GEMMs its
  // weight stream counts.
  for (int tile = blockIdx.x; tile < MT; tile += gridDim.x) {
    // global row of tile row r (-1: padding row or walker past the end)
    auto grow_of = [&](int r) -> long long {
      const int walker = tile * G + (r >> lnp), el = r & (NP - 1);
      return (el < N && walker < p.walkers) ? (long long)walker * N + el : -1;
    };
    // ---- tile load: the warpgroup's embedding rows -> residual stream and the operand buffer (loads in batches of 8 ahead
    // of the stores)
#pragma unroll 1
    for (int i0 = 0; i0 < 64 * 64 / 128; i0 += 8) {
      float4 x[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int idx = (tid & 127) + 128 * (i0 + i), r = 64 * wg + (idx >> 6), c = 4 * (idx & 63);
        const long long row = grow_of(r);
        x[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row >= 0) {
          const float* xrow = p.X0 + (size_t)row * p.ldx;
          float sw = 0.f;
          if (p.vper > 0) {
            const int walker = tile * G + (r >> lnp), el = r & (NP - 1);
            const VirtualMove mv = virtual_move((int)p.v0 + walker, p.vper, N, p.n_up, p.vlayout, p.pairs);
            if (mv.e1 < 0) {  // ECP: the moved electron's row is new
              xrow = el == mv.e0 ? p.X0 + (size_t)walker * p.ldx : p.Xbase + ((size_t)mv.base * N + el) * p.ldx;
            } else {  // spin swap: up electron e0 sits at r_e1 and down electron e1 at r_e0, each with its own spin:
                      // emb(r, +-1) = emb(r, -+1) +- 2 w_spin
              const int src = el == mv.e0 ? mv.e1 : (el == mv.e1 ? mv.e0 : el);
              xrow = p.Xbase + ((size_t)mv.base * N + src) * p.ldx;
              sw = el == mv.e0 ? 2.f : (el == mv.e1 ? -2.f : 0.f);
            }
          }
          x[i] = __ldg((const float4*)(xrow + c));
          if (sw != 0.f) {
            const float4 ws = __ldg((const float4*)(p.wspin + c));
            x[i].x += sw * ws.x; x[i].y += sw * ws.y; x[i].z += sw * ws.z; x[i].w += sw * ws.w;
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int idx = (tid & 127) + 128 * (i0 + i), r = 64 * wg + (idx >> 6), c = 4 * (idx & 63);
        *(float4*)(resid + r * 256 + c) = x[i];
        const float sc = p.a_scale;
        store_operand_quad(smem, r, c, make_float4(x[i].x * sc, x[i].y * sc, x[i].z * sc, x[i].w * sc));
      }
    }
    fence_proxy_async();
    wg_sync(wg);
    pc.mark(kPhLoad);
    for (int l = 0; l < L; ++l) {
      const bool last = l == L - 1;
      // ---- K | V | Q = X Wqkv, 256 columns at a time, split for the attention
#pragma unroll 1
      for (int j = 0; j < 3; ++j) {
        const int blk = j == 2 ? 0 : j + 1;  // column block: K, V, then Q (its epilogue overwrites the operand X)
        // one hold of the tensor-core lock per column block: the other warpgroup's MMAs may run under the K and V epilogues
        gemm_abuf<256>(acc, smem, ring, ws, tile, l, j, kTurnOwn, p.err_flag, pc);
        pc.mark(kPhQkv);
        const float us = p.us[l][0];
        const int odd = ag & 1;  // fragment rows fr, fr + 8 have the parity of ag
        // K / V: where column pair (c, c + 1) of fragment row h goes, c = 64 q + 8 jj + fc -> gdst[h] + 32 q + 4 jj (K) or
        // + 64 q + 8 jj (V: even rows keys (r, r + 1) of column c, odd rows keys (r - 1, r) of column c + 1)
        uint2* gdst[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = f.fr + 8 * h;
          gdst[h] = blk == 1 ? kbuf + r * 128 + (f.fc >> 1) : vbuf + (r >> 1) * 256 + f.fc + odd;
        }
        const int gq = blk == 1 ? 32 : 64;
        // one body for the three blocks, rolled over column quarters as in mlp_epilogue: the quarter's values are always
        // acc[0 .. 31]
#pragma unroll 1
        for (int q = 0; q < 4; ++q) {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = f.fr + 8 * h, c = 64 * q + 8 * jj + f.fc;
              // (acc us) kAmQS, two roundings: what the fp32 loaders split from a stored fp32 value
              float x0 = acc[4 * jj + 2 * h] * us * kAmQS, x1 = acc[4 * jj + 2 * h + 1] * us * kAmQS;
              if (blk == 2) {  // the key pair: one value from the lane of the neighbouring row
                const float y = __shfl_xor_sync(0xffffffffu, odd ? x0 : x1, 4);
                x0 = odd ? y : x0;
                x1 = odd ? x1 : y;
              }
              uint2 v;
              am_split2(x0, x1, v.x, v.y);
              if (blk != 0) {
                gdst[h][gq * q + (gq >> 3) * jj] = v;
              } else if ((r & (NP - 1)) < N) {  // Q of head q; padding rows keep their finite X operand
                const int off = operand_off(r, c);
                *(uint32_t*)(smem + MlpSmem::abuf(q, 0) + off) = v.x;
                *(uint32_t*)(smem + MlpSmem::abuf(q, 1) + off) = v.y;
              }
            }
#pragma unroll
          for (int i = 0; i < 96; ++i) acc[i] = acc[i + 32];
        }
        pc.mark(kPhQkvEpi);
      }
      wg_sync(wg);  // K / V rows of the warpgroup are in the scratch buffer, Q in the operand buffer
      // ---- attention on the tensor cores, head by head -> k-block h of the operand buffer
      for (int h = 0; h < 4; ++h) {
        const uint32_t qhi = smem_u32(smem + MlpSmem::abuf(h, 0)), qlo = smem_u32(smem + MlpSmem::abuf(h, 1));
        auto ldq = [&](int kt, uint32_t (&qh)[4], uint32_t (&ql)[4]) {
          const int off = operand_off(r0 + (lane & 15), 16 * kt + 8 * (lane >> 4));
          ldsm_x4(qhi + off, qh);
          ldsm_x4(qlo + off, ql);
        };
        auto ldk = [&](int nt, int kt, uint32_t (&kh)[2], uint32_t (&kl)[2]) {
          const uint2* kp = kbuf + (k0 + nt * 8 + ag) * 128 + 32 * h + 8 * kt + (lane & 3);
          const uint2 a = kp[0], b = kp[4];
          kh[0] = a.x; kl[0] = a.y; kh[1] = b.x; kl[1] = b.y;
        };
        auto ldv = [&](int kk, int nt, auto keep, uint32_t (&vh)[2], uint32_t (&vl)[2]) {
          const int j = 16 * kk + 2 * (lane & 3);
          const uint2* vp = vbuf + ((k0 + j) >> 1) * 256 + 64 * h + 8 * nt + ag;
          const uint2 a = vp[0], b = vp[4 * 256];
          // halves of keys outside keep() are zeros: the split of a zero is a zero pair
          auto sel = [](uint32_t x, bool lo, bool hi) { return (lo ? x & 0xFFFFu : 0u) | (hi ? x & 0xFFFF0000u : 0u); };
          vh[0] = sel(a.x, keep(j), keep(j + 1)); vl[0] = sel(a.y, keep(j), keep(j + 1));
          vh[1] = sel(b.x, keep(j + 8), keep(j + 9)); vl[1] = sel(b.y, keep(j + 8), keep(j + 9));
        };
        auto valid = [&](int i, int j) {
          const int r = r0 + ag + 8 * i, k = k0 + j;
          return (k >> lnp) == (r >> lnp) && (k & (NP - 1)) < N;
        };
        auto store = [&](int i, int c, float o0, float o1) {
          const int r = r0 + ag + 8 * i;
          if ((r & (NP - 1)) < N) store_operand_pair(smem, r, 64 * h + c, o0 * p.a_scale, o1 * p.a_scale);
        };
        attn_task_frag<(NP > 16 ? 4 : 2)>(p.attn_scale, ldq, ldk, ldv, valid, store, NP < 16 ? NP : 0);
      }
      fence_proxy_async();
      wg_sync(wg);
      pc.mark(kPhAttn);
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
      mlp3<256>(acc, smem, ring, ws, tile, l, p.us[l][1], p.us[l][2], p.us[l][3], p.a_scale, p.b1[l], p.b2[l], xin, aout,
                xout, !last, p.err_flag, pc);
      fence_proxy_async();
      wg_sync(wg);  // next layer's operand rows complete / next tile's load may overwrite the residual rows
      pc.mark(kPhW2Epi);
      if (tid < 128) pc.count(kPhPairs);
    }
  }
  if (pc.acc)
    for (int k = 0; k < kPhases; ++k) atomicAdd(p.phase + k, pc.acc[k]);
}

}  // namespace tc
}  // namespace dq
