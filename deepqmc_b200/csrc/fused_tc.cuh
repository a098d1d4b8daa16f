// Fused Psiformer MLP block of a plain forward (S = 1) on the Hopper tensor cores (wgmma), "3xFP16" operands (see
// gemm_wgmma.cuh):
//
//     A  = X + O Wo                      (attention output projection + residual)
//     M1 = tanh(A W1 + b1)
//     X' = A + tanh(M1 W2 + b2)          (reference: gnn/update_features.py:241-286 attention layer with
//                                          conf/ansatz/psiformer.yaml:84-101 MLP; hkext.py:22-113, residual rule :116-137)
//
// for a tile of 128 rows (row = walker x electron) per CTA, persistent over tiles.  The three GEMMs of a tile run back to back
// with the operand of the next GEMM written by the epilogue of the previous one straight from the accumulator registers into
// the 128-byte-swizzled K-major operand buffer in shared memory (split into hi / lo halves): one launch per layer instead of
// three, and M1 never leaves the SM.  A is written to the output rows and read back by the same thread in the last epilogue
// (the accumulator of the next GEMM already fills the register file).
//
// 256 threads = two warpgroups; warpgroup w computes tile rows 64 w .. +63 over all d columns (wgmma m64 n = d, fp32
// accumulators in registers) and owns those rows from the tile load to the output: its half of the operand buffer, its
// residual rows, its weight ring.  The two warpgroups never wait for each other except for the MMA token (ping-pong): each
// runs its own copy of the layer, and one warpgroup's epilogues (and the trunk's attention) run while the other's MMAs
// keep the tensor cores busy.  Thread 0 of a warpgroup streams the pre-split weight half-planes [d rows x 32 halves] (hi,
// lo per k-block, two halves each) of the GEMM through the warpgroup's 3-slot ring (TMA, 64-byte swizzle): the slots of the
// next two k-steps land while the current one is multiplied.  A warpgroup takes the token before the first MMA of a GEMM
// (of the trunk's whole QKV projection: its three column blocks have epilogues much shorter than a GEMM) and hands it to
// the other after issuing the last one, so the two warpgroups' GEMMs alternate on the tensor cores.
// shared memory: operand buffer 4 k-blocks x {hi, lo} x 16 KB = 128 KB, weight rings 2 x 3 x 16 KB, barriers (224 KB).
#pragma once
#include <cstdint>

#include "tc_ptx.cuh"

namespace dq {
namespace tc {

constexpr int kMlpThreads = 256;
constexpr int kMlpSlots = 3;  // weight ring of a warpgroup: a slot is refilled 3 slots ahead, i.e. under the MMAs of the next two

struct MlpParams {
  const float* O; int ldo;     // attention output rows [M][d]
  const float* X; int ldx;     // residual stream rows [M][d]
  float* Out; int ldout;       // X' rows [M][d]; may alias O (a warpgroup reads its O rows before it writes them)
  const float* b1; const float* b2;
  int M, d;
  float a_scale;               // power of two applied to every activation operand before the hi / lo split
  float us0, us1, us2;         // accumulator unscale of the three GEMMs: 1 / (a_scale * weight scale)
  int* err_flag;
};

struct MlpSmem {
  static __host__ __device__ int abuf(int kb, int plane) { return (kb * 2 + plane) * 16384; }   // [128 rows][128 B]
  static __host__ __device__ int wring(int wg, int s) { return 131072 + (wg * kMlpSlots + s) * 16384; }  // [<= 256 rows][64 B]
  static __host__ __device__ int bars() { return 131072 + 2 * kMlpSlots * 16384; }  // full [2][kMlpSlots], token [2]
  static __host__ __device__ int phases() { return bars() + 64; }                                 // [2][16] u64
  static __host__ __device__ int total() { return phases() + 2 * 8 * 16; }
};
// mbarriers: slot s of warpgroup wg's ring landed (TMA tx); the MMA token of warpgroup wg (arrived by the other one)
__device__ __forceinline__ uint64_t* ring_full(unsigned char* smem, int wg) {
  return (uint64_t*)(smem + MlpSmem::bars()) + wg * kMlpSlots;
}
__device__ __forceinline__ uint64_t* mma_token(unsigned char* smem, int wg) {
  return (uint64_t*)(smem + MlpSmem::bars()) + 2 * kMlpSlots + wg;
}
// Kernel prologue (thread 0 with the CTA barrier after it): the barriers of both rings and both tokens.
__device__ __forceinline__ void init_rings(unsigned char* smem) {
  for (int i = 0; i < 2 * kMlpSlots + 2; ++i) mbar_init((uint64_t*)(smem + MlpSmem::bars()) + i, 1);
  fence_barrier_init();
}
// After that CTA barrier: warpgroup 0 holds the token for the first GEMM.
__device__ __forceinline__ void start_pingpong(unsigned char* smem) {
  if (threadIdx.x == 128) mbar_arrive(mma_token(smem, 0));
}

// Phase timers of the whole-trunk kernel (TrunkParams::phase): clock64() cycles summed over the consumer warpgroups of all
// CTAs, in this order; kPhWait (waiting for weight slots to land) and kPhTurn (waiting for the other warpgroup to hand over
// the MMA token) are not part of the mainloop phases.
enum Phase {
  kPhLoad, kPhQkv, kPhQkvEpi, kPhAttn, kPhWo, kPhWoEpi, kPhW1, kPhW1Epi, kPhW2, kPhW2Epi, kPhWait, kPhTurn, kPhPairs, kPhases
};
static_assert(kPhases <= 16, "MlpSmem::phases() holds 16 counters per warpgroup");
struct PhaseClock {
  unsigned long long* acc;  // this warpgroup's shared-memory counters on its timing thread, nullptr: not timing
  long long t;
  __device__ __forceinline__ explicit PhaseClock(unsigned long long* a) : acc(a), t(0) {
    if (a) t = clock64();
  }
  // the time since the last mark goes to phase k
  __device__ __forceinline__ void mark(int k) {
    if (acc) {
      const long long n = clock64();
      acc[k] += (unsigned long long)(n - t);
      t = n;
    }
  }
  __device__ __forceinline__ void count(int k) { if (acc) acc[k] += 1; }
  // w cycles of waiting inside the current phase: booked to phase k (kPhWait, kPhTurn) instead
  __device__ __forceinline__ void waited(long long w, int k) {
    acc[k] += (unsigned long long)w;
    t += w;
  }
};

// tanh of the plain-forward epilogues (same as gemm_wgmma.cuh tanh_fwd): absolute error <= ~3e-7
__device__ __forceinline__ float mlp_tanh(float x) {
  const float x2 = x * x;
  const float poly = x + x * x2 * (-0.33333333333f + x2 * (0.13333333333f + x2 * (-0.05396825397f)));
  const float e = ex2_approx(x * 2.8853900817779268f);
  const float big = 1.f - fast_div(2.f, 1.f + e);
  return fabsf(x) < 0.15f ? poly : big;
}

// (x0, x1) -> packed hi halves and packed lo halves, x = hi + lo to 22 significant bits.  hi is formed in fp32 by Veltkamp's
// splitting (c = 8193 x, hi = c - (c - x): x rounded to 11 bits, three full-rate instructions) instead of converting the packed
// half back; x - hi is exact, both packs are then plain cvt.rn.f16x2.  Values below the normal half range (2^-14 after
// scaling) keep the absolute floor of 2^-25 that the split has anyway.
__device__ __forceinline__ void split_half2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const float c0 = __fmul_rn(x0, 8193.f), c1 = __fmul_rn(x1, 8193.f);
  const float h0 = __fsub_rn(c0, __fsub_rn(c0, x0)), h1 = __fsub_rn(c1, __fsub_rn(c1, x1));
  hi = pack_half2_rn(h0, h1);
  lo = pack_half2_rn(__fsub_rn(x0, h0), __fsub_rn(x1, h1));
}

// byte offset of operand element (row, col) inside its k-block plane: 64 halves per 128-byte row, 16-byte chunks XOR row % 8
__device__ __forceinline__ int operand_off(int row, int col) {
  const int cc = col & 63;
  return (row >> 3) * 1024 + (row & 7) * 128 + ((((cc >> 3) ^ row) & 7) << 4) + (cc & 7) * 2;
}
// two adjacent columns (col even) of tile row `row`, already scaled by a_scale
__device__ __forceinline__ void store_operand_pair(unsigned char* smem, int row, int col, float a0, float a1) {
  uint32_t h, l;
  split_half2(a0, a1, h, l);
  const int off = operand_off(row, col), kb = col >> 6;
  *(uint32_t*)(smem + MlpSmem::abuf(kb, 0) + off) = h;
  *(uint32_t*)(smem + MlpSmem::abuf(kb, 1) + off) = l;
}
// four adjacent columns (col % 4 == 0) of tile row `row`, already scaled
__device__ __forceinline__ void store_operand_quad(unsigned char* smem, int row, int col, float4 a) {
  uint32_t h01, l01, h23, l23;
  split_half2(a.x, a.y, h01, l01);
  split_half2(a.z, a.w, h23, l23);
  const int off = operand_off(row, col), kb = col >> 6;
  *(uint2*)(smem + MlpSmem::abuf(kb, 0) + off) = make_uint2(h01, h23);
  *(uint2*)(smem + MlpSmem::abuf(kb, 1) + off) = make_uint2(l01, l23);
}

// Per-warpgroup pipeline state: ring slots used so far (slot g lives in ring stage g % 3 and completes phase (g / 3) & 1 of
// its barrier) and MMA tokens taken so far (token u completes phase u & 1 of the warpgroup's token barrier).
struct Ring {
  uint32_t nslot = 0, nturn = 0;
};
// What a GEMM does with the MMA token: take it before its first MMA, pass it to the other warpgroup after its last.  A run of
// GEMMs with short epilogues in between (the three column blocks of the QKV projection) holds the token throughout.
enum Turn { kTurnTake = 1, kTurnPass = 2, kTurnOwn = kTurnTake | kTurnPass, kTurnKeep = 0 };

// acc = (this warpgroup's 64 operand rows, K = D) x (rows y0 .. y0 + D - 1 of W^T), hi / lo half-planes through the
// warpgroup's 3-slot weight ring.  Called by the 128 threads of a warpgroup with its operand rows complete (fenced +
// wg_sync); returns with every MMA retired and the ring free.
//
// The MMAs run in the same order as with whole 64-half planes (per k-block: lo A x hi W and hi A x hi W for k-steps 0 .. 3,
// then hi A x lo W for k-steps 0 .. 3), so every output element sums the same products in the same order.
template <int D>
__device__ __forceinline__ void gemm_abuf(float (&acc)[D / 2], unsigned char* smem, Ring& ring, const CUtensorMap* mh,
                                          const CUtensorMap* ml, int y0, int turn, int* err, PhaseClock& pc) {
  uint32_t& nslot = ring.nslot;
  constexpr int KB = D / 64;
  constexpr int NS = 4 * KB;  // slots of this GEMM: slot i = k-steps 2 (i % 2) .. +1 of plane (i / 2) % 2 (hi, lo) of k-block i / 4
  static_assert(NS >= kMlpSlots, "the ring is filled at the start of a GEMM");
  constexpr uint32_t kSlot = D * 64u;
  const int wg = threadIdx.x >> 7;
  const bool leader = (threadIdx.x & 127) == 0;
  uint64_t* full = ring_full(smem, wg);
#pragma unroll
  for (int i = 0; i < D / 2; ++i) acc[i] = 0.f;  // the previous contents are dead: registers free between GEMMs
  auto stage = [&](int i) { return (int)((nslot + (uint32_t)i) % (uint32_t)kMlpSlots); };
  auto load = [&](int i) {
    const int st = stage(i);
    mbar_expect_tx(&full[st], kSlot);
    tma_load_2d(((i >> 1) & 1) ? ml : mh, &full[st], smem + MlpSmem::wring(wg, st), (i >> 2) * 64 + (i & 1) * 32, y0);
  };
  if (leader)
    for (int i = 0; i < kMlpSlots; ++i) load(i);
  // the first slots land while this warpgroup waits for the token
  if (turn & kTurnTake) {
    const long long t0 = pc.acc ? clock64() : 0;
    mbar_wait(mma_token(smem, wg), ring.nturn & 1u, err);
    ++ring.nturn;
    if (pc.acc) pc.waited(clock64() - t0, kPhTurn);
  }
  // waits for slot i and returns its shared-memory address
  auto acquire = [&](int i) {
    const int st = stage(i);
    const long long t0 = pc.acc ? clock64() : 0;
    mbar_wait(&full[st], ((nslot + (uint32_t)i) / (uint32_t)kMlpSlots) & 1u, err);
    if (pc.acc) pc.waited(clock64() - t0, kPhWait);
    return smem_u32(smem + MlpSmem::wring(wg, st));
  };
  // slot i's MMAs were just committed: once the previous slot's have retired in every warp of the warpgroup, its stage takes
  // slot i + 2
  auto retire = [&](int i) {
    wgmma_wait1();
    if (i == 0) return;
    wg_sync(wg);
    if (leader && i + kMlpSlots - 1 < NS) load(i + kMlpSlots - 1);
  };
  auto mma = [&](float (&d)[D / 2], uint32_t a, uint32_t w, int accumulate) {
    if constexpr (D == 256) wgmma_f16_n256(d, make_desc(a), make_desc64(w), accumulate);
    else wgmma_f16_n128(d, make_desc(a), make_desc64(w), accumulate);
  };
  // The MMAs of one slot are straight-line code; between slots nothing touches the accumulator, so the wgmmas of one GEMM
  // stay in flight back to back.
#pragma unroll 1
  for (int kb = 0; kb < KB; ++kb) {
    const uint32_t ah = smem_u32(smem + MlpSmem::abuf(kb, 0)) + wg * 8192, al = smem_u32(smem + MlpSmem::abuf(kb, 1)) + wg * 8192;
#pragma unroll
    for (int q = 0; q < 2; ++q) {  // hi plane, k-steps 2 q, 2 q + 1 (16 halves = 32 bytes per instruction)
      const uint32_t w = acquire(4 * kb + q);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        const int k = 2 * q + kk;
        mma(acc, al + 32 * k, w + 32 * kk, (kb | k) ? 1 : 0);
        mma(acc, ah + 32 * k, w + 32 * kk, 1);
      }
      wgmma_commit();
      retire(4 * kb + q);
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) {  // lo plane
      const uint32_t w = acquire(4 * kb + 2 + q);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) mma(acc, ah + 32 * (2 * q + kk), w + 32 * kk, 1);
      wgmma_commit();
      retire(4 * kb + 2 + q);
    }
  }
  // every MMA of the GEMM is issued: the other warpgroup's GEMM queues behind them
  if ((turn & kTurnPass) && leader) mbar_arrive(mma_token(smem, wg ^ 1));
  wgmma_wait0();
  fence_acc(acc);
  wg_sync(wg);  // the last slots are retired in every warp: the next GEMM may refill their stages
  nslot += NS;
}

// The rows a thread's accumulator fragment covers: tile rows fr and fr + 8, columns 8 j + fc + {0, 1}.
struct Frag {
  int fr, fc;
  __device__ __forceinline__ Frag() {
    const int tid = threadIdx.x, lane = tid & 31;
    fr = 64 * (tid >> 7) + 16 * ((tid >> 5) & 3) + (lane >> 2);
    fc = 2 * (lane & 3);
  }
};

// The epilogues of the MLP block's three GEMMs (mlp3), per accumulator pair (acc0, acc1) = columns c, c + 1 of tile row `row`
// with its row r of the residual input (A for kEpiW2, X for kEpiWo):
//   kEpiWo: A = X + acc us -> gout (parked A), operand
//   kEpiW1: M1 = tanh(acc us + b) -> operand
//   kEpiW2: X' = A + tanh(acc us + b) -> gout (X'), operand if `operand`
enum MlpEpi { kEpiWo, kEpiW1, kEpiW2 };
template <int E>
__device__ __forceinline__ void mlp_epi_pair(unsigned char* smem, int row, int c, float acc0, float acc1, float2 r, float us,
                                             const float* bias, float a_scale, float* gout, bool operand) {
  float v0, v1;
  if constexpr (E == kEpiWo) {
    v0 = r.x + acc0 * us;
    v1 = r.y + acc1 * us;
  } else {
    const float2 b = make_float2(__ldg(bias + c), __ldg(bias + c + 1));  // (the parameter table gives no 8-byte alignment)
    if constexpr (E == kEpiW1) {
      v0 = mlp_tanh(acc0 * us + b.x);
      v1 = mlp_tanh(acc1 * us + b.y);
    } else {
      v0 = r.x + mlp_tanh(acc0 * us + b.x);
      v1 = r.y + mlp_tanh(acc1 * us + b.y);
    }
  }
  if (E != kEpiW1 && gout) *(float2*)(gout + c) = make_float2(v0, v1);
  if (operand) store_operand_pair(smem, row, c, v0 * a_scale, v1 * a_scale);
}

// Epilogue E of the MLP block on this warpgroup's accumulator: per fragment row h (tile rows fr, fr + 8) the residual input
// rin[h] (nullptr: zero for kEpiWo, row skipped for kEpiW2) and the row output gout[h] (nullptr: not stored).  A rolled loop
// over column quarters keeps the code to one quarter: the quarter's values are always acc[0 .. D / 8 - 1] (static register
// indices), the next quarter's move down after each.  This clobbers acc, dead after the epilogue.
template <int D, int E>
__device__ __forceinline__ void mlp_epilogue(float (&acc)[D / 2], unsigned char* smem, float us, const float* bias,
                                             float a_scale, const float* const (&rin)[2], float* const (&gout)[2], bool operand) {
  const Frag f;
  constexpr int QJ = D / 32;  // fragment columns of 8 per quarter
  // Row loads are issued in batches of kJ fragment columns ahead of the stores: rin / gout may alias, so the compiler would
  // otherwise wait for every load behind the previous store.
  constexpr int kJ = 4;
#pragma unroll 1
  for (int q = 0; q < 4; ++q) {
#pragma unroll
    for (int jb = 0; jb < QJ; jb += kJ) {
      float2 r[kJ][2];
#pragma unroll
      for (int j = 0; j < kJ; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          r[j][h] = E != kEpiW1 && rin[h] ? *(const float2*)(rin[h] + 8 * (QJ * q + jb + j) + f.fc) : make_float2(0.f, 0.f);
#pragma unroll
      for (int j = 0; j < kJ; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (E == kEpiW2 && !rin[h]) continue;
          mlp_epi_pair<E>(smem, f.fr + 8 * h, 8 * (QJ * q + jb + j) + f.fc, acc[4 * (jb + j) + 2 * h],
                          acc[4 * (jb + j) + 2 * h + 1], r[j][h], us, bias, a_scale, gout[h], E != kEpiW2 || operand);
        }
    }
#pragma unroll
    for (int i = 0; i < D / 2 - D / 8; ++i) acc[i] = acc[i + D / 8];
  }
}

// The three GEMMs of the MLP block with their epilogues, run by one warpgroup on its 64 rows, its operand rows holding O
// (scaled, split) on entry.  Per fragment row h (tile rows fr, fr + 8): xin[h] residual X (nullptr: zero), aout[h] where A is
// parked (nullptr: row not stored), xout[h] where X' goes (nullptr: not stored); operand_out: X' also becomes the operand
// rows (next layer of the trunk).  wmaps: (Wo, W1, W2) x (hi, lo) tensor maps; b1, b2: the biases in global memory (read
// through the read-only cache).  One call site of the GEMM for all three (a rolled loop): the kernel's code stays small.
template <int D>
__device__ __forceinline__ void mlp3(float (&acc)[D / 2], unsigned char* smem, Ring& ring, const CUtensorMap* const (&wmaps)[6],
                                     float us0, float us1, float us2, float a_scale, const float* b1, const float* b2,
                                     const float* const (&xin)[2], float* const (&aout)[2], float* const (&xout)[2],
                                     bool operand_out, int* err, PhaseClock& pc) {
  const int wg = threadIdx.x >> 7;
#pragma unroll 1
  for (int g = 0; g < 3; ++g) {
    const CUtensorMap* mh = g == 0 ? wmaps[0] : (g == 1 ? wmaps[2] : wmaps[4]);
    const CUtensorMap* ml = g == 0 ? wmaps[1] : (g == 1 ? wmaps[3] : wmaps[5]);
    gemm_abuf<D>(acc, smem, ring, mh, ml, 0, kTurnOwn, err, pc);
    pc.mark(kPhWo + 2 * g);
    if (g == 0) {  // ---- A = X + O Wo -> parked rows and the operand buffer
      mlp_epilogue<D, kEpiWo>(acc, smem, us0, nullptr, a_scale, xin, aout, true);
      fence_proxy_async();
      wg_sync(wg);
      pc.mark(kPhWoEpi);
    } else if (g == 1) {  // ---- M1 = tanh(A W1 + b1) -> operand buffer
      mlp_epilogue<D, kEpiW1>(acc, smem, us1, b1, a_scale, xin, aout, true);
      fence_proxy_async();
      wg_sync(wg);
      pc.mark(kPhW1Epi);
    } else {  // ---- X' = A + tanh(M1 W2 + b2)
      const float* const ain[2] = {aout[0], aout[1]};
      mlp_epilogue<D, kEpiW2>(acc, smem, us2, b2, a_scale, ain, xout, operand_out);
      pc.mark(kPhW2Epi);
    }
  }
}

template <int D>
__global__ void __launch_bounds__(kMlpThreads, 1)
mlp_block_f16_kernel(const __grid_constant__ CUtensorMap wo_hi, const __grid_constant__ CUtensorMap wo_lo,
                     const __grid_constant__ CUtensorMap w1_hi, const __grid_constant__ CUtensorMap w1_lo,
                     const __grid_constant__ CUtensorMap w2_hi, const __grid_constant__ CUtensorMap w2_lo, MlpParams p) {
  DQMC_TC_SMEM(smem);
  if ((smem_u32(smem) & 1023u) != 0u) tc_trap();
  const int tid = threadIdx.x, wg = tid >> 7;
  const int MT = (p.M + 127) / 128;

  if (tid == 0) {
    init_rings(smem);
    tma_prefetch_desc(&wo_hi); tma_prefetch_desc(&wo_lo); tma_prefetch_desc(&w1_hi);
    tma_prefetch_desc(&w1_lo); tma_prefetch_desc(&w2_hi); tma_prefetch_desc(&w2_lo);
  }
  __syncthreads();
  start_pingpong(smem);
  const Frag f;
  Ring ring;
  float acc[D / 2];
  PhaseClock pc(nullptr);
  // Both warpgroups run every tile of the CTA (a warpgroup without valid rows computes on zeros and stores nothing), so
  // they take the MMA token equally often.
  for (int tile = blockIdx.x; tile < MT; tile += gridDim.x) {
    // ---- stage this warpgroup's 64 rows of the O tile: coalesced float4 loads, hi / lo split
    for (int idx = tid & 127; idx < 64 * (D / 4); idx += 128) {
      const int r = 64 * wg + idx / (D / 4), c = 4 * (idx % (D / 4));
      const int grow = tile * 128 + r;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (grow < p.M) v = __ldg((const float4*)(p.O + (size_t)grow * p.ldo + c));
      const float sc = p.a_scale;
      store_operand_quad(smem, r, c, make_float4(v.x * sc, v.y * sc, v.z * sc, v.w * sc));
    }
    fence_proxy_async();
    wg_sync(wg);  // also: every O row of the warpgroup has been read before A is parked in the (possibly aliasing) Out rows
    const float* xin[2];
    float* aout[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int grow = tile * 128 + f.fr + 8 * h;
      const bool valid = grow < p.M;
      xin[h] = valid ? p.X + (size_t)grow * p.ldx : nullptr;
      aout[h] = valid ? p.Out + (size_t)grow * p.ldout : nullptr;
    }
    const CUtensorMap* const wmaps[6] = {&wo_hi, &wo_lo, &w1_hi, &w1_lo, &w2_hi, &w2_lo};
    mlp3<D>(acc, smem, ring, wmaps, p.us0, p.us1, p.us2, p.a_scale, p.b1, p.b2, xin, aout, aout, false, p.err_flag, pc);
  }
}

}  // namespace tc
}  // namespace dq
