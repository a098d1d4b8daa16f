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
// residual rows, its weight ring.  The two warpgroups never wait for each other except for the tensor-core lock
// (ping-pong): each runs its own copy of the layer, and one warpgroup's epilogues (and the trunk's attention) run while the
// other's MMAs keep the tensor cores busy.  Thread 0 of a warpgroup streams the pre-split weight half-planes [d rows x 32
// halves] (hi, lo per k-block, two halves each) through the warpgroup's 3-slot ring (TMA, 64-byte swizzle): the slots of
// the next two k-steps land while the current one is multiplied.  The ring runs along one stream of slots per warpgroup
// across GEMM boundaries (WeightStream): the last k-steps of a GEMM load the first slots of the warpgroup's next GEMM, so
// they land during the epilogue in between.  A warpgroup takes the lock before the first MMA of a GEMM (each of the
// trunk's three QKV column blocks is a GEMM of its own) and releases it after issuing the last one; whichever warpgroup
// asks first gets the tensor cores next, so neither waits on a fixed turn order.
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
  static __host__ __device__ int bars() { return 131072 + 2 * kMlpSlots * 16384; }  // full [2][kMlpSlots], lock word
  static __host__ __device__ int phases() { return bars() + 64; }                                 // [2][16] u64
  static __host__ __device__ int total() { return phases() + 2 * 8 * 16; }
};
// mbarriers: slot s of warpgroup wg's ring landed (TMA tx)
__device__ __forceinline__ uint64_t* ring_full(unsigned char* smem, int wg) {
  return (uint64_t*)(smem + MlpSmem::bars()) + wg * kMlpSlots;
}
// the CTA's tensor-core lock: 0 free, 1 + w held by warpgroup w
__device__ __forceinline__ uint32_t* mma_lock(unsigned char* smem) {
  return (uint32_t*)((uint64_t*)(smem + MlpSmem::bars()) + 2 * kMlpSlots);
}
static_assert(2 * kMlpSlots * 8 + 4 <= 64, "the ring barriers and the lock word fit below MlpSmem::phases()");
// Kernel prologue (thread 0 with the CTA barrier after it): the barriers of both rings, the lock free.
__device__ __forceinline__ void init_rings(unsigned char* smem) {
  for (int i = 0; i < 2 * kMlpSlots; ++i) mbar_init((uint64_t*)(smem + MlpSmem::bars()) + i, 1);
  *mma_lock(smem) = 0u;
  fence_barrier_init();
}

// Taken by the leader of warpgroup wg before the first MMA of a GEMM (then wg_sync releases the other 127 threads): a
// shared-memory CAS, retried after a short sleep, since the spinning warp shares its SM sub-partition with an epilogue warp
// of the other warpgroup and must leave it the issue slots.  Bounded like mbar_wait, but nothing the warpgroups compute
// depends on the lock (their rows, accumulators and rings are disjoint; it only orders their MMAs on the tensor cores), so
// on timeout the error flag is set and the warpgroup goes on without it.
constexpr unsigned kLockSleepNs = 64;
__device__ __forceinline__ void lock_take(unsigned char* smem, int wg, int* err) {
  const uint32_t a = smem_u32(mma_lock(smem)), me = 1u + (uint32_t)wg;
  if (smem_cas_acquire(a, 0u, me) == 0u) return;
  const long long t0 = clock64();
  while (true) {
    __nanosleep(kLockSleepNs);
    if (smem_cas_acquire(a, 0u, me) == 0u) return;
    if (clock64() - t0 > 4000000000LL) {
      if (err) atomicExch(err, 1);
      return;
    }
  }
}
// By the same leader right after issuing the last MMA of the GEMM (release: no MMA issue moves below it).  Only a lock
// this warpgroup holds is released.
__device__ __forceinline__ void lock_release(unsigned char* smem, int wg) {
  smem_cas_release(smem_u32(mma_lock(smem)), 1u + (uint32_t)wg, 0u);
}

// Phase timers of the whole-trunk kernel (TrunkParams::phase): clock64() cycles summed over the consumer warpgroups of all
// CTAs, in this order; kPhWait (waiting for weight slots to land) and kPhTurn (waiting for the tensor-core lock while the
// other warpgroup's MMAs are issued) are not part of the mainloop phases.
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

// Per-warpgroup pipeline state: ring slots used so far (slot g of the warpgroup's weight stream lives in ring stage g % 3 and
// completes phase (g / 3) & 1 of its barrier).
struct Ring {
  uint32_t nslot = 0;
};
// What a GEMM does with the tensor-core lock: take it before its first MMA, release it after its last.  A run of GEMMs may
// hold it throughout (take, keep, ..., release); the kernels take and release it per GEMM (kTurnOwn).
enum Turn { kTurnTake = 1, kTurnRelease = 2, kTurnOwn = kTurnTake | kTurnRelease, kTurnKeep = 0 };

// One GEMM's weights: the hi / lo half-plane maps of W^T and the first W^T row of its column block (hi == nullptr: none).
struct WTile {
  const CUtensorMap* hi;
  const CUtensorMap* lo;
  int y0;
};
// The weight stream of a warpgroup: every GEMM it runs, in order.  For each of the CTA's tiles (blockIdx.x, + gridDim.x,
// ... < MT) and each of its L layers, the G = Maps::G GEMMs Maps::at(l, g), g = 0 .. G - 1.  A GEMM loads the first slots of
// the next one (after()), and the stream ends with the last GEMM the CTA runs: no slot is loaded that no GEMM consumes, so
// no TMA is in flight when the CTA exits.
template <class Maps>
struct WeightStream {
  Maps maps;
  int L, MT;
  __device__ __forceinline__ WTile after(int tile, int l, int g) const {
    if (++g == Maps::G) {
      g = 0;
      if (++l == L) {
        l = 0;
        tile += gridDim.x;
      }
    }
    return tile < MT ? maps.at(l, g) : WTile{nullptr, nullptr, 0};
  }
};

// TMA of slot i of a GEMM's weights (k-steps 2 (i % 2) .. +1 of plane (i / 2) % 2 (hi, lo) of k-block i / 4) into stage st of
// warpgroup wg's ring
template <int D>
__device__ __forceinline__ void load_slot(unsigned char* smem, int wg, int st, const WTile& w, int i) {
  uint64_t* full = ring_full(smem, wg) + st;
  mbar_expect_tx(full, D * 64u);
  tma_load_2d(((i >> 1) & 1) ? w.lo : w.hi, full, smem + MlpSmem::wring(wg, st), (i >> 2) * 64 + (i & 1) * 32, w.y0);
}
// Kernel prologue, after the CTA barrier that follows init_rings: the first kMlpSlots slots of the warpgroup's stream (GEMM
// 0 of layer 0 of tile blockIdx.x).  Ring::nslot starts at 0.
template <int D, class Maps>
__device__ __forceinline__ void stream_start(unsigned char* smem, const WeightStream<Maps>& ws) {
  if ((threadIdx.x & 127) == 0 && (int)blockIdx.x < ws.MT) {
    const WTile w = ws.maps.at(0, 0);
    for (int i = 0; i < kMlpSlots; ++i) load_slot<D>(smem, threadIdx.x >> 7, i, w, i);
  }
}

// acc = (this warpgroup's 64 operand rows, K = D) x (rows y0 .. y0 + D - 1 of W^T) for GEMM g of layer l of tile `tile` of
// the warpgroup's weight stream, hi / lo half-planes through its 3-slot ring.  Called by the 128 threads of a warpgroup with
// its operand rows complete (fenced + wg_sync) and the first kMlpSlots slots of the GEMM loaded (stream_start or the GEMM
// before); returns with every MMA retired and the first kMlpSlots slots of the next GEMM loaded.
//
// The MMAs run in the same order as with whole 64-half planes (per k-block: lo A x hi W and hi A x hi W for k-steps 0 .. 3,
// then hi A x lo W for k-steps 0 .. 3), so every output element sums the same products in the same order.
template <int D, class Maps>
__device__ __forceinline__ void gemm_abuf(float (&acc)[D / 2], unsigned char* smem, Ring& ring, const WeightStream<Maps>& ws,
                                          int tile, int l, int g, int turn, int* err, PhaseClock& pc) {
  uint32_t& nslot = ring.nslot;
  constexpr int KB = D / 64;
  constexpr int NS = 4 * KB;  // slots of this GEMM
  static_assert(NS >= kMlpSlots, "a GEMM has at least as many slots as the ring has stages");
  const int wg = threadIdx.x >> 7;
  const bool leader = (threadIdx.x & 127) == 0;
  uint64_t* full = ring_full(smem, wg);
  const WTile cur = ws.maps.at(l, g), nxt = ws.after(tile, l, g);
#pragma unroll
  for (int i = 0; i < D / 2; ++i) acc[i] = 0.f;  // the previous contents are dead: registers free between GEMMs
  // stage of slot i of this GEMM; i >= NS: slot i - NS of the next one
  auto stage = [&](int i) { return (int)((nslot + (uint32_t)i) % (uint32_t)kMlpSlots); };
  // the lock is asked for once the first slot has landed: a warpgroup never holds the tensor cores while it waits for L2.
  // (This wait, bounded by a trap like every ring wait, also keeps ptxas from serialising the GEMM's wgmmas behind the
  // lock's divergent spin loop.)
  if (turn & kTurnTake) {
    long long t0 = pc.acc ? clock64() : 0;
    if (leader) mbar_wait(&full[stage(0)], (nslot / (uint32_t)kMlpSlots) & 1u, err);
    if (pc.acc) {
      const long long t1 = clock64();
      pc.waited(t1 - t0, kPhWait);
      t0 = t1;
    }
    if (leader) lock_take(smem, wg, err);
    wg_sync(wg);
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
  // slot i + 2, of this GEMM or (only after a lo-plane slot, `cross`) of the next one
  auto retire = [&](int i, bool cross) {
    wgmma_wait1();
    if (i == 0) return;
    wg_sync(wg);
    const int s = i + kMlpSlots - 1;
    const bool own = !cross || s < NS;
    if (leader && (own || nxt.hi))
      load_slot<D>(smem, wg, stage(s), WTile{own ? cur.hi : nxt.hi, own ? cur.lo : nxt.lo, own ? cur.y0 : nxt.y0},
                   own ? s : s - NS);
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
      retire(4 * kb + q, false);
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) {  // lo plane
      const uint32_t w = acquire(4 * kb + 2 + q);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) mma(acc, ah + 32 * (2 * q + kk), w + 32 * kk, 1);
      wgmma_commit();
      retire(4 * kb + 2 + q, true);
    }
  }
  // every MMA of the GEMM is issued: the other warpgroup's GEMM may queue behind them
  if ((turn & kTurnRelease) && leader) lock_release(smem, wg);
  wgmma_wait0();
  fence_acc(acc);
  wg_sync(wg);  // the last slot is retired in every warp: its stage takes the next GEMM's third slot
  if (leader && nxt.hi) load_slot<D>(smem, wg, stage(NS + kMlpSlots - 1), nxt, kMlpSlots - 1);
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
// rows (next layer of the trunk).  Wo, W1, W2 are the last three GEMMs of layer l of tile `tile` in the weight stream ws;
// b1, b2: the biases in global memory (read through the read-only cache).  One call site of the GEMM for all three (a rolled
// loop): the kernel's code stays small.
template <int D, class Maps>
__device__ __forceinline__ void mlp3(float (&acc)[D / 2], unsigned char* smem, Ring& ring, const WeightStream<Maps>& ws,
                                     int tile, int l, float us0, float us1, float us2, float a_scale, const float* b1,
                                     const float* b2, const float* const (&xin)[2], float* const (&aout)[2],
                                     float* const (&xout)[2], bool operand_out, int* err, PhaseClock& pc) {
  const int wg = threadIdx.x >> 7;
#pragma unroll 1
  for (int g = 0; g < 3; ++g) {
    gemm_abuf<D>(acc, smem, ring, ws, tile, l, Maps::G - 3 + g, kTurnOwn, err, pc);
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

// The MLP block's weight stream: per tile Wo, W1, W2
struct MlpMaps {
  static constexpr int G = 3;
  const CUtensorMap *wo_hi, *wo_lo, *w1_hi, *w1_lo, *w2_hi, *w2_lo;
  __device__ __forceinline__ WTile at(int, int g) const {
    return g == 0 ? WTile{wo_hi, wo_lo, 0} : (g == 1 ? WTile{w1_hi, w1_lo, 0} : WTile{w2_hi, w2_lo, 0});
  }
};

template <int D>
__global__ void __launch_bounds__(kMlpThreads, 1)
mlp_block_f16_kernel(const __grid_constant__ CUtensorMap wo_hi, const __grid_constant__ CUtensorMap wo_lo,
                     const __grid_constant__ CUtensorMap w1_hi, const __grid_constant__ CUtensorMap w1_lo,
                     const __grid_constant__ CUtensorMap w2_hi, const __grid_constant__ CUtensorMap w2_lo, MlpParams p) {
  DQMC_TC_SMEM(smem);
  if ((smem_u32(smem) & 1023u) != 0u) tc_trap();
  const int tid = threadIdx.x, wg = tid >> 7;
  const int MT = (p.M + 127) / 128;
  const WeightStream<MlpMaps> ws{MlpMaps{&wo_hi, &wo_lo, &w1_hi, &w1_lo, &w2_hi, &w2_lo}, 1, MT};

  if (tid == 0) {
    init_rings(smem);
    tma_prefetch_desc(&wo_hi); tma_prefetch_desc(&wo_lo); tma_prefetch_desc(&w1_hi);
    tma_prefetch_desc(&w1_lo); tma_prefetch_desc(&w2_hi); tma_prefetch_desc(&w2_lo);
  }
  __syncthreads();
  stream_start<D>(smem, ws);
  const Frag f;
  Ring ring;
  float acc[D / 2];
  PhaseClock pc(nullptr);
  // Both warpgroups run every tile of the CTA (a warpgroup without valid rows computes on zeros and stores nothing): each
  // runs the GEMMs its weight stream counts.
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
    mlp3<D>(acc, smem, ring, ws, tile, 0, p.us0, p.us1, p.us2, p.a_scale, p.b1, p.b2, xin, aout, aout, false, p.err_flag, pc);
  }
}

}  // namespace tc
}  // namespace dq
