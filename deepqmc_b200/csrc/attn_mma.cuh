// Softmax attention of a plain forward (S = 1) on the tensor cores: warp-level mma.sync.m16n8k16 with "3xFP16" operands.
//
//   O[b, i, h, :] = sum_j softmax_j(q_i . k_j / sqrt(dh)) v_j        (reference: gnn/update_features.py:273-280
//                                                                      hk.MultiHeadAttention; algebra hkext.py:215-253)
// One warp task = 16 queries of one (walker, head) pair against all of its keys (electrons, plus the TransPsiformer's constant
// nuclear tokens).  Scores S = Q K^T and outputs O = P V are m16n8k16 products of half operands split into hi + lo
// (x 2^e = hi + lo, 22 significant bits; three products  hi.lo + lo.hi + hi.hi  accumulated in fp32: fp32-class accuracy, the
// power-of-two scales are undone exactly).  The task body (attn_task_frag) takes its Q / K / V fragments from the caller,
// already split: attn_task_mma loads them from fp32 rows in global memory and splits them in registers, the whole-trunk
// kernel (trunk_tc.cuh) splits each operand once where it is produced.  The probabilities move from the accumulator layout
// of S to the A-operand layout of P V without leaving the register file (the C fragment of two adjacent 8-key tiles IS the
// A fragment of one 16-key tile).
// dh = 64 only (4 k-tiles of 16); keys <= 8 NK8.
#pragma once
#include <cstdint>

#include "common.cuh"

namespace dq {

#ifdef DQMC_EMU
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  float c[4] = {d[0], d[1], d[2], d[3]};
  emu::mma_m16n8k16_f16(d, a, b, c);
}
__device__ __forceinline__ uint32_t am_pack_half2(float lo, float hi);
__device__ __forceinline__ float am_half_to_float(uint32_t h16) { return emu::h2f((uint16_t)h16); }
#else
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ uint32_t am_pack_half2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float am_half_to_float(uint32_t h16) {
  float f;
  asm("{\n\t.reg .b16 h;\n\tcvt.u16.u32 h, %1;\n\tcvt.f32.f16 %0, h;\n\t}" : "=f"(f) : "r"(h16));
  return f;
}
#endif

#ifdef DQMC_EMU
namespace attn_emu {
inline uint16_t f2h(float f) {  // round to nearest even
  uint32_t x;
  std::memcpy(&x, &f, 4);
  const uint32_t sign = (x >> 16) & 0x8000u;
  const int32_t e = (int32_t)((x >> 23) & 255u) - 127;
  uint32_t m = x & 0x7FFFFFu;
  if (((x >> 23) & 255u) == 255u) return (uint16_t)(sign | 0x7C00u | (m ? 0x200u : 0));
  if (e > 15) return (uint16_t)(sign | 0x7C00u);
  if (e >= -14) {
    uint32_t h = ((uint32_t)(e + 15) << 10) | (m >> 13);
    const uint32_t rem = m & 0x1FFFu;
    if (rem > 0x1000u || (rem == 0x1000u && (h & 1u))) ++h;
    return (uint16_t)(sign | h);
  }
  if (e < -25) return (uint16_t)sign;
  m |= 0x800000u;
  const int shift = -e - 14 + 13;
  uint32_t h = m >> shift;
  const uint32_t rem = m & ((1u << shift) - 1u), half = 1u << (shift - 1);
  if (rem > half || (rem == half && (h & 1u))) ++h;
  return (uint16_t)(sign | h);
}
}  // namespace attn_emu
__device__ __forceinline__ uint32_t am_pack_half2(float lo, float hi) {
  return (uint32_t)attn_emu::f2h(lo) | ((uint32_t)attn_emu::f2h(hi) << 16);
}
#endif

// (x0, x1) -> packed hi halves and packed lo halves (x - hi)
__device__ __forceinline__ void am_split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  hi = am_pack_half2(x0, x1);
  lo = am_pack_half2(x0 - am_half_to_float(hi & 0xFFFFu), x1 - am_half_to_float(hi >> 16));
}

// Operand scales of the task: q, k, v by 2^4, probabilities by 2^10 (undone exactly).  A caller that hands over pre-split
// fragments splits x * kAmQS with am_split2, the split of the fp32 loaders below.
constexpr float kAmQS = 16.f, kAmPS = 1024.f;

// One warp task: 16 query rows of one head against 8 NK8 keys (dh = 64), from fragments the caller loads already split
// (lane: g = lane / 4, t = lane % 4, query rows g (i = 0) and g + 8 (i = 1)):
//   ldq(kt, qh, ql)             A fragments of Q x kAmQS, k-tile kt (hi / lo: rows g, g + 8 x columns 16 kt + 2 t (+1, +8, +9))
//   ldk(nt, kt, kh, kl)         B fragments of K x kAmQS: key nt * 8 + g, columns 16 kt + 2 t (+1) and + 8 (+9)
//   ldv(kk, nt, keep, vh, vl)   B fragments of V x kAmQS: keys 16 kk + 2 t (+1) and + 8 (+9), column nt * 8 + g; the pair
//                               halves of keys j with !keep(j) are zeros (substituted, never multiplied)
//   valid(i, j)                 key j takes part in the softmax of query row i (every row needs at least one)
//   store(i, c, o0, o1)         normalised output of query row i, head columns c, c + 1
// Padded keys must load finite fragments: their scores are masked, their V pairs enter P V with probability zero.
// slot > 0 (NK8 = 2, keys = the task's own 16 rows, every key masked to the query rows of its own slot of `slot` rows): a masked
// key's probability is an exact zero, but its V row still enters P V, and 0 x Inf = NaN, so one slot with a non-finite V row
// (or one past the range of the scaled half split, |v| >= 65504 / 16) would make the outputs of every slot in the 16-row window
// non-finite.  If any output of the task is non-finite, P V is therefore recomputed slot by slot with the V rows of the other
// slots read as zeros: the other slots' outputs come out exactly as without the bad slot, the bad slot's stay non-finite.
template <int NK8, class LdQ, class LdK, class LdV, class Valid, class Store>
__device__ __forceinline__ void attn_task_frag(float scale, LdQ ldq, LdK ldk, LdV ldv, Valid valid, Store store, int slot = 0) {
  constexpr int NK16 = (NK8 + 1) / 2;
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  // ---- Q fragments of this query tile (rows g, g + 8), hi / lo, 4 k-tiles of 16
  uint32_t qh[4][4], ql[4][4];
#pragma unroll
  for (int kt = 0; kt < 4; ++kt) ldq(kt, qh[kt], ql[kt]);
  // ---- scores: S[16 x 8 NK8] = Q K^T; B fragment of key tile nt: (k = dh index, n = key nt * 8 + g)
  float s[NK8][4];
#pragma unroll
  for (int nt = 0; nt < NK8; ++nt) {
    s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
    for (int kt = 0; kt < 4; ++kt) {
      uint32_t kh[2], kl[2];
      ldk(nt, kt, kh, kl);
      mma16816(s[nt], qh[kt], kl);
      mma16816(s[nt], ql[kt], kh);
      mma16816(s[nt], qh[kt], kh);
    }
  }
  // ---- softmax over the keys of rows g (c0, c1) and g + 8 (c2, c3); a lane holds keys nt * 8 + 2 t, + 1
  const float us = scale / (kAmQS * kAmQS);
  float m0 = -3.0e38f, m1 = -3.0e38f;
#pragma unroll
  for (int nt = 0; nt < NK8; ++nt) {
    const int j0 = nt * 8 + 2 * t;
    s[nt][0] = valid(0, j0) ? s[nt][0] * us : -3.0e38f;
    s[nt][1] = valid(0, j0 + 1) ? s[nt][1] * us : -3.0e38f;
    s[nt][2] = valid(1, j0) ? s[nt][2] * us : -3.0e38f;
    s[nt][3] = valid(1, j0 + 1) ? s[nt][3] * us : -3.0e38f;
    m0 = fmaxf(m0, fmaxf(s[nt][0], s[nt][1]));
    m1 = fmaxf(m1, fmaxf(s[nt][2], s[nt][3]));
  }
  m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
  m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
  float l0 = 0.f, l1 = 0.f;
#pragma unroll
  for (int nt = 0; nt < NK8; ++nt) {
    s[nt][0] = m_exp(s[nt][0] - m0); s[nt][1] = m_exp(s[nt][1] - m0);
    s[nt][2] = m_exp(s[nt][2] - m1); s[nt][3] = m_exp(s[nt][3] - m1);
    l0 += s[nt][0] + s[nt][1];
    l1 += s[nt][2] + s[nt][3];
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  // ---- probabilities as A fragments of P V: key tile pair (2 kk, 2 kk + 1) = one 16-key k-tile
  uint32_t ph[NK16][4], pl[NK16][4];
#pragma unroll
  for (int kk = 0; kk < NK16; ++kk) {
    const int n0 = 2 * kk, n1 = 2 * kk + 1;
    am_split2(s[n0][0] * kAmPS, s[n0][1] * kAmPS, ph[kk][0], pl[kk][0]);
    am_split2(s[n0][2] * kAmPS, s[n0][3] * kAmPS, ph[kk][1], pl[kk][1]);
    if (n1 < NK8) {
      am_split2(s[n1 < NK8 ? n1 : n0][0] * kAmPS, s[n1 < NK8 ? n1 : n0][1] * kAmPS, ph[kk][2], pl[kk][2]);
      am_split2(s[n1 < NK8 ? n1 : n0][2] * kAmPS, s[n1 < NK8 ? n1 : n0][3] * kAmPS, ph[kk][3], pl[kk][3]);
    } else {
      ph[kk][2] = ph[kk][3] = pl[kk][2] = pl[kk][3] = 0u;
    }
  }
  // ---- O[16 x 64] = P V: B fragment of dh tile nt: (k = key 16 kk + 2 t (+1, +8, +9), n = dh nt * 8 + g)
  const float uo0 = 1.f / (l0 * kAmPS * kAmQS), uo1 = 1.f / (l1 * kAmPS * kAmQS);
  // dh tile nt of P V, V rows of the keys j with keep(j) (the others read as zeros)
  auto pv = [&](int nt, float (&o)[4], auto keep) {
    o[0] = o[1] = o[2] = o[3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < NK16; ++kk) {
      uint32_t vh[2], vl[2];
      ldv(kk, nt, keep, vh, vl);
      mma16816(o, ph[kk], vl);
      mma16816(o, pl[kk], vh);
      mma16816(o, ph[kk], vh);
    }
  };
  int bad = 0;  // this lane stored a non-finite output (NaN fails the comparison)
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    float o[4];
    pv(nt, o, [](int) { return true; });
    o[0] *= uo0; o[1] *= uo0; o[2] *= uo1; o[3] *= uo1;
#pragma unroll
    for (int e = 0; e < 4; ++e) bad |= !(fabsf(o[e]) <= 3.4e38f);
    store(0, nt * 8 + 2 * t, o[0], o[1]);
    store(1, nt * 8 + 2 * t, o[2], o[3]);
  }
  if (slot > 0) {
#pragma unroll
    for (int m = 1; m < 32; m *= 2) bad |= __shfl_xor_sync(0xffffffffu, bad, m);
  }
  if (slot > 0 && bad) {
    const int sm = ~(slot - 1);
    for (int s0 = 0; s0 < 16; s0 += slot) {
      const bool mine0 = (g & sm) == s0, mine1 = ((g + 8) & sm) == s0;
#pragma unroll 1
      for (int nt = 0; nt < 8; ++nt) {
        float o[4];
        pv(nt, o, [&](int j) { return (j & sm) == s0; });
        if (mine0) store(0, nt * 8 + 2 * t, o[0] * uo0, o[1] * uo0);
        if (mine1) store(1, nt * 8 + 2 * t, o[2] * uo1, o[3] * uo1);
      }
    }
  }
}

// The task on fp32 rows in global memory (read-only path), split in registers: every fragment is loaded in the layout the
// instruction wants -- a quad of lanes reads 32 contiguous bytes of a row per instruction (full sectors).
//   qrow(i)            query row i (64 fp32)
//   krow(j), vrow(j)   key / value row j < 8 NK8 (padded keys must point at readable rows: their scores are masked)
template <int NK8, class QRow, class KRow, class VRow, class Valid, class Store>
__device__ __forceinline__ void attn_task_mma(float scale, QRow qrow, KRow krow, VRow vrow, Valid valid, Store store) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const float* qp0 = qrow(0);
  const float* qp1 = qrow(1);
  auto ldq = [&](int kt, uint32_t (&qh)[4], uint32_t (&ql)[4]) {
    const float2 a0 = __ldg((const float2*)(qp0 + kt * 16 + 2 * t)), a1 = __ldg((const float2*)(qp1 + kt * 16 + 2 * t));
    const float2 a2 = __ldg((const float2*)(qp0 + kt * 16 + 8 + 2 * t)), a3 = __ldg((const float2*)(qp1 + kt * 16 + 8 + 2 * t));
    am_split2(a0.x * kAmQS, a0.y * kAmQS, qh[0], ql[0]);
    am_split2(a1.x * kAmQS, a1.y * kAmQS, qh[1], ql[1]);
    am_split2(a2.x * kAmQS, a2.y * kAmQS, qh[2], ql[2]);
    am_split2(a3.x * kAmQS, a3.y * kAmQS, qh[3], ql[3]);
  };
  auto ldk = [&](int nt, int kt, uint32_t (&kh)[2], uint32_t (&kl)[2]) {
    const float* kp = krow(nt * 8 + g);
    const float2 b0 = __ldg((const float2*)(kp + kt * 16 + 2 * t)), b1 = __ldg((const float2*)(kp + kt * 16 + 8 + 2 * t));
    am_split2(b0.x * kAmQS, b0.y * kAmQS, kh[0], kl[0]);
    am_split2(b1.x * kAmQS, b1.y * kAmQS, kh[1], kl[1]);
  };
  auto ldv = [&](int kk, int nt, auto keep, uint32_t (&vh)[2], uint32_t (&vl)[2]) {
    const int j = kk * 16 + 2 * t;
    const float v00 = keep(j) ? __ldg(vrow(j) + nt * 8 + g) : 0.f;
    const float v01 = keep(j + 1) ? __ldg(vrow(j + 1) + nt * 8 + g) : 0.f;
    const float v10 = keep(j + 8) ? __ldg(vrow(j + 8) + nt * 8 + g) : 0.f;
    const float v11 = keep(j + 9) ? __ldg(vrow(j + 9) + nt * 8 + g) : 0.f;
    am_split2(v00 * kAmQS, v01 * kAmQS, vh[0], vl[0]);
    am_split2(v10 * kAmQS, v11 * kAmQS, vh[1], vl[1]);
  };
  attn_task_frag<NK8>(scale, ldq, ldk, ldv, valid, store);
}

// NK8 = number of 8-key tiles (keys padded to 8 NK8 <= 48); block = 4 warps, each warp walks over (pair, query tile) tasks.
template <int NK8>
__global__ void __launch_bounds__(128)
attn_fwd_mma_kernel(const float* __restrict__ QKV, int ldq, float* __restrict__ O, int ldo, int N, int H, int dmodel, float scale,
                    int n_pairs, const float* __restrict__ Kn, const float* __restrict__ Vn, int Mn) {
  constexpr int DH = 64;
  const int NKEY = N + Mn;
  const int MT = (N + 15) / 16;  // query tiles per pair
  const int n_tasks = n_pairs * MT;
  const int g = (threadIdx.x & 31) >> 2;
  const int wglobal = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), wtotal = gridDim.x * (blockDim.x >> 5);
  for (int task = wglobal; task < n_tasks; task += wtotal) {
    const int pair = task / MT, mt = task - pair * MT;
    const int b = pair / H, h = pair - b * H;
    const float* base = QKV + (size_t)b * N * ldq + h * DH;
    // row pointers of key j (K part); the V part sits dmodel further (nuclear tokens: separate arrays)
    auto krow = [&](int j) -> const float* {
      j = j < NKEY ? j : NKEY - 1;  // padded keys read a valid row, their scores are masked
      return j < N ? base + (size_t)j * ldq + dmodel : Kn + (size_t)(j - N) * dmodel + h * DH;
    };
    auto vrow = [&](int j) -> const float* {
      j = j < NKEY ? j : NKEY - 1;
      return j < N ? base + (size_t)j * ldq + 2 * dmodel : Vn + (size_t)(j - N) * dmodel + h * DH;
    };
    const int q0 = mt * 16 + g, q1 = q0 + 8;
    auto qrow = [&](int i) -> const float* {
      const int q = i ? q1 : q0;
      return base + (size_t)(q < N ? q : N - 1) * ldq;
    };
    auto valid = [&](int, int j) { return j < NKEY; };
    auto store = [&](int i, int c, float o0, float o1) {
      const int q = i ? q1 : q0;
      if (q < N) *(float2*)(O + ((size_t)b * N + q) * ldo + h * DH + c) = make_float2(o0, o1);
    };
    attn_task_mma<NK8>(scale, qrow, krow, vrow, valid, store);
  }
}

}  // namespace dq
