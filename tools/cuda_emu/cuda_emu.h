// Minimal CPU emulation of the CUDA execution model, DEVELOPMENT/TEST TOOL ONLY.
//
// The build container has no GPU; this header lets the *same kernel sources* under
// deepqmc_b200/csrc be compiled with g++ (-DDQMC_EMU) and executed block by block on the
// CPU so that indexing / reduction / barrier logic can be checked against the oracle before
// spending GPU minutes.  Threads of a block are ucontext fibers scheduled round-robin;
// __syncthreads / warp shuffles are cooperative yields.  It is never linked into the shipped
// library (libdqmc_b200.so is built by nvcc only) and the product path never falls back to it.
#pragma once
#include <ucontext.h>

#include <cassert>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <functional>
#include <map>
#include <vector>

struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct uint3_emu { unsigned x, y, z; };

namespace emu {
struct Fiber {
  ucontext_t ctx;
  std::vector<char> stack;
  uint3_emu tidx{0, 0, 0};
  int lin = 0;
  bool done = false;
};
struct State {
  std::vector<Fiber> fibers;
  ucontext_t main_ctx;
  int cur = 0;
  int nthreads = 0;
  uint3_emu bidx{0, 0, 0};
  dim3 bdim, gdim;
  // block barrier
  long bar_gen = 0;
  int bar_count = 0;
  // warp exchange
  std::vector<uint64_t> shfl_buf;      // [nthreads]
  std::vector<int> warp_count;         // arrivals per warp
  std::vector<long> warp_gen;          // generation per warp
  std::vector<unsigned char> dyn_smem;
  std::function<void()> body;
  std::map<const void*, size_t> max_dyn_smem;  // cudaFuncSetAttribute(MaxDynamicSharedMemorySize) opt-ins per kernel
};
inline State& S() { static thread_local State s; return s; }
// Scheduling order of the fibers of a block.  DQMC_EMU_REVERSE=1 runs the highest thread first and walks downwards:
// a missing __syncthreads()/__syncwarp() between a shared-memory write and a read by another thread gives the right
// answer in at most one of the two orders, so running a test in both orders exposes the race.
inline int sched_dir() {
  static const int d = (std::getenv("DQMC_EMU_REVERSE") && std::getenv("DQMC_EMU_REVERSE")[0] == '1') ? -1 : 1;
  return d;
}
inline int sched_next(int me, int k, int n) { return ((me + sched_dir() * k) % n + n) % n; }

inline void yield() {
  State& s = S();
  int me = s.cur;
  // next runnable fiber (round robin); if none other, continue
  for (int k = 1; k <= s.nthreads; ++k) {
    int nxt = sched_next(me, k, s.nthreads);
    if (!s.fibers[nxt].done) {
      if (nxt == me) return;
      s.cur = nxt;
      swapcontext(&s.fibers[me].ctx, &s.fibers[nxt].ctx);
      return;
    }
  }
}
inline void fiber_entry() {
  State& s = S();
  s.body();
  int me = s.cur;
  s.fibers[me].done = true;
  // switch to next unfinished fiber or back to main
  for (int k = 1; k <= s.nthreads; ++k) {
    int nxt = sched_next(me, k, s.nthreads);
    if (!s.fibers[nxt].done) {
      s.cur = nxt;
      setcontext(&s.fibers[nxt].ctx);
    }
  }
  setcontext(&s.main_ctx);
}
inline void syncthreads() {
  State& s = S();
  long gen = s.bar_gen;
  if (++s.bar_count == s.nthreads) {
    s.bar_count = 0;
    s.bar_gen++;
    return;
  }
  while (s.bar_gen == gen) yield();
}
inline void syncwarp() {
  State& s = S();
  int w = s.fibers[s.cur].lin / 32;
  int wsize = std::min(32, s.nthreads - w * 32);
  long gen = s.warp_gen[w];
  if (++s.warp_count[w] == wsize) {
    s.warp_count[w] = 0;
    s.warp_gen[w]++;
    return;
  }
  while (s.warp_gen[w] == gen) yield();
}
template <class T>
inline T shfl_idx(T v, int src_lane) {
  static_assert(sizeof(T) <= 8, "shfl of <=8 byte types");
  State& s = S();
  int lin = s.fibers[s.cur].lin;
  int w = lin / 32;
  uint64_t raw = 0;
  std::memcpy(&raw, &v, sizeof(T));
  s.shfl_buf[lin] = raw;
  syncwarp();
  int src = w * 32 + (src_lane & 31);
  if (src >= s.nthreads) src = lin;
  uint64_t got = s.shfl_buf[src];
  syncwarp();
  T out;
  std::memcpy(&out, &got, sizeof(T));
  return out;
}
// Launch limits of sm_90 that a CPU run would otherwise never notice: 1024 threads per block, grid.y/z <= 65535,
// dynamic shared memory <= 48 KiB unless the kernel opted in (<= 227 KiB), and no write past the requested bytes.
inline void check_limits(dim3 grid, dim3 block, size_t smem, const void* fn, const char* name) {
  State& s = S();
  bool ok = block.x >= 1 && block.x <= 1024 && grid.x >= 1 && grid.y >= 1 && grid.z >= 1 && grid.x <= 2147483647u &&
            grid.y <= 65535u && grid.z <= 65535u;
  size_t cap = 48 * 1024;
  auto it = s.max_dyn_smem.find(fn);
  if (it != s.max_dyn_smem.end()) cap = std::max(cap, it->second);
  if (!ok || smem > cap || cap > 227 * 1024) {
    std::fprintf(stderr, "cuda_emu: invalid launch of %s: grid (%u,%u,%u) block %u smem %zu (cap %zu)\n", name, grid.x, grid.y,
                 grid.z, block.x, smem, cap);
    std::abort();
  }
}
inline void launch(dim3 grid, dim3 block, size_t smem, std::function<void()> body, const void* fn = nullptr,
                   const char* name = "?") {
  State& s = S();
  assert(block.y == 1 && block.z == 1 && "emulator supports 1-D blocks");
  check_limits(grid, block, smem, fn, name);
  s.nthreads = block.x;
  s.bdim = block;
  s.gdim = grid;
  s.body = body;
  const size_t kGuard = 64;
  s.dyn_smem.assign(smem + 1024 + kGuard, 0);  // 1024-byte aligned base (SWIZZLE_128B atoms of the tensor-core kernels)
  unsigned char* smem_base = (unsigned char*)(((uintptr_t)s.dyn_smem.data() + 1023) & ~(uintptr_t)1023);
  size_t guard_len = s.dyn_smem.data() + s.dyn_smem.size() - (smem_base + smem);
  if ((int)s.fibers.size() < s.nthreads) s.fibers.resize(s.nthreads);
  s.shfl_buf.assign(s.nthreads, 0);
  int nw = (s.nthreads + 31) / 32;
  const size_t kStack = 256 * 1024;
  // DQMC_EMU_REVERSE_BLOCKS=1 walks the grid from the last block to the first: blocks of one launch may run in any order
  // on the GPU, so a kernel whose blocks depend on each other (without atomics) passes in one of the two orders at most.
  static const bool rev_blocks = std::getenv("DQMC_EMU_REVERSE_BLOCKS") && std::getenv("DQMC_EMU_REVERSE_BLOCKS")[0] == '1';
  for (unsigned iz = 0; iz < grid.z; ++iz)
    for (unsigned iy = 0; iy < grid.y; ++iy)
      for (unsigned ix = 0; ix < grid.x; ++ix) {
        const unsigned bx = rev_blocks ? grid.x - 1 - ix : ix, by = rev_blocks ? grid.y - 1 - iy : iy,
                       bz = rev_blocks ? grid.z - 1 - iz : iz;
        s.bidx = {bx, by, bz};
        s.bar_gen = 0;
        s.bar_count = 0;
        s.warp_count.assign(nw, 0);
        s.warp_gen.assign(nw, 0);
        for (int t = 0; t < s.nthreads; ++t) {
          Fiber& f = s.fibers[t];
          if (f.stack.size() != kStack) f.stack.resize(kStack);
          f.tidx = {(unsigned)t, 0, 0};
          f.lin = t;
          f.done = false;
          getcontext(&f.ctx);
          f.ctx.uc_stack.ss_sp = f.stack.data();
          f.ctx.uc_stack.ss_size = kStack;
          f.ctx.uc_link = nullptr;
          makecontext(&f.ctx, (void (*)())fiber_entry, 0);
        }
        std::memset(s.dyn_smem.data(), 0xFF, s.dyn_smem.size());  // shared memory of a fresh block holds garbage, not zeros
        std::memset(smem_base + smem, 0xA5, guard_len);
        s.cur = sched_dir() > 0 ? 0 : s.nthreads - 1;
        swapcontext(&s.main_ctx, &s.fibers[s.cur].ctx);
        for (size_t g = 0; g < guard_len; ++g)
          if (smem_base[smem + g] != 0xA5) {
            std::fprintf(stderr, "cuda_emu: %s wrote past its %zu bytes of dynamic shared memory (block %u,%u,%u)\n", name, smem,
                         bx, by, bz);
            std::abort();
          }
      }
}
}  // namespace emu

struct alignas(16) float4 { float x, y, z, w; };
struct alignas(16) double2 { double x, y; };
struct alignas(8) float2 { float x, y; };
inline float2 make_float2(float x, float y) { return float2{x, y}; }
struct alignas(8) uint2 { unsigned x, y; };
inline uint2 make_uint2(unsigned x, unsigned y) { return uint2{x, y}; }
struct alignas(16) uint4 { unsigned x, y, z, w; };
inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
inline float __uint_as_float(unsigned u) { float f; std::memcpy(&f, &u, 4); return f; }
inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }
inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
template <class T> inline T __ldg(const T* p) { return *p; }

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static thread_local
#define threadIdx (emu::S().fibers[emu::S().cur].tidx)
#define blockIdx (emu::S().bidx)
#define blockDim (emu::S().bdim)
#define gridDim (emu::S().gdim)
inline void __syncthreads() { emu::syncthreads(); }
inline void __syncwarp(unsigned = 0xffffffffu) { emu::syncwarp(); }
inline void __threadfence_block() {}
inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
inline long long clock64() { return 0; }
inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
inline void __threadfence() {}
template <class T> inline T __shfl_sync(unsigned, T v, int src) { return emu::shfl_idx(v, src); }
template <class T> inline T __shfl_xor_sync(unsigned, T v, int m) {
  return emu::shfl_idx(v, (emu::S().fibers[emu::S().cur].lin & 31) ^ m);
}
template <class T> inline T __shfl_down_sync(unsigned, T v, int d) {
  int lane = emu::S().fibers[emu::S().cur].lin & 31;
  return emu::shfl_idx(v, lane + d < 32 ? lane + d : lane);
}
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline unsigned __ballot_sync(unsigned, int pred) {  // every lane of the warp calls it (as the kernels do)
  unsigned m = pred ? 1u << (emu::S().fibers[emu::S().cur].lin & 31) : 0u;
  for (int o = 16; o > 0; o >>= 1) m |= __shfl_xor_sync(0xffffffffu, m, o);
  return m;
}
template <class T> inline T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }
template <class T> inline T atomicMax(T* p, T v) { T o = *p; if (v > o) *p = v; return o; }

// ---- warp-level mma.sync.m16n8k16 (f16 inputs, f32 accumulate): functional model with the PTX fragment layouts ------------
// A (16x16, row): a0 = (g, 2t..2t+1), a1 = (g+8, 2t..), a2 = (g, 2t+8..), a3 = (g+8, 2t+8..);  B (16x8, col): b0 = (k 2t..2t+1, n g),
// b1 = (k 2t+8.., n g);  C/D (16x8): c0 = (g, 2t), c1 = (g, 2t+1), c2 = (g+8, 2t), c3 = (g+8, 2t+1);  g = lane / 4, t = lane % 4.
namespace emu {
inline float h2f(uint16_t h) {
  const uint32_t s = (h >> 15) & 1u, e = (h >> 10) & 31u, m = h & 1023u;
  float v;
  if (e == 0) v = std::ldexp((float)m, -24);
  else if (e == 31) v = m ? NAN : INFINITY;
  else v = std::ldexp((float)(m | 1024u), (int)e - 25);
  return s ? -v : v;
}
inline void mma_m16n8k16_f16(float* d, const uint32_t* a, const uint32_t* b, const float* c) {
  static thread_local std::vector<uint32_t> abuf, bbuf;
  State& s = S();
  if ((int)abuf.size() < s.nthreads * 4) { abuf.assign(s.nthreads * 4, 0); bbuf.assign(s.nthreads * 2, 0); }
  const int lin = s.fibers[s.cur].lin, w = lin / 32, lane = lin & 31;
  for (int i = 0; i < 4; ++i) abuf[lin * 4 + i] = a[i];
  for (int i = 0; i < 2; ++i) bbuf[lin * 2 + i] = b[i];
  syncwarp();
  auto A = [&](int r, int k) {  // element (row r, col k) of the 16x16 A tile
    const int gl = r & 7, t = (k & 7) >> 1, reg = (r >> 3) + 2 * (k >> 3);
    const uint32_t v = abuf[(w * 32 + gl * 4 + t) * 4 + reg];
    return h2f((uint16_t)((k & 1) ? v >> 16 : v & 0xFFFFu));
  };
  auto B = [&](int k, int n) {  // element (k, n) of the 16x8 B tile
    const int t = (k & 7) >> 1, reg = k >> 3;
    const uint32_t v = bbuf[(w * 32 + n * 4 + t) * 2 + reg];
    return h2f((uint16_t)((k & 1) ? v >> 16 : v & 0xFFFFu));
  };
  const int g = lane >> 2, t = lane & 3;
  for (int i = 0; i < 4; ++i) {
    const int r = g + 8 * (i >> 1), n = 2 * t + (i & 1);
    double acc = (double)c[i];
    for (int k = 0; k < 16; ++k) acc += (double)A(r, k) * (double)B(k, n);
    d[i] = (float)acc;
  }
  syncwarp();
}
// mma.sync.m16n8k8 .tf32: A a0 (g, t) a1 (g + 8, t) a2 (g, t + 4) a3 (g + 8, t + 4); B b0 (k = t, n = g) b1 (k = t + 4, n = g)
inline void mma_m16n8k8_tf32(float* d, const uint32_t* a, const uint32_t* b, const float* c) {
  static thread_local std::vector<uint32_t> abuf, bbuf;
  State& s = S();
  if ((int)abuf.size() < s.nthreads * 4) { abuf.assign(s.nthreads * 4, 0); bbuf.assign(s.nthreads * 2, 0); }
  const int lin = s.fibers[s.cur].lin, w = lin / 32, lane = lin & 31;
  for (int i = 0; i < 4; ++i) abuf[lin * 4 + i] = a[i];
  for (int i = 0; i < 2; ++i) bbuf[lin * 2 + i] = b[i];
  syncwarp();
  auto f = [](uint32_t u) { u &= 0xFFFFE000u; float x; std::memcpy(&x, &u, 4); return x; };
  auto A = [&](int r, int k) { return f(abuf[(w * 32 + (r & 7) * 4 + (k & 3)) * 4 + (r >> 3) + 2 * (k >> 2)]); };
  auto B = [&](int k, int n) { return f(bbuf[(w * 32 + n * 4 + (k & 3)) * 2 + (k >> 2)]); };
  const int g = lane >> 2, t = lane & 3;
  for (int i = 0; i < 4; ++i) {
    const int r = g + 8 * (i >> 1), n = 2 * t + (i & 1);
    double acc = (double)c[i];
    for (int k = 0; k < 8; ++k) acc += (double)A(r, k) * (double)B(k, n);
    d[i] = (float)acc;
  }
  syncwarp();
}
}  // namespace emu

// ---- tiny runtime shim ---------------------------------------------------------------
typedef int cudaError_t;
typedef void* cudaStream_t;
enum { cudaSuccess = 0 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
// fresh device memory holds garbage on the GPU, fresh mmap-backed malloc memory holds zeros: poison it (0xFF = NaN in every
// float format, -1 in every integer) so that code relying on zero-initialised cudaMalloc memory fails here as well
inline cudaError_t cudaMemset(void* p, int v, size_t n) { std::memset(p, v, n); return 0; }
inline cudaError_t cudaMalloc(void** p, size_t n) {
  *p = std::malloc(n ? n : 1);
  if (*p) std::memset(*p, 0xFF, n ? n : 1);
  return 0;
}
inline cudaError_t cudaFree(void* p) { std::free(p); return 0; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { std::memcpy(d, s, n); return 0; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { std::memcpy(d, s, n); return 0; }
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) { std::memset(d, v, n); return 0; }
inline cudaError_t cudaGetLastError() { return 0; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return 0; }
inline cudaError_t cudaSetDevice(int) { return 0; }
inline cudaError_t cudaGetDevice(int* d) { *d = 0; return 0; }
inline const char* cudaGetErrorString(cudaError_t) { return "emu"; }
template <class F> inline cudaError_t cudaFuncSetAttribute(F f, int, int bytes) {
  emu::S().max_dyn_smem[(const void*)f] = (size_t)bytes;
  return 0;
}
enum { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
#define DQMC_DYN_SMEM(name) unsigned char* name = (unsigned char*)(((uintptr_t)emu::S().dyn_smem.data() + 1023) & ~(uintptr_t)1023)
#define DQMC_LAUNCH(kern, grid, block, smem, stream, ...) \
  emu::launch(dim3(grid), dim3(block), smem, [=]() { kern(__VA_ARGS__); }, (const void*)(kern), #kern)
