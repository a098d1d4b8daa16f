// Metropolis walker update and non-local ECP quadrature kernels.
#pragma once
#include "common.cuh"

namespace dq {

// Gaussian proposal r' = r + tau * N(0,1), all electrons at once.
// reference: src/deepqmc/sampling/electron_samplers.py:102-104.
// noise != nullptr: injected standard normals (parity tests); else Philox keyed by
// (seed; global element pair index, step).
template <class T>
__global__ void propose_kernel(const T* __restrict__ r, T* __restrict__ r_prop, const T* __restrict__ tau,
                               const T* __restrict__ noise, uint64_t seed, uint64_t step, uint64_t elem_offset,
                               int n_elem) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;  // pair index
  const int e0 = 2 * p;
  if (e0 >= n_elem) return;
  const T t = tau[0];
  T z0, z1;
  if (noise) {
    z0 = noise[e0];
    z1 = e0 + 1 < n_elem ? noise[e0 + 1] : T(0);
  } else {
    uint32_t w[4];
    Philox::gen(seed, elem_offset / 2 + (uint64_t)p, step, w);
    double u1 = Philox::u01(w[0], w[1]), u2 = Philox::u01(w[2], w[3]);
    double rad = ::sqrt(-2.0 * ::log(u1)), ang = 6.283185307179586 * u2;
    z0 = (T)(rad * ::cos(ang));
    z1 = (T)(rad * ::sin(ang));
  }
  r_prop[e0] = r[e0] + t * z0;
  if (e0 + 1 < n_elem) r_prop[e0 + 1] = r[e0 + 1] + t * z1;
}

// Spin-exchange proposal (reference: sampling/electron_samplers.py:235-285 OppositeSpinExchangeSampler.exchange_proposal with
// the default uniform logits): r' = r with the positions of one spin-up electron and one spin-down electron swapped.
// idx[b][2] = (up index, down index) injected by parity tests, else drawn from Philox.  One thread per walker.
template <class T>
__global__ void exchange_propose_kernel(const T* __restrict__ r, T* __restrict__ r_prop, const int* __restrict__ idx,
                                        uint64_t seed, uint64_t step, uint64_t walker_offset, int n_up, int N, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  int iu, id;
  if (idx) { iu = idx[2 * b]; id = idx[2 * b + 1]; }
  else {
    uint32_t w[4];
    Philox::gen(seed ^ 0xD1B54A32D192ED03ull, walker_offset + (uint64_t)b, step, w);
    iu = (int)(Philox::u01(w[0], w[1]) * n_up);
    id = (int)(Philox::u01(w[2], w[3]) * (N - n_up));
    iu = iu < n_up ? iu : n_up - 1;
    id = id < N - n_up ? id : N - n_up - 1;
  }
  const T* rb = r + (size_t)b * 3 * N;
  T* pb = r_prop + (size_t)b * 3 * N;
  for (int e = 0; e < 3 * N; ++e) pb[e] = rb[e];
  for (int c = 0; c < 3; ++c) {
    pb[3 * iu + c] = rb[3 * (n_up + id) + c];
    pb[3 * (n_up + id) + c] = rb[3 * iu + c];
  }
}

// Accept/reject, one thread per walker.  reference: electron_samplers.py:106-138
// (2 dlog|psi| > log u, max_age override, age bookkeeping, per-walker select of r/psi/age).
template <class T>
__global__ void accept_kernel(T* __restrict__ r, const T* __restrict__ r_prop, T* __restrict__ sign,
                              const T* __restrict__ sign_p, T* __restrict__ logp, const T* __restrict__ logp_p,
                              int* __restrict__ age, const T* __restrict__ unoise, uint64_t seed, uint64_t step,
                              uint64_t walker_offset, int max_age, int B, int N, int* __restrict__ acc_count) {
  __shared__ int s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) {
    double u;
    if (unoise) u = (double)unoise[b];
    else {
      uint32_t w[4];
      Philox::gen(seed ^ 0x9E3779B97F4A7C15ull, walker_offset + (uint64_t)b, step, w);
      u = Philox::u01(w[0], w[1]);
    }
    double lp = 2.0 * ((double)logp_p[b] - (double)logp[b]);
    bool acc = lp > ::log(u);
    if (max_age >= 0) acc = acc || (age[b] >= max_age);
    if (acc) {
      for (int e = 0; e < 3 * N; ++e) r[(size_t)b * 3 * N + e] = r_prop[(size_t)b * 3 * N + e];
      sign[b] = sign_p[b];
      logp[b] = logp_p[b];
      age[b] = 0;
      atomicAdd(&s_cnt, 1);
    } else {
      age[b] += 1;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_cnt) atomicAdd(acc_count, s_cnt);
}

// ---- Metropolis-adjusted Langevin sampler (reference: sampling/electron_samplers.py:176-232) --------------------
// clean_force (sampling_utils.py:71-101): damp the drift near the nuclei.  grad[B][3N] = d log|psi| / dr from the
// forward-Laplacian pass; z = r_i - R_nearest (plain distances), a = (1 + f^.z^)/2 + Z^2 z^2 / (10 (4 + Z^2 z^2)),
// f <- f 2 / (sqrt(1 + 2 a |f|^2 tau) + 1), then |f| limited to |z| / tau.  One thread per (walker, electron).
template <class T>
__global__ void langevin_force_kernel(const T* __restrict__ grad, const T* __restrict__ r, const T* __restrict__ R,
                                      int R_batched, const T* __restrict__ charges, const T* __restrict__ tau, int N,
                                      int M, int total, T* __restrict__ force) {
  const int bi = blockIdx.x * blockDim.x + threadIdx.x;
  if (bi >= total) return;
  const int b = bi / N;
  const T* ri = r + (size_t)bi * 3;
  const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
  T z0 = 0, z1 = 0, z2 = 0, zz = T(-1), zch = 0;
  for (int m = 0; m < M; ++m) {
    const T d0 = ri[0] - Rb[3 * m], d1 = ri[1] - Rb[3 * m + 1], d2 = ri[2] - Rb[3 * m + 2];
    const T dd = d0 * d0 + d1 * d1 + d2 * d2;
    if (zz < T(0) || dd < zz) { zz = dd; z0 = d0; z1 = d1; z2 = d2; zch = charges[m]; }  // argmin: first minimum
  }
  T f0 = grad[(size_t)bi * 3], f1 = grad[(size_t)bi * 3 + 1], f2 = grad[(size_t)bi * 3 + 2];
  const T eps = Num<T>::eps(), t = tau[0];
  const T zn = m_sqrt(zz);
  T fn = m_sqrt(f0 * f0 + f1 * f1 + f2 * f2);
  const T fc = fn > eps ? fn : eps;
  const T cosfz = (f0 * z0 + f1 * z1 + f2 * z2) / (fc * zn);
  const T Z2z2 = zch * zch * zz;
  const T a = (T(1) + cosfz) / T(2) + Z2z2 / (T(10) * (T(4) + Z2z2));
  const T factor = T(2) / (m_sqrt(T(1) + T(2) * a * fn * fn * t) + T(1));
  f0 *= factor; f1 *= factor; f2 *= factor;
  fn = m_sqrt(f0 * f0 + f1 * f1 + f2 * f2);
  const T lim = zn / (t * (fn > eps ? fn : eps));
  const T nf = lim < T(1) ? lim : T(1);
  force[(size_t)bi * 3] = f0 * nf; force[(size_t)bi * 3 + 1] = f1 * nf; force[(size_t)bi * 3 + 2] = f2 * nf;
}

// proposal r' = r + tau F + sqrt(tau) N(0, 1)  (electron_samplers.py:213-220); noise / Philox as propose_kernel
template <class T>
__global__ void langevin_propose_kernel(const T* __restrict__ r, const T* __restrict__ force, T* __restrict__ r_prop,
                                        const T* __restrict__ tau, const T* __restrict__ noise, uint64_t seed,
                                        uint64_t step, uint64_t elem_offset, int n_elem) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int e0 = 2 * p;
  if (e0 >= n_elem) return;
  const T t = tau[0], st = m_sqrt(t);
  T z0, z1;
  if (noise) {
    z0 = noise[e0];
    z1 = e0 + 1 < n_elem ? noise[e0 + 1] : T(0);
  } else {
    uint32_t w[4];
    Philox::gen(seed, elem_offset / 2 + (uint64_t)p, step, w);
    double u1 = Philox::u01(w[0], w[1]), u2 = Philox::u01(w[2], w[3]);
    double rad = ::sqrt(-2.0 * ::log(u1)), ang = 6.283185307179586 * u2;
    z0 = (T)(rad * ::cos(ang));
    z1 = (T)(rad * ::sin(ang));
  }
  r_prop[e0] = r[e0] + t * force[e0] + st * z0;
  if (e0 + 1 < n_elem) r_prop[e0 + 1] = r[e0 + 1] + t * force[e0 + 1] + st * z1;
}

// accept with log G ratio = sum (F + F') . ((r - r') + tau / 2 (F - F')) plus 2 dlog|psi| (electron_samplers.py:222-232);
// the force travels with the walker state.  One thread per walker.
template <class T>
__global__ void langevin_accept_kernel(T* __restrict__ r, const T* __restrict__ r_prop, T* __restrict__ force,
                                       const T* __restrict__ force_p, T* __restrict__ sign, const T* __restrict__ sign_p,
                                       T* __restrict__ logp, const T* __restrict__ logp_p, int* __restrict__ age,
                                       const T* __restrict__ tau, const T* __restrict__ unoise, uint64_t seed,
                                       uint64_t step, uint64_t walker_offset, int max_age, int B, int N,
                                       int* __restrict__ acc_count) {
  __shared__ int s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) {
    double u;
    if (unoise) u = (double)unoise[b];
    else {
      uint32_t w[4];
      Philox::gen(seed ^ 0x9E3779B97F4A7C15ull, walker_offset + (uint64_t)b, step, w);
      u = Philox::u01(w[0], w[1]);
    }
    const double t = (double)tau[0];
    double lg = 0.0;
    for (int e = 0; e < 3 * N; ++e) {
      const size_t k = (size_t)b * 3 * N + e;
      const double f = (double)force[k], fp = (double)force_p[k];
      lg += (f + fp) * (((double)r[k] - (double)r_prop[k]) + 0.5 * t * (f - fp));
    }
    const double lp = lg + 2.0 * ((double)logp_p[b] - (double)logp[b]);
    bool acc = lp > ::log(u);
    if (max_age >= 0) acc = acc || (age[b] >= max_age);
    if (acc) {
      for (int e = 0; e < 3 * N; ++e) {
        const size_t k = (size_t)b * 3 * N + e;
        r[k] = r_prop[k];
        force[k] = force_p[k];
      }
      sign[b] = sign_p[b];
      logp[b] = logp_p[b];
      age[b] = 0;
      atomicAdd(&s_cnt, 1);
    } else {
      age[b] += 1;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_cnt) atomicAdd(acc_count, s_cnt);
}

// tau <- tau * max(acceptance, 0.05) / target   (reference: electron_samplers.py:121-126)
template <class T>
__global__ void tau_kernel(T* tau, int* acc_count, int B, T target, T* acc_out) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    T acc = (T)acc_count[0] / (T)B;
    if (target > T(0)) {
      T a = acc > T(0.05) ? acc : T(0.05);
      tau[0] = tau[0] / (target / a);
    }
    acc_out[0] = acc;
    acc_count[0] = 0;
  }
}

// Sampler statistics of the final sub-step (reference: electron_samplers.py:154-163):
// out[0]=acceptance (written by tau_kernel), [1]=tau, [2]=age mean, [3]=age max,
// [4]=log|psi| mean, [5]=log|psi| std (population), [6]=mean e-e distance.  Single block.
template <class T>
__global__ void sampler_stats_kernel(const T* __restrict__ r, const T* __restrict__ logp, const int* __restrict__ age,
                                     const T* __restrict__ tau, int B, int N, T* __restrict__ out) {
  __shared__ T scratch[66];
  __shared__ int s_max;
  if (threadIdx.x == 0) s_max = 0;
  __syncthreads();
  T sa = 0, sl = 0, sd = 0;
  int amax = 0;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    sa += (T)age[b];
    amax = age[b] > amax ? age[b] : amax;
    sl += logp[b];
    const T* rb = r + (size_t)b * 3 * N;
    for (int i = 0; i < N; ++i)
      for (int j = i + 1; j < N; ++j) {
        T d0 = rb[3 * i] - rb[3 * j], d1 = rb[3 * i + 1] - rb[3 * j + 1], d2 = rb[3 * i + 2] - rb[3 * j + 2];
        sd += m_sqrt(Num<T>::eps() + d0 * d0 + d1 * d1 + d2 * d2);
      }
  }
  atomicMax(&s_max, amax);
  block_sum2(sa, sl, scratch);
  T mean_l = sl / (T)B;
  T dummy = 0, sv = 0;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    T dl = logp[b] - mean_l;
    sv += dl * dl;
  }
  block_sum2(sd, sv, scratch);
  (void)dummy;
  if (threadIdx.x == 0) {
    out[1] = tau[0];
    out[2] = sa / (T)B;
    out[3] = (T)s_max;
    out[4] = mean_l;
    out[5] = m_sqrt(sv / (T)B);
    int npair = N * (N - 1) / 2;
    out[6] = sd / ((T)B * (T)(npair > 0 ? npair : 1));
  }
}

// Per-rank part of the step statistics (reference: loss/energy.py:63-74 mean energy over all devices,
// observable.py:474-479): out[0] = sum E, [1] = sum E^2, [2] = B, [3..8] = sums of the six hamil stats,
// [9] = max E, [10] = -min E, accumulated in fp64.  Single block; the caller all-gathers the 11 doubles.
template <class T>
__global__ void stats_pack_kernel(const T* __restrict__ E, const T* __restrict__ stats, int B, double* __restrict__ out) {
  __shared__ double sh[32][9];
  __shared__ double shm[32][2];
  double acc[9];
  for (int k = 0; k < 9; ++k) acc[k] = 0.0;
  double mx = -1e300, mn = 1e300;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const double e = (double)E[b];
    acc[0] += e; acc[1] += e * e; acc[2] += 1.0;
    if (stats)
      for (int k = 0; k < 6; ++k) acc[3 + k] += (double)stats[(size_t)k * B + b];
    mx = e > mx ? e : mx;
    mn = e < mn ? e : mn;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  for (int off = 16; off > 0; off >>= 1) {
    for (int k = 0; k < 9; ++k) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], off);
    const double omx = __shfl_xor_sync(0xffffffffu, mx, off), omn = __shfl_xor_sync(0xffffffffu, mn, off);
    mx = omx > mx ? omx : mx;
    mn = omn < mn ? omn : mn;
  }
  if (lane == 0) {
    for (int k = 0; k < 9; ++k) sh[warp][k] = acc[k];
    shm[warp][0] = mx; shm[warp][1] = mn;
  }
  __syncthreads();
  if (threadIdx.x < 11) {
    const int k = threadIdx.x;
    double v = k < 9 ? 0.0 : (k == 9 ? -1e300 : 1e300);
    for (int w = 0; w < nw; ++w) {
      if (k < 9) v += sh[w][k];
      else if (k == 9) v = shm[w][0] > v ? shm[w][0] : v;
      else v = shm[w][1] < v ? shm[w][1] : v;
    }
    out[k] = k == 10 ? -v : v;
  }
}

// ------------------------------------------------------------------------------------------
// Non-local ECP: 12-point icosahedron quadrature, rotated onto r_i - R_I with a random twist
// about the local z axis.  reference: src/deepqmc/ecp/ecp_utils.py:24-60,
// gaussian_type_ecp.py:161-255.  One block per active pair a of the group (ecp_pairs_kernel): pair p = pairs[a] =
// (b*J + j)*N + i (walker b, ecp nucleus slot j, electron i); writes 12 virtual walkers r_virt[v][N][3], v = a*12 + q.
// phi: injected twists [B][J][N] in [0, pi/5) or nullptr -> Philox.  Twist and Philox counter belong to the pair (b, j, i),
// not to its place in the list: a pair's quadrature points do not depend on which other pairs are active.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void ico_vertex(int q, double& th, double& ph) {
  const double pi = 3.141592653589793, at2 = 1.1071487177940904;  // atan(2)
  if (q == 0) { th = 0; ph = 0; }
  else if (q == 1) { th = pi; ph = 0; }
  else {
    int j = (q - 2) / 2;
    if ((q & 1) == 0) { th = at2; ph = pi / 5 * 2 * j; }
    else { th = pi - at2; ph = pi / 5 * (2 * j - 1); }
  }
}

// The twist of pair (walker b of the group, nucleus slot j, electron i): injected phi[B][J][N] or Philox(seed) keyed by the
// pair's global index (ecp_points_kernel and ecp_force_accumulate_kernel draw the same one).
template <class T>
__device__ __forceinline__ double ecp_pair_twist(const T* __restrict__ phi, uint64_t seed, uint64_t walker_offset, int b, int j,
                                                 int i, int J, int N) {
  if (phi) return (double)phi[((size_t)b * J + j) * N + i];
  uint32_t w[4];
  Philox::gen(seed ^ 0xD1B54A32D192ED03ull, (walker_offset + (uint64_t)b) * (uint64_t)(J * N) + (uint64_t)(j * N + i), 0, w);
  return Philox::u01(w[0], w[1]) * (3.141592653589793 / 5);
}

template <class T>
__global__ void ecp_points_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M,
                                  int J, const int* __restrict__ nl_nuc, const T* __restrict__ phi, uint64_t seed,
                                  uint64_t walker_offset, const int* __restrict__ pairs, T* __restrict__ r_virt) {
  __shared__ double pts[12][3];
  const int blk = blockIdx.x, pr = pairs[blk];
  const int i = pr % N, j = (pr / N) % J, b = pr / (N * J);
  const T* rb = r + (size_t)b * 3 * N;
  const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
  const int I = nl_nuc[j];
  if (threadIdx.x < 12) {
    const int q = threadIdx.x;
    double dx = (double)rb[3 * i] - (double)Rb[3 * I], dy = (double)rb[3 * i + 1] - (double)Rb[3 * I + 1],
           dz = (double)rb[3 * i + 2] - (double)Rb[3 * I + 2];
    double radius = ::sqrt(dx * dx + dy * dy + dz * dz);
    double cz = dz / radius;
    cz = cz > 1.0 ? 1.0 : (cz < -1.0 ? -1.0 : cz);
    double theta = ::acos(cz), ph0 = ::atan2(dy, dx);
    const double pr = ecp_pair_twist(phi, seed, walker_offset, b, j, i, J, N);
    double th, ph;
    ico_vertex(q, th, ph);
    double ux = ::sin(th) * ::cos(ph), uy = ::sin(th) * ::sin(ph), uz = ::cos(th);
    // rot_z(pr)
    double ax = ::cos(pr) * ux - ::sin(pr) * uy, ay = ::sin(pr) * ux + ::cos(pr) * uy, az = uz;
    // rot_y(theta)
    double bx = ::cos(theta) * ax + ::sin(theta) * az, by = ay, bz = -::sin(theta) * ax + ::cos(theta) * az;
    // rot_z(ph0)
    double cx = ::cos(ph0) * bx - ::sin(ph0) * by, cy = ::sin(ph0) * bx + ::cos(ph0) * by;
    pts[q][0] = radius * cx + (double)Rb[3 * I];
    pts[q][1] = radius * cy + (double)Rb[3 * I + 1];
    pts[q][2] = radius * bz + (double)Rb[3 * I + 2];
  }
  __syncthreads();
  T* out = r_virt + (size_t)blk * 12 * 3 * N;
  for (int idx = threadIdx.x; idx < 12 * 3 * N; idx += blockDim.x) {
    int q = idx / (3 * N), e = idx % (3 * N);
    out[idx] = (e / 3 == i) ? (T)pts[q][e % 3] : rb[e];
  }
}

// Active (nucleus, electron) pairs of a group of B walkers (ecp_pair_active, common.cuh), in the order walker, nucleus slot,
// electron: pairs[] = the group-local pair indices (b J + j) N + i, offs[b] = the walker's first entry, *total = the count.
// One block: warp w counts walkers w, w + 32, ... (ballot per 32 pairs), a block scan turns the counts into offsets, the
// warps write their walkers' pairs at the ballot ranks.  The list is a subsequence of all B J N pairs in their natural order.
template <class T>
__global__ void __launch_bounds__(1024)
ecp_pairs_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M, int J,
                 const int* __restrict__ nl_nuc, const double* __restrict__ rc2, int B, int* __restrict__ offs,
                 int* __restrict__ pairs, int* __restrict__ total) {
  __shared__ int wsum[32];
  __shared__ int carry;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5, JN = J * N;
  auto active = [&](int b, int p) {
    if (p >= JN) return false;
    const int j = p / N, i = p - j * N, I = nl_nuc[j];
    const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
    double d2;
    return ecp_pair_active(r + ((size_t)b * N + i) * 3, Rb + 3 * I, rc2[j], d2);
  };
  for (int b = warp; b < B; b += nw) {
    int cnt = 0;
    for (int p0 = 0; p0 < JN; p0 += 32) cnt += __popc(__ballot_sync(0xffffffffu, active(b, p0 + lane)));
    if (lane == 0) offs[b] = cnt;
  }
  if (tid == 0) carry = 0;
  for (int base = 0; base < B; base += blockDim.x) {  // exclusive scan of offs[0 .. B) in place
    __syncthreads();  // counts written / previous round's carry and wsum read
    const int idx = base + tid;
    const int c = idx < B ? offs[idx] : 0;
    int x = c;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_sync(0xffffffffu, x, lane >= o ? lane - o : lane);
      if (lane >= o) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int s = lane < nw ? wsum[lane] : 0;
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_sync(0xffffffffu, s, lane >= o ? lane - o : lane);
        if (lane >= o) s += y;
      }
      if (lane < nw) wsum[lane] = s;
    }
    __syncthreads();
    if (idx < B) offs[idx] = carry + (warp ? wsum[warp - 1] : 0) + x - c;
    __syncthreads();
    if (tid == 0) carry += wsum[nw - 1];
  }
  __syncthreads();
  if (tid == 0) *total = carry;
  for (int b = warp; b < B; b += nw) {
    int slot = offs[b];
    for (int p0 = 0; p0 < JN; p0 += 32) {
      const bool act = active(b, p0 + lane);
      const unsigned m = __ballot_sync(0xffffffffu, act);
      if (act) pairs[slot + __popc(m & ((1u << lane) - 1u))] = b * JN + p0 + lane;
      slot += __popc(m);
    }
  }
}

// V_nl[b] = sum_{j,i,l} (2l+1)/12 v_l(|r_i - R_I|) sum_q P_l(cos th_q) psi(r_i->q)/psi(r)
// (reference: ecp/gaussian_type_ecp.py:161-255).  One WARP per walker: lanes stride over the
// (nucleus, electron) pairs, 12 quadrature ratios each, warp-shuffle reduction; accumulation in
// double.  Only the pairs inside the cutoff (ecp_pair_active) have quadrature forwards: the walker's
// active pairs are entries offs[b], offs[b] + 1, ... of the group's pair list (ecp_pairs_kernel), in
// the order of this loop; a pair outside adds nothing.  Adds V_nl to E_loc and to stats[3].
template <class T>
__global__ void ecp_accumulate_kernel(const T* __restrict__ r, const T* __restrict__ R, int R_batched, int N, int M,
                                      int J, const int* __restrict__ nl_nuc, const T* __restrict__ nl_params,
                                      const double* __restrict__ rc2, const int* __restrict__ offs,
                                      int L, int Tm, const T* __restrict__ sign0, const T* __restrict__ log0,
                                      const T* __restrict__ sign_v, const T* __restrict__ log_v, int B, int Bstat,
                                      T* __restrict__ out_E, T* __restrict__ out_stats) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;  // warp-uniform
  const T* rb = r + (size_t)b * 3 * N;
  const T* Rb = R + (R_batched ? (size_t)b * M * 3 : 0);
  const double l0 = (double)log0[b], s0 = (double)sign0[b];
  double total = 0.0;
  int slot = offs[b];
  for (int p0 = 0; p0 < J * N; p0 += 32) {  // warp-uniform trip count: every lane takes part in the ballot
    const int p = p0 + lane;
    const int j = p / N, i = p - j * N;
    const int I = p < J * N ? nl_nuc[j] : 0;
    double d2 = 0.0;
    const bool act = p < J * N && ecp_pair_active(rb + 3 * i, Rb + 3 * I, rc2[j], d2);
    const unsigned m = __ballot_sync(0xffffffffu, act);
    const int a = slot + __popc(m & ((1u << lane) - 1u));
    slot += __popc(m);
    if (!act) continue;
    const T* nl = nl_params + (size_t)I * L * 2 * Tm;
    double integ[4] = {0, 0, 0, 0};
    for (int q = 0; q < 12; ++q) {
      size_t v = (size_t)a * 12 + q;
      double ratio = ::exp((double)log_v[v] - l0) * (double)sign_v[v] * s0;
      double th, ph;
      ico_vertex(q, th, ph);
      double x = ::cos(th);
      double pl[4] = {1.0, x, 0.5 * (3 * x * x - 1), 0.5 * (5 * x * x * x - 3 * x)};
      for (int l = 0; l < L; ++l) integ[l] += ratio * pl[l];
    }
    for (int l = 0; l < L; ++l) {
      double vl = 0.0;
      for (int t = 0; t < Tm; ++t) vl += (double)nl[(l * 2 + 1) * Tm + t] * ::exp(-(double)nl[(l * 2 + 0) * Tm + t] * d2);
      total += vl * (2 * l + 1) / 12.0 * integ[l];
    }
  }
  total = warp_sum(total);
  if (lane == 0) {
    out_E[b] += (T)total;
    out_stats[3 * (size_t)Bstat + b] = (T)total;
  }
}

// Non-local ECP force (reference: ecp/gaussian_type_ecp.py:257-328, ecp_force_utils.py): out[b][I] = -grad_{R_I} of
// nucleus I's share of V_nl, sum_i sum_l (2l+1)/12 v_l(rho) sum_q P_l(cos th_q) psi(r_q(R), R) / psi(r, R), rho = |r_i - R_I|;
// rows of nuclei without a non-local term are zero.  With d = r_i - R_I, r_q = R_I + f_q(d), f_q = rho Rz(phi) Ry(theta) w_q,
// w_q = Rz(twist) u_q (ecp_points_kernel):
//   d ratio_q / d R_I = ratio_q [g_R(r_q)[I] + (1 - df_q/dd)^T g_r(r_q)[i] - g_R(r)[I]],
//   df_q/dd = (f_q / rho) d^T / rho + rho Rz(phi) Ry'(theta) w_q (dtheta/dd)^T + rho Rz'(phi) Ry(theta) w_q (dphi/dd)^T,
//   dtheta/dd = (d_z d / rho^2 - e_z) / s, dphi/dd = (-d_y, d_x, 0) / s^2, s = sqrt(d_x^2 + d_y^2),
//   d v_l / d R_I = 2 d sum_t alpha beta exp(-alpha rho^2).
// g_r, g_R = grad_r, grad_R log|psi| from the position reverse pass: of the base walkers (gR0[nb][M][3], sign0, log0) and of
// the virtual walkers of the active pairs (gr_v[V][N][3], gR_v[V][M][3], sign_v, log_v, v = 12 a + q for the pair's entry a in
// the group's list, ecp_pairs_kernel with the force's cutoff rc2).  One WARP per walker: nucleus slot by nucleus slot, lanes
// stride over the electrons, everything in double, a fixed shuffle tree per slot -- no atomics.
template <class T>
__global__ void ecp_force_accumulate_kernel(const T* __restrict__ r, const T* __restrict__ R, int N, int M, int J,
                                            const int* __restrict__ nl_nuc, const T* __restrict__ nl_params,
                                            const double* __restrict__ rc2, const int* __restrict__ offs, int L, int Tm,
                                            const T* __restrict__ phi, uint64_t seed, uint64_t walker_offset,
                                            const T* __restrict__ sign0, const T* __restrict__ log0, const T* __restrict__ gR0,
                                            const T* __restrict__ sign_v, const T* __restrict__ log_v,
                                            const T* __restrict__ gr_v, const T* __restrict__ gR_v, int B, T* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;  // warp-uniform
  const T* rb = r + (size_t)b * 3 * N;
  T* ob = out + (size_t)b * M * 3;
  for (int k = lane; k < 3 * M; k += 32) ob[k] = T(0);
  __syncwarp();
  const double l0 = (double)log0[b], s0 = (double)sign0[b];
  int slot = offs[b];
  for (int j = 0; j < J; ++j) {
    const int I = nl_nuc[j];
    const T* nl = nl_params + (size_t)I * L * 2 * Tm;
    const double g0[3] = {(double)gR0[((size_t)b * M + I) * 3], (double)gR0[((size_t)b * M + I) * 3 + 1],
                          (double)gR0[((size_t)b * M + I) * 3 + 2]};
    double acc[3] = {0.0, 0.0, 0.0};
    for (int i0 = 0; i0 < N; i0 += 32) {  // warp-uniform trip count: every lane takes part in the ballot
      const int i = i0 + lane;
      double d2 = 0.0;
      const bool act = i < N && ecp_pair_active(rb + 3 * i, R + 3 * I, rc2[j], d2);
      const unsigned m = __ballot_sync(0xffffffffu, act);
      const int a = slot + __popc(m & ((1u << lane) - 1u));
      slot += __popc(m);
      if (!act) continue;
      const double d[3] = {(double)rb[3 * i] - (double)R[3 * I], (double)rb[3 * i + 1] - (double)R[3 * I + 1],
                           (double)rb[3 * i + 2] - (double)R[3 * I + 2]};
      const double rho = ::sqrt(d2), s2 = d[0] * d[0] + d[1] * d[1], s = ::sqrt(s2);
      double cz = d[2] / rho;
      cz = cz > 1.0 ? 1.0 : (cz < -1.0 ? -1.0 : cz);
      const double th = ::acos(cz), ph = ::atan2(d[1], d[0]), tw = ecp_pair_twist(phi, seed, walker_offset, b, j, i, J, N);
      const double ct = ::cos(th), st = ::sin(th), cp = ::cos(ph), sp = ::sin(ph), cw = ::cos(tw), sw = ::sin(tw);
      const double dth[3] = {(d[2] * d[0] / d2) / s, (d[2] * d[1] / d2) / s, (d[2] * d[2] / d2 - 1.0) / s};
      const double dph[3] = {-d[1] / s2, d[0] / s2, 0.0};
      double integ[4] = {0, 0, 0, 0}, dinteg[4][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
      for (int q = 0; q < 12; ++q) {
        const size_t v = (size_t)a * 12 + q;
        const double ratio = ::exp((double)log_v[v] - l0) * (double)sign_v[v] * s0;
        double qt, qp;
        ico_vertex(q, qt, qp);
        const double ux = ::sin(qt) * ::cos(qp), uy = ::sin(qt) * ::sin(qp), uz = ::cos(qt);
        const double wx = cw * ux - sw * uy, wy = sw * ux + cw * uy, wz = uz;               // Rz(twist) u
        const double A[3] = {ct * wx + st * wz, wy, -st * wx + ct * wz};                     // Ry(theta) w
        const double Ad[3] = {-st * wx + ct * wz, 0.0, -ct * wx - st * wz};                  // Ry'(theta) w
        const double f[3] = {rho * (cp * A[0] - sp * A[1]), rho * (sp * A[0] + cp * A[1]), rho * A[2]};
        const double t1[3] = {rho * (cp * Ad[0] - sp * Ad[1]), rho * (sp * Ad[0] + cp * Ad[1]), rho * Ad[2]};
        const double t2[3] = {rho * (-sp * A[0] - cp * A[1]), rho * (cp * A[0] - sp * A[1]), 0.0};
        const T* gr = gr_v + (v * N + i) * 3;
        const T* gR = gR_v + (v * M + I) * 3;
        const double g[3] = {(double)gr[0], (double)gr[1], (double)gr[2]};
        const double fg = (f[0] * g[0] + f[1] * g[1] + f[2] * g[2]) / d2, t1g = t1[0] * g[0] + t1[1] * g[1] + t1[2] * g[2],
                     t2g = t2[0] * g[0] + t2[1] * g[1] + t2[2] * g[2];
        double dr[3];
        for (int c = 0; c < 3; ++c)  // ratio_q [g_R(r_q) + g_r(r_q) - J^T g_r(r_q) - g_R(r)]
          dr[c] = ratio * ((double)gR[c] + g[c] - (d[c] * fg + dth[c] * t1g + dph[c] * t2g) - g0[c]);
        const double x = ::cos(qt);
        const double pl[4] = {1.0, x, 0.5 * (3 * x * x - 1), 0.5 * (5 * x * x * x - 3 * x)};
        for (int l = 0; l < L; ++l) {
          integ[l] += ratio * pl[l];
          for (int c = 0; c < 3; ++c) dinteg[l][c] += dr[c] * pl[l];
        }
      }
      for (int l = 0; l < L; ++l) {
        double vl = 0.0, dvl = 0.0;
        for (int t = 0; t < Tm; ++t) {
          const double al = (double)nl[(l * 2 + 0) * Tm + t], be = (double)nl[(l * 2 + 1) * Tm + t], e = ::exp(-al * d2);
          vl += be * e;
          dvl += al * be * e;
        }
        const double c = (2 * l + 1) / 12.0;
        for (int k = 0; k < 3; ++k) acc[k] += c * (2 * d[k] * dvl * integ[l] + vl * dinteg[l][k]);
      }
    }
    for (int k = 0; k < 3; ++k) acc[k] = warp_sum(acc[k]);
    if (lane == 0)
      for (int k = 0; k < 3; ++k) ob[(size_t)I * 3 + k] = (T)(-acc[k]);
  }
}

// Virtual walkers of the spin pass: r_virt[b P + p] = r[b] with the positions of electrons a and beta of pair p swapped.
// One thread per coordinate of r_virt.
template <class T>
__global__ void spin_pairs_kernel(const T* __restrict__ r, int N, int n_up, int down_idx, int P, int64_t n_elem,
                                  T* __restrict__ r_virt) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_elem) return;
  const int64_t v = idx / (3 * N);
  const int e = (int)(idx - v * 3 * N), i = e / 3, c = e - 3 * i;
  const int64_t b = v / P;
  int a, beta;
  spin_pair((int)(v - b * P), n_up, N, down_idx, a, beta);
  const int src = i == a ? beta : (i == beta ? a : i);
  r_virt[idx] = r[(b * N + src) * 3 + c];
}

// Spin estimators from the swapped forwards (reference: physics.py:159-239).  rho_p = sign' sign exp(log' - log) in fp64;
// s2[b] = c0 - sum_p rho_p with c0 = D/2 (D/2 + 1) + n_down (exact) or 1 (spin-raising).  One WARP per walker: lane l sums
// the pairs p = l, l + 32, ... in order, then a fixed shuffle tree -- no atomics, so a repeated call is bitwise identical.
// P = 0 (no down electrons): s2 = c0 without reading the forwards.  ratio[B][P] (nullable) receives rho.
template <class T>
__global__ void spin_accumulate_kernel(const T* __restrict__ sign0, const T* __restrict__ log0, const T* __restrict__ sign_v,
                                       const T* __restrict__ log_v, int P, int B, double c0, T* __restrict__ s2,
                                       T* __restrict__ ratio) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;  // warp-uniform
  double total = 0.0;
  if (P > 0) {
    const double l0 = (double)log0[b], s0 = (double)sign0[b];
    for (int p = lane; p < P; p += 32) {
      const size_t v = (size_t)b * P + p;
      const double rho = (double)sign_v[v] * s0 * ::exp((double)log_v[v] - l0);
      total += rho;
      if (ratio) ratio[v] = (T)rho;
    }
  }
  total = warp_sum(total);
  if (lane == 0) s2[b] = (T)(c0 - total);
}

}  // namespace dq
