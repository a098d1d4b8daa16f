// Host side of libdqmc_b200.so: engine object, parameter table, workspace planning, kernel
// sequencing, C ABI (include/dqmc_b200.h).  Built by nvcc for sm_90a (H100); with -DDQMC_EMU -DDQMC_NO_TCGEN05 the
// same file builds against tools/cuda_emu for CPU-side logic checks of the SIMT kernels during development (never shipped).
#include <algorithm>
#include <array>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <map>
#include <mutex>
#include <optional>
#include <string>
#include <type_traits>
#include <vector>

#include "dqmc_b200.h"
#include "kernels_mcmc.cuh"
#include "kernels_slater.cuh"
#include "kernels_trunk.cuh"
#include "kernels_gnn.cuh"
#include "kernels_bwd.cuh"
#include "kernels_zv.cuh"
#include "attn_mma.cuh"
#if !defined(DQMC_NO_TCGEN05)
#include "gemm_wgmma.cuh"
#include "fused_tc.cuh"
#include "trunk_tc.cuh"
#endif

namespace dq {

struct ParamEntry {
  std::string name;
  int64_t offset;
  int rows, cols;
};

static inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// largest d2 >= lo with w(d2) >= eps, for w falling on [lo, inf) with w(lo) >= eps: doubling, then bisection to adjacent doubles
template <class W>
static double last_above(W w, double lo, double eps) {
  double hi = lo > 0.0 ? 2 * lo : 1.0;
  while (w(hi) >= eps) { lo = hi; hi *= 2; }
  for (;;) {
    const double mid = lo + 0.5 * (hi - lo);
    if (mid <= lo || mid >= hi) break;
    (w(mid) >= eps ? lo : hi) = mid;
  }
  return lo;
}

// Squared cutoff radius of one non-local ECP nucleus, nl[l][alpha | beta][t] as the accumulator reads it: the largest d2 with
// w(d2) = sum_l (2l+1) sum_t |beta_lt| exp(-alpha_lt d2) >= 2^-100.  A pair's term in V_nl is at most w(d2) max_q |psi ratio|
// (sum_q |P_l(cos th_q)| <= 12), so the pairs beyond it are skipped (common.cuh ecp_pair_active).  w falls monotonically
// when every alpha with beta != 0 is positive, and the bisection runs to adjacent doubles.  +inf: no cutoff (on == false,
// DQMC_ECP_CUTOFF=0, or a term that does not decay).
template <class T>
static double ecp_cutoff_rc2(const T* nl, int L, int Tn, bool on) {
  const double inf = std::numeric_limits<double>::infinity(), eps = std::ldexp(1.0, -100);
  if (!on) return inf;
  for (int l = 0; l < L; ++l)
    for (int t = 0; t < Tn; ++t)
      if ((double)nl[(l * 2 + 1) * Tn + t] != 0.0 && !((double)nl[(l * 2) * Tn + t] > 0.0)) return inf;
  auto w = [&](double d2) {
    double s = 0.0;
    for (int l = 0; l < L; ++l)
      for (int t = 0; t < Tn; ++t)
        s += (2 * l + 1) * std::fabs((double)nl[(l * 2 + 1) * Tn + t]) * std::exp(-(double)nl[(l * 2) * Tn + t] * d2);
    return s;
  };
  if (w(0.0) < eps) return -inf;  // no pair is ever active
  return last_above(w, 0.0, eps);
}

// Squared cutoff radius of the non-local ECP force (dqmc_ecp_force): a pair's share of grad_R V_nl is bounded by the weight w
// above and by its radial derivative w'(rho) = sum_l (2l+1) sum_t 2 alpha_lt |beta_lt| rho exp(-alpha_lt rho^2) times the
// ratios and their gradients, so the radius bounds both by 2^-100.  Each term of w' rises up to rho^2 = 1 / (2 alpha) and falls
// beyond, so w' falls from the largest of those points on and the bisection starts there; a radius inside it keeps that whole
// ball.  Never smaller than the energy's radius; +inf wherever that one is.
template <class T>
static double ecp_force_cutoff_rc2(const T* nl, int L, int Tn, bool on) {
  const double rc2 = ecp_cutoff_rc2(nl, L, Tn, on), eps = std::ldexp(1.0, -100);
  if (rc2 == std::numeric_limits<double>::infinity()) return rc2;
  double peak = 0.0;
  for (int l = 0; l < L; ++l)
    for (int t = 0; t < Tn; ++t)
      if ((double)nl[(l * 2 + 1) * Tn + t] != 0.0) peak = std::max(peak, 0.5 / (double)nl[(l * 2) * Tn + t]);
  auto wd = [&](double d2) {
    double s = 0.0;
    for (int l = 0; l < L; ++l)
      for (int t = 0; t < Tn; ++t) {
        const double a = (double)nl[(l * 2) * Tn + t];
        s += (2 * l + 1) * 2 * a * std::fabs((double)nl[(l * 2 + 1) * Tn + t]) * std::sqrt(d2) * std::exp(-a * d2);
      }
    return s;
  };
  return std::max(rc2, wd(peak) >= eps ? last_above(wd, peak, eps) : peak);
}

// The A/B switches (DESIGN §9), read from the environment once, when an engine is created.  A flag switch is on when its
// variable is set, whatever the value; the DQMC_ATTN_TB / DQMC_ATTN_NT values are range-checked where they are used.
struct Switches {
  bool tc_trunk = true;              // DQMC_TC_TRUNK=0: plain forwards without the whole-trunk kernel
  bool tc_f16 = true;                // DQMC_TC_F16=0: plain forwards on 3xTF32 instead of 3xFP16 row GEMMs
  std::optional<bool> attn_fl_mma;   // DQMC_ATTN_FL_MMA=0 / 1: force the SIMT / tensor-core forward-Laplacian attention
  std::optional<int> attn_tb, attn_nt;  // DQMC_ATTN_TB, DQMC_ATTN_NT: its tangent slots per chunk, threads per block
  bool attn_generic = false;         // DQMC_ATTN_GENERIC
  bool no_fuse_tanh = false;         // DQMC_NO_FUSE_TANH
  bool slater_generic = false;       // DQMC_SLATER_GENERIC
  bool slater_fwd1 = false;          // DQMC_SLATER_FWD1
  bool ecp_cutoff = true;            // DQMC_ECP_CUTOFF=0: every (nucleus, electron) pair runs its quadrature forwards
  bool ecp_env_table = true;         // DQMC_ECP_ENV_TABLE_OFF
  bool ecp_emb_table = true;         // DQMC_ECP_EMB_TABLE_OFF
  int nsms = 0;                      // DQMC_NSMS >= 1: SM count the persistent kernels size their grids by (test hook)
  bool trunk_phases = false;         // DQMC_TRUNK_PHASES=1: the whole-trunk kernel's phase timers
};

inline Switches read_switches() {
  auto env = [](const char* name) { return std::getenv(name); };
  auto num = [&](const char* name) { const char* ev = env(name); return ev ? std::optional<int>(std::atoi(ev)) : std::nullopt; };
  Switches s;
  s.tc_trunk = num("DQMC_TC_TRUNK").value_or(1) != 0;
  s.tc_f16 = num("DQMC_TC_F16").value_or(1) != 0;
  if (auto v = num("DQMC_ATTN_FL_MMA")) s.attn_fl_mma = *v != 0;
  s.attn_tb = num("DQMC_ATTN_TB");
  s.attn_nt = num("DQMC_ATTN_NT");
  s.attn_generic = env("DQMC_ATTN_GENERIC");
  s.no_fuse_tanh = env("DQMC_NO_FUSE_TANH");
  s.slater_generic = env("DQMC_SLATER_GENERIC");
  s.slater_fwd1 = env("DQMC_SLATER_FWD1");
  s.ecp_cutoff = num("DQMC_ECP_CUTOFF").value_or(1) != 0;
  s.ecp_env_table = !env("DQMC_ECP_ENV_TABLE_OFF");
  s.ecp_emb_table = !env("DQMC_ECP_EMB_TABLE_OFF");
  s.nsms = num("DQMC_NSMS").value_or(0);
  s.trunk_phases = num("DQMC_TRUNK_PHASES").value_or(0) != 0;
  return s;
}

struct EngineBase {
  dqmc_config cfg;
  int device = 0;
  std::string err;
  int64_t launches = 0;
  int64_t ecp_forwards = 0;  // quadrature virtual walkers run by the non-local ECP pass (12 per active pair)
  std::vector<ParamEntry> entries;
  int64_t total = 0;
  // Planning pass: the host code of an entry point is walked with every CUDA call skipped, so that the number of workspace
  // bytes a call carves is computed by the SAME code that carves them (dqmc_workspace_bytes, dqmc_debug_plan).  An engine
  // created with device < 0 is plan-only (dry for its whole life: no CUDA context, no allocation).
  bool dry = false;
  bool plan_only = false;
  mutable const char* dry_hwm = nullptr;  // highest workspace address carved during a dry pass
  void note_hwm(const void* q) const { if (dry && (const char*)q > dry_hwm) dry_hwm = (const char*)q; }
  mutable std::vector<unsigned char*> emu_guards;  // emulator builds only: guard zones behind the carved workspace buffers
  // optional per-launch timing of the dominant (GEMM) kernels with CUDA events on the caller's stream
  bool prof = false;
  double prof_flops = 0;
  int64_t prof_n = 0;
  // per kernel class: 0 row GEMM (one dense layer per launch), 1 fused MLP block, 2 whole trunk (all layers in one launch)
  double prof_cls_flops[3] = {0, 0, 0};
  int64_t prof_cls_n[3] = {0, 0, 0};
  std::vector<int> prof_cls;
#ifndef DQMC_EMU
  std::vector<cudaEvent_t> prof_ev;
  void prof_note(cudaEvent_t e0, cudaEvent_t e1, double flops, int cls) {
    prof_ev.push_back(e0); prof_ev.push_back(e1);
    prof_cls.push_back(cls);
    prof_flops += flops; prof_cls_flops[cls] += flops;
    ++prof_n; ++prof_cls_n[cls];
  }
#endif
  virtual ~EngineBase() {}
  virtual int set_params(const double* host, int64_t n, cudaStream_t st) = 0;
  virtual int64_t ws_bytes(int B, int mode) = 0;
  virtual int64_t ws_bytes_min(int B, int mode) = 0;
  virtual int debug_plan(int B, int mode, int64_t wsb, int64_t* planned, int64_t* carved) = 0;
  virtual int stats_pack(const void* E, const void* stats, int B, double* out, cudaStream_t st) = 0;
  virtual int debug_mlp_block(int layer, const void* O, const void* X, void* Out, int rows, cudaStream_t st) = 0;
  virtual int debug_trunk(const void* X0, void* Out, int rows, cudaStream_t st) = 0;
  virtual int debug_attention(int layer, const void* QKV, void* O, int rows, int S, int32_t* kernel, cudaStream_t st) = 0;
  virtual int debug_mlp(int layer, int S, const void* O, const void* X, void* Out, void* scratch, int rows, int32_t* path,
                        cudaStream_t st) = 0;
  virtual int debug_trunk_phases(uint64_t* out, int n) = 0;
  virtual int debug_tc_error(int32_t* flag) = 0;
  virtual int debug_slater(const void* r, const void* R, const void* BF, int rows, int S, void* dsign, void* dlog, void* dgrad,
                           void* dlap, int32_t* kernel, cudaStream_t st) = 0;
  virtual int debug_det_sum(const void* r, const void* R, const void* dsign, const void* dlog, const void* dgrad,
                            const void* dlap, int B, int S, void* sign, void* logp, void* grad, void* stats,
                            cudaStream_t st) = 0;
  virtual int debug_wgrad(const void* A, const void* dY, int rows, int Kc, int Nc, int lo, int hi, void* dW, void* db,
                          cudaStream_t st) = 0;
  virtual int debug_attention_bwd(int layer, const void* QKV, const void* dO, void* dQKV, void* dKn, void* dVn, int rows,
                                  cudaStream_t st) = 0;
  virtual int forward(const void* r, const void* R, int Rb, int B, void* sign, void* logp, void* ws, int64_t wsb,
                      cudaStream_t st) = 0;
  virtual int local_energy(const void* r, const void* R, int Rb, int B, uint64_t seed, const void* twist, void* E,
                           void* stats, void* sign, void* logp, void* grad, void* ws, int64_t wsb,
                           cudaStream_t st) = 0;
  virtual int langevin(void* r, void* sign, void* logp, void* force, int32_t* age, void* tau, const void* R, int Rb, int B,
                       int n_sub, double target, int max_age, uint64_t seed, uint64_t step0, uint64_t woff, const void* nn,
                       const void* nu, void* stats, void* ws, int64_t wsb, cudaStream_t st) = 0;
  virtual int vjp_params(const void* r, const void* R, int Rb, int B, const void* weights, void* sign, void* logp,
                         void* grad_params, void* ws, int64_t wsb, cudaStream_t st) = 0;
  virtual int spin(const void* r, const void* R, int Rb, int B, const void* sign, const void* logp, int down_idx, void* s2,
                   void* ratio, void* ws, int64_t wsb, cudaStream_t st) = 0;
  virtual int grad_positions(const void* r, const void* R, int Rb, int B, void* sign, void* logp, void* grad_r, void* grad_R,
                             void* ws, int64_t wsb, cudaStream_t st) = 0;
  virtual int force_terms(const void* r, const void* R, int Rb, int B, const void* grad_r, void* bare, void* zvq, void* Q,
                          cudaStream_t st) = 0;
  virtual int ecp_force(const void* r, const void* R, int Rb, int B, uint64_t seed, const void* twist, void* bare, void* nl,
                        void* ws, int64_t wsb, cudaStream_t st) = 0;
  virtual int zv_force(const void* r, const void* R, int Rb, int B, void* zv, void* grad_R, void* ws, int64_t wsb,
                       cudaStream_t st) = 0;
  virtual int orbitals(const void* r, const void* R, int Rb, int B, void* out, void* ws, int64_t wsb, cudaStream_t st) = 0;
  virtual int set_ph(int n_tab, int n_grid, double r_max, const double* tables, const int32_t* tab_of_nuc) = 0;
  virtual int debug_gemm(const char* wname, const char* bname, const void* A, const void* Res, void* C, int Mr, int S,
                         int sliced, int backend, cudaStream_t st) = 0;
  virtual int mcmc(void* r, void* sign, void* logp, int32_t* age, void* tau, const void* R, int Rb, int B, int n_sub,
                   double target, int max_age, uint64_t seed, uint64_t step0, uint64_t woff, const void* nn,
                   const void* nu, void* stats, void* ws, int64_t wsb, cudaStream_t st, double p_exchange = 0.0,
                   const int32_t* ex_flags = nullptr, const int32_t* ex_idx = nullptr) = 0;

  // width of the type-t edge stream (same / anti / ne) entering layer l: the raw features, or edge_dim after a deep layer
  int gnn_ein(int t, int l) const {
    if (cfg.gnn_deep_edges && l > 0) return cfg.edge_dim;
    return cfg.gnn_edge_in[t] > 0 ? cfg.gnn_edge_in[t] : 4;
  }
  // width of the h_ne rows of layer l: the filter's width, i.e. the ne edge stream itself when it is the filter
  int gnn_hne_w(int l) const { return cfg.gnn_ne_identity ? gnn_ein(2, l) : cfg.edge_dim; }
  // convolution columns of layer l: [conv_same | conv_anti (| conv_ne)] or [conv_same + conv_anti | conv_ne]
  int gnn_conv_w(int l) const {
    return (cfg.gnn_ne_identity ? 1 : 2) * cfg.edge_dim + (cfg.gnn_conv_ne ? gnn_hne_w(l) : 0);
  }
  void add(const std::string& n, int rows, int cols) {
    entries.push_back({n, total, rows, cols});
    total += (int64_t)rows * cols;
  }
  void build_layout() {
    const int N = cfg.n_up + cfg.n_down, M = cfg.n_nuc, d = cfg.embedding_dim, K = cfg.n_determinants;
    const int rep = cfg.n_env_per_nuc > 1 ? cfg.n_env_per_nuc : 1;
    if (cfg.kind == DQMC_PSIFORMER || cfg.kind == DQMC_TRANSPSIFORMER) {
      add("emb.w", 4 * M + 1, d);
      for (int l = 0; l < cfg.n_layers; ++l) {
        std::string p = "L" + std::to_string(l) + ".";
        add(p + "wqkv", d, 3 * d);
        add(p + "wo", d, d);
        add(p + "w1", d, d);
        add(p + "b1", 1, d);
        add(p + "w2", d, d);
        add(p + "b2", 1, d);
        if (cfg.kind == DQMC_TRANSPSIFORMER && cfg.n_nuc_tokens > 0) {
          add(p + "kn", cfg.n_nuc_tokens, d);  // key / value rows of the nuclear tokens (host-evaluated stream)
          add(p + "vn", cfg.n_nuc_tokens, d);
        }
      }
    }
    int bf_in = d;  // input width of the final backflow layer
    if (cfg.kind == DQMC_PAULINET) {
      // reference tests/conf/ansatz.yaml and conf/ansatz/default.yaml; entry names mirror the Haiku modules
      const int e = cfg.edge_dim, nl = cfg.gnn_sub_n > 0 ? cfg.gnn_sub_n : 1;
      if (!cfg.gnn_features) add("emb.table", cfg.n_elec_types > 0 ? cfg.n_elec_types : 1, d);
      int dcur = cfg.gnn_features ? 4 * M : d;
      const int nt = cfg.gnn_conv_ne ? 3 : 2;
      const char* tn[3] = {"same", "anti", "ne"};
      for (int l = 0; l < cfg.n_layers; ++l) {
        std::string p = "G" + std::to_string(l) + ".";
        for (int t = 0; t < nt; ++t) {
          int din = gnn_ein(t, l);
          for (int i = 0; i < nl && !(t == 2 && cfg.gnn_ne_identity); ++i) {
            const std::string q = p + "w_" + tn[t] + "." + std::to_string(i);
            add(q + ".w", din, cfg.gnn_w_dims[l][i]);
            if (cfg.gnn_w_bias) add(q + ".b", 1, cfg.gnn_w_dims[l][i]);
            din = cfg.gnn_w_dims[l][i];
          }
          if (t < 2) {
            din = dcur;
            for (int i = 0; i < nl; ++i) {
              const std::string q = p + "h_" + tn[t] + "." + std::to_string(i);
              add(q + ".w", din, cfg.gnn_h_dims[l][i]); add(q + ".b", 1, cfg.gnn_h_dims[l][i]);
              din = cfg.gnn_h_dims[l][i];
            }
          } else {
            add(p + "hne", M, gnn_hne_w(l));  // h_ne(nuclear embedding table): walker-independent, evaluated on the host
          }
          if (!cfg.gnn_concat) { add(p + "g_" + tn[t] + ".w", e, d); add(p + "g_" + tn[t] + ".b", 1, d); }
        }
        if (cfg.gnn_concat) {
          add(p + "g.w", 3 * dcur + gnn_conv_w(l), d);
          if (cfg.gnn_g_bias) add(p + "g.b", 1, d);
        }
        if (cfg.gnn_deep_edges && l < cfg.n_layers - 1) {
          for (int t = 0; t < (cfg.gnn_sep_edges ? nt : 1); ++t) {
            int din = gnn_ein(t, l);
            for (int i = 0; i < nl; ++i) {
              const std::string q = p + (cfg.gnn_sep_edges ? std::string("u_") + tn[t] : std::string("u")) + "." + std::to_string(i);
              add(q + ".w", din, cfg.gnn_u_dims[l][i]); add(q + ".b", 1, cfg.gnn_u_dims[l][i]);
              din = cfg.gnn_u_dims[l][i];
            }
          }
        }
        dcur = d;
      }
      int din = d;
      for (int i = 0; i < cfg.jastrow_n; ++i) {
        add("J" + std::to_string(i) + ".w", din, cfg.jastrow_dims[i]);
        if (i < cfg.jastrow_n - 1) add("J" + std::to_string(i) + ".b", 1, cfg.jastrow_dims[i]);
        din = cfg.jastrow_dims[i];
      }
      din = d;
      for (int i = 0; i < cfg.backflow_n; ++i) {
        const std::string q = std::to_string(i);
        add("bfh" + q + ".up", din, cfg.backflow_dims[i]); add("bfh" + q + ".dn", din, cfg.backflow_dims[i]);
        add("bfb" + q + ".up", 1, cfg.backflow_dims[i]); add("bfb" + q + ".dn", 1, cfg.backflow_dims[i]);
        din = cfg.backflow_dims[i];
      }
      bf_in = din;
      add("bfb.up", 1, K * N); add("bfb.dn", 1, K * N);
      if (cfg.conf_linear) add("conf.w", 1, K);
    }
    if (cfg.kind == DQMC_FERMINET) {
      const int de = cfg.edge_dim;
      int din = 4 * M, ein = 4;
      for (int l = 0; l < cfg.n_layers; ++l) {
        std::string p = "F" + std::to_string(l) + ".";
        add(p + "wg", 3 * din + 2 * ein, d);
        add(p + "bg", 1, d);
        if (l < cfg.n_layers - 1) {
          add(p + "wu", ein, de);
          add(p + "bu", 1, de);
        }
        din = d; ein = de;
      }
    }
    add("bf.up", bf_in, K * N * (cfg.backflow_add == 2 ? 2 : 1));
    add("bf.dn", bf_in, K * N * (cfg.backflow_add == 2 ? 2 : 1));
    add("env.pi_up", K * N, M * rep);
    add("env.pi_dn", K * N, M * rep);
    add("env.zeta_up", K * N, M * rep);
    add("env.zeta_dn", K * N, M * rep);
    add("cusp.alpha", 1, 2);
    if (cfg.nuc_cusp_kind) add("cusp.nuc", 1, 1 + M);  // alpha_nuc, nuclear charges
  }
  int64_t off(const std::string& n) const {
    for (auto& e : entries)
      if (e.name == n) return e.offset;
    return -1;
  }
};

// Bump allocator over a caller's workspace: every buffer of every entry point is carved through one.  Buffers are 256-byte
// aligned; emulator builds (tools/cuda_emu) put a 256-byte guard zone behind each one, verified after each chunk
// (Engine::check_guards), so a buffer that is individually too small (with a consistent total) cannot hide.  The guard bytes
// are part of what take() advances by, so the PLAN (a dry pass of the same code) contains them too: emulator and hardware
// builds plan by the same rule, there is no build-dependent slack.
struct Arena {
  const EngineBase* e;
  char* base;
  char* top;    // next free byte
  int64_t cap;  // bytes of the workspace behind base
  Arena(const EngineBase* e_, void* base_, int64_t cap_ = INT64_MAX) : e(e_), base((char*)base_), top((char*)base_), cap(cap_) {}
  template <class U>
  U* take(size_t n) {
    U* q = (U*)top;
    top += align_up(sizeof(U) * n);
#ifdef DQMC_EMU
    if (!e->dry) { std::memset(top, 0xC3, 256); e->emu_guards.push_back((unsigned char*)top); }
    top += 256;
#endif
    e->note_hwm(top);
    return q;
  }
  int64_t left() const { return cap - (top - base); }  // < 0: the buffers taken exceed the workspace
};

// Size probes and dqmc_debug_plan walk the carving code on a dummy base with every CUDA call skipped (EngineBase::dry); the
// scope restores the caller's dry state and high-water mark, so probes nest inside a planning pass.
static char* plan_base() { return (char*)(uintptr_t)0x100000; }
struct DryPass {
  EngineBase* e;
  bool was;
  const char* hw;
  explicit DryPass(const EngineBase* e_) : e(const_cast<EngineBase*>(e_)), was(e->dry), hw(e->dry_hwm) {
    e->dry = true;  // no guard writes through the dummy base
    e->dry_hwm = plan_base();
  }
  ~DryPass() { e->dry = was; e->dry_hwm = hw; }
  int64_t bytes() const { return e->dry_hwm - plan_base(); }  // highest offset carved so far
};

// largest n in [1, hi] with bytes(n) <= wsb (bytes monotone in n), 0 if there is none
template <class F>
static int64_t largest_fit(int64_t hi, int64_t wsb, F bytes) {
  if (hi < 1 || bytes(1) > wsb) return 0;
  if (bytes(hi) <= wsb) return hi;
  int64_t lo = 1;
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) / 2;
    (bytes(mid) <= wsb ? lo : hi) = mid;
  }
  return lo;
}

static constexpr int64_t kRowCap = 2000000000;  // elements per chunk buffer: keeps 32-bit row * ld products safe

template <class T>
__global__ void convert_kernel(const double* __restrict__ src, T* __restrict__ dst, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = (T)src[i];
}

// W[K][N] (row-major) -> W^T hi/lo [N][K]: hi = rna_tf32(w), lo = rna_tf32(w - hi)
__global__ void split_transpose_kernel(const float* __restrict__ W, int K, int N, float* __restrict__ hi,
                                       float* __restrict__ lo) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= K * N) return;
  int n = idx / K, k = idx % K;
  float w = W[(size_t)k * N + n];
#if !defined(DQMC_NO_TCGEN05)
  float h = tc::tf32_rna(w);
  hi[idx] = h;
  lo[idx] = tc::tf32_rna(w - h);
#else
  float h = __uint_as_float(__float_as_uint(w) & 0xFFFFE000u);
  hi[idx] = h;
  lo[idx] = w - h;
#endif
}

#if !defined(DQMC_NO_TCGEN05)
// W[K][N] (row-major) -> (W 2^e)^T as IEEE halves, hi / lo planes [N][K]: hi = rn(w'), lo = rn(w' - hi)
__global__ void split_transpose_f16_kernel(const float* __restrict__ W, int K, int N, float scale, uint16_t* __restrict__ hi,
                                           uint16_t* __restrict__ lo) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= K * N) return;
  int n = idx / K, k = idx % K;
  const float w = W[(size_t)k * N + n] * scale;
  const uint32_t h = tc::pack_half2_rn(w, 0.f) & 0xFFFFu;
  const uint32_t l = tc::pack_half2_rn(w - tc::half_bits_to_float(h), 0.f) & 0xFFFFu;
  hi[idx] = (uint16_t)h;
  lo[idx] = (uint16_t)l;
}
#endif

#define DQ_CHECK(call)                                                             \
  do {                                                                             \
    if (dry) break; /* planning pass: no CUDA calls */                             \
    cudaError_t e_ = (call);                                                       \
    if (e_ != cudaSuccess) {                                                       \
      err = std::string(#call) + ": " + cudaGetErrorString(e_);                    \
      return 1;                                                                    \
    }                                                                              \
  } while (0)

// cudaFuncAttributeMaxDynamicSharedMemorySize belongs to the kernel, not to an engine, and engines for molecules of different
// size share one process: the opt-in therefore only ever grows (a later, smaller engine must not lower the cap under an
// earlier, larger one).
template <class F>
inline cudaError_t raise_dyn_smem(F fn, int bytes) {
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, int> high;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lock(mu);
  int& h = high[std::make_pair(dev, (const void*)fn)];
  if (bytes > h) h = bytes;
  return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, h);
}

#define DQ_LAUNCH(kern, grid, block, smem, stream, ...)          \
  do {                                                           \
    if (dry) break; /* planning pass */                          \
    auto kfn_ = kern;                                            \
    DQMC_LAUNCH(kfn_, grid, block, smem, stream, __VA_ARGS__);   \
    ++launches;                                                  \
  } while (0)

template <class T>
struct Engine : EngineBase {
  T* d_params = nullptr;
  T* d_params_t = nullptr;  // every entry transposed ([cols][rows]): operands of the dA = dY W^T products of the reverse pass
  double* d_stage = nullptr;
  T* d_zval = nullptr;
  T* d_znuc = nullptr;  // full nuclear charges (Langevin clean_force)
  int* d_ecp_mask = nullptr;
  T* d_ecp_loc = nullptr;
  T* d_nl_params = nullptr;
  int* d_nl_nuc = nullptr;
  double* d_nl_rc2 = nullptr;  // [J] squared cutoff radius of each non-local nucleus slot (ecp_cutoff_rc2)
  double* d_nl_rc2f = nullptr;  // [J] ... of the non-local force (ecp_force_cutoff_rc2)
  int J = 0;  // nuclei with a non-local channel
  // pseudo-Hamiltonian (reference ecp/pseudo_hamiltonian.py): tables r V_loc / r V_L2 per element on a uniform grid
  T* d_ph_tabs = nullptr;
  int* d_ph_nuc = nullptr;
  int ph_G = 0;
  double ph_rmax = 0;
  int check_guards() {
#ifdef DQMC_EMU
    for (unsigned char* g : emu_guards)
      for (int i = 0; i < 256; ++i)
        if (g[i] != 0xC3) { emu_guards.clear(); err = "emulator: a workspace buffer was overrun (guard zone modified)"; return 4; }
    emu_guards.clear();
#endif
    return 0;
  }
  bool ph_on = false;      // tables uploaded
  int attn_tb = 1, attn_tb1 = 1;
  bool attn_gen_mma = false;  // ... same for the generic kernel (TransPsiformer: extra key / value tokens)
  bool attn_fl_mma = false;   // fp32 forward-Laplacian attention: tangent chunks as warp-level 3xTF32 mma.sync products
  int attn_fl_threads = 128;  // block size of the fp32 forward-Laplacian attention (large molecules: one block per SM fits -> more warps)
  bool attn_f32 = false;
  bool embed_fwd_ok = false;
  bool attn_mma_ok = false;  // plain-forward attention on mma.sync (attn_mma.cuh)
  bool slater_fwd2_ok = false;
  int N, M, d, K, KN, H, dh, T3;
  int BFW = 0;      // row width of the backflow buffer: K N, or 2 K N with multiplicative + additive heads
  int add_off = 0;  // column offset of the additive head in it
  bool gnn = false;    // conv-GNN ("PauliNet" test ansatz)
  int bf_in = 0;       // input width of the final backflow layer
  bool trans = false;  // TransPsiformer: nuclear attention tokens + nucleus-dependent envelopes
  int Mn = 0, env_rep = 1;
  size_t max_smem = 0;
  int n_sms = 132;
  Switches sw;  // read_switches() at the start of init()
  // What a plain forward (run_batched) takes besides positions and outputs; the default value is an ordinary forward.
  struct FwdIn {
    // compact virtual-walker group (non-local ECP quadrature or spin swaps, virtual_groups): envelope table of its base
    // walkers [nb][N][K N], their embedding rows [nb][N][d] (whole-trunk kernel only), the ECP group's active-pair list
    // (ecp_pairs_kernel), virtual walkers per base walker (J N 12, or the swapped pairs) and the layout of virtual_move
    // (common.cuh)
    const T* env = nullptr;
    const T* emb = nullptr;
    const int* pairs = nullptr;
    int vper = 0;
    int layout = kVirtEcp;
    T* mos = nullptr;  // orbitals(): the tail writes the orbital matrices [B][K][N][N] here and stops
    bool ph = false;   // the pseudo-Hamiltonian metric applies to the forward-Laplacian pass (needs ph_on)
  };
#if !defined(DQMC_NO_TCGEN05)
  struct TcWeight {
    float* hi = nullptr; float* lo = nullptr; CUtensorMap mh, ml; int N = 0, K = 0;
    // "3xFP16" operands of the plain-forward kernels: (W 2^e)^T as halves, hi / lo planes [N][K]; maps with BN-row boxes
    // (row GEMM) and with all-N-row boxes of 32 halves (64-byte swizzle: the per-warpgroup weight slots of the fused MLP
    // block, N <= 256, fused_tc.cuh)
    uint16_t* h16 = nullptr; CUtensorMap m16h, m16l, m16h_all, m16l_all; float wscale = 1.f; bool f16 = false, f16_all = false;
    CUtensorMap m16h_256, m16l_256; bool f16_256 = false;  // 256-row boxes of 32 halves: weight slots of the whole-trunk kernel (trunk_tc.cuh)
  };
  CUtensorMap* d_trunk_maps = nullptr;       // [L][4][2]
  unsigned char* d_trunk_scratch = nullptr;  // n_sms x 384 KB: split K / V and residual rows of a tile
  int* d_tc_err = nullptr;                     // error word of the whole-trunk and MLP-block kernels (tc::lock_take past its bound)
  unsigned long long* d_trunk_phase = nullptr;  // DQMC_TRUNK_PHASES=1: the whole-trunk kernel's phase timers (tc::kPhases)
  static constexpr float kActScale = 16.f;  // 2^4: |activation| < 4094 representable, absolute floor 2^-29
  std::map<std::string, TcWeight> tcw;
  bool use_tc() const { return std::is_same<T, float>::value && cfg.gemm_backend == DQMC_GEMM_TCGEN05; }
  int prepare_tc_weight(const std::string& name, const float* W, int Kc, int Nc, cudaStream_t st, double wmax) {
    TcWeight& w = tcw[name];
    if (!w.hi) {
      DQ_CHECK(cudaMalloc((void**)&w.hi, sizeof(float) * (size_t)Kc * Nc));
      DQ_CHECK(cudaMalloc((void**)&w.lo, sizeof(float) * (size_t)Kc * Nc));
      w.N = Nc; w.K = Kc;
      if (tc::make_weight_map(&w.mh, w.hi, Nc, Kc, tc::kBN) || tc::make_weight_map(&w.ml, w.lo, Nc, Kc, tc::kBN)) {
        err = "cuTensorMapEncodeTiled failed for " + name;
        return 4;
      }
      if (Kc % 64 == 0) {
        DQ_CHECK(cudaMalloc((void**)&w.h16, sizeof(uint16_t) * 2 * (size_t)Kc * Nc));
        const uint16_t* lo16 = w.h16 + (size_t)Kc * Nc;
        if (tc::make_kmajor_map(&w.m16h, w.h16, 2, Nc, Kc, 64, tc::kBN) || tc::make_kmajor_map(&w.m16l, lo16, 2, Nc, Kc, 64, tc::kBN)) {
          err = "cuTensorMapEncodeTiled (half planes) failed for " + name;
          return 4;
        }
        w.f16 = true;
        if (Nc <= 256 && Nc % 16 == 0) {
          if (tc::make_kmajor_map(&w.m16h_all, w.h16, 2, Nc, Kc, 32, Nc) || tc::make_kmajor_map(&w.m16l_all, lo16, 2, Nc, Kc, 32, Nc)) {
            err = "cuTensorMapEncodeTiled (whole-N half planes) failed for " + name;
            return 4;
          }
          w.f16_all = true;
        }
        if (Kc == 256 && Nc % 256 == 0 &&
            !tc::make_kmajor_map(&w.m16h_256, w.h16, 2, Nc, Kc, 32, 256) && !tc::make_kmajor_map(&w.m16l_256, lo16, 2, Nc, Kc, 32, 256))
          w.f16_256 = true;
      }
    }
    DQ_LAUNCH(split_transpose_kernel, dim3((Kc * Nc + 255) / 256), dim3(256), 0, st, W, Kc, Nc, w.hi, w.lo);
    if (w.f16) {
      // power-of-two weight scale: the largest |w| of the matrix (of the spin pair for the per-spin heads) lands in [512, 1024)
      int e = 0;
      if (wmax > 0) { std::frexp(wmax, &e); e = 10 - e; }
      e = e > 24 ? 24 : (e < -24 ? -24 : e);
      w.wscale = std::ldexp(1.f, e);
      DQ_LAUNCH(split_transpose_f16_kernel, dim3((Kc * Nc + 255) / 256), dim3(256), 0, st, W, Kc, Nc, w.wscale, w.h16,
                w.h16 + (size_t)Kc * Nc);
    }
    return 0;
  }
#else
  bool use_tc() const { return false; }
#endif

  int init() {
    sw = read_switches();
    N = cfg.n_up + cfg.n_down; M = cfg.n_nuc; d = cfg.embedding_dim; K = cfg.n_determinants;
    KN = K * N; H = cfg.n_heads; dh = d / H; T3 = 3 * N;
    BFW = KN * (cfg.backflow_add == 2 ? 2 : 1);
    add_off = cfg.backflow_add == 2 ? KN : 0;
    if (cfg.backflow_add && cfg.kind == DQMC_PAULINET) { err = "additive backflow: linear-head ansatz kinds only"; return 2; }
    if (cfg.kind != DQMC_PSIFORMER && cfg.kind != DQMC_FERMINET && cfg.kind != DQMC_TRANSPSIFORMER &&
        cfg.kind != DQMC_PAULINET) {
      err = "unknown ansatz kind"; return 2;
    }
    trans = cfg.kind == DQMC_TRANSPSIFORMER;
    Mn = trans ? cfg.n_nuc_tokens : 0;
    env_rep = cfg.n_env_per_nuc > 1 ? cfg.n_env_per_nuc : 1;
    if (M * env_rep > 4 * DQMC_MAX_NUC || Mn < 0 || Mn > DQMC_MAX_NUC) { err = "bad config (envelope terms / nuclear tokens)"; return 2; }
    if (H < 1) H = 1;
    if (cfg.kind == DQMC_FERMINET || cfg.kind == DQMC_PAULINET) { H = 1; dh = d; }
    gnn = cfg.kind == DQMC_PAULINET;
    if (gnn && (cfg.jastrow_n > 8 || cfg.backflow_n > 8 || cfg.jastrow_n < 0 || cfg.backflow_n < 0)) { err = "bad MLP depth"; return 2; }
    for (int t = 0; t < 3; ++t)
      if (cfg.gnn_edge_in[t] != 0 && cfg.gnn_edge_in[t] != 1 && cfg.gnn_edge_in[t] != 4) { err = "bad edge feature width"; return 2; }
    if (gnn && ((cfg.gnn_ne_identity && (!cfg.gnn_concat || !cfg.gnn_conv_ne || cfg.edge_dim < 4)) ||
                (cfg.gnn_no_res && !cfg.gnn_concat) || (cfg.gnn_sep_edges && !cfg.gnn_deep_edges) ||
                (cfg.gnn_sub_n > 1 && (cfg.gnn_edge_in[0] || cfg.gnn_edge_in[1] || cfg.gnn_edge_in[2])))) {
      err = "bad conv-GNN config (identity ne filter / no residual need the concatenate update with ne edges, separate u "
            "needs deep edges, per-type edge widths need one-layer w / u MLPs)";
      return 2;
    }
    bf_in = d;
    if (gnn && cfg.backflow_n > 0) bf_in = cfg.backflow_dims[cfg.backflow_n - 1];
    if (M > DQMC_MAX_NUC || d % H != 0 || N < 2) { err = "bad config"; return 2; }
    build_layout();
    DQ_CHECK(cudaSetDevice(device));
    DQ_CHECK(cudaMalloc((void**)&d_params, sizeof(T) * total));
    DQ_CHECK(cudaMalloc((void**)&d_params_t, sizeof(T) * total));
    DQ_CHECK(cudaMalloc((void**)&d_stage, sizeof(double) * total));
    std::vector<T> z(M);
    for (int m = 0; m < M; ++m) z[m] = (T)cfg.z_valence[m];
    DQ_CHECK(cudaMalloc((void**)&d_zval, sizeof(T) * M));
    DQ_CHECK(cudaMemcpy(d_zval, z.data(), sizeof(T) * M, cudaMemcpyHostToDevice));
    {
      std::vector<T> zn(M);
      for (int m = 0; m < M; ++m) zn[m] = (T)cfg.z_nuclear[m];
      DQ_CHECK(cudaMalloc((void**)&d_znuc, sizeof(T) * M));
      DQ_CHECK(cudaMemcpy(d_znuc, zn.data(), sizeof(T) * M, cudaMemcpyHostToDevice));
    }
    DQ_CHECK(cudaMalloc((void**)&d_ecp_mask, sizeof(int) * M));
    DQ_CHECK(cudaMemcpy(d_ecp_mask, cfg.ecp_mask, sizeof(int) * M, cudaMemcpyHostToDevice));
    const int Tm = cfg.ecp_loc_terms;
    if (Tm > 0) {
      std::vector<T> lp((size_t)M * 6 * Tm);
      for (int m = 0; m < M; ++m)
        for (int n = 0; n < 3; ++n)
          for (int ab = 0; ab < 2; ++ab)
            for (int t = 0; t < Tm; ++t) lp[(((size_t)m * 3 + n) * 2 + ab) * Tm + t] = (T)cfg.ecp_loc[m][n][ab][t];
      DQ_CHECK(cudaMalloc((void**)&d_ecp_loc, sizeof(T) * lp.size()));
      DQ_CHECK(cudaMemcpy(d_ecp_loc, lp.data(), sizeof(T) * lp.size(), cudaMemcpyHostToDevice));
    }
    const int L = cfg.ecp_nl_lmax_p1, Tn = cfg.ecp_nl_terms;
    if (L > 0 && Tn > 0) {
      std::vector<T> np((size_t)M * L * 2 * Tn);
      std::vector<int> nuc;
      for (int m = 0; m < M; ++m) {
        bool any = false;
        for (int l = 0; l < L; ++l)
          for (int ab = 0; ab < 2; ++ab)
            for (int t = 0; t < Tn; ++t) {
              double v = cfg.ecp_nl[m][l][ab][t];
              np[(((size_t)m * L + l) * 2 + ab) * Tn + t] = (T)v;
              any = any || v != 0.0;
            }
        if (any) nuc.push_back(m);  // nuc_with_nl_pot, gaussian_type_ecp.py:120
      }
      J = (int)nuc.size();
      if (J > 0) {
        DQ_CHECK(cudaMalloc((void**)&d_nl_params, sizeof(T) * np.size()));
        DQ_CHECK(cudaMemcpy(d_nl_params, np.data(), sizeof(T) * np.size(), cudaMemcpyHostToDevice));
        DQ_CHECK(cudaMalloc((void**)&d_nl_nuc, sizeof(int) * J));
        DQ_CHECK(cudaMemcpy(d_nl_nuc, nuc.data(), sizeof(int) * J, cudaMemcpyHostToDevice));
        std::vector<double> rc2(J), rc2f(J);
        for (int j = 0; j < J; ++j) {
          rc2[j] = ecp_cutoff_rc2(np.data() + (size_t)nuc[j] * L * 2 * Tn, L, Tn, sw.ecp_cutoff);
          rc2f[j] = ecp_force_cutoff_rc2(np.data() + (size_t)nuc[j] * L * 2 * Tn, L, Tn, sw.ecp_cutoff);
        }
        DQ_CHECK(cudaMalloc((void**)&d_nl_rc2, sizeof(double) * J));
        DQ_CHECK(cudaMemcpy(d_nl_rc2, rc2.data(), sizeof(double) * J, cudaMemcpyHostToDevice));
        DQ_CHECK(cudaMalloc((void**)&d_nl_rc2f, sizeof(double) * J));
        DQ_CHECK(cudaMemcpy(d_nl_rc2f, rc2f.data(), sizeof(double) * J, cudaMemcpyHostToDevice));
      }
    }
#ifndef DQMC_EMU
    {
      int v = 0;
      DQ_CHECK(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, device));
      if (v > 0) n_sms = v;
    }
#endif
    if (sw.nsms >= 1) n_sms = sw.nsms;
    // opt in to large dynamic shared memory
    const bool psif = cfg.kind == DQMC_PSIFORMER || trans;
    // the specialised fp32 attention kernels do not take extra tokens yet: TransPsiformer runs the generic one
    attn_f32 = psif && !trans && std::is_same<T, float>::value && dh % 16 == 0 && !sw.attn_generic;
    // forward-Laplacian tangent slots per chunk: DQMC_ATTN_TB if it is in 1 .. 3N; fp32: ~7 blocks/SM for small molecules
    if (sw.attn_tb && *sw.attn_tb >= 1 && *sw.attn_tb <= T3) attn_tb = *sw.attn_tb;
    else attn_tb = attn_f32 ? attn_f32_pick_tb(N, dh, T3, 32 * 1024) : attn_pick_tb<T>(N, dh, T3, 100 * 1024, Mn);
    size_t s_attn = !psif ? 0 : attn_f32 ? attn_f32_smem_bytes(N, dh, attn_tb) : attn_smem_bytes<T>(N, dh, attn_tb, Mn);
    // few resident blocks per SM (large molecules: the tangent chunk fills the shared memory) -> more warps per block
    // (benzene, one 170 KB block per SM: 128 threads 707 ms per 512-walker step, 512 threads 684 ms)
    if (!sw.attn_nt) attn_fl_threads = s_attn > 110 * 1024 ? 512 : (s_attn > 56 * 1024 ? 256 : 128);
    else if (*sw.attn_nt >= 32 && *sw.attn_nt <= 1024 && *sw.attn_nt % 32 == 0) attn_fl_threads = *sw.attn_nt;
    // 16 x 8 tiles: worthwhile from about 20 electrons (benzene, N = 30: 686 -> 648 ms per 512-walker step; LiH, N = 4, where
    // 7/8 of every tile is padding: 6.9 -> 15.7 ms, so small molecules keep the SIMT variant)
    attn_fl_mma = attn_f32 && N <= 32 && dh % 16 == 0 && sw.attn_fl_mma.value_or(N >= 20);
    if (attn_fl_mma && !sw.attn_tb) {  // two resident blocks of 8 warps per SM
      attn_tb = attn_f32_pick_tb(N, dh, T3, 110 * 1024);
      s_attn = attn_f32_smem_bytes(N, dh, attn_tb);
    }
    // generic kernel (extra key / value tokens: TransPsiformer) in fp32: same tensor-core products, row pitch dh + 4
    attn_gen_mma = psif && !attn_f32 && std::is_same<T, float>::value && dh % 16 == 0 &&
                   sw.attn_fl_mma.value_or(N >= 20 && !sw.attn_generic);
    if (attn_gen_mma) {
      if (!sw.attn_tb) attn_tb = attn_pick_tb<T>(N, dh, T3, 110 * 1024, Mn, 4);
      s_attn = attn_smem_bytes<T>(N, dh, attn_tb, Mn, 4);
    }
    size_t s_sl = slater_smem_bytes<T>(N);
    max_smem = s_attn > s_sl ? s_attn : s_sl;
    if (max_smem > 227 * 1024) { err = "system too large for the shared-memory tiling (N)"; return 2; }
    if (attn_f32) {
      if (launch_attn_f32(nullptr, nullptr, 0, 0, 0, 0.f, 0, (int)s_attn, nullptr, true)) return 1;
    } else if (psif) {
      DQ_CHECK(raise_dyn_smem(attn_fl_kernel<T>, (int)s_attn));
      if constexpr (std::is_same<T, float>::value) DQ_CHECK(raise_dyn_smem((attn_fl_kernel<T, true>), (int)s_attn));
    }
    DQ_CHECK(raise_dyn_smem(slater_kernel<T>, (int)s_sl));
    slater_fwd2_ok = N <= 32 && slater_fwd2_smem_bytes<T>(N, M, K) <= 110 * 1024 && !sw.slater_generic && !sw.slater_fwd1;
    if (slater_fwd2_ok) {
      DQ_CHECK(raise_dyn_smem(slater_fwd2_kernel<T, 14>, (int)slater_fwd2_smem_bytes<T>(N, M, K)));
      DQ_CHECK(raise_dyn_smem(slater_fwd2_kernel<T, 16>, (int)slater_fwd2_smem_bytes<T>(N, M, K)));
      DQ_CHECK(raise_dyn_smem(slater_fwd2_kernel<T, 28>, (int)slater_fwd2_smem_bytes<T>(N, M, K)));
      DQ_CHECK(raise_dyn_smem(slater_fwd2_kernel<T, 30>, (int)slater_fwd2_smem_bytes<T>(N, M, K)));
      DQ_CHECK(raise_dyn_smem(slater_fwd2_kernel<T, 32>, (int)slater_fwd2_smem_bytes<T>(N, M, K)));
    }
    attn_mma_ok = psif && std::is_same<T, float>::value && dh == 64 && N + Mn <= 48 && d % 4 == 0 && !sw.attn_generic;
    embed_fwd_ok = psif && d % 4 == 0 && embed_fwd_smem_bytes<T>(M, d) <= 200 * 1024;
    if (embed_fwd_ok)
      DQ_CHECK(raise_dyn_smem(embed_fwd_kernel<T>, (int)embed_fwd_smem_bytes<T>(M, d)));
    if (cfg.gemm_backend == DQMC_GEMM_TCGEN05) {
#if !defined(DQMC_NO_TCGEN05)
      if (!std::is_same<T, float>::value) { err = "DQMC_GEMM_TCGEN05 needs dtype DQMC_F32"; return 2; }
      if (d % 32 != 0) { err = "DQMC_GEMM_TCGEN05 needs embedding_dim % 32 == 0"; return 2; }
      DQ_CHECK(raise_dyn_smem(tc::gemm3x_kernel<false>, tc::SmemLayout::total()));
      DQ_CHECK(raise_dyn_smem(tc::gemm3x_kernel<true>, tc::SmemLayout::total()));
      DQ_CHECK(raise_dyn_smem(tc::mlp_block_f16_kernel<128>, tc::MlpSmem::total()));
      DQ_CHECK(raise_dyn_smem(tc::mlp_block_f16_kernel<256>, tc::MlpSmem::total()));
      DQ_CHECK(raise_dyn_smem(tc::trunk_f16_kernel<1>, tc::TrSmem::total()));
      DQ_CHECK(raise_dyn_smem(tc::trunk_f16_kernel<2>, tc::TrSmem::total()));
      DQ_CHECK(raise_dyn_smem(tc::trunk_f16_kernel<4>, tc::TrSmem::total()));
      DQ_CHECK(raise_dyn_smem(tc::trunk_f16_kernel<8>, tc::TrSmem::total()));
      DQ_CHECK(raise_dyn_smem(tc::trunk_f16_kernel<16>, tc::TrSmem::total()));
      DQ_CHECK(raise_dyn_smem(tc::trunk_f16_kernel<32>, tc::TrSmem::total()));
      DQ_CHECK(cudaMalloc((void**)&d_tc_err, sizeof(int)));
      DQ_CHECK(cudaMemset(d_tc_err, 0, sizeof(int)));
      if (psif && !trans && d == 256 && H == 4 && N <= 32 && cfg.n_layers <= tc::kTrMaxLayers) {
        DQ_CHECK(cudaMalloc((void**)&d_trunk_maps, sizeof(CUtensorMap) * 8 * cfg.n_layers));
        DQ_CHECK(cudaMalloc((void**)&d_trunk_scratch, (size_t)n_sms * tc::kTrScratchPerCta));
        if (sw.trunk_phases) {
          DQ_CHECK(cudaMalloc((void**)&d_trunk_phase, sizeof(unsigned long long) * tc::kPhases));
          DQ_CHECK(cudaMemset(d_trunk_phase, 0, sizeof(unsigned long long) * tc::kPhases));
        }
      }
#else
      err = "this build has no tensor-core backend"; return 2;
#endif
    }
    return 0;
  }
  ~Engine() override {
    if (plan_only) return;  // nothing was allocated, no CUDA context
    cudaFree(d_params); cudaFree(d_params_t); cudaFree(d_stage); cudaFree(d_znuc); cudaFree(d_zval); cudaFree(d_ecp_mask);
    if (d_ecp_loc) cudaFree(d_ecp_loc);
    if (d_nl_params) cudaFree(d_nl_params);
    if (d_nl_nuc) cudaFree(d_nl_nuc);
    if (d_nl_rc2) cudaFree(d_nl_rc2);
    if (d_nl_rc2f) cudaFree(d_nl_rc2f);
    if (d_ph_tabs) cudaFree(d_ph_tabs);
    if (d_ph_nuc) cudaFree(d_ph_nuc);
#if !defined(DQMC_NO_TCGEN05)
    for (auto& kv : tcw) {
      if (kv.second.hi) cudaFree(kv.second.hi);
      if (kv.second.lo) cudaFree(kv.second.lo);
      if (kv.second.h16) cudaFree(kv.second.h16);
    }
    if (d_trunk_maps) cudaFree(d_trunk_maps);
    if (d_trunk_scratch) cudaFree(d_trunk_scratch);
    if (d_trunk_phase) cudaFree(d_trunk_phase);
    if (d_tc_err) cudaFree(d_tc_err);
#endif
  }
  const T* P(const std::string& n) const { return d_params + off(n); }

  int set_ph(int n_tab, int n_grid, double r_max, const double* tables, const int32_t* tab_of_nuc) override {
    if (J > 0 || cfg.ecp_loc_terms > 0) { err = "pseudo-Hamiltonian and Gaussian-type ECP are mutually exclusive"; return 2; }
    if (n_tab < 1 || n_grid < 2 || !(r_max > 0) || !tables || !tab_of_nuc) { err = "bad pseudo-Hamiltonian tables"; return 2; }
    for (int m = 0; m < M; ++m)
      if (tab_of_nuc[m] >= n_tab) { err = "pseudo-Hamiltonian table index out of range"; return 2; }
    std::vector<T> h((size_t)n_tab * 2 * n_grid);
    for (size_t i = 0; i < h.size(); ++i) h[i] = (T)tables[i];
    if (d_ph_tabs) cudaFree(d_ph_tabs);
    if (d_ph_nuc) cudaFree(d_ph_nuc);
    DQ_CHECK(cudaMalloc((void**)&d_ph_tabs, sizeof(T) * h.size()));
    DQ_CHECK(cudaMemcpy(d_ph_tabs, h.data(), sizeof(T) * h.size(), cudaMemcpyHostToDevice));
    DQ_CHECK(cudaMalloc((void**)&d_ph_nuc, sizeof(int) * M));
    DQ_CHECK(cudaMemcpy(d_ph_nuc, tab_of_nuc, sizeof(int) * M, cudaMemcpyHostToDevice));
    ph_G = n_grid; ph_rmax = r_max; ph_on = true;
    return 0;
  }
  PhArgs<T> ph_args(const T* QA) const {
    PhArgs<T> a;
    a.QA = QA; a.tabs = d_ph_tabs; a.tab_of_nuc = d_ph_nuc; a.G = ph_G; a.rmax = (T)ph_rmax;
    return a;
  }

  int set_params(const double* host, int64_t n, cudaStream_t st) override {
    if (n != total) { err = "parameter count mismatch"; return 2; }
    DQ_CHECK(cudaMemcpyAsync(d_stage, host, sizeof(double) * n, cudaMemcpyHostToDevice, st));
    DQ_LAUNCH(convert_kernel<T>, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, (const double*)d_stage, d_params, n);
    for (auto& e : entries)  // (vectors included: a [n][1] weight such as the Jastrow's last layer is its own transpose)
      if (e.rows >= 1 && e.cols >= 1)
        DQ_LAUNCH(transpose_kernel<T>, dim3((e.rows * e.cols + 255) / 256), dim3(256), 0, st, (const T*)(d_params + e.offset),
                  e.rows, e.cols, d_params_t + e.offset);
#if !defined(DQMC_NO_TCGEN05)
    if (use_tc()) {
      // largest |w| per matrix (the two spin heads of a per-spin layer share one scale: they are used in one launch)
      std::map<std::string, double> wmax;
      auto group = [](const std::string& n) {
        const size_t k = n.size();
        return (k > 3 && (n.compare(k - 3, 3, ".up") == 0 || n.compare(k - 3, 3, ".dn") == 0)) ? n.substr(0, k - 3) : n;
      };
      for (auto& e : entries) {
        double m = 0;
        for (int64_t i = 0; i < (int64_t)e.rows * e.cols; ++i) m = std::max(m, std::fabs(host[e.offset + i]));
        double& g = wmax[group(e.name)];
        g = std::max(g, m);
      }
      for (auto& e : entries) {
        bool is_w = e.name.find(".w") != std::string::npos || e.name.rfind("bf.", 0) == 0;
        if (!is_w || e.name == "emb.w" || e.rows % 32 != 0 || e.cols < 64) continue;
        int rc = prepare_tc_weight(e.name, (const float*)(d_params + e.offset), e.rows, e.cols, st, wmax[group(e.name)]);
        if (rc) return rc;
      }
      if (d_trunk_maps && trunk_weights_ok()) {
        std::vector<CUtensorMap> hm((size_t)8 * cfg.n_layers);
        for (int l = 0; l < cfg.n_layers; ++l) {
          const std::string pfx = "L" + std::to_string(l) + ".";
          int g = 0;
          for (const char* n : {"wqkv", "wo", "w1", "w2"}) {
            const TcWeight& w = tcw.at(pfx + n);
            hm[(size_t)8 * l + 2 * g] = w.m16h_256;
            hm[(size_t)8 * l + 2 * g + 1] = w.m16l_256;
            ++g;
          }
        }
        DQ_CHECK(cudaMemcpy(d_trunk_maps, hm.data(), sizeof(CUtensorMap) * hm.size(), cudaMemcpyHostToDevice));
      }
    }
#endif
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  // ---- workspace ---------------------------------------------------------------------------
  struct Ws {
    T *X, *O, *A, *M1, *QKV, *BF, *dsign, *dlog, *dlap, *dgrad;
    T* QA = nullptr;  // pseudo-Hamiltonian records [Bc][N][PH_STRIDE]
    T* Gadd = nullptr;  // additive-backflow factor g_i = cutoff * envelope norm with gradient / Laplacian [Bc][N][5]
    T *G0 = nullptr, *G1 = nullptr, *G2 = nullptr, *Hs = nullptr, *Ha = nullptr, *C = nullptr, *Fc = nullptr, *HT = nullptr,
      *E0 = nullptr, *E1 = nullptr, *ET0 = nullptr, *ET1 = nullptr, *W3 = nullptr,
      *Y0 = nullptr, *Y1 = nullptr, *Jb = nullptr;  // conv-GNN trunk
  };
  int gnn_hmax() const {
    int h = 1;
    for (int i = 0; i < cfg.backflow_n; ++i) h = cfg.backflow_dims[i] > h ? cfg.backflow_dims[i] : h;
    return h;
  }
  size_t fermi_dmax() const { return (size_t)(4 * M > d ? 4 * M : d); }
  size_t fermi_emax() const { return (size_t)(cfg.edge_dim > 4 ? cfg.edge_dim : 4); }
  int gnn_dmax() const { return cfg.gnn_features && 4 * M > d ? 4 * M : d; }
  int gnn_emax() const {  // widest edge-side row (raw features, w / u hidden and output widths)
    int m = cfg.edge_dim > 4 ? cfg.edge_dim : 4;
    for (int l = 0; l < cfg.n_layers && l < 8; ++l)
      for (int i = 0; i < cfg.gnn_sub_n && i < 4; ++i) {
        m = cfg.gnn_w_dims[l][i] > m ? cfg.gnn_w_dims[l][i] : m;
        m = cfg.gnn_u_dims[l][i] > m ? cfg.gnn_u_dims[l][i] : m;
      }
    return m;
  }
  int gnn_hnode_max() const {
    int m = cfg.edge_dim;
    for (int l = 0; l < cfg.n_layers && l < 8; ++l)
      for (int i = 0; i < cfg.gnn_sub_n && i < 4; ++i) m = cfg.gnn_h_dims[l][i] > m ? cfg.gnn_h_dims[l][i] : m;
    return m;
  }
  int gnn_jsum() const {
    int j = d;
    for (int i = 0; i < cfg.jastrow_n; ++i) j += cfg.jastrow_dims[i];
    return j;
  }
  // Workspace plan == the carve itself: every planned size is a dry pass of the functions that carve the buffers (chunk_bytes
  // runs carve(), prefixed_bytes an entry point's prefix carve followed by carve(), vjp_chunk_bytes the reverse-pass chunk),
  // so a buffer added to a carve can never be forgotten in the plan (round 1 planned dgrad for S > 1 only while carve()
  // always took it).
  int64_t chunk_bytes(int Bc, int S) const {
    DryPass dp(this);
    carve(plan_base(), Bc, S);
    return dp.bytes();
  }
  Ws carve(void* base, int Bc, int S) const {
    Ws w;
    size_t rows = (size_t)Bc * N * S;
    Arena a(this, base);
    if (gnn) {
      const size_t e = cfg.edge_dim, hm = gnn_hmax(), dm = gnn_dmax(), em = gnn_emax(), hn = gnn_hnode_max();
      const size_t pairs8 = (size_t)Bc * N * (N + (cfg.gnn_conv_ne ? M : 0)) * 8;
      w.X = a.take<T>(rows * dm); w.O = a.take<T>(rows * dm); w.G0 = a.take<T>(rows * d); w.G1 = a.take<T>(rows * d);
      w.G2 = a.take<T>(rows * d); w.Fc = a.take<T>(rows * (3 * dm + 3 * e)); w.Hs = a.take<T>(rows * e);
      w.Ha = a.take<T>(rows * e); w.HT = a.take<T>(rows * hn); w.C = a.take<T>(rows * 3 * e);
      w.E0 = a.take<T>(pairs8 * em); w.E1 = a.take<T>(pairs8 * em); w.ET0 = a.take<T>(pairs8 * em); w.ET1 = a.take<T>(pairs8 * em);
      w.W3 = a.take<T>(pairs8 * 3 * e);
      w.Y0 = a.take<T>(rows * hm); w.Y1 = a.take<T>(rows * hm); w.Jb = a.take<T>((size_t)Bc * S * gnn_jsum());
      w.A = w.M1 = w.QKV = nullptr;
      w.BF = a.take<T>(rows * KN);
    } else if (cfg.kind == DQMC_FERMINET) {
      const size_t dm = fermi_dmax(), em = fermi_emax(), fin = 3 * dm + 2 * em;
      w.X = a.take<T>(rows * dm); w.O = a.take<T>(rows * dm); w.QKV = a.take<T>(rows * fin);  // H, H2, F
      w.A = a.take<T>(rows * N * em); w.M1 = a.take<T>(rows * N * em);                        // E, E2
      w.BF = a.take<T>(rows * BFW);
    } else {
      w.X = a.take<T>(rows * d); w.O = a.take<T>(rows * d); w.A = a.take<T>(rows * d); w.M1 = a.take<T>(rows * d);
      w.QKV = a.take<T>(rows * 3 * d); w.BF = a.take<T>(rows * BFW);
    }
    w.dsign = a.take<T>((size_t)Bc * K); w.dlog = a.take<T>((size_t)Bc * K); w.dlap = a.take<T>((size_t)Bc * K);
    w.dgrad = a.take<T>((size_t)Bc * K * (S > 1 ? T3 : 1));
    if (ph_on && S > 1) w.QA = a.take<T>((size_t)Bc * N * PH_STRIDE);
    if (cfg.backflow_add) w.Gadd = a.take<T>((size_t)Bc * N * 5);
    return w;
  }
  // bytes of the buffers `prefix` carves followed by a forward chunk of Bc walkers with S slots
  template <class Prefix>
  int64_t prefixed_bytes(Prefix prefix, int64_t Bc, int S) const {
    DryPass dp(this);
    Arena a(this, plan_base());
    prefix(a);
    carve(a.top, (int)Bc, S);
    return dp.bytes();
  }
  // largest walker chunk (<= B, <= the 32-bit row cap) whose carve fits wsb bytes
  int max_chunk(int64_t wsb, int S, int B) const {
    int64_t row_cap = kRowCap / ((int64_t)N * S * 3 * d);
    if (cfg.kind == DQMC_FERMINET) row_cap = kRowCap / ((int64_t)N * N * S * (3 * (int64_t)fermi_dmax() + 64));
    if (gnn) row_cap = kRowCap / ((int64_t)N * (N + M + S) * (8 * gnn_emax() + 3 * gnn_dmax() + 3 * cfg.edge_dim + KN));
    return (int)largest_fit(std::min<int64_t>(B, row_cap), wsb, [&](int64_t n) { return chunk_bytes((int)n, S); });
  }
  // Virtual-walker group of nb base walkers (non-local ECP quadrature points, spin swaps): the V virtual walkers r[V][N][3],
  // their sign[V] and log[V], and the base walkers' envelope table [nb][N][K N] and embedding rows [nb][N][d] that the
  // forwards gather the unmoved electrons from.  The ECP group adds its active-pair list int[nb J N] and the per-walker
  // offsets into it int[nb + 1] (the last entry is the group's pair count), the spin group the base walkers' sign[nb] and
  // log[nb].
  struct VirtGroup {
    T *r, *sign, *logp, *env = nullptr, *emb = nullptr, *sign0 = nullptr, *logp0 = nullptr;
    int *pairs = nullptr, *offs = nullptr;
    T *gr = nullptr, *gR = nullptr, *gR0 = nullptr;  // ECP force group: grad_r / grad_R of the virtual walkers, grad_R of the base walkers
  };
  VirtGroup carve_virt_group(Arena& a, int64_t nb, int64_t V) const {
    VirtGroup g;
    g.r = a.take<T>(V * 3 * N); g.sign = a.take<T>(V); g.logp = a.take<T>(V);
    g.env = a.take<T>(nb * N * K * N); g.emb = a.take<T>(nb * N * d);
    return g;
  }
  // Sized for every pair active (V = nb J N 12), so the plan does not depend on the walkers; the cutoff only shortens the
  // list the forwards run over.
  VirtGroup carve_ecp_group(Arena& a, int64_t nb) const {
    VirtGroup g = carve_virt_group(a, nb, nb * J * N * 12);
    g.pairs = a.take<int>(nb * J * N); g.offs = a.take<int>(nb + 1);
    return g;
  }
  // ECP force group (dqmc_ecp_force): the virtual walkers are materialised (no base-walker tables) and the position reverse
  // pass writes their sign, log, grad_r [V][N][3] and grad_R [V][M][3]; the base walkers' sign, log and grad_R [nb][M][3].
  // Sized for every pair active, like carve_ecp_group.
  VirtGroup carve_ecp_force_group(Arena& a, int64_t nb) const {
    const int64_t V = nb * J * N * 12;
    VirtGroup g;
    g.r = a.take<T>(V * 3 * N); g.sign = a.take<T>(V); g.logp = a.take<T>(V);
    g.gr = a.take<T>(V * 3 * N); g.gR = a.take<T>(V * 3 * M);
    g.pairs = a.take<int>(nb * J * N); g.offs = a.take<int>(nb + 1);
    g.sign0 = a.take<T>(nb); g.logp0 = a.take<T>(nb); g.gR0 = a.take<T>(nb * 3 * M);
    return g;
  }
  VirtGroup carve_spin_group(Arena& a, int64_t nb, int64_t P) const {  // P swapped pairs per walker
    VirtGroup g = carve_virt_group(a, nb, nb * P);
    g.sign0 = a.take<T>(nb); g.logp0 = a.take<T>(nb);
    return g;
  }
  // base walkers per virtual-walker group (vper virtual walkers each) are bounded by the 32-bit row cap of the plain-forward
  // chunk: the plan never asks for more
  int64_t group_cap(int64_t vper) const { return std::max<int64_t>(1, kRowCap / ((int64_t)N * 3 * d) / vper); }
  // bytes of an ECP / spin group of nb walkers + a plain-forward chunk of Vc virtual walkers
  int64_t ecp_bytes(int64_t nb, int64_t Vc) const { return prefixed_bytes([&](Arena& a) { carve_ecp_group(a, nb); }, Vc, 1); }
  // what one chunk of Vc virtual walkers carves after a group's prefix: a plain forward (ECP energy, spin), or a position
  // reverse pass (ECP force); the chunk-size functions of virtual_groups
  void fwd_chunk_carve(Arena& a, int64_t Vc) const { carve(a.top, (int)Vc, 1); }
  void pos_chunk_carve(Arena& a, int64_t Vc) {
    const PosOut none{nullptr, nullptr};
    reverse_chunk(nullptr, nullptr, 0, (int)Vc, nullptr, nullptr, nullptr, nullptr, Arena(this, a.top), nullptr, &none);
  }
  // bytes of an ECP force group of nb walkers + a position reverse-pass chunk of Vc virtual walkers
  int64_t ecp_force_bytes(int64_t nb, int64_t Vc) {
    DryPass dp(this);
    Arena a(this, plan_base());
    carve_ecp_force_group(a, nb);
    pos_chunk_carve(a, Vc);
    return dp.bytes();
  }
  // the non-local ECP force needs grad_r and grad_R of log|psi| by the reverse pass (TransPsiformer: grad_r only)
  bool has_nl_force() const { return has_pos_pass() && !trans; }
  int64_t spin_bytes(int64_t nb, int64_t P, int64_t Vc) const {
    return prefixed_bytes([&](Arena& a) { carve_spin_group(a, nb, P); }, Vc, 1);
  }
  // Metropolis / Langevin sweep over B walkers: the proposed walkers (Langevin: and their drift), their sign and log, the
  // acceptance counter (one 256-byte slot)
  struct Proposals { T *r, *force, *sign, *logp; int* cnt; };
  Proposals carve_proposals(Arena& a, int B, bool with_force) const {
    Proposals q;
    q.r = a.take<T>((size_t)B * 3 * N); q.force = with_force ? a.take<T>((size_t)B * 3 * N) : nullptr;
    q.sign = a.take<T>(B); q.logp = a.take<T>(B); q.cnt = a.take<int>(1);
    return q;
  }
  struct ForceBufs { T *E, *stats, *grad; };  // value_and_force: E, 6 stats, grad of the forward-Laplacian pass
  ForceBufs carve_force(Arena& a, int B) const {
    ForceBufs f;
    f.E = a.take<T>(B); f.stats = a.take<T>((size_t)6 * B); f.grad = a.take<T>((size_t)B * T3);
    return f;
  }
  // prefix of a Metropolis (langevin false) or Langevin sweep over B walkers + a forward chunk of Bc walkers
  int64_t sweep_bytes(int B, bool langevin, int Bc) const {
    auto prefix = [&](Arena& a) { carve_proposals(a, B, langevin); if (langevin) carve_force(a, B); };
    return prefixed_bytes(prefix, Bc, langevin ? T3 + 2 : 1);
  }
  // bytes one reverse-pass chunk of Bc walkers carves: a dry pass of the chunk function itself
  // (pos: the position mode of dqmc_wf_grad_positions, Psiformer kinds and FermiNet)
  int64_t vjp_chunk_bytes(int Bc, bool pos = false) {
    DryPass dp(this);
    const PosOut none{nullptr, nullptr};
    reverse_chunk(nullptr, nullptr, 0, Bc, nullptr, nullptr, nullptr, nullptr, Arena(this, plan_base()), nullptr,
                  pos ? &none : nullptr);
    return dp.bytes();
  }
  bool has_pos_pass() const { return !gnn && !cfg.backflow_add; }
  int64_t ws_bytes(int B, int mode) override {
    if (B < 1) B = 1;
    if (mode == DQMC_MODE_VJP) return vjp_chunk_bytes(B);
    if (mode == DQMC_MODE_GRAD_POS) return has_pos_pass() ? vjp_chunk_bytes(B, true) : 0;
    if (mode == DQMC_MODE_MCMC) return sweep_bytes(B, false, B);
    if (mode == DQMC_MODE_LANGEVIN) return sweep_bytes(B, true, B);
    if (mode == DQMC_MODE_ECP_FORCE) {  // out_nl; out_bare alone needs no workspace
      if (!J || !has_nl_force()) return 0;
      const int64_t vper = (int64_t)J * N * 12, nb = std::min<int64_t>(B, group_cap(vper));
      return ecp_force_bytes(nb, nb * vper);
    }
    if (mode == DQMC_MODE_ZV_FORCE) return zv_refusal() ? 0 : zv_chunk_bytes(B);
    if (mode == DQMC_MODE_SPIN) {  // sized for the exact estimator, the larger of the two; no down electrons: no forwards
      const int64_t P = (int64_t)cfg.n_up * cfg.n_down;
      if (!P) return 0;
      const int64_t nb = std::min<int64_t>(B, group_cap(P));
      return spin_bytes(nb, P, nb * P);
    }
    int S = mode == DQMC_MODE_FORWARD ? 1 : T3 + 2;
    int64_t need = chunk_bytes(B, S);
    if (mode == DQMC_MODE_LOCAL_ENERGY && J > 0) {
      const int64_t vper = (int64_t)J * N * 12, nb = std::min<int64_t>(B, group_cap(vper));
      need = std::max(need, ecp_bytes(nb, nb * vper));
    }
    return need;
  }
  // least workspace with which a call for B walkers proceeds (walkers chunked down to one at a time)
  int64_t ws_bytes_min(int B, int mode) override {
    if (B < 1) B = 1;
    const int S = T3 + 2;
    switch (mode) {
      case DQMC_MODE_VJP: return vjp_chunk_bytes(1);
      case DQMC_MODE_GRAD_POS: return has_pos_pass() ? vjp_chunk_bytes(1, true) : 0;
      case DQMC_MODE_MCMC: return sweep_bytes(B, false, 1);
      case DQMC_MODE_LANGEVIN: return sweep_bytes(B, true, 1);
      case DQMC_MODE_LOCAL_ENERGY: return std::max<int64_t>(chunk_bytes(1, S), J > 0 ? ecp_bytes(1, 1) : 0);
      case DQMC_MODE_ECP_FORCE: return J > 0 && has_nl_force() ? ecp_force_bytes(1, 1) : 0;
      case DQMC_MODE_ZV_FORCE: return zv_refusal() ? 0 : zv_chunk_bytes(1);
      case DQMC_MODE_SPIN: {
        const int64_t P = (int64_t)cfg.n_up * cfg.n_down;
        return P ? spin_bytes(1, P, 1) : 0;
      }
      default: return chunk_bytes(1, 1);
    }
  }
  // dqmc_debug_plan: walk the entry point of `mode` with a workspace of wsb bytes (<= 0: the planned size) on a dummy base
  // and report the highest offset it carves.  Host-only (works on plan-only engines).
  int debug_plan(int B, int mode, int64_t wsb, int64_t* planned, int64_t* carved) override {
    const int64_t pl = ws_bytes(B, mode);
    if (planned) *planned = pl;
    if (wsb <= 0) wsb = pl;
    DryPass dp(this);
    void* ws = plan_base();
    int rc = 0;
    switch (mode) {
      case DQMC_MODE_FORWARD: rc = forward(nullptr, nullptr, 0, B, nullptr, nullptr, ws, wsb, nullptr); break;
      case DQMC_MODE_LOCAL_ENERGY:
        rc = local_energy(nullptr, nullptr, 0, B, 0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, ws, wsb, nullptr);
        break;
      case DQMC_MODE_VJP: rc = vjp_params(nullptr, nullptr, 0, B, nullptr, nullptr, nullptr, nullptr, ws, wsb, nullptr); break;
      case DQMC_MODE_MCMC:
        rc = mcmc(nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, B, 1, 0.5, -1, 0, 0, 0, nullptr, nullptr, nullptr, ws, wsb,
                  nullptr, 0.0, nullptr, nullptr);
        break;
      case DQMC_MODE_LANGEVIN:
        rc = langevin(nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, B, 1, 0.5, -1, 0, 0, 0, nullptr, nullptr,
                      nullptr, ws, wsb, nullptr);
        break;
      case DQMC_MODE_SPIN: rc = spin(nullptr, nullptr, 0, B, nullptr, nullptr, -1, nullptr, nullptr, ws, wsb, nullptr); break;
      case DQMC_MODE_GRAD_POS:
        rc = grad_positions(nullptr, nullptr, 0, B, nullptr, nullptr, nullptr, nullptr, ws, wsb, nullptr);
        break;
      case DQMC_MODE_ECP_FORCE:
        rc = ecp_force(nullptr, nullptr, 0, B, 0, nullptr, nullptr, has_nl_force() ? ws : nullptr, ws, wsb, nullptr);
        break;
      case DQMC_MODE_ZV_FORCE: rc = zv_force(nullptr, nullptr, 0, B, nullptr, nullptr, ws, wsb, nullptr); break;
      default: err = "unknown mode"; rc = 2;
    }
    if (carved) *carved = dp.bytes();
    return rc;
  }

  // ---- GEMM dispatch ------------------------------------------------------------------------
  // dense layers can absorb the tanh propagation in the tensor-core epilogue when whole slot
  // groups fit a 128-row tile with little padding
  bool can_fuse_act(int S) const {
    if (!use_tc() || sw.no_fuse_tanh) return false;
    if (S == 1) return true;
    return S <= 128 && (128 / S) * S >= 112;
  }
  // gemm() runs the tensor-core kernel for these operands (else the CUDA-core gemm_kernel)
  bool gemm_on_tc(const char* w0, const char* w1, int lda, int ldc, int Kc, const T* bias1) const {
#if !defined(DQMC_NO_TCGEN05)
    return use_tc() && !bias1 && Kc % 32 == 0 && lda % 4 == 0 && ldc % 4 == 0 && tcw.count(w0) && (!w1 || tcw.count(w1));
#else
    return false;
#endif
  }
  int gemm(const T* A, int lda, const char* w0, const char* w1, int zsplit, int ldw, const T* bias, const T* Res,
           int ldr, T* C, int ldc, int Mr, int Nc, int Kc, int S, int sliced, int Nel, cudaStream_t st, int act = 0,
           const T* bias1 = nullptr) {
    if (dry) return 0;  // planning pass
    const T* W0 = P(w0);
    const T* W1 = w1 ? P(w1) : nullptr;
#if !defined(DQMC_NO_TCGEN05)
    if constexpr (std::is_same<T, float>::value) {
      if (gemm_on_tc(w0, w1, lda, ldc, Kc, bias1)) {
        const TcWeight& t0 = tcw.at(w0);
        const TcWeight& t1 = w1 ? tcw.at(w1) : t0;
        tc::Params p;
        p.A = A; p.lda = lda; p.bias = bias; p.Res = Res; p.ldr = ldr; p.C = C; p.ldc = ldc; p.M = Mr; p.N = Nc;
        p.K = Kc; p.S = S; p.sliced = sliced; p.Nel = Nel; p.z_split = zsplit; p.err_flag = nullptr;
        p.act = act;
        p.rpt = (act && S > 1) ? (128 / S) * S : tc::kBM;
        p.a_scale = 1.f; p.unscale = 1.f;
        // plain forwards: half operands (hi / lo), f16 wgmma -- twice the MMA rate, half the shared-memory bytes per k
        const bool f16 = S == 1 && sw.tc_f16 && Kc % 64 == 0 && t0.f16 && t1.f16 && t0.wscale == t1.wscale;
        if (f16) { p.a_scale = kActScale; p.unscale = 1.f / (kActScale * t0.wscale); }
        const int MT = (Mr + p.rpt - 1) / p.rpt, NT = (Nc + tc::kBN - 1) / tc::kBN;
        const int n_tiles = (sliced ? Nel : 1) * MT * NT;  // one tile per CTA
#ifndef DQMC_EMU
        cudaEvent_t e0 = nullptr, e1 = nullptr;
        if (prof) { cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventRecord(e0, st); }
#endif
        if (f16)
          DQ_LAUNCH(tc::gemm3x_kernel<true>, dim3(n_tiles), dim3(tc::kThreads), tc::SmemLayout::total(), st, t0.m16h, t0.m16l,
                    t1.m16h, t1.m16l, p);
        else
          DQ_LAUNCH(tc::gemm3x_kernel<false>, dim3(n_tiles), dim3(tc::kThreads), tc::SmemLayout::total(), st, t0.mh, t0.ml,
                    t1.mh, t1.ml, p);
#ifndef DQMC_EMU
        if (prof) {
          cudaEventRecord(e1, st);
          prof_note(e0, e1, 2.0 * (double)Mr * (sliced ? Nel : 1) * (double)Nc * (double)Kc, 0);
        }
#endif
        return 0;
      }
    }
#endif
    if (act) { err = "internal: fused activation requested on the CUDA-core GEMM"; return 5; }
    GemmArgs<T> g;
    g.A = A; g.lda = lda; g.W0 = W0; g.W1 = W1; g.z_split = zsplit; g.ldw = ldw; g.bias = bias; g.Res = Res;
    g.ldr = ldr; g.C = C; g.ldc = ldc; g.M = Mr; g.N = Nc; g.K = Kc; g.S = S; g.sliced = sliced; g.Nel = Nel;
    g.bias1 = bias1;
    constexpr int BM = 64, BN = 64, BK = 16, TM = 4, TN = 4;
    dim3 grid((Nc + BN - 1) / BN, (Mr + BM - 1) / BM, sliced ? Nel : 1);
#ifndef DQMC_EMU
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (prof) { cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventRecord(e0, st); }
#endif
    DQ_LAUNCH((gemm_kernel<T, BM, BN, BK, TM, TN>), grid, dim3(256), 0, st, g);
#ifndef DQMC_EMU
    if (prof) {
      cudaEventRecord(e1, st);
      prof_note(e0, e1, 2.0 * (double)Mr * (sliced ? Nel : 1) * (double)Nc * (double)Kc, 0);
    }
#endif
    return 0;
  }

  // Fused MLP block of a plain forward: Out = A + tanh(tanh(A W1 + b1) W2 + b2), A = X + O Wo  (one launch; fused_tc.cuh)
  bool can_fuse_mlp(int S, const std::string& pfx) const {
#if !defined(DQMC_NO_TCGEN05)
    if (S != 1 || !use_tc() || !sw.tc_f16 || (d != 128 && d != 256)) return false;
    for (const char* n : {"wo", "w1", "w2"}) {
      auto it = tcw.find(pfx + n);
      if (it == tcw.end() || !it->second.f16_all) return false;
    }
    return true;
#else
    return false;
#endif
  }
  int mlp_block(const std::string& pfx, const T* O, const T* X, T* Out, int rows, cudaStream_t st) {
    if (dry) return 0;
#if !defined(DQMC_NO_TCGEN05)
    if constexpr (std::is_same<T, float>::value) {
      const TcWeight& wo = tcw.at(pfx + "wo");
      const TcWeight& w1 = tcw.at(pfx + "w1");
      const TcWeight& w2 = tcw.at(pfx + "w2");
      tc::MlpParams p;
      p.O = O; p.ldo = d; p.X = X; p.ldx = d; p.Out = Out; p.ldout = d; p.b1 = P(pfx + "b1"); p.b2 = P(pfx + "b2");
      p.M = rows; p.d = d; p.a_scale = kActScale;
      p.us0 = 1.f / (kActScale * wo.wscale); p.us1 = 1.f / (kActScale * w1.wscale); p.us2 = 1.f / (kActScale * w2.wscale);
      p.err_flag = d_tc_err;
      const int MT = (rows + 127) / 128;
      const int grid = MT < n_sms ? MT : n_sms;
#ifndef DQMC_EMU
      cudaEvent_t e0 = nullptr, e1 = nullptr;
      if (prof) { cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventRecord(e0, st); }
#endif
      if (d == 256)
        DQ_LAUNCH(tc::mlp_block_f16_kernel<256>, dim3(grid), dim3(tc::kMlpThreads), tc::MlpSmem::total(), st, wo.m16h_all,
                  wo.m16l_all, w1.m16h_all, w1.m16l_all, w2.m16h_all, w2.m16l_all, p);
      else
        DQ_LAUNCH(tc::mlp_block_f16_kernel<128>, dim3(grid), dim3(tc::kMlpThreads), tc::MlpSmem::total(), st, wo.m16h_all,
                  wo.m16l_all, w1.m16h_all, w1.m16l_all, w2.m16h_all, w2.m16l_all, p);
#ifndef DQMC_EMU
      if (prof) {
        cudaEventRecord(e1, st);
        prof_note(e0, e1, 3 * 2.0 * (double)rows * (double)d * (double)d, 1);
      }
#endif
      return 0;
    }
#endif
    err = "internal: fused MLP block without the tensor-core backend";
    return 5;
  }

  int debug_mlp_block(int layer, const void* O, const void* X, void* Out, int rows, cudaStream_t st) override {
    const std::string pfx = "L" + std::to_string(layer) + ".";
    if (!can_fuse_mlp(1, pfx)) { err = "fused MLP block not available for this configuration"; return 2; }
    int rc = mlp_block(pfx, (const T*)O, (const T*)X, (T*)Out, rows, st);
    if (rc) return rc;
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  // Whole trunk of a plain forward in one launch (trunk_tc.cuh): needs the shipped Psiformer shape (d = 256, 4 heads of 64)
  bool trunk_weights_ok() const {
#if !defined(DQMC_NO_TCGEN05)
    for (int l = 0; l < cfg.n_layers; ++l)
      for (const char* n : {"wqkv", "wo", "w1", "w2"}) {
        auto it = tcw.find("L" + std::to_string(l) + "." + n);
        if (it == tcw.end() || !it->second.f16_256) return false;
      }
    return true;
#else
    return false;
#endif
  }
  bool can_trunk(int S) const {
#if !defined(DQMC_NO_TCGEN05)
    return S == 1 && use_tc() && sw.tc_f16 && sw.tc_trunk && d_trunk_maps && d_trunk_scratch && cfg.n_layers >= 1 && trunk_weights_ok();
#else
    return false;
#endif
  }
  // in.emb set: compact virtual-walker forwards, walker w of the launch is virtual walker v0 + w
  int trunk_block(const T* X0, T* Out, int rows, cudaStream_t st, const FwdIn& in, int64_t v0) {
    if (dry) return 0;
#if !defined(DQMC_NO_TCGEN05)
    if constexpr (std::is_same<T, float>::value) {
      tc::TrunkParams p;
      p.X0 = X0; p.ldx = d; p.Out = Out; p.ldout = d; p.maps = d_trunk_maps; p.scratch = d_trunk_scratch;
      p.Xbase = in.emb; p.v0 = in.emb ? (long long)v0 : 0; p.vper = in.emb ? in.vper : 0;
      p.n_up = cfg.n_up; p.vlayout = in.layout; p.pairs = in.pairs; p.wspin = P("emb.w") + (size_t)(4 * M) * d;  // the +-1 spin feature's row
      int np2 = 1;
      while (np2 < N) np2 *= 2;  // walker slot of the tile: electrons rounded up to a power of two (<= 32)
      p.walkers = rows / N; p.N = N; p.L = cfg.n_layers; p.a_scale = kActScale;
      p.attn_scale = (float)(1.0 / std::sqrt((double)dh)); p.err_flag = d_tc_err; p.phase = d_trunk_phase;
      for (int l = 0; l < cfg.n_layers; ++l) {
        const std::string pfx = "L" + std::to_string(l) + ".";
        p.b1[l] = P(pfx + "b1"); p.b2[l] = P(pfx + "b2");
        int g = 0;
        for (const char* n : {"wqkv", "wo", "w1", "w2"}) p.us[l][g++] = 1.f / (kActScale * tcw.at(pfx + n).wscale);
      }
      const int G = 128 / np2, MT = (p.walkers + G - 1) / G;
      const int grid = MT < n_sms ? MT : n_sms;
#ifndef DQMC_EMU
      cudaEvent_t e0 = nullptr, e1 = nullptr;
      if (prof) { cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventRecord(e0, st); }
#endif
      switch (np2) {  // one kernel instance per walker slot
        case 1: DQ_LAUNCH(tc::trunk_f16_kernel<1>, dim3(grid), dim3(tc::kTrThreads), tc::TrSmem::total(), st, p); break;
        case 2: DQ_LAUNCH(tc::trunk_f16_kernel<2>, dim3(grid), dim3(tc::kTrThreads), tc::TrSmem::total(), st, p); break;
        case 4: DQ_LAUNCH(tc::trunk_f16_kernel<4>, dim3(grid), dim3(tc::kTrThreads), tc::TrSmem::total(), st, p); break;
        case 8: DQ_LAUNCH(tc::trunk_f16_kernel<8>, dim3(grid), dim3(tc::kTrThreads), tc::TrSmem::total(), st, p); break;
        case 16: DQ_LAUNCH(tc::trunk_f16_kernel<16>, dim3(grid), dim3(tc::kTrThreads), tc::TrSmem::total(), st, p); break;
        case 32: DQ_LAUNCH(tc::trunk_f16_kernel<32>, dim3(grid), dim3(tc::kTrThreads), tc::TrSmem::total(), st, p); break;
        default: err = "internal: fused trunk walker slot above 32"; return 5;
      }
#ifndef DQMC_EMU
      if (prof) {
        cudaEventRecord(e1, st);
        // dense layers 12 d^2 and attention 4 N d (scores + weighted sum) flops per row and layer
        prof_note(e0, e1, (double)cfg.n_layers * 2.0 * (double)rows * (6.0 * d * d + 2.0 * N * d), 2);
      }
#endif
      return 0;
    }
#endif
    err = "internal: fused trunk without the tensor-core backend";
    return 5;
  }
  int debug_trunk_phases(uint64_t* out, int n) override {
#if !defined(DQMC_NO_TCGEN05)
    if (!d_trunk_phase) { err = "trunk phase timers are off (set DQMC_TRUNK_PHASES=1 before creating the engine)"; return 2; }
    if (n < tc::kPhases) { err = "dqmc_debug_trunk_phases: the output holds fewer than the kernel's counters"; return 2; }
    DQ_CHECK(cudaMemcpy(out, d_trunk_phase, sizeof(unsigned long long) * tc::kPhases, cudaMemcpyDeviceToHost));
    DQ_CHECK(cudaMemset(d_trunk_phase, 0, sizeof(unsigned long long) * tc::kPhases));
    return 0;
#else
    err = "this build has no tensor-core backend"; return 2;
#endif
  }
  int debug_tc_error(int32_t* flag) override {
#if !defined(DQMC_NO_TCGEN05)
    if (!d_tc_err) { err = "no tensor-core backend in this engine"; return 2; }
    int v = 0;
    DQ_CHECK(cudaMemcpy(&v, d_tc_err, sizeof(int), cudaMemcpyDeviceToHost));
    DQ_CHECK(cudaMemset(d_tc_err, 0, sizeof(int)));
    *flag = v;
    return 0;
#else
    err = "this build has no tensor-core backend"; return 2;
#endif
  }
  int debug_trunk(const void* X0, void* Out, int rows, cudaStream_t st) override {
    if (!can_trunk(1)) { err = "fused trunk not available for this configuration"; return 2; }
    if (rows % N != 0) { err = "debug_trunk: rows must be a multiple of the electron count"; return 2; }
    int rc = trunk_block((const T*)X0, (T*)Out, rows, st, FwdIn{}, 0);
    if (rc) return rc;
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  int debug_attention(int layer, const void* QKV, void* O, int rows, int S, int32_t* kernel, cudaStream_t st) override {
    if (!(cfg.kind == DQMC_PSIFORMER || trans)) { err = "debug_attention: the configuration has no softmax attention layers"; return 2; }
    if (layer < 0 || layer >= cfg.n_layers) { err = "debug_attention: layer out of range"; return 2; }
    // the tangent chunk and the shared memory of the forward-Laplacian kernels were sized for T3 = 3N at creation
    if (S != 1 && S != T3 + 2) { err = "debug_attention: S must be 1 or 3N + 2"; return 2; }
    if (rows < 1 || rows % (N * S) != 0) { err = "debug_attention: rows must be a positive multiple of N S"; return 2; }
    int rc = attention((const T*)QKV, (T*)O, rows / (N * S), S, layer, st, kernel);
    if (rc) return rc;
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  int debug_mlp(int layer, int S, const void* O, const void* X, void* Out, void* scratch, int rows, int32_t* path,
                cudaStream_t st) override {
    if (!(cfg.kind == DQMC_PSIFORMER || trans)) { err = "debug_mlp: the configuration has no attention layers"; return 2; }
    if (layer < 0 || layer >= cfg.n_layers) { err = "debug_mlp: layer out of range"; return 2; }
    if (S != 1 && S != T3 + 2) { err = "debug_mlp: S must be 1 or 3N + 2"; return 2; }
    if (rows < 1 || rows % (N * S) != 0) { err = "debug_mlp: rows must be a positive multiple of N S"; return 2; }
    T* A = (T*)scratch;
    int rc = mlp("L" + std::to_string(layer) + ".", (const T*)O, (const T*)X, (T*)Out, A, A + (size_t)rows * d, rows / (N * S), S,
                 st, path);
    if (rc) return rc;
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  int debug_slater(const void* r, const void* R, const void* BF, int rows, int S, void* dsign, void* dlog, void* dgrad,
                   void* dlap, int32_t* kernel, cudaStream_t st) override {
    if (S != 1 && S != T3 + 2) { err = "debug_slater: S must be 1 or 3N + 2"; return 2; }
    if (rows < 1 || rows % (N * S) != 0) { err = "debug_slater: rows must be a positive multiple of N S"; return 2; }
    if (S > 1 && (!dgrad || !dlap)) { err = "debug_slater: S = 3N + 2 needs the gradient and Laplacian outputs"; return 2; }
    const int Bc = rows / (N * S);
    // the activation runs in place: work on a copy so that the caller's rows stay as they were
    T* bf = nullptr;
    T* gadd = nullptr;
    DQ_CHECK(cudaMalloc((void**)&bf, sizeof(T) * (size_t)rows * BFW));
    if (cfg.backflow_add && cudaMalloc((void**)&gadd, sizeof(T) * (size_t)Bc * N * 5) != cudaSuccess) {
      cudaFree(bf);
      err = "debug_slater: out of device memory";
      return 1;
    }
    int rc = 0;
    if (cudaMemcpyAsync(bf, BF, sizeof(T) * (size_t)rows * BFW, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
      err = "debug_slater: copy of the backflow rows failed";
      rc = 1;
    }
    if (!rc) rc = slater((const T*)r, (const T*)R, 0, Bc, S, bf, gadd, (T*)dsign, (T*)dlog, (T*)dgrad, (T*)dlap, st, nullptr,
                         FwdIn{}, 0, kernel);
    if (!rc && cudaStreamSynchronize(st) != cudaSuccess) { err = "debug_slater: kernel failed"; rc = 1; }
    cudaFree(bf);
    cudaFree(gadd);
    if (rc) return rc;
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  int debug_det_sum(const void* r, const void* R, const void* dsign, const void* dlog, const void* dgrad, const void* dlap,
                    int B, int S, void* sign, void* logp, void* grad, void* stats, cudaStream_t st) override {
    if (S != 1 && S != T3 + 2) { err = "debug_det_sum: S must be 1 or 3N + 2"; return 2; }
    if (B < 1) { err = "debug_det_sum: needs at least one walker"; return 2; }
    if (S > 1 && (!dgrad || !dlap || !grad || !stats)) { err = "debug_det_sum: S = 3N + 2 needs every jet array"; return 2; }
    T* E = nullptr;  // the local energy finalize_kernel also writes; not part of the hook's outputs
    DQ_CHECK(cudaMalloc((void**)&E, sizeof(T) * (size_t)B));
    const FinalizeCfg fc = finalize_cfg(S);
    DQ_LAUNCH(finalize_kernel<T>, dim3(B), dim3(128), finalize_smem_bytes<T>(N, K), st, fc, (const T*)r, (const T*)R, 0,
              (const T*)dsign, (const T*)dlog, (const T*)dgrad, (const T*)dlap, P("cusp.alpha"), (const T*)d_zval,
              (const T*)d_ecp_loc, (const int*)d_ecp_mask, B, (T*)sign, (T*)logp, E, (T*)stats, (T*)grad,
              cfg.conf_linear ? P("conf.w") : (const T*)nullptr, (const T*)nullptr,
              cfg.nuc_cusp_kind ? P("cusp.nuc") : (const T*)nullptr, PhArgs<T>());
    const bool ok = cudaStreamSynchronize(st) == cudaSuccess;
    cudaFree(E);
    if (!ok) { err = "debug_det_sum: kernel failed"; return 1; }
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  int debug_attention_bwd(int layer, const void* QKV, const void* dO, void* dQKV, void* dKn, void* dVn, int rows,
                          cudaStream_t st) override {
    if (!(cfg.kind == DQMC_PSIFORMER || trans)) { err = "debug_attention_bwd: the configuration has no softmax attention layers"; return 2; }
    if (layer < 0 || layer >= cfg.n_layers) { err = "debug_attention_bwd: layer out of range"; return 2; }
    if (rows < 1 || rows % N != 0) { err = "debug_attention_bwd: rows must be a positive multiple of N"; return 2; }
    if (Mn > 0 && (!dKn || !dVn)) { err = "debug_attention_bwd: nuclear tokens need the dKn / dVn outputs"; return 2; }
    int rc = attention_bwd(layer, (const T*)QKV, (const T*)dO, (T*)dQKV, rows / N, Mn > 0 ? (T*)dKn : nullptr,
                           Mn > 0 ? (T*)dVn : nullptr, st);
    if (rc) return rc;
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  int debug_wgrad(const void* A, const void* dY, int rows, int Kc, int Nc, int lo, int hi, void* dW, void* db,
                  cudaStream_t st) override {
    if (rows < 1 || Kc < 1 || Nc < 1) { err = "debug_wgrad: rows, K and Nc must be positive"; return 2; }
    if (hi != ALL_ROWS && (lo < 0 || hi < lo || hi > N)) { err = "debug_wgrad: the electron range must lie in [0, N]"; return 2; }
    wgrad((const T*)A, Kc, (const T*)dY, Nc, rows, Kc, Nc, (T*)dW, lo, hi, st);
    bgrad((const T*)dY, Nc, rows, Nc, (T*)db, st, lo, hi);
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  int debug_gemm(const char* wname, const char* bname, const void* A, const void* Res, void* C, int Mr, int S,
                 int sliced, int backend, cudaStream_t st) override {
    int64_t o = off(wname);
    if (o < 0) { err = "unknown weight"; return 2; }
    int rows = 0, cols = 0;
    for (auto& e : entries) if (e.name == wname) { rows = e.rows; cols = e.cols; }
    int saved = cfg.gemm_backend;
    cfg.gemm_backend = backend;
    int rc = gemm((const T*)A, rows, wname, sliced ? "bf.dn" : nullptr, cfg.n_up, cols, bname ? P(bname) : nullptr,
                  (const T*)Res, cols, (T*)C, cols, Mr, cols, rows, S, sliced, N, st);
    cfg.gemm_backend = saved;
    if (rc) return rc;
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  // fp32 attention: pick the <N, dh> specialisation (compile-time index arithmetic) when there is one
  template <int NE, int DH>
  int attn_f32_go(const float* QKV, float* O, int Bc, int S, int tb, float scale, int smem, cudaStream_t st, bool setup) {
    if (setup) {
      DQ_CHECK(raise_dyn_smem((attn_fl_f32_kernel<NE, DH, false>), smem));
      DQ_CHECK(raise_dyn_smem((attn_fl_f32_kernel<NE, DH, true>), smem));
      return 0;
    }
    if (attn_fl_mma && S > 1)  // tangent chunks on the tensor cores (8 warp tasks per phase: 256 threads)
      DQ_LAUNCH((attn_fl_f32_kernel<NE, DH, true>), dim3(Bc, H), dim3(256), smem, st, QKV, 3 * d, O, d, N, S, dh, d, scale, tb);
    else
      DQ_LAUNCH((attn_fl_f32_kernel<NE, DH, false>), dim3(Bc, H), dim3(attn_fl_threads), smem, st, QKV, 3 * d, O, d, N, S, dh, d, scale, tb);
    return 0;
  }
  // generic forward-Laplacian attention (any dtype, extra key / value tokens); fp32 with tangents: tensor-core variant
  int launch_attn_generic(const T* QKV, T* O, int Bc, int S, int tb, T scale, const T* kn, const T* vn, cudaStream_t st) {
    if constexpr (std::is_same<T, float>::value) {
      if (attn_gen_mma && S > 1) {
        DQ_LAUNCH((attn_fl_kernel<T, true>), dim3(Bc, H), dim3(256), attn_smem_bytes<T>(N, dh, tb, Mn, 4), st, QKV, 3 * d, O, d, N, S,
                  dh, d, scale, tb, kn, vn, Mn);
        return 0;
      }
    }
    DQ_LAUNCH(attn_fl_kernel<T>, dim3(Bc, H), dim3(S > 1 ? attn_fl_threads : 128), attn_smem_bytes<T>(N, dh, tb, Mn), st, QKV, 3 * d,
              O, d, N, S, dh, d, scale, tb, kn, vn, Mn);
    return 0;
  }
  int launch_attn_f32(const float* QKV, float* O, int Bc, int S, int tb, float scale, int, int smem, cudaStream_t st,
                      bool setup) {
    if (dh == 64) {
      switch (N) {
        case 4: return attn_f32_go<4, 64>(QKV, O, Bc, S, tb, scale, smem, st, setup);
        case 10: return attn_f32_go<10, 64>(QKV, O, Bc, S, tb, scale, smem, st, setup);
        case 14: return attn_f32_go<14, 64>(QKV, O, Bc, S, tb, scale, smem, st, setup);
        case 28: return attn_f32_go<28, 64>(QKV, O, Bc, S, tb, scale, smem, st, setup);
        case 30: return attn_f32_go<30, 64>(QKV, O, Bc, S, tb, scale, smem, st, setup);
        default: return attn_f32_go<0, 64>(QKV, O, Bc, S, tb, scale, smem, st, setup);
      }
    }
    return attn_f32_go<0, 0>(QKV, O, Bc, S, tb, scale, smem, st, setup);
  }

  // ---- one chunk of the wave-function pipeline ---------------------------------------------
  // FermiNet trunk (reference: conf/ansatz/ferminet.yaml; gnn/electron_gnn.py:160-259 with
  // Residual / NodeSum / EdgeSum update features and a shared edge MLP): leaves the final electron
  // embeddings in *Xout.
  int ferminet_trunk(const T* r, const T* R, int Rb, int Bc, int S, Ws& w, T** Xout, cudaStream_t st, const T* qa = nullptr) {
    const int rows = Bc * N * S, rowsE = Bc * N * N * S, de = cfg.edge_dim, d0 = 4 * M;
    const T isq2 = (T)0.70710678118654752440;
    DQ_LAUNCH(embed_kernel<T>, dim3(Bc * N), dim3(128), sizeof(T) * 5 * d0, st, r, R, Rb, N, M, cfg.n_up, S, 0, 0,
              (const T*)nullptr, d0, w.X, Bc * N, 1, qa);
    DQ_LAUNCH(edge_feat_kernel<T>, dim3((Bc * N * N + 127) / 128), dim3(128), 0, st, r, N, S, w.A, Bc * N * N, qa);
    T* Hc = w.X; T* Hn = w.O; T* Ec = w.A; T* En = w.M1;
    int dcur = d0, ecur = 4;
    for (int l = 0; l < cfg.n_layers; ++l) {
      std::string p = "F" + std::to_string(l) + ".";
      const int fin = 3 * dcur + 2 * ecur;
      DQ_LAUNCH(fermi_agg_kernel<T>, dim3(Bc * S, N), dim3(128), 0, st, (const T*)Hc, dcur, (const T*)Ec, ecur, N, cfg.n_up,
                S, w.QKV);
      int rc = gemm(w.QKV, fin, (p + "wg").c_str(), nullptr, 0, d, P(p + "bg"), nullptr, 0, Hn, d, rows, d, fin, S, 0, N, st);
      if (rc) return rc;
      DQ_LAUNCH(tanh_fl_kernel<T>, dim3(Bc * N, (d + 127) / 128), dim3(128), 0, st, Hn, d,
                (const T*)(dcur == d ? Hc : nullptr), dcur, S, d, dcur == d ? isq2 : T(1));
      if (l < cfg.n_layers - 1) {
        rc = gemm(Ec, ecur, (p + "wu").c_str(), nullptr, 0, de, P(p + "bu"), nullptr, 0, En, de, rowsE, de, ecur, S, 0, N, st);
        if (rc) return rc;
        DQ_LAUNCH(tanh_fl_kernel<T>, dim3(Bc * N * N, 1), dim3(32), 0, st, En, de, (const T*)(ecur == de ? Ec : nullptr),
                  ecur, S, de, ecur == de ? isq2 : T(1));
        T* t2 = Ec; Ec = En; En = t2;
        ecur = de;
      }
      T* t1 = Hc; Hc = Hn; Hn = t1;
      dcur = d;
    }
    *Xout = Hc;
    return 0;
  }

  // conv-GNN trunk (reference tests/conf/ansatz.yaml): embedding lookup, per layer edge filters w_t, node
  // transforms h_t, convolution over same / anti / ne edges, featurewise update sum_t g_t(conv_t) + residual;
  // then the Jastrow MLP on sum_i x_i and the hidden layers of the per-spin backflow MLPs (ssp).
  // MLP of `nl` Linear(+bias)+tanh layers on augmented rows (groups of Sg slots): in -> out, ping-pong through tmp
  // (lda: row stride of `in` when its first din columns are the input, 0 = din)
  int gnn_mlp(const T* in, int din, const std::string& base, const int* dims, int nl, bool bias, T* tmp, T* out, int rows_,
              int Sg, cudaStream_t st, int lda = 0) {
    const T* cur = in;
    int dc = din, ld = lda > 0 ? lda : din;
    for (int i = 0; i < nl; ++i) {
      T* dst = (i == nl - 1) ? out : tmp;
      const std::string q = base + "." + std::to_string(i);
      int rc = gemm(cur, ld, (q + ".w").c_str(), nullptr, 0, dims[i], bias ? P(q + ".b") : nullptr, nullptr, 0, dst, dims[i], rows_,
                    dims[i], dc, Sg, 0, 1, st);
      if (rc) return rc;
      DQ_LAUNCH(act_fl_kernel<T>, dim3(rows_ / Sg, (dims[i] + 63) / 64), dim3(64), 0, st, dst, dims[i], (const T*)nullptr, 0, Sg,
                dims[i], T(1), 0);
      cur = dst; dc = ld = dims[i];
    }
    return 0;
  }

  int paulinet_trunk(const T* r, const T* R, int Rb, int Bc, int S, Ws& w, T** Xbf, const T** jastrow, cudaStream_t st,
                     const T* qa = nullptr) {
    const int rows = Bc * N * S, e = cfg.edge_dim, groups = Bc * N, nl = cfg.gnn_sub_n > 0 ? cfg.gnn_sub_n : 1;
    const int Mne = cfg.gnn_conv_ne ? M : 0, NS = N + Mne, nt = cfg.gnn_conv_ne ? 3 : 2;
    const int pairs = Bc * N * NS, prow = pairs * 8;  // compact edge rows: 8 slots per (receiver, sender) pair
    const T isq2 = (T)0.70710678118654752440;
    int dcur = d, ecur = 4;
    if (cfg.gnn_features) {
      dcur = 4 * M;
      DQ_LAUNCH(embed_kernel<T>, dim3(Bc * N), dim3(128), sizeof(T) * 5 * dcur, st, r, R, Rb, N, M, cfg.n_up, S, 0, 0,
                (const T*)nullptr, dcur, w.X, Bc * N, 1, qa);
    } else {
      DQ_LAUNCH(gnn_embed_kernel<T>, dim3((Bc * N * d + 127) / 128), dim3(128), 0, st, P("emb.table"),
                cfg.n_elec_types > 0 ? cfg.n_elec_types : 1, N, cfg.n_up, S, d, w.X, Bc * N);
    }
    DQ_LAUNCH(gnn_edge_feat_kernel<T>, dim3((pairs + 63) / 64), dim3(64), 0, st, r, R, Rb, N, M, Mne, w.E0, pairs, S > 1 ? qa : (const T*)nullptr,
              cfg.gnn_self_edges);
    T* X = w.X;
    T* Xn = w.O;
    T* E = w.E0;
    T* En = w.E1;
    const char* tn[3] = {"same", "anti", "ne"};
    for (int l = 0; l < cfg.n_layers; ++l) {
      const std::string p = "G" + std::to_string(l) + ".";
      // edge filters of every type on all pairs (compact rows), node transforms h_same / h_anti
      // (E holds ecur columns; the type-t stream is its first gnn_ein(t, l), e.g. [|d|] of the raw [|d|, d])
      for (int t = 0; t < nt; ++t) {
        if (t == 2 && cfg.gnn_ne_identity) continue;  // w_for_ne = false: the ne edge stream is the filter
        int rc = gnn_mlp(E, gnn_ein(t, l), p + "w_" + tn[t], cfg.gnn_w_dims[l], nl, cfg.gnn_w_bias != 0, w.ET0,
                         w.W3 + (size_t)t * prow * e, prow, 8, st, ecur);
        if (rc) return rc;
      }
      int rc = gnn_mlp(X, dcur, p + "h_same", cfg.gnn_h_dims[l], nl, true, w.HT, w.Hs, rows, S, st);
      if (rc) return rc;
      rc = gnn_mlp(X, dcur, p + "h_anti", cfg.gnn_h_dims[l], nl, true, w.HT, w.Ha, rows, S, st);
      if (rc) return rc;
      const int dconv = gnn_conv_w(l);
      DQ_LAUNCH(gnn_conv_kernel<T>, dim3(groups), dim3(128), 0, st, (const T*)w.W3, (const T*)(w.W3 + (size_t)prow * e),
                cfg.gnn_ne_identity ? (const T*)E : (const T*)(w.W3 + (size_t)2 * prow * e), cfg.gnn_ne_identity ? ecur : e,
                gnn_hne_w(l), (const T*)w.Hs, (const T*)w.Ha, cfg.gnn_conv_ne ? P(p + "hne") : (const T*)nullptr, N, Mne,
                cfg.n_up, S, e, cfg.gnn_ne_identity, cfg.gnn_self_edges, w.C);
      T* Xout;
      if (cfg.gnn_concat) {
        // x <- [(x +) tanh(g([x, mean_up x, mean_down x, conv_*]))] (/ sqrt 2)   (electron_gnn.py:243-259)
        const int fin = 3 * dcur + dconv;
        DQ_LAUNCH(gnn_concat_kernel<T>, dim3(Bc * S, N), dim3(128), 0, st, (const T*)X, dcur, (const T*)w.C, dconv, N, cfg.n_up,
                  S, w.Fc);
        rc = gemm(w.Fc, fin, (p + "g.w").c_str(), nullptr, 0, d, cfg.gnn_g_bias ? P(p + "g.b") : nullptr, nullptr, 0, Xn, d, rows,
                  d, fin, S, 0, N, st);
        if (rc) return rc;
        const bool res = dcur == d && !cfg.gnn_no_res;
        DQ_LAUNCH(act_fl_kernel<T>, dim3(groups, (d + 63) / 64), dim3(64), 0, st, Xn, d, res ? (const T*)X : (const T*)nullptr,
                  d, S, d, (res && cfg.gnn_res_norm) ? isq2 : T(1), 0);
        Xout = Xn; Xn = X;
      } else {
        // featurewise update: x <- x + sum_t tanh(g_t(conv_t))   (residual hkext.py:116-137)
        T* G[3] = {w.G0, w.G1, w.G2};
        const T* res = dcur == d ? X : nullptr;
        for (int t = 0; t < nt; ++t) {
          rc = gemm(w.C + t * e, nt * e, (p + "g_" + tn[t] + ".w").c_str(), nullptr, 0, d, P(p + "g_" + tn[t] + ".b"), nullptr,
                    0, G[t], d, rows, d, e, S, 0, N, st);
          if (rc) return rc;
          const bool last = t == nt - 1;
          DQ_LAUNCH(act_fl_kernel<T>, dim3(groups, (d + 63) / 64), dim3(64), 0, st, G[t], d, res, d, S, d,
                    (last && res && cfg.gnn_res_norm) ? isq2 : T(1), 0);
          res = G[t];
        }
        Xout = G[nt - 1];
        // the accumulated buffer becomes the new x; hand the old x buffer to the G slot
        T* old = X;
        if (nt == 3) w.G2 = old; else w.G1 = old;
      }
      X = Xout;
      dcur = d;
      if (cfg.gnn_deep_edges && l < cfg.n_layers - 1 && cfg.gnn_sep_edges) {
        // one edge MLP u_t per edge type on the compact rows (into the free filter buffer), then per pair its own type's
        // output + normalised residual (electron_gnn.py:176-188)
        int res_mask = 0;
        for (int t = 0; t < nt; ++t) {
          rc = gnn_mlp(E, gnn_ein(t, l), p + "u_" + tn[t], cfg.gnn_u_dims[l], nl, true, w.ET0, w.W3 + (size_t)t * prow * e, prow,
                       8, st, ecur);
          if (rc) return rc;
          if (gnn_ein(t, l) == e && ecur == e) res_mask |= 1 << t;
        }
        DQ_LAUNCH((gnn_edge_select_kernel<T>), dim3((unsigned)(((size_t)prow * e + 255) / 256)), dim3(256), 0, st, (const T*)E,
                  (const T*)w.W3, (const T*)(w.W3 + (size_t)prow * e), (const T*)(w.W3 + (size_t)2 * prow * e), 8, N, Mne,
                  cfg.n_up, e, res_mask, isq2, En, (size_t)prow * e);
        T* tmp = E; E = En; En = tmp;
        ecur = e;
      } else if (cfg.gnn_deep_edges && l < cfg.n_layers - 1) {
        // shared edge MLP u on the compact rows + normalised residual (electron_gnn.py:160-192)
        rc = gnn_mlp(E, ecur, p + "u", cfg.gnn_u_dims[l], nl, true, w.ET0, w.ET1, prow, 8, st);
        if (rc) return rc;
        if (ecur == e) {
          // (e + u(e)) / sqrt 2: u's last tanh already applied -> plain scaled add on all slots
          DQ_LAUNCH((axpby_kernel<T>), dim3((unsigned)(((size_t)prow * e + 255) / 256)), dim3(256), 0, st, (const T*)E,
                    (const T*)w.ET1, isq2, En, (size_t)prow * e);
          T* tmp = E; E = En; En = tmp;
        } else {
          T* tmp = E; E = w.ET1; w.ET1 = tmp;
        }
        ecur = e;
      }
    }
    *jastrow = nullptr;
    if (cfg.jastrow_n > 0) {
      const int jr = Bc * S;
      T* cur = w.Jb;
      int din = d;
      DQ_LAUNCH(sum_electrons_kernel<T>, dim3((jr * d + 127) / 128), dim3(128), 0, st, (const T*)X, N, S, d, cur, jr * d);
      for (int i = 0; i < cfg.jastrow_n; ++i) {
        const int dout = cfg.jastrow_dims[i];
        T* nxt = cur + (size_t)jr * din;
        const bool last = i == cfg.jastrow_n - 1;
        const std::string q = "J" + std::to_string(i);
        int rc = gemm(cur, din, (q + ".w").c_str(), nullptr, 0, dout, last ? nullptr : P(q + ".b"), nullptr, 0, nxt, dout, jr,
                      dout, din, S, 0, 1, st);
        if (rc) return rc;
        if (!last) DQ_LAUNCH(act_fl_kernel<T>, dim3(Bc, (dout + 31) / 32), dim3(32), 0, st, nxt, dout, (const T*)nullptr, 0, S, dout, T(1), 1);
        cur = nxt; din = dout;
      }
      *jastrow = cur;  // [Bc][S] scalar rows
    }
    T* Y = X;
    int din = d;
    for (int i = 0; i < cfg.backflow_n; ++i) {
      const int dout = cfg.backflow_dims[i];
      const std::string q = std::to_string(i);
      T* out = (i & 1) ? w.Y1 : w.Y0;
      int rc = gemm(Y, din, ("bfh" + q + ".up").c_str(), ("bfh" + q + ".dn").c_str(), cfg.n_up, dout, P("bfb" + q + ".up"),
                    nullptr, 0, out, dout, Bc * S, dout, din, S, 1, N, st, 0, P("bfb" + q + ".dn"));
      if (rc) return rc;
      DQ_LAUNCH(act_fl_kernel<T>, dim3(groups, (dout + 31) / 32), dim3(32), 0, st, out, dout, (const T*)nullptr, 0, S, dout, T(1), 1);
      Y = out; din = dout;
    }
    *Xbf = Y;
    return 0;
  }

  // softmax attention of layer l on the Q | K | V rows [Bc N S][3d] -> O [Bc N S][d], with the kernel the configuration picks
  // (TransPsiformer: plus the layer's nuclear key / value tokens); *kernel (if given) = that kernel, DQMC_ATTN_KERNEL_*
  int attention(const T* QKV, T* O, int Bc, int S, int l, cudaStream_t st, int32_t* kernel = nullptr) {
    int32_t which = DQMC_ATTN_KERNEL_GENERIC;
    const std::string p = "L" + std::to_string(l) + ".";
    const T scale = (T)(1.0 / std::sqrt((double)dh));
    const int tb = S > 1 ? attn_tb : 1;
    const T* kn = Mn > 0 ? P(p + "kn") : nullptr;
    const T* vn = Mn > 0 ? P(p + "vn") : nullptr;
    if constexpr (std::is_same<T, float>::value) {
      if (S == 1 && attn_mma_ok) {
        which = DQMC_ATTN_KERNEL_MMA;
        // tensor-core attention: a warp per (walker, head, 16-query tile), fragments straight from global memory
        const int n_pairs = Bc * H, tasks = n_pairs * ((N + 15) / 16);
        int nblk = (tasks + 3) / 4;
        if (nblk > n_sms * 8) nblk = n_sms * 8;
        const dim3 grid(nblk), block(128);
#define DQ_ATTN_MMA(NK_)                                                                                                     \
  DQ_LAUNCH(attn_fwd_mma_kernel<NK_>, grid, block, 0, st, (const float*)QKV, 3 * d, (float*)O, d, N, H, d, (float)scale, \
        n_pairs, (const float*)kn, (const float*)vn, Mn)
        switch ((N + Mn + 7) / 8) {
          case 1: DQ_ATTN_MMA(1); break;
          case 2: DQ_ATTN_MMA(2); break;
          case 3: DQ_ATTN_MMA(3); break;
          case 4: DQ_ATTN_MMA(4); break;
          case 5: DQ_ATTN_MMA(5); break;
          default: DQ_ATTN_MMA(6); break;
        }
#undef DQ_ATTN_MMA
      } else if (attn_f32) {
        which = attn_fl_mma && S > 1 ? DQMC_ATTN_KERNEL_FL_F32_MMA : DQMC_ATTN_KERNEL_FL_F32;
        if (launch_attn_f32((const float*)QKV, (float*)O, Bc, S, tb, (float)scale, 0,
                            (int)attn_f32_smem_bytes(N, dh, tb), st, false))
          return 1;
      } else {
        if (attn_gen_mma && S > 1) which = DQMC_ATTN_KERNEL_GENERIC_MMA;
        int rc = launch_attn_generic((const T*)QKV, O, Bc, S, tb, scale, kn, vn, st);
        if (rc) return rc;
      }
    } else {
      int rc = launch_attn_generic((const T*)QKV, O, Bc, S, tb, scale, kn, vn, st);
      if (rc) return rc;
    }
    if (kernel) *kernel = which;
    return 0;
  }

  // what follows the attention of a layer, on [Bc N S] slot rows: A = X + O Wo; M1 = tanh(A W1 + b1); Out = A + tanh(M1 W2 + b2),
  // with the forward-Laplacian propagation of the tanh for S > 1.  A / M1: [Bc N S][d] scratch (unused by the fused block);
  // Out may alias O.  *path (if given) = the path that ran, DQMC_MLP_PATH_*
  int mlp(const std::string& p, const T* O, const T* X, T* Out, T* A, T* M1, int Bc, int S, cudaStream_t st,
          int32_t* path = nullptr) {
    const int rows = Bc * N * S;
    int32_t which;
    if (can_fuse_mlp(S, p)) {
      // plain forward: attention projection + residual and both MLP layers in ONE launch
      which = DQMC_MLP_PATH_BLOCK;
      int rc = mlp_block(p, O, X, Out, rows, st);
      if (rc) return rc;
    } else {
      gemm(O, d, (p + "wo").c_str(), nullptr, 0, d, nullptr, X, d, A, d, rows, d, d, S, 0, N, st);
      if (can_fuse_act(S)) {
        // MLP with the tanh (and its Jacobian/Laplacian propagation) inside the GEMM epilogues
        which = DQMC_MLP_PATH_GEMM_ACT;
        gemm(A, d, (p + "w1").c_str(), nullptr, 0, d, P(p + "b1"), nullptr, 0, M1, d, rows, d, d, S, 0, N, st, 1);
        gemm(M1, d, (p + "w2").c_str(), nullptr, 0, d, P(p + "b2"), A, d, Out, d, rows, d, d, S, 0, N, st, 1);
      } else {
        gemm(A, d, (p + "w1").c_str(), nullptr, 0, d, P(p + "b1"), nullptr, 0, M1, d, rows, d, d, S, 0, N, st);
        which = gemm_on_tc((p + "w1").c_str(), nullptr, d, d, d, nullptr) ? DQMC_MLP_PATH_GEMM_TANH : DQMC_MLP_PATH_SIMT_TANH;
        DQ_LAUNCH(tanh_fl_kernel<T>, dim3(Bc * N, (d + 127) / 128), dim3(128), 0, st, M1, d, (const T*)nullptr, 0, S, d, T(1));
        gemm(M1, d, (p + "w2").c_str(), nullptr, 0, d, P(p + "b2"), nullptr, 0, Out, d, rows, d, d, S, 0, N, st);
        DQ_LAUNCH(tanh_fl_kernel<T>, dim3(Bc * N, (d + 127) / 128), dim3(128), 0, st, Out, d, (const T*)A, d, S, d, T(1));
      }
    }
    if (path) *path = which;
    return 0;
  }

  // one chunk of run_batched: walkers v0 .. v0 + Bc - 1 of its batch
  int run_chunk(const T* r, const T* R, int Rb, int Bc, int S, int Bstat, T* sign, T* logp, T* E, T* stats, T* grad,
                void* wsbase, cudaStream_t st, const FwdIn& in, int64_t v0) {
    Ws w = carve(wsbase, Bc, S);
    const int rows = Bc * N * S;
    const T* qa = nullptr;  // pseudo-Hamiltonian: per-electron metric of the forward-Laplacian pass
    if (in.ph && S > 1) {
      DQ_LAUNCH(ph_coeff_kernel<T>, dim3((Bc * N + 127) / 128), dim3(128), 0, st, r, R, Rb, N, M, ph_args(nullptr), w.QA,
                Bc * N);
      qa = w.QA;
    }
    if (gnn) {
      T* Xbf = nullptr;
      const T* jas = nullptr;
      int rc = paulinet_trunk(r, R, Rb, Bc, S, w, &Xbf, &jas, st, qa);
      if (rc) return rc;
      return tail(r, R, Rb, Bc, S, Bstat, sign, logp, E, stats, grad, w, Xbf, st, in, v0, jas, qa);
    }
    if (cfg.kind == DQMC_FERMINET) {
      T* Xf = nullptr;
      int rc = ferminet_trunk(r, R, Rb, Bc, S, w, &Xf, st, qa);
      if (rc) return rc;
      return tail(r, R, Rb, Bc, S, Bstat, sign, logp, E, stats, grad, w, Xf, st, in, v0, nullptr, qa);
    }
    const int F = 4 * M + 1;
    const bool compact = S == 1 && embed_fwd_ok && in.emb && can_trunk(S);
    if (compact && in.layout != kVirtEcp) {
      // spin swaps: no embedding launch -- the whole-trunk kernel's tile load forms the two swapped rows from the base walkers'
      // table (the embedding is linear in the spin feature)
    } else if (compact) {
      // quadrature forwards of the non-local ECP: only the moved electron's embedding row is new, the whole-trunk kernel
      // takes the other rows from the base walkers' table
      int epb = (Bc / (2 * n_sms)) / 32 * 32;
      epb = epb < 32 ? 32 : (epb > 512 ? 512 : epb);
      DQ_LAUNCH(embed_fwd_kernel<T>, dim3((Bc + epb - 1) / epb), dim3(256), embed_fwd_smem_bytes<T>(M, d), st, r, R, Rb, N,
                M, cfg.n_up, 1, P("emb.w"), d, w.X, Bc, epb, (long long)v0, in.vper, in.pairs);
    } else if (S == 1 && embed_fwd_ok) {
      // plain forwards (Metropolis, ECP quadrature): register-tiled projection, W staged per block
      const int tot = Bc * N;
      int epb = (tot / (2 * n_sms)) / 32 * 32;
      epb = epb < 32 ? 32 : (epb > 512 ? 512 : epb);
      DQ_LAUNCH(embed_fwd_kernel<T>, dim3((tot + epb - 1) / epb), dim3(256), embed_fwd_smem_bytes<T>(M, d), st, r, R, Rb, N,
                M, cfg.n_up, 1, P("emb.w"), d, w.X, tot, epb, 0LL, 0, (const int*)nullptr);
    } else {
      const int epb = S == 1 ? 8 : 1;  // plain forwards: several electrons per block (tiny per-electron work)
      DQ_LAUNCH(embed_kernel<T>, dim3((Bc * N + epb - 1) / epb), dim3(128), sizeof(T) * 5 * F, st, r, R, Rb, N, M,
                cfg.n_up, S, 1, 1, P("emb.w"), d, w.X, Bc * N, epb, qa);
    }
    T* X = w.X;
    T* O = w.O;
    if (can_trunk(S)) {  // plain forward: every layer in one persistent tensor-core launch
      int rc = trunk_block(X, O, rows, st, in, v0);
      if (rc) return rc;
      return tail(r, R, Rb, Bc, S, Bstat, sign, logp, E, stats, grad, w, O, st, in, v0, nullptr, qa);
    }
    for (int l = 0; l < cfg.n_layers; ++l) {
      std::string p = "L" + std::to_string(l) + ".";
      gemm(X, d, (p + "wqkv").c_str(), nullptr, 0, 3 * d, nullptr, nullptr, 0, w.QKV, 3 * d, rows, 3 * d, d, S, 0, N, st);
      int rc = attention(w.QKV, O, Bc, S, l, st);
      if (rc) return rc;
      rc = mlp(p, O, X, O, w.A, w.M1, Bc, S, st);
      if (rc) return rc;
      T* tmp = X; X = O; O = tmp;
    }
    return tail(r, R, Rb, Bc, S, Bstat, sign, logp, E, stats, grad, w, X, st, in, v0, nullptr, qa);
  }

  // Backflow activation -> K signed log-determinants (+ 3N tangents, Laplacian for S > 1), the kernel picked for the shape:
  // BF [Bc N S][BFW] holds the backflow head rows before activation (row (b N + i) S + s) and is activated IN PLACE; Gadd
  // [Bc N][5] receives the additive branch's electron factor.  in.env: the virtual-walker group's envelope table
  // (slater_fwd2_kernel; the chunk's walkers are virtual walkers v0 ..), qa: the pseudo-Hamiltonian metric (slater_kernel),
  // both null outside those passes.  With in.mos set, the chunk's orbital matrices are written there from walker v0 on
  // instead of determinants.  *kernel (if given) = {DQMC_SLATER_KERNEL_*, the template instance NS / NM, 0 for the
  // runtime-N kernels}.  The forward tails and dqmc_debug_slater both call this.
  int slater(const T* r, const T* R, int Rb, int Bc, int S, T* BF, T* Gadd, T* dsign, T* dlog, T* dgrad, T* dlap,
             cudaStream_t st, const T* qa, const FwdIn& in, int64_t v0, int32_t* kernel = nullptr) {
    if (cfg.mult_act == 1)  // default mult_act 1 + 2 tanh(x / 4) of the BackflowOp (nn_wave_function.py:14-33)
      DQ_LAUNCH(act_fl_kernel<T>, dim3(Bc * N, (KN + 127) / 128), dim3(128), 0, st, BF, KN, (const T*)nullptr, 0, S, KN, T(1), 2);
    const int full_det = cfg.factorized_det ? 0 : 1;
    const int mult_on = cfg.backflow_add == 1 ? 0 : 1;
    const T* gadd = nullptr;
    if (cfg.backflow_add) {
      // additive branch (wf/nn_wave_function.py:26-32): add_act on its head, electron-local factor cutoff * |envelope|
      if (qa) { err = "additive backflow with a pseudo-Hamiltonian is not supported"; return 2; }
      DQ_LAUNCH(act_fl_kernel<T>, dim3(Bc * N, (KN + 127) / 128), dim3(128), 0, st, BF + add_off, BFW, (const T*)nullptr, 0, S, KN,
                T(1), 3);
      DQ_LAUNCH(bf_add_factor_kernel<T>, dim3((Bc * N + 63) / 64), dim3(64), 0, st, r, R, Rb, N, M, cfg.n_up, K, P("env.pi_up"),
                P("env.pi_dn"), P("env.zeta_up"), P("env.zeta_dn"), env_rep, full_det, Gadd, Bc * N);
      gadd = Gadd;
    }
    if (in.mos) {  // Ansatz.apply(..., return_mos=True): orbital matrices instead of determinants
      const size_t tot = (size_t)Bc * K * N * N;
      DQ_LAUNCH(orbitals_kernel<T>, dim3((unsigned)((tot + 255) / 256)), dim3(256), 0, st, r, R, Rb, N, M, cfg.n_up, K,
                P("env.pi_up"), P("env.pi_dn"), P("env.zeta_up"), P("env.zeta_dn"), (const T*)BF, BFW, env_rep, full_det,
                in.mos + (size_t)v0 * K * N * N, tot, gadd, add_off, mult_on);
      return 0;
    }
    int32_t which = DQMC_SLATER_KERNEL_GENERIC, inst = 0;
    const int sl_wpb = slater_warps_per_block<T>(N);
    if ((N <= 4 || (N <= 6 && std::is_same<T, float>::value)) && !qa && !gadd && !sw.slater_generic) {
      const int tot = Bc * K;
      which = DQMC_SLATER_KERNEL_SMALL;
#define DQ_SL_SMALL(NS_)                                                                                           \
  inst = NS_;                                                                                                      \
  DQ_LAUNCH((slater_small_kernel<T, NS_>), dim3((tot + 63) / 64), dim3(64), 0, st, r, R, Rb, M, cfg.n_up, K, S, tot,    \
            P("env.pi_up"), P("env.pi_dn"), P("env.zeta_up"), P("env.zeta_dn"), (const T*)BF, KN, dsign, dlog, \
            dgrad, dlap, env_rep, full_det)
      switch (N) {
        case 2: DQ_SL_SMALL(2); break;
        case 3: DQ_SL_SMALL(3); break;
        case 4: DQ_SL_SMALL(4); break;
        case 5: DQ_SL_SMALL(5); break;
        default: DQ_SL_SMALL(6); break;
      }
#undef DQ_SL_SMALL
    } else if (S == 1 && N <= 32 && slater_fwd2_ok && !gadd) {
      const int nthr = 32 * K < 256 ? 32 * K : 256;
      const int grid = Bc < 3 * n_sms ? Bc : 3 * n_sms;
      which = DQMC_SLATER_KERNEL_FWD2;
      // register-resident LU: the row array is sized to the electron count where an exact instance exists (every padded
      // column costs a shuffle + FMA per elimination step)
#define DQ_SL_FWD2(NMV)                                                                                                        \
  inst = NMV;                                                                                                                  \
  DQ_LAUNCH((slater_fwd2_kernel<T, NMV>), dim3(grid), dim3(nthr), slater_fwd2_smem_bytes<T>(N, M, K), st, r, R, Rb, N, M,      \
            cfg.n_up, K, Bc, P("env.pi_up"), P("env.pi_dn"), P("env.zeta_up"), P("env.zeta_dn"), (const T*)BF, KN, dsign,     \
            dlog, env_rep, full_det, in.env, (long long)v0, in.vper, in.layout, in.pairs)
      if (N == 14) { DQ_SL_FWD2(14); }
      else if (N <= 16) { DQ_SL_FWD2(16); }
      else if (N == 28) { DQ_SL_FWD2(28); }
      else if (N == 30) { DQ_SL_FWD2(30); }
      else { DQ_SL_FWD2(32); }
#undef DQ_SL_FWD2
    } else if (S == 1 && N <= 32 && !gadd && !sw.slater_generic) {
      const int wpb = K < 8 ? K : 8;
      which = DQMC_SLATER_KERNEL_FWD_REG;
      DQ_LAUNCH(slater_fwd_reg_kernel<T>, dim3(Bc), dim3(32 * wpb), sizeof(T) * N * M, st, r, R, Rb, N, M, cfg.n_up, K,
                P("env.pi_up"), P("env.pi_dn"), P("env.zeta_up"), P("env.zeta_dn"), (const T*)BF, KN, dsign, dlog,
                env_rep, full_det);
    } else
    DQ_LAUNCH(slater_kernel<T>, dim3((Bc * K + sl_wpb - 1) / sl_wpb), dim3(32 * sl_wpb), slater_smem_bytes<T>(N), st, r, R,
              Rb, N, M, cfg.n_up, K, S, Bc * K, P("env.pi_up"), P("env.pi_dn"), P("env.zeta_up"), P("env.zeta_dn"), (const T*)BF, BFW, dsign, dlog,
              dgrad, dlap, env_rep, full_det, qa, gadd, add_off, mult_on);
    if (kernel) { kernel[0] = which; kernel[1] = inst; }
    return 0;
  }

  // the determinant sum's configuration (finalize_kernel): cusp, ECP and nuclear-cusp terms as the engine was created
  FinalizeCfg finalize_cfg(int S) const {
    FinalizeCfg fc;
    fc.N = N; fc.M = M; fc.n_up = cfg.n_up; fc.K = K; fc.S = S; fc.cusp_kind = cfg.cusp_kind;
    fc.cusp_same_scale = cfg.cusp_same_scale; fc.cusp_anti_scale = cfg.cusp_anti_scale;
    fc.ecp_terms = cfg.ecp_loc_terms;
    fc.nuc_cusp_kind = cfg.nuc_cusp_kind;
    return fc;
  }

  // backflow heads -> Slater determinants -> det sum / cusp / potentials (shared by all trunks)
  int tail(const T* r, const T* R, int Rb, int Bc, int S, int Bstat, T* sign, T* logp, T* E, T* stats, T* grad, Ws& w,
           T* X, cudaStream_t st, const FwdIn& in, int64_t v0, const T* jastrow = nullptr, const T* qa = nullptr) {
    // per-spin backflow heads: rows of electron e across walkers, weights by spin
    gemm(X, bf_in, "bf.up", "bf.dn", cfg.n_up, BFW, gnn ? P("bfb.up") : nullptr, nullptr, 0, w.BF, BFW, Bc * S, BFW, bf_in, S, 1, N,
         st, 0, gnn ? P("bfb.dn") : nullptr);
    int rc = slater(r, R, Rb, Bc, S, w.BF, w.Gadd, w.dsign, w.dlog, w.dgrad, w.dlap, st, qa, in, v0);
    if (rc || in.mos) return rc;
    const FinalizeCfg fc = finalize_cfg(S);
    DQ_LAUNCH(finalize_kernel<T>, dim3(Bc), dim3(128), finalize_smem_bytes<T>(N, K), st, fc, r, R, Rb,
              (const T*)w.dsign, (const T*)w.dlog, (const T*)w.dgrad, (const T*)w.dlap, P("cusp.alpha"),
              (const T*)d_zval, (const T*)d_ecp_loc, (const int*)d_ecp_mask, Bstat, sign, logp, E, stats, grad,
              cfg.conf_linear ? P("conf.w") : (const T*)nullptr, jastrow,
              cfg.nuc_cusp_kind ? P("cusp.nuc") : (const T*)nullptr, qa ? ph_args(qa) : PhArgs<T>());
    return 0;
  }

  int run_batched(const T* r, const T* R, int Rb, int B, int S, T* sign, T* logp, T* E, T* stats, T* grad, void* ws,
                  int64_t wsb, cudaStream_t st, const FwdIn& in = {}) {
    int Bc = max_chunk(wsb, S, B);
    if (Bc < 1) { err = "workspace too small for a single walker"; return 3; }
    if (chunk_bytes(Bc, S) > wsb) { err = "internal: carved workspace exceeds the planned size"; return 3; }
    if (dry) { carve(ws, Bc, S); return 0; }  // planning pass: record the extent of the largest chunk
    for (int b0 = 0; b0 < B; b0 += Bc) {
      int nb = std::min(Bc, B - b0);
      int rc = run_chunk(r + (size_t)b0 * 3 * N, R + (Rb ? (size_t)b0 * 3 * M : 0), Rb, nb, S, B, sign ? sign + b0 : nullptr,
                         logp ? logp + b0 : nullptr, E ? E + b0 : nullptr, stats ? stats + b0 : nullptr,
                         grad ? grad + (size_t)b0 * T3 : nullptr, ws, st, in, b0);
      if (rc) return rc;
      rc = check_guards();
      if (rc) return rc;
    }
    return 0;
  }

  // ---- Metropolis-adjusted Langevin sweep (SURVEY.md 8(f) N3): value + drift from the forward-Laplacian pass ----
  // state = {r, sign, log, force}; force == clean_force(grad log|psi|) with the CURRENT tau (electron_samplers.py:197-211)
  int value_and_force(const T* r, const T* R, int Rb, int B, const T* tau, T* sign, T* logp, T* force, void* ws, int64_t wsb,
                      cudaStream_t st) {
    Arena a(this, ws, wsb);
    const ForceBufs f = carve_force(a, B);
    if (a.left() < 0) { err = "workspace too small (Langevin force buffers)"; return 3; }
    FwdIn in;
    in.ph = false;  // the drift is the gradient of log|psi| alone (electron_samplers.py:201-209): no pseudo-Hamiltonian metric
    int rc = run_batched(r, R, Rb, B, T3 + 2, sign, logp, f.E, f.stats, f.grad, a.top, a.left(), st, in);
    if (rc) return rc;
    DQ_LAUNCH(langevin_force_kernel<T>, dim3((B * N + 127) / 128), dim3(128), 0, st, (const T*)f.grad, r, R, Rb, (const T*)d_znuc,
              tau, N, M, B * N, force);
    return 0;
  }
  int langevin(void* r_, void* sign_, void* logp_, void* force_, int32_t* age, void* tau_, const void* R_, int Rb, int B, int n_sub,
               double target, int max_age, uint64_t seed, uint64_t step0, uint64_t woff, const void* nn, const void* nu,
               void* stats_, void* ws, int64_t wsb, cudaStream_t st) override {
    T* r = (T*)r_; T* sign = (T*)sign_; T* logp = (T*)logp_; T* force = (T*)force_; T* tau = (T*)tau_; T* stats = (T*)stats_;
    const T* R = (const T*)R_;
    if (n_sub == 0) return langevin_update(r, R, Rb, B, tau, sign, logp, force, ws, wsb, st);
    Arena a(this, ws, wsb);
    const Proposals q = carve_proposals(a, B, true);
    if (a.left() < 0) { err = "workspace too small (Langevin proposal buffers)"; return 3; }
    DQ_CHECK(cudaMemsetAsync(q.cnt, 0, sizeof(int), st));
    const int ne = B * 3 * N;
    for (int s = 0; s < n_sub; ++s) {
      const T* nns = nn ? (const T*)nn + (size_t)s * ne : nullptr;
      const T* nus = nu ? (const T*)nu + (size_t)s * B : nullptr;
      DQ_LAUNCH(langevin_propose_kernel<T>, dim3((ne / 2 + 1 + 127) / 128), dim3(128), 0, st, (const T*)r, (const T*)force, q.r,
                (const T*)tau, nns, seed, step0 + (uint64_t)s, woff * (uint64_t)(3 * N), ne);
      int rc = value_and_force(q.r, R, Rb, B, tau, q.sign, q.logp, q.force, a.top, a.left(), st);
      if (rc) return rc;
      DQ_LAUNCH(langevin_accept_kernel<T>, dim3((B + 127) / 128), dim3(128), 0, st, r, (const T*)q.r, force, (const T*)q.force,
                sign, (const T*)q.sign, logp, (const T*)q.logp, age, (const T*)tau, nus, seed, step0 + (uint64_t)s, woff, max_age, B,
                N, q.cnt);
      DQ_LAUNCH(tau_kernel<T>, dim3(1), dim3(32), 0, st, tau, q.cnt, B, (T)target, stats);
    }
    DQ_LAUNCH(sampler_stats_kernel<T>, dim3(1), dim3(256), 0, st, (const T*)r, (const T*)logp, (const int*)age, (const T*)tau, B,
              N, stats);
    DQ_CHECK(cudaGetLastError());
    return check_guards();  // the proposal buffers' guards, after the last accept (and with n_sub == 0)
  }
  // n_sub == 0 with force output: (re)compute psi and the drift of the current walkers (sampler.update)
  int langevin_update(const T* r, const T* R, int Rb, int B, const T* tau, T* sign, T* logp, T* force, void* ws, int64_t wsb,
                      cudaStream_t st) {
    int rc = value_and_force(r, R, Rb, B, tau, sign, logp, force, ws, wsb, st);
    if (rc) return rc;
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  // ---- parameter VJP of the plain forward (Psiformer): SURVEY.md 8(f) N1 ------------------------
  const T* PT(const std::string& n) const { return d_params_t + off(n); }
  // entry n's slot in the parameter cotangent G; null when G is (the position mode accumulates no parameter gradients)
  T* PG(T* G, const std::string& n) const { return G ? G + off(n) : nullptr; }
  // C = (Res) + A @ W with a raw weight pointer (CUDA-core kernel; used by the reverse pass with transposed weights)
  int gemm_raw(const T* A, int lda, const T* W0, const T* W1, int zsplit, int ldw, const T* Res, int ldr, T* C, int ldc,
               int Mr, int Nc, int Kc, int sliced, cudaStream_t st) {
    GemmArgs<T> g;
    g.A = A; g.lda = lda; g.W0 = W0; g.W1 = W1; g.z_split = zsplit; g.ldw = ldw; g.bias = nullptr; g.Res = Res;
    g.ldr = ldr; g.C = C; g.ldc = ldc; g.M = Mr; g.N = Nc; g.K = Kc; g.S = 1; g.sliced = sliced; g.Nel = N;
    constexpr int BM = 64, BN = 64, BK = 16, TM = 4, TN = 4;
    dim3 grid((Nc + BN - 1) / BN, (Mr + BM - 1) / BM, sliced ? N : 1);
    DQ_LAUNCH((gemm_kernel<T, BM, BN, BK, TM, TN>), grid, dim3(256), 0, st, g);
    return 0;
  }
  // dW += A^T dY over `rows` rows, db += column sums.  The rows are (walker, electron i) pairs; [lo, hi) selects electrons
  // lo <= i < hi of every walker (the per-spin heads), hi = ALL_ROWS takes every row.  An empty selection (a spin block with
  // no electrons) accumulates nothing, and so does a null dW / db (PG in the position mode).
  static constexpr int ALL_ROWS = -1;
  void wgrad(const T* A, int lda, const T* dY, int ldy, int rows, int Kc, int Nc, T* dW, int lo, int hi, cudaStream_t st) {
    if (!dW || (hi != ALL_ROWS && hi <= lo)) return;
    int nz = (rows + 4095) / 4096;
    if (nz > 256) nz = 256;
    if (nz < 1) nz = 1;
    const int rpb = ((rows + nz - 1) / nz + 31) / 32 * 32;
    DQ_LAUNCH(gemm_tn_kernel<T>, dim3((Nc + 31) / 32, (Kc + 31) / 32, (rows + rpb - 1) / rpb), dim3(256), 0, st, A, lda, dY, ldy,
              rows, Kc, Nc, rpb, hi == ALL_ROWS ? 0 : N, lo, hi, dW, Nc);
  }
  void bgrad(const T* dZ, int ld, int rows, int Nc, T* db, cudaStream_t st, int lo = 0, int hi = ALL_ROWS) {
    if (!db || (hi != ALL_ROWS && hi <= lo)) return;
    int ny = (rows + 2047) / 2048;
    if (ny > 128) ny = 128;
    if (ny < 1) ny = 1;
    const int rpb = (rows + ny - 1) / ny;
    DQ_LAUNCH(colsum_kernel<T>, dim3((Nc + 127) / 128, (rows + rpb - 1) / rpb), dim3(128), 0, st, dZ, ld, rows, Nc, rpb, db,
              hi == ALL_ROWS ? 0 : N, lo, hi);
  }

  // Position mode of the reverse passes (dqmc_wf_grad_positions): cotangent 1 per walker, no parameter gradients, the chain
  // carried on into the electron-nucleus features, the envelopes and the cusps.  gr [Bc][N][3] / gR [Bc][M][3] nullable.
  struct PosOut { T* gr; T* gR; };
  // pair-cotangent buffers of the position mode: per-(walker, determinant) envelope shares and their per-walker sum
  struct PosBufs { T *cpart = nullptr, *cbuf = nullptr; };
  PosBufs carve_pos(Arena& a, int Bc) const {
    PosBufs p;
    p.cpart = a.take<T>((size_t)Bc * K * N * M * 3);
    p.cbuf = a.take<T>((size_t)Bc * N * M * 3);
    return p;
  }
  void launch_pos_reduce(const T* r, const T* R, int Rb, int Bc, const PosBufs& pb, const T* dFeat, int ldf, int log_rescale,
                         const T* dE, const PosOut* po, cudaStream_t st) {
    DQ_LAUNCH(pos_grad_reduce_kernel<T>, dim3(Bc), dim3(128), 0, st, r, R, Rb, N, M, cfg.n_up, K, (const T*)pb.cpart, dFeat, ldf,
              log_rescale, dE, cfg.cusp_kind, (T)cfg.cusp_same_scale, (T)cfg.cusp_anti_scale, P("cusp.alpha"), cfg.nuc_cusp_kind,
              cfg.nuc_cusp_kind ? P("cusp.nuc") : (const T*)nullptr, pb.cbuf, po->gr, po->gR);
  }

  // slater_bwd_kernel's launch: as many warps per block (1 ... 4) as fit 96 KiB of dynamic shared memory.  The launch and
  // the shared-memory opt-in both take it from here, so the opt-in always covers the launch (DESIGN §8).
  int slater_bwd_shape(int& wpb, size_t& smem) {
    const size_t pw = slater_bwd_smem_per_warp<T>(N);
    wpb = (int)((96 * 1024) / pw);
    wpb = wpb < 1 ? 1 : (wpb > 4 ? 4 : wpb);
    smem = pw * wpb;
    if (smem > 227 * 1024) { err = "system too large for the shared-memory tiling of the reverse pass (N)"; return 2; }
    return 0;
  }

  // Determinant head of the reverse passes, from the backflow output BF [Bc N][KN] to its cotangent dBF: determinants and
  // their sum (sign, logp), then back through both.  The conv-GNN kinds' spin-factorised determinants, hk.Linear determinant
  // weights and Jastrow (jastrow: the Jastrow tape's output, null without one) follow from cfg.  G null: position mode, no
  // parameter gradients; cpart: its pair-cotangent buffer (null otherwise).
  int det_head_bwd(const T* r, const T* R, int Rb, int Bc, const T* BF, T* dBF, const T* wts, T* sign, T* logp, T* G,
                   const T* jastrow, T* cpart, Arena& a, cudaStream_t st) {
    T* dsign = a.take<T>((size_t)Bc * K); T* dlog = a.take<T>((size_t)Bc * K); T* dld = a.take<T>((size_t)Bc * K);
    if (a.left() < 0) { err = "internal: reverse-pass buffers exceed the planned workspace"; return 3; }
    int wpb;
    size_t smem;
    int rc = slater_bwd_shape(wpb, smem);
    if (rc) return rc;
    const int full_det = cfg.factorized_det ? 0 : 1;
    const T* conf = cfg.conf_linear ? P("conf.w") : nullptr;
    const T* nuc = cfg.nuc_cusp_kind ? P("cusp.nuc") : nullptr;
    const int sl_wpb = slater_warps_per_block<T>(N);
    DQ_LAUNCH(slater_kernel<T>, dim3((Bc * K + sl_wpb - 1) / sl_wpb), dim3(32 * sl_wpb), slater_smem_bytes<T>(N), st, r, R, Rb, N,
              M, cfg.n_up, K, 1, Bc * K, P("env.pi_up"), P("env.pi_dn"), P("env.zeta_up"), P("env.zeta_dn"), BF, KN, dsign, dlog,
              (T*)nullptr, (T*)nullptr, env_rep, full_det, (const T*)nullptr, (const T*)nullptr, 0, 1);
    FinalizeCfg fc = finalize_cfg(1);
    fc.ecp_terms = 0;  // sign and log only: no local energy, no ECP table
    DQ_LAUNCH(finalize_kernel<T>, dim3(Bc), dim3(128), finalize_smem_bytes<T>(N, K), st, fc, r, R, Rb, (const T*)dsign,
              (const T*)dlog, (const T*)nullptr, (const T*)nullptr, P("cusp.alpha"), (const T*)d_zval, (const T*)nullptr,
              (const int*)d_ecp_mask, Bc, sign, logp, (T*)nullptr, (T*)nullptr, (T*)nullptr, conf, jastrow, nuc, PhArgs<T>());
    // ---- reverse ------------------------------------------------------------------------------------------------
    // the conv-GNN kinds pass cusp kind 0 (fixed cusp exponent: no gradient)
    DQ_LAUNCH(finalize_bwd_kernel<T>, dim3((Bc + 127) / 128), dim3(128), 0, st, r, N, cfg.n_up, K, Bc, (const T*)dsign,
              (const T*)dlog, wts, gnn ? 0 : cfg.cusp_kind, (T)cfg.cusp_same_scale, (T)cfg.cusp_anti_scale, P("cusp.alpha"), dld,
              gnn ? (T*)nullptr : PG(G, "cusp.alpha"), R, Rb, M, cfg.nuc_cusp_kind, nuc,
              cfg.nuc_cusp_kind ? PG(G, "cusp.nuc") : (T*)nullptr, conf, cfg.conf_linear ? PG(G, "conf.w") : (T*)nullptr);
    DQ_LAUNCH(slater_bwd_kernel<T>, dim3((Bc * K + wpb - 1) / wpb), dim3(32 * wpb), smem, st, r, R, Rb, N, M, cfg.n_up, K, Bc * K,
              P("env.pi_up"), P("env.pi_dn"), P("env.zeta_up"), P("env.zeta_dn"), BF, KN, (const T*)dld, dBF, PG(G, "env.pi_up"),
              PG(G, "env.pi_dn"), PG(G, "env.zeta_up"), PG(G, "env.zeta_dn"), env_rep, full_det, cpart);
    return 0;
  }
  // linear backflow heads of the Psiformer kinds and FermiNet: dX_L = dBF W_spin^T, dW_spin += X_L[spin rows]^T dBF[spin rows]
  void bf_head_bwd(const T* XL, const T* dBF, T* dXL, int Bc, T* G, cudaStream_t st) {
    gemm_raw(dBF, KN, PT("bf.up"), PT("bf.dn"), cfg.n_up, d, nullptr, 0, dXL, d, Bc, d, KN, 1, st);
    wgrad(XL, d, dBF, KN, Bc * N, d, KN, PG(G, "bf.up"), 0, cfg.n_up, st);
    wgrad(XL, d, dBF, KN, Bc * N, d, KN, PG(G, "bf.dn"), cfg.n_up, N, st);
  }

  // Softmax attention backward of layer `layer` (plain forward, one slot), one block per (walker, head): QKV / dQKV rows
  // [Bc N][3d], dO [Bc N][d].  With nuclear tokens (TransPsiformer) the cotangents of their keys / values are accumulated
  // over walkers into dKn / dVn [Mn][d] (null: not wanted).  vjp_chunk and dqmc_debug_attention_bwd both run this.
  int attention_bwd(int layer, const T* QKV, const T* dO, T* dQKV, int Bc, T* dKn, T* dVn, cudaStream_t st) {
    const std::string q = "L" + std::to_string(layer) + ".";
    const size_t smem = attn_bwd_smem_bytes<T>(N, dh, Mn);
    if (smem > 227 * 1024) { err = "system too large for the shared-memory tiling of the attention reverse pass (N)"; return 2; }
    DQ_CHECK(raise_dyn_smem(attn_bwd_kernel<T>, (int)smem));
    DQ_LAUNCH(attn_bwd_kernel<T>, dim3(Bc, H), dim3(128), smem, st, QKV, 3 * d, dO, d, N, dh, d, (T)(1.0 / std::sqrt((double)dh)),
              dQKV, Mn > 0 ? P(q + "kn") : (const T*)nullptr, Mn > 0 ? P(q + "vn") : (const T*)nullptr, Mn, dKn, dVn);
    return 0;
  }

  int vjp_chunk(const T* r, const T* R, int Rb, int Bc, const T* wts, T* sign, T* logp, T* G, Arena a, cudaStream_t st,
                const PosOut* po) {
    const int L = cfg.n_layers, rows = Bc * N, F = 4 * M + 1;
    std::vector<T*> X(L + 1), QKV(L), O(L), A(L), M1(L);
    for (int l = 0; l <= L; ++l) X[l] = a.take<T>((size_t)rows * d);
    for (int l = 0; l < L; ++l) { QKV[l] = a.take<T>((size_t)rows * 3 * d); O[l] = a.take<T>((size_t)rows * d); A[l] = a.take<T>((size_t)rows * d); M1[l] = a.take<T>((size_t)rows * d); }
    T* BF = a.take<T>((size_t)rows * KN); T* dBF = a.take<T>((size_t)rows * KN);
    T* dXn = a.take<T>((size_t)rows * d); T* dZ = a.take<T>((size_t)rows * d); T* dM1 = a.take<T>((size_t)rows * d);
    T* dA = a.take<T>((size_t)rows * d); T* dO = a.take<T>((size_t)rows * d); T* dQKV = a.take<T>((size_t)rows * 3 * d);
    T* dX = a.take<T>((size_t)rows * d); T* Feat = a.take<T>((size_t)rows * F);
    const PosBufs pb = po ? carve_pos(a, Bc) : PosBufs();
    if (a.left() < 0) { err = "internal: reverse-pass buffers exceed the planned workspace"; return 3; }
    const T scale = (T)(1.0 / std::sqrt((double)dh));
    // ---- forward with every layer's activations kept --------------------------------------------------------
    DQ_LAUNCH(embed_kernel<T>, dim3((rows + 7) / 8), dim3(128), sizeof(T) * 5 * F, st, r, R, Rb, N, M, cfg.n_up, 1, 1, 1,
              P("emb.w"), d, X[0], rows, 8, (const T*)nullptr);
    for (int l = 0; l < L; ++l) {
      const std::string q = "L" + std::to_string(l) + ".";
      gemm(X[l], d, (q + "wqkv").c_str(), nullptr, 0, 3 * d, nullptr, nullptr, 0, QKV[l], 3 * d, rows, 3 * d, d, 1, 0, N, st);
      const T* kn = Mn > 0 ? P(q + "kn") : nullptr;
      const T* vn = Mn > 0 ? P(q + "vn") : nullptr;
      DQ_LAUNCH(attn_fl_kernel<T>, dim3(Bc, H), dim3(128), attn_smem_bytes<T>(N, dh, 1, Mn), st, (const T*)QKV[l], 3 * d, O[l], d, N,
                1, dh, d, scale, 1, kn, vn, Mn);
      gemm(O[l], d, (q + "wo").c_str(), nullptr, 0, d, nullptr, X[l], d, A[l], d, rows, d, d, 1, 0, N, st);
      gemm(A[l], d, (q + "w1").c_str(), nullptr, 0, d, P(q + "b1"), nullptr, 0, M1[l], d, rows, d, d, 1, 0, N, st);
      DQ_LAUNCH(tanh_fl_kernel<T>, dim3(rows, (d + 127) / 128), dim3(128), 0, st, M1[l], d, (const T*)nullptr, 0, 1, d, T(1));
      gemm(M1[l], d, (q + "w2").c_str(), nullptr, 0, d, P(q + "b2"), nullptr, 0, X[l + 1], d, rows, d, d, 1, 0, N, st);
      DQ_LAUNCH(tanh_fl_kernel<T>, dim3(rows, (d + 127) / 128), dim3(128), 0, st, X[l + 1], d, (const T*)A[l], d, 1, d, T(1));
    }
    gemm(X[L], d, "bf.up", "bf.dn", cfg.n_up, KN, nullptr, nullptr, 0, BF, KN, Bc, KN, d, 1, 1, N, st);
    int rc = det_head_bwd(r, R, Rb, Bc, BF, dBF, wts, sign, logp, G, nullptr, pb.cpart, a, st);
    if (rc) return rc;
    bf_head_bwd(X[L], dBF, dXn, Bc, G, st);
    const size_t nel = (size_t)rows * d;
    for (int l = L - 1; l >= 0; --l) {
      const std::string q = "L" + std::to_string(l) + ".";
      // X_{l+1} = A + tanh(M1 W2 + b2)
      DQ_LAUNCH(tanh_bwd_kernel<T>, dim3((unsigned)((nel + 255) / 256)), dim3(256), 0, st, (const T*)dXn, (const T*)X[l + 1],
                (const T*)A[l], dZ, nel);
      bgrad(dZ, d, rows, d, PG(G, q + "b2"), st);
      wgrad(M1[l], d, dZ, d, rows, d, d, PG(G, q + "w2"), 0, ALL_ROWS, st);
      gemm_raw(dZ, d, PT(q + "w2"), nullptr, 0, d, nullptr, 0, dM1, d, rows, d, d, 0, st);
      // M1 = tanh(A W1 + b1)
      DQ_LAUNCH(tanh_bwd_kernel<T>, dim3((unsigned)((nel + 255) / 256)), dim3(256), 0, st, (const T*)dM1, (const T*)M1[l],
                (const T*)nullptr, dZ, nel);
      bgrad(dZ, d, rows, d, PG(G, q + "b1"), st);
      wgrad(A[l], d, dZ, d, rows, d, d, PG(G, q + "w1"), 0, ALL_ROWS, st);
      gemm_raw(dZ, d, PT(q + "w1"), nullptr, 0, d, dXn, d, dA, d, rows, d, d, 0, st);  // dA = dX_{l+1} + dZ1 W1^T
      // A = X + O Wo
      wgrad(O[l], d, dA, d, rows, d, d, PG(G, q + "wo"), 0, ALL_ROWS, st);
      gemm_raw(dA, d, PT(q + "wo"), nullptr, 0, d, nullptr, 0, dO, d, rows, d, d, 0, st);
      rc = attention_bwd(l, QKV[l], dO, dQKV, Bc, Mn > 0 ? PG(G, q + "kn") : (T*)nullptr, Mn > 0 ? PG(G, q + "vn") : (T*)nullptr, st);
      if (rc) return rc;
      wgrad(X[l], d, dQKV, 3 * d, rows, d, 3 * d, PG(G, q + "wqkv"), 0, ALL_ROWS, st);
      gemm_raw(dQKV, 3 * d, PT(q + "wqkv"), nullptr, 0, d, dA, d, dX, d, rows, d, 3 * d, 0, st);  // dX_l = dA + dQKV Wqkv^T
      T* t = dXn; dXn = dX; dX = t;
    }
    if (po) {  // dFeat = dX0 W_emb^T (the spin column is not read), then features, envelopes and cusps per walker
      gemm_raw(dXn, d, PT("emb.w"), nullptr, 0, F, nullptr, 0, Feat, F, rows, F, d, 0, st);
      launch_pos_reduce(r, R, Rb, Bc, pb, Feat, F, 1, (const T*)nullptr, po, st);
      return 0;
    }
    DQ_LAUNCH(embed_feat_kernel<T>, dim3((rows * M + 127) / 128), dim3(128), 0, st, r, R, Rb, N, M, cfg.n_up, Feat, rows);
    wgrad(Feat, F, dXn, d, rows, F, d, G + off("emb.w"), 0, ALL_ROWS, st);
    return 0;
  }

  // FermiNet reverse pass (conf/ansatz/ferminet.yaml): node update g on concat[h, spin means of h, spin means of the
  // incoming edges], shared edge MLP u, residuals / sqrt(2).  The raw input features carry no parameters, so the
  // parameter chain stops at the first layer's weights; the position mode carries it on to the raw node and edge features.
  int vjp_chunk_ferminet(const T* r, const T* R, int Rb, int Bc, const T* wts, T* sign, T* logp, T* G, Arena a,
                         cudaStream_t st, const PosOut* po) {
    const int L = cfg.n_layers, rows = Bc * N, rowsE = Bc * N * N, de = cfg.edge_dim, d0 = 4 * M;
    const T isq2 = (T)0.70710678118654752440;
    std::vector<T*> Hs(L + 1), Es(L), Fs(L);
    std::vector<int> dH(L + 1), dEd(L);
    dH[0] = d0;
    for (int l = 1; l <= L; ++l) dH[l] = d;
    for (int l = 0; l < L; ++l) dEd[l] = l == 0 ? 4 : de;
    for (int l = 0; l <= L; ++l) Hs[l] = a.take<T>((size_t)rows * dH[l]);
    for (int l = 0; l < L; ++l) { Es[l] = a.take<T>((size_t)rowsE * dEd[l]); Fs[l] = a.take<T>((size_t)rows * (3 * dH[l] + 2 * dEd[l])); }
    const int fmax = 3 * (d > d0 ? d : d0) + 2 * (de > 4 ? de : 4);
    T* BF = a.take<T>((size_t)rows * KN); T* dBF = a.take<T>((size_t)rows * KN);
    const int dx = po ? std::max(d, d0) : d, dex = po ? std::max(de, 4) : de;  // the position mode reaches layer 0's inputs
    T* dXa = a.take<T>((size_t)rows * dx); T* dXb = a.take<T>((size_t)rows * dx); T* dZ = a.take<T>((size_t)rows * d);
    T* dF = a.take<T>((size_t)rows * fmax);
    T* dEa = a.take<T>((size_t)rowsE * dex); T* dEb = a.take<T>((size_t)rowsE * dex); T* dZe = a.take<T>((size_t)rowsE * de);
    const PosBufs pb = po ? carve_pos(a, Bc) : PosBufs();
    if (a.left() < 0) { err = "internal: reverse-pass buffers exceed the planned workspace"; return 3; }
    // ---- forward, activations kept -----------------------------------------------------------------------------
    DQ_LAUNCH(embed_kernel<T>, dim3(Bc * N), dim3(128), sizeof(T) * 5 * d0, st, r, R, Rb, N, M, cfg.n_up, 1, 0, 0,
              (const T*)nullptr, d0, Hs[0], Bc * N, 1, (const T*)nullptr);
    DQ_LAUNCH(edge_feat_kernel<T>, dim3((rowsE + 127) / 128), dim3(128), 0, st, r, N, 1, Es[0], rowsE, (const T*)nullptr);
    for (int l = 0; l < L; ++l) {
      const std::string q = "F" + std::to_string(l) + ".";
      const int dc = dH[l], ec = dEd[l], fin = 3 * dc + 2 * ec;
      DQ_LAUNCH(fermi_agg_kernel<T>, dim3(Bc, N), dim3(128), 0, st, (const T*)Hs[l], dc, (const T*)Es[l], ec, N, cfg.n_up, 1, Fs[l]);
      int rc = gemm(Fs[l], fin, (q + "wg").c_str(), nullptr, 0, d, P(q + "bg"), nullptr, 0, Hs[l + 1], d, rows, d, fin, 1, 0, N, st);
      if (rc) return rc;
      DQ_LAUNCH(tanh_fl_kernel<T>, dim3(rows, (d + 127) / 128), dim3(128), 0, st, Hs[l + 1], d,
                (const T*)(dc == d ? Hs[l] : nullptr), dc, 1, d, dc == d ? isq2 : T(1));
      if (l < L - 1) {
        rc = gemm(Es[l], ec, (q + "wu").c_str(), nullptr, 0, de, P(q + "bu"), nullptr, 0, Es[l + 1], de, rowsE, de, ec, 1, 0, N, st);
        if (rc) return rc;
        DQ_LAUNCH(tanh_fl_kernel<T>, dim3(rowsE, 1), dim3(32), 0, st, Es[l + 1], de, (const T*)(ec == de ? Es[l] : nullptr), ec,
                  1, de, ec == de ? isq2 : T(1));
      }
    }
    gemm(Hs[L], d, "bf.up", "bf.dn", cfg.n_up, KN, nullptr, nullptr, 0, BF, KN, Bc, KN, d, 1, 1, N, st);
    int rc = det_head_bwd(r, R, Rb, Bc, BF, dBF, wts, sign, logp, G, nullptr, pb.cpart, a, st);
    if (rc) return rc;
    T* dHn = dXa;   // gradient w.r.t. H_{l+1}
    T* dHc = dXb;   // gradient w.r.t. H_l (being built)
    T* dEn = dEa;   // gradient w.r.t. E_{l+1} (valid for l < L - 1)
    T* dEc = dEb;
    bf_head_bwd(Hs[L], dBF, dHn, Bc, G, st);
    for (int l = L - 1; l >= 0; --l) {
      const std::string q = "F" + std::to_string(l) + ".";
      const int dc = dH[l], ec = dEd[l], fin = 3 * dc + 2 * ec;
      const bool res_h = dc == d, res_e = ec == de;
      const size_t nel = (size_t)rows * d;
      // H_{l+1} = s (H_l + tanh(F Wg + bg))  |  tanh(F Wg + bg)
      DQ_LAUNCH(tanh_res_bwd_kernel<T>, dim3((unsigned)((nel + 255) / 256)), dim3(256), 0, st, (const T*)dHn, (const T*)Hs[l + 1],
                (const T*)(res_h ? Hs[l] : nullptr), res_h ? isq2 : T(1), dZ, nel);
      bgrad(dZ, d, rows, d, PG(G, q + "bg"), st);
      wgrad(Fs[l], fin, dZ, d, rows, fin, d, PG(G, q + "wg"), 0, ALL_ROWS, st);
      if (l > 0 || po) {
        gemm_raw(dZ, d, PT(q + "wg"), nullptr, 0, fin, nullptr, 0, dF, fin, rows, fin, d, 0, st);
        DQ_LAUNCH(fermi_agg_bwd_kernel<T>, dim3(Bc, N), dim3(128), 0, st, (const T*)dF, dc, ec, N, cfg.n_up,
                  (const T*)(res_h ? dHn : nullptr), isq2, dHc, dEc, 0);
      }
      if (l < L - 1) {
        // E_{l+1} = s (E_l + tanh(E_l Wu + bu))  |  tanh(E_l Wu + bu)
        const size_t nee = (size_t)rowsE * de;
        DQ_LAUNCH(tanh_res_bwd_kernel<T>, dim3((unsigned)((nee + 255) / 256)), dim3(256), 0, st, (const T*)dEn, (const T*)Es[l + 1],
                  (const T*)(res_e ? Es[l] : nullptr), res_e ? isq2 : T(1), dZe, nee);
        bgrad(dZe, de, rowsE, de, PG(G, q + "bu"), st);
        wgrad(Es[l], ec, dZe, de, rowsE, ec, de, PG(G, q + "wu"), 0, ALL_ROWS, st);
        if (l > 0 || po) {
          gemm_raw(dZe, de, PT(q + "wu"), nullptr, 0, ec, dEc, ec, dEc, ec, rowsE, ec, de, 0, st);  // dE_l += dZe Wu^T
          if (res_e) {
            const size_t ne2 = (size_t)rowsE * ec;
            DQ_LAUNCH(axpy_kernel<T>, dim3((unsigned)((ne2 + 255) / 256)), dim3(256), 0, st, (const T*)dEn, isq2, dEc, ne2);
          }
        }
      }
      T* t1 = dHn; dHn = dHc; dHc = t1;
      T* t2 = dEn; dEn = dEc; dEc = t2;
    }
    if (po) launch_pos_reduce(r, R, Rb, Bc, pb, dHn, d0, 0, dEn, po, st);  // dH_0 [rows][4 M], dE_0 [rows N][4]
    return 0;
  }
  // ---- conv-GNN reverse pass: the reference's test ansatz (tests/conf/ansatz.yaml: hk.Embed embeddings, 'featurewise'
  // update over same / anti / ne convolutions, no deep edge features), Jastrow and per-spin backflow MLPs (ssp), default
  // mult_act, spin-factorised determinants, hk.Linear determinant weights.  Value layouts of kernels_bwd.cuh.
  struct Tape {
    std::vector<T*> a;     // a[0] input, a[k] output of layer k (after its activation)
    std::vector<int> dim;  // widths
    int lda0 = 0;          // row stride of the input a[0] (its first dim[0] columns are the input)
  };
  int tape_fwd(const T* in, int din, const int* dims, int nl, const std::string& base, bool bias, int act, bool last_linear,
               int rows_, Arena& a, Tape& t, cudaStream_t st, int lda = 0) {
    t.a.assign(1, const_cast<T*>(in));
    t.dim.assign(1, din);
    t.lda0 = lda > 0 ? lda : din;
    for (int i = 0; i < nl; ++i) {
      T* out = a.take<T>((size_t)rows_ * dims[i]);
      const std::string q = base + std::to_string(i);
      const bool b_i = bias && (!last_linear || base[0] != 'J' || i < nl - 1);  // Jastrow: bias 'not_last'
      int rc = gemm(t.a.back(), i == 0 ? t.lda0 : t.dim.back(), (q + ".w").c_str(), nullptr, 0, dims[i], b_i ? P(q + ".b") : nullptr, nullptr, 0, out,
                    dims[i], rows_, dims[i], t.dim.back(), 1, 0, 1, st);
      if (rc) return rc;
      if (i < nl - 1 || !last_linear)
        DQ_LAUNCH(act_fl_kernel<T>, dim3(rows_, (dims[i] + 63) / 64), dim3(64), 0, st, out, dims[i], (const T*)nullptr, 0, 1, dims[i],
                  T(1), act);
      t.a.push_back(out);
      t.dim.push_back(dims[i]);
    }
    return 0;
  }
  // dY = gradient w.r.t. the tape's output (destroyed).  s0 / s1: scratch of rows_ x max width.  dIn (nullable) receives
  // (accumulate: is increased by) the gradient w.r.t. the tape's input.
  int tape_bwd(const Tape& t, T* dY, const std::string& base, bool bias, int act, bool last_linear, int rows_, T* s0, T* s1,
               T* dIn, bool accumulate, T* G, cudaStream_t st) {
    const int nl = (int)t.a.size() - 1;
    T* cur = dY;
    for (int i = nl - 1; i >= 0; --i) {
      const int dout = t.dim[i + 1], din = t.dim[i];
      const std::string q = base + std::to_string(i);
      const size_t n = (size_t)rows_ * dout;
      if (i < nl - 1 || !last_linear)
        DQ_LAUNCH(act_bwd_kernel<T>, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, cur, (const T*)t.a[i + 1], act, n);
      const bool b_i = bias && (!last_linear || base[0] != 'J' || i < nl - 1);
      if (b_i) bgrad(cur, dout, rows_, dout, G + off(q + ".b"), st);
      const int lda = i == 0 ? t.lda0 : din;
      wgrad(t.a[i], lda, cur, dout, rows_, din, dout, G + off(q + ".w"), 0, ALL_ROWS, st);
      if (i > 0) {
        T* nxt = (cur == s0) ? s1 : s0;
        gemm_raw(cur, dout, PT(q + ".w"), nullptr, 0, din, nullptr, 0, nxt, din, rows_, din, dout, 0, st);
        cur = nxt;
      } else if (dIn) {  // dIn has the input's row stride; its columns past din are left alone
        gemm_raw(cur, dout, PT(q + ".w"), nullptr, 0, din, accumulate ? dIn : nullptr, lda, dIn, lda, rows_, din, dout, 0, st);
      }
    }
    return 0;
  }
  int vjp_chunk_paulinet(const T* r, const T* R, int Rb, int Bc, const T* wts, T* sign, T* logp, T* G, Arena a,
                         cudaStream_t st) {
    const int L = cfg.n_layers, rows = Bc * N, e = cfg.edge_dim, nl = cfg.gnn_sub_n > 0 ? cfg.gnn_sub_n : 1;
    const int Mne = cfg.gnn_conv_ne ? M : 0, NS = N + Mne, nt = cfg.gnn_conv_ne ? 3 : 2, pairs = Bc * N * NS;
    const int n_types = cfg.n_elec_types > 0 ? cfg.n_elec_types : 1;
    const bool deep = cfg.gnn_deep_edges != 0;
    const T isq2 = (T)0.70710678118654752440;
    const char* tn[3] = {"same", "anti", "ne"};
    // ---- forward, everything kept --------------------------------------------------------------------------------
    std::vector<T*> X(L + 1), C(L), Fc(L), E(L);
    std::vector<int> xd(L + 1), ed(L);
    std::vector<std::array<T*, 3>> Gt(L);
    std::vector<std::array<Tape, 3>> Wt(L);
    std::vector<std::array<Tape, 2>> Ht(L);
    std::vector<Tape> Ut(L);
    std::vector<std::array<Tape, 3>> Us(L);  // deep_features 'separate': one u tape per edge type
    const bool dw = cfg.gnn_ne_identity != 0, sep = cfg.gnn_sep_edges != 0;
    xd[0] = cfg.gnn_features ? 4 * M : d;
    X[0] = a.take<T>((size_t)rows * xd[0]);
    if (cfg.gnn_features)  // raw nucleus-electron features [|d|, d]: no parameters
      DQ_LAUNCH(embed_kernel<T>, dim3(rows), dim3(128), sizeof(T) * 5 * xd[0], st, r, R, Rb, N, M, cfg.n_up, 1, 0, 0, (const T*)nullptr,
                xd[0], X[0], rows, 1, (const T*)nullptr);
    else
      DQ_LAUNCH(gnn_embed_kernel<T>, dim3((rows * d + 127) / 128), dim3(128), 0, st, P("emb.table"), n_types, N, cfg.n_up, 1, d, X[0], rows);
    E[0] = a.take<T>((size_t)pairs * 4);
    ed[0] = 4;
    DQ_LAUNCH(gnn_edge_val_kernel<T>, dim3((pairs + 127) / 128), dim3(128), 0, st, r, R, Rb, N, M, Mne, E[0], pairs,
              cfg.gnn_self_edges);
    for (int l = 0; l < L; ++l) {
      const std::string q = "G" + std::to_string(l) + ".";
      for (int t = 0; t < nt; ++t) {
        if (t == 2 && dw) continue;  // identity ne filter
        int rc = tape_fwd(E[l], gnn_ein(t, l), cfg.gnn_w_dims[l], nl, q + "w_" + tn[t] + ".", cfg.gnn_w_bias != 0, 0, false, pairs,
                          a, Wt[l][t], st, ed[l]);
        if (rc) return rc;
      }
      for (int t = 0; t < 2; ++t) {
        int rc = tape_fwd(X[l], xd[l], cfg.gnn_h_dims[l], nl, q + "h_" + tn[t] + ".", true, 0, false, rows, a, Ht[l][t], st);
        if (rc) return rc;
      }
      const int dconv = gnn_conv_w(l);
      C[l] = a.take<T>((size_t)rows * dconv);
      if (dw)
        DQ_LAUNCH(gnn_conv_val_dw_kernel<T>, dim3(rows), dim3(64), 0, st, (const T*)Wt[l][0].a.back(), (const T*)Wt[l][1].a.back(),
                  (const T*)E[l], ed[l], gnn_hne_w(l), (const T*)Ht[l][0].a.back(), (const T*)Ht[l][1].a.back(), P(q + "hne"), N,
                  Mne, cfg.n_up, e, cfg.gnn_self_edges, C[l]);
      else
        DQ_LAUNCH(gnn_conv_val_kernel<T>, dim3(rows), dim3(64), 0, st, (const T*)Wt[l][0].a.back(), (const T*)Wt[l][1].a.back(),
                  (const T*)(nt == 3 ? Wt[l][2].a.back() : nullptr), (const T*)Ht[l][0].a.back(), (const T*)Ht[l][1].a.back(),
                  nt == 3 ? P(q + "hne") : (const T*)nullptr, N, Mne, cfg.n_up, e, C[l]);
      xd[l + 1] = d;
      if (cfg.gnn_concat) {  // x <- [(x +) tanh(g([x, mean_up x, mean_down x, conv_*]))] (/ sqrt 2)
        const int fin = 3 * xd[l] + dconv;
        Fc[l] = a.take<T>((size_t)rows * fin);
        DQ_LAUNCH(gnn_concat_kernel<T>, dim3(Bc, N), dim3(128), 0, st, (const T*)X[l], xd[l], (const T*)C[l], dconv, N, cfg.n_up, 1, Fc[l]);
        X[l + 1] = a.take<T>((size_t)rows * d);
        int rc = gemm(Fc[l], fin, (q + "g.w").c_str(), nullptr, 0, d, cfg.gnn_g_bias ? P(q + "g.b") : nullptr, nullptr, 0, X[l + 1], d,
                      rows, d, fin, 1, 0, N, st);
        if (rc) return rc;
        const bool res = xd[l] == d && !cfg.gnn_no_res;
        DQ_LAUNCH(act_fl_kernel<T>, dim3(rows, (d + 63) / 64), dim3(64), 0, st, X[l + 1], d, res ? (const T*)X[l] : (const T*)nullptr, d, 1,
                  d, (res && cfg.gnn_res_norm) ? isq2 : T(1), 0);
      } else {  // featurewise: x <- x + sum_t tanh(g_t(conv_t)); each G_t holds the running sum
        const T* res = xd[l] == d ? X[l] : nullptr;
        for (int t = 0; t < nt; ++t) {
          Gt[l][t] = a.take<T>((size_t)rows * d);
          int rc = gemm(C[l] + t * e, nt * e, (q + "g_" + tn[t] + ".w").c_str(), nullptr, 0, d, P(q + "g_" + tn[t] + ".b"), nullptr, 0,
                        Gt[l][t], d, rows, d, e, 1, 0, N, st);
          if (rc) return rc;
          DQ_LAUNCH(act_fl_kernel<T>, dim3(rows, (d + 63) / 64), dim3(64), 0, st, Gt[l][t], d, res, d, 1, d, T(1), 0);
          res = Gt[l][t];
        }
        if (cfg.gnn_res_norm) { err = "dqmc_wf_vjp_params: normalised featurewise residual not supported"; return 2; }
        X[l + 1] = Gt[l][nt - 1];
      }
      if (deep && l < L - 1 && sep) {  // one u per edge type, each pair keeps its own type's (electron_gnn.py:176-188)
        int res_mask = 0;
        for (int t = 0; t < nt; ++t) {
          int rc = tape_fwd(E[l], gnn_ein(t, l), cfg.gnn_u_dims[l], nl, q + "u_" + tn[t] + ".", true, 0, false, pairs, a, Us[l][t], st,
                            ed[l]);
          if (rc) return rc;
          if (gnn_ein(t, l) == e && ed[l] == e) res_mask |= 1 << t;
        }
        ed[l + 1] = e;
        E[l + 1] = a.take<T>((size_t)pairs * e);
        DQ_LAUNCH((gnn_edge_select_kernel<T>), dim3((unsigned)(((size_t)pairs * e + 255) / 256)), dim3(256), 0, st, (const T*)E[l],
                  (const T*)Us[l][0].a.back(), (const T*)Us[l][1].a.back(), (const T*)(nt == 3 ? Us[l][2].a.back() : nullptr), 1, N,
                  Mne, cfg.n_up, e, res_mask, isq2, E[l + 1], (size_t)pairs * e);
      } else if (deep && l < L - 1) {  // shared edge MLP u + normalised residual (electron_gnn.py:160-192)
        int rc = tape_fwd(E[l], ed[l], cfg.gnn_u_dims[l], nl, q + "u.", true, 0, false, pairs, a, Ut[l], st);
        if (rc) return rc;
        ed[l + 1] = e;
        if (ed[l] == e) {
          E[l + 1] = a.take<T>((size_t)pairs * e);
          DQ_LAUNCH((axpby_kernel<T>), dim3((unsigned)(((size_t)pairs * e + 255) / 256)), dim3(256), 0, st, (const T*)E[l],
                    (const T*)Ut[l].a.back(), isq2, E[l + 1], (size_t)pairs * e);
        } else {
          E[l + 1] = Ut[l].a.back();
        }
      } else if (l < L - 1) {
        E[l + 1] = E[l]; ed[l + 1] = ed[l];
      }
    }
    // Jastrow on sum_i x_i
    Tape Jt;
    T* Js = nullptr;
    if (cfg.jastrow_n > 0) {
      Js = a.take<T>((size_t)Bc * d);
      DQ_LAUNCH(sum_electrons_kernel<T>, dim3((Bc * d + 127) / 128), dim3(128), 0, st, (const T*)X[L], N, 1, d, Js, Bc * d);
      int rc = tape_fwd(Js, d, cfg.jastrow_dims, cfg.jastrow_n, "J", true, 1, true, Bc, a, Jt, st);
      if (rc) return rc;
    }
    // per-spin backflow MLPs: hidden layers (ssp), then the orbital head (+ default mult_act)
    std::vector<T*> Y(cfg.backflow_n + 1);
    std::vector<int> yd(cfg.backflow_n + 1);
    Y[0] = X[L]; yd[0] = d;
    for (int i = 0; i < cfg.backflow_n; ++i) {
      const int dout = cfg.backflow_dims[i];
      const std::string q = std::to_string(i);
      Y[i + 1] = a.take<T>((size_t)rows * dout); yd[i + 1] = dout;
      int rc = gemm(Y[i], yd[i], ("bfh" + q + ".up").c_str(), ("bfh" + q + ".dn").c_str(), cfg.n_up, dout, P("bfb" + q + ".up"), nullptr,
                    0, Y[i + 1], dout, Bc, dout, yd[i], 1, 1, N, st, 0, P("bfb" + q + ".dn"));
      if (rc) return rc;
      DQ_LAUNCH(act_fl_kernel<T>, dim3(rows, (dout + 31) / 32), dim3(32), 0, st, Y[i + 1], dout, (const T*)nullptr, 0, 1, dout, T(1), 1);
    }
    T* BF = a.take<T>((size_t)rows * KN); T* dBF = a.take<T>((size_t)rows * KN);
    int rc = gemm(Y.back(), yd.back(), "bf.up", "bf.dn", cfg.n_up, KN, P("bfb.up"), nullptr, 0, BF, KN, Bc, KN, yd.back(), 1, 1, N, st, 0,
                  P("bfb.dn"));
    if (rc) return rc;
    if (cfg.mult_act == 1)
      DQ_LAUNCH(act_fl_kernel<T>, dim3(rows, (KN + 127) / 128), dim3(128), 0, st, BF, KN, (const T*)nullptr, 0, 1, KN, T(1), 2);
    rc = det_head_bwd(r, R, Rb, Bc, BF, dBF, wts, sign, logp, G, cfg.jastrow_n > 0 ? (const T*)Jt.a.back() : nullptr, nullptr,
                      a, st);
    if (rc) return rc;
    // scratch for the reverse sweep
    const int xm = std::max(d, xd[0]);
    const int hm = std::max(gnn_hmax(), xm), hn = std::max(gnn_hnode_max(), e), em = gnn_emax();
    int fmax = 0, cmax = 0;
    for (int l = 0; l < L; ++l) { fmax = std::max(fmax, 3 * xd[l] + gnn_conv_w(l)); cmax = std::max(cmax, gnn_conv_w(l)); }
    T* dXa = a.take<T>((size_t)rows * xm); T* dXb = a.take<T>((size_t)rows * xm);
    T* sr0 = a.take<T>((size_t)rows * std::max(hm, hn)); T* sr1 = a.take<T>((size_t)rows * std::max(hm, hn));
    T* dCb = a.take<T>((size_t)rows * cmax); T* dCt = a.take<T>((size_t)rows * e);
    T* dFb = cfg.gnn_concat ? a.take<T>((size_t)rows * fmax) : nullptr;
    T* dWb[3] = {a.take<T>((size_t)pairs * e), a.take<T>((size_t)pairs * e), a.take<T>((size_t)pairs * e)};
    T* sp0 = a.take<T>((size_t)pairs * em); T* sp1 = a.take<T>((size_t)pairs * em);
    T* dHb[2] = {a.take<T>((size_t)rows * e), a.take<T>((size_t)rows * e)};
    T* dEa = deep ? a.take<T>((size_t)pairs * e) : nullptr;
    T* dEb = deep ? a.take<T>((size_t)pairs * e) : nullptr;
    T* dUb = deep ? a.take<T>((size_t)pairs * e) : nullptr;
    T* dUs[3] = {dUb, sep ? a.take<T>((size_t)pairs * e) : nullptr, sep && nt == 3 ? a.take<T>((size_t)pairs * e) : nullptr};
    // orbital head
    if (cfg.mult_act == 1) {
      const size_t n = (size_t)rows * KN;
      DQ_LAUNCH(act_bwd_kernel<T>, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, dBF, (const T*)BF, 2, n);
    }
    bgrad(dBF, KN, rows, KN, G + off("bfb.up"), st, 0, cfg.n_up);
    bgrad(dBF, KN, rows, KN, G + off("bfb.dn"), st, cfg.n_up, N);
    wgrad(Y.back(), yd.back(), dBF, KN, rows, yd.back(), KN, G + off("bf.up"), 0, cfg.n_up, st);
    wgrad(Y.back(), yd.back(), dBF, KN, rows, yd.back(), KN, G + off("bf.dn"), cfg.n_up, N, st);
    T* cur = cfg.backflow_n > 0 ? sr0 : dXa;
    gemm_raw(dBF, KN, PT("bf.up"), PT("bf.dn"), cfg.n_up, yd.back(), nullptr, 0, cur, yd.back(), Bc, yd.back(), KN, 1, st);
    for (int i = cfg.backflow_n - 1; i >= 0; --i) {
      const int dout = yd[i + 1], din = yd[i];
      const std::string q = std::to_string(i);
      const size_t n = (size_t)rows * dout;
      DQ_LAUNCH(act_bwd_kernel<T>, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, cur, (const T*)Y[i + 1], 1, n);
      bgrad(cur, dout, rows, dout, G + off("bfb" + q + ".up"), st, 0, cfg.n_up);
      bgrad(cur, dout, rows, dout, G + off("bfb" + q + ".dn"), st, cfg.n_up, N);
      wgrad(Y[i], din, cur, dout, rows, din, dout, G + off("bfh" + q + ".up"), 0, cfg.n_up, st);
      wgrad(Y[i], din, cur, dout, rows, din, dout, G + off("bfh" + q + ".dn"), cfg.n_up, N, st);
      T* nxt = i == 0 ? dXa : (cur == sr0 ? sr1 : sr0);
      gemm_raw(cur, dout, PT("bfh" + q + ".up"), PT("bfh" + q + ".dn"), cfg.n_up, din, nullptr, 0, nxt, din, Bc, din, dout, 1, st);
      cur = nxt;
    }
    T* dXn = dXa;  // gradient w.r.t. X_L
    T* dXc = dXb;
    if (cfg.jastrow_n > 0) {  // d log|psi| / d jastrow = w_b
      T* dJ = a.take<T>((size_t)Bc);  // [Bc] scalars
      T* js0 = a.take<T>((size_t)Bc * d); T* js1 = a.take<T>((size_t)Bc * d); T* dJs = a.take<T>((size_t)Bc * d);
      DQ_CHECK(cudaMemcpyAsync(dJ, wts, sizeof(T) * Bc, cudaMemcpyDeviceToDevice, st));
      tape_bwd(Jt, dJ, "J", true, 1, true, Bc, js0, js1, dJs, false, G, st);
      const size_t n = (size_t)rows * d;
      DQ_LAUNCH(bcast_add_kernel<T>, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, (const T*)dJs, N, d, dXn, n);
    }
    T* dEn = dEa;  // gradient w.r.t. E_{l+1} (deep edge features only)
    T* dEc = dEb;
    for (int l = L - 1; l >= 0; --l) {
      const std::string q = "G" + std::to_string(l) + ".";
      const size_t nd = (size_t)rows * d;
      const bool need_dx = l > 0 || !cfg.gnn_features;  // layer 0 of the raw-feature variant has nothing trainable upstream
      if (cfg.gnn_concat) {
        const int dconv = gnn_conv_w(l), fin = 3 * xd[l] + dconv;
        const bool res = xd[l] == d && !cfg.gnn_no_res;
        const T sc = (res && cfg.gnn_res_norm) ? isq2 : T(1);
        DQ_LAUNCH(tanh_res_bwd_kernel<T>, dim3((unsigned)((nd + 255) / 256)), dim3(256), 0, st, (const T*)dXn, (const T*)X[l + 1],
                  (const T*)(res ? X[l] : nullptr), sc, sr0, nd);
        if (cfg.gnn_g_bias) bgrad(sr0, d, rows, d, G + off(q + "g.b"), st);
        wgrad(Fc[l], fin, sr0, d, rows, fin, d, G + off(q + "g.w"), 0, ALL_ROWS, st);
        gemm_raw(sr0, d, PT(q + "g.w"), nullptr, 0, fin, nullptr, 0, dFb, fin, rows, fin, d, 0, st);
        // dF -> dX_l (own row + spin means + residual) and dC (the convolution columns); F = [x, mean_up, mean_down, conv_*]
        if (nt != 2 && !dw) { err = "dqmc_wf_vjp_params: concatenate update with nucleus-electron convolutions not supported"; return 2; }
        DQ_LAUNCH(fermi_agg_bwd_kernel<T>, dim3(Bc, N), dim3(128), 0, st, (const T*)dFb, xd[l], e, N, cfg.n_up,
                  (const T*)(res ? dXn : nullptr), sc, dXc, (T*)nullptr, fin);
        const size_t nc = (size_t)rows * dconv;
        DQ_LAUNCH(slice_cols_kernel<T>, dim3((unsigned)((nc + 255) / 256)), dim3(256), 0, st, (const T*)dFb, fin, 3 * xd[l], dconv, dCb, nc);
      } else {
        // X_{l+1} = X_l + sum_t tanh(z_t): tanh outputs are the differences of the running sums
        if (xd[l] == d) DQ_CHECK(cudaMemcpyAsync(dXc, dXn, sizeof(T) * nd, cudaMemcpyDeviceToDevice, st));  // residual
        else DQ_CHECK(cudaMemsetAsync(dXc, 0, sizeof(T) * (size_t)rows * xd[l], st));
        for (int t = 0; t < nt; ++t) {
          const T* prev = t == 0 ? (xd[l] == d ? X[l] : nullptr) : Gt[l][t - 1];
          DQ_LAUNCH(tanh_bwd_kernel<T>, dim3((unsigned)((nd + 255) / 256)), dim3(256), 0, st, (const T*)dXn, (const T*)Gt[l][t], prev, sr0, nd);
          bgrad(sr0, d, rows, d, G + off(q + "g_" + tn[t] + ".b"), st);
          const size_t ne_ = (size_t)rows * e;  // conv_t is a column slice of C: copy it out for the weight gradient
          DQ_LAUNCH(slice_cols_kernel<T>, dim3((unsigned)((ne_ + 255) / 256)), dim3(256), 0, st, (const T*)C[l], nt * e, t * e, e, dCt, ne_);
          wgrad(dCt, e, sr0, d, rows, e, d, G + off(q + "g_" + tn[t] + ".w"), 0, ALL_ROWS, st);
          gemm_raw(sr0, d, PT(q + "g_" + tn[t] + ".w"), nullptr, 0, e, nullptr, 0, dCb + t * e, nt * e, rows, e, d, 0, st);
        }
      }
      DQ_CHECK(cudaMemsetAsync(dHb[0], 0, sizeof(T) * (size_t)rows * e, st));
      DQ_CHECK(cudaMemsetAsync(dHb[1], 0, sizeof(T) * (size_t)rows * e, st));
      // gradient w.r.t. this layer's edge features E_l (only the deep-edge variant carries it; E_0 has nothing upstream)
      const bool need_de = deep && l > 0;
      if (need_de) DQ_CHECK(cudaMemsetAsync(dEc, 0, sizeof(T) * (size_t)pairs * ed[l], st));
      if (dw)
        DQ_LAUNCH(gnn_conv_bwd_dw_kernel<T>, dim3(rows), dim3(64), 0, st, (const T*)dCb, (const T*)Wt[l][0].a.back(),
                  (const T*)Wt[l][1].a.back(), (const T*)E[l], ed[l], gnn_hne_w(l), (const T*)Ht[l][0].a.back(),
                  (const T*)Ht[l][1].a.back(), P(q + "hne"), N, Mne, cfg.n_up, e, cfg.gnn_self_edges, dWb[0], dWb[1],
                  need_de ? dEc : (T*)nullptr, dHb[0], dHb[1], G + off(q + "hne"));
      else
        DQ_LAUNCH(gnn_conv_bwd_kernel<T>, dim3(rows), dim3(64), 0, st, (const T*)dCb, (const T*)Wt[l][0].a.back(),
                  (const T*)Wt[l][1].a.back(), (const T*)(nt == 3 ? Wt[l][2].a.back() : nullptr), (const T*)Ht[l][0].a.back(),
                  (const T*)Ht[l][1].a.back(), nt == 3 ? P(q + "hne") : (const T*)nullptr, N, Mne, cfg.n_up, e, dWb[0], dWb[1], dWb[2],
                  dHb[0], dHb[1], nt == 3 ? G + off(q + "hne") : (T*)nullptr);
      for (int t = 0; t < nt; ++t)
        if (!(t == 2 && dw)) tape_bwd(Wt[l][t], dWb[t], q + "w_" + tn[t] + ".", cfg.gnn_w_bias != 0, 0, false, pairs, sp0, sp1, need_de ? dEc : nullptr, true, G, st);
      for (int t = 0; t < 2; ++t)
        tape_bwd(Ht[l][t], dHb[t], q + "h_" + tn[t] + ".", true, 0, false, rows, sr0, sr1, need_dx ? dXc : nullptr, true, G, st);
      if (deep && l < L - 1 && sep) {  // E_{l+1} = per pair s (E_l + u_t(E_l)) | u_t(E_l) of its type t
        int res_mask = 0;
        for (int t = 0; t < nt; ++t)
          if (gnn_ein(t, l) == e && ed[l] == e) res_mask |= 1 << t;
        const size_t ne2 = (size_t)pairs * e;
        DQ_LAUNCH(gnn_edge_select_bwd_kernel<T>, dim3((unsigned)((ne2 + 255) / 256)), dim3(256), 0, st, (const T*)dEn, N, Mne, cfg.n_up,
                  e, res_mask, isq2, dUs[0], dUs[1], dUs[2], need_de ? dEc : (T*)nullptr, ne2);
        for (int t = 0; t < nt; ++t)
          tape_bwd(Us[l][t], dUs[t], q + "u_" + tn[t] + ".", true, 0, false, pairs, sp0, sp1, need_de ? dEc : nullptr, true, G, st);
      } else if (deep && l < L - 1) {  // E_{l+1} = s (E_l + u(E_l))  |  u(E_l); dEn holds the gradient w.r.t. E_{l+1}
        const bool res_e = ed[l] == e;
        const size_t ne2 = (size_t)pairs * e;
        DQ_LAUNCH((axpby_kernel<T>), dim3((unsigned)((ne2 + 255) / 256)), dim3(256), 0, st, (const T*)dEn, (const T*)dEn, res_e ? isq2 / T(2) : T(0.5),
                  dUb, ne2);  // dU = s dE_{l+1}
        tape_bwd(Ut[l], dUb, q + "u.", true, 0, false, pairs, sp0, sp1, need_de ? dEc : nullptr, true, G, st);
        if (need_de && res_e) DQ_LAUNCH(axpy_kernel<T>, dim3((unsigned)((ne2 + 255) / 256)), dim3(256), 0, st, (const T*)dEn, isq2, dEc, ne2);
      }
      T* tmp = dXn; dXn = dXc; dXc = tmp;
      T* tmq = dEn; dEn = dEc; dEc = tmq;
    }
    if (!cfg.gnn_features)
      DQ_LAUNCH(embed_table_bwd_kernel<T>, dim3((d + 63) / 64, 64), dim3(64), 0, st, (const T*)dXn, n_types, N, cfg.n_up, d, rows,
                G + off("emb.table"));
    if (a.left() < 0) { err = "internal: reverse-pass buffers exceed the planned workspace"; return 3; }
    return 0;
  }

  // one reverse-pass chunk of the engine's kind; po: position mode (Psiformer kinds and FermiNet only)
  int reverse_chunk(const T* r, const T* R, int Rb, int Bc, const T* wts, T* sign, T* logp, T* G, const Arena& a,
                    cudaStream_t st, const PosOut* po) {
    if (gnn) return vjp_chunk_paulinet(r, R, Rb, Bc, wts, sign, logp, G, a, st);
    if (cfg.kind == DQMC_FERMINET) return vjp_chunk_ferminet(r, R, Rb, Bc, wts, sign, logp, G, a, st, po);
    return vjp_chunk(r, R, Rb, Bc, wts, sign, logp, G, a, st, po);
  }

  // The reverse pass over B walkers in chunks: activations of every layer stay resident for the reverse pass, so a chunk is
  // the largest one whose buffers (a dry pass of the chunk function) fit the caller's workspace.  po: position mode, its
  // outputs from walker 0 on (wts and G null there); what: the entry point the workspace refusal names.
  int reverse_pass(const T* r, const T* R, int Rb, int B, const T* wts, T* sign, T* logp, T* G, const PosOut* po, void* ws,
                   int64_t wsb, cudaStream_t st, const char* what) {
    // (not const: nvcc 12.9's front end aborts on a const local initialised through this lambda)
    int64_t Bc = largest_fit(B, wsb, [&](int64_t n) { return vjp_chunk_bytes((int)n, po != nullptr); });
    if (Bc < 1) { err = std::string("workspace too small for a single walker (") + what + ")"; return 3; }
    if (!gnn && cfg.kind != DQMC_FERMINET) {
      // the chunk's forward runs the generic attention with one slot, which fp32 engines on the specialised kernels never
      // opted in at creation (benzene, N = 30, dh = 64: 69 KB)
      DQ_CHECK(raise_dyn_smem(attn_fl_kernel<T>, (int)attn_smem_bytes<T>(N, dh, 1, Mn)));
    }
    int wpb;
    size_t smem;
    int rc = slater_bwd_shape(wpb, smem);
    if (rc) return rc;
    DQ_CHECK(raise_dyn_smem(slater_bwd_kernel<T>, (int)smem));
    for (int b0 = 0; b0 < B; b0 += (int)Bc) {
      const int nb = (int)std::min<int64_t>(Bc, B - b0);
      PosOut pc{nullptr, nullptr};
      if (po) pc = {po->gr ? po->gr + (size_t)b0 * 3 * N : nullptr, po->gR ? po->gR + (size_t)b0 * 3 * M : nullptr};
      rc = reverse_chunk(r + (size_t)b0 * 3 * N, R + (Rb ? (size_t)b0 * 3 * M : 0), Rb, nb, wts ? wts + b0 : nullptr, sign + b0,
                         logp + b0, G, Arena(this, ws, wsb), st, po ? &pc : nullptr);
      if (rc) return rc;
      rc = check_guards();
      if (rc) return rc;
      if (dry) break;  // planning pass: the first chunk is the largest
    }
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  int vjp_params(const void* r, const void* R, int Rb, int B, const void* weights, void* sign, void* logp,
                 void* grad_params, void* ws, int64_t wsb, cudaStream_t st) override {
    if (cfg.backflow_add) { err = "dqmc_wf_vjp_params: additive backflow branch has no reverse pass"; return 2; }
    DQ_CHECK(cudaMemsetAsync(grad_params, 0, sizeof(T) * total, st));
    if (B == 0) return 0;  // empty batch: zero gradient
    return reverse_pass((const T*)r, (const T*)R, Rb, B, (const T*)weights, (T*)sign, (T*)logp, (T*)grad_params, nullptr, ws,
                        wsb, st, "vjp");
  }

  // d log|psi| / d r and / d R per walker: the parameter reverse pass in its position mode, chunked like vjp_params
  int grad_positions(const void* r, const void* R, int Rb, int B, void* sign, void* logp, void* grad_r, void* grad_R, void* ws,
                     int64_t wsb, cudaStream_t st) override {
    if (gnn) { err = "dqmc_wf_grad_positions: the conv-GNN kinds have no position reverse pass"; return 2; }
    if (cfg.backflow_add) { err = "dqmc_wf_grad_positions: additive backflow branch has no reverse pass"; return 2; }
    if (cfg.kind == DQMC_TRANSPSIFORMER && grad_R) {
      err = "dqmc_wf_grad_positions: the TransPsiformer's nuclear tokens and envelope exponents depend on R through the host-side "
            "nuclear stream; only grad_r is available (out_grad_R must be null)";
      return 2;
    }
    if (B == 0) return 0;
    const PosOut po{(T*)grad_r, (T*)grad_R};
    return reverse_pass((const T*)r, (const T*)R, Rb, B, nullptr, (T*)sign, (T*)logp, nullptr, &po, ws, wsb, st, "grad_positions");
  }

  // closed-form force terms per walker (force_terms_kernel); all-electron Hamiltonians only
  int force_terms(const void* r, const void* R, int Rb, int B, const void* grad_r, void* bare, void* zvq, void* Q,
                  cudaStream_t st) override {
    if (J > 0 || cfg.ecp_loc_terms > 0 || d_ph_tabs) {
      err = "dqmc_force_terms: effective core potentials and pseudo-Hamiltonians are not supported (all-electron only)";
      return 2;
    }
    if (zvq && !grad_r) { err = "dqmc_force_terms: out_zvq needs grad_r"; return 2; }
    if (B == 0) return 0;
    DQ_LAUNCH(force_terms_kernel<T>, dim3(B), dim3(32), 0, st, (const T*)r, (const T*)R, Rb, N, M, (const T*)d_zval,
              (const T*)grad_r, (T*)bare, (T*)zvq, (T*)Q, (const T*)nullptr, 0);
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  // ---- AC-ZV force term: nuclear-coordinate companion of the forward-Laplacian pass (kernels_zv.cuh) ----------------
  // Companion buffers of one chunk of Bc walkers, carved in front of the primal forward chunk (carve()): the companion rows
  // of the trunk (X, O, QKV and for the Psiformer A, M1) and of the backflow heads, the determinants' companions zl [Bc K],
  // zg [Bc K T3], zlap [Bc K], and the primal outputs the companion pass reads or finalize_kernel writes (sign, log, E,
  // stats [6][Bc], grad [Bc T3]).
  struct ZvWs { T *X, *O, *QKV, *A, *M1, *BF, *zl, *zg, *zlap, *sign, *logp, *E, *stats, *grad; };
  ZvWs carve_zv(Arena& a, int Bc) const {
    ZvWs z;
    const size_t rows = (size_t)Bc * N * (T3 + 2);
    if (cfg.kind == DQMC_FERMINET) {
      const size_t dm = fermi_dmax(), fin = 3 * dm + 2 * fermi_emax();
      z.X = a.take<T>(rows * dm); z.O = a.take<T>(rows * dm); z.QKV = a.take<T>(rows * fin);
      z.A = z.M1 = nullptr;
    } else {
      z.X = a.take<T>(rows * d); z.O = a.take<T>(rows * d); z.QKV = a.take<T>(rows * 3 * d);
      z.A = a.take<T>(rows * d); z.M1 = a.take<T>(rows * d);
    }
    z.BF = a.take<T>(rows * BFW);
    z.zl = a.take<T>((size_t)Bc * K); z.zg = a.take<T>((size_t)Bc * K * T3); z.zlap = a.take<T>((size_t)Bc * K);
    z.sign = a.take<T>(Bc); z.logp = a.take<T>(Bc); z.E = a.take<T>(Bc); z.stats = a.take<T>((size_t)6 * Bc);
    z.grad = a.take<T>((size_t)Bc * T3);
    return z;
  }
  int64_t zv_chunk_bytes(int Bc) const {
    return prefixed_bytes([&](Arena& a) { carve_zv(a, Bc); }, Bc, T3 + 2);
  }
  // why dqmc_zv_force refuses this engine (null: it does not)
  const char* zv_refusal() const {
    if (trans) return "the TransPsiformer's nuclear tokens and envelope exponents depend on R through the host-side nuclear stream";
    if (gnn) return "the conv-GNN kinds have no nuclear companion pass";
    if (cfg.kind != DQMC_PSIFORMER && cfg.kind != DQMC_FERMINET) return "Psiformer and FermiNet only";
    if (cfg.backflow_add) return "the additive backflow branch has no nuclear companion pass";
    if (J > 0 || cfg.ecp_loc_terms > 0) return "effective core potentials are not supported (all-electron only)";
    if (d_ph_tabs || ph_on) return "pseudo-Hamiltonians are not supported (all-electron only)";
    return nullptr;
  }

  // one chunk, one nuclear coordinate kappa = (m, c): the primal forward-Laplacian pass (its dense layers without fused
  // epilogues, so that every pre-activation is there for its companion rule) and the companion pass beside it.  Writes
  // zv[b][kappa] (and gR[b][kappa]) with row stride 3 M.
  int zv_chunk(const T* r, const T* R, int Rb, int Bc, int kappa, const ZvWs& z, Ws& w, T* zv, T* gR, cudaStream_t st) {
    const int S = T3 + 2, rows = Bc * N * S, m = kappa / 3, c = kappa % 3;
    const T isq2 = (T)0.70710678118654752440;
    const dim3 blk(128);
    T* X;
    T* Xd;
    int rc;
    if (cfg.kind == DQMC_FERMINET) {
      const int de = cfg.edge_dim, d0 = 4 * M;
      DQ_LAUNCH(embed_kernel<T>, dim3(Bc * N), blk, sizeof(T) * 5 * d0, st, r, R, Rb, N, M, cfg.n_up, S, 0, 0, (const T*)nullptr,
                d0, w.X, Bc * N, 1, (const T*)nullptr);
      DQ_LAUNCH(zv_embed_kernel<T>, dim3(Bc * N), blk, 0, st, r, R, Rb, N, M, S, 0, (const T*)nullptr, d0, z.X, Bc * N, m, c);
      DQ_LAUNCH(edge_feat_kernel<T>, dim3((Bc * N * N + 127) / 128), blk, 0, st, r, N, S, w.A, Bc * N * N, (const T*)nullptr);
      T *Hc = w.X, *Hn = w.O, *Ec = w.A, *En = w.M1, *Hcd = z.X, *Hnd = z.O;
      int dcur = d0, ecur = 4;
      for (int l = 0; l < cfg.n_layers; ++l) {
        const std::string p = "F" + std::to_string(l) + ".";
        const int fin = 3 * dcur + 2 * ecur;
        const T sc = dcur == d ? isq2 : T(1);
        DQ_LAUNCH(fermi_agg_kernel<T>, dim3(Bc * S, N), blk, 0, st, (const T*)Hc, dcur, (const T*)Ec, ecur, N, cfg.n_up, S, w.QKV);
        DQ_LAUNCH(zv_agg_kernel<T>, dim3(Bc * S, N), blk, 0, st, (const T*)Hcd, dcur, ecur, N, cfg.n_up, S, z.QKV);
        if ((rc = gemm(w.QKV, fin, (p + "wg").c_str(), nullptr, 0, d, P(p + "bg"), nullptr, 0, Hn, d, rows, d, fin, S, 0, N, st)))
          return rc;
        if ((rc = gemm(z.QKV, fin, (p + "wg").c_str(), nullptr, 0, d, nullptr, nullptr, 0, Hnd, d, rows, d, fin, S, 0, N, st)))
          return rc;
        DQ_LAUNCH(zv_act_kernel<T>, dim3(Bc * N, (d + 127) / 128), blk, 0, st, (const T*)Hn, d, Hnd, d,
                  (const T*)(dcur == d ? Hcd : nullptr), dcur, S, d, sc, 0);
        DQ_LAUNCH(tanh_fl_kernel<T>, dim3(Bc * N, (d + 127) / 128), blk, 0, st, Hn, d, (const T*)(dcur == d ? Hc : nullptr), dcur,
                  S, d, sc);
        if (l < cfg.n_layers - 1) {  // the two-particle stream: primal only (its companion is zero)
          if ((rc = gemm(Ec, ecur, (p + "wu").c_str(), nullptr, 0, de, P(p + "bu"), nullptr, 0, En, de, Bc * N * N * S, de, ecur, S,
                         0, N, st)))
            return rc;
          DQ_LAUNCH(tanh_fl_kernel<T>, dim3(Bc * N * N, 1), dim3(32), 0, st, En, de, (const T*)(ecur == de ? Ec : nullptr), ecur,
                    S, de, ecur == de ? isq2 : T(1));
          std::swap(Ec, En);
          ecur = de;
        }
        std::swap(Hc, Hn);
        std::swap(Hcd, Hnd);
        dcur = d;
      }
      X = Hc;
      Xd = Hcd;
    } else {
      DQ_LAUNCH(embed_kernel<T>, dim3(Bc * N), blk, sizeof(T) * 5 * (4 * M + 1), st, r, R, Rb, N, M, cfg.n_up, S, 1, 1,
                P("emb.w"), d, w.X, Bc * N, 1, (const T*)nullptr);
      DQ_LAUNCH(zv_embed_kernel<T>, dim3(Bc * N), blk, 0, st, r, R, Rb, N, M, S, 1, P("emb.w"), d, z.X, Bc * N, m, c);
      T *O = w.O, *Od = z.O;
      X = w.X;
      Xd = z.X;
      const T scale = (T)(1.0 / std::sqrt((double)dh));
      const int dblk = (d + 127) / 128;
      for (int l = 0; l < cfg.n_layers; ++l) {
        const std::string p = "L" + std::to_string(l) + ".";
        if ((rc = gemm(X, d, (p + "wqkv").c_str(), nullptr, 0, 3 * d, nullptr, nullptr, 0, w.QKV, 3 * d, rows, 3 * d, d, S, 0, N, st)))
          return rc;
        if ((rc = gemm(Xd, d, (p + "wqkv").c_str(), nullptr, 0, 3 * d, nullptr, nullptr, 0, z.QKV, 3 * d, rows, 3 * d, d, S, 0, N, st)))
          return rc;
        DQ_LAUNCH(zv_attn_kernel<T>, dim3(Bc, H), blk, zv_attn_smem_bytes<T>(N, dh), st, (const T*)w.QKV, (const T*)z.QKV, 3 * d,
                  Od, d, N, S, dh, d, scale);
        if ((rc = attention(w.QKV, O, Bc, S, l, st))) return rc;
        if ((rc = gemm(O, d, (p + "wo").c_str(), nullptr, 0, d, nullptr, X, d, w.A, d, rows, d, d, S, 0, N, st))) return rc;
        if ((rc = gemm(Od, d, (p + "wo").c_str(), nullptr, 0, d, nullptr, Xd, d, z.A, d, rows, d, d, S, 0, N, st))) return rc;
        if ((rc = gemm(w.A, d, (p + "w1").c_str(), nullptr, 0, d, P(p + "b1"), nullptr, 0, w.M1, d, rows, d, d, S, 0, N, st)))
          return rc;
        if ((rc = gemm(z.A, d, (p + "w1").c_str(), nullptr, 0, d, nullptr, nullptr, 0, z.M1, d, rows, d, d, S, 0, N, st))) return rc;
        DQ_LAUNCH(zv_act_kernel<T>, dim3(Bc * N, dblk), blk, 0, st, (const T*)w.M1, d, z.M1, d, (const T*)nullptr, 0, S, d, T(1), 0);
        DQ_LAUNCH(tanh_fl_kernel<T>, dim3(Bc * N, dblk), blk, 0, st, w.M1, d, (const T*)nullptr, 0, S, d, T(1));
        if ((rc = gemm(w.M1, d, (p + "w2").c_str(), nullptr, 0, d, P(p + "b2"), nullptr, 0, O, d, rows, d, d, S, 0, N, st))) return rc;
        if ((rc = gemm(z.M1, d, (p + "w2").c_str(), nullptr, 0, d, nullptr, nullptr, 0, Od, d, rows, d, d, S, 0, N, st))) return rc;
        DQ_LAUNCH(zv_act_kernel<T>, dim3(Bc * N, dblk), blk, 0, st, (const T*)O, d, Od, d, (const T*)z.A, d, S, d, T(1), 0);
        DQ_LAUNCH(tanh_fl_kernel<T>, dim3(Bc * N, dblk), blk, 0, st, O, d, (const T*)w.A, d, S, d, T(1));
        std::swap(X, O);
        std::swap(Xd, Od);
      }
    }
    // backflow heads (no bias for these kinds), mult_act, determinants, determinant sum
    if ((rc = gemm(X, bf_in, "bf.up", "bf.dn", cfg.n_up, BFW, nullptr, nullptr, 0, w.BF, BFW, Bc * S, BFW, bf_in, S, 1, N, st)))
      return rc;
    if ((rc = gemm(Xd, bf_in, "bf.up", "bf.dn", cfg.n_up, BFW, nullptr, nullptr, 0, z.BF, BFW, Bc * S, BFW, bf_in, S, 1, N, st)))
      return rc;
    if (cfg.mult_act == 1)
      DQ_LAUNCH(zv_act_kernel<T>, dim3(Bc * N, (KN + 127) / 128), blk, 0, st, (const T*)w.BF, KN, z.BF, KN, (const T*)nullptr, 0,
                S, KN, T(1), 2);
    if ((rc = slater(r, R, Rb, Bc, S, w.BF, w.Gadd, w.dsign, w.dlog, w.dgrad, w.dlap, st, nullptr, FwdIn{}, 0))) return rc;
    const int full_det = cfg.factorized_det ? 0 : 1;
    const int wpb = zv_slater_warps_per_block<T>(N);
    DQ_LAUNCH(zv_slater_kernel<T>, dim3((Bc * K + wpb - 1) / wpb), dim3(32 * wpb), zv_slater_smem_per_warp<T>(N) * wpb, st, r, R,
              Rb, N, M, cfg.n_up, K, S, Bc * K, P("env.pi_up"), P("env.pi_dn"), P("env.zeta_up"), P("env.zeta_dn"),
              (const T*)w.BF, (const T*)z.BF, BFW, z.zl, z.zg, z.zlap, env_rep, full_det, m, c);
    const FinalizeCfg fc = finalize_cfg(S);
    const T* nuc = cfg.nuc_cusp_kind ? P("cusp.nuc") : (const T*)nullptr;
    const T* conf = cfg.conf_linear ? P("conf.w") : (const T*)nullptr;
    DQ_LAUNCH(finalize_kernel<T>, dim3(Bc), blk, finalize_smem_bytes<T>(N, K), st, fc, r, R, Rb, (const T*)w.dsign,
              (const T*)w.dlog, (const T*)w.dgrad, (const T*)w.dlap, P("cusp.alpha"), (const T*)d_zval, (const T*)d_ecp_loc,
              (const int*)d_ecp_mask, Bc, z.sign, z.logp, z.E, z.stats, z.grad, conf, (const T*)nullptr, nuc, PhArgs<T>());
    DQ_LAUNCH(zv_finalize_kernel<T>, dim3(Bc), blk, zv_finalize_smem_bytes<T>(K), st, N, M, K, S, cfg.nuc_cusp_kind, r, R, Rb,
              (const T*)w.dsign, (const T*)w.dlog, (const T*)w.dgrad, (const T*)w.dlap, (const T*)z.zl, (const T*)z.zg,
              (const T*)z.zlap, conf, (const T*)z.grad, nuc, m, c, 3 * M, kappa, zv, gR);
    return 0;
  }

  // -dT/dR and (optionally) grad_R log|psi| per walker [B][M][3]: for every chunk and nuclear coordinate one zv_chunk
  int zv_force(const void* r_, const void* R_, int Rb, int B, void* zv_, void* gR_, void* ws, int64_t wsb,
               cudaStream_t st) override {
    if (const char* why = zv_refusal()) { err = std::string("dqmc_zv_force: ") + why; return 2; }
    if (B == 0) return 0;
    const size_t s_attn = cfg.kind == DQMC_PSIFORMER ? zv_attn_smem_bytes<T>(N, dh) : 0;
    const size_t s_sl = zv_slater_smem_per_warp<T>(N) * zv_slater_warps_per_block<T>(N);
    if (s_attn > 227 * 1024 || s_sl > 227 * 1024) {
      err = "dqmc_zv_force: system too large for the companion kernels' shared memory (N, head width)";
      return 2;
    }
    int64_t row_cap = kRowCap / ((int64_t)N * (T3 + 2) * 3 * d);
    if (cfg.kind == DQMC_FERMINET) row_cap = kRowCap / ((int64_t)N * N * (T3 + 2) * (3 * (int64_t)fermi_dmax() + 64));
    const int Bc = (int)largest_fit(std::min<int64_t>(B, row_cap), wsb, [&](int64_t n) { return zv_chunk_bytes((int)n); });
    if (Bc < 1) { err = "workspace too small for a single walker"; return 3; }
    Arena a(this, ws, wsb);
    const ZvWs z = carve_zv(a, Bc);
    Ws w = carve(a.top, Bc, T3 + 2);
    if (dry) return 0;
    if (s_attn) DQ_CHECK(raise_dyn_smem(zv_attn_kernel<T>, (int)s_attn));
    DQ_CHECK(raise_dyn_smem(zv_slater_kernel<T>, (int)s_sl));
    const T* r = (const T*)r_;
    const T* R = (const T*)R_;
    T* zv = (T*)zv_;
    T* gR = (T*)gR_;
    for (int b0 = 0; b0 < B; b0 += Bc) {
      const int nb = std::min(Bc, B - b0);
      for (int kappa = 0; kappa < 3 * M; ++kappa) {
        int rc = zv_chunk(r + (size_t)b0 * 3 * N, R + (Rb ? (size_t)b0 * 3 * M : 0), Rb, nb, kappa, z, w,
                          zv + (size_t)b0 * 3 * M, gR ? gR + (size_t)b0 * 3 * M : nullptr, st);
        if (rc) return rc;
        if ((rc = check_guards())) return rc;
      }
    }
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  int stats_pack(const void* E, const void* stats, int B, double* out, cudaStream_t st) override {
    DQ_LAUNCH(stats_pack_kernel<T>, dim3(1), dim3(1024), 0, st, (const T*)E, (const T*)stats, B, out);
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  // orbital matrices out[B][K][N][N] (electron i, orbital mu) of a plain forward
  int orbitals(const void* r, const void* R, int Rb, int B, void* out, void* ws, int64_t wsb, cudaStream_t st) override {
    FwdIn in;
    in.mos = (T*)out;
    int rc = run_batched((const T*)r, (const T*)R, Rb, B, 1, nullptr, nullptr, nullptr, nullptr, nullptr, ws, wsb, st, in);
    if (rc) return rc;
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  int forward(const void* r, const void* R, int Rb, int B, void* sign, void* logp, void* ws, int64_t wsb,
              cudaStream_t st) override {
    int rc = run_batched((const T*)r, (const T*)R, Rb, B, 1, (T*)sign, (T*)logp, nullptr, nullptr, nullptr, ws, wsb, st);
    if (rc) return rc;
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  // Virtual walkers (vper per base walker: ECP quadrature points, spin swaps) through a per-group pass in groups of nb base
  // walkers: the largest group whose prefix (carve_group) + one pass chunk of all its virtual walkers (chunk_carve, a dry carve
  // after the prefix) fits wsb, else one walker (the pass chunks its virtual walkers).  Per group, setup() launches the kind's
  // work before the pass and sets V, the virtual walkers to run, pass(g, in, V, rest) runs them in the workspace after the
  // prefix (run_batched: plain forwards; reverse_pass: position gradients), and finish() reduces their results.  With `tables`
  // (and slater_fwd2, N <= 32) the forwards take the unmoved electrons' envelopes and, with `emb_table`, embedding rows from
  // tables of the base walkers: `in` describes them (default: none).
  template <class CarveGroup, class Setup, class Pass, class ChunkCarve, class Finish>
  int virtual_groups(const T* r, const T* R, int B, int64_t vper, int layout, bool tables, bool emb_table, void* ws,
                     int64_t wsb, const char* too_small, CarveGroup carve_group, Setup setup, Pass pass, ChunkCarve chunk_carve,
                     Finish finish, cudaStream_t st) {
    auto bytes = [&](int64_t nb, int64_t Vc) {
      DryPass dp(this);
      Arena a(this, plan_base());
      carve_group(a, nb);
      chunk_carve(a, Vc);
      return dp.bytes();
    };
    int64_t Be = largest_fit(std::min<int64_t>(B, group_cap(vper)), wsb, [&](int64_t nb) { return bytes(nb, nb * vper); });
    if (Be < 1) Be = 1;  // one walker's virtual walkers do not fit at once: the pass chunks them
    if (bytes(Be, 1) > wsb) { err = too_small; return 3; }
    tables = tables && slater_fwd2_ok && N <= 32 && !dry;
    emb_table = tables && emb_table && embed_fwd_ok && can_trunk(1);
    for (int b0 = 0; b0 < B; b0 += (int)Be) {
      const int nb = (int)std::min<int64_t>(Be, B - b0);
      const T* rb = r + (size_t)b0 * 3 * N;
      Arena a(this, ws, wsb);
      const VirtGroup g = carve_group(a, nb);
      int64_t V = 0;
      int rc = setup(b0, nb, g, a, V);
      if (rc) return rc;
      FwdIn in;
      if (tables) {
        DQ_LAUNCH(env_table_kernel<T>, dim3(nb), dim3(256), sizeof(T) * N * M, st, rb, R, N, M, cfg.n_up, K * N, P("env.pi_up"),
                  P("env.pi_dn"), P("env.zeta_up"), P("env.zeta_dn"), env_rep, g.env);
        in.env = g.env; in.vper = (int)vper; in.layout = layout; in.pairs = g.pairs;
        if (emb_table) {
          DQ_LAUNCH(embed_fwd_kernel<T>, dim3((nb * N + 31) / 32), dim3(256), embed_fwd_smem_bytes<T>(M, d), st, rb, R, 0, N, M,
                    cfg.n_up, 1, P("emb.w"), d, g.emb, nb * N, 32, 0LL, 0, (const int*)nullptr);
          in.emb = g.emb;
        }
      }
      if (V > 0) rc = pass(g, in, V, a);
      if (rc) return rc;
      rc = finish(b0, nb, g);
      if (!rc) rc = check_guards();  // the prefix's guards, also when no forward ran (V == 0)
      if (rc) return rc;
      if (dry) break;  // planning pass: the first group is the largest
    }
    return 0;
  }

  // the plain-forward pass of a virtual-walker group (ECP energy, spin), in the workspace after the group's prefix
  int virt_forwards(const VirtGroup& g, const FwdIn& in, const T* R, int64_t V, const Arena& rest, cudaStream_t st) {
    return run_batched(g.r, R, 0, (int)V, 1, g.sign, g.logp, nullptr, nullptr, nullptr, rest.top, rest.left(), st, in);
  }

  // The non-local ECP's virtual walkers of the group g of nb base walkers from walker b0 on (nuclei shared by all walkers):
  // the electron-nucleus pairs inside the cutoff radii rc2 (ecp_pairs_kernel), whose quadrature forwards alone run, and
  // their quadrature points (ecp_points_kernel) with the twists `twist` [B][J][N] or, if null, twists drawn from `seed`.
  // V = the number of quadrature points.  The energy and the force pass share it, each with its own radii.
  int ecp_group_points(const T* r, const T* R, int b0, int nb, const VirtGroup& g, const double* rc2, const T* twist,
                       uint64_t seed, int64_t& V, cudaStream_t st) {
    const T* rb = r + (size_t)b0 * 3 * N;
    DQ_LAUNCH(ecp_pairs_kernel<T>, dim3(1), dim3(1024), 0, st, rb, R, 0, N, M, J, (const int*)d_nl_nuc, rc2, nb, g.offs,
              g.pairs, g.offs + nb);
    int n_act = nb * J * N;  // the planning pass sizes every buffer for all pairs
    if (!dry) {
      DQ_CHECK(cudaMemcpyAsync(&n_act, g.offs + nb, sizeof(int), cudaMemcpyDeviceToHost, st));
      DQ_CHECK(cudaStreamSynchronize(st));
      ecp_forwards += (int64_t)n_act * 12;
    }
    V = (int64_t)n_act * 12;
    if (n_act > 0)
      DQ_LAUNCH(ecp_points_kernel<T>, dim3(n_act), dim3(64), 0, st, rb, R, 0, N, M, J, (const int*)d_nl_nuc,
                twist ? twist + (size_t)b0 * J * N : nullptr, seed, (uint64_t)b0, (const int*)g.pairs, g.r);
    return 0;
  }

  // Hellmann-Feynman force terms with effective core potentials (reference force.py:252-301): bare = F_nuc(Z_eff) - grad_R V_loc
  // (force_terms_kernel with the local ECP table), nl = -grad_R V_nl per walker.  The non-local part runs in groups of base
  // walkers (virtual_groups): a position reverse pass of the base walkers (sign, log, grad_R), the active pairs inside the
  // force's cutoff radius with their quadrature points (the energy pass's twists for the same seed / ecp_twist), a position
  // reverse pass over those virtual walkers, and ecp_force_accumulate_kernel.
  int ecp_force(const void* r_, const void* R_, int Rb, int B, uint64_t seed, const void* twist, void* bare, void* nl, void* ws,
                int64_t wsb, cudaStream_t st) override {
    const T* r = (const T*)r_;
    const T* R = (const T*)R_;
    if (d_ph_tabs) { err = "dqmc_ecp_force: pseudo-Hamiltonians are not supported"; return 2; }
    if (nl && !has_nl_force()) {
      err = "dqmc_ecp_force: the non-local force needs grad_r and grad_R of log|psi| by the reverse pass (Psiformer and FermiNet "
            "with multiplicative backflow); out_nl must be null";
      return 2;
    }
    if (nl && Rb) { err = "non-local ECP with per-walker nuclei is not supported"; return 2; }
    if (B == 0) return 0;
    if (bare)
      DQ_LAUNCH(force_terms_kernel<T>, dim3(B), dim3(32), 0, st, r, R, Rb, N, M, (const T*)d_zval, (const T*)nullptr, (T*)bare,
                (T*)nullptr, (T*)nullptr, (const T*)d_ecp_loc, cfg.ecp_loc_terms);
    if (nl && !J && !dry) DQ_CHECK(cudaMemsetAsync(nl, 0, sizeof(T) * (size_t)B * M * 3, st));
    if (nl && J) {
      auto setup = [&](int b0, int nb, const VirtGroup& g, const Arena& rest, int64_t& V) {
        const T* rb = r + (size_t)b0 * 3 * N;
        const PosOut p0{nullptr, g.gR0};
        int rc = reverse_pass(rb, R, 0, nb, nullptr, g.sign0, g.logp0, nullptr, &p0, rest.top, rest.left(), st, "ecp_force");
        if (rc) return rc;
        return ecp_group_points(r, R, b0, nb, g, d_nl_rc2f, (const T*)twist, seed, V, st);
      };
      auto pass = [&](const VirtGroup& g, const FwdIn&, int64_t V, const Arena& rest) {
        const PosOut pv{g.gr, g.gR};
        return reverse_pass(g.r, R, 0, (int)V, nullptr, g.sign, g.logp, nullptr, &pv, rest.top, rest.left(), st, "ecp_force");
      };
      auto finish = [&](int b0, int nb, const VirtGroup& g) {
        DQ_LAUNCH(ecp_force_accumulate_kernel<T>, dim3((nb + 3) / 4), dim3(128), 0, st, r + (size_t)b0 * 3 * N, R, N, M, J,
                  (const int*)d_nl_nuc, (const T*)d_nl_params, (const double*)d_nl_rc2f, (const int*)g.offs, cfg.ecp_nl_lmax_p1,
                  cfg.ecp_nl_terms, twist ? (const T*)twist + (size_t)b0 * J * N : nullptr, seed, (uint64_t)b0,
                  (const T*)g.sign0, (const T*)g.logp0, (const T*)g.gR0, (const T*)g.sign, (const T*)g.logp, (const T*)g.gr,
                  (const T*)g.gR, nb, (T*)nl + (size_t)b0 * M * 3);
        return 0;
      };
      int rc = virtual_groups(r, R, B, (int64_t)J * N * 12, kVirtEcp, false, false, ws, wsb,
                              "workspace too small for the non-local ECP force", [&](Arena& a, int64_t nb) { return carve_ecp_force_group(a, nb); },
                              setup, pass, [&](Arena& a, int64_t Vc) { pos_chunk_carve(a, Vc); }, finish, st);
      if (rc) return rc;
    }
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  int local_energy(const void* r_, const void* R_, int Rb, int B, uint64_t seed, const void* twist, void* E,
                   void* stats, void* sign, void* logp, void* grad, void* ws, int64_t wsb, cudaStream_t st) override {
    const T* r = (const T*)r_;
    const T* R = (const T*)R_;
    if (J > 0 && Rb) { err = "non-local ECP with per-walker nuclei is not supported"; return 2; }
    FwdIn in;
    in.ph = ph_on;
    int rc = run_batched(r, R, Rb, B, T3 + 2, (T*)sign, (T*)logp, (T*)E, (T*)stats, (T*)grad, ws, wsb, st, in);
    if (rc) return rc;
    if (J > 0) {
      // non-local ECP: virtual walkers (12 quadrature points x electrons x ECP nuclei)
      auto setup = [&](int b0, int nb, const VirtGroup& g, const Arena&, int64_t& V) {
        return ecp_group_points(r, R, b0, nb, g, d_nl_rc2, (const T*)twist, seed, V, st);
      };
      auto finish = [&](int b0, int nb, const VirtGroup& g) {
        DQ_LAUNCH(ecp_accumulate_kernel<T>, dim3((nb + 3) / 4), dim3(128), 0, st, r + (size_t)b0 * 3 * N, R, Rb, N, M, J,
                  (const int*)d_nl_nuc, (const T*)d_nl_params, (const double*)d_nl_rc2, (const int*)g.offs,
                  cfg.ecp_nl_lmax_p1, cfg.ecp_nl_terms,
                  (const T*)sign + b0, (const T*)logp + b0, (const T*)g.sign, (const T*)g.logp, nb, B, (T*)E + b0,
                  (T*)stats + b0);
        return 0;
      };
      rc = virtual_groups(r, R, B, (int64_t)J * N * 12, kVirtEcp, sw.ecp_env_table, sw.ecp_emb_table, ws, wsb,
                          "workspace too small for the non-local ECP pass", [&](Arena& a, int64_t nb) { return carve_ecp_group(a, nb); }, setup,
                          [&](const VirtGroup& g, const FwdIn& in, int64_t V, const Arena& a) { return virt_forwards(g, in, R, V, a, st); },
                          [&](Arena& a, int64_t Vc) { fwd_chunk_carve(a, Vc); }, finish, st);
      if (rc) return rc;
    }
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  // <S^2> estimators (reference physics.py:159-239): every walker's virtual walkers (one up / down pair swapped each) run
  // through the plain forward in groups of whole walkers; spin_accumulate_kernel reduces their ratios per walker.  A group
  // whose virtual walkers do not fit the workspace at once is split across plain-forward chunks by run_batched.
  int spin(const void* r_, const void* R_, int Rb, int B, const void* sign_, const void* logp_, int down_idx, void* s2_,
           void* ratio_, void* ws, int64_t wsb, cudaStream_t st) override {
    const T* r = (const T*)r_;
    const T* R = (const T*)R_;
    const int nd = cfg.n_down, nu = cfg.n_up;
    if (Rb) { err = "spin: per-walker nuclei are not supported"; return 2; }
    if (down_idx != -1 && (nd == 0 || down_idx < nu || down_idx >= N)) { err = "spin: down_idx out of range"; return 2; }
    if (!sign_ != !logp_) { err = "spin: pass both sign and log of the walkers, or neither"; return 2; }
    if (B < 1) return 0;
    const int64_t Pn = down_idx < 0 ? (int64_t)nu * nd : nu;
    const double D = nu - nd;
    const double c0 = down_idx < 0 ? D / 2 * (D / 2 + 1) + nd : 1.0;
    if (Pn == 0) {  // no down electrons: the constant, no forwards
      DQ_LAUNCH(spin_accumulate_kernel<T>, dim3((B + 3) / 4), dim3(128), 0, st, (const T*)nullptr, (const T*)nullptr,
                (const T*)nullptr, (const T*)nullptr, 0, B, c0, (T*)s2_, (T*)nullptr);
      DQ_CHECK(cudaGetLastError());
      return 0;
    }
    auto setup = [&](int b0, int nb, const VirtGroup& g, const Arena& rest, int64_t& V) {
      const T* rb = r + (size_t)b0 * 3 * N;
      if (!sign_) {
        int rc = run_batched(rb, R, 0, nb, 1, g.sign0, g.logp0, nullptr, nullptr, nullptr, rest.top, rest.left(), st);
        if (rc) return rc;
      }
      V = (int64_t)nb * Pn;
      const int64_t ne = V * 3 * N;
      DQ_LAUNCH(spin_pairs_kernel<T>, dim3((unsigned)((ne + 255) / 256)), dim3(256), 0, st, rb, N, nu, down_idx, (int)Pn, ne, g.r);
      return 0;
    };
    auto finish = [&](int b0, int nb, const VirtGroup& g) {
      DQ_LAUNCH(spin_accumulate_kernel<T>, dim3((nb + 3) / 4), dim3(128), 0, st,
                sign_ ? (const T*)sign_ + b0 : (const T*)g.sign0, sign_ ? (const T*)logp_ + b0 : (const T*)g.logp0,
                (const T*)g.sign, (const T*)g.logp, (int)Pn, nb, c0, (T*)s2_ + b0, ratio_ ? (T*)ratio_ + (size_t)b0 * Pn : (T*)nullptr);
      return 0;
    };
    // a swapped walker differs from its base walker in two electrons: the forwards take every other electron's envelopes and
    // embedding rows from tables of the base walkers
    int rc = virtual_groups(r, R, B, Pn, down_idx, cfg.kind == DQMC_PSIFORMER, true, ws, wsb, "workspace too small for the spin pass",
                            [&](Arena& a, int64_t nb) { return carve_spin_group(a, nb, Pn); }, setup,
                            [&](const VirtGroup& g, const FwdIn& in, int64_t V, const Arena& a) { return virt_forwards(g, in, R, V, a, st); },
                            [&](Arena& a, int64_t Vc) { fwd_chunk_carve(a, Vc); }, finish, st);
    if (rc) return rc;
    DQ_CHECK(cudaGetLastError());
    return 0;
  }

  int mcmc(void* r_, void* sign_, void* logp_, int32_t* age, void* tau_, const void* R_, int Rb, int B, int n_sub,
           double target, int max_age, uint64_t seed, uint64_t step0, uint64_t woff, const void* nn, const void* nu,
           void* stats_, void* ws, int64_t wsb, cudaStream_t st, double p_exchange, const int32_t* ex_flags,
           const int32_t* ex_idx) override {
    // p_exchange > 0 (or ex_flags given): some sub-steps are spin-exchange steps (OppositeSpinExchangeSampler,
    // electron_samplers.py:286-330): the whole batch swaps one up / down pair per walker, plain Metropolis acceptance without
    // max_age override and without step-size adaptation.  ex_flags[n_sub] (host) / ex_idx[n_sub][B][2] (device): injected.
    T* r = (T*)r_; T* sign = (T*)sign_; T* logp = (T*)logp_; T* tau = (T*)tau_; T* stats = (T*)stats_;
    const T* R = (const T*)R_;
    Arena a(this, ws, wsb);
    const Proposals q = carve_proposals(a, B, false);
    if (a.left() < 0) { err = "workspace too small (proposal buffers)"; return 3; }
    DQ_CHECK(cudaMemsetAsync(q.cnt, 0, sizeof(int), st));
    const int ne = B * 3 * N;
    for (int s = 0; s < n_sub; ++s) {
      const T* nns = nn ? (const T*)nn + (size_t)s * ne : nullptr;
      const T* nus = nu ? (const T*)nu + (size_t)s * B : nullptr;
      bool exchange = false;
      if (ex_flags) exchange = ex_flags[s] != 0;
      else if (p_exchange > 0.0) {  // one decision per sub-step for the whole batch (as the reference's lax.cond on a scalar)
        uint32_t w4[4];
        Philox::gen(seed ^ 0xA0761D6478BD642Full, 0, step0 + (uint64_t)s, w4);
        exchange = Philox::u01(w4[0], w4[1]) < p_exchange;
      }
      if (exchange)
        DQ_LAUNCH(exchange_propose_kernel<T>, dim3((B + 127) / 128), dim3(128), 0, st, (const T*)r, q.r,
                  ex_idx ? ex_idx + (size_t)s * 2 * B : (const int32_t*)nullptr, seed, step0 + (uint64_t)s, woff, cfg.n_up, N, B);
      else
      DQ_LAUNCH(propose_kernel<T>, dim3((ne / 2 + 1 + 127) / 128), dim3(128), 0, st, (const T*)r, q.r, (const T*)tau, nns,
                seed, step0 + (uint64_t)s, woff * (uint64_t)(3 * N), ne);
      int rc = run_batched(q.r, R, Rb, B, 1, q.sign, q.logp, nullptr, nullptr, nullptr, a.top, a.left(), st);
      if (rc) return rc;
      DQ_LAUNCH(accept_kernel<T>, dim3((B + 127) / 128), dim3(128), 0, st, r, (const T*)q.r, sign, (const T*)q.sign, logp,
                (const T*)q.logp, age, nus, seed, step0 + (uint64_t)s, woff, exchange ? -1 : max_age, B, N, q.cnt);
      DQ_LAUNCH(tau_kernel<T>, dim3(1), dim3(32), 0, st, tau, q.cnt, B, exchange ? T(0) : (T)target, stats);
    }
    DQ_LAUNCH(sampler_stats_kernel<T>, dim3(1), dim3(256), 0, st, (const T*)r, (const T*)logp, (const int*)age,
              (const T*)tau, B, N, stats);
    DQ_CHECK(cudaGetLastError());
    return check_guards();  // the proposal buffers' guards, after the last accept (and with n_sub == 0)
  }
};

}  // namespace dq

// ================================= C ABI ======================================================
struct dqmc_engine {
  dq::EngineBase* e;
};

#define DQ_NEED_DEVICE(h)                                                                        \
  do {                                                                                            \
    if ((h)->e->plan_only) {                                                                      \
      (h)->e->err = "plan-only engine (created with device < 0): no compute entry points";        \
      return 2;                                                                                   \
    }                                                                                             \
  } while (0)

extern "C" {

const char* dqmc_version(void) { return "dqmc_b200 0.1 (sm_90a)"; }

int dqmc_create(const dqmc_config* cfg, int device, dqmc_handle* out) {
  if (!cfg || !out) return 2;
  dq::EngineBase* e = nullptr;
  int rc = 0;
  const bool plan = device < 0;  // plan-only engine: workspace planning without a CUDA device (dqmc_debug_plan)
  if (cfg->dtype == DQMC_F64) {
    auto* x = new dq::Engine<double>();
    x->cfg = *cfg; x->device = device; x->dry = x->plan_only = plan; rc = x->init(); e = x;
  } else if (cfg->dtype == DQMC_F32) {
    auto* x = new dq::Engine<float>();
    x->cfg = *cfg; x->device = device; x->dry = x->plan_only = plan; rc = x->init(); e = x;
  } else {
    return 2;
  }
  if (rc) {
    std::fprintf(stderr, "dqmc_create failed: %s\n", e->err.c_str());
    delete e;
    return rc;
  }
  *out = new dqmc_engine{e};
  return 0;
}
int dqmc_destroy(dqmc_handle h) {
  if (!h) return 2;
  delete h->e;
  delete h;
  return 0;
}
const char* dqmc_last_error(dqmc_handle h) { return h ? h->e->err.c_str() : "null handle"; }
int dqmc_param_count(dqmc_handle h) { return h ? (int)h->e->entries.size() : -1; }
int64_t dqmc_param_total(dqmc_handle h) { return h ? h->e->total : -1; }
int dqmc_param_entry(dqmc_handle h, int idx, char* name, int name_len, int64_t* offset, int32_t* rows, int32_t* cols) {
  if (!h || idx < 0 || idx >= (int)h->e->entries.size()) return 2;
  auto& en = h->e->entries[idx];
  if (name && name_len > 0) {
    std::strncpy(name, en.name.c_str(), name_len - 1);
    name[name_len - 1] = 0;
  }
  if (offset) *offset = en.offset;
  if (rows) *rows = en.rows;
  if (cols) *cols = en.cols;
  return 0;
}
int dqmc_set_params(dqmc_handle h, const double* host_params, int64_t n, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  return h->e->set_params(host_params, n, (cudaStream_t)stream);
}
int64_t dqmc_workspace_bytes(dqmc_handle h, int32_t n_walkers, int32_t mode) {
  return h ? h->e->ws_bytes(n_walkers, mode) : -1;
}
int64_t dqmc_workspace_bytes_min(dqmc_handle h, int32_t n_walkers, int32_t mode) {
  return h ? h->e->ws_bytes_min(n_walkers, mode) : -1;
}
int dqmc_wf_forward(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers, void* out_sign,
                    void* out_log, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (n_walkers < 0) { h->e->err = "negative walker count"; return 2; }
  if (n_walkers == 0) return 0;  // empty batch: nothing to evaluate
  return h->e->forward(r, R, R_batched, n_walkers, out_sign, out_log, workspace, workspace_bytes, (cudaStream_t)stream);
}
int dqmc_wf_orbitals(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers, void* out_orbitals,
                     void* workspace, int64_t workspace_bytes, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (n_walkers < 0) { h->e->err = "negative walker count"; return 2; }
  if (n_walkers == 0) return 0;
  return h->e->orbitals(r, R, R_batched, n_walkers, out_orbitals, workspace, workspace_bytes, (cudaStream_t)stream);
}
int dqmc_local_energy(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers, uint64_t seed,
                      const void* ecp_twist, void* out_E, void* out_stats, void* out_sign, void* out_log,
                      void* out_grad, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (n_walkers < 0) { h->e->err = "negative walker count"; return 2; }
  if (n_walkers == 0) return 0;  // empty batch: nothing to evaluate
  return h->e->local_energy(r, R, R_batched, n_walkers, seed, ecp_twist, out_E, out_stats, out_sign, out_log, out_grad,
                            workspace, workspace_bytes, (cudaStream_t)stream);
}
int dqmc_mcmc_sweep(dqmc_handle h, void* r, void* sign, void* log, int32_t* age, void* tau, const void* R,
                    int32_t R_batched, int32_t n_walkers, int32_t n_sub, double target_acceptance, int32_t max_age,
                    uint64_t seed, uint64_t step0, uint64_t walker_offset, const void* noise_normal,
                    const void* noise_uniform, void* out_stats, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (n_walkers < 1) { h->e->err = "the sampler needs at least one walker"; return 2; }
  return h->e->mcmc(r, sign, log, age, tau, R, R_batched, n_walkers, n_sub, target_acceptance, max_age, seed, step0,
                    walker_offset, noise_normal, noise_uniform, out_stats, workspace, workspace_bytes,
                    (cudaStream_t)stream);
}
int dqmc_mcmc_sweep_exchange(dqmc_handle h, void* r, void* sign, void* log, int32_t* age, void* tau, const void* R,
                             int32_t R_batched, int32_t n_walkers, int32_t n_sub, double target_acceptance, int32_t max_age,
                             uint64_t seed, uint64_t step0, uint64_t walker_offset, const void* noise_normal,
                             const void* noise_uniform, double exchange_step_probability, const int32_t* exchange_flags,
                             const int32_t* exchange_idx, void* out_stats, void* workspace, int64_t workspace_bytes,
                             void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (n_walkers < 1) { h->e->err = "the sampler needs at least one walker"; return 2; }
  if (h->e->cfg.n_up < 1 || h->e->cfg.n_down < 1) { h->e->err = "spin exchange needs electrons of both spins"; return 2; }
  return h->e->mcmc(r, sign, log, age, tau, R, R_batched, n_walkers, n_sub, target_acceptance, max_age, seed, step0,
                    walker_offset, noise_normal, noise_uniform, out_stats, workspace, workspace_bytes, (cudaStream_t)stream,
                    exchange_step_probability, exchange_flags, exchange_idx);
}
int dqmc_langevin_sweep(dqmc_handle h, void* r, void* sign, void* log, void* force, int32_t* age, void* tau, const void* R,
                        int32_t R_batched, int32_t n_walkers, int32_t n_sub, double target_acceptance, int32_t max_age,
                        uint64_t seed, uint64_t step0, uint64_t walker_offset, const void* noise_normal,
                        const void* noise_uniform, void* out_stats, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (n_walkers < 1) { h->e->err = "the sampler needs at least one walker"; return 2; }
  return h->e->langevin(r, sign, log, force, age, tau, R, R_batched, n_walkers, n_sub, target_acceptance, max_age, seed, step0,
                        walker_offset, noise_normal, noise_uniform, out_stats, workspace, workspace_bytes, (cudaStream_t)stream);
}
int dqmc_wf_vjp_params(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers, const void* weights,
                       void* out_sign, void* out_log, void* out_grad_params, void* workspace, int64_t workspace_bytes,
                       void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (n_walkers < 0) { h->e->err = "negative walker count"; return 2; }
  return h->e->vjp_params(r, R, R_batched, n_walkers, weights, out_sign, out_log, out_grad_params, workspace, workspace_bytes,
                          (cudaStream_t)stream);
}
int dqmc_spin(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers, const void* sign,
              const void* log, int32_t down_idx, void* out_s2, void* out_ratio, void* workspace, int64_t workspace_bytes,
              void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (n_walkers < 0) { h->e->err = "negative walker count"; return 2; }
  return h->e->spin(r, R, R_batched, n_walkers, sign, log, down_idx, out_s2, out_ratio, workspace, workspace_bytes,
                    (cudaStream_t)stream);
}
int dqmc_wf_grad_positions(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers, void* out_sign,
                           void* out_log, void* out_grad_r, void* out_grad_R, void* workspace, int64_t workspace_bytes,
                           void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (n_walkers < 0) { h->e->err = "negative walker count"; return 2; }
  if (n_walkers > 0 && (!r || !R || !out_sign || !out_log)) { h->e->err = "dqmc_wf_grad_positions: null array"; return 2; }
  return h->e->grad_positions(r, R, R_batched, n_walkers, out_sign, out_log, out_grad_r, out_grad_R, workspace, workspace_bytes,
                              (cudaStream_t)stream);
}
int dqmc_force_terms(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers, const void* grad_r,
                     void* out_bare, void* out_zvq, void* out_Q, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (n_walkers < 0) { h->e->err = "negative walker count"; return 2; }
  if (n_walkers > 0 && (!r || !R)) { h->e->err = "dqmc_force_terms: null array"; return 2; }
  return h->e->force_terms(r, R, R_batched, n_walkers, grad_r, out_bare, out_zvq, out_Q, (cudaStream_t)stream);
}
int dqmc_ecp_force(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers, uint64_t seed,
                   const void* ecp_twist, void* out_bare, void* out_nl, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (n_walkers < 0) { h->e->err = "negative walker count"; return 2; }
  if (n_walkers > 0 && (!r || !R)) { h->e->err = "dqmc_ecp_force: null array"; return 2; }
  return h->e->ecp_force(r, R, R_batched, n_walkers, seed, ecp_twist, out_bare, out_nl, workspace, workspace_bytes,
                         (cudaStream_t)stream);
}
int dqmc_zv_force(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers, void* out_zv,
                  void* out_grad_R, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (n_walkers < 0) { h->e->err = "negative walker count"; return 2; }
  if (n_walkers > 0 && (!r || !R || !out_zv)) { h->e->err = "dqmc_zv_force: null array"; return 2; }
  return h->e->zv_force(r, R, R_batched, n_walkers, out_zv, out_grad_R, workspace, workspace_bytes, (cudaStream_t)stream);
}
int dqmc_set_pseudo_hamiltonian(dqmc_handle h, int32_t n_tab, int32_t n_grid, double r_max, const double* tables,
                                const int32_t* tab_of_nuc) {
  if (!h) return 2;
  if (!h->e->plan_only) cudaSetDevice(h->e->device);
  return h->e->set_ph(n_tab, n_grid, r_max, tables, tab_of_nuc);
}
int dqmc_debug_plan(dqmc_handle h, int32_t n_walkers, int32_t mode, int64_t workspace_bytes, int64_t* planned_bytes,
                    int64_t* carved_bytes) {
  if (!h) return 2;
  if (n_walkers < 1) { h->e->err = "dqmc_debug_plan needs at least one walker"; return 2; }
  return h->e->debug_plan(n_walkers, mode, workspace_bytes, planned_bytes, carved_bytes);
}
int dqmc_stats_pack(dqmc_handle h, const void* E_loc, const void* stats, int32_t n_walkers, double* out11, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (n_walkers < 1 || !E_loc || !out11) { h->e->err = "dqmc_stats_pack: bad arguments"; return 2; }
  return h->e->stats_pack(E_loc, stats, n_walkers, out11, (cudaStream_t)stream);
}
int64_t dqmc_launch_count(dqmc_handle h) { return h ? h->e->launches : -1; }
int64_t dqmc_ecp_forward_count(dqmc_handle h) { return h ? h->e->ecp_forwards : -1; }

int dqmc_debug_gemm(dqmc_handle h, const char* weight, const char* bias, const void* A, const void* Res, void* C,
                    int32_t rows, int32_t S, int32_t sliced, int32_t backend, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  return h->e->debug_gemm(weight, bias, A, Res, C, rows, S, sliced, backend, (cudaStream_t)stream);
}

int dqmc_debug_mlp_block(dqmc_handle h, int32_t layer, const void* O, const void* X, void* Out, int32_t rows, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  return h->e->debug_mlp_block(layer, O, X, Out, rows, (cudaStream_t)stream);
}
int dqmc_debug_trunk(dqmc_handle h, const void* X0, void* Out, int32_t rows, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  return h->e->debug_trunk(X0, Out, rows, (cudaStream_t)stream);
}
int dqmc_debug_attention(dqmc_handle h, int32_t layer, const void* QKV, void* O, int32_t rows, int32_t S, int32_t* kernel,
                         void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (!QKV || !O) { h->e->err = "dqmc_debug_attention: null array"; return 2; }
  return h->e->debug_attention(layer, QKV, O, rows, S, kernel, (cudaStream_t)stream);
}
int dqmc_debug_mlp(dqmc_handle h, int32_t layer, int32_t S, const void* O, const void* X, void* Out, void* scratch, int32_t rows,
                   int32_t* path, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (!O || !X || !Out || !scratch) { h->e->err = "dqmc_debug_mlp: null array"; return 2; }
  return h->e->debug_mlp(layer, S, O, X, Out, scratch, rows, path, (cudaStream_t)stream);
}
int dqmc_debug_slater(dqmc_handle h, const void* r, const void* R, const void* BF, int32_t rows, int32_t S, void* det_sign,
                      void* det_log, void* det_grad, void* det_lap, int32_t* kernel, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (!r || !R || !BF || !det_sign || !det_log) { h->e->err = "dqmc_debug_slater: null array"; return 2; }
  return h->e->debug_slater(r, R, BF, rows, S, det_sign, det_log, det_grad, det_lap, kernel, (cudaStream_t)stream);
}
int dqmc_debug_det_sum(dqmc_handle h, const void* r, const void* R, const void* det_sign, const void* det_log,
                       const void* det_grad, const void* det_lap, int32_t B, int32_t S, void* sign, void* logp, void* grad,
                       void* stats, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (!r || !R || !det_sign || !det_log || !sign || !logp) { h->e->err = "dqmc_debug_det_sum: null array"; return 2; }
  return h->e->debug_det_sum(r, R, det_sign, det_log, det_grad, det_lap, B, S, sign, logp, grad, stats, (cudaStream_t)stream);
}
int dqmc_debug_attention_bwd(dqmc_handle h, int32_t layer, const void* QKV, const void* dO, void* dQKV, void* dKn, void* dVn,
                             int32_t rows, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (!QKV || !dO || !dQKV) { h->e->err = "dqmc_debug_attention_bwd: null array"; return 2; }
  return h->e->debug_attention_bwd(layer, QKV, dO, dQKV, dKn, dVn, rows, (cudaStream_t)stream);
}
int dqmc_debug_wgrad(dqmc_handle h, const void* A, const void* dY, int32_t rows, int32_t K, int32_t Nc, int32_t lo, int32_t hi,
                     void* dW, void* db, void* stream) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (!A || !dY || !dW || !db) { h->e->err = "dqmc_debug_wgrad: null array"; return 2; }
  return h->e->debug_wgrad(A, dY, rows, K, Nc, lo, hi, dW, db, (cudaStream_t)stream);
}
int dqmc_debug_trunk_phases(dqmc_handle h, uint64_t* out, int32_t n) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (!out) { h->e->err = "dqmc_debug_trunk_phases: null output"; return 2; }
  return h->e->debug_trunk_phases(out, n);
}
int dqmc_debug_tc_error(dqmc_handle h, int32_t* flag) {
  if (!h) return 2;
  DQ_NEED_DEVICE(h);
  if (!flag) { h->e->err = "dqmc_debug_tc_error: null output"; return 2; }
  return h->e->debug_tc_error(flag);
}

int dqmc_profile_begin(dqmc_handle h) {
  if (!h) return 2;
  h->e->prof = true; h->e->prof_flops = 0; h->e->prof_n = 0;
  for (int c = 0; c < 3; ++c) { h->e->prof_cls_flops[c] = 0; h->e->prof_cls_n[c] = 0; }
  h->e->prof_cls.clear();
  return 0;
}
int dqmc_profile_end_classes(dqmc_handle h, double* ms3, double* flops3, int64_t* n3) {
  if (!h) return 2;
  double ms[3] = {0, 0, 0};
#ifndef DQMC_EMU
  for (size_t i = 0; i + 1 < h->e->prof_ev.size(); i += 2) {
    cudaEventSynchronize(h->e->prof_ev[i + 1]);
    float t = 0;
    cudaEventElapsedTime(&t, h->e->prof_ev[i], h->e->prof_ev[i + 1]);
    ms[h->e->prof_cls[i / 2]] += t;
    cudaEventDestroy(h->e->prof_ev[i]); cudaEventDestroy(h->e->prof_ev[i + 1]);
  }
  h->e->prof_ev.clear();
#endif
  h->e->prof_cls.clear();
  h->e->prof = false;
  for (int c = 0; c < 3; ++c) {
    if (ms3) ms3[c] = ms[c];
    if (flops3) flops3[c] = h->e->prof_cls_flops[c];
    if (n3) n3[c] = h->e->prof_cls_n[c];
  }
  return 0;
}
int dqmc_profile_end(dqmc_handle h, double* gemm_ms, double* gemm_flops, int64_t* n_gemm) {
  double ms[3], fl[3];
  int64_t n[3];
  const int rc = dqmc_profile_end_classes(h, ms, fl, n);
  if (rc) return rc;
  if (gemm_ms) *gemm_ms = ms[0] + ms[1] + ms[2];
  if (gemm_flops) *gemm_flops = fl[0] + fl[1] + fl[2];
  if (n_gemm) *n_gemm = n[0] + n[1] + n[2];
  return 0;
}

}  // extern "C"
