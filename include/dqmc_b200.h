/* dqmc_b200.h -- C ABI of the H100-native local-energy engine (libdqmc_b200.so).
 *
 * Drop-in boundary for the per-walker local-energy hot path of deepqmc/deepqmc.  The
 * reference has no FFI of its own (pure JAX); each entry point below names the reference
 * interface it stands in for (paths relative to the reference repo).  Conventions follow
 * what an XLA-FFI / ctypes binding needs (SURVEY.md 8b): caller-owned DEVICE pointers,
 * no allocation on the call path except the caller-provided workspace, work is enqueued on
 * the caller's cudaStream_t, every call returns an int status (0 = ok) and never throws,
 * handles are re-entrant per stream-ordered use.  Array dtype is the handle's compute dtype
 * (cfg.dtype): double for the fp64 parity mode, float for the production mode
 * (reference: src/deepqmc/__init__.py:9-34 fp32, tests/conftest.py:20 fp64).
 * Empty batches: n_walkers = 0 is a no-op for dqmc_wf_forward / dqmc_local_energy and yields a zero gradient from
 * dqmc_wf_vjp_params; the samplers need at least one walker (status 2).  Status 2 = bad argument / unsupported
 * configuration, 3 = workspace too small, other non-zero = CUDA error; dqmc_last_error gives the text.
 * Several handles (molecules of different size, electronic states, dtypes) may live in one process and be used in any
 * order; concurrent calls on ONE handle from several host threads are not supported.
 */
#ifndef DQMC_B200_H
#define DQMC_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DQMC_MAX_NUC 32
#define DQMC_MAX_ECP_TERMS 4
#define DQMC_MAX_ECP_L 4

enum { DQMC_PSIFORMER = 0, DQMC_FERMINET = 1, DQMC_TRANSPSIFORMER = 2, DQMC_PAULINET = 3 };
enum { DQMC_F64 = 0, DQMC_F32 = 1 };
enum { DQMC_GEMM_SIMT = 0, DQMC_GEMM_TCGEN05 = 1 };
enum { DQMC_MODE_FORWARD = 0, DQMC_MODE_LOCAL_ENERGY = 1, DQMC_MODE_VJP = 2, DQMC_MODE_MCMC = 3, DQMC_MODE_LANGEVIN = 4,
       DQMC_MODE_SPIN = 5, DQMC_MODE_GRAD_POS = 6, DQMC_MODE_ECP_FORCE = 7,
       DQMC_MODE_ZV_FORCE = 8 };

/* Ansatz + Hamiltonian constants that fix the kernel shapes.
 * reference: src/deepqmc/conf/ansatz/psiformer.yaml, ferminet.yaml (SURVEY.md 8(a0));
 *            src/deepqmc/hamil.py:97-154 (n_up, n_down, ns_valence, ecp_mask);
 *            src/deepqmc/ecp/gaussian_type_ecp.py:32-95 (loc/nl parameter layout). */
typedef struct dqmc_config {
  int32_t kind;            /* DQMC_PSIFORMER | DQMC_FERMINET | DQMC_TRANSPSIFORMER | DQMC_PAULINET */
  int32_t dtype;           /* DQMC_F64 | DQMC_F32 */
  int32_t gemm_backend;    /* DQMC_GEMM_SIMT | DQMC_GEMM_TCGEN05 (f32 only) */
  int32_t n_up, n_down, n_nuc;
  int32_t embedding_dim, n_layers, n_heads, n_determinants, edge_dim;
  int32_t cusp_kind;       /* 0 none, 1 PsiformerCusp (wf/cusp.py:17-26), 2 DeepQMCCusp (wf/cusp.py:5-14) */
  double cusp_same_scale, cusp_anti_scale;
  double z_valence[DQMC_MAX_NUC];                                   /* pot.ns_valence */
  int32_t ecp_mask[DQMC_MAX_NUC];
  int32_t ecp_loc_terms;                                            /* 0: plain Coulomb */
  double ecp_loc[DQMC_MAX_NUC][3][2][DQMC_MAX_ECP_TERMS];           /* [I][r^-1,r^0,r^1][alpha,beta][term] */
  int32_t ecp_nl_lmax_p1, ecp_nl_terms;
  double ecp_nl[DQMC_MAX_NUC][DQMC_MAX_ECP_L][2][DQMC_MAX_ECP_TERMS]; /* [I][l][alpha,beta][term] */
  /* DQMC_TRANSPSIFORMER (conf/ansatz/transpsiformer.yaml): envelope terms per nucleus
   * (SimplifiedNucleusDependentEnvelopes.n_envelope_per_nucleus, wf/env.py:111-226; 0/1 otherwise) and the
   * number of walker-independent nuclear attention tokens (gnn/update_features.py:385-451, elec_to_nuc =
   * false), whose per-layer key/value rows are entries "L<l>.kn" / "L<l>.vn" of the parameter table. */
  int32_t n_env_per_nuc;
  int32_t n_nuc_tokens;
  /* DQMC_PAULINET = the conv-GNN ansatz of the reference's own CPU tests (tests/conf/ansatz.yaml; BASELINE
   * configs[0]).  All zero for the other kinds. */
  int32_t factorized_det;   /* 1: det_up(n_up x n_up) det_down(n_down x n_down) (wf/nn_wave_function.py:143-151) */
  int32_t conf_linear;      /* 1: hk.Linear(1, no bias) determinant combination, entry "conf.w" (else SumPool) */
  int32_t mult_act;         /* 0 identity, 1: 1 + 2 tanh(x / 4) on the backflow (wf/nn_wave_function.py:17) */
  int32_t n_elec_types;     /* rows of the electron embedding table (gnn/electron_gnn.py:337-343) */
  int32_t jastrow_n;        /* layers of the Jastrow MLP on sum_i x_i (wf/omni.py:13-40); 0: none */
  int32_t jastrow_dims[8];  /* their widths (the last one is 1) */
  int32_t backflow_n;       /* HIDDEN layers of the per-spin backflow MLPs (wf/omni.py:43-88), ssp activation */
  int32_t backflow_dims[8]; /* their widths, padded to the larger of the two spins */
  /* conv-GNN variants (tests/conf/ansatz.yaml vs conf/ansatz/default.yaml) */
  int32_t gnn_features;     /* 0: hk.Embed lookup; 1: raw nucleus-electron features [|d|, d] (4 M wide) */
  int32_t gnn_concat;       /* 0: 'featurewise' update; 1: 'concatenate' of [h, mean_up, mean_down, conv_*] */
  int32_t gnn_conv_ne;      /* nucleus -> electron convolution present */
  int32_t gnn_sub_n;        /* layers of the w / h / u MLPs (1..4) */
  int32_t gnn_deep_edges;   /* shared edge MLP u + normalised residual between layers */
  int32_t gnn_res_norm;     /* electron residual divided by sqrt(2) */
  int32_t gnn_g_bias, gnn_w_bias;
  int32_t gnn_w_dims[8][4]; /* per layer: widths of the w MLP layers (last = edge_dim) */
  int32_t gnn_h_dims[8][4]; /* per layer: widths of the h MLP layers (last = edge_dim) */
  int32_t gnn_u_dims[8][4]; /* per layer: widths of the u MLP layers (last = edge_dim) */
  /* NuclearCuspAsymptotic (wf/cusp.py:81-101): 0 none, 1 PsiformerCusp, 2 DeepQMCCusp form with scale = nuclear
   * charge; alpha is entry "cusp.alpha_nuc", the charges are z_nuclear (all kinds) */
  int32_t nuc_cusp_kind;
  double z_nuclear[DQMC_MAX_NUC];
  /* BackflowOp branches (wf/nn_wave_function.py:14-33,111-125 backflow_transform): 0 'mult' (every shipped config),
   * 1 'add', 2 'both'.  With an additive branch the heads "bf.up" / "bf.dn" are [d][K N] ('add') or
   * [d][2 K N] ('both': multiplicative head first), add_act = 0.1 tanh(x / 4), with_envelope = true.
   * Linear-head ansatz kinds (Psiformer, FermiNet, TransPsiformer) only. */
  int32_t backflow_add;
  /* DeepErwin conv-GNN variant (conf/ansatz/deeperwin.yaml); all zero for the other kinds. */
  int32_t gnn_sep_edges;    /* deep_features 'separate': one u MLP per edge type, entries "G<l>.u_<type>.<i>" */
  int32_t gnn_self_edges;   /* self_interaction: the same-spin edges include (i, i), |d| = sqrt(eps) constant */
  int32_t gnn_ne_identity;  /* w_for_ne = false: the ne edge stream is the filter of the ne convolution, and the
                             * electron-electron convolutions enter the update as one sum conv_same + conv_anti ('ee') */
  int32_t gnn_no_res;       /* electron_residual = false: x <- tanh(g(...)) */
  int32_t gnn_edge_in[3];   /* raw feature widths of the same / anti / ne edges: 1 = [|d|], 4 = [|d|, d]; 0 reads 4 */
} dqmc_config;

typedef struct dqmc_engine* dqmc_handle;

/* Build / tear down an engine bound to one CUDA device.  device < 0 builds a PLAN-ONLY engine: no CUDA context and no
 * allocation; only the parameter-table queries, dqmc_workspace_bytes and dqmc_debug_plan work on it (every compute entry
 * point returns status 2).
 * replaces: app.py:82-105 instantiate_ansatz + hamil.py:97-154 MolecularHamiltonian.__init__ */
int dqmc_create(const dqmc_config* cfg, int device, dqmc_handle* out);
int dqmc_destroy(dqmc_handle h);
const char* dqmc_last_error(dqmc_handle h);
const char* dqmc_version(void);

/* Parameter table: the engine's packed layout (one fp64 host buffer, converted on upload).
 * replaces: the Haiku params pytree passed to Ansatz.apply (types.py:133-150). */
int dqmc_param_count(dqmc_handle h);
int dqmc_param_entry(dqmc_handle h, int idx, char* name, int name_len, int64_t* offset, int32_t* rows,
                     int32_t* cols);
int64_t dqmc_param_total(dqmc_handle h);
int dqmc_set_params(dqmc_handle h, const double* host_params, int64_t n, void* stream);

/* Workspace the caller must provide for n_walkers in one call of the entry point `mode` names (bytes; DQMC_MODE_MCMC =
 * dqmc_mcmc_sweep(_exchange), DQMC_MODE_LANGEVIN = dqmc_langevin_sweep, proposal buffers included).  The engine chunks
 * walkers internally if given less (>= dqmc_workspace_bytes_min(h, n_walkers, mode) required).  The figure is computed by a dry pass of
 * the code that carves the workspace, so plan and use cannot drift apart.
 * replaces: XLA buffer assignment / loss/energy.py:44-48 local_energy_batch_size chunking. */
int64_t dqmc_workspace_bytes(dqmc_handle h, int32_t n_walkers, int32_t mode);
/* The least workspace with which a call for n_walkers proceeds at all (walkers processed one at a time). */
int64_t dqmc_workspace_bytes_min(dqmc_handle h, int32_t n_walkers, int32_t mode);

/* psi(r) for a batch of walkers.  r[B][N][3], R[M][3] (R_batched = 0) or R[B][M][3].
 * replaces: vmap(ansatz.apply)(params, phys_conf) -> Psi(sign, log)
 *           (types.py:133-150; wf/nn_wave_function.py:127-173; callers
 *           sampling/electron_samplers.py:76-81). */
int dqmc_wf_forward(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers,
                    void* out_sign, void* out_log, void* workspace, int64_t workspace_bytes, void* stream);

/* Local energies.  out_stats[6][B] = V_el, E_kin, V_loc, V_nl, lap, quantum_force^2
 * (hamil.py:172-180 order); out_grad[B][3N] (nullable) = grad log|psi| (quantum force).
 * ecp_twist (nullable) = injected quadrature twists [B][J][N] in [0, pi/5) replacing the
 * rng stream (gaussian_type_ecp.py:217-223); otherwise Philox(seed).
 * replaces: loss/energy.py:19-60 compute_local_energy -> hamil.py:156-184 local_energy
 *           -> physics.py:79-109 kinetic_term with a forward-Laplacian factory
 *           (conf/hamil/qc_forward_laplacian.yaml). */
int dqmc_local_energy(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers,
                      uint64_t seed, const void* ecp_twist, void* out_E, void* out_stats, void* out_sign,
                      void* out_log, void* out_grad, void* workspace, int64_t workspace_bytes, void* stream);

/* Orbital matrices of a plain forward: out_orbitals[B][K][N][N] (determinant k, electron i, orbital mu) =
 * envelope * mult_act(backflow), the matrices whose determinants dqmc_wf_forward takes.  With spin-factorised
 * determinants the spin-off-diagonal blocks are zero; the caller slices the n_up x n_up / n_down x n_down blocks.
 * Workspace: dqmc_workspace_bytes(h, B, DQMC_MODE_FORWARD).
 * replaces: Ansatz.apply(params, phys_conf, return_mos=True) (types.py:133-150, wf/nn_wave_function.py:131-142;
 *           caller pretrain/pretraining.py:73-78). */
int dqmc_wf_orbitals(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers, void* out_orbitals,
                     void* workspace, int64_t workspace_bytes, void* stream);

/* n_sub Metropolis sub-steps on the walker state {r, sign, log, age, tau} (updated in place).
 * noise_normal[n_sub][B][N][3] / noise_uniform[n_sub][B] (nullable): injected random numbers.
 * out_stats[7] (device, compute dtype) = acceptance, tau, age mean, age max, log|psi| mean,
 * log|psi| std, mean e-e distance of the LAST sub-step.
 * replaces: sampling/electron_samplers.py:140-163 MetropolisSampler.sample inside
 *           :347-357 DecorrSampler.sample (lax.scan of `length` sub-steps). */
int dqmc_mcmc_sweep(dqmc_handle h, void* r, void* sign, void* log, int32_t* age, void* tau, const void* R,
                    int32_t R_batched, int32_t n_walkers, int32_t n_sub, double target_acceptance, int32_t max_age,
                    uint64_t seed, uint64_t step0, uint64_t walker_offset, const void* noise_normal,
                    const void* noise_uniform, void* out_stats, void* workspace, int64_t workspace_bytes,
                    void* stream);

/* dqmc_mcmc_sweep with spin-exchange steps mixed in: every sub-step is, for the whole batch, an exchange step with
 * probability exchange_step_probability (proposal = swap the positions of one random spin-up / spin-down pair per walker,
 * acceptance 2 dlog|psi| > log u, no max_age override, no step-size adaptation) and an ordinary Metropolis step otherwise.
 * exchange_flags[n_sub] (HOST int32, nullable) / exchange_idx[n_sub][B][2] (device int32, nullable): injected decisions and
 * (up, down) indices for parity tests.
 * replaces: sampling/electron_samplers.py:235-330 OppositeSpinExchangeSampler chained in front of MetropolisSampler
 *           (conf/task/sampler_factory/elec_sampler/decorr_spin_exchange_metropolis.yaml). */
int dqmc_mcmc_sweep_exchange(dqmc_handle h, void* r, void* sign, void* log, int32_t* age, void* tau, const void* R,
                             int32_t R_batched, int32_t n_walkers, int32_t n_sub, double target_acceptance, int32_t max_age,
                             uint64_t seed, uint64_t step0, uint64_t walker_offset, const void* noise_normal,
                             const void* noise_uniform, double exchange_step_probability, const int32_t* exchange_flags,
                             const int32_t* exchange_idx, void* out_stats, void* workspace, int64_t workspace_bytes,
                             void* stream);

/* Metropolis-adjusted Langevin sweep: like dqmc_mcmc_sweep with the drift force[B][N][3] (= clean_force of
 * grad log|psi|, sampling_utils.py:71-101) as an extra piece of walker state; proposals r + tau F + sqrt(tau) N(0,1),
 * acceptance with the Green's-function ratio.  Every sub-step costs one forward-Laplacian pass (value + gradient).
 * n_sub = 0 recomputes sign / log / force of the walkers in place (ElectronSampler.update).
 * replaces: sampling/electron_samplers.py:176-232 LangevinSampler (inside DecorrSampler). */
int dqmc_langevin_sweep(dqmc_handle h, void* r, void* sign, void* log, void* force, int32_t* age, void* tau, const void* R,
                        int32_t R_batched, int32_t n_walkers, int32_t n_sub, double target_acceptance, int32_t max_age,
                        uint64_t seed, uint64_t step0, uint64_t walker_offset, const void* noise_normal,
                        const void* noise_uniform, void* out_stats, void* workspace, int64_t workspace_bytes, void* stream);

/* Parameter VJP of the wave function: out_grad_params[dqmc_param_total] (compute dtype, the packed layout of
 * dqmc_param_entry) = d/dparams sum_b weights[b] log|psi(r_b)|; also returns sign/log of the batch.
 * With weights = 2 (E_loc - <E_loc>) / B this is the energy gradient (all ansatz kinds; no additive backflow branch).
 * replaces: loss/loss_function.py:53-82 compute_log_psi_tangent / jax.grad through ansatz.apply,
 *           loss/energy.py:77-102 compute_mean_energy_tangent. */
int dqmc_wf_vjp_params(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers,
                       const void* weights, void* out_sign, void* out_log, void* out_grad_params, void* workspace,
                       int64_t workspace_bytes, void* stream);

/* Total spin <S^2> per walker -> out_s2[B].
 *   down_idx = -1: exact estimator over all n_up n_down (up a, down b) pairs,
 *                  s2 = D/2 (D/2 + 1) + n_down - sum_{a,b} rho_ab,  D = n_up - n_down;
 *   down_idx in [n_up, N): spin-raising contribution 1 - sum_a rho_{a,down_idx}.
 * rho = sign' sign exp(log' - log), (sign', log') = psi with the positions of a and b swapped, formed and summed in fp64
 * in a fixed order (a repeated call is bitwise identical).  sign / log [B] of the base walkers are given together or both
 * null (null: a plain forward inside the call; exactly one of them: status 2).  out_ratio [B][P] (nullable) receives rho:
 * P = n_up n_down with p = a n_down + (b - n_up), or P = n_up with p = a.  Every swapped walker is one plain forward.
 * Psiformer engines take the N - 2 unmoved electrons' envelope rows (slater_fwd2_kernel) and embedding rows (whole-trunk
 * kernel; the two swapped rows are formed from the table as emb(r, +-1) = emb(r, -+1) +- 2 w_spin) from tables of the base
 * walkers; the other kinds run dqmc_wf_forward's path on the swapped walkers.  Walkers are grouped to fit the workspace,
 * one walker's pairs split across forward chunks if need be.  n_walkers = 0 is a no-op; n_down = 0 gives the constant
 * D/2 (D/2 + 1) without forwards (and needs no workspace) for down_idx = -1, and status 2 otherwise.  Status 2 also for
 * down_idx out of range and for R_batched = 1.  Workspace: dqmc_workspace_bytes(h, B, DQMC_MODE_SPIN).
 * replaces: physics.py:159-239 evaluate_spin / make_stochastic_spin_raising_operator (observable.py:193-200 SpinMonitor,
 *           loss/spin.py). */
int dqmc_spin(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers, const void* sign,
              const void* log, int32_t down_idx, void* out_s2, void* out_ratio, void* workspace, int64_t workspace_bytes,
              void* stream);

/* Position gradients of log|psi| per walker: out_grad_r[B][N][3] = grad_r log|psi|, out_grad_R[B][M][3] = grad_R log|psi|
 * (either nullable), plus sign / log [B] (required).  The reverse pass of dqmc_wf_vjp_params with cotangent 1 per walker and no
 * parameter gradients, carried on through the electron-nucleus features, the envelopes and the cusps into the pair cotangent
 * c_im = d log|psi| / d(r_i - R_m); grad_{r_i} = sum_m c_im + the e-e terms, grad_{R_m} = -sum_i c_im.  No atomics: every sum
 * runs in a fixed order, a repeated call is bitwise identical.  Psiformer and FermiNet: both outputs; TransPsiformer: grad_r
 * only (its nuclear tokens and envelope exponents depend on R through the host-side nuclear stream; a non-null out_grad_R is
 * status 2); conv-GNN kinds and the additive backflow branch: status 2.  n_walkers = 0 is a no-op.
 * Workspace: dqmc_workspace_bytes(h, B, DQMC_MODE_GRAD_POS) (walkers are chunked to fit).
 * replaces: force.py:96-118 make_grad_nuc_log_wf / make_grad_log_wf (jax.grad of wf(...).log with respect to R and r). */
int dqmc_wf_grad_positions(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers,
                           void* out_sign, void* out_log, void* out_grad_r, void* out_grad_R,
                           void* workspace, int64_t workspace_bytes, void* stream);

/* Closed-form force terms per walker [B][M][3] (device, every output nullable), d_im = r_i - R_m, Z = the nuclear charges:
 *   out_bare = F_nuc + Z_m sum_i d_im / |d_im|^3                    (bare Hellmann-Feynman force, all-electron)
 *   out_zvq  = F_nuc + sum_i (dQ_m / dr_i)^T grad_i log|psi|        (needs grad_r[B][N][3]; otherwise status 2)
 *   out_Q    = Q_m = Z_m sum_i d_im / |d_im|
 * F_nuc = -grad_R E_nuc (eps-safe nucleus-nucleus distances); dQ_ma / dr_ib = Z_m (delta_ab / |d| - d_a d_b / |d|^3).
 * Engines with an effective core potential (local or non-local) or a pseudo-Hamiltonian return status 2.  One block per
 * walker, sums in a fixed order.
 * replaces: force.py:30-38 nuclear_force, :122-132 Q, :172-194 make_bare_plus_zvq_term, :252-301 evaluate_hf_force_bare
 *           (all-electron part). */
int dqmc_force_terms(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers,
                     const void* grad_r, void* out_bare, void* out_zvq, void* out_Q, void* stream);

/* Hellmann-Feynman force terms with effective core potentials, per walker [B][M][3] (device, both outputs nullable):
 *   out_bare = F_nuc(Z_eff) - grad_R V_loc: dqmc_force_terms' out_bare with the local ECP's Gaussian terms added (equal to it
 *              on an all-electron engine); any ansatz kind.
 *   out_nl   = -grad_R V_nl (the reference's -grad_nonloc_potential): for every nucleus I with a non-local term and electron i,
 *              d/dR_I of v_l(|r_i - R_I|) (2l+1)/12 sum_q P_l(cos th_q) psi(r_q(R), R) / psi(r, R), where the quadrature point
 *              r_q moves with R_I and psi depends on R_I explicitly, in the numerator and the denominator; rows of nuclei
 *              without a non-local term are zero.  Written into row I, the nucleus' own row (the reference writes row j, the
 *              nucleus' index among the non-local nuclei; the two agree when those nuclei come first).  Needs grad_r and
 *              grad_R of log|psi| by the reverse pass: Psiformer and FermiNet with multiplicative backflow; the other kinds,
 *              R_batched = 1 and a non-null out_nl return status 2.
 * Quadrature twists: seed / ecp_twist [B][J][N] as in dqmc_local_energy, so the same seed gives the energy pass's
 * quadrature points.  Pairs beyond the force's cutoff radius (the weight sum_l (2l+1) sum_t |beta| exp(-alpha rho^2) and its
 * radial derivative below 2^-100; DQMC_ECP_CUTOFF=0: none) add nothing and run no reverse pass; their quadrature walkers
 * count in dqmc_ecp_forward_count.  Every sum runs in a fixed order without atomics: a repeated call is bitwise identical.
 * Pseudo-Hamiltonians: status 2.  n_walkers = 0 is a no-op.
 * Workspace: dqmc_workspace_bytes(h, B, DQMC_MODE_ECP_FORCE) (0 where out_nl has nothing to compute; walkers are grouped
 * and the reverse passes chunked to fit).
 * replaces: force.py:252-301 evaluate_hf_force_bare with a GaussianTypeECP (local_potential gradient,
 *           ecp/gaussian_type_ecp.py:257-328 grad_nonloc_potential, ecp/ecp_force_utils.py). */
int dqmc_ecp_force(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers, uint64_t seed,
                   const void* ecp_twist, void* out_bare, void* out_nl, void* workspace, int64_t workspace_bytes, void* stream);

/* Zero-variance term of the AC-ZV / AC-ZVZB force estimators per walker [B][M][3] (device):
 *   out_zv     = -dT/dR = 1/2 d/dR (Lap_r log|psi| + |grad_r log|psi||^2) at fixed electron positions, T the local kinetic
 *                energy (stats E_kin of dqmc_local_energy).  With an all-electron Hamiltonian the potential cancels in the
 *                reference's -(E'_kappa - E_loc) g_kappa (E'_kappa: local energy of d psi / dR_kappa, g_kappa = d log|psi| / dR_kappa)
 *                when E_loc is the walker's exact local energy; this closed form needs no division by g_kappa and no E_loc.
 *   out_grad_R = grad_R log|psi| (nullable), the companion of the value slot (equal to dqmc_wf_grad_positions' grad_R).
 * Each nuclear coordinate runs a forward-Laplacian pass with a companion state dX/dR of every activation beside it
 * (kernels_zv.cuh).  Psiformer and FermiNet with multiplicative backflow (nuclear cusp included), shared or per-walker R;
 * the TransPsiformer, the conv-GNN kinds, the additive backflow branch, engines with an effective core potential and
 * pseudo-Hamiltonians return status 2.  Every sum runs in a fixed order without atomics: a repeated call is bitwise
 * identical.  n_walkers = 0 is a no-op.  Workspace: dqmc_workspace_bytes(h, B, DQMC_MODE_ZV_FORCE) (walkers are chunked to fit).
 * replaces: force.py:135-169 make_zv_term_via_jvp (the local energy of the nuclear-JVP wave function, scanned over the 3M
 *           tangents), used by :304-411 evaluate_hf_force_ac_zv / evaluate_hf_force_ac_zvzb. */
int dqmc_zv_force(dqmc_handle h, const void* r, const void* R, int32_t R_batched, int32_t n_walkers, void* out_zv,
                  void* out_grad_R, void* workspace, int64_t workspace_bytes, void* stream);

/* Switch the handle's Hamiltonian to a pseudo-Hamiltonian (fully local replacement of the semi-local ECP):
 * tables[n_tab][2][n_grid] (host, fp64) = r V_loc(r) and r V_L2(r) per tabulated element on the uniform grid
 * [0, r_max]; tab_of_nuc[n_nuc] = table index of each nucleus or -1.  z_valence of the config carries the
 * effective charges.  dqmc_local_energy then evaluates  sum_i [A(r_i) : Hess_i + b(r_i) . grad_i] psi / psi  with
 * A = 1/2 + sum_I (r V_L2 |d| 1 - V_L2 d d^T), b = 2 sum_I V_L2 d  by seeding the forward-Laplacian tangents with
 * the Cholesky factor of A, and adds r V_loc / r to V_loc; stats lap / quantum_force are those of the transformed
 * coordinates as in the reference.  Call once after dqmc_create (changes the workspace size).
 * replaces: ecp/pseudo_hamiltonian.py:165-278 PseudoHamiltonian.{local_potential, kinetic_term},
 *           :71-112 load_PH_functions (RegularGridInterpolator tables). */
int dqmc_set_pseudo_hamiltonian(dqmc_handle h, int32_t n_tab, int32_t n_grid, double r_max, const double* tables,
                                const int32_t* tab_of_nuc);

/* This rank's contribution to the per-step statistics in ONE launch: out11[0] = sum E_loc, [1] = sum E_loc^2,
 * [2] = n_walkers, [3..8] = sums of the six rows of `stats` (dqmc_local_energy's out_stats[6][B]; nullable),
 * [9] = max E_loc, [10] = -min E_loc, fp64 on the device.  The caller exchanges the 11 doubles with one all-gather
 * (deepqmc_b200/parallel.py) -- the only per-step collective of the data-parallel path.
 * replaces: loss/energy.py:63-74 (pmean of the mean energy), observable.py:474-479, parallel.py:239-245. */
int dqmc_stats_pack(dqmc_handle h, const void* E_loc, const void* stats, int32_t n_walkers, double* out11, void* stream);

/* Self-test hook (host only, also on plan-only engines): *planned_bytes = dqmc_workspace_bytes(h, n_walkers, mode);
 * *carved_bytes = the highest workspace offset the entry point of `mode` carves when it is given workspace_bytes bytes
 * (<= 0: the planned size) -- found by walking that entry point's host code with every CUDA call skipped.
 * Status 3 if that workspace is too small for one walker.  tests/test_plan.py sweeps ansatz kind x mode x batch size x
 * dtype and asserts carved <= given.  No reference analogue (XLA assigns buffers itself). */
int dqmc_debug_plan(dqmc_handle h, int32_t n_walkers, int32_t mode, int64_t workspace_bytes, int64_t* planned_bytes,
                    int64_t* carved_bytes);

/* Number of kernels this handle has launched so far (bench.py's gpu_launches claim). */
int64_t dqmc_launch_count(dqmc_handle h);
/* Number of non-local ECP quadrature forwards (virtual walkers, 12 per active electron-nucleus pair) this handle has run so far
   in local-energy and dqmc_ecp_force calls: pairs beyond the nucleus' cutoff radius run none (DQMC_ECP_CUTOFF=0: every pair runs). */
int64_t dqmc_ecp_forward_count(dqmc_handle h);

/* Self-test hook: run ONE dense-layer row GEMM  C = (Res) + A @ W[weight] (+ bias on value rows)
 * with the named weight of the handle's parameter table, on the requested backend
 * (DQMC_GEMM_SIMT | DQMC_GEMM_TCGEN05).  A[rows][K], Res/C[rows][N] device arrays in the compute
 * dtype; sliced = 1 exercises the per-spin backflow mapping (weight "bf.up"/"bf.dn", rows = B*S).
 * Used by tests to validate the wgmma 3xTF32 kernel against the CUDA-core kernel and fp64.
 * No reference analogue (the reference's dense layers are hk.Linear -> XLA dot). */
int dqmc_debug_gemm(dqmc_handle h, const char* weight, const char* bias, const void* A, const void* Res, void* C,
                    int32_t rows, int32_t S, int32_t sliced, int32_t backend, void* stream);

/* Self-test hook: ONE launch of the fused plain-forward MLP block of layer `layer` (Psiformer kinds, fp32 tensor-core
 * backend, embedding_dim 128 | 256):  Out = A + tanh(tanh(A W1 + b1) W2 + b2),  A = X + O Wo,  O / X / Out [rows][d] device
 * arrays (Out may alias O).  Status 2 if the configuration has no fused block.
 * reference: gnn/update_features.py:241-286 (attention output projection + residual, MLP + residual), hkext.py:22-137. */
int dqmc_debug_mlp_block(dqmc_handle h, int32_t layer, const void* O, const void* X, void* Out, int32_t rows, void* stream);

/* Self-test hook: ONE launch of the whole-trunk kernel of a plain forward (deepqmc_b200/csrc/trunk_tc.cuh; fp32 engines with the
 * tensor-core backend and the shipped Psiformer shape: embedding_dim 256, 4 heads of 64, N <= 32 electrons): every attention layer
 * (QKV projection, softmax attention, output projection + residual, tanh-MLP + residual) applied to the embedding rows
 * X0 [rows][256] (rows = walkers x electrons, walker-major), result Out [rows][256].  Status 2 if the configuration has none.
 * reference: gnn/electron_gnn.py:403-432 (layer loop), gnn/update_features.py:241-286, hkext.py:22-137, :215-253. */
int dqmc_debug_trunk(dqmc_handle h, const void* X0, void* Out, int32_t rows, void* stream);

/* Self-test hook: the softmax attention of layer `layer` with S slots per electron, run by the kernel the engine picks for it
 * (the same Engine::attention the forward calls), on caller-supplied rows QKV [rows][3d] (Q | K | V, head h in columns
 * h dh .. h dh + dh - 1 of each) -> O [rows][d].  rows = walkers x electrons x S in the engine's slot layout: row
 * (b N + i) S + s holds slot s of electron i of walker b.  S = 1: plain forward (fp32, dh = 64, N + nuclear tokens <= 48: the
 * tensor-core attn_fwd_mma_kernel; otherwise the forward-Laplacian kernel of the configuration with one slot).  S = 3N + 2: forward-Laplacian pass, slot 0 the value, slots 1 .. 3N the tangents, slot
 * 3N + 1 the Laplacian (the tangent chunk and the shared memory were sized for this S when the engine was created).
 * TransPsiformer: the keys and values also hold the layer's nuclear tokens from the parameter table (L<layer>.kn / .vn).
 * *kernel (if not null) receives the kernel that ran, one of DQMC_ATTN_KERNEL_*.
 * Status 2 for kinds without softmax attention, a layer out of range, S other than 1 or 3N + 2, or rows not a multiple of N S.
 * reference: gnn/update_features.py:273-280 (hk.MultiHeadAttention), algebra hkext.py:215-253; derivative rules
 * folxext.py:70-171. */
enum {
  DQMC_ATTN_KERNEL_MMA = 0,     /* attn_fwd_mma_kernel: 3xFP16 mma.sync, fp32 dh = 64, N + nuclear tokens <= 48 */
  DQMC_ATTN_KERNEL_FL_F32 = 1,  /* attn_fl_f32_kernel<., ., false>: fp32 forward-Laplacian attention, SIMT tangent chunks */
  DQMC_ATTN_KERNEL_GENERIC = 2, /* attn_fl_kernel<T, false>: generic, any dtype, SIMT */
  DQMC_ATTN_KERNEL_FL_F32_MMA = 3,  /* attn_fl_f32_kernel<., ., true>: tangent chunks as 3xTF32 mma.sync products */
  DQMC_ATTN_KERNEL_GENERIC_MMA = 4  /* attn_fl_kernel<float, true>: generic fp32 kernel, tangent chunks on the tensor cores */
};
int dqmc_debug_attention(dqmc_handle h, int32_t layer, const void* QKV, void* O, int32_t rows, int32_t S, int32_t* kernel,
                         void* stream);

/* Self-test hook: what follows the attention in layer `layer`, with S slots per electron (1 or 3N + 2, rows in the layout of
 * dqmc_debug_attention), run by the same Engine::mlp the forward calls:  A = X + O Wo;  M1 = tanh(A W1 + b1);
 * Out = A + tanh(M1 W2 + b2), the tanh with its forward-Laplacian propagation for S > 1 (y_t = y' z_t,
 * y_L = y' z_L + y'' sum_t z_t^2).  O / X / Out [rows][d] device arrays; scratch: 2 rows d elements (A and M1).
 * *path (if not null) receives the path that ran, one of DQMC_MLP_PATH_*.
 * Status 2 for kinds without attention layers, a layer out of range, S other than 1 or 3N + 2, or rows not a multiple of N S.
 * reference: gnn/update_features.py:241-286, hkext.py:22-137 (MLP), :104-113 (activation). */
enum {
  DQMC_MLP_PATH_BLOCK = 0,      /* plain forward: one fused MLP-block launch (fused_tc.cuh) */
  DQMC_MLP_PATH_GEMM_ACT = 1,   /* 3xTF32 row GEMMs, tanh (+ forward-Laplacian rule) in the W1 / W2 epilogues */
  DQMC_MLP_PATH_GEMM_TANH = 2,  /* 3xTF32 row GEMMs, tanh_fl_kernel after W1 and W2 */
  DQMC_MLP_PATH_SIMT_TANH = 3   /* CUDA-core gemm_kernel, tanh_fl_kernel after W1 and W2 */
};
int dqmc_debug_mlp(dqmc_handle h, int32_t layer, int32_t S, const void* O, const void* X, void* Out, void* scratch, int32_t rows,
                   int32_t* path, void* stream);

/* Self-test hook: the Slater determinants of the engine, run by the same Engine::slater the forward tails call: the backflow
 * activation (mult_act, the additive head's add_act and its electron factor) and the determinant kernel the engine picks for
 * the shape, on caller-supplied inputs.  r [B][N][3] walker positions, R [M][3] the nuclei; BF [rows][BFW] the backflow head
 * rows BEFORE activation, exactly as the bf.up / bf.dn GEMM writes them: rows = B N S, row (b N + i) S + s; BFW = K N, or
 * 2 K N with backflow_transform 'both' (the multiplicative head, then the additive one).  The activation runs on a copy: BF
 * is not changed.  S = 1: plain forward; S = 3N + 2: slot 0 the value, slots 1 .. 3N the r-tangents, slot 3N + 1 the
 * r-Laplacian.  Outputs det_sign / det_log [B][K] (slogdet convention: an exactly singular matrix gives sign 0, log -inf);
 * for S = 3N + 2 also det_grad [B][K][3N] and det_lap [B][K] (not meaningful where the matrix is singular).
 * kernel (if not null) receives two values: the kernel that ran, one of DQMC_SLATER_KERNEL_*, and its template instance (NS
 * of slater_small_kernel, NM of slater_fwd2_kernel, 0 for the runtime-N kernels).
 * Status 2 for S other than 1 or 3N + 2, rows not a positive multiple of N S, or null arrays.
 * reference: wf/env.py:57-75, wf/nn_wave_function.py:14-33, :111-151. */
enum {
  DQMC_SLATER_KERNEL_SMALL = 0,    /* slater_small_kernel<NS>: one thread per determinant, N <= 4 (fp32: N <= 6) */
  DQMC_SLATER_KERNEL_FWD2 = 1,     /* slater_fwd2_kernel<NM>: persistent plain forward, N <= 32 */
  DQMC_SLATER_KERNEL_FWD_REG = 2,  /* slater_fwd_reg_kernel: plain forward, lane = row, when fwd2 does not fit */
  DQMC_SLATER_KERNEL_GENERIC = 3   /* slater_kernel: warp Gauss-Jordan with an explicit inverse, every other case */
};
int dqmc_debug_slater(dqmc_handle h, const void* r, const void* R, const void* BF, int32_t rows, int32_t S, void* det_sign,
                      void* det_log, void* det_grad, void* det_lap, int32_t* kernel, void* stream);

/* Self-test hook: the determinant sum (finalize_kernel with the engine's cusp, conf_coeff and nuclear-cusp settings; no
 * Jastrow, no pseudo-Hamiltonian) on caller-supplied determinants det_sign / det_log [B][K], and for S = 3N + 2 det_grad
 * [B][K][3N] / det_lap [B][K]; r [B][N][3], R [M][3] as in dqmc_debug_slater (the e-e cusp and the potentials read them).
 * -> sign / logp [B] (log|psi| = log|sum_k c_k s_k exp(l_k)|, sign 0 and log -inf when the sum vanishes); for S = 3N + 2
 * also grad [B][3N] = grad log|psi| and stats [6][B] in the layout of dqmc_local_energy (stats[4] = lap log|psi|,
 * stats[5] = |grad log|psi||^2).  Status 2 for S other than 1 or 3N + 2, B < 1, or null arrays.
 * reference: wf/nn_wave_function.py:152-171. */
int dqmc_debug_det_sum(dqmc_handle h, const void* r, const void* R, const void* det_sign, const void* det_log,
                       const void* det_grad, const void* det_lap, int32_t B, int32_t S, void* sign, void* logp, void* grad,
                       void* stats, void* stream);

/* Self-test hook: the softmax attention backward of layer `layer` (plain forward), run by the same Engine::attention_bwd the
 * parameter and position reverse passes call, on caller-supplied Q | K | V rows QKV [rows][3d] (layout of dqmc_debug_attention
 * with S = 1) and output cotangents dO [rows][d] -> dQKV [rows][3d] (dQ | dK | dV).  TransPsiformer: the keys and values also
 * hold the layer's nuclear tokens from the parameter table, and the cotangents of those tokens are ADDED over every walker into
 * dKn / dVn [Mn][d] (caller-zeroed; not read without nuclear tokens).  Status 2 for kinds without softmax attention, a layer out
 * of range, rows not a positive multiple of N, or missing dKn / dVn.  reference: the cotangents jax.grad takes through
 * hk.MultiHeadAttention (gnn/update_features.py:273-280). */
int dqmc_debug_attention_bwd(dqmc_handle h, int32_t layer, const void* QKV, const void* dO, void* dQKV, void* dKn, void* dVn,
                             int32_t rows, void* stream);

/* Self-test hook: the weight- and bias-gradient reductions of the reverse passes (Engine::wgrad / Engine::bgrad, the row split
 * the reverse passes use) on caller-supplied A [rows][K] and dY [rows][Nc]:  dW [K][Nc] += A^T dY and db [Nc] += column sums of
 * dY, over the rows (b N + i) whose electron i lies in [lo, hi) (N of the handle; the per-spin backflow heads), or over every row
 * with hi = -1.  An empty range (lo = hi) adds nothing.  dW / db must be zeroed by the caller to read the sums.
 * Status 2 for rows, K or Nc < 1, or a range outside [0, N].  reference: the parameter cotangents jax.grad takes through
 * hk.Linear. */
int dqmc_debug_wgrad(dqmc_handle h, const void* A, const void* dY, int32_t rows, int32_t K, int32_t Nc, int32_t lo, int32_t hi,
                     void* dW, void* db, void* stream);

/* Measurement aid: the phase timers of the whole-trunk kernel, summed over every launch since the last call, then reset.  On
 * only for an engine created with DQMC_TRUNK_PHASES=1 in the environment (status 2 otherwise); n >= 13.  out[0..11]: clock64()
 * cycles of the consumer warpgroups in tile load, QKV mainloop, QKV epilogue, attention, Wo mainloop, Wo epilogue, W1
 * mainloop, W1 epilogue, W2 mainloop, W2 epilogue, waiting for weight slots (not part of the mainloops), waiting for the
 * tensor-core lock; out[12]: the number of (tile, layer) pairs processed. */
int dqmc_debug_trunk_phases(dqmc_handle h, uint64_t* out, int32_t n);

/* Self-test hook: the error word of the whole-trunk and fused MLP-block kernels since the engine was created or the last
 * call (synchronous), then reset; *flag = 0: no error.  A kernel sets it when a wait passes its bound (the tensor-core lock:
 * the warpgroup goes on without it, the results are unchanged).  Status 2 for an engine without the tensor-core backend. */
int dqmc_debug_tc_error(dqmc_handle h, int32_t* flag);

/* Measurement aid (bench.py roofline): between begin/end every dense-layer GEMM launch is
 * bracketed by CUDA events on the caller's stream; end() returns their summed duration [ms],
 * the algorithmic flops they performed (2*M*N*K each) and their count.  No reference analogue
 * (the reference ships no profiler hooks, SURVEY.md 5). */
int dqmc_profile_begin(dqmc_handle h);
int dqmc_profile_end(dqmc_handle h, double* gemm_ms, double* gemm_flops, int64_t* n_gemm);
/* Same, split by kernel class (arrays of 3): [0] row GEMM (one dense layer per launch), [1] fused MLP block,
 * [2] whole-trunk kernel (all layers incl. attention in one launch). */
int dqmc_profile_end_classes(dqmc_handle h, double* ms3, double* flops3, int64_t* n3);

#ifdef __cplusplus
}
#endif
#endif /* DQMC_B200_H */
