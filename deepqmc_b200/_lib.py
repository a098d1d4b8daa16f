"""ctypes binding of libdqmc_b200.so (C ABI declared in include/dqmc_b200.h).

The shared library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).  There is
NO fallback: if the library is missing or a symbol cannot be resolved, importing the engine
raises.  ``load(path)`` with an explicit path exists only so the development-time CPU emulator
build (tools/emu_check.py) can drive the same host code; the product never passes a path.
"""
from __future__ import annotations

import ctypes as C
import os

MAX_NUC, MAX_T, MAX_L = 32, 4, 4
LIB_NAME = 'libdqmc_b200.so'
LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), LIB_NAME)

SYMBOLS = [
    'dqmc_create', 'dqmc_destroy', 'dqmc_last_error', 'dqmc_version', 'dqmc_param_count',
    'dqmc_param_entry', 'dqmc_param_total', 'dqmc_set_params', 'dqmc_workspace_bytes',
    'dqmc_wf_forward', 'dqmc_local_energy', 'dqmc_mcmc_sweep', 'dqmc_launch_count',
    'dqmc_profile_begin', 'dqmc_profile_end', 'dqmc_debug_gemm', 'dqmc_wf_vjp_params', 'dqmc_langevin_sweep',
    'dqmc_set_pseudo_hamiltonian', 'dqmc_wf_orbitals', 'dqmc_mcmc_sweep_exchange',
    'dqmc_workspace_bytes_min', 'dqmc_debug_plan', 'dqmc_stats_pack', 'dqmc_debug_mlp_block', 'dqmc_debug_trunk',
    'dqmc_profile_end_classes', 'dqmc_debug_trunk_phases', 'dqmc_debug_attention', 'dqmc_debug_mlp',
    'dqmc_debug_slater', 'dqmc_debug_det_sum', 'dqmc_spin', 'dqmc_ecp_forward_count', 'dqmc_wf_grad_positions',
    'dqmc_force_terms', 'dqmc_ecp_force', 'dqmc_debug_wgrad', 'dqmc_zv_force',
    'dqmc_debug_attention_bwd', 'dqmc_debug_tc_error',
]


class DqmcConfig(C.Structure):
    _fields_ = [
        ('kind', C.c_int32), ('dtype', C.c_int32), ('gemm_backend', C.c_int32),
        ('n_up', C.c_int32), ('n_down', C.c_int32), ('n_nuc', C.c_int32),
        ('embedding_dim', C.c_int32), ('n_layers', C.c_int32), ('n_heads', C.c_int32),
        ('n_determinants', C.c_int32), ('edge_dim', C.c_int32),
        ('cusp_kind', C.c_int32), ('cusp_same_scale', C.c_double), ('cusp_anti_scale', C.c_double),
        ('z_valence', C.c_double * MAX_NUC), ('ecp_mask', C.c_int32 * MAX_NUC),
        ('ecp_loc_terms', C.c_int32), ('ecp_loc', C.c_double * (MAX_NUC * 3 * 2 * MAX_T)),
        ('ecp_nl_lmax_p1', C.c_int32), ('ecp_nl_terms', C.c_int32),
        ('ecp_nl', C.c_double * (MAX_NUC * MAX_L * 2 * MAX_T)),
        ('n_env_per_nuc', C.c_int32), ('n_nuc_tokens', C.c_int32),
        ('factorized_det', C.c_int32), ('conf_linear', C.c_int32), ('mult_act', C.c_int32),
        ('n_elec_types', C.c_int32), ('jastrow_n', C.c_int32), ('jastrow_dims', C.c_int32 * 8),
        ('backflow_n', C.c_int32), ('backflow_dims', C.c_int32 * 8),
        ('gnn_features', C.c_int32), ('gnn_concat', C.c_int32), ('gnn_conv_ne', C.c_int32), ('gnn_sub_n', C.c_int32),
        ('gnn_deep_edges', C.c_int32), ('gnn_res_norm', C.c_int32), ('gnn_g_bias', C.c_int32), ('gnn_w_bias', C.c_int32),
        ('gnn_w_dims', C.c_int32 * 32), ('gnn_h_dims', C.c_int32 * 32), ('gnn_u_dims', C.c_int32 * 32),
        ('nuc_cusp_kind', C.c_int32), ('z_nuclear', C.c_double * MAX_NUC), ('backflow_add', C.c_int32),
        ('gnn_sep_edges', C.c_int32), ('gnn_self_edges', C.c_int32), ('gnn_ne_identity', C.c_int32),
        ('gnn_no_res', C.c_int32), ('gnn_edge_in', C.c_int32 * 3),
    ]


_cache = {}


def load(path: str | None = None) -> C.CDLL:
    path = path or LIB_PATH
    if path in _cache:
        return _cache[path]
    if not os.path.exists(path):
        raise ImportError(
            f'{path} not found: the CUDA engine is not built. Run `python -c "import __graft_entry__ as g; '
            'g.build()"` (nvcc, sm_90a). There is no CPU fallback.'
        )
    lib = C.CDLL(path)
    for s in SYMBOLS:
        if not hasattr(lib, s):
            raise ImportError(f'{path} does not export {s}')
    vp, i32, i64, u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64
    lib.dqmc_create.argtypes = [C.POINTER(DqmcConfig), C.c_int, C.POINTER(vp)]
    lib.dqmc_destroy.argtypes = [vp]
    lib.dqmc_last_error.argtypes = [vp]
    lib.dqmc_last_error.restype = C.c_char_p
    lib.dqmc_version.restype = C.c_char_p
    lib.dqmc_param_count.argtypes = [vp]
    lib.dqmc_param_entry.argtypes = [vp, C.c_int, C.c_char_p, C.c_int, C.POINTER(i64), C.POINTER(i32), C.POINTER(i32)]
    lib.dqmc_param_total.argtypes = [vp]
    lib.dqmc_param_total.restype = i64
    lib.dqmc_set_params.argtypes = [vp, C.POINTER(C.c_double), i64, vp]
    lib.dqmc_workspace_bytes.argtypes = [vp, i32, i32]
    lib.dqmc_workspace_bytes.restype = i64
    lib.dqmc_workspace_bytes_min.argtypes = [vp, i32, i32]
    lib.dqmc_workspace_bytes_min.restype = i64
    lib.dqmc_debug_plan.argtypes = [vp, i32, i32, i64, C.POINTER(i64), C.POINTER(i64)]
    lib.dqmc_stats_pack.argtypes = [vp, vp, vp, i32, vp, vp]
    lib.dqmc_debug_mlp_block.argtypes = [vp, i32, vp, vp, vp, i32, vp]
    lib.dqmc_debug_trunk.argtypes = [vp, vp, vp, i32, vp]
    lib.dqmc_debug_trunk_phases.argtypes = [vp, C.POINTER(u64), i32]
    lib.dqmc_debug_tc_error.argtypes = [vp, C.POINTER(i32)]
    lib.dqmc_debug_attention.argtypes = [vp, i32, vp, vp, i32, i32, C.POINTER(i32), vp]
    lib.dqmc_debug_mlp.argtypes = [vp, i32, i32, vp, vp, vp, vp, i32, C.POINTER(i32), vp]
    lib.dqmc_debug_slater.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, C.POINTER(i32), vp]
    lib.dqmc_debug_det_sum.argtypes = [vp, vp, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp]
    lib.dqmc_debug_wgrad.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, vp, vp, vp]
    lib.dqmc_debug_attention_bwd.argtypes = [vp, i32, vp, vp, vp, vp, vp, i32, vp]
    lib.dqmc_wf_forward.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp, i64, vp]
    lib.dqmc_wf_orbitals.argtypes = [vp, vp, vp, i32, i32, vp, vp, i64, vp]
    lib.dqmc_local_energy.argtypes = [vp, vp, vp, i32, i32, u64, vp, vp, vp, vp, vp, vp, vp, i64, vp]
    lib.dqmc_mcmc_sweep.argtypes = [vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, C.c_double, i32, u64, u64, u64,
                                    vp, vp, vp, vp, i64, vp]
    lib.dqmc_mcmc_sweep_exchange.argtypes = [vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, C.c_double, i32, u64, u64, u64,
                                             vp, vp, C.c_double, C.POINTER(i32), vp, vp, vp, i64, vp]
    lib.dqmc_langevin_sweep.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, C.c_double, i32, u64, u64, u64,
                                        vp, vp, vp, vp, i64, vp]
    lib.dqmc_wf_vjp_params.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, i64, vp]
    lib.dqmc_spin.argtypes = [vp, vp, vp, i32, i32, vp, vp, i32, vp, vp, vp, i64, vp]
    lib.dqmc_wf_grad_positions.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, i64, vp]
    lib.dqmc_force_terms.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp, vp, vp]
    lib.dqmc_ecp_force.argtypes = [vp, vp, vp, i32, i32, u64, vp, vp, vp, vp, i64, vp]
    lib.dqmc_zv_force.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp, i64, vp]
    lib.dqmc_set_pseudo_hamiltonian.argtypes = [vp, i32, i32, C.c_double, C.POINTER(C.c_double), C.POINTER(i32)]
    lib.dqmc_launch_count.argtypes = [vp]
    lib.dqmc_launch_count.restype = i64
    lib.dqmc_ecp_forward_count.argtypes = [vp]
    lib.dqmc_ecp_forward_count.restype = i64
    lib.dqmc_profile_begin.argtypes = [vp]
    lib.dqmc_debug_gemm.argtypes = [vp, C.c_char_p, C.c_char_p, vp, vp, vp, i32, i32, i32, i32, vp]
    lib.dqmc_profile_end.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(i64)]
    lib.dqmc_profile_end_classes.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(i64)]
    _cache[path] = lib
    return lib
