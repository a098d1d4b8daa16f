#!/usr/bin/env python
"""Rate of the Hellmann-Feynman force with effective core potentials (dqmc_ecp_force).

  python tools/ecp_force_rate.py OUT_DIR [--workloads benzene_psiformer,lih_ccecp_psiformer] [--walkers B] [--reps 2]

For every workload (fp32, tensor-core backend, bench.py's molecule, ansatz and walker count unless --walkers overrides it;
random-init weights and the benchmark's synthetic walkers; lih_ccecp_psiformer is lih_psiformer with ccECP on lithium) it
times, with CUDA events after one warm-up call,
  - the bare force with its non-local part (Engine.ecp_force), as forces (walker samples) per second, and out_bare alone;
and reports
  - the share of (nucleus, electron) pairs inside the force's cutoff radius (quadrature walkers run / 12 B J N);
  - from one further call under torch.profiler, the CUDA time of the position reverse passes (every kernel that is not one of
    the three ECP kernels below or the force-terms kernel) and of the accumulation (ecp_force_accumulate_kernel), the pair
    list and the quadrature points (ecp_pairs_kernel, ecp_points_kernel).
Reports the fastest rep, and the card's name and power limit read in the same run (read-only nvidia-smi query).
Writes OUT_DIR/ecp_force_rate.json.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import WORKLOADS, make_problem  # noqa: E402
from deepqmc_b200.ansatz import B200Ansatz  # noqa: E402

EXTRA = {'lih_ccecp_psiformer': dict(WORKLOADS['lih_psiformer'], ecp='ccECP')}
GROUPS = {'accumulate': ('ecp_force_accumulate_kernel',), 'pairs_and_points': ('ecp_pairs_kernel', 'ecp_points_kernel'),
          'force_terms': ('force_terms_kernel',)}


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True,
                         check=True).stdout.strip().splitlines()[0]
    return dict(zip(q.split(','), (x.strip() for x in out.split(','))))


def timed(fn, reps_out):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    e1.synchronize()
    reps_out.append(e0.elapsed_time(e1) / 1e3)
    return out


def kernel_split(fn):
    """CUDA time [s] per group of GROUPS, the rest counted as the reverse passes, from one profiled call."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {k: 0.0 for k in GROUPS}
    split['reverse_passes'] = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, 'device_time_total', None)
        t = ev.cuda_time_total if t is None else t
        if not t:
            continue
        grp = next((k for k, names in GROUPS.items() if any(n in ev.key for n in names)), 'reverse_passes')
        split[grp] += t / 1e6
    return split


def run(wl_name, walkers, reps):
    wl = EXTRA.get(wl_name) or WORKLOADS[wl_name]
    B = walkers or wl['walkers']
    mol, hamil, r_np, PN = make_problem(wl, B, 0)
    a = B200Ansatz(hamil, wl['kind'], dtype='float32', gemm_backend=1, **wl['hyper'])
    params = PN.perturb_params(a.init(0))
    eng = a.engine_for(hamil, params)
    r = torch.as_tensor(r_np, dtype=torch.float32, device='cuda')
    R = torch.as_tensor(mol.coords, dtype=torch.float32, device='cuda')
    N, J = hamil.n_up + hamil.n_down, len(hamil.pot.nuc_with_nl_pot)
    res = {'walkers': B, 'n_elec': N, 'n_nuc': len(mol.charges), 'n_ecp_nuc': J}
    paths = {'bare_and_nonlocal': lambda: eng.ecp_force(r, R, seed=1), 'bare_only': lambda: eng.ecp_force(r, R, want_nl=False)}
    n0 = eng.lib.dqmc_ecp_forward_count(eng.h)
    for f in paths.values():  # warm-up (workspace, allocator, modules)
        f()
    torch.cuda.synchronize()
    res['active_pair_share'] = (eng.lib.dqmc_ecp_forward_count(eng.h) - n0) / (12 * B * J * N)
    times = {k: [] for k in paths}
    for _ in range(reps):
        for k, f in paths.items():
            timed(f, times[k])
    for k in paths:
        t = min(times[k])
        res[k] = {'s': times[k], 'forces_per_s': B / t}
        print(f'{wl_name:20s} {k:18s} {B / t:12.2f} forces/s', flush=True)
    res['cuda_time_split_s'] = kernel_split(paths['bare_and_nonlocal'])
    print(f"{wl_name:20s} active pairs {res['active_pair_share']:.3f}, CUDA time split {res['cuda_time_split_s']}", flush=True)
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out_dir')
    ap.add_argument('--workloads', default='benzene_psiformer,lih_ccecp_psiformer')
    ap.add_argument('--walkers', type=int, default=0, help='override the workloads\' walker count')
    ap.add_argument('--reps', type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('ecp_force_rate.py measures on a CUDA device; none found')
    os.makedirs(a.out_dir, exist_ok=True)
    out = {'card': card(), 'dtype': 'float32', 'gemm_backend': 'tensor', 'reps': a.reps, 'timing': 'min over reps, CUDA events'}
    print(f"{out['card']['name']}, power limit {out['card']['power.limit']}", flush=True)
    for w in a.workloads.split(','):
        out[w] = run(w, a.walkers, a.reps)
    with open(os.path.join(a.out_dir, 'ecp_force_rate.json'), 'w') as f:
        json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
