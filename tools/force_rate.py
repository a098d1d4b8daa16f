#!/usr/bin/env python
"""Rate of the position gradients (dqmc_wf_grad_positions) and of the force estimators, on the benchmark's workloads.

  python tools/force_rate.py OUT_DIR [--workloads lih_psiformer,n2_psiformer,n2_ferminet] [--reps 3]

For every workload (fp32, tensor-core backend, bench.py's molecule, ansatz and walker count; random-init weights and the
benchmark's synthetic walkers) it times, with CUDA events after one warm-up call of each,
  - the two ways to get grad_r log|psi|: the reverse pass (Engine.grad_positions, grad_r only, and grad_r + grad_R) and the
    forward-Laplacian pass (Engine.local_energy(want_grad=True)), alternating rep by rep, with their largest difference
    relative to max(1, |grad_r|_inf);
  - every estimator of deepqmc_b200/force.py built for all-electron systems (bare, AC-ZVQ, AC-ZVZBQ, AC-ZB, AC-ZVQZB),
    as forces (walker samples) per second; E_loc is given to the estimators that take it.
Reports the fastest rep, and the card's name and power limit read in the same run (read-only nvidia-smi query).
Writes OUT_DIR/force_rate.json.
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
from deepqmc_b200 import force as FO  # noqa: E402
from deepqmc_b200.ansatz import B200Ansatz  # noqa: E402
from deepqmc_b200.types import PhysicalConfiguration  # noqa: E402


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


def run(wl_name, reps):
    wl = WORKLOADS[wl_name]
    B = wl['walkers']
    mol, hamil, r_np, PN = make_problem(wl, B, 0)
    a = B200Ansatz(hamil, wl['kind'], dtype='float32', gemm_backend=1, **wl['hyper'])
    params = PN.perturb_params(a.init(0))
    eng = a.engine_for(hamil, params)
    r = torch.as_tensor(r_np, dtype=torch.float32, device='cuda')
    R = torch.as_tensor(mol.coords, dtype=torch.float32, device='cuda')
    res = {'walkers': B, 'n_elec': hamil.n_up + hamil.n_down, 'n_nuc': len(mol.charges)}
    paths = {
        'reverse_grad_r': lambda: eng.grad_positions(r, R, want_R=False)[2],
        'reverse_grad_r_and_R': lambda: eng.grad_positions(r, R)[2],
        'forward_laplacian_grad_r': lambda: eng.local_energy(r, R, want_grad=True)[4].reshape(r.shape),
    }
    outs = {k: f() for k, f in paths.items()}  # warm-up (workspace, allocator, modules)
    torch.cuda.synchronize()
    times = {k: [] for k in paths}
    for _ in range(reps):
        for k, f in paths.items():
            outs[k] = timed(f, times[k])
    scale = max(1.0, float(outs['forward_laplacian_grad_r'].abs().max()))
    for k in paths:
        t = min(times[k])
        res[k] = {'s': times[k], 'walkers_per_s': B / t}
        print(f'{wl_name:16s} {k:26s} {B / t:12.1f} walkers/s', flush=True)
    res['reverse_vs_forward_laplacian_time'] = min(times['reverse_grad_r']) / min(times['forward_laplacian_grad_r'])
    res['max_rel_diff_grad_r'] = float((outs['reverse_grad_r'].double() - outs['forward_laplacian_grad_r'].double()).abs().max()
                                       / scale)
    pc = PhysicalConfiguration(R, r, torch.zeros(B, device='cuda'))
    e_loc = hamil.local_energy(a.apply)(None, params, pc)[0]
    energy = float(e_loc.double().mean())
    est = {
        'bare': lambda: FO.evaluate_hf_force_bare(hamil, a.apply)(0, params, pc),
        'ac_zvq': lambda: FO.evaluate_hf_force_ac_zvq(hamil, a.apply)(params, pc),
        'ac_zvzbq': lambda: FO.evaluate_hf_force_ac_zvzbq(hamil, a.apply)(params, pc, e_loc, energy),
        'ac_zb': lambda: FO.evaluate_hf_force_ac_zb(hamil, a.apply)(0, params, pc, e_loc, energy),
        'ac_zvqzb': lambda: FO.evaluate_hf_force_ac_zvqzb(hamil, a.apply)(params, pc, e_loc, energy),
    }
    for k, f in est.items():
        f()
        torch.cuda.synchronize()
        t = []
        for _ in range(reps):
            timed(f, t)
        res[k] = {'s': t, 'forces_per_s': B / min(t)}
        print(f'{wl_name:16s} {k:26s} {B / min(t):12.1f} forces/s', flush=True)
    del outs
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out_dir')
    ap.add_argument('--workloads', default='lih_psiformer,n2_psiformer,n2_ferminet')
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('force_rate.py measures on a CUDA device; none found')
    os.makedirs(a.out_dir, exist_ok=True)
    out = {'card': card(), 'dtype': 'float32', 'gemm_backend': 'tensor', 'reps': a.reps, 'timing': 'min over reps, CUDA events'}
    print(f"{out['card']['name']}, power limit {out['card']['power.limit']}", flush=True)
    for w in a.workloads.split(','):
        out[w] = run(w, a.reps)
    with open(os.path.join(a.out_dir, 'force_rate.json'), 'w') as f:
        json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
