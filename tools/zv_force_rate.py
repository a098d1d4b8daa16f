#!/usr/bin/env python
"""Rate of the AC-ZV force estimator (dqmc_zv_force + the bare force) on the benchmark's all-electron workloads.

  python tools/zv_force_rate.py OUT_DIR [--workloads lih_psiformer,n2_psiformer,n2_ferminet] [--reps 3]

For every workload (fp32, tensor-core backend, bench.py's molecule, ansatz and walker count; random-init weights and the
benchmark's synthetic walkers) it times with CUDA events, after one warm-up call of each, the local energy
(Engine.local_energy: one forward-Laplacian pass), the zero-variance term alone (Engine.zv_force: 3M companion passes, each
with its primal forward-Laplacian pass) and the AC-ZV estimator of deepqmc_b200/force.py, as walker samples per second.
Reports the fastest rep, and the card's name and power limit read in the same run (read-only nvidia-smi query).
Writes OUT_DIR/zv_force_rate.json.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

from bench import WORKLOADS, make_problem  # noqa: E402
from deepqmc_b200 import force as FO  # noqa: E402
from deepqmc_b200.ansatz import B200Ansatz  # noqa: E402
from deepqmc_b200.types import PhysicalConfiguration  # noqa: E402
from force_rate import card, timed  # noqa: E402


def run(wl_name, reps):
    wl = WORKLOADS[wl_name]
    B = wl['walkers']
    mol, hamil, r_np, PN = make_problem(wl, B, 0)
    a = B200Ansatz(hamil, wl['kind'], dtype='float32', gemm_backend=1, **wl['hyper'])
    params = PN.perturb_params(a.init(0))
    eng = a.engine_for(hamil, params)
    r = torch.as_tensor(r_np, dtype=torch.float32, device='cuda')
    R = torch.as_tensor(mol.coords, dtype=torch.float32, device='cuda')
    pc = PhysicalConfiguration(R, r, torch.zeros(B, device='cuda'))
    res = {'walkers': B, 'n_elec': hamil.n_up + hamil.n_down, 'n_nuc': len(mol.charges)}
    paths = {
        'local_energy': lambda: eng.local_energy(r, R),
        'zv_term': lambda: eng.zv_force(r, R),
        'ac_zv': lambda: FO.evaluate_hf_force_ac_zv(hamil, a.apply)(0, params, pc),
    }
    for f in paths.values():  # warm-up (workspace, allocator, modules)
        f()
    torch.cuda.synchronize()
    times = {k: [] for k in paths}
    for _ in range(reps):
        for k, f in paths.items():
            timed(f, times[k])
    for k in paths:
        t = min(times[k])
        res[k] = {'s': times[k], 'walkers_per_s': B / t}
        print(f'{wl_name:16s} {k:14s} {B / t:12.1f} walkers/s', flush=True)
    res['ac_zv_vs_local_energy_time'] = min(times['ac_zv']) / min(times['local_energy'])
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out_dir')
    ap.add_argument('--workloads', default='lih_psiformer,n2_psiformer,n2_ferminet')
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('zv_force_rate.py measures on a CUDA device; none found')
    os.makedirs(a.out_dir, exist_ok=True)
    out = {'card': card(), 'dtype': 'float32', 'gemm_backend': 'tensor', 'reps': a.reps, 'timing': 'min over reps, CUDA events'}
    print(f"{out['card']['name']}, power limit {out['card']['power.limit']}", flush=True)
    for w in a.workloads.split(','):
        out[w] = run(w, a.reps)
    with open(os.path.join(a.out_dir, 'zv_force_rate.json'), 'w') as f:
        json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
