#!/usr/bin/env python
"""Rate of the spin pass (dqmc_spin) against the materialised-copy path, on the benchmark's workloads.

  python tools/spin_rate.py OUT_DIR [--workloads n2_psiformer,benzene_psiformer,cyclobutadiene_transpsiformer] [--reps 3]

For every workload (fp32, tensor-core backend, bench.py's molecule, ansatz and walker count; random-init weights and the
benchmark's synthetic walkers) it times, with CUDA events after one warm-up call of each,
  - the exact estimator (n_up n_down swapped forwards per walker) and the spin-raising estimator (n_up per walker) of
    Engine.spin, and
  - the materialised-copy path: the swapped walkers built in torch, one dqmc_wf_forward over all of them, the ratios and
    their sum in torch (fp64),
alternating the two paths rep by rep.  Reports S^2 evaluations per second and virtual forwards per second (fastest rep),
the largest difference between the two paths' results relative to max(1, sum |rho|), and the card's name and power limit
read in the same run (read-only nvidia-smi query).  Writes OUT_DIR/spin_rate.json.
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


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True,
                         check=True).stdout.strip().splitlines()[0]
    return dict(zip(q.split(','), (x.strip() for x in out.split(','))))


def copy_path(eng, r, R, n_up, n_down, down_idx):
    """The swapped walkers built in torch, one dqmc_wf_forward over all of them, ratios and sums in fp64."""
    B, N = r.shape[:2]
    if down_idx < 0:
        a = torch.arange(n_up, device=r.device).repeat_interleave(n_down)
        b = n_up + torch.arange(n_down, device=r.device).repeat(n_up)
        c0 = (n_up - n_down) / 2 * ((n_up - n_down) / 2 + 1) + n_down
    else:
        a = torch.arange(n_up, device=r.device)
        b = torch.full_like(a, down_idx)
        c0 = 1.0
    P = a.numel()
    idx = torch.arange(N, device=r.device).repeat(P, 1)  # [P, N]: source electron of every row
    p = torch.arange(P, device=r.device)
    idx[p, a], idx[p, b] = b, a
    sw = r[:, idx]  # [B, P, N, 3]
    s0, l0 = eng.wf_forward(r, R)
    s, l = eng.wf_forward(sw.reshape(B * P, N, 3), R)
    rho = s.double().reshape(B, P) * s0.double()[:, None] * torch.exp(l.double().reshape(B, P) - l0.double()[:, None])
    return (c0 - rho.sum(1)).to(r.dtype), rho.abs().sum(1)


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
    eng = a.engine_for(hamil, PN.perturb_params(a.init(0)))
    r = torch.as_tensor(r_np, dtype=torch.float32, device='cuda')
    R = torch.as_tensor(mol.coords, dtype=torch.float32, device='cuda')
    n_up, n_down = hamil.n_up, hamil.n_down
    res = {'walkers': B, 'n_up': n_up, 'n_down': n_down}
    for est, down_idx, P in (('exact', -1, n_up * n_down), ('raising', n_up + n_down - 1, n_up)):
        new = lambda: eng.spin(r, R, down_idx=down_idx)[0]
        cpy = lambda: copy_path(eng, r, R, n_up, n_down, down_idx)[0]
        s_new, (s_cpy, abs_sum) = new(), copy_path(eng, r, R, n_up, n_down, down_idx)  # warm-up (workspace, allocator, modules)
        torch.cuda.synchronize()
        t_new, t_cpy = [], []
        for _ in range(reps):
            s_new = timed(new, t_new)
            s_cpy = timed(cpy, t_cpy)
        tn, tc = min(t_new), min(t_cpy)
        res[est] = {
            'virtual_forwards_per_walker': P,
            'spin_pass_s': t_new, 'copy_path_s': t_cpy,
            'spin_pass_s2_per_s': B / tn, 'spin_pass_virtual_forwards_per_s': B * P / tn,
            'copy_path_s2_per_s': B / tc, 'copy_path_virtual_forwards_per_s': B * P / tc,
            'speedup_vs_copy_path': tc / tn,
            # s2 is a sum of P ratios: the difference relative to max(1, sum |rho|) (the bound of tests/test_gpu_spin.py)
            'max_rel_diff_vs_copy_path': float(((s_new.double() - s_cpy.double()).abs() / abs_sum.clamp(min=1.0)).max()),
        }
        print(f'{wl_name:32s} {est:8s} P={P:4d}  spin pass {B / tn:10.1f} S2/s {B * P / tn / 1e6:8.3f} M fwd/s   '
              f'copy path {B / tc:10.1f} S2/s   x{tc / tn:.3f}   max rel diff {res[est]["max_rel_diff_vs_copy_path"]:.2e}', flush=True)
        del s_new, s_cpy, abs_sum
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out_dir')
    ap.add_argument('--workloads', default='n2_psiformer,benzene_psiformer,cyclobutadiene_transpsiformer')
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('spin_rate.py measures on a CUDA device; none found')
    os.makedirs(a.out_dir, exist_ok=True)
    out = {'card': card(), 'dtype': 'float32', 'gemm_backend': 'tensor', 'reps': a.reps, 'timing': 'min over reps, CUDA events'}
    print(f"{out['card']['name']}, power limit {out['card']['power.limit']}", flush=True)
    for w in a.workloads.split(','):
        out[w] = run(w, a.reps)
    with open(os.path.join(a.out_dir, 'spin_rate.json'), 'w') as f:
        json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
