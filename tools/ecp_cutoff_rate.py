#!/usr/bin/env python
"""The non-local ECP cutoff radius on the flagship workload: step time, outputs and the share of active pairs.

  python tools/ecp_cutoff_rate.py OUT_DIR [--parent DIR] [--reps 2] [--steps 2] [--warmup 1]

Arms: 'default' (this tree, cutoff on), 'cutoff_off' (this tree under DQMC_ECP_CUTOFF=0: every pair runs its quadrature
forwards) and, with --parent DIR, 'parent' (DIR: a plain export of another revision of the project, e.g. `git archive`
of the parent commit, built here by its own __graft_entry__.build()).  It
  - prints the card's name and power limit (read-only nvidia-smi query),
  - runs `bench.py --gpus 1 --steps S --warmup W` (benzene_psiformer, the defaults) for every arm, alternating the arms rep
    by rep, and reports ms per step and walker.E_loc/s of each run and the ratios of the arms' best runs,
  - runs `bench.py --dump-outputs` (one step, no equilibration) for every arm and compares each array with the first arm's:
    bitwise equal or not, elements that differ and the largest |difference|,
  - reports the active-pair share on the benchmark's equilibrated walkers: bench.py's problem, parameters and equilibration
    sweeps, one local-energy call, Engine.ecp_forward_count over 12 B J N.
Writes OUT_DIR/ecp_cutoff_rate.json (and the dumps under OUT_DIR/dump_<arm>/).
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    q = 'name,power.limit,clocks.max.sm'
    out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True,
                         check=True).stdout.strip().splitlines()[0]
    return dict(zip(q.split(','), (x.strip() for x in out.split(','))))


def build(tree):
    subprocess.run([sys.executable, '-c', 'import __graft_entry__ as g; g.build()'], cwd=tree, check=True)


def bench(tree, env, args):
    cp = subprocess.run([sys.executable, 'bench.py', '--gpus', '1', *args], cwd=tree, env=env, capture_output=True,
                        text=True)
    if cp.returncode:
        raise SystemExit(f'bench.py failed in {tree}:\n{cp.stdout[-2000:]}\n{cp.stderr[-4000:]}')
    return json.loads(cp.stdout.strip().splitlines()[-1])


def active_share(steps_seed=100):
    """Active pairs of bench.py's equilibrated walkers, from the engine's quadrature-forward counter."""
    sys.path.insert(0, ROOT)
    import torch

    from bench import WORKLOADS, make_problem
    from deepqmc_b200 import parallel
    from deepqmc_b200.ansatz import B200Ansatz

    wl = WORKLOADS['benzene_psiformer']
    B = wl['walkers']
    mol, hamil, r_np, PN = make_problem(wl, B, seed=1000)
    a = B200Ansatz(hamil, wl['kind'], dtype='float32', gemm_backend=1, **wl['hyper'])
    eng = a.engine_for(hamil, PN.perturb_params(a.init(0), seed=0))
    R = torch.as_tensor(mol.coords, dtype=torch.float32, device='cuda')
    r = torch.as_tensor(r_np[:B], dtype=torch.float32, device='cuda')
    N, J = hamil.n_up + hamil.n_down, len(hamil.pot.nuc_with_nl_pot)
    out = {}
    for name in ('synthetic', 'equilibrated'):
        if name == 'equilibrated':  # bench.py's untimed equilibration of the heavy workloads: 5 sweeps x 10 sub-steps
            sign, log = eng.wf_forward(r, R)
            st = dict(r=r.clone(), sign=sign, log=log, age=torch.zeros(B, dtype=torch.int32, device='cuda'),
                      tau=torch.tensor([0.5], dtype=torch.float32, device='cuda'))
            for it in range(5):
                eng.mcmc_sweep(st, R, 10, seed=parallel.rank_seed(7), step0=10 * it, walker_offset=0)
            r = st['r']
        n0 = eng.ecp_forward_count
        eng.local_energy(r, R, seed=steps_seed)
        torch.cuda.synchronize()
        n = eng.ecp_forward_count - n0
        out[name] = {'quadrature_forwards': n, 'all_pairs_forwards': 12 * B * J * N, 'active_share': n / (12 * B * J * N)}
    return out


def compare(ref_dir, dirs):
    res = {}
    for arm, d in dirs.items():
        res[arm] = {}
        for f in sorted(os.listdir(ref_dir)):
            x, y = np.load(os.path.join(ref_dir, f)), np.load(os.path.join(d, f))
            diff = np.abs(x.astype(np.float64) - y.astype(np.float64))
            res[arm][f[:-4]] = {'bitwise_equal': bool(np.array_equal(x, y, equal_nan=True)),
                                'n_differ': int((x != y).sum() - (np.isnan(x) & np.isnan(y)).sum()),
                                'max_abs_diff': float(np.nanmax(diff)) if diff.size else 0.0}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out_dir')
    ap.add_argument('--parent', default=None, help='an exported tree of the revision to compare against')
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--steps', type=int, default=2)
    ap.add_argument('--warmup', type=int, default=1)
    a = ap.parse_args()
    os.makedirs(a.out_dir, exist_ok=True)
    out = {'card': card(), 'workload': 'benzene_psiformer (bench.py defaults)', 'steps': a.steps, 'warmup': a.warmup}
    print(f"{out['card']['name']}, power limit {out['card']['power.limit']}", flush=True)
    env = dict(os.environ)
    env.pop('DQMC_ECP_CUTOFF', None)
    arms = {'default': (ROOT, env), 'cutoff_off': (ROOT, dict(env, DQMC_ECP_CUTOFF='0'))}
    if a.parent:
        arms = {'parent': (os.path.abspath(a.parent), env), **arms}
    for tree in {t for t, _ in arms.values()}:
        build(tree)

    runs = {k: [] for k in arms}
    for rep in range(a.reps):
        for arm, (tree, e) in arms.items():
            j = bench(tree, e, ['--steps', str(a.steps), '--warmup', str(a.warmup)])
            cls = (j.get('roofline') or {}).get('classes') or {}
            runs[arm].append({'value': j['value'], 'ms_per_step': j['ms_per_step'], 'ms_per_step_min': j['ms_per_step_min'],
                              'energy_mean': j['energy_mean'], 'gpu_launches': j['gpu_launches'],
                              'classes': cls, 'clocks': j.get('clocks')})
            print(f'rep {rep} {arm:10s} {j["ms_per_step"]:10.1f} ms/step {j["value"]:9.2f} walker.E_loc/s  '
                  f'trunk share {cls.get("trunk", {}).get("share_of_step", float("nan")):.3f}', flush=True)
    out['runs'] = runs
    best = {k: max(r['value'] for r in v) for k, v in runs.items()}
    out['best_value'] = best
    out['ratios'] = {'default_over_cutoff_off': best['default'] / best['cutoff_off']}
    if a.parent:
        out['ratios'].update(default_over_parent=best['default'] / best['parent'],
                             cutoff_off_over_parent=best['cutoff_off'] / best['parent'])
    print('ratios', json.dumps(out['ratios']), flush=True)

    dumps = {}
    for arm, (tree, e) in arms.items():
        dumps[arm] = os.path.join(os.path.abspath(a.out_dir), f'dump_{arm}')
        bench(tree, e, ['--steps', '1', '--warmup', '0', '--dump-outputs', dumps[arm]])
    ref = 'parent' if a.parent else 'cutoff_off'
    out['outputs_vs_' + ref] = compare(dumps[ref], {k: v for k, v in dumps.items() if k != ref})
    for arm, arrs in out['outputs_vs_' + ref].items():
        for name, c in arrs.items():
            print(f'{arm:10s} vs {ref:10s} {name:28s} bitwise {c["bitwise_equal"]}  differ {c["n_differ"]}  '
                  f'max |d| {c["max_abs_diff"]:.3e}', flush=True)

    out['active_pairs'] = active_share()
    print('active pairs', json.dumps(out['active_pairs']), flush=True)
    with open(os.path.join(a.out_dir, 'ecp_cutoff_rate.json'), 'w') as f:
        json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
