#!/usr/bin/env python
"""Local-energy rate of the DeepErwin ansatz (conf/ansatz/deeperwin.yaml as shipped) on LiH and N2.

  python tools/deeperwin_rate.py OUT_DIR [--walkers 2048] [--reps 5] [--dtype float32]

For each molecule: random-init weights, walkers drawn around the nuclei, one warm-up call, then the fastest of --reps
dqmc_local_energy calls timed with CUDA events -> walker E_loc per second, and the same for dqmc_wf_vjp_params (the
gradient of the mean log|psi|, host pull-back included) -> walkers per second.  The card's name and
power limit are read in the same run (read-only nvidia-smi query) and printed beside every number.  Writes
OUT_DIR/deeperwin_rate.json.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from deepqmc_b200.ansatz import B200Ansatz  # noqa: E402
from deepqmc_b200.hamil import MolecularHamiltonian  # noqa: E402
from deepqmc_b200.molecule import Molecule  # noqa: E402


def card():
    q = 'name,power.limit'
    out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True,
                         check=True).stdout.strip().splitlines()[0]
    return dict(zip(q.split(','), (x.strip() for x in out.split(','))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out')
    ap.add_argument('--walkers', type=int, default=2048)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--dtype', default='float32')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('deeperwin_rate needs a CUDA device')
    c = card()
    res = {'card': c, 'walkers': a.walkers, 'dtype': a.dtype, 'rates': {}}
    for name in ('LiH', 'N2'):
        mol = Molecule.from_name(name)
        hamil = MolecularHamiltonian(mol=mol)
        ans = B200Ansatz(hamil, 'deeperwin', dtype=a.dtype, gemm_backend=1 if a.dtype == 'float32' else 0)
        params = ans.init(0)
        eng = ans.engine_for(hamil, params)
        rng = np.random.default_rng(0)
        N = hamil.n_up + hamil.n_down
        r = mol.coords[rng.integers(0, len(mol.coords), size=(a.walkers, N))] + rng.normal(size=(a.walkers, N, 3))
        r = torch.as_tensor(r, dtype=eng.dtype, device='cuda')
        R = torch.as_tensor(mol.coords, dtype=eng.dtype, device='cuda')
        w = torch.full((a.walkers,), 1.0 / a.walkers, dtype=eng.dtype, device='cuda')

        def best_of(fn):
            fn()
            torch.cuda.synchronize()
            best = float('inf')
            for _ in range(a.reps):
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                fn()
                t1.record()
                torch.cuda.synchronize()
                best = min(best, t0.elapsed_time(t1) / 1e3)
            return best

        te = best_of(lambda: eng.local_energy(r, R))
        tv = best_of(lambda: eng.vjp_params(r, R, w))
        res['rates'][name] = {'walker_eloc_per_s': a.walkers / te, 'eloc_seconds': te,
                              'vjp_walkers_per_s': a.walkers / tv, 'vjp_seconds': tv}
        print(f'{name}: {a.walkers / te:.4g} walker E_loc/s, {a.walkers / tv:.4g} walker parameter-VJP/s ({a.walkers} '
              f'walkers, {a.dtype}) on {c["name"]} at {c["power.limit"]}', flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'deeperwin_rate.json'), 'w') as f:
        json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
