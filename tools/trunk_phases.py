#!/usr/bin/env python
"""Where the whole-trunk kernel's time goes: phase timers of `tc::trunk_f16_kernel` at the production tile shape.

  python tools/trunk_phases.py OUT_DIR [--mol benzene|LiH] [--walkers 16384] [--launches 20]

Builds the benzene / ccECP Psiformer engine (fp32, tensor-core backend; N = 30 electrons, walker slot 32, 4 walkers per
128-row tile) or the LiH one (N = 4, walker slot 4, 32 walkers per tile) and runs the trunk alone (dqmc_debug_trunk) on random embedding rows.  Two engines: one without timers for the
kernel time (CUDA events over --launches launches after a warm-up), one created with DQMC_TRUNK_PHASES=1 for the phase shares.
Prints and writes OUT_DIR/trunk_phases_<mol>.json: us per (tile, layer) per SM, algorithmic TFLOP/s (counted as the engine's
profiler counts the trunk class: 2 rows (6 d^2 + 2 N d) per layer), each phase's share of the consumer warpgroups' cycles,
and the card's name, power limit and SM clocks (read-only nvidia-smi query).  The two warpgroups of a CTA share the tensor
cores through a lock that whichever asks first takes: 'mma_turn' is the time a warpgroup waited for that lock while the
other one issued its MMAs (the part of those MMAs its own non-MMA work did not cover), 'weight_wait' the time it waited
for weight slots to land.

'sass_bytes' is the machine code of the trunk instance the run launched (cuobjdump -sass of the built library), split at the
phase timers in address order: the code between two timer marks belongs to the phase the later mark books, a mark whose
counter index is only known at run time books to 'shared', and code after the last mark to 'other'.  Where the compiler lays
out the code of several phases before one mark (the rolled loop over the MLP GEMMs with its three epilogues), that mark's
phase gets all of it; 'total' is exact.  Code size matters because a (tile, layer) runs the kernel's body once per warp as straight-line code.
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from deepqmc_b200 import params as PN  # noqa: E402
from deepqmc_b200.ansatz import B200Ansatz  # noqa: E402
from deepqmc_b200.hamil import MolecularHamiltonian  # noqa: E402
from deepqmc_b200.molecule import Molecule  # noqa: E402


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True,
                         check=True).stdout.strip().splitlines()[0]
    return dict(zip(q.split(','), (x.strip() for x in out.split(','))))


def cuobjdump():
    for c in (os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'cuobjdump'), shutil.which('cuobjdump')):
        if c and os.access(c, os.X_OK):
            return c
    return None


def sass_bytes(lib, np2, names):
    """{phase: bytes} of the trunk instance for walker slot np2 in `lib`, split at the phase timer marks (see the module
    docstring); None without cuobjdump.  A mark is a predicated clock read followed by the same-predicate read of its
    counter `[R + 8 k]`; reads of the weight_wait / mma_turn counters (waits inside a phase) do not split."""
    tool = cuobjdump()
    if tool is None:
        return None
    out = ''
    for fn in (f'_ZN2dq2tc16trunk_f16_kernelILi{np2}EEEvNS0_11TrunkParamsE', '_ZN2dq2tc16trunk_f16_kernelENS0_11TrunkParamsE'):
        r = subprocess.run([tool, '-sass', '-fun', fn, lib], capture_output=True, text=True)
        if r.returncode == 0 and 'Function : ' in r.stdout:
            out = r.stdout
            break
    ins = [t.strip() for t in re.findall(r'/\*[0-9a-f]{4,}\*/\s+([^;]*);', out)]
    assert ins, f'no trunk kernel in {lib}'
    waits = {names.index('weight_wait'), names.index('mma_turn')}
    res = {k: 0 for k in names if k != 'tile_layer_pairs'}
    res.update(shared=0, other=0)
    start = 0
    for i, txt in enumerate(ins):
        if not (txt.startswith('@') and 'SR_CLOCKLO' in txt):
            continue
        pred = txt.split()[0]
        for nxt in ins[i + 1:i + 4]:
            m = re.match(re.escape(pred) + r'\s+LDS\.64\s+\S+,\s+\[(.*)\]', nxt)
            if m is None:
                continue
            addr = re.fullmatch(r'R\d+(?:\+(0x[0-9a-f]+))?', m.group(1))
            if addr is None:
                key = 'shared'
            else:
                k = int(addr.group(1) or '0', 16) // 8
                key = None if k in waits else names[k]
            if key is not None:
                res[key] += 16 * (i - start)
                start = i
            break
    res['other'] += 16 * (len(ins) - start)
    res['total'] = 16 * len(ins)
    return res


def engine(hamil, params, phases):
    os.environ.pop('DQMC_TRUNK_PHASES', None)
    if phases:
        os.environ['DQMC_TRUNK_PHASES'] = '1'
    try:
        return B200Ansatz(hamil, 'psiformer', dtype='float32', gemm_backend=1).engine_for(hamil, params)
    finally:
        os.environ.pop('DQMC_TRUNK_PHASES', None)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument('out_dir')
    ap.add_argument('--mol', choices=('benzene', 'LiH'), default='benzene')
    ap.add_argument('--walkers', type=int, default=16384)
    ap.add_argument('--launches', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    a = ap.parse_args()
    assert a.walkers >= 16384 and a.launches >= 20, 'production shape: >= 16384 walkers, >= 20 timed launches'
    assert torch.cuda.is_available(), 'the trunk phase timers need a GPU'
    torch.cuda.set_device(0)
    hamil = MolecularHamiltonian(mol=Molecule.from_name(a.mol), ecp_type='ccECP' if a.mol == 'benzene' else None)
    params = PN.perturb_params(B200Ansatz(hamil, 'psiformer', dtype='float32', gemm_backend=1).init(0))
    N, d, L = hamil.n_up + hamil.n_down, 256, 4
    g = torch.Generator(device='cpu').manual_seed(0)
    X0 = torch.randn(a.walkers * N, d, generator=g).cuda()

    plain = engine(hamil, params, False)
    for _ in range(a.warmup):
        plain.debug_trunk(X0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.launches):
        plain.debug_trunk(X0)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.launches

    timed = engine(hamil, params, True)
    timed.debug_trunk(X0)
    torch.cuda.synchronize()
    timed.debug_trunk_phases()  # drop the warm-up launch
    for _ in range(a.launches):
        timed.debug_trunk(X0)
    torch.cuda.synchronize()
    ph = timed.debug_trunk_phases()

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    np2 = 1 << (N - 1).bit_length()
    tiles = -(-a.walkers // (128 // np2))
    grid = min(tiles, sms)
    pairs = ph.pop('tile_layer_pairs') / a.launches
    assert pairs == tiles * L, (pairs, tiles * L)
    flops = L * 2.0 * a.walkers * N * (6 * d * d + 2 * N * d)
    total = sum(ph.values())
    res = dict(
        kernel='tc::trunk_f16_kernel', mol=a.mol, ecp=hamil.ecp_type, walkers=a.walkers, N=N, slot=np2, walkers_per_tile=128 // np2,
        launches=a.launches, grid=grid, ms_per_launch=ms, us_per_tile_layer=ms * 1e3 * grid / pairs,
        algorithmic_tflops=flops / (ms * 1e-3) / 1e12, phase_share={k: v / total for k, v in ph.items()},
        phase_cycles={k: int(v) for k, v in ph.items()},
        sass_bytes=sass_bytes(os.path.join(ROOT, 'deepqmc_b200', 'libdqmc_b200.so'), np2, timed.TRUNK_PHASES), card=card())
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, f'trunk_phases_{a.mol}.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(f"{res['card']['name']}, power limit {res['card']['power.limit']}, SM clock {res['card']['clocks.sm']} "
          f"(max {res['card']['clocks.max.sm']})")
    print(f'{ms:.3f} ms per launch, {res["us_per_tile_layer"]:.1f} us per (tile, layer) per SM, '
          f'{res["algorithmic_tflops"]:.1f} algorithmic TFLOP/s')
    for k, v in res['phase_share'].items():
        print(f'  {k:14s} {100 * v:5.1f} %')
    if res['sass_bytes']:
        print('SASS bytes: ' + ', '.join(f'{k} {v}' for k, v in res['sass_bytes'].items() if v))


if __name__ == '__main__':
    main()
