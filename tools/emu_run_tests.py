"""Development tool: run tests of tests/test_gpu_*.py against the CPU emulation of the SIMT kernels (tools/cuda_emu).

NOT part of the product and not a parity claim -- the container this was written in has no GPU, so everything added after the
round's GPU minutes ran out was first checked here (DESIGN.md section 8).  What a run checks beyond the test's own assertions:
  * the engine workspace, every cudaMalloc and every torch.empty of the host mirrors start poisoned (0xFF bytes: NaN / -1),
  * launch limits of sm_90 (block size, grid dims, dynamic shared memory vs the opt-in) and a canary behind the dynamic
    shared memory of every block (tools/cuda_emu/cuda_emu.h),
  * DQMC_EMU_REVERSE=1: the threads of a block run from the highest index down (a missing barrier passes in one order at most),
  * DQMC_EMU_REVERSE_BLOCKS=1: the grid is walked backwards (blocks of one launch that depend on each other),
  * guard zones behind every buffer carved from the engine workspace (engine.cu Arena::take), verified after each chunk,
  * --asan: the kernels are compiled with AddressSanitizer (out-of-bounds global accesses; run with
    LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0:detect_stack_use_after_return=0).
The wgmma / TMA kernels are not emulated (the build sets DQMC_NO_TCGEN05): engines are created with gemm_backend = 0.

The emulator replaces ex2.approx / rcp.approx / redux.sync by exact code: it checks layouts and protocols, never accuracy.

Usage:  python tools/emu_run_tests.py [--lib PATH] [--nobuild] [--asan] test_name[substring] [test_name ...]
        python tools/emu_run_tests.py --all-small          (every test small enough for the emulator, parity files)
Tests come from test_gpu_parity.py, test_gpu_z_next_rows.py, test_gpu_ecp_cutoff.py, test_gpu_force.py, test_gpu_reverse_chunks.py,
test_gpu_reverse_conformance.py, test_gpu_slater_conformance.py, test_gpu_zv_force.py and test_gpu_deeperwin.py; stacked parametrize marks run
as their cartesian product, and `name[substring]` keeps the cases whose arguments' repr contains the substring.
"""
import argparse
import importlib
import os
import pathlib
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

# full-size / tensor-core tests: hours on the emulator, or not emulable
TOO_BIG = {'test_full_size_properties_4096_walkers', 'test_benzene_full_psiformer_fp32_tensor_core_vs_fp64',
           'test_ferminet_n2_full_fp32_tensor_core_vs_fp64', 'test_engine_external_fixtures',
           'test_benzene_fp32_cutoff_equals_all_pairs', 'test_benzene_walker_isolation_mixed_active_counts',
           'test_cutoff_quadrature_chunking_bitwise'}


def build(out, asan=False):
    cmd = ['g++', '-std=c++17', '-O1', '-g', '-DDQMC_EMU', '-DDQMC_NO_TCGEN05', '-x', 'c++', f'-I{ROOT}/tools/cuda_emu', f'-I{ROOT}/include',
           f'-I{ROOT}/deepqmc_b200/csrc', '-fPIC', '-shared', f'{ROOT}/deepqmc_b200/csrc/engine.cu', '-o', out]
    if asan:
        cmd[1:1] = ['-fsanitize=address', '-fno-omit-frame-pointer']
    subprocess.check_call(cmd)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', default='/tmp/libdqmc_emu.so')
    ap.add_argument('--nobuild', action='store_true')
    ap.add_argument('--asan', action='store_true')
    ap.add_argument('--all-small', action='store_true')
    ap.add_argument('names', nargs='*')
    a = ap.parse_args()
    if not a.nobuild:
        build(a.lib, a.asan)

    import torch

    import deepqmc_b200.engine as E

    engine_init = E.Engine.__init__

    def init(self, *args, **kw):
        kw['_lib_path'], kw['gemm_backend'] = a.lib, 0
        engine_init(self, *args, **kw)

    E.Engine.__init__ = init
    workspace = E.Engine.workspace

    def poisoned_workspace(self, *args, **kw):
        w = workspace(self, *args, **kw)
        w.fill_(255)
        return w

    E.Engine.workspace = poisoned_workspace

    class TorchProxy:  # torch.empty / empty_like of the host mirrors return poisoned memory, like fresh device memory may
        def __getattr__(self, k):
            return getattr(torch, k)

        @staticmethod
        def _poison(t):
            if t.numel():
                t.view(-1).view(torch.uint8).fill_(255)
            return t

        def empty(self, *args, **kw):
            return self._poison(torch.empty(*args, **kw))

        def empty_like(self, *args, **kw):
            return self._poison(torch.empty_like(*args, **kw))

    for m in ('engine', 'hamil', 'sampling', 'ansatz', 'energy', 'overlap', 'parallel', 'force'):
        mod = importlib.import_module('deepqmc_b200.' + m)
        if hasattr(mod, 'torch'):
            mod.torch = TorchProxy()

    import itertools

    import pytest

    pytest_param_type = type(pytest.param(0))
    import test_gpu_deeperwin as DW
    import test_gpu_ecp_cutoff as EC
    import test_gpu_force as FC
    import test_gpu_parity as P
    import test_gpu_reverse_chunks as RC
    import test_gpu_reverse_conformance as RV
    import test_gpu_slater_conformance as SC
    import test_gpu_z_next_rows as Z
    import test_gpu_zv_force as ZV

    P.DEV = Z.DEV = SC.DEV = EC.DEV = FC.DEV = RC.DEV = RV.DEV = ZV.DEV = DW.DEV = 'cpu'
    torch.cuda.synchronize = lambda *args, **kw: None
    names = list(a.names)
    if a.all_small:
        names += [n for mod in (P, Z, EC) for n in vars(mod) if n.startswith('test_') and n not in TOO_BIG and n not in names]
    for name in names:
        # name or name[substring]: the cases whose printed arguments contain the substring
        name, _, sel = name.partition('[')
        sel = sel.rstrip(']')
        f = (getattr(Z, name, None) or getattr(P, name, None) or getattr(EC, name, None) or getattr(FC, name, None)
             or getattr(RC, name, None) or getattr(RV, name, None) or getattr(ZV, name, None) or getattr(DW, name, None)
             or getattr(SC, name))
        wants_tmp = 'tmp_path' in f.__code__.co_varnames[:f.__code__.co_argcount]
        # stacked parametrize marks: the cartesian product of their cases, passed by argument name
        axes = []
        for m in (m for m in getattr(f, 'pytestmark', []) if m.name == 'parametrize'):
            argnames, values = m.args[:2]
            argnames = [s.strip() for s in argnames.split(',')] if isinstance(argnames, str) else list(argnames)
            tups = [tuple(v.values) if isinstance(v, pytest_param_type) else (v,) if len(argnames) == 1 else tuple(v)
                    for v in values]
            axes.append([dict(zip(argnames, t)) for t in tups])
        for combo in itertools.product(*axes):
            kw = {k: v for d in combo for k, v in d.items()}
            if sel and sel not in repr(kw):
                continue
            if wants_tmp:
                kw['tmp_path'] = pathlib.Path(tempfile.mkdtemp())
            f(**kw)
            print('ok', name, kw, flush=True)


if __name__ == '__main__':
    main()
