"""CPU: the wgmmas of the whole-trunk kernel and the fused MLP block stay in flight back to back (cuobjdump -sass).

ptxas serialises a kernel's wgmmas (one warpgroup arrive and one wait around every HGMMA, warning C7518) when it cannot
prove the code between them warpgroup-convergent, for example after a divergent spin loop in front of a GEMM.  The
pipelined code has one WARPGROUP.ARRIVE per slot of a GEMM call site (4 per site: the trunk has two sites, the MLP block
one), far fewer than its HGMMAs.  Skips when the library or cuobjdump is missing.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'deepqmc_b200', 'libdqmc_b200.so')
KERNELS = {f'_ZN2dq2tc16trunk_f16_kernelILi{np}EEEvNS0_11TrunkParamsE': 2 for np in (1, 2, 4, 8, 16, 32)}
KERNELS.update({f'_ZN2dq2tc20mlp_block_f16_kernelILi{d}EEEv14CUtensorMap_stS2_S2_S2_S2_S2_NS0_9MlpParamsE': 1 for d in (128, 256)})


def _cuobjdump():
    for c in (os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'cuobjdump'), shutil.which('cuobjdump')):
        if c and os.access(c, os.X_OK):
            return c
    return None


@pytest.mark.parametrize('name', sorted(KERNELS))
def test_wgmmas_not_serialised(name):
    tool = _cuobjdump()
    if tool is None or not os.path.exists(LIB):
        pytest.skip('needs the built library and cuobjdump')
    out = subprocess.run([tool, '-sass', '-fun', name, LIB], capture_output=True, text=True).stdout
    ins = [t.strip() for t in re.findall(r'/\*[0-9a-f]{4,}\*/\s+([^;]*);', out)]
    assert ins, f'{name} is not in the library'
    hgmma = sum('HGMMA' in t for t in ins)
    arrive = sum('WARPGROUP.ARRIVE' in t for t in ins)
    assert hgmma == 12 * KERNELS[name], (name, hgmma)
    assert arrive == 4 * KERNELS[name], f'{name}: {arrive} warpgroup arrives for {hgmma} HGMMAs (serialised wgmmas)'
