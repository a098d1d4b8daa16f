"""CPU: code size of the whole-trunk kernel and the fused MLP block in the built library (cuobjdump -sass).

The trunk runs its whole layer body once per (tile, layer) and warp as straight-line code, and its two warpgroups sit at
different points of it (ping-pong), so the body has to stay small: one instance per walker slot carrying only its own
attention variant, one call site per GEMM shape, and epilogues rolled over column quarters.  Skips when the library or
cuobjdump is missing.
"""
import os
import re
import shutil
from collections import Counter

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'deepqmc_b200', 'libdqmc_b200.so')
SLOTS = (1, 2, 4, 8, 16, 32)
TRUNK_BUDGET = 128 * 1024  # bytes of SASS per trunk instance
MLP_BUDGET = 64 * 1024     # bytes of SASS per fused MLP block instance


def _cuobjdump():
    for c in (os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'cuobjdump'), shutil.which('cuobjdump')):
        if c and os.access(c, os.X_OK):
            return c
    return None


@pytest.fixture(scope='module')
def sass():
    tool = _cuobjdump()
    if tool is None or not os.path.exists(LIB):
        pytest.skip('needs the built library and cuobjdump')
    import subprocess

    funcs = {}
    for name in [f'_ZN2dq2tc16trunk_f16_kernelILi{np}EEEvNS0_11TrunkParamsE' for np in SLOTS] + [
            f'_ZN2dq2tc20mlp_block_f16_kernelILi{d}EEEv14CUtensorMap_stS2_S2_S2_S2_S2_NS0_9MlpParamsE' for d in (128, 256)]:
        out = subprocess.run([tool, '-sass', '-fun', name, LIB], capture_output=True, text=True).stdout
        ins = [t.strip() for t in re.findall(r'/\*[0-9a-f]{4,}\*/\s+([^;]*);', out)]
        assert ins, f'{name} is not in the library'
        funcs[name] = Counter(re.sub(r'^@!?U?P\w+\s+', '', t).split()[0] for t in ins)
    return funcs


def _trunk(sass, np):
    return sass[f'_ZN2dq2tc16trunk_f16_kernelILi{np}EEEvNS0_11TrunkParamsE']


def _ops(c, prefix):
    return sum(v for k, v in c.items() if k.split('.')[0] == prefix)


@pytest.mark.parametrize('np', SLOTS)
def test_trunk_instance_size(sass, np):
    c = _trunk(sass, np)
    size = 16 * sum(c.values())
    assert size <= TRUNK_BUDGET, f'trunk_f16_kernel<{np}>: {size} bytes of SASS'
    assert _ops(c, 'LDL') == 0 and _ops(c, 'STL') == 0, 'the trunk keeps its accumulator in registers'


def test_trunk_one_attention_variant_per_instance(sass):
    """Slots of at most 16 rows run the 2-key-tile attention task, 32-row slots the 4-key-tile one, and every instance
    carries the tensor-core MMAs (HMMA) of exactly one of the two: a small-slot instance has fewer than the 32-row one, and
    the 32-row one (twice the key tiles: about twice the MMAs) fewer than twice the largest small-slot one, where both
    tasks together would come to about three times."""
    hmma = {np: _ops(_trunk(sass, np), 'HMMA') for np in SLOTS}
    small = [hmma[np] for np in SLOTS if np <= 16]
    assert min(small) > 0 and max(small) < hmma[32] < 2 * max(small), hmma


@pytest.mark.parametrize('d', (128, 256))
def test_mlp_block_size(sass, d):
    c = sass[f'_ZN2dq2tc20mlp_block_f16_kernelILi{d}EEEv14CUtensorMap_stS2_S2_S2_S2_S2_NS0_9MlpParamsE']
    size = 16 * sum(c.values())
    assert size <= MLP_BUDGET, f'mlp_block_f16_kernel<{d}>: {size} bytes of SASS'
    assert _ops(c, 'LDL') == 0 and _ops(c, 'STL') == 0
    assert _ops(c, 'HGMMA') == 12, 'one call site of the GEMM for Wo, W1 and W2'
