"""GPU: the parameter reverse pass in chunks.  dqmc_wf_vjp_params over a workspace capped to two walkers per chunk against
one chunk, for every ansatz kind.  Sign and log of psi are per-walker values and must be bitwise equal; the parameter
gradients are atomic sums over walkers, so they agree to round-off: fp64 1e-12, fp32 1e-5 of each array's largest entry."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from deepqmc_b200.engine import MODE_VJP
from test_gpu_parity import DEV, make

HYPER = {
    'psiformer': dict(embedding_dim=32, n_layers=2, n_heads=4, n_determinants=4),
    'transpsiformer': dict(embedding_dim=32, n_layers=2, n_heads=4, n_determinants=4),
    'ferminet': dict(embedding_dim=32, n_layers=2, n_determinants=4, edge_dim=8),
    'paulinet': dict(),
    'paulinet_default': dict(embedding_dim=16, n_determinants=3, edge_dim=8),
}
TOL = {'float64': 1e-12, 'float32': 1e-5}


@pytest.mark.parametrize('dtype', ['float64', 'float32'])
@pytest.mark.parametrize('kind', list(HYPER))
def test_vjp_params_in_chunks_matches_one_chunk(kind, dtype):
    B = 7
    mol, hamil, oh, ansatz, params, r, R = make('LiH', B=B, kind=kind, dtype=dtype, **HYPER[kind])
    ansatz.gemm_backend = 1 if dtype == 'float32' and ansatz.spec.embedding_dim % 32 == 0 else 0  # tensor cores where they serve
    eng = ansatz.engine_for(hamil, params)
    r, R = r.to(eng.dtype), R.to(eng.dtype)
    w = torch.as_tensor(np.random.default_rng(3).normal(size=B), device=DEV).to(eng.dtype)
    s1, l1, g1 = eng.vjp_params(r, R, w)  # the first call may also upload parameters (TransPsiformer: nuclear stream at R)
    n0 = eng.launch_count
    s3, l3, g3 = eng.vjp_params(r, R, w, max_ws_bytes=eng.workspace_bytes(2, MODE_VJP))
    n1 = eng.launch_count
    eng.vjp_params(r, R, w)
    n2 = eng.launch_count
    assert n1 - n0 >= 3 * (n2 - n1)  # every chunk launches the same kernels: at least three chunks ran
    assert torch.equal(s1, s3) and torch.equal(l1, l3)
    assert set(g1) == set(g3)
    for k, g in g1.items():
        assert float((g3[k] - g).abs().max()) <= TOL[dtype] * float(g.abs().max()), k
