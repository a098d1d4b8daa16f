"""Development tool: run the kernel sources on the CPU emulator (tools/cuda_emu) and compare
with the oracle.  NOT part of the product or of the pytest suites' parity claims -- it exists
because the build container has no GPU and GPU minutes are scarce.  Usage:
    python tools/emu_check.py [--mol LiH] [--d 16] [--layers 2] [--B 3]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch


def build_emu(out='/tmp/libdqmc_emu.so'):
    cmd = ['g++', '-std=c++17', '-O1', '-g', '-DDQMC_EMU', '-DDQMC_NO_TCGEN05', '-x', 'c++', f'-I{ROOT}/tools/cuda_emu',
           f'-I{ROOT}/include', f'-I{ROOT}/deepqmc_b200/csrc', '-fPIC', '-shared',
           f'{ROOT}/deepqmc_b200/csrc/engine.cu', '-o', out]
    subprocess.check_call(cmd)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--mol', default='LiH')
    ap.add_argument('--d', type=int, default=16)
    ap.add_argument('--layers', type=int, default=2)
    ap.add_argument('--heads', type=int, default=2)
    ap.add_argument('--K', type=int, default=3)
    ap.add_argument('--B', type=int, default=3)
    ap.add_argument('--ecp', default=None)
    ap.add_argument('--kind', default='psiformer')
    ap.add_argument('--dtype', default='float64')
    ap.add_argument('--nobuild', action='store_true')
    a = ap.parse_args()
    lib = '/tmp/libdqmc_emu.so' if a.nobuild else build_emu()
    from deepqmc_b200 import params as PN
    from deepqmc_b200.engine import Engine
    from deepqmc_b200.molecule import Molecule
    from deepqmc_b200.spec import ferminet_spec, paulinet_default_spec, paulinet_spec, psiformer_spec, transpsiformer_spec
    from oracle import wf
    from oracle.hamil import OracleHamiltonian

    mol = Molecule.from_name(a.mol)
    h = OracleHamiltonian(mol, ecp_type=a.ecp)
    mk = {'psiformer': psiformer_spec, 'ferminet': ferminet_spec, 'transpsiformer': transpsiformer_spec, 'paulinet': paulinet_spec, 'paulinet_default': paulinet_default_spec}[a.kind]
    spec = (mk(h, n_layers=a.layers) if a.kind == 'paulinet' else mk(h, n_layers=a.layers, embedding_dim=a.d, n_determinants=a.K, edge_dim=8)) if a.kind.startswith('paulinet') else mk(h, embedding_dim=a.d, n_layers=a.layers, n_heads=a.heads, n_determinants=a.K)
    params = PN.perturb_params(PN.init_params(spec, 0))
    pt = wf.to_torch(params)
    rng = np.random.default_rng(0)
    N = spec.n_elec
    R = torch.as_tensor(mol.coords)
    r = torch.as_tensor(mol.coords[rng.integers(0, len(mol.coords), size=(a.B, N))] + rng.normal(size=(a.B, N, 3)))
    eng = Engine(spec, h, dtype=a.dtype, _lib_path=lib)
    eng.set_params(params)
    sign, log = eng.wf_forward(r, R)
    J = 0 if h.nl_params is None else len(np.unique(np.nonzero(h.nl_params)[0]))
    twist = torch.as_tensor(rng.uniform(0, np.pi / 5, size=(a.B, max(J, 1), N)))
    E, stats, s2, l2, grad = eng.local_energy(r, R, ecp_twist=twist if J else None, want_grad=True)
    for b in range(a.B):
        f = lambda x: wf.log_psi(spec, pt, x, R)
        so, lo = f(r[b])
        eo, st = h.local_energy(f, r[b], R, phi_random=twist[b] if J else None)
        print(f'b={b} sign {sign[b].item():+.0f}/{so.item():+.0f} dlog {abs(log[b].item()-lo.item()):.2e} '
              f'dlogFL {abs(l2[b].item()-lo.item()):.2e} dE {abs(E[b].item()-eo.item()):.2e} (E={eo.item():.6f}) '
              + ' '.join(f"{k.split('/')[1]}:{abs(stats[i, b].item()-v.item()):.1e}" for i, (k, v) in enumerate(st.items())))
    # Metropolis with injected noise
    from oracle.sampling import metropolis_step
    nsub = 3
    nn = torch.as_tensor(rng.normal(size=(nsub, a.B, N, 3)))
    nu = torch.as_tensor(rng.uniform(size=(nsub, a.B)))
    dt = eng.dtype
    state = dict(r=r.to(dt).clone(), sign=sign.clone(), log=log.clone(), age=torch.zeros(a.B, dtype=torch.int32),
                 tau=torch.tensor([0.3], dtype=dt))
    ost = dict(r=r.clone(), sign=sign.to(torch.float64).clone(), log=log.to(torch.float64).clone(),
               age=torch.zeros(a.B, dtype=torch.int32), tau=torch.tensor(0.3, dtype=torch.float64))
    stats = eng.mcmc_sweep(state, R, nsub, max_age=2, noise_normal=nn, noise_uniform=nu)
    wfb = lambda rr: tuple(torch.stack(x) for x in zip(*[wf.log_psi(spec, pt, rr[b], R) for b in range(a.B)]))
    for s in range(nsub):
        ost, acc = metropolis_step(wfb, ost, nn[s], nu[s], 0.57, 2)
    print('mcmc dr', (state['r'] - ost['r']).abs().max().item(), 'dlog', (state['log'] - ost['log']).abs().max().item(),
          'age', state['age'].tolist(), ost['age'].tolist(), 'tau', state['tau'].item(), ost['tau'].item(),
          'acc', stats[0].item(), acc.item())
    print('stats', stats.tolist())


if __name__ == '__main__':
    main()
