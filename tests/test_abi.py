"""CPU: the C-ABI library loads and exports every symbol include/dqmc_b200.h declares
(no compute calls without a GPU), and the product fails loudly without its CUDA library."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, 'include', 'dqmc_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(dqmc_[a-z_0-9]+)\s*\(', src)))


def test_header_symbols_exported(built_lib):
    syms = _declared_symbols()
    assert len(syms) >= 14
    for s in syms:
        assert hasattr(built_lib, s), f'libdqmc_b200.so does not export {s}'
    from deepqmc_b200 import _lib

    assert sorted(_lib.SYMBOLS) == syms
    assert b'sm_90a' in built_lib.dqmc_version()


def test_sass_is_sm90a(built_lib):
    import subprocess

    from deepqmc_b200 import _lib

    out = subprocess.run(['cuobjdump', '-lelf', _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert 'sm_90a' in out


def test_no_cpu_fallback(monkeypatch, tmp_path):
    """Missing library -> ImportError; present library but no GPU -> RuntimeError."""
    import torch

    from deepqmc_b200 import _lib

    with pytest.raises(ImportError):
        _lib.load(str(tmp_path / 'libdqmc_b200.so'))
    if not torch.cuda.is_available():
        from deepqmc_b200.ansatz import B200Ansatz
        from deepqmc_b200.hamil import MolecularHamiltonian
        from deepqmc_b200.molecule import Molecule
        from deepqmc_b200.types import PhysicalConfiguration

        h = MolecularHamiltonian(mol=Molecule.from_name('LiH'))
        a = B200Ansatz(h, embedding_dim=16, n_layers=1, n_heads=2, n_determinants=2)
        pc = PhysicalConfiguration(torch.zeros(2, 3), torch.zeros(4, 3), torch.zeros(()))
        with pytest.raises(RuntimeError):
            a.apply(a.init(0), pc)


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, 'deepqmc_b200')
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith(('.py', '.cu', '.cuh', '.h')):
                txt = open(os.path.join(dp, f)).read()
                assert not re.search(r'^\s*(from|import)\s+oracle\b', txt, flags=re.M), f


def test_oracle_does_not_import_product():
    """The checker is independent of the thing it checks: nothing under oracle/ imports deepqmc_b200 (own table of the reference's
    Haiku parameter names in oracle/names.py, own jax.random / haiku-init restatement in oracle/jaxrand.py); hyper-parameter
    records (``spec``) and parameter dicts are handed in by the tests."""
    for dp, _, fs in os.walk(os.path.join(ROOT, 'oracle')):
        for f in fs:
            if f.endswith('.py'):
                txt = open(os.path.join(dp, f)).read()
                assert not re.search(r'^\s*(from|import)\s+deepqmc_b200\b', txt, flags=re.M), f
