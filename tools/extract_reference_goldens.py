"""Extract the PARAM-FREE goldens of the reference's own test-suite into a small JSON fixture.

Run against a checkout of the reference (reads <reference>/tests/**/*.npz):
    python tools/extract_reference_goldens.py <reference>/tests
Only numbers are extracted (regression *data*), no reference source.  The parameter-dependent
goldens (psi, its parameter gradient, Laplacian, E_loc of the Haiku-initialised test ansatz) are
reproduced in tests/test_oracle_goldens.py by regenerating the Haiku / jax.random initialisation
in numpy (oracle/jaxrand.py); the walker is recovered from the edge-builder golden.
"""
import json
import os
import sys

import numpy as np

REF = sys.argv[1] if len(sys.argv) > 1 else 'tests'
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden', 'reference_goldens.json')


def npz(path):
    d = np.load(os.path.join(REF, path))
    return {k: d[k].tolist() for k in d.files}


def main():
    g = {
        'source': 'deepqmc/deepqmc v1.3.0 tests/*.npz (ndarrays_regression fixtures)',
        'molecule': {n: npz(f'test_molecule/test_from_name_{n}_.npz') for n in ('LiH', 'C', 'H2O', 'NH3', 'H10', 'ScO', 'bicyclobutane')},
        'hamil_init': {
            'Molecular': npz('test_hamil/test_init_Molecular_.npz'),
            'Molecular_PP': npz('test_hamil/test_init_Molecular_PP_.npz'),
        },
        'edge_builder_LiH': npz('test_gnn/test_molecular_graph_edge_builder.npz'),
        'graph_edge_builder_mask_self_True': npz('test_gnn/test_graph_edge_builder_mask_self_True_.npz'),
        'graph_edge_builder_mask_self_False': npz('test_gnn/test_graph_edge_builder_mask_self_False_.npz'),
        'potential_LiH_None': npz('test_potential/test_pseudo_potentials_LiH_None_.npz'),
        'potential_C_None': npz('test_potential/test_pseudo_potentials_C_None_.npz'),
        # parameter-tree names and shapes of the reference's test ansatz (tests/conf/ansatz.yaml on LiH): the keys of
        # tests/test_wf/test_grad_psi.npz are the Haiku paths (values are gradients, which need the Haiku-initialised
        # parameters and are not reproducible here)
        'test_ansatz_param_shapes': {k: list(np.load(os.path.join(REF, 'test_wf/test_grad_psi.npz'))[k].shape)
                                     for k in np.load(os.path.join(REF, 'test_wf/test_grad_psi.npz')).files},
        # d log|psi| / d params of the test ansatz with its Haiku-initialised parameters (tests/test_wf.py test_grad_psi)
        'wf_grad_psi': npz('test_wf/test_grad_psi.npz'),
        'wf_psi': npz('test_wf/test_psi.npz'),
        # electron embeddings of the bare 4-interaction ElectronGNN of tests/conf/gnn.yaml (tests/test_gnn.py TestGNN)
        'gnn_embedding': npz('test_gnn/test_embedding.npz'),
        # walkers drawn by AtomCenteredElectronInitializer(ShellBasedDistribution()) from split(PRNGKey(0), 5)
        'init_sample_Molecular': npz('test_hamil/test_init_sample_Molecular_.npz'),
        # carbon atom: plain Coulomb and ccECP potentials on the PRNGKey(0) walker (tests/test_potential.py)
        'potential_C_ccECP': npz('test_potential/test_pseudo_potentials_C_ccECP_.npz'),
        'potential_C_bfd': npz('test_potential/test_pseudo_potentials_C_bfd_.npz'),
        # LiH with ccECP on lithium: walkers, potentials and E_loc (tests/test_hamil.py, tests/test_potential.py)
        'init_sample_Molecular_PP': npz('test_hamil/test_init_sample_Molecular_PP_.npz'),
        'potential_LiH_ccECP': npz('test_potential/test_pseudo_potentials_LiH_ccECP_.npz'),
        'local_energy_Molecular_PP': npz('test_hamil/test_local_energy_Molecular_PP_.npz'),
        # sampler fixtures (tests/test_sampling.py): state after init(PRNGKey(0)) and after sample(PRNGKey(step)), step < 4
        'sampling': {k: npz(f'test_sampling/test_sampler_{k}_.npz') for k in
                     ('init_Metropolis', 'init_Langevin', 'sample_Metropolis', 'sample_DecorrMetropolis', 'sample_Langevin')},
        # MultiNuclearGeometrySampler over two copies of LiH (tests/test_sampling.py TestMultimoleculeSampling)
        'sampling_multi': {k: npz(f'test_sampling/test_multi_nuclear_geometry_sampler_{k}_Metropolis_.npz') for k in ('init', 'sample')},
        'wf_laplace': npz('test_wf/test_laplace_psi.npz'),
        'local_energy_Molecular': npz('test_hamil/test_local_energy_Molecular_.npz'),
        # reference tests/test_physics.py:7-17 and tests/test_geom.py:8-18 (inline known answers)
        'coulomb_kat': {'R': [[0, 0, 0], [0, 0, 1.4]], 'r': [[0, 0, 0], [0, 0, 1.0]], 'ns_valence': [1.0, 1.0],
                        'nuclear_energy': 1 / 1.4, 'electronic_potential': 1.0,
                        'pairwise_distance': [[0.0, 1.4], [1.0, 0.4]]},
    }
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    with open(OUT, 'w') as f:
        json.dump(g, f, indent=1)
    print('wrote', OUT)


if __name__ == '__main__':
    main()
