"""deepqmc_b200 -- H100-native (sm_90a) local-energy / Metropolis hot path for DeepQMC-style
neural wave functions, behind the reference's Ansatz / Hamiltonian / ElectronSampler plugin
interfaces.  See DESIGN.md and INTEGRATION.md."""
from .molecule import Molecule
from .spec import AnsatzSpec, deeperwin_spec, ferminet_spec, psiformer_spec
from .types import PhysicalConfiguration, Psi

__all__ = ['Molecule', 'AnsatzSpec', 'psiformer_spec', 'ferminet_spec', 'deeperwin_spec', 'PhysicalConfiguration', 'Psi']
