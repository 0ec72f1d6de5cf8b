"""pyscf_b200 — H100-native J/K Fock-matrix builder behind PySCF's get_jk surface."""
__version__ = '0.1.0'
from . import gto
