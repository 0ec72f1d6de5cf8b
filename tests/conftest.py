import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run with -m gpu on an H100)')


from pyscf_b200.gto.mole import geometry
H2O = geometry('h2o')
BENZENE = geometry('benzene')

EMU_LIB = os.path.join(ROOT, 'tests', 'emu', 'libb200jk_emu.so')


@pytest.fixture(scope='session')
def emu_lib():
    import subprocess
    subprocess.check_call(['make', '-s', '-C', os.path.join(ROOT, 'pyscf_b200', 'csrc'), 'emu'])  # incremental
    return EMU_LIB


@pytest.fixture(scope='session')
def emu_lib_experimental():
    """The emulation compiled with the experimental lane layouts on (-DB2_PBMAX=4 -DB2_PPW=1 -DB2_TPQ_KOUTER=1), see DESIGN.md §4.1."""
    import subprocess
    subprocess.check_call(['make', '-s', '-C', os.path.join(ROOT, 'pyscf_b200', 'csrc'), 'emu_x'])
    return os.path.join(ROOT, 'tests', 'emu', 'libb200jk_emu_pbppw.so')
