import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


EMULATE = os.environ.get("BDEPTH_EMULATE") == "1"


# BDEPTH_EMULATE=1 (TEST INFRASTRUCTURE): the `gpu` tests run on the CPU against tests/emul/libbdepth_emul.so, the same pipeline
# and kernels compiled with g++ over a CUDA-on-CPU emulation (tests/emul/cuda_shim.hpp).  The multi-GPU tests run with ranks
# as threads over an NCCL stand-in; every gpu test has an emulation-sized variant of its input.  Nothing of this ever touches
# the product library.


@pytest.fixture(scope="session", autouse=True)
def _build_everything():
    """Build the oracle, the generator, the emulation harness and (cross-compile) libbdepth.so once."""
    import __graft_entry__ as g
    g.build(quiet=True)
    if EMULATE:
        import helpers
        import sambamba_b200._lib as L
        emul = os.path.join(ROOT, "tests", "emul")
        L.lib_path = lambda: os.path.join(emul, "libbdepth_emul.so")
        L._lib = None                      # build() has loaded the product library: drop the cached handle
        helpers.CLI = os.path.join(emul, "sambamba-depth-emul")
    yield
