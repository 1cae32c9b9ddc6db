"""Test configuration.

`-m "not gpu"` tests run on a CPU-only box: oracle vs golden vectors, host
logic, C-ABI exports.  `-m gpu` tests are the parity tests proper: they drive
libbifrost_b200.so through the Python/ctypes boundary on a real H100 and
compare with the oracle (and with stored outputs of the reference's own CUDA code).
"""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# bfProcLog* / ring status files of the test processes go to a scratch directory
# (read by the library on first use; default /dev/shm/bifrost as in the reference)
if 'BIFROST_B200_PROCLOG_DIR' not in os.environ:
    import tempfile
    os.environ['BIFROST_B200_PROCLOG_DIR'] = tempfile.mkdtemp(prefix='bfb_proclog_')
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on a machine with an H100)")
    lib = os.path.join(ROOT, 'bifrost_b200', 'lib', 'libbifrost_b200.so')
    if not os.path.exists(lib):
        # Building the product library is allowed from tests (it is never *used*
        # for compute on a CPU-only box).
        subprocess.check_call(['make', '-C', os.path.join(ROOT, 'bifrost_b200', 'csrc'), '-j8'])


def _has_gpu():
    try:
        import ctypes
        from bifrost_b200.libbifrost import _bf
        n = ctypes.c_int(-1)
        return _bf.bfDeviceGet(ctypes.byref(n)) == 0
    except Exception:
        return False


HAS_GPU = None


def pytest_collection_modifyitems(config, items):
    global HAS_GPU
    if HAS_GPU is None:
        HAS_GPU = _has_gpu()
    if HAS_GPU:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)
