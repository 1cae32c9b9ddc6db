"""bifrost_b200 -- H100-native (sm_90a) implementation of the Bifrost GPU DSP
hot path behind the reference's C ABI and ``bifrost.blocks`` operator surface.

``import bifrost_b200 as bf`` exposes the subset of ``import bifrost as bf``
that the per-gulp path uses: ``bf.ndarray``/``asarray``/``empty``/..., the op
wrappers ``bf.transpose``, ``bf.reduce``, ``bf.fft.Fft``, ``bf.fdmt.Fdmt``,
``bf.pulse_search.PulseSearch``, ``bf.sk_flag.SkFlag``,
``bf.coherent_dedisp.CoherentDedisp``, ``bf.fold.Fold``,
``bf.period_search.PeriodSearch``,
``bf.linalg.LinAlg``, ``bf.unpack``, ``bf.map`` (fixed-kernel subset) and the
block classes in ``bf.blocks``.
"""
from bifrost_b200 import libbifrost, device, memory
from bifrost_b200.libbifrost import _bf, _th, _check, _get, EndOfDataStop, BifrostObject
from bifrost_b200.DataType import DataType
from bifrost_b200.Space import Space
from bifrost_b200.ndarray import (ndarray, asarray, empty, zeros, empty_like,
                                  zeros_like, copy_array, memset_array)
from bifrost_b200 import fdmt, fft, linalg, visibilities, pulse_search, sk_flag, coherent_dedisp, fold, \
    period_search
from bifrost_b200.reduce import reduce
from bifrost_b200.transpose import transpose
from bifrost_b200.unpack import unpack
from bifrost_b200.quantize import quantize
from bifrost_b200.map import map, detect, accumulate, clear_map_cache
from bifrost_b200.spectrometer import spectrometer
from bifrost_b200 import views
from bifrost_b200 import affinity, proclog
from bifrost_b200 import blocks
from bifrost_b200.pipeline import Pipeline, get_default_pipeline, block_scope, block_view

__version__ = '0.1.0'


def launch_count():
    """Number of kernels libbifrost_b200 has launched in this process."""
    import ctypes
    n = ctypes.c_ulonglong()
    _check(_bf.bfGetLaunchCount(ctypes.byref(n)))
    return n.value
