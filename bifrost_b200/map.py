"""bf.map (python/bifrost/map.py -> bfMap) and the fixed-kernel entry points
behind the hot-path expressions.

``bf.map`` takes an arbitrary C++ expression over named arrays, like the
reference's: the library compiles it at run time with NVRTC for sm_90a
(csrc/map_jit.cu).  The two expression families the hot-path blocks use -- the
detect products (blocks/detect.py:87-136) and the accumulate update
(blocks/accumulate.py:67) -- are recognised and run as compiled kernels
(``bfDetect`` / ``bfAccumulate``), which is also what ``detect`` /
``accumulate`` below call directly.
"""
import ctypes

import numpy as np

from bifrost_b200.libbifrost import _bf, _check, _array, BFarray
from bifrost_b200.ndarray import asarray, ndarray

DETECT_MODES = {'scalar': 0, 'jones': 1, 'stokes': 2, 'stokes_i': 3, 'coherence': 4}


def detect(idata, odata, mode='stokes', axis=None):
    """odata = detect(idata): |x|^2 ('scalar') or polarisation products along
    `axis` (length-2 pol axis of idata).  Semantics of blocks/detect.py:86-138."""
    mode = DETECT_MODES[mode] if isinstance(mode, str) else int(mode)
    if axis is None:
        axis = 0
    _check(_bf.bfDetect(asarray(idata).as_BFarray(), asarray(odata).as_BFarray(),
                        mode, int(axis)))
    return odata


def accumulate(idata, odata, beta=1.0):
    """odata = beta*odata + idata  (blocks/accumulate.py:63-74)."""
    _check(_bf.bfAccumulate(asarray(idata).as_BFarray(), asarray(odata).as_BFarray(),
                            float(beta)))
    return odata


def _is_scalar(x):
    return isinstance(x, (int, float, complex, np.number))


def _convert_to_array(arg):
    """Literals become immutable 1-element system arrays, which bfMap passes to
    the kernel by value (python/bifrost/map.py:44-56: int32 / float32 /
    complex64)."""
    if _is_scalar(arg):
        arr = np.array(arg)
        if isinstance(arg, (int, np.integer)) and -(1 << 31) <= int(arg) < (1 << 31):
            arr = arr.astype(np.int32)
        elif isinstance(arg, (float, np.floating)):
            arr = arr.astype(np.float32)
        elif isinstance(arg, (complex, np.complexfloating)):
            arr = arr.astype(np.complex64)
        arr = arr.reshape(1).view(ndarray)
        arr.flags['WRITEABLE'] = False
        arg = arr
    return asarray(arg)


def _marshal(data, shape, axis_names, block_axes):
    arg_arrays, arg_names, keepalive = [], [], []
    for key, arg in data.items():
        arg = _convert_to_array(arg)
        keepalive.append(arg)
        arg_arrays.append(arg.as_BFarray())
        arg_names.append(key)
    if block_axes is not None and axis_names is not None:
        block_axes = [list(axis_names).index(a) if isinstance(a, str) else a for a in block_axes]
    if block_axes is not None and len(block_axes) != 2:
        raise ValueError("block_axes must contain exactly 2 entries")
    return arg_arrays, arg_names, keepalive, block_axes


def _enc(x):
    return x.encode() if isinstance(x, str) else x


def map(func_string, data, axis_names=None, shape=None, func_name=None,
        extra_code=None, block_shape=None, block_axes=None):
    """Apply `func_string` to the arrays in `data` (dict name -> array/scalar).
    Signature and semantics of python/bifrost/map.py:map, e.g.

      bf.map("c = a + b", {'c': c, 'a': a, 'b': b})
      bf.map("c(i,j) = a(i) * b(j)", {'c': c, 'a': a, 'b': b}, axis_names=('i','j'))
      bf.map("c(i) = a(i,k)", {'c': c, 'a': a, 'k': 7}, ['i'], shape=c.shape)

    block_shape / block_axes are accepted for compatibility (tuning hints of
    the reference's launch; this implementation runs one flat grid-stride loop)."""
    if block_shape is not None and len(block_shape) != 2:
        raise ValueError("block_shape must contain exactly 2 entries")
    ndim = len(shape) if shape is not None else 0
    arg_arrays, arg_names, keepalive, block_axes = _marshal(data, shape, axis_names, block_axes)
    _check(_bf.bfMap(ndim, _array(shape, dtype=ctypes.c_long), _array(axis_names),
                     len(arg_arrays), _array(arg_arrays), _array(arg_names),
                     _enc(func_name), _enc(func_string), _enc(extra_code),
                     _array(block_shape), _array(block_axes)))


def compile_only(func_string, data, axis_names=None, shape=None, func_name=None,
                 extra_code=None, block_axes=None):
    """Compiles the kernel ``map`` would launch and returns 0 (array names are
    element references) or 1 (callable views).  Needs no GPU (bfMapCompile)."""
    ndim = len(shape) if shape is not None else 0
    arg_arrays, arg_names, keepalive, block_axes = _marshal(data, shape, axis_names, block_axes)
    mode = ctypes.c_int(-1)
    _check(_bf.bfMapCompile(ndim, _array(shape, dtype=ctypes.c_long), _array(axis_names),
                            len(arg_arrays), _array(arg_arrays), _array(arg_names),
                            _enc(func_name), _enc(func_string), _enc(extra_code),
                            _array(block_axes), ctypes.byref(mode)))
    return mode.value


def clear_map_cache():
    _check(_bf.bfMapClearCache())
