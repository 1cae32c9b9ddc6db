"""Overlay of the H100 hot path on a stock libbifrost binding.

The reference's Python package binds ``libbifrost.so`` through a ctypes
namespace (``bifrost/libbifrost.py:38-40``: ``import
bifrost.libbifrost_generated as _bf``).  ``apply(_bf, lib)`` rebinds the
hot-path symbols of that namespace to ``libbifrost_b200.so`` and leaves every
other symbol -- rings, proclog, affinity, UDP, file I/O, ``bfMap`` for arbitrary
expressions -- with the stock library.  Argument types and struct layouts are
identical (``include/bifrost_b200.h`` vs ``src/bifrost/*.h``), so the stock
prototypes are carried over to the new functions.

    import bifrost.libbifrost_generated as _bf
    from bifrost_b200.overlay import apply
    apply(_bf, '/path/to/libbifrost_b200.so')

INTEGRATION.md section 2 shows the same thing inline; tests/test_overlay.py
runs it against a stand-in for the stock library.
"""
import ctypes

HOT_PATH = (
    'bfTranspose', 'bfReduce', 'bfUnpack', 'bfQuantize',
    'bfFdmtCreate', 'bfFdmtInit', 'bfFdmtSetStream', 'bfFdmtExecute', 'bfFdmtDestroy',
    'bfFftCreate', 'bfFftInit', 'bfFftExecute', 'bfFftDestroy',
    'bfLinAlgCreate', 'bfLinAlgDestroy', 'bfLinAlgMatMul',
)
# Both libraries keep a per-thread stream / device: calls that set them go to both.
MIRRORED = ('bfStreamSet', 'bfDeviceSet', 'bfDeviceSetById')


def apply(namespace, lib, names=HOT_PATH):
    """Rebinds `names` in `namespace` to the functions of `lib` (a path or a
    loaded ctypes.CDLL).  Returns the list of names rebound (a name the
    namespace does not have, or `lib` does not export, is skipped)."""
    if not isinstance(lib, ctypes.CDLL):
        lib = ctypes.CDLL(lib, mode=ctypes.RTLD_GLOBAL)
    done = []
    for name in names:
        old = getattr(namespace, name, None)
        new = getattr(lib, name, None)
        if old is None or new is None:
            continue
        # same prototypes: keep the stock binding's argument / result types
        if getattr(old, 'argtypes', None) is not None:
            new.argtypes = old.argtypes
        new.restype = getattr(old, 'restype', ctypes.c_int)
        setattr(namespace, name, new)
        done.append(name)
    for name in MIRRORED:
        stock = getattr(namespace, name, None)
        ours = getattr(lib, name, None)
        if stock is None or ours is None:
            continue
        if getattr(stock, 'argtypes', None) is not None:
            ours.argtypes = stock.argtypes
        ours.restype = getattr(stock, 'restype', ctypes.c_int)

        def both(*args, _stock=stock, _ours=ours):
            _ours(*args)
            return _stock(*args)
        setattr(namespace, name, both)
    return done
