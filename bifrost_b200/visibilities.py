"""bf.visibilities: the correlator's output in the forms that follow it
(the data path of blocks/convert_visibilities.py, python/bifrost/blocks/
convert_visibilities.py:86-180 of the reference, as compiled kernels).

All arrays are cf32 in CUDA space; leading (time) dims are batch dims.  Only
the lower triangle of a matrix input (r >= s over r = 2 station + pol) is read.
"""
from bifrost_b200.libbifrost import _bf, _check
from bifrost_b200.ndarray import asarray


def fill_hermitian(idata, odata):
    """idata, odata: [..., n, n].  odata = idata on and below the diagonal,
    conj(idata.T) above it."""
    _check(_bf.bfVisibilitiesFillHermitian(asarray(idata).as_BFarray(), asarray(odata).as_BFarray()))
    return odata


def to_storage(idata, odata):
    """idata: [..., nchan, nstand, 2, nstand, 2] (lower-filled),
    odata: [..., nstand (nstand + 1) / 2, nchan, 4] Stokes I, Q, U, V of
    baseline b = i (i + 1) / 2 + j, i >= j."""
    _check(_bf.bfVisibilitiesToStorage(asarray(idata).as_BFarray(), asarray(odata).as_BFarray()))
    return odata


def from_storage(idata, odata):
    """The inverse of to_storage: odata [..., nchan, nstand, 2, nstand, 2] is
    written in full (the upper triangle mirrors the lower)."""
    _check(_bf.bfVisibilitiesFromStorage(asarray(idata).as_BFarray(), asarray(odata).as_BFarray()))
    return odata
