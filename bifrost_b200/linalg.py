"""bf.linalg.LinAlg (mirrors python/bifrost/linalg.py:38-67 -> bfLinAlg*)."""
from bifrost_b200.libbifrost import _bf, _check, BifrostObject
from bifrost_b200.ndarray import asarray


class LinAlg(BifrostObject):
    def __init__(self):
        BifrostObject.__init__(self, _bf.bfLinAlgCreate, _bf.bfLinAlgDestroy)

    def matmul(self, alpha, a, b, beta, c):
        """c = alpha*a.b + beta*c; b None: alpha*a.a^H + beta*c; a None:
        alpha*b^H.b + beta*c.  Batch dims follow numpy.matmul.  The a.a^H /
        b^H.b forms write the lower triangle of c and take ci8, ci16, cf32
        or ci4 (high nibble real; bfLinAlgCorrelateCi4, which gives the bits
        of the ci8 call on the same integers)."""
        alpha = 1. if alpha is None else float(alpha)
        beta = 0. if beta is None else float(beta)
        a_array = asarray(a).as_BFarray() if a is not None else None
        b_array = asarray(b).as_BFarray() if b is not None else None
        fn = _bf.bfLinAlgMatMul
        x_array = b_array if a_array is None else a_array if b_array is None else None
        if x_array is not None and x_array.dtype == _bf.BF_DTYPE_CI4:
            fn = _bf.bfLinAlgCorrelateCi4
        _check(fn(self.obj, alpha, a_array, b_array, beta, asarray(c).as_BFarray()))
        return c

    def correlate_to_storage(self, x, vis):
        """vis = the Stokes storage layout of x^H.x, written straight from the
        correlator: x [nchan, ntime, 2 nstand] (ci8 / ci16 / cf32, or ci4
        through bfLinAlgCorrelateCi4ToStorage), vis [nstand (nstand + 1) / 2,
        nchan, 4] cf32.  Bit for bit visibilities.to_storage(matmul(1, None,
        x, 0, C)) with C [nchan, n, n]."""
        x_array = asarray(x).as_BFarray()
        fn = _bf.bfLinAlgCorrelateCi4ToStorage if x_array.dtype == _bf.BF_DTYPE_CI4 else \
            _bf.bfLinAlgCorrelateToStorage
        _check(fn(self.obj, x_array, asarray(vis).as_BFarray()))
        return vis
