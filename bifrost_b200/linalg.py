"""bf.linalg.LinAlg (mirrors python/bifrost/linalg.py:38-67 -> bfLinAlg*)."""
from bifrost_b200.libbifrost import _bf, _check, BifrostObject
from bifrost_b200.ndarray import asarray
from bifrost_b200.map import DETECT_MODES


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

    def beamform_detect(self, w, x, out, mode='stokes', nint=1):
        """out = power beams of w.x: the beams C = w.x (w [..., nb, K],
        x [..., K, ntime], as matmul's a.b), detected with `mode` ('scalar',
        'stokes', 'stokes_i' or 'coherence'; polarised modes take beam rows
        2j, 2j+1 as pols x, y of beam j) and summed over nint samples:
        out f32 [..., nb/npb, nprod, ntime/nint].  Bit for bit
        reduce(detect(matmul(1, w, x, 0, C) as [..., nb/npb, npb, ntime]), nint),
        in one kernel for cf32 / ci16 w and ci4 / ci8 x (bfLinAlgBeamformDetect)."""
        m = DETECT_MODES[mode] if isinstance(mode, str) else int(mode)
        _check(_bf.bfLinAlgBeamformDetect(self.obj, asarray(w).as_BFarray(), asarray(x).as_BFarray(),
                                          m, int(nint), asarray(out).as_BFarray()))
        return out
