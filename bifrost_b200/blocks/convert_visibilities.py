"""convert_visibilities block (same contract as
python/bifrost/blocks/convert_visibilities.py:38-209 of the reference; the data
path is bfVisibilities*, compiled sm_90a kernels, instead of bfMap strings).

    matrix  ['time','freq','station_i','pol_i','station_j','pol_j'] (lower or hermitian)
      -> 'matrix'   the same tensor, Hermitian-filled
      -> 'storage'  ['time','baseline','freq','stokes'], Stokes I, Q, U, V
    storage ['time','baseline','freq','stokes']
      -> 'matrix'   the six-axis tensor, Hermitian-filled

Deliberate differences from the reference (DESIGN.md §8): diagonal entries of
the matrix fill are kept as they are, there is no 2048-station limit, storage
headers carry one scales / units entry per output axis, storage -> matrix sets
matrix_fill_mode = 'hermitian', and only cf32 with npol = 2 (storage forms) is
accepted."""
from bifrost_b200.pipeline import TransformBlock
from bifrost_b200.blocks import _header as H
from bifrost_b200 import visibilities

MATRIX_AXES = ['time', 'freq', 'station_i', 'pol_i', 'station_j', 'pol_j']
STORAGE_AXES = ['time', 'baseline', 'freq', 'stokes']
STOKES_UNITS = ['I', 'Q', 'U', 'V']
POL_UNITS = ['X', 'Y']


def _nstand(nbaseline):
    """nstand with nstand (nstand + 1) / 2 == nbaseline (integers only)."""
    lo, hi = 0, 1
    while hi * (hi + 1) // 2 < nbaseline:
        hi *= 2
    while lo < hi:
        mid = (lo + hi) // 2
        if mid * (mid + 1) // 2 < nbaseline:
            lo = mid + 1
        else:
            hi = mid
    if lo * (lo + 1) // 2 != nbaseline:
        raise ValueError("%i is not a triangular number of baselines" % nbaseline)
    return lo


def matrix_to_storage_header(ohdr):
    """Rewrites, in place, a copy of a matrix sequence header into the header
    of its storage form (also the header of correlate(..., output='storage'))."""
    otensor = ohdr['_tensor']
    nchan, nstand, npol = otensor['shape'][1:4]
    if npol != 2:
        raise ValueError("The storage form needs npol = 2, got %i" % npol)
    del ohdr['matrix_fill_mode']
    otensor['shape'] = [-1, nstand * (nstand + 1) // 2, nchan, 4]
    otensor['labels'] = list(STORAGE_AXES)
    if 'scales' in otensor:
        s = otensor['scales']
        otensor['scales'] = [s[0], None, s[1], None]
    if 'units' in otensor:
        u = otensor['units']
        otensor['units'] = [u[0], None, u[1], list(STOKES_UNITS)]
    return ohdr


class ConvertVisibilitiesBlock(TransformBlock):
    def __init__(self, iring, fmt, *args, **kwargs):
        super(ConvertVisibilitiesBlock, self).__init__(iring, *args, **kwargs)
        self.ofmt = fmt

    def define_valid_input_spaces(self):
        return ('cuda',)

    def on_sequence(self, iseq):
        ihdr = iseq.header
        itensor = ihdr['_tensor']
        labels = itensor['labels']
        if labels[0] != 'time':
            raise ValueError("Expected 'time' as the first axis, got %s" % labels)
        if itensor['dtype'] != 'cf32':
            raise ValueError("Expected cf32 visibilities, got %s" % itensor['dtype'])
        ohdr, otensor = H.derive(ihdr)
        if labels == MATRIX_AXES:
            nchan, nstand, npol, nstand_j, npol_j = itensor['shape'][1:]
            if nstand_j != nstand or npol_j != npol:
                raise ValueError("station_i / pol_i and station_j / pol_j differ: %s" % itensor['shape'])
            mode = ihdr.get('matrix_fill_mode')
            if mode not in ('lower', 'hermitian'):
                raise ValueError("matrix_fill_mode must be 'lower' or 'hermitian', got %r" % mode)
            self.ifmt = 'matrix'
            if self.ofmt == 'matrix':
                ohdr['matrix_fill_mode'] = 'hermitian'
            elif self.ofmt == 'storage':
                matrix_to_storage_header(ohdr)
            else:
                raise NotImplementedError("Unsupported conversion from matrix to %s" % self.ofmt)
        elif labels == STORAGE_AXES:
            nbaseline, nchan, nstokes = itensor['shape'][1:]
            if nstokes != 4:
                raise ValueError("The storage form needs 4 Stokes parameters, got %i" % nstokes)
            nstand = _nstand(nbaseline)
            self.ifmt = 'storage'
            if self.ofmt != 'matrix':
                raise NotImplementedError("Unsupported conversion from storage to %s" % self.ofmt)
            otensor['shape'] = [-1, nchan, nstand, 2, nstand, 2]
            otensor['labels'] = list(MATRIX_AXES)
            if 'scales' in otensor:
                s = otensor['scales']
                otensor['scales'] = [s[0], s[2], None, None, None, None]
            if 'units' in otensor:
                u = otensor['units']
                otensor['units'] = [u[0], u[2], None, list(POL_UNITS), None, list(POL_UNITS)]
            ohdr['matrix_fill_mode'] = 'hermitian'
        else:
            raise NotImplementedError("Cannot convert input from %s to %s" % (labels, self.ofmt))
        return ohdr

    def on_data(self, ispan, ospan):
        idata, odata = ispan.data, ospan.data
        if self.ifmt == 'matrix' and self.ofmt == 'matrix':
            # [..., nstand, npol, nstand, npol] -> [..., n, n]: same memory
            n = idata.shape[2] * idata.shape[3]
            visibilities.fill_hermitian(idata.reshape(idata.shape[:2] + (n, n)),
                                        odata.reshape(odata.shape[:2] + (n, n)))
        elif self.ifmt == 'matrix':
            visibilities.to_storage(idata, odata)
        else:
            visibilities.from_storage(idata, odata)


def convert_visibilities(iring, fmt, *args, **kwargs):
    """Convert visibility data to a new format: 'matrix' or 'storage'.

    Input ['time','freq','station_i','pol_i','station_j','pol_j'] cf32 (lower
    triangle or Hermitian), CUDA space:
      fmt='matrix'   the same tensor, fully (Hermitian) filled
      fmt='storage'  ['time','baseline','freq','stokes'] (UVFITS / FITS-IDI / MS order)
    Input ['time','baseline','freq','stokes'] cf32, CUDA space:
      fmt='matrix'   the six-axis tensor, fully filled
    """
    return ConvertVisibilitiesBlock(iring, fmt, *args, **kwargs)
