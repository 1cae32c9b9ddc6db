"""bf.spectrometer: the fused GUPPI spectrometer gulp (extension).

One kernel for transpose -> fft(fine_time, fftshift) -> detect('stokes') ->
reduce(freq, f_avg) -> accumulate(nframe) (testbench/gpuspec_simple.py:44-55).
"""
from bifrost_b200.libbifrost import _bf, _check
from bifrost_b200.ndarray import asarray


def spectrometer(idata, odata, nfft=4096, f_avg=4, beta=0.0):
    """idata: ci8 [nframe, nchan, nfft, 2] (or [nchan, nfft, 2]) in CUDA space,
    odata: f32 [4, nchan*nfft/f_avg].  odata = beta*odata + sum over frames."""
    _check(_bf.bfSpectrometerFused(asarray(idata).as_BFarray(), asarray(odata).as_BFarray(),
                                   int(nfft), int(f_avg), float(beta)))
    return odata
