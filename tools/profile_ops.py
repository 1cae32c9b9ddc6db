"""One launch each of the fused spectrometer and the wgmma correlator for ncu
captures (not a benchmark: numbers under ncu are never reported)."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import bifrost_b200 as bf

rng = np.random.default_rng(5)
which = sys.argv[1] if len(sys.argv) > 1 else 'spectrometer,correlate'
if 'spectrometer' in which:
    nframe, nchan, nfft = 8, 4096, 4096
    raw = rng.integers(-127, 128, size=(nframe, nchan, nfft, 2, 2), dtype=np.int8)
    x = bf.asarray(raw.view(bf.DataType('ci8').as_numpy_dtype()).reshape(nframe, nchan, nfft, 2), space='cuda')
    o = bf.zeros((4, nchan * nfft // 4), 'f32', 'cuda')
    for _ in range(2):
        bf.spectrometer(x, o, nfft, 4, 0.0)
    bf.device.stream_synchronize()
    del x, o
if 'correlate' in which:
    ntime, nchan, n = 2048, 512, 512
    raw = rng.integers(-127, 128, size=(ntime, nchan, n, 2), dtype=np.int8)
    x = bf.asarray(raw.view(bf.DataType('ci8').as_numpy_dtype()).reshape(ntime, nchan, n), space='cuda')
    c = bf.zeros((nchan, n, n), 'cf32', 'cuda')
    la = bf.linalg.LinAlg()
    for _ in range(2):
        la.matmul(1, None, x.transpose(1, 0, 2), 0, c)
    bf.device.stream_synchronize()
if 'beamform' in which:
    # weights x voltages on the tensor cores (ab_tc_kernel): 64 beams, 512 inputs, 8192 samples, 64 channels
    import time
    nbeam, nin, ntime, nchan = 64, 512, 8192, 64
    CI8 = bf.DataType('ci8').as_numpy_dtype()
    w = bf.asarray(rng.integers(-127, 128, size=(nchan, nbeam, nin, 2), dtype=np.int8).view(CI8).reshape(nchan, nbeam, nin), space='cuda')
    v = bf.asarray(rng.integers(-127, 128, size=(nchan, nin, ntime, 2), dtype=np.int8).view(CI8).reshape(nchan, nin, ntime), space='cuda')
    c = bf.zeros((nchan, nbeam, ntime), 'cf32', 'cuda')
    la = bf.linalg.LinAlg()
    for _ in range(3):
        la.matmul(1, w, v, 0, c)
    bf.device.stream_synchronize()
    if 'time' in which:
        import json
        for env in ('', '1'):
            if env:
                os.environ['BFB_LINALG_SIMT'] = '1'
            la.matmul(1, w, v, 0, c)
            bf.device.stream_synchronize()
            t0 = time.perf_counter()
            for _ in range(10):
                la.matmul(1, w, v, 0, c)
            bf.device.stream_synchronize()
            ms = (time.perf_counter() - t0) * 100
            ops = 8.0 * nchan * nbeam * nin * ntime
            print(json.dumps(dict(op='a.b ci8 beamformer %dx%dx%d x%d chan' % (nbeam, nin, ntime, nchan),
                                  path='simt' if env else 'wgmma', ms=ms, TOPs=ops / ms / 1e9,
                                  out_GBps=nchan * nbeam * ntime * 8 / ms / 1e6)))
        os.environ.pop('BFB_LINALG_SIMT', None)
print('done')
