"""Per-op timings of the C-ABI entry points on BASELINE-sized inputs, next to
the reference's own CUDA kernels (oracle/_ref/libbifrost_ref.so, same device
buffers, same harness) where that library provides the op.

    python tools/bench_ops.py [--nframe 32] [--ops fdmt,transpose,fft,visibilities,beamform,correlate_storage,correlate_ci4,beamform_detect,pulse_search,sk_flag,coherent_dedisp,coherent_filterbank,fold,period_search,candidates,...]

Prints one JSON line per op: ms (median of runs, CUDA events on the launching
stream), algorithmic GB/s = in+out bytes at the C ABI / time (SURVEY 8d), and
the reference's time when available.  Not the headline benchmark (bench.py is).
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import torch  # noqa: E402
import bifrost_b200 as bf  # noqa: E402
from bifrost_b200.libbifrost import _bf, _check  # noqa: E402
import reflib  # noqa: E402


def timeit(fn, nrep=10, nwarm=3, stream=None):
    for _ in range(nwarm):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(nrep):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(np.median(times))


def cufft_ms(nbatch, nfft, stream, shift=False):
    """cuFFT (through torch.fft: bench tooling only, never on the product path)
    on the same number of transforms: cf32 -> cf32 c2c, the kernel the reference
    calls for this op (src/fft.cu:224-239).  The reference additionally converts
    ci8 -> cf32 in a load callback, so cuFFT's own traffic is 16 B/sample."""
    x = torch.randn(nbatch, nfft, dtype=torch.complex64, device='cuda')
    fn = (lambda: torch.fft.fftshift(torch.fft.fft(x, dim=1), dim=1)) if shift else (lambda: torch.fft.fft(x, dim=1))
    ms = timeit(fn, nrep=5, stream=stream)
    del x
    return ms


def report(name, ms, nbytes, ref_ms=None, **extra):
    line = dict(op=name, ms=round(ms, 4), alg_GBps=round(nbytes / ms / 1e6, 1))
    if ref_ms is not None:
        line['ref_ms'] = round(ref_ms, 4)
        line['speedup_vs_ref'] = round(ref_ms / ms, 2)
    line.update(extra)
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--nframe', type=int, default=32)
    ap.add_argument('--ops', default='config1,fdmt,transpose,fft,detect,reduce,accumulate,correlate')
    args = ap.parse_args()
    ops = args.ops.split(',')
    stream = torch.cuda.current_stream()
    bf.device.set_stream(stream.cuda_stream)
    ref = reflib.load()
    if ref is not None:
        h = ctypes.c_void_p(stream.cuda_stream)
        ref.bfStreamSet(ctypes.byref(h))
    rng = np.random.default_rng(1234)

    if 'config1' in ops:
        # BASELINE config 1: f32 [4096 frames, 256 chan]
        a = bf.asarray(rng.normal(size=(4096, 256)).astype(np.float32), space='cuda')
        t = bf.empty((256, 4096), 'f32', 'cuda')
        ms = timeit(lambda: bf.transpose(t, a, (1, 0)), stream=stream)
        rms = None
        if ref is not None:
            ax = (ctypes.c_int * 2)(1, 0)
            rms = timeit(lambda: ref.bfTranspose(a.as_BFarray(), t.as_BFarray(), ax), stream=stream)
        report('config1.transpose f32[4096,256]', ms, 2 * 4 * 4096 * 256, rms)
        r1 = bf.empty((4096, 64), 'f32', 'cuda')
        ms = timeit(lambda: bf.reduce(a, r1, 'sum'), stream=stream)
        rms = timeit(lambda: ref.bfReduce(a.as_BFarray(), r1.as_BFarray(), 0), stream=stream) if ref else None
        report('config1.reduce chan/4', ms, 4 * 4096 * 256 * 1.25, rms)
        r2 = bf.empty((512, 256), 'f32', 'cuda')
        ms = timeit(lambda: bf.reduce(a, r2, 'sum'), stream=stream)
        rms = timeit(lambda: ref.bfReduce(a.as_BFarray(), r2.as_BFarray(), 0), stream=stream) if ref else None
        report('config1.reduce time/8', ms, 4 * 4096 * 256 * 1.125, rms)

    if 'fdmt' in ops:
        import bench
        w = bench.workload(0)
        x = bench.make_input(w, 1)
        d_in = bf.asarray(x, space='cuda')
        d_out = bf.zeros((w['max_delay'], w['ntime']), 'f32', 'cuda')
        plan = bf.fdmt.Fdmt()
        plan.init(w['nchan'], w['max_delay'], w['f0'], w['df'])
        ms = timeit(lambda: plan.execute(d_in, d_out), stream=stream)
        rms = None
        if ref is not None:
            rp = ctypes.c_void_p()
            _check(ref.bfFdmtCreate(ctypes.byref(rp)))
            _check(ref.bfFdmtInit(rp, w['nchan'], w['max_delay'], w['f0'], w['df'], -2.0, 2, None, None))
            h = ctypes.c_void_p(stream.cuda_stream)
            ref.bfFdmtSetStream(rp, ctypes.byref(h))
            st = ref.bfFdmtExecute(rp, d_in.as_BFarray(), d_out.as_BFarray(), 0, None, None)
            if st == 0:
                rms = timeit(lambda: ref.bfFdmtExecute(rp, d_in.as_BFarray(), d_out.as_BFarray(), 0, None, None),
                             nrep=5, stream=stream)
            ref.bfFdmtDestroy(rp)
        report('fdmt 4096x%d i8 md=%d' % (w['ntime'], w['max_delay']), ms,
               w['ntime'] * (w['nchan'] + 4 * w['max_delay']), rms,
               Msamples_per_s=round(w['nchan'] * bench.NTIME_OUT / ms / 1e3, 1))
        del d_in, d_out, plan

    if 'fdmt_scaling' in ops:
        # SURVEY 8d: the same 4096-channel gulp at max_delay 204 / 1621
        import bench
        for md, f0, bw in ((204, 1000., 400.), (1621, 1200., 300.)):
            ntime = bench.NTIME_OUT + md
            x = rng.integers(-64, 64, size=(4096, ntime), dtype=np.int8)
            d_in = bf.asarray(x, space='cuda')
            d_out = bf.zeros((md, ntime), 'f32', 'cuda')
            plan = bf.fdmt.Fdmt()
            plan.init(4096, md, f0, bw / 4096)
            ms = timeit(lambda: plan.execute(d_in, d_out), stream=stream)
            report('fdmt 4096x%d i8 md=%d' % (ntime, md), ms, ntime * (4096 + 4 * md),
                   Msamples_per_s=round(4096 * bench.NTIME_OUT / ms / 1e3, 1))
            del d_in, d_out, plan

    # ---- GUPPI chain (config 3): ci8 [nframe, 4096 chan, 4096 fine_time, 2 pol]
    nframe, nchan, nfft, npol = args.nframe, 4096, 4096, 2
    I = nframe * nchan * nfft * npol * 2         # bytes of ci8 in the gulp
    chain = [o for o in ops if o in ('transpose', 'fft', 'detect', 'reduce', 'accumulate')]
    if chain:
        raw = rng.integers(-127, 128, size=(nframe, nchan, nfft, npol, 2), dtype=np.int8)
        x = raw.view(bf.DataType('ci8').as_numpy_dtype()).reshape(nframe, nchan, nfft, npol)
        d_x = bf.asarray(x, space='cuda')
        d_t = bf.empty((nframe, npol, nchan, nfft), 'ci8', 'cuda')
        ms = timeit(lambda: bf.transpose(d_t, d_x, (0, 3, 1, 2)), nrep=5, stream=stream)
        report('chain.transpose ci8 [t,f,ft,p]->[t,p,f,ft]', ms, 2 * I, Msamples_per_s=round(nframe * nchan * nfft / ms / 1e3, 1))
        del d_x
        d_f = bf.empty((nframe, npol, nchan, nfft), 'cf32', 'cuda')
        plan = bf.fft.Fft()
        plan.init(d_t, d_f, axes=[3], apply_fftshift=True)
        ms = timeit(lambda: plan.execute(d_t, d_f), nrep=5, stream=stream)
        del d_t
        cu = cufft_ms(nframe * npol * nchan, nfft, stream)
        report('chain.fft ci8->cf32 n=4096 fftshift', ms, 5 * I, Msamples_per_s=round(nframe * nchan * nfft / ms / 1e3, 1),
               cufft_c2c_cf32_ms=round(cu, 4), cufft_GBps=round(16 * nframe * npol * nchan * nfft / cu / 1e6, 1),
               speedup_vs_cufft=round(cu / ms, 2))
        d_d = bf.empty((nframe, 4, nchan, nfft), 'f32', 'cuda')
        ms = timeit(lambda: bf.detect(d_f, d_d, 'stokes', 1), nrep=5, stream=stream)
        report('chain.detect stokes', ms, 8 * I, Msamples_per_s=round(nframe * nchan * nfft / ms / 1e3, 1))
        del d_f
        d_dm = d_d.reshape(nframe, 4, nchan * nfft)
        d_r = bf.empty((nframe, 4, nchan * nfft // 4), 'f32', 'cuda')
        ms = timeit(lambda: bf.reduce(d_dm, d_r, 'sum'), nrep=5, stream=stream)
        rms = timeit(lambda: ref.bfReduce(d_dm.as_BFarray(), d_r.as_BFarray(), 0), nrep=5, stream=stream) if ref else None
        report('chain.reduce freq/4', ms, 5 * I, rms, Msamples_per_s=round(nframe * nchan * nfft / ms / 1e3, 1))
        del d_d, d_dm
        d_acc = bf.zeros((1, 4, nchan * nfft // 4), 'f32', 'cuda')
        one = d_r[0:1]
        ms = timeit(lambda: bf.accumulate(one, d_acc, 1.0), stream=stream)
        report('chain.accumulate one frame', ms, 3 * 4 * 4 * nchan * nfft // 4)
        del d_r, d_acc

    if 'fftsizes' in ops:
        # c2c forward FFTs of other lengths (ci8 -> cf32), 2^28 complex samples each
        for nfft_ in (256, 1024, 2048, 8192, 16384, 131072):
            nbatch = (1 << 27) // nfft_
            raw = rng.integers(-127, 128, size=(nbatch, nfft_, 2), dtype=np.int8)
            xi = raw.view(bf.DataType('ci8').as_numpy_dtype()).reshape(nbatch, nfft_)
            d_i = bf.asarray(xi, space='cuda')
            d_o = bf.empty((nbatch, nfft_), 'cf32', 'cuda')
            plan = bf.fft.Fft()
            plan.init(d_i, d_o, axes=[1], apply_fftshift=False)
            ms = timeit(lambda: plan.execute(d_i, d_o), nrep=5, stream=stream)
            del d_i, d_o, plan
            cu = cufft_ms(nbatch, nfft_, stream)
            report('fft ci8->cf32 n=%d batch=%d' % (nfft_, nbatch), ms, 10 * nbatch * nfft_,
                   Msamples_per_s=round(nbatch * nfft_ / ms / 1e3, 1),
                   cufft_c2c_cf32_ms=round(cu, 4), cufft_GBps=round(16 * nbatch * nfft_ / cu / 1e6, 1),
                   speedup_vs_cufft=round(cu / ms, 2))

    if 'correlate' in ops:
        nchan_c, nstand, npol_c = 512, 256, 2
        n = nstand * npol_c
        la = bf.linalg.LinAlg()
        for ntime in (512, 2048, 8192):
            raw = rng.integers(-127, 128, size=(ntime, nchan_c, n, 2), dtype=np.int8)
            x = raw.view(bf.DataType('ci8').as_numpy_dtype()).reshape(ntime, nchan_c, n)
            d_x = bf.asarray(x, space='cuda')
            xv = d_x.transpose(1, 0, 2)               # [chan, time, stand*pol] view
            d_c = bf.zeros((nchan_c, n, n), 'cf32', 'cuda')
            try:
                la.matmul(1, None, xv, 0, d_c)
            except RuntimeError as e:
                print(json.dumps(dict(op='correlate', error=str(e))))
                break
            ms = timeit(lambda: la.matmul(1, None, xv, 0, d_c), nrep=5, stream=stream)
            rms = None
            if ref is not None:
                rl = ctypes.c_void_p()
                _check(ref.bfLinAlgCreate(ctypes.byref(rl)))
                st = ref.bfLinAlgMatMul(rl, 1.0, None, xv.as_BFarray(), 0.0, d_c.as_BFarray())
                if st == 0:
                    rms = timeit(lambda: ref.bfLinAlgMatMul(rl, 1.0, None, xv.as_BFarray(), 0.0, d_c.as_BFarray()),
                                 nrep=3, stream=stream)
                ref.bfLinAlgDestroy(rl)
            flops = nchan_c * ntime * n * (n + 1) / 2 * 8
            report('correlate ci8 ntime=%d n=%d nchan=%d' % (ntime, n, nchan_c), ms,
                   2 * ntime * nchan_c * n + 8 * nchan_c * n * (n + 1) / 2, rms,
                   TFLOPs=round(flops / ms / 1e9, 1))
            del d_x, d_c

    if 'visibilities' in ops:
        # BASELINE config 4 correlator output, one frame: 512 chan x (256 stations x 2 pols)^2 cf32.
        # Compulsory bytes: the lower triangle read (or the storage tensor) plus the output
        # written.  copy_* is a device-to-device copy moving the same bytes (half read, half
        # written), timed in the same run: the practical ceiling for a streaming kernel.
        nchan_v, nstand = 512, 256
        n, nb = 2 * nstand, nstand * (nstand + 1) // 2
        low = 8 * nchan_v * n * (n + 1) // 2
        full, sto = 8 * nchan_v * n * n, 32 * nchan_v * nb
        c = rng.standard_normal(size=(nchan_v, n, n), dtype=np.float32).astype(np.complex64)
        d_m = bf.asarray(c, space='cuda')
        del c
        d_f = bf.empty((nchan_v, n, n), 'cf32', 'cuda')
        d_s = bf.empty((nb, nchan_v, 4), 'cf32', 'cuda')
        m6 = d_m.reshape(nchan_v, nstand, 2, nstand, 2)
        f6 = d_f.reshape(nchan_v, nstand, 2, nstand, 2)
        buf = torch.empty(full, dtype=torch.uint8, device='cuda')
        dst = torch.empty_like(buf)
        for name, fn, nbytes in (
                ('fill_hermitian', lambda: bf.visibilities.fill_hermitian(d_m, d_f), low + full),
                ('to_storage', lambda: bf.visibilities.to_storage(m6, d_s), low + sto),
                ('from_storage', lambda: bf.visibilities.from_storage(d_s, f6), sto + full)):
            ms = timeit(fn, nrep=20, stream=stream)
            half = nbytes // 2
            cms = timeit(lambda: dst[:half].copy_(buf[:half]), nrep=20, stream=stream)
            report('visibilities.%s nchan=%d nstand=%d' % (name, nchan_v, nstand), ms, nbytes,
                   copy_ms=round(cms, 4), copy_GBps=round(nbytes / cms / 1e6, 1),
                   of_copy=round(cms / ms, 3))
        del d_m, d_f, d_s, buf, dst

    if 'beamform' in ops:
        bench_beamform(stream, ref, rng)

    if 'correlate_storage' in ops:
        bench_correlate_storage(stream, rng)

    if 'correlate_ci4' in ops:
        bench_correlate_ci4(stream, rng)

    if 'beamform_detect' in ops:
        bench_beamform_detect(stream, rng)

    if 'pulse_search' in ops:
        bench_pulse_search(stream)

    if 'sk_flag' in ops:
        bench_sk_flag(stream)

    if 'sk_flag_kernels' in ops:
        bench_sk_flag_kernels()

    if 'coherent_dedisp' in ops:
        bench_coherent_dedisp(stream)

    if 'coherent_filterbank' in ops:
        bench_coherent_filterbank(stream)

    if 'fold' in ops:
        bench_fold(stream)

    if 'period_search' in ops:
        bench_period_search(stream)

    if 'candidates' in ops:
        bench_candidates(stream)


def gpu_name():
    """Card name, power limit and max SM clock, read in the same run as the timings."""
    import subprocess
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else None


def bench_correlate_storage(stream, rng, nrep=20):
    """bfLinAlgCorrelateToStorage against the two calls it replaces
    (bfLinAlgMatMul into a [chan, n, n] matrix, then bfVisibilitiesToStorage)
    on BASELINE config 4: 512 chan, 256 stations x 2 pols, ci8.  The two are
    timed alternately in the same loop, and their outputs compared bit for
    bit.  HBM share: compulsory bytes (voltages read + Stokes written for the
    fused call; + the lower triangle written and read back for the two calls)
    at 3.35 TB/s (H100 SXM data sheet, 700 W) over the time."""
    print(json.dumps({'op': 'correlate_storage.device', 'gpu': gpu_name()}), flush=True)
    nchan, nstand = 512, 256
    n, nb = 2 * nstand, nstand * (nstand + 1) // 2
    la = bf.linalg.LinAlg()
    d_c = bf.empty((nchan, n, n), 'cf32', 'cuda')
    c6 = d_c.reshape(nchan, nstand, 2, nstand, 2)
    d_f = bf.empty((nb, nchan, 4), 'cf32', 'cuda')
    d_s = bf.empty((nb, nchan, 4), 'cf32', 'cuda')
    fused = lambda: la.correlate_to_storage(xv, d_f)                                    # noqa: E731
    two = lambda: (la.matmul(1, None, xv, 0, d_c), bf.visibilities.to_storage(c6, d_s))   # noqa: E731
    for ntime in (512, 2048, 8192):
        raw = rng.integers(-128, 128, size=(ntime, nchan, n, 2), dtype=np.int8)
        d_x = bf.asarray(raw.view(bf.DataType('ci8').as_numpy_dtype()).reshape(ntime, nchan, n), space='cuda')
        del raw
        xv = d_x.transpose(1, 0, 2)                   # [chan, time, stand*pol] view of the ring frame
        for fn in (fused, two, fused, two):
            fn()
        torch.cuda.synchronize()
        times = {'fused': [], 'two': []}
        for _ in range(nrep):
            for key, fn in (('fused', fused), ('two', two)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                fn()
                e1.record(stream)
                torch.cuda.synchronize()
                times[key].append(e0.elapsed_time(e1))
        identical = bool(np.array_equal(np.asarray(d_f.copy('system')).view(np.uint64),
                                        np.asarray(d_s.copy('system')).view(np.uint64)))
        ms, two_ms = float(np.median(times['fused'])), float(np.median(times['two']))
        vin, vout, low = 2 * ntime * nchan * n, 32 * nchan * nb, 8 * nchan * n * (n + 1) // 2
        report('correlate_storage ci8 ntime=%d nstand=%d nchan=%d' % (ntime, nstand, nchan), ms, vin + vout,
               hbm_share=round((vin + vout) / 3.35e12 * 1e3 / ms, 3), two_call_ms=round(two_ms, 4),
               two_call_hbm_share=round((vin + 2 * low + vout) / 3.35e12 * 1e3 / two_ms, 3),
               speedup_vs_two_calls=round(two_ms / ms, 3), identical=identical)
        del d_x, xv


def bench_correlate_ci4(stream, rng, nrep=20):
    """The correlator on ci4 voltages, BASELINE config 4 (512 chan, 256
    stations x 2 pols) as the correlate block passes a ring frame: the ci4 call,
    bfUnpack to ci8 followed by the ci8 call (what a ci4 pipeline ran before),
    and the ci8 call alone, timed alternately in the same loop.  The ci4 and
    ci8 outputs are compared bit for bit.  bfUnpack reads the byte-reversed
    nibble order, so it unpacks a byte-reversed copy of the same samples."""
    print(json.dumps({'op': 'correlate_ci4.device', 'gpu': gpu_name()}), flush=True)
    nchan, n = 512, 512
    la = bf.linalg.LinAlg()
    d_c4 = bf.empty((nchan, n, n), 'cf32', 'cuda')
    d_c8 = bf.empty((nchan, n, n), 'cf32', 'cuda')
    ci4 = bf.DataType('ci4').as_numpy_dtype()
    for ntime in (512, 2048, 8192):
        x4 = rng.integers(0, 256, size=(ntime, nchan, n), dtype=np.uint8).view(ci4)
        d_x4 = bf.asarray(bf.ndarray(x4, dtype='ci4'), space='cuda')
        d_x4r = bf.asarray(bf.ndarray(x4, dtype='ci4').byteswap(), space='cuda')
        del x4
        d_x8 = bf.empty((ntime, nchan, n), 'ci8', 'cuda')
        x4v, x8v = d_x4.transpose(1, 0, 2), d_x8.transpose(1, 0, 2)
        fns = {'ci4': lambda: la.matmul(1, None, x4v, 0, d_c4),
               'unpack_ci8': lambda: (bf.unpack(d_x4r, d_x8), la.matmul(1, None, x8v, 0, d_c8)),
               'ci8': lambda: la.matmul(1, None, x8v, 0, d_c8)}
        for _ in range(2):
            for fn in fns.values():
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in fns}
        for _ in range(nrep):
            for key, fn in fns.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                fn()
                e1.record(stream)
                torch.cuda.synchronize()
                times[key].append(e0.elapsed_time(e1))
        identical = bool(np.array_equal(np.asarray(d_c4.copy('system')).view(np.uint64),
                                        np.asarray(d_c8.copy('system')).view(np.uint64)))
        ms = {k: float(np.median(v)) for k, v in times.items()}
        vin, vout = ntime * nchan * n, 8 * nchan * n * (n + 1) // 2
        report('correlate ci4 ntime=%d n=%d nchan=%d' % (ntime, n, nchan), ms['ci4'], vin + vout,
               unpack_ci8_ms=round(ms['unpack_ci8'], 4), ci8_ms=round(ms['ci8'], 4),
               speedup_vs_unpack_ci8=round(ms['unpack_ci8'] / ms['ci4'], 3),
               vs_ci8_alone=round(ms['ci8'] / ms['ci4'], 3), identical=identical)
        del d_x4, d_x4r, d_x8, x4v, x8v


def bench_beamform(stream, ref, rng):
    """The beamformer layout of bfLinAlgMatMul: 512 chan, K = 256 stations x 2
    pols, ntime 4096, cf32 weights, ci8 / ci4 voltages.  Times the sm_90a kernel,
    the generic kernel (BFB_LINALG_SIMT=1), the reference's kernel (nbeam <= 16,
    ci8: its CI8 @ CF32 path) and a device copy of the voltage bytes.  Bounds:
    compulsory bytes (voltages + weights + output) at 3.35 TB/s and 8 flops per
    complex multiply-add at 67 TFLOP/s (H100 SXM data sheet, 700 W)."""
    print(json.dumps({'op': 'beamform.device', 'gpu': gpu_name()}), flush=True)
    nchan, K, ntime = 512, 512, 4096
    for xk in ('ci8', 'ci4'):
        vb = 2 if xk == 'ci8' else 1
        raw = rng.integers(0, 256, size=(ntime, nchan, K * vb), dtype=np.uint8)
        xnp = raw.view(bf.DataType(xk).as_numpy_dtype()).reshape(ntime, nchan, K)
        d_x = bf.asarray(bf.ndarray(xnp, dtype=xk), space='cuda')
        del raw, xnp
        xv = d_x.transpose((1, 2, 0))
        buf = torch.empty(ntime * nchan * K * vb, dtype=torch.uint8, device='cuda')
        dst = torch.empty_like(buf)
        cms = timeit(lambda: dst.copy_(buf), nrep=20, stream=stream)
        del buf, dst
        for nbeam in (1, 4, 16, 64):
            if xk == 'ci4' and nbeam == 64:
                continue
            w = (rng.normal(size=(nchan, nbeam, K)) + 1j * rng.normal(size=(nchan, nbeam, K))).astype(np.complex64)
            d_w = bf.asarray(w, space='cuda')
            d_c = bf.zeros((nchan, nbeam, ntime), 'cf32', 'cuda')
            la = bf.linalg.LinAlg()
            ms = timeit(lambda: la.matmul(1, d_w, xv, 0, d_c), nrep=20, stream=stream)
            got = np.asarray(d_c.copy('system'))
            os.environ['BFB_LINALG_SIMT'] = '1'
            try:
                sms = timeit(lambda: la.matmul(1, d_w, xv, 0, d_c), nrep=3, nwarm=1, stream=stream)
                simt = np.asarray(d_c.copy('system'))
            finally:
                del os.environ['BFB_LINALG_SIMT']
            # sum_k |w_k| |x_k| <= 128 sqrt(2) sum_k |w_k|: each kernel is within 1e-6 of it
            tol = 2e-6 * 128 * np.sqrt(2) * np.abs(w).sum(-1)[..., None]
            agree = bool(np.all(np.abs(got - simt) <= tol))
            rms = None
            if ref is not None and nbeam <= 16 and xk == 'ci8':
                rl = ctypes.c_void_p()
                _check(ref.bfLinAlgCreate(ctypes.byref(rl)))
                st = ref.bfLinAlgMatMul(rl, 1.0, d_w.as_BFarray(), xv.as_BFarray(), 0.0, d_c.as_BFarray())
                if st == 0:
                    rms = timeit(lambda: ref.bfLinAlgMatMul(rl, 1.0, d_w.as_BFarray(), xv.as_BFarray(), 0.0,
                                                            d_c.as_BFarray()), nrep=3, nwarm=1, stream=stream)
                ref.bfLinAlgDestroy(rl)
            nbytes = ntime * nchan * K * vb + nchan * nbeam * K * 8 + nchan * nbeam * ntime * 8
            flops = 8.0 * nchan * nbeam * K * ntime
            t_hbm, t_fp = nbytes / 3.35e12 * 1e3, flops / 67e12 * 1e3
            report('beamform %s x cf32 nbeam=%d nchan=%d K=%d ntime=%d' % (xk, nbeam, nchan, K, ntime), ms, nbytes,
                   rms, TFLOPs=round(flops / ms / 1e9, 2), bound_by='HBM' if t_hbm >= t_fp else 'FP32',
                   share_of_bound=round(max(t_hbm, t_fp) / ms, 3), simt_ms=round(sms, 4),
                   speedup_vs_simt=round(sms / ms, 1), copy_ms=round(cms, 4), agrees_with_simt=agree,
                   max_abs_diff_vs_simt=float(np.abs(got - simt).max()))
            del d_w, d_c
        del d_x


def bench_beamform_detect(stream, rng, nrep=10):
    """Power beams, bfLinAlgBeamformDetect, against the three calls it
    replaces (bfLinAlgMatMul into cf32 beams, bfDetect, bfReduce over time)
    and the beamformer alone, timed alternately in the same loop: 512 chan,
    K = 512, ntime 4096, cf32 weights, ci8 / ci4 voltages, nb dual-pol beam
    rows, stokes and stokes_i, nint 16.  The fused and chain outputs are
    compared bit for bit.  Bounds as bench_beamform: compulsory bytes
    (voltages + weights + power beams) at 3.35 TB/s and 8 flops per complex
    multiply-add at 67 TFLOP/s (H100 SXM data sheet, 700 W)."""
    print(json.dumps({'op': 'beamform_detect.device', 'gpu': gpu_name()}), flush=True)
    nchan, K, ntime, nint = 512, 512, 4096, 16
    la = bf.linalg.LinAlg()
    for xk in ('ci8', 'ci4'):
        vb = 2 if xk == 'ci8' else 1
        raw = rng.integers(0, 256, size=(ntime, nchan, K * vb), dtype=np.uint8)
        xnp = raw.view(bf.DataType(xk).as_numpy_dtype()).reshape(ntime, nchan, K)
        d_x = bf.asarray(bf.ndarray(xnp, dtype=xk), space='cuda')
        del raw, xnp
        xv = d_x.transpose((1, 2, 0))
        for nb in (2, 8, 32, 64):
            w = (rng.normal(size=(nchan, nb, K)) + 1j * rng.normal(size=(nchan, nb, K))).astype(np.complex64)
            d_w = bf.asarray(w, space='cuda')
            d_c = bf.empty((nchan, nb, ntime), 'cf32', 'cuda')
            for mode in ('stokes', 'stokes_i'):
                nprod = 4 if mode == 'stokes' else 1
                d_d = bf.empty((nchan, nb // 2, nprod, ntime), 'f32', 'cuda')
                d_f = bf.empty((nchan, nb // 2, nprod, ntime // nint), 'f32', 'cuda')
                d_o = bf.empty((nchan, nb // 2, nprod, ntime // nint), 'f32', 'cuda')
                cv = d_c.reshape(nchan, nb // 2, 2, ntime)
                fns = {'fused': lambda: la.beamform_detect(d_w, xv, d_f, mode, nint),
                       'chain': lambda: (la.matmul(1, d_w, xv, 0, d_c), bf.detect(cv, d_d, mode, 2),
                                         bf.reduce(d_d, d_o, 'sum')),
                       'beamform': lambda: la.matmul(1, d_w, xv, 0, d_c)}
                for _ in range(2):
                    for fn in fns.values():
                        fn()
                torch.cuda.synchronize()
                times = {k: [] for k in fns}
                for _ in range(nrep):
                    for key, fn in fns.items():
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(stream)
                        fn()
                        e1.record(stream)
                        torch.cuda.synchronize()
                        times[key].append(e0.elapsed_time(e1))
                identical = bool(np.array_equal(np.asarray(d_f.copy('system')).view(np.uint32),
                                                np.asarray(d_o.copy('system')).view(np.uint32)))
                ms = {k: float(np.median(v)) for k, v in times.items()}
                nbytes = ntime * nchan * K * vb + nchan * nb * K * 8 + nchan * (nb // 2) * nprod * (ntime // nint) * 4
                flops = 8.0 * nchan * nb * K * ntime
                t_hbm, t_fp = nbytes / 3.35e12 * 1e3, flops / 67e12 * 1e3
                report('beamform_detect %s x cf32 %s nint=%d nb=%d nchan=%d K=%d ntime=%d'
                       % (xk, mode, nint, nb, nchan, K, ntime), ms['fused'], nbytes,
                       chain_ms=round(ms['chain'], 4), beamform_ms=round(ms['beamform'], 4),
                       speedup_vs_chain=round(ms['chain'] / ms['fused'], 3),
                       bound_by='HBM' if t_hbm >= t_fp else 'FP32', share_of_bound=round(max(t_hbm, t_fp) / ms['fused'], 3),
                       identical=identical)
                del d_d, d_f, d_o, cv
            del d_w, d_c
        del d_x, xv


def bench_pulse_search(stream, nrep=20):
    """bfPulseSearchExecute on the config-2 bank: the 794 x 131072 f32 output
    of the config-2 bfFdmtExecute (bench.make_input, made on the device),
    widths 1..256 in powers of two, decim 256.  Timed alternately in the same
    loop with a device-to-device copy of the bank and with the config-2
    bfFdmtExecute itself.  The search reads the bank once and writes a peak
    map nblk x 3 f32 per row; its HBM share is those bytes at 3.35 TB/s (H100
    SXM data sheet, 700 W) over the time.  Two runs are compared bit for bit."""
    import bench
    print(json.dumps({'op': 'pulse_search.device', 'gpu': gpu_name()}), flush=True)
    w = bench.workload(0)
    d_in = bf.asarray(bench.make_input(w, 1), space='cuda')
    md, ntime = w['max_delay'], w['ntime']
    bank = bf.zeros((md, ntime), 'f32', 'cuda')
    fplan = bf.fdmt.Fdmt()
    fplan.init(w['nchan'], md, w['f0'], w['df'])
    fplan.execute(d_in, bank)
    bview = bank[:, :bench.NTIME_OUT]                         # the 131072 fully-summed samples of each row
    widths, decim = [1 << k for k in range(9)], 256
    nblk = bf.pulse_search.output_nblock(bench.NTIME_OUT, widths, decim)
    plan = bf.pulse_search.PulseSearch()
    plan.init(widths, decim)
    d_a = bf.zeros((md, nblk, 3), 'f32', 'cuda')
    d_b = bf.zeros((md, nblk, 3), 'f32', 'cuda')
    nbytes_bank = md * bench.NTIME_OUT * 4
    src = torch.empty(nbytes_bank, dtype=torch.uint8, device='cuda')
    dst = torch.empty_like(src)
    fbank = bf.zeros((md, ntime), 'f32', 'cuda')
    fns = {'search': lambda: plan.execute(bview, d_a),
           'copy': lambda: dst.copy_(src),
           'fdmt': lambda: fplan.execute(d_in, fbank)}
    for _ in range(3):
        for fn in fns.values():
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(nrep):
        for key, fn in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            fn()
            e1.record(stream)
            torch.cuda.synchronize()
            times[key].append(e0.elapsed_time(e1))
    plan.execute(bview, d_b)
    torch.cuda.synchronize()
    a, b = np.asarray(d_a.copy('system')), np.asarray(d_b.copy('system'))
    ms = {k: float(np.median(v)) for k, v in times.items()}
    nbytes = nbytes_bank + md * nblk * 3 * 4
    top = np.argsort(a[..., 0].ravel())[::-1][:3]
    report('pulse_search f32 %dx%d widths=1..256 decim=%d' % (md, bench.NTIME_OUT, decim), ms['search'], nbytes,
           bank_GBps=round(nbytes_bank / ms['search'] / 1e6, 1),
           hbm_share=round(nbytes / 3.35e12 * 1e3 / ms['search'], 3),
           copy_ms=round(ms['copy'], 4), copy_GBps=round(2 * nbytes_bank / ms['copy'] / 1e6, 1),
           fdmt_ms=round(ms['fdmt'], 4), search_over_fdmt=round(ms['search'] / ms['fdmt'], 3),
           identical=bool(np.array_equal(a.view(np.uint32), b.view(np.uint32))),
           top_peaks=[[int(i // nblk), int(i % nblk) * decim + int(a.reshape(-1, 3)[i, 1]),
                       int(a.reshape(-1, 3)[i, 2]), round(float(a.reshape(-1, 3)[i, 0]), 2)] for i in top])
    del d_in, bank, fbank, d_a, d_b, src, dst


def sk_flag_input(nrow, ntime, dtype, window, bad=0.03, seed=0):
    """Gamma(4, 8) power drawn on the device (the sum of four exponentials),
    with a `bad` share of its windows given four samples of +150, which sk
    flags; returned as a bf device array of `dtype` ('u8' or 'f32')."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.zeros(nrow, ntime, device='cuda')
    for _ in range(4):
        x += torch.empty(nrow, ntime, device='cuda').exponential_(generator=g)
    x *= 8
    hit = torch.rand(nrow, ntime // window, 1, device='cuda', generator=g) < bad
    x.view(nrow, ntime // window, window)[..., 100:104] += 150 * hit
    x = torch.clamp(torch.round(x), 0, 255).to(torch.uint8) if dtype == 'u8' else x
    d = bf.empty((nrow, ntime), dtype, 'cuda')
    nbytes = x.numel() * x.element_size()
    _check(_bf.bfMemcpy(d.ctypes.data, _bf.BF_SPACE_CUDA, x.data_ptr(), _bf.BF_SPACE_CUDA, nbytes))
    bf.device.stream_synchronize()
    return d


SK_CASES = (('u8', 4096, 131072, 256, 4), ('f32', 4096, 32768, 256, 4))


def bench_sk_flag(stream, nrep=20):
    """bfSkFlagExecute on a u8 [4096, 131072] filterbank (the config-2 gulp),
    window 256, nacc 4, out of place and in place, and on f32 [4096, 32768],
    window 256, nacc 4.  Inputs are Gamma(4, 8) power with about 3 % of the windows
    corrupted (sk_flag_input).  Each case is timed alternately in one loop
    with a device-to-device copy of x.  Compulsory bytes: |x| + |y| out of
    place, |x| + the flagged windows in place; their HBM share is those bytes
    at 3.35 TB/s (H100 SXM data sheet, 700 W) over the time.  The in-place
    case restores x from a pristine copy before every run (that copy is not
    timed); two out-of-place runs are compared bit for bit."""
    print(json.dumps({'op': 'sk_flag.device', 'gpu': gpu_name()}), flush=True)
    for dt, nrow, ntime, M, N in SK_CASES:
        isz = 1 if dt == 'u8' else 4
        nbytes = nrow * ntime * isz
        d_x = sk_flag_input(nrow, ntime, dt, M)
        d_y = bf.empty((nrow, ntime), dt, 'cuda')
        d_w = bf.empty((nrow, ntime), dt, 'cuda')
        d_k = bf.empty((nrow, ntime // M), 'f32', 'cuda')
        plan = bf.sk_flag.SkFlag()
        plan.init(M, N)
        src = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
        dst = torch.empty_like(src)

        def restore():
            _check(_bf.bfMemcpy(d_w.ctypes.data, _bf.BF_SPACE_CUDA, d_x.ctypes.data, _bf.BF_SPACE_CUDA, nbytes))
        fns = {'out': (None, lambda: plan.execute(d_x, d_y)),
               'copy': (None, lambda: dst.copy_(src))}
        if dt == 'u8':
            fns['inplace'] = (restore, lambda: plan.execute(d_w, d_w))
        for _ in range(3):
            for pre, fn in fns.values():
                if pre:
                    pre()
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in fns}
        for _ in range(nrep):
            for key, (pre, fn) in fns.items():
                if pre:
                    pre()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                fn()
                e1.record(stream)
                torch.cuda.synchronize()
                times[key].append(e0.elapsed_time(e1))
        y1 = np.asarray(d_y.copy('system'))
        plan.execute(d_x, d_y, d_k)
        bf.device.stream_synchronize()
        y2, k = np.asarray(d_y.copy('system')), np.asarray(d_k.copy('system'))
        lo, hi = plan.lo, plan.hi
        flagged = float(np.mean(~((lo <= k) & (k <= hi))))
        ms = {key: float(np.median(v)) for key, v in times.items()}
        fields = dict(copy_ms=round(ms['copy'], 4), over_copy=round(ms['out'] / ms['copy'], 3),
                      hbm_share=round(2 * nbytes / 3.35e12 * 1e3 / ms['out'], 3),
                      flagged_share=round(flagged, 4), identical=bool(np.array_equal(y1, y2)))
        if 'inplace' in ms:
            inb = nbytes * (1 + flagged)
            fields.update(inplace_ms=round(ms['inplace'], 4),
                          inplace_hbm_share=round(inb / 3.35e12 * 1e3 / ms['inplace'], 3))
        report('sk_flag %s %dx%d window=%d nacc=%d' % (dt, nrow, ntime, M, N), ms['out'], 2 * nbytes, **fields)
        del d_x, d_y, d_w, d_k, src, dst


def bench_sk_flag_kernels(nrep=10):
    """Per-kernel device time of bfSkFlagExecute (out of place) on the
    bench_sk_flag cases, from torch.profiler in a run of its own."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    print(json.dumps({'op': 'sk_flag_kernels.device', 'gpu': gpu_name()}), flush=True)
    for dt, nrow, ntime, M, N in SK_CASES:
        d_x = sk_flag_input(nrow, ntime, dt, M)
        d_y = bf.empty((nrow, ntime), dt, 'cuda')
        plan = bf.sk_flag.SkFlag()
        plan.init(M, N)
        for _ in range(3):
            plan.execute(d_x, d_y)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(nrep):
                plan.execute(d_x, d_y)
            bf.device.stream_synchronize()
            torch.cuda.synchronize()
        per = {}
        for e in prof.profiler.kineto_results.events():
            if e.device_type() == DeviceType.CUDA and e.name().startswith('void bfb::sk_'):
                name = e.name().split('<')[0].replace('void bfb::', '')
                per.setdefault(name, []).append((e.end_ns() - e.start_ns()) / 1e6)
        print(json.dumps(dict(op='sk_flag.kernels %s %dx%d window=%d' % (dt, nrow, ntime, M),
                              **{k: round(float(np.median(v)), 4) for k, v in per.items()})), flush=True)
        del d_x, d_y


CD_CASES = ((100., 4096), (1000., 65536))            # (DM, nfft): one case on each kernel path


def bench_coherent_dedisp(stream, nrep=10):
    """bfCoherentDedispExecute on ci8 [64 chan, 2 pol, 2^20 + M] (0.67 s of a
    100 MHz band: f0 = 1300.78125 MHz, df = 1.5625 MHz) at DM 100 (M = 921,
    N = 4096, fused kernel) and DM 1000 (M = 9204, N = 65536, bfFft path).
    Timed alternately in one loop with: the same filter from today's public
    calls at the same N on pre-gathered cf32 segments (bfFft forward, bfMap
    times a precomputed cf32 chirp, bfFft inverse); cuFFT through torch.fft on
    the same segments (bench tooling only); a device-to-device copy of the
    output bytes.  Compulsory bytes per sample: 2 N / L (ci8 read N / L times)
    + 8 (cf32 written); their HBM share is those bytes at 3.35 TB/s (H100 SXM
    data sheet, 700 W) over the time.  FP32 work: 2 x 5 N log2 N / L flop per
    sample.  Every pair of outputs is compared on the kept samples: max |a - b|
    over max |b| per row."""
    from oracle import coherent_dedisp as ocd
    print(json.dumps({'op': 'coherent_dedisp.device', 'gpu': gpu_name()}), flush=True)
    nchan, npol, f0, df = 64, 2, 1300.78125, 1.5625
    for dm, n in CD_CASES:
        m = ocd.overlap(nchan, f0, df, dm)
        L = n - m
        ntime = (1 << 20) + m
        nseg = -(-ntime // L)
        rows = nchan * npol
        g = torch.Generator(device='cuda').manual_seed(1)
        raw = torch.randint(-127, 128, (nchan, npol, ntime, 2), dtype=torch.int8, device='cuda', generator=g)
        d_x = bf.empty((nchan, npol, ntime), 'ci8', 'cuda')
        _check(_bf.bfMemcpy(d_x.ctypes.data, _bf.BF_SPACE_CUDA, raw.data_ptr(), _bf.BF_SPACE_CUDA, raw.numel()))
        d_y = bf.empty((nchan, npol, ntime), 'cf32', 'cuda')
        plan = bf.coherent_dedisp.CoherentDedisp()
        plan.init(nchan, f0, df, dm, n)
        # cf32 segments [rows, nseg, N] (zeros past the end) and the chirp with 1/N folded in
        xc = torch.view_as_complex(raw.float()).reshape(rows, ntime)
        xp = torch.zeros(rows, (nseg - 1) * L + n, dtype=torch.complex64, device='cuda')
        xp[:, :ntime] = xc
        seg = xp.unfold(1, n, L).contiguous()
        del xp, xc
        h = np.stack([ocd.chirp(n, f0 + c * df, df, dm) / n for c in range(nchan)])
        h_t = torch.from_numpy(np.repeat(h, npol, axis=0).astype(np.complex64)).cuda()
        d_src = bf.empty((rows, nseg, n), 'cf32', 'cuda')
        _check(_bf.bfMemcpy(d_src.ctypes.data, _bf.BF_SPACE_CUDA, seg.data_ptr(), _bf.BF_SPACE_CUDA,
                            rows * nseg * n * 8))
        d_seg = bf.empty((rows, nseg, n), 'cf32', 'cuda')
        d_h = bf.empty((rows, n), 'cf32', 'cuda')
        _check(_bf.bfMemcpy(d_h.ctypes.data, _bf.BF_SPACE_CUDA, h_t.data_ptr(), _bf.BF_SPACE_CUDA, rows * n * 8))
        fft = bf.fft.Fft()
        fft.init(d_src, d_seg, axes=[2])

        def composed():
            fft.execute(d_src, d_seg, inverse=False)
            bf.map("y(r,s,k) = y(r,s,k) * h(r,k)", {'y': d_seg, 'h': d_h}, axis_names=('r', 's', 'k'),
                   shape=d_seg.shape)
            fft.execute(d_seg, d_seg, inverse=True)
        t_out = {}

        def torchfft():
            t_out['y'] = torch.fft.ifft(torch.fft.fft(seg, dim=2) * h_t[:, None, :], dim=2, norm='forward')
        nbytes_out = rows * ntime * 8
        src = torch.empty(nbytes_out, dtype=torch.uint8, device='cuda')
        dst = torch.empty_like(src)
        fns = {'new': lambda: plan.execute(d_x, d_y), 'composed': composed, 'torch': torchfft,
               'copy': lambda: dst.copy_(src)}
        for _ in range(2):
            for fn in fns.values():
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in fns}
        for _ in range(nrep):
            for key, fn in fns.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                fn()
                e1.record(stream)
                torch.cuda.synchronize()
                times[key].append(e0.elapsed_time(e1))
        # kept samples of every output, [rows, ntime]
        y_new = np.asarray(d_y.copy('system')).reshape(rows, ntime)
        plan.execute(d_x, d_y)
        bf.device.stream_synchronize()
        identical = bool(np.array_equal(y_new.view(np.uint64),
                                        np.asarray(d_y.copy('system')).reshape(rows, ntime).view(np.uint64)))
        y_cmp = np.asarray(d_seg.copy('system'))[:, :, :L].reshape(rows, nseg * L)[:, :ntime]
        y_tor = t_out['y'][:, :, :L].reshape(rows, nseg * L)[:, :ntime].cpu().numpy()

        def maxrel(a, b):
            return float(max(np.abs(a[r] - b[r]).max() / np.abs(b[r]).max() for r in range(rows)))
        ms = {key: float(np.median(v)) for key, v in times.items()}
        per_sample = 2.0 * n / L + 8
        nsamp = rows * ntime
        flop = 2 * 5 * n * np.log2(n) / L
        report('coherent_dedisp ci8 %dx%dx%d DM=%g N=%d M=%d' % (nchan, npol, ntime, dm, n, m), ms['new'],
               per_sample * nsamp,
               path='fused' if n <= 4096 else 'bfFft',
               realtime=round(ntime / (df * 1e6) / (ms['new'] * 1e-3), 1),
               hbm_share=round(per_sample * nsamp / 3.35e12 * 1e3 / ms['new'], 3),
               compulsory_GB=round(per_sample * nsamp / 1e9, 3),
               flop_per_sample=round(flop, 1), fp32_TFLOPs=round(flop * nsamp / ms['new'] / 1e9, 2),
               composed_ms=round(ms['composed'], 4), torch_fft_ms=round(ms['torch'], 4),
               copy_ms=round(ms['copy'], 4),
               err_new_vs_composed=maxrel(y_new, y_cmp), err_new_vs_torch=maxrel(y_new, y_tor),
               err_composed_vs_torch=maxrel(y_cmp, y_tor), identical=identical)
        del d_x, d_y, d_src, d_seg, d_h, seg, raw, h_t, src, dst, t_out, fft, plan
        torch.cuda.empty_cache()


def bench_coherent_filterbank(stream, nrep=10):
    """bfCoherentDedispFilterbank on ci8 [64 chan, 2 pol, ntime] with ntime =
    2^20 + M rounded up to a multiple of nfine (the bench_coherent_dedisp
    band), at DM 100 / N 4096 (fused kernel) and DM 1000 / N 65536 (bfFft
    path), nfine 1 and 16, stokes_i and stokes, nint 1.  Timed alternately in
    one loop with: the three calls it replaces (bfCoherentDedispExecute into
    cf32, bfDetect; no bfReduce at nint 1), bfCoherentDedispExecute alone, and
    a device-to-device copy of the output bytes.  Compulsory bytes: the ci8
    input read N / S times (S the segment step) plus the f32 output; their HBM
    share is those bytes at 3.35 TB/s (H100 SXM data sheet, 700 W) over the
    time.  At nfine 1 the fused and three-call outputs are compared bit for
    bit; two fused runs always are."""
    from oracle import coherent_dedisp as ocd
    print(json.dumps({'op': 'coherent_filterbank.device', 'gpu': gpu_name()}), flush=True)
    nchan, npol, f0, df, nint = 64, 2, 1300.78125, 1.5625, 1
    for dm, n in CD_CASES:
        m = ocd.overlap(nchan, f0, df, dm)
        for nfine in (1, 16):
            q = nfine * nint
            ntime = -(-((1 << 20) + m) // q) * q
            step = q * ((n - m) // q)
            g = torch.Generator(device='cuda').manual_seed(1)
            raw = torch.randint(-127, 128, (nchan, npol, ntime, 2), dtype=torch.int8, device='cuda', generator=g)
            d_x = bf.empty((nchan, npol, ntime), 'ci8', 'cuda')
            _check(_bf.bfMemcpy(d_x.ctypes.data, _bf.BF_SPACE_CUDA, raw.data_ptr(), _bf.BF_SPACE_CUDA, raw.numel()))
            del raw
            plan = bf.coherent_dedisp.CoherentDedisp()
            plan.init(nchan, f0, df, dm, n)
            d_y = bf.empty((nchan, npol, ntime), 'cf32', 'cuda')
            for mode in ('stokes_i', 'stokes'):
                shape = bf.coherent_dedisp.filterbank_shape(nchan, npol, ntime, nfine, mode, nint)
                d_o = bf.empty(shape, 'f32', 'cuda')
                d_d = bf.empty((nchan, shape[1], ntime), 'f32', 'cuda')
                nbytes_out = int(np.prod(shape)) * 4
                src = torch.empty(nbytes_out, dtype=torch.uint8, device='cuda')
                dst = torch.empty_like(src)
                fns = {'fused': lambda: plan.filterbank(d_x, d_o, nfine, mode, nint),
                       'chain': lambda: (plan.execute(d_x, d_y), bf.detect(d_y, d_d, mode, 1)),
                       'execute': lambda: plan.execute(d_x, d_y),
                       'copy': lambda: dst.copy_(src)}
                for _ in range(2):
                    for fn in fns.values():
                        fn()
                torch.cuda.synchronize()
                times = {k: [] for k in fns}
                for _ in range(nrep):
                    for key, fn in fns.items():
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(stream)
                        fn()
                        e1.record(stream)
                        torch.cuda.synchronize()
                        times[key].append(e0.elapsed_time(e1))
                a = np.asarray(d_o.copy('system'))
                plan.filterbank(d_x, d_o, nfine, mode, nint)
                bf.device.stream_synchronize()
                fields = dict(repeatable=bool(np.array_equal(a.view(np.uint32),
                                                             np.asarray(d_o.copy('system')).view(np.uint32))))
                if nfine == 1:
                    plan.execute(d_x, d_y)
                    bf.detect(d_y, d_d, mode, 1)
                    bf.device.stream_synchronize()
                    fields['identical_to_chain'] = bool(np.array_equal(
                        a.view(np.uint32), np.asarray(d_d.copy('system')).view(np.uint32)))
                ms = {key: float(np.median(v)) for key, v in times.items()}
                nbytes = nchan * npol * ntime * 2 * n / step + nbytes_out
                report('coherent_filterbank ci8 %dx%dx%d DM=%g N=%d M=%d nfine=%d %s nint=%d'
                       % (nchan, npol, ntime, dm, n, m, nfine, mode, nint), ms['fused'], nbytes,
                       path='fused' if n <= 4096 else 'bfFft',
                       realtime=round(ntime / (df * 1e6) / (ms['fused'] * 1e-3), 1),
                       hbm_share=round(nbytes / 3.35e12 * 1e3 / ms['fused'], 3), compulsory_GB=round(nbytes / 1e9, 3),
                       chain_ms=round(ms['chain'], 4), execute_ms=round(ms['execute'], 4),
                       copy_ms=round(ms['copy'], 4), speedup_vs_chain=round(ms['chain'] / ms['fused'], 3),
                       over_execute=round(ms['fused'] / ms['execute'], 3), **fields)
                del d_o, d_d, src, dst
            del d_x, d_y, plan
            torch.cuda.empty_cache()


FOLD_FP64_OPS = 11          # fp64 operations per sample in the phase and bin (DESIGN section 8)
FOLD_FP64_RATE = 16.7e12    # fp64 operations / s: 132 SMs x 64 FP64 lanes x 1.98 GHz (H100 SXM, 700 W)


def bench_fold(stream, nrep=10):
    """bfFoldExecute on three inputs: f32 [64, 4, 2^20] at nbin 1024, nu 641.9
    Hz, tsamp 0.64 us (Stokes from the coherent chain; channels 1300.78125 +
    1.5625 c MHz, top-edge delays at DM 100), and u8 [4096, 131072] at nbin
    256, tsamp 64 us (a config-2 filterbank, 1500 MHz down to 1200 MHz, DM
    100) with nu 1.4 Hz and 300 Hz.  Timed alternately in one loop with the
    same fold composed in torch (fp64 bins, then scatter_add_ of f32 into
    [rows, nbin]; bench tooling only) and a device-to-device copy of the
    input.  Bounds: the input bytes at 3.35 TB/s, and FOLD_FP64_OPS fp64
    operations per sample at FOLD_FP64_RATE (H100 SXM data sheet, 700 W).
    Counts are compared exactly with the torch composition, sums to 1e-5 of
    the bin's magnitude, and two runs bit for bit."""
    print(json.dumps({'op': 'fold.device', 'gpu': gpu_name()}), flush=True)
    cases = [('f32', (64, 4, 1 << 20), 1024, 0.64e-6, 641.9, 1300.78125, 1.5625, True),
             ('u8', (4096, 131072), 256, 64e-6, 1.4, 1500.0, -300.0 / 4096, False),
             ('u8', (4096, 131072), 256, 64e-6, 300.0, 1500.0, -300.0 / 4096, False)]
    for dt, shape, nbin, tsamp, nu, f0, df, coherent in cases:
        nchan, ntime = shape[0], shape[-1]
        rows = int(np.prod(shape[:-1]))
        freqs = f0 + df * np.arange(nchan) + (0.5 * abs(df) if coherent else 0.0)
        delays = bf.fold.dispersion_delays(freqs, 100.0, freqs.max())
        g = torch.Generator(device='cuda').manual_seed(2)
        if dt == 'u8':
            xt = torch.randint(0, 256, shape, dtype=torch.uint8, device='cuda', generator=g)
        else:
            xt = torch.rand(shape, dtype=torch.float32, device='cuda', generator=g) * 100
        d_x = bf.empty(shape, dt, 'cuda')
        nbytes = xt.numel() * xt.element_size()
        _check(_bf.bfMemcpy(d_x.ctypes.data, _bf.BF_SPACE_CUDA, xt.data_ptr(), _bf.BF_SPACE_CUDA, nbytes))
        plan = bf.fold.Fold()
        plan.init(nbin, delays, tsamp, 0.0, nu)
        d_o = bf.empty(shape[:-1] + (nbin,), 'f32', 'cuda')
        d_n = bf.empty((nchan, nbin), 'i32', 'cuda')
        a_t = torch.from_numpy(0.0 - delays).cuda()
        t_out = {}

        def torch_fold():
            t = torch.arange(ntime, dtype=torch.int64, device='cuda').double()
            tau = a_t[:, None] + t[None, :] * tsamp
            phi = tau * nu
            frac = phi - torch.floor(phi)
            b = torch.clamp(torch.floor(frac * nbin).long(), max=nbin - 1)          # [nchan, ntime]
            idx = b.reshape((nchan,) + (1,) * (len(shape) - 2) + (ntime,)).expand(shape).reshape(rows, ntime)
            out = torch.zeros(rows, nbin, dtype=torch.float32, device='cuda')
            out.scatter_add_(1, idx, xt.reshape(rows, ntime).float())
            cnt = torch.zeros(nchan, nbin, dtype=torch.int64, device='cuda')
            cnt.scatter_add_(1, b, torch.ones_like(b))
            t_out['out'], t_out['cnt'] = out, cnt
        dst = torch.empty_like(xt)
        fns = {'new': lambda: plan.execute(d_x, d_o, d_n), 'torch': torch_fold, 'copy': lambda: dst.copy_(xt)}
        for _ in range(3):
            for fn in fns.values():
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in fns}
        for _ in range(nrep):
            for key, fn in fns.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                fn()
                e1.record(stream)
                torch.cuda.synchronize()
                times[key].append(e0.elapsed_time(e1))
        ms = {key: float(np.median(v)) for key, v in times.items()}
        o1 = np.asarray(d_o.copy('system')).reshape(rows, nbin)
        n1 = np.asarray(d_n.copy('system'))
        plan.execute(d_x, d_o, d_n)
        bf.device.stream_synchronize()
        identical = bool(np.array_equal(o1.view(np.uint32), np.asarray(d_o.copy('system')).reshape(rows, nbin)
                                        .view(np.uint32)))
        to = t_out['out'].cpu().numpy()
        counts_match = bool(np.array_equal(n1, t_out['cnt'].cpu().numpy()))
        rel = float(np.max(np.abs(o1.astype(np.float64) - to) / np.maximum(np.abs(to), 1e-30)))
        nsamp = rows * ntime
        hbm_ms = nbytes / 3.35e12 * 1e3
        fp64_ms = nsamp * FOLD_FP64_OPS / FOLD_FP64_RATE * 1e3
        report('fold %s %s nbin=%d nu=%g tsamp=%g' % (dt, 'x'.join(map(str, shape)), nbin, nu, tsamp), ms['new'],
               nbytes, samples_per_bin_turn=round(1.0 / (nu * tsamp) / nbin, 3),
               hbm_bound_ms=round(hbm_ms, 4), fp64_bound_ms=round(fp64_ms, 4),
               bound='fp64' if fp64_ms > hbm_ms else 'HBM',
               share_of_bound=round(max(hbm_ms, fp64_ms) / ms['new'], 3),
               torch_ms=round(ms['torch'], 4), copy_ms=round(ms['copy'], 4),
               speedup_vs_torch=round(ms['torch'] / ms['new'], 2),
               counts_match_torch=counts_match, max_rel_vs_torch=rel, identical=identical)
        del d_x, d_o, d_n, xt, dst, t_out, plan
        torch.cuda.empty_cache()


def bench_period_search(stream, nrep=20):
    """bfPeriodSearchExecute on the config-2 bank shape: 794 x 131072 f32 of
    seeded noise with a periodic pulse train in a few rows, through a bfFft r2c
    to [794, 65537] cf32, then nharm 32, window 1024, decim 64.  The bfFft, the
    search and a torch composition of the same definition (torch.fft.rfft, a
    lower median over unfolded windows, fp64 gather sums, block maxima) are
    timed alternately in one loop; a torch.profiler run of its own splits the
    search by kernel.  Shape bound: the cf32 spectrum read, p written and read
    once, and the peak map written, at 3.35 TB/s (H100 SXM data sheet, 700 W).
    Two runs are compared bit for bit.  The torch composition transforms
    with cuFFT, whose spectrum differs from bfFft's in the last bits, so its
    output is timed but not compared."""
    from torch.profiler import ProfilerActivity, profile
    print(json.dumps({'op': 'period_search.device', 'gpu': gpu_name()}), flush=True)
    nrow, ntime, nharm, window, decim = 794, 131072, 32, 1024, 64
    nbin = ntime // 2 + 1
    nlevel = nharm.bit_length()
    nblk = bf.period_search.output_nblock(nbin, decim)
    gen = torch.Generator(device='cuda').manual_seed(1234)
    xt = torch.randn(nrow, ntime, generator=gen, device='cuda', dtype=torch.float32)
    period = 517.3                                              # samples: fundamental at 253.4 bins
    pulses = torch.arange(0, ntime - 1, period, device='cuda').round().long()
    for r in (100, 400, 700):
        xt[r, pulses] += 3.0
    x = bf.asarray(xt)
    spec = bf.empty((nrow, nbin), 'cf32', 'cuda')
    fft = bf.fft.Fft()
    fft.init(x, spec, axes=1)
    plan = bf.period_search.PeriodSearch()
    plan.init(nharm, window, decim)
    d_a = bf.zeros((nrow, nlevel, nblk, 2), 'f32', 'cuda')
    d_b = bf.zeros((nrow, nlevel, nblk, 2), 'f32', 'cuda')

    ln2 = 0.6931471805599453
    kk = torch.arange(nbin, device='cuda', dtype=torch.int64)
    gathers = [[(2 * i * kk + (1 << l)) // (2 << l) for i in range(1, 1 << l, 2)] for l in range(1, nlevel)]

    def torch_search():
        X = torch.fft.rfft(xt, dim=1)
        P = X.real.double() ** 2 + X.imag.double() ** 2
        full = (nbin // window) * window
        med = torch.median(P[:, :full].unfold(1, window, window), dim=2).values
        med = med.repeat_interleave(window, dim=1)
        if full < nbin:
            med = torch.cat([med, torch.median(P[:, full:], dim=1, keepdim=True).values.expand(-1, nbin - full)], 1)
        p = torch.where(med > 0, ((P / med) * ln2).float(), torch.zeros((), device='cuda'))
        p[:, 0] = 0
        p64 = p.double()
        S = [p64]
        for idx in gathers:
            t = torch.zeros_like(p64)
            for g in idx:
                t = t + p64[:, g]
            S.append(S[-1] + t)
        pad = nblk * decim - nbin
        out = torch.empty(nrow, nlevel, nblk, 2, device='cuda')
        for l, s in enumerate(S):
            sp = torch.nn.functional.pad(s, (0, pad), value=-float('inf')).view(nrow, nblk, decim)
            v, i = sp.max(dim=2)
            out[:, l, :, 0] = v.float()
            out[:, l, :, 1] = i.float()
        return out

    fns = {'fft': lambda: fft.execute(x, spec),
           'search': lambda: plan.execute(spec, d_a),
           'torch': torch_search}
    for _ in range(3):
        for fn in fns.values():
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(nrep):
        for key, fn in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            fn()
            e1.record(stream)
            torch.cuda.synchronize()
            times[key].append(e0.elapsed_time(e1))
    plan.execute(spec, d_b)
    torch.cuda.synchronize()
    a, b = np.asarray(d_a.copy('system')), np.asarray(d_b.copy('system'))
    ms = {k: float(np.median(v)) for k, v in times.items()}

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(nrep):
            plan.execute(spec, d_a)
        torch.cuda.synchronize()
    per_kernel = {}
    for e in prof.key_averages():
        if 'period_search' in e.key:
            per_kernel[e.key.split('(')[0].split('<')[0].split()[-1]] = round(
                e.device_time_total / max(e.count, 1) / 1e3, 4)

    nbytes = nrow * nbin * 8 + 2 * nrow * nbin * 4 + nrow * nlevel * nblk * 2 * 4
    sig = np.stack([bf.period_search.significance(a[:, l, :, 0], 1 << l) for l in range(nlevel)], axis=1)
    r, l, j = np.unravel_index(int(np.argmax(sig)), sig.shape)
    report('period_search cf32 %dx%d nharm=%d window=%d decim=%d' % (nrow, nbin, nharm, window, decim),
           ms['search'], nbytes, bound_ms=round(nbytes / 3.35e12 * 1e3, 4),
           hbm_share=round(nbytes / 3.35e12 * 1e3 / ms['search'], 3), kernels_ms=per_kernel,
           fft_ms=round(ms['fft'], 4), torch_ms=round(ms['torch'], 4),
           torch_over_search=round(ms['torch'] / ms['search'], 2),
           identical=bool(np.array_equal(a.view(np.uint32), b.view(np.uint32))),
           best=dict(row=int(r), nharm=1 << int(l), k=int(j) * decim + int(a[r, l, j, 1]),
                     fundamental=round((int(j) * decim + int(a[r, l, j, 1])) / (1 << int(l)), 2),
                     expected=round(ntime / period, 2), sigma=round(float(sig[r, l, j]), 2)))
    del xt, x, spec, d_a, d_b



def bench_candidates(stream, nrep=20):
    """bfCandidatesExecute (trial_radius 8, pos_radius 256: the widest boxcar)
    on the peak maps of the config-2 bank: the 794 x 131072 f32 output of the
    config-2 bfFdmtExecute (bench.make_input, made on the device) through
    bfPulseSearchExecute (widths 1..256 in powers of two) at decim 256 and 16,
    at thresholds 6 and 5, plus one dense case (every cell a member, one
    cluster).  The bound is the map's bytes at 3.35 TB/s (H100 SXM data sheet,
    700 W).  The alternative it replaces, a device-to-host copy of the map and
    oracle/candidates.py on the host, is timed once per case on the wall
    clock and must give the same table.  Two runs are compared bit for bit."""
    import time
    import bench
    from torch.profiler import ProfilerActivity, profile
    from oracle import candidates as oc
    print(json.dumps({'op': 'candidates.device', 'gpu': gpu_name()}), flush=True)
    w = bench.workload(0)
    d_in = bf.asarray(bench.make_input(w, 1), space='cuda')
    md, ntime = w['max_delay'], w['ntime']
    bank = bf.zeros((md, ntime), 'f32', 'cuda')
    fplan = bf.fdmt.Fdmt()
    fplan.init(w['nchan'], md, w['f0'], w['df'])
    fplan.execute(d_in, bank)
    bview = bank[:, :bench.NTIME_OUT]
    widths, ncap = [1 << k for k in range(9)], 4096
    for decim in (256, 16):
        nblk = bf.pulse_search.output_nblock(bench.NTIME_OUT, widths, decim)
        d_map = bf.zeros((md, nblk, 3), 'f32', 'cuda')
        ps = bf.pulse_search.PulseSearch()
        ps.init(widths, decim)
        ps.execute(bview, d_map)
        nbytes = md * nblk * 3 * 4
        cases = [(6., False), (5., False)] + ([(-1e30, True)] if decim == 256 else [])
        for threshold, dense in cases:
            plan = bf.candidates.Candidates()
            plan.init(threshold, 8, 256, decim)
            tabs = [bf.zeros((ncap, 9), 'f64', 'cuda') for _ in range(2)]
            cnts = [bf.zeros((1,), 'i32', 'cuda') for _ in range(2)]
            ms = timeit(lambda: plan.execute(d_map, tabs[0], cnts[0]), nrep=nrep, stream=stream)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(nrep):
                    plan.execute(d_map, tabs[0], cnts[0])
                torch.cuda.synchronize()
            per_kernel = {e.key.split('(')[0].split()[-1].replace('bfb::', ''):
                          round(e.device_time_total / max(e.count, 1) / 1e3, 4)
                          for e in prof.key_averages() if 'candidates_' in e.key}
            plan.execute(d_map, tabs[1], cnts[1])
            torch.cuda.synchronize()
            a, b = (np.asarray(x.copy('system')) for x in tabs)
            count = int(np.asarray(cnts[0].copy('system'))[0])
            t0 = time.perf_counter()
            host = np.asarray(d_map.copy('system'))
            t1 = time.perf_counter()
            want = oc.cluster(host, threshold, 8, 256, decim)
            t2 = time.perf_counter()
            n = min(count, ncap)
            report('candidates %dx%d decim=%d threshold=%s' % (md, nblk, decim, 'all' if dense else threshold),
                   ms, nbytes, map_MB=round(nbytes / 1e6, 2), bound_ms=round(nbytes / 3.35e12 * 1e3, 4),
                   share_of_bound=round(nbytes / 3.35e12 * 1e3 / ms, 3), kernels_ms=per_kernel,
                   members=int(np.count_nonzero((host[..., 0].astype(np.float64) >= threshold))),
                   clusters=count, host_copy_ms=round((t1 - t0) * 1e3, 2),
                   host_cluster_ms=round((t2 - t1) * 1e3, 1),
                   host_total_over_op=round((t2 - t0) * 1e3 / ms, 1),
                   matches_host=bool(len(want) == count and np.array_equal(a[:n].view(np.uint64),
                                                                           want[:n].view(np.uint64))),
                   identical=bool(np.array_equal(a.view(np.uint64), b.view(np.uint64))),
                   brightest=[[int(r[1]), int(r[2]), int(r[3]), round(float(r[0]), 2)]
                              for r in a[:n][np.argsort(a[:n, 0])[::-1][:3]]])
            del tabs, cnts
        del d_map
    del d_in, bank


if __name__ == '__main__':
    main()
