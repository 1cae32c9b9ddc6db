"""Where the time of bfFdmtExecute goes, pass by pass, on the int8 gulps of
BASELINE config 2 (4096 channels x (131072 + max_delay) samples):

    python tools/fdmt_passes.py [--md 794 204 1621] [--nrep 20] [--out FILE] ["KNOBS" ...]

For each max_delay (1621 runs at f0 1200 MHz / 300 MHz, as `tools/fdmt_time.py
--md 1621 --f0 1200 --bw 300`; the others at 1000 / 400) and each knob set
(space-separated NAME=VALUE, "" = defaults) it prints one JSON line with

  * `call_ms`: the whole call, CUDA events, median of --nrep;
  * `kernels`: the time of every FDMT kernel per call, from torch.profiler with
    CUDA activities, in a run of its own;
  * `model`: bytes per pass of the packed schedule, from bfFdmtPackedQuery --
    the pass output written (workspace rows, or the bank for the last pass),
    its unique bytes read by the next pass, the bytes staged into shared
    memory, and the compulsory bytes ntime * (nchan + 4 * max_delay);
  * `copy_ms`: a device-to-device copy that moves the compulsory bytes (half
    read, half written), timed in the same run as a practical ceiling;
  * the card's name and power limit, read in the same call.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import bifrost_b200 as bf  # noqa: E402
from bifrost_b200.fdmt import Fdmt  # noqa: E402
from bifrost_b200.libbifrost import _bf  # noqa: E402

SHAPES = {204: (1000., 400.), 794: (1000., 400.), 1621: (1200., 300.)}
NCHAN, NTIME = 4096, 131072


def _ip(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))


def packed_passes(nchan, md, f0, df):
    """Header fields and per-program tables of every pass of the packed schedule."""
    hdr = np.zeros(24, np.int32)
    if _bf.bfFdmtPackedQuery(nchan, md, f0, df, -2.0, -1, _ip(hdr), None, None, None) != 0:
        return []
    keys = ('s0 s1 nlev esize src_kind dst_kind T nprog nwarp slots src_slots data_bytes '
            'lookback nrow_out smem_bytes nops lv fused prefetch early').split()
    passes = []
    for k in range(int(hdr[0])):
        h = np.zeros(24, np.int32)
        assert _bf.bfFdmtPackedQuery(nchan, md, f0, df, -2.0, k, _ip(h), None, None, None) == 0
        p = dict(zip(keys, (int(v) for v in h)))
        ops = np.zeros((p['nprog'] * p['nlev'] * p['nwarp'] * p['slots'], 4), np.int32)
        src = np.zeros((p['nprog'], p['src_slots'], 4), np.int32)
        ph = np.zeros((p['nprog'], 4), np.int32)
        assert _bf.bfFdmtPackedQuery(nchan, md, f0, df, -2.0, k, _ip(h), _ip(ops), _ip(src), _ip(ph)) == 0
        p.update(src=src, hdr=ph)
        passes.append(p)
    return passes


def traffic_model(passes, nchan, md, ntime):
    """Bytes per pass for one gulp of `ntime` samples (the time ranges of
    packed_geometry in csrc/fdmt.cu: each pass starts early enough for the
    backward reach of the next one)."""
    n = len(passes)
    tb, nt = [0] * n, [0] * n
    nt[-1] = -(-ntime // passes[-1]['T'])
    te = nt[-1] * passes[-1]['T']
    for k in range(n - 2, -1, -1):
        tb[k] = -((passes[k + 1]['lookback'] - tb[k + 1] + 7) // 8 * 8)
        nt[k] = -(-(te - tb[k]) // passes[k]['T'])
        te = tb[k] + nt[k] * passes[k]['T']
    out = []
    for k, p in enumerate(passes):
        width = nt[k] * p['T']
        if p['dst_kind'] == 2:
            written = md * ntime * 4
        else:
            esz = 4 if p['dst_kind'] == 1 else p['esize']
            written = p['nrow_out'] * width * esz
        nsrc = p['hdr'][:, 1]
        staged_per_tile = 0
        for prog in range(p['nprog']):
            w = p['src'][prog, :nsrc[prog], 3].astype(np.int64)
            staged_per_tile += int(w.sum()) * (1 if p['src_kind'] == 0 else p['esize'])
        out.append(dict(steps='%d-%d' % (p['s0'], p['s1']), T=p['T'], nprog=p['nprog'], tiles=nt[k],
                        ws_written_MB=round((written if p['dst_kind'] != 2 else 0) / 1e6, 1),
                        ws_read_MB=round((written if k + 1 < n else 0) / 1e6, 1),
                        bank_MB=round((written if p['dst_kind'] == 2 else 0) / 1e6, 1),
                        staged_MB=round(staged_per_tile * nt[k] / 1e6, 1)))
    return out


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader',
                             '-i', str(torch.cuda.current_device())],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:          # the name alone still identifies the card
        pl = 'unavailable (%s)' % e
    return name, pl


def event_ms(fn, nrep, stream):
    times = []
    for _ in range(nrep):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(np.median(times)), float(min(times))


def kernel_times(fn, nrep):
    """Per-call CUDA time of every kernel fn launches (torch.profiler)."""
    from torch.profiler import profile, ProfilerActivity
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(nrep):
            fn()
        torch.cuda.synchronize()
    ks = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        d = ks.setdefault(ev.name, [0.0, 0])
        d[0] += ev.device_time_total if hasattr(ev, 'device_time_total') else ev.cuda_time_total
        d[1] += 1
    return {name: dict(ms_per_call=round(t / 1e3 / nrep, 4), launches_per_call=c / nrep)
            for name, (t, c) in sorted(ks.items(), key=lambda kv: -kv[1][0]) if 'fdmt' in name}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--md', type=int, nargs='+', default=[794, 204, 1621])
    ap.add_argument('--nrep', type=int, default=20)
    ap.add_argument('--out', default=None, help='also append the JSON lines to this file')
    ap.add_argument('knobs', nargs='*', default=[''])
    args = ap.parse_args()
    name, power = card()
    stream = torch.cuda.current_stream()
    bf.device.set_stream(stream.cuda_stream)
    rng = np.random.default_rng(1234)
    for md in args.md:
        f0, bw = SHAPES.get(md, (1000., 400.))
        ntime = NTIME + md
        x = np.clip(np.rint(rng.normal(0, 20, size=(NCHAN, ntime))), -127, 127).astype(np.int8)
        d_in = bf.asarray(x, space='cuda')
        d_out = bf.empty((md, ntime), 'f32', 'cuda')
        alg = ntime * (NCHAN + 4 * md)
        model = traffic_model(packed_passes(NCHAN, md, f0, bw / NCHAN), NCHAN, md, ntime)
        a = torch.empty(alg // 2, dtype=torch.uint8, device='cuda')
        b = torch.empty_like(a)
        for knob in args.knobs:
            env = dict(kv.split('=', 1) for kv in knob.split() if '=' in kv)
            old = {k: os.environ.get(k) for k in env}
            os.environ.update(env)
            try:
                plan = Fdmt()
                plan.init(NCHAN, md, f0, bw / NCHAN)
                run = lambda: plan.execute(d_in, d_out)  # noqa: E731
                for _ in range(3):
                    run()
                    b.copy_(a)
                torch.cuda.synchronize()
                # the call and the copy alternate so that both see the same clocks
                call, copy = [], []
                for _ in range(args.nrep):
                    call.append(event_ms(run, 1, stream)[0])
                    copy.append(event_ms(lambda: b.copy_(a), 1, stream)[0])
                ks = kernel_times(run, max(5, args.nrep // 2))
                line = dict(card=name, power_limit_max_sm_clock=power, md=md, f0=f0, bw=bw, knobs=knob,
                            call_ms=round(float(np.median(call)), 4), call_min_ms=round(min(call), 4),
                            copy_ms=round(float(np.median(copy)), 4),
                            compulsory_MB=round(alg / 1e6, 1),
                            compulsory_GBps=round(alg / float(np.median(call)) / 1e6, 1),
                            kernels=ks, model=model)
                del plan
            except Exception as e:      # a knob set that cannot be planned
                line = dict(md=md, knobs=knob, error=str(e))
            finally:
                for k, v in old.items():
                    if v is None:
                        os.environ.pop(k, None)
                    else:
                        os.environ[k] = v
            s = json.dumps(line)
            print(s, flush=True)
            if args.out:
                with open(args.out, 'a') as f:
                    f.write(s + '\n')


if __name__ == '__main__':
    main()
