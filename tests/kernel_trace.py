"""Which device kernels a call ran, read from torch.profiler's device activity
(it sees launches from libbifrost_b200.so too).  Shared by the edge suites
that assert the kernel path as well as the values."""
import time

import bifrost_b200 as bf

# Seconds of host time spent inside each profiler session before the work.
# Late in a long process the profiler can open its capture window after the
# first kernels of a session and drop their records as out of range; a wait
# at the start moves the work back inside the window.  It grows while
# sessions miss launches and is kept for the rest of the process.
_margin = [0.0]


def device_kernels(fn, reset=None, attempts=5):
    """Names of the device kernels that `fn` ran, in execution order.

    A session counts only if it recorded exactly as many kernels as the
    library launched (bf.launch_count()).  If a session misses some or all of
    the device activity, `reset` (if given) puts the operands back and `fn`
    runs again in a new session with a longer wait before the work, up to
    `attempts` times.  If no session records every launch the helper fails:
    a path check must never pass vacuously."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    seen = []
    for _ in range(attempts):
        if reset is not None:
            reset()
        torch.cuda.synchronize()
        before = bf.launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            time.sleep(_margin[0])
            fn()
            bf.device.stream_synchronize()
            torch.cuda.synchronize()
        launched = bf.launch_count() - before
        events = sorted((e.start_ns(), e.name()) for e in prof.profiler.kineto_results.events()
                        if e.device_type() == DeviceType.CUDA)
        names = [name for _, name in events if not name.startswith(('Memcpy', 'Memset'))]
        if names and len(names) == launched:
            return names
        seen.append((launched, len(names)))
        _margin[0] = min(4.0, max(0.05, 4 * _margin[0]))
    raise AssertionError("torch.profiler did not record every kernel launch "
                         "(launched, recorded per session: %s)" % seen)
