"""The measurement harness every script under tools/ times, counts and labels its numbers with, so that "GPU time",
"host synchronisations" and "launches" mean the same thing in every results file.

  card              the GPU's name, power limit and maximum SM clock, to store beside every number
  time_call         GPU time of a call on CUDA events, from an idle device (the host's issue time counts)
  time_queued       GPU time of a call on CUDA events, queued behind work already on the stream (it hides the launch)
  host_ms           host-clock time of a call that ends in a device synchronise
  capture           a CUDA graph of a call, captured after a warm-up on a side stream
  replay_ms         device time of one replay of a captured graph
  graph_us          capture + replay_ms in µs, or why the call cannot be captured
  peak_alloc        the peak allocation a call adds
  syncs             synchronising calls, counted under torch.cuda.set_sync_debug_mode('warn')
  profile           every CUDA activity of a call, by name, from a torch.profiler run
  launches          every CUDA activity of a call: kernels, memcpys and memsets
  kernel_launches   kernels alone
  summary           median / min / max / all of a list; ms_summary the same as median_ms / min_ms / max_ms

Imports only torch and the standard library.
"""
import statistics
import subprocess
import time
import warnings

import torch


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip().splitlines()[:1]}


def time_queued(fn):
    """(ms, result): CUDA events around one call of fn, recorded behind whatever the stream already holds."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def time_call(fn, reps=1, warmup=0):
    """(ms per call, last result): CUDA events around `reps` back-to-back calls of fn after `warmup` calls, started from
    an idle device so that the host's time to issue the work counts."""
    def run():
        for _ in range(reps - 1):
            fn()
        return fn()
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms, out = time_queued(run)
    return ms / reps, out


def host_ms(fn):
    """(ms, result): host clock around one call of fn and a device synchronise, started from an idle device."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def capture(fn):
    """fn captured into a CUDA graph.  Two calls on a side stream come first, so that lazy initialisation and the
    allocator's growth happen outside the capture."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    return graph


def replay_ms(graph, reps):
    """Device time (ms) of one replay: CUDA events around `reps` replays, after three untimed ones."""
    return time_call(graph.replay, reps=reps, warmup=3)[0]


def graph_us(fn, reps, per_graph=1):
    """Device time (µs) of one call of fn, replayed from a graph that holds `per_graph` calls; or, as a string, why fn
    cannot be captured (it reads the host or synchronises), so that a table of many calls records which ones."""
    try:
        graph = capture(lambda: [fn() for _ in range(per_graph)])
    except Exception as exc:                                            # noqa: BLE001
        torch.cuda.synchronize()
        return 'not capturable: ' + str(exc).split('\n')[0][:80]
    return replay_ms(graph, reps) * 1e3 / per_graph


def peak_alloc(fn):
    """(bytes, result): the peak allocation during one call of fn above what was allocated before it."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base, out


def syncs(fn):
    """Synchronising calls in one call of fn: the warnings torch raises under set_sync_debug_mode('warn').  Only torch's
    own text, 'called a synchronizing CUDA operation', counts; another warning that mentions synchronisation does not."""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as seen:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode('default')
    return sum('called a synchronizing' in str(w.message) for w in seen)


def profile(fn):
    """{name: (count, device ms)} of every CUDA activity of one call of fn -- kernels, memcpys and memsets -- from a
    torch.profiler run of its own."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.key: (e.count, e.device_time_total / 1e3) for e in prof.key_averages()
            if e.device_type.name == 'CUDA' and e.count}


def launches(fn):
    """Every CUDA activity of one call of fn: kernels, memcpys and memsets (the 'launches' of tools/results/*.json)."""
    return sum(c for c, _ in profile(fn).values())


def kernel_launches(fn):
    """Kernels of one call of fn, memcpys and memsets left out (the kernel launches of bench_box2mask_head.py and
    bench_discobox_half.py)."""
    return sum(c for name, (c, _) in profile(fn).items() if 'Memcpy' not in name and 'Memset' not in name)


def summary(xs):
    return {'median': statistics.median(xs), 'min': min(xs), 'max': max(xs), 'all': xs}


def ms_summary(xs):
    return {'median_ms': statistics.median(xs), 'min_ms': min(xs), 'max_ms': max(xs)}
