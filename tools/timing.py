"""The measurement code the benchmark scripts under tools/ share: the card read, CUDA-event timing of routes run
alternately after a warm-up, one summary of the times, per-kernel device time from torch.profiler, and the JSON line.

    from tools import timing      # after the script's repo-root sys.path insert

A time is only comparable to another taken the same way on the same card, so every script takes it here.
"""
import json
import os
import subprocess

import torch

CARD_FIELDS = ("name", "power_limit", "max_sm_clock")


def card(index=0):
    """Name, power limit and max SM clock of GPU `index` from one read-only nvidia-smi query; "unknown" each when the
    query fails."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(index)], capture_output=True, text=True, timeout=20)
        fields = [f.strip() for f in r.stdout.strip().rsplit(",", 2)]
        if r.returncode == 0 and len(fields) == 3:
            return dict(zip(CARD_FIELDS, fields))
    except (OSError, subprocess.SubprocessError):
        pass
    return dict.fromkeys(CARD_FIELDS, "unknown")


def summary(ms):
    """Median, p10, p90, min and max of the times `ms`, in ms.  The q-th percentile is sorted(ms)[min(n - 1, int(q n))],
    so the median is sorted(ms)[n // 2]."""
    t = sorted(ms)
    pct = lambda q: t[min(len(t) - 1, int(q * len(t)))]
    return {k: round(v, 4) for k, v in (("median_ms", pct(0.5)), ("p10_ms", pct(0.1)), ("p90_ms", pct(0.9)),
                                        ("min_ms", t[0]), ("max_ms", t[-1]))}


def timed(fn):
    """(ms, fn()): `fn` run alone on the idle device between two CUDA events, host work included."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1), out


def alternate(routes, steps, warmup, before=None):
    """Time the routes ({name: callable}, run in order) against each other: `warmup` untimed rounds, then `steps`
    rounds each timed with `timed`.  `before()`, if given, runs ahead of every route call, outside the events.
    Returns ({name: summary}, {name: the route's last return value}); a route's previous value is dropped before it
    runs again."""
    times = {name: [] for name in routes}
    last = {}
    for step in range(warmup + steps):
        for name, fn in routes.items():
            if before is not None:
                before()
            last.pop(name, None)
            ms, last[name] = timed(fn)
            if step >= warmup:
                times[name].append(ms)
    return {name: summary(t) for name, t in times.items()}, last


def kernel_times(fn, steps, groups=None):
    """Device time (ms per step) of each kernel and memset `fn` launches, from torch.profiler (CUDA activity) over
    `steps` calls after one warm call, slowest first, names cut at 100 characters.  `groups` ({group: name
    substrings}) also gives the sum over the kernels whose name contains one of a group's substrings.
    Returns (kernels, group sums)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        if e.self_device_time_total > 0:
            kernels[e.key[:100]] = kernels.get(e.key[:100], 0.0) + e.self_device_time_total / 1e3 / steps
    kernels = {k: round(v, 4) for k, v in sorted(kernels.items(), key=lambda kv: -kv[1])}
    sums = {g: round(sum(v for k, v in kernels.items() if any(n in k for n in names)), 4)
            for g, names in (groups or {}).items()}
    return kernels, sums


def emit(result, out=None):
    """Print `result` as one JSON line and, with `out`, write the line to that file.  The card is read again here,
    after the run, as "card_after", beside the read the script took before it as "card"."""
    result["card_after"] = card()
    line = json.dumps(result)
    print(line, flush=True)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            f.write(line + "\n")
