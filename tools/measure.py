"""What the tools/time_*.py scripts share: the repository root on sys.path (import this module before the package), the
card a number was measured on, the H100 SXM data-sheet peaks, and the timing primitives.  Each script keeps its own
protocol (sizes, warm-up, repetitions, operand rotation, statistics); only the plumbing lives here.
"""
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12     # H100 SXM data sheet: HBM3 bandwidth
TF32_FLOP_PER_S = 495e12      # H100 SXM data sheet: dense TF32


def card(sm_clock=False, split=False):
    """nvidia-smi's line for the current device: name, power limit, (with ``sm_clock`` the SM clock now,) maximum SM
    clock.  With ``split``: the pair (name, power limit).  The runtime's device name when nvidia-smi cannot be read."""
    fields = "name,power.limit" + (",clocks.sm" if sm_clock else "") + ",clocks.max.sm"
    try:
        q = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30, check=True).stdout.strip().splitlines()
        line = q[torch.cuda.current_device()]
    except (OSError, subprocess.SubprocessError, IndexError):
        name = torch.cuda.get_device_name()
        return (name, "not readable") if split else name + " (power limit not readable)"
    return tuple(s.strip() for s in line.split(",")[:2]) if split else line


def timed(fn, reps=1, rotate=None):
    """One pair of CUDA events around ``reps`` back-to-back calls of ``fn``, a device synchronise before and after:
    (the last call's result, ms per call).  With ``rotate``, call i is ``fn(rotate[i % len(rotate)])``."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(reps):
        out = fn() if rotate is None else fn(rotate[i % len(rotate)])
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1) / reps


def per_call(fn, reps):
    """A pair of CUDA events around each of ``reps`` calls of ``fn``, one device synchronise after the last: (the last
    call's result, [ms of each call])."""
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for e0, e1 in ev:
        e0.record()
        out = fn()
        e1.record()
    torch.cuda.synchronize()
    return out, [e0.elapsed_time(e1) for e0, e1 in ev]


def host_ms(fn):
    """A host clock around ``fn()``, with a device synchronise before and after: (its result, ms)."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


class Probe:
    """Named windows around the stages of one larger call: ``cuda`` wraps a library binding in CUDA events (its kernels,
    in stream order), ``clock`` wraps a Python stage in ``host_ms``.  ``take`` synchronises and returns each name's
    total ms since the last ``take``."""

    def __init__(self):
        self.ev, self.host = {}, {}

    def cuda(self, name, fn):
        def wrapped(*a):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = fn(*a)
            e1.record()
            self.ev.setdefault(name, []).append((e0, e1))
            return rc
        return wrapped

    def clock(self, name, fn):
        def wrapped(*a, **k):
            out, ms = host_ms(lambda: fn(*a, **k))
            self.host[name] = self.host.get(name, 0.0) + ms
            return out
        return wrapped

    def take(self):
        torch.cuda.synchronize()
        out = {k: sum(a.elapsed_time(b) for a, b in v) for k, v in self.ev.items()}
        out.update(self.host)
        self.ev, self.host = {}, {}
        return out
