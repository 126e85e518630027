"""What the timing tools under tools/ share: the card line, the L2 flush, CUDA-event timing of steps, alternating arms round by round, and
the summaries they print.  bench.py keeps its own timing code; nothing here imports it."""
import statistics
import subprocess
import sys
import time

import torch


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def card():
    """The current CUDA device's name, power limit, current SM clock and max SM clock as one nvidia-smi line.  Without nvidia-smi: the
    device name and "power limit and clocks unknown".  Never raises, so a measurement always has a card line beside it."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30, check=True)
        return q.stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception:
        pass
    try:
        name = torch.cuda.get_device_name()
    except Exception:
        name = "no CUDA device"
    return name + ", power limit and clocks unknown"


class Flush:
    """256 MB, five times the H100's 50 MB L2: zeroing it before a timed step evicts what earlier steps left in the L2."""

    def __init__(self, device="cuda"):
        self.buf = torch.empty(256 << 20, dtype=torch.uint8, device=device)

    def flush(self):
        self.buf.zero_()


def time_events(fn, steps, warmup=0, flush=None):
    """Milliseconds of each of `steps` calls of fn() on the current stream, one CUDA-event pair per call, after `warmup` untimed calls and a
    synchronize.  With `flush` (a Flush), the L2 is flushed before every timed call, outside its event pair.  The events are read after
    one synchronize at the end, so the host may run ahead of the device across steps.  A CUDA graph is timed with fn = graph.replay."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for e0, e1 in evs:
        if flush is not None:
            flush.flush()
        e0.record()
        fn()
        e1.record()
    torch.cuda.synchronize()
    return [e0.elapsed_time(e1) for e0, e1 in evs]


def time_call(fn, flush=None):
    """(fn()'s result, CUDA-event ms, host ms up to a synchronize) of one call that starts on an idle device, after the L2 is flushed when
    `flush` is given: for calls long enough, or host-bound enough, that each is measured on its own."""
    if flush is not None:
        flush.flush()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    h0 = time.perf_counter()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1), (time.perf_counter() - h0) * 1e3


def alternate(arms, rounds, run, reverse=True):
    """{arm: [run(arm) of every round]}: each round runs every arm once, in the order given, or with `reverse` in reverse order on odd
    rounds, so that no arm always follows the same other arm."""
    out = {arm: [] for arm in arms}
    for r in range(rounds):
        for arm in (arms[::-1] if reverse and r % 2 else arms):
            out[arm].append(run(arm))
    return out


def stats(values):
    return dict(mean=sum(values) / len(values), min=min(values), max=max(values))


def median_spread(values):
    """The median and the spread (max - min): the summary of the tools that time a few long rounds."""
    return dict(median=float(statistics.median(values)), spread=float(max(values) - min(values)))
