"""Parity tests share their workload set-up with bench.py / tools: the code lives in tools/workload_setup.py.  The
profiler helpers below prove which CUDA kernels a call launched."""
from tools.workload_setup import *  # noqa: F401,F403


def kernels_launched(fn, repeatable=True):
    """Runs fn() under torch.profiler with CUDA activities -> (fn's result, Counter of the names of the CUDA kernels it
    launched: launches per name).
    A torch kernel before fn's launches (add) and one behind them (mul) show that the trace kept its device records.  A
    trace that lost them is taken again with one more call of fn when the caller says the call is repeatable (its
    repetition changes nothing the test checks later and launches the same kernels), and the first call's result is
    returned.  Any other call (an index commit, say) is traced once: check trace_complete before concluding that a
    kernel did not run.
    The profiler drops device records now and then.  On an H100, about one session in 350 loses all of them.  One in 350
    loses a single record: the two bracket kernels are told apart, so that loss alone does not mark a trace with both
    of them as incomplete.  Another loses every record before the trailing bracket.  Total losses can come back to back,
    so each retake waits longer before its session (0.05 s, doubling up to 0.8 s)."""
    import time
    from collections import Counter

    import torch
    from torch.profiler import ProfilerActivity, profile
    out, names = None, Counter()
    for attempt in range(6 if repeatable else 1):
        if attempt:
            time.sleep(0.05 * (1 << (attempt - 1)))
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.ones(1, device="cuda").add_(1)
            r = fn()
            torch.cuda.synchronize()
            torch.ones(1, device="cuda").mul_(2)
            torch.cuda.synchronize()
        if attempt == 0:
            out = r
        events = prof.events()
        names = Counter(e.name for e in events)
        if trace_complete(names):
            break
    return out, names


def trace_complete(names):
    """The trace of kernels_launched kept the device records of the torch kernels before (add) and behind (mul) fn's
    launches."""
    before = any("at::native::" in n and "_add<" in n for n in names)
    behind = any("at::native::" in n and "MulFunctor" in n for n in names)
    return before and behind


def ran(names, kernel):
    return any(kernel in n for n in names)


def assert_ran(names, kernel, absent=(), where=""):
    assert ran(names, kernel), f"{where}: {kernel} did not run; kernels: {sorted(names)}"
    for k in absent:
        assert not ran(names, k), f"{where}: {k} ran; kernels: {sorted(names)}"
