"""What per-request endpoint subsets cost (epp_schedule_subset, csrc/subset_pick.cu).

    python tools/subset_probe.py [--window-ms W] [--reps N] [--out FILE]

Config 3 (E = 4096, R = 65536 device batch) with every request restricted to S = 1, 8, 64, 1024 slots (R = 8192 for
S = E: 2^25 slots per call) against the same batch without subsets.  Each request's slots are S distinct slots spread
over the pool ((r * 7919 + k * E / S) mod E).  Per S, alternating with the batch without subsets N times: the time of
one synchronous call (host clock around enough calls to fill a window of W ms, ending in a device synchronise: the
subset arrays are host memory, validated and copied by every call), and the subset kernel's CUDA-event time
(epp_stats.last_kernel_ms[6]) and the match kernels' (last_kernel_ms[3]) of single calls; min / median / max over the
repeats.
Then synchronous host batches of 1 / 16 / 256 requests -- what one batcher flush runs -- restricted to 8 slots each
against unrestricted ones (median host time of many calls; restricted batches take the chunked host path, unrestricted
ones the single-launch small-batch path).  Prints one JSON line (and writes it to --out)."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    return [x.strip() for x in q.split(",")]


def spread_subsets(R, E, S):
    """counts / offsets / slots of epp_subset: request r holds S distinct slots, ascending."""
    k = np.arange(S, dtype=np.int64)
    base = (np.arange(R, dtype=np.int64) * 7919)[:, None]
    slots = np.sort((base + k[None, :] * (E // S)) % E, axis=1).astype(np.uint32)
    return (np.full(R, S, np.uint32), np.arange(R, dtype=np.uint64) * np.uint64(S), np.ascontiguousarray(slots.reshape(-1)))


class Caller:
    """epp_schedule[_subset] on pre-packed arrays (no Python packing inside the timed window)."""

    def __init__(self, epp, eng, tokens, w, packed=None):
        self.epp, self.eng, self.keep = epp, eng, [tokens]
        self.b, self.R, self.dev, k = eng._batch(tokens, uniform_len=w.prompt_bytes)
        self.keep.append(k)
        if self.dev:
            import torch
            self.dec = torch.empty((self.R, 32), dtype=torch.uint8, device="cuda")
        else:
            self.dec = np.zeros(self.R, dtype=epp.DECISION_DTYPE)
        self.sub = None
        if packed is not None:
            self.keep.append(packed)
            self.sub = epp.capi.Subset()
            self.sub.struct_size = C.sizeof(epp.capi.Subset)
            self.sub.counts, self.sub.offsets, self.sub.slots = (a.ctypes.data for a in packed)
        self.lib = eng._lib
        self.ptr = self.dec.data_ptr() if self.dev else self.dec.ctypes.data

    def __call__(self):
        if self.sub is not None:
            rc = self.lib.epp_schedule_subset(self.eng._h, C.byref(self.b), C.byref(self.sub), self.ptr, None, 0, None)
        else:
            rc = self.lib.epp_schedule(self.eng._h, C.byref(self.b), self.ptr, None, 0)
        assert rc == 0, self.lib.epp_last_error()


def timed(fn, window_ms):
    """ms per call over a window of at least window_ms (and at least 5 calls)."""
    import torch
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    one = (time.perf_counter() - t0) * 1e3
    calls = max(5, int(window_ms / max(one, 1e-3)))
    t0 = time.perf_counter()
    for _ in range(calls):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / calls


def spread(xs):
    return {"min": float(np.min(xs)), "median": float(np.median(xs)), "max": float(np.max(xs)), "all": [float(x) for x in xs]}


def median_ms(fn, calls=200):
    for _ in range(20):
        fn()
    t = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-ms", type=float, default=300.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch

    import epp_b200 as epp
    from tools import tracegen as tg
    from tools import workload_setup as helpers
    if not torch.cuda.is_available():
        raise SystemExit("subset_probe needs a CUDA device")
    gpu, power, max_sm = card()
    w = tg.baseline_configs()["config3"]
    trace = tg.Trace(w)
    tokens, _, _ = trace.requests(0, w.R)
    dev_tokens = torch.from_numpy(tokens.view(np.int32)).cuda()
    eng = helpers.make_engine(w)
    helpers.setup_engine(eng, w, trace)
    out = {"what": "endpoint-subset cost per scheduling call (config 3, synchronous device batches)", "gpu": gpu,
           "power_limit": power, "max_sm_clock": max_sm, "window_ms": args.window_ms,
           "reps": args.reps, "E": w.E, "batches": []}
    for S in (1, 8, 64, 1024, w.E):
        R = w.R if S < w.E else 8192
        toks = dev_tokens[:R]
        plain = Caller(epp, eng, toks, w)
        restricted = Caller(epp, eng, toks, w, spread_subsets(R, w.E, S))
        acc = {label: {"call_ms": [], "match_pick_ms": [], "subset_kernel_ms": []} for label in ("without", "with")}
        for _ in range(args.reps):                          # alternate the two
            for label, fn in (("without", plain), ("with", restricted)):
                acc[label]["call_ms"].append(timed(fn, args.window_ms))
                for _ in range(5):
                    fn()
                    st = eng.stats()
                    acc[label]["match_pick_ms"].append(st["last_kernel_ms"][3])
                    acc[label]["subset_kernel_ms"].append(st["last_kernel_ms"][6])
        rows = {}
        for label, a in acc.items():
            rows[label] = {k: spread(v) for k, v in a.items()}
            rows[label]["decisions_per_s_median"] = R / rows[label]["call_ms"]["median"] * 1e3
        out["batches"].append({"S": S, "R": R, **rows})
    small = {}
    for n in (1, 16, 256):
        h = tokens[:n]
        plain = Caller(epp, eng, h, w)
        restricted = Caller(epp, eng, h, w, spread_subsets(n, w.E, 8))
        small[str(n)] = {"without_ms": spread([median_ms(plain) for _ in range(args.reps)]),
                         "with_ms": spread([median_ms(restricted) for _ in range(args.reps)])}
    out["host_flushes_S8"] = small
    eng.close()
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
