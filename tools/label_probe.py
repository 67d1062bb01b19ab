"""What the label filters cost (epp_label_filters_set / epp_pool_set_labels; include/epp_engine.h "Label filters").

    python tools/label_probe.py [--reps N] [--bench-log FILE] [--out FILE]

1. Synchronised epp_pool_set + epp_pool_set_labels at E = 4096 and 131 073, 8 labels per endpoint, on an engine with the
   config-3 profile and no label filter, and on one whose profile holds 4 label requirements (host clock around the two
   calls, which both end in a device synchronise; min / median / max over N repeats).
2. The config-3 step (R = 65536 device batch, E = 4096) without a label filter and with one that keeps half the pool
   (CUDA events around one synchronous call; median over N).
--bench-log: lines "<tag> <bench.py JSON line>" (bench.py config 3 run for the parent and this build, alternated in the
same session by the caller) are copied into the record.  Prints one JSON line (and writes it to --out)."""
from __future__ import annotations

import argparse
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


def labels_for(E):
    """8 labels per endpoint; `zone` splits the pool in half."""
    return [{"zone": "a" if e % 2 else "b", "rack": f"r{e % 64}", "model": "m", "tier": "gold",
             "app.kubernetes.io/name": "vllm", "lws/worker-index": str(e % 4), "hw": "h100", "pool": "p0"}
            for e in range(E)]


REQS = [("zone", 0, ["a"]), ("tier", 1, ["silver"]), ("hw", 2, []), ("deprecated", 3, [])]   # keeps zone = a


def pool_set_times(epp, E, with_filter, reps):
    from tools import tracegen as tg
    w = tg.baseline_configs()["config3"].scaled(E=E, R=64, T=512)
    spec = epp.ProfileSpec(0, [epp.ScorerSpec(*s) for s in w.primary_scorers], labels=REQS if with_filter else [])
    rng = np.random.default_rng(1)
    ids = np.arange(E, dtype=np.uint32)
    role, kv, waiting, running = np.zeros(E, np.uint8), rng.random(E), rng.integers(0, 50, E), rng.integers(0, 50, E)
    labels = labels_for(E)
    out = []
    with epp.Engine(E, spec) as eng:
        for _ in range(reps + 1):
            t0 = time.perf_counter()
            eng.pool_set(ids, role, kv, waiting, running)
            eng.pool_set_labels(ids, labels)
            out.append((time.perf_counter() - t0) * 1e3)
    out = sorted(out[1:])
    return {"min_ms": out[0], "median_ms": out[len(out) // 2], "max_ms": out[-1]}


def step_times(epp, half, reps):
    import torch
    from tools import tracegen as tg
    from tools import workload_setup as ws
    w = tg.baseline_configs()["config3"]
    trace = tg.Trace(w)
    eng = ws.make_engine(w)
    if half:
        eng.label_filters_set(0, [("zone", 0, ["a"])])
    ws.setup_engine(eng, w, trace)
    if half:
        eng.pool_set_labels(np.arange(w.E, dtype=np.uint32), [{"zone": "a" if e % 2 else "b"} for e in range(w.E)])
    tokens, _, _ = trace.requests()
    dt = torch.from_numpy(tokens.view(np.int32)).cuda()
    out = torch.empty((w.R, 32), dtype=torch.uint8, device="cuda")
    for _ in range(3):
        eng.schedule(dt, uniform_len=w.prompt_bytes, out=out, detail=False)
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        eng.schedule(dt, uniform_len=w.prompt_bytes, out=out, detail=False)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    dec = epp.decisions_from_torch(out)
    eng.close()
    ms.sort()
    return {"median_ms": ms[len(ms) // 2], "min_ms": ms[0], "max_ms": ms[-1],
            "odd_picks": int((dec["pick"][dec["status"] == 0] % 2 == 1).sum()), "decided": int((dec["status"] == 0).sum())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--bench-log", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import epp_b200 as epp
    name, power, clock = card()
    rec = {"gpu": name, "power_limit": power, "max_sm_clock": clock, "pool_set_plus_labels": {}, "config3_step": {}}
    for E in (4096, 131073):
        for f in (False, True):
            rec["pool_set_plus_labels"][f"E={E} {'4 requirements' if f else 'no label filter'}"] = pool_set_times(epp, E, f, a.reps)
    for half in (False, True):
        rec["config3_step"]["label filter keeping half" if half else "no label filter"] = step_times(epp, half, a.reps)
    if a.bench_log:
        runs = [ln.split(" ", 1) for ln in open(a.bench_log) if ln.strip()]
        rec["bench_config3_alternated"] = [{"build": t, "result": json.loads(j) if j.strip().startswith("{") else None}
                                           for t, j in (r + [""] if len(r) == 1 else r for r in runs)]
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
