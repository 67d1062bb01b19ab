"""What the inflight-load producer costs per scheduling call.

    python tools/inflight_probe.py [--steps K] [--reps N] [--out FILE]

Config 3 with a token-load and an active-request scorer appended to its profile, once with the producer (the engine keeps
the counters and updates them behind every call) and once without (the same scorers read two ext columns set by
epp_pool_set, i.e. what a caller without the producer has).  In one process the two engines alternate over `reps` rounds
of K async device batches enqueued back to back (the pipelined two-chunk path), timed with CUDA events on the engine's
stream like bench.py's `value`.  Per engine it also reports the update's own CUDA-event time of a synchronous batch
(epp_stats.last_kernel_ms[5]), the host time of one synchronous host batch of 1 / 16 / 256 requests (median of many
calls), and the host time of folding releases.  Prints one JSON line (and writes it to --out)."""
from __future__ import annotations

import argparse
import dataclasses
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

TOKEN_LOAD = (6, 1.0, 0.0, 0, 0.0)
ACTIVE_REQUEST = (7, 1.0, 1.0, 1, 0.0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in q.split(",")]
    return name, power


def time_steps(eng, dev_tokens, w, steps):
    eng.event_record(0)
    for _ in range(steps):
        eng.schedule(dev_tokens, uniform_len=w.prompt_bytes, detail=False, asynchronous=True)
    eng.event_record(1)
    eng.synchronize()
    return eng.event_elapsed_ms() / steps


def small_call_ms(eng, tokens, w, n, calls=200):
    for _ in range(20):
        eng.schedule(tokens[:n], uniform_len=w.prompt_bytes, detail=False)
    t = []
    for _ in range(calls):
        t0 = time.perf_counter()
        eng.schedule(tokens[:n], uniform_len=w.prompt_bytes, detail=False)
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch

    import epp_b200 as epp
    from tools import tracegen as tg
    from tools import workload_setup as helpers
    if not torch.cuda.is_available():
        raise SystemExit("inflight_probe needs a CUDA device")
    gpu, power = card()
    result = {"what": "inflight-load producer cost per scheduling call (config 3 + token-load + active-request)",
              "gpu": gpu, "power_limit": power, "steps": args.steps, "reps": args.reps}
    base = tg.baseline_configs()["config3"]
    w = dataclasses.replace(base, primary_scorers=tuple(base.primary_scorers) + (TOKEN_LOAD, ACTIVE_REQUEST))
    trace = tg.Trace(w)
    tokens, _, _ = trace.requests(0, w.R)
    dev_tokens = torch.from_numpy(tokens.view(np.int32)).cuda()
    engines = {}
    for label in ("without", "with"):
        eng = helpers.make_engine(w, **({"inflight_load": True} if label == "with" else {"n_ext_cols": 2}))
        mid = eng.register_model(tg.MODEL)
        assert mid == 0
        role, kv, waiting, running = trace.pool()
        eng.pool_set(np.arange(w.E, dtype=np.uint32), role, kv, waiting, running,
                     None if label == "with" else np.zeros((2, w.E)))
        fh, _ = eng.hash_prompts(trace.family_tokens(), uniform_len=w.prompt_bytes)
        eng.index_load_snapshot(*trace.index_pairs(fh))
        for _ in range(2):
            eng.schedule(dev_tokens, uniform_len=w.prompt_bytes, detail=False)
        engines[label] = eng
    steps = {"without": [], "with": []}
    for _ in range(args.reps):                          # alternate the two engines
        for label, eng in engines.items():
            steps[label].append(time_steps(eng, dev_tokens, w, args.steps))
    out = {"R": w.R, "E": w.E}
    for label, eng in engines.items():
        eng.schedule(dev_tokens, uniform_len=w.prompt_bytes, detail=False)         # synchronous: per-kernel events
        st = eng.stats()
        out[label] = {"step_ms": steps[label], "step_ms_min": min(steps[label]), "match_pick_ms": st["last_kernel_ms"][3],
                      "update_ms": st["last_kernel_ms"][5]}
    for label, eng in engines.items():
        out[label]["small_call_ms"] = {str(n): small_call_ms(eng, tokens, w, n) for n in (1, 16, 256)}
    eng = engines["with"]
    req, tok = eng.inflight_get()
    n_dec = eng.stats()["n_decisions"]
    out["with"]["requests_counted_equal_decisions"] = bool(int(req.sum()) == int(n_dec))
    rel = np.random.default_rng(1).integers(0, w.E, size=w.R).astype(np.uint32)
    lens = np.full(w.R, w.prompt_bytes, np.uint64)
    t0 = time.perf_counter()
    eng.inflight_release(rel, lens)
    out["with"]["release_fold_ns_per_entry"] = (time.perf_counter() - t0) * 1e9 / w.R
    eng.schedule(dev_tokens, uniform_len=w.prompt_bytes, detail=False)             # applies them, then adds
    req2, _ = eng.inflight_get()
    out["with"]["release_then_add_exact"] = bool(int(req2.sum()) == int(req.sum()))   # R releases, then R adds
    for e in engines.values():
        e.close()
    result["config3"] = out
    line = json.dumps(result)
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
