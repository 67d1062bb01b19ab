"""Device time of the match + score + pick kernel on a config-3-sized batch (4 096 endpoints, 65 536 requests of 16 KiB,
the populated config-3 index) on three engines with the config-3 profile (queue 2, kv-cache-utilization 2, prefix 3):
  plain       as configured: the throughput path (k_match_pick_sparse + its overflow pass)
  cl_score    + the context-length-aware scorer (weight 1): a chain engine, k_match_pick_lat
  cl_filter   the same with enableFiltering
Every endpoint carries a range label (a quarter each of 0-2048, 2048-4096, 4096-8192, none); requests carry context lengths
spread over 0 .. 10 000 tokens.  Times are the engine's CUDA events around that kernel (epp_stats.last_kernel_ms[3]) of
synchronous device-pointer batches, the three engines alternating, with the card name and power limit beside them.

    python tools/context_length_probe.py [--reps 10] > profiles/h100_context_length_probe.json
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import torch
    import epp_b200 as epp
    from tools import tracegen as tg
    from tools import workload_setup as helpers
    w = tg.baseline_configs()["config3"]
    trace = tg.Trace(w)
    tokens, _, _ = trace.requests(0, w.R)
    data = torch.from_numpy(tokens.view(np.int32)).cuda()
    rng = np.random.default_rng(1)
    values = ["0-2048", "2048-4096", "4096-8192", None]
    labels = [None if values[e % 4] is None else {"llm-d.ai/context-length-range": values[e % 4]} for e in range(w.E)]
    ctx = rng.integers(0, 10000, w.R).astype(np.int64)
    base = [epp.ScorerSpec(*s) for s in w.primary_scorers]
    engines = {}
    for name in ("plain", "cl_score", "cl_filter"):
        scorers = base if name == "plain" else base + [epp.ScorerSpec(11, 1.0, 0.0)]
        cl = None if name == "plain" else dict(enable_filtering=name == "cl_filter")
        eng = epp.Engine(w.E, epp.ProfileSpec(w.primary_filter, scorers, context_length=cl),
                         block_size_tokens=w.block_size_tokens, max_prefix_blocks=w.max_prefix_blocks)
        helpers.setup_engine(eng, w, trace)
        eng.pool_set_labels(np.arange(w.E, dtype=np.uint32), labels)
        engines[name] = eng
    times = {n: [] for n in engines}
    status = {}
    for rep in range(args.reps + 2):
        for name, eng in engines.items():
            dec, _ = eng.schedule(data, uniform_len=w.prompt_bytes, detail=False,
                                  context_tokens=None if name == "plain" else ctx)
            torch.cuda.synchronize()
            st = eng.stats()
            if rep >= 2:                                   # two warm-up rounds
                times[name].append(st["last_kernel_ms"][3])
            status[name] = int((epp.decisions_from_torch(dec)["status"] != 0).sum())
    for eng in engines.values():
        eng.close()
    res = {n: dict(match_pick_ms_median=float(np.median(t)), match_pick_ms_min=float(np.min(t)),
                   match_pick_ms_max=float(np.max(t)), requests_without_endpoint=status[n]) for n, t in times.items()}
    print(json.dumps({"gpu": card(), "workload": f"config3: {w.E} endpoints, {w.R} requests of {w.prompt_bytes} B, "
                      f"synchronous device-pointer batches, {args.reps} timed rounds, engines alternating",
                      "kernel": "match + score + pick (epp_stats.last_kernel_ms[3])", "results": res}))


if __name__ == "__main__":
    main()
