"""What the chart's predicted-latency profile costs (include/epp_engine.h "Latency predictions").

    python tools/predicted_latency_probe.py [--reps N] [--leg pool|subset|all] [--out FILE]

Pools of 64 and 1024 endpoints, batches of 1, 64 and 1024 requests of 1 KiB prompts against an index that holds every
prompt's first blocks on a few endpoints, each request carrying a prediction for every candidate.  Three engines on
the same pool: the chart profile (affinity 0.99 -> slo-headroom-tier-filter -> affinity 0.80 -> latency-scorer ->
weighted-random picker) with predictions, the same engine without predictions, and the default profile (queue 2, kv 2,
prefix 3, max-score).  Paths per cell:
  host    Engine.schedule of a host batch: host clock around the synchronous call, packing the per-request prediction
          arrays included (median over N);
  device  the same batch in device memory: epp_stats.last_kernel_ms[3], the match + score + pick kernel (median);
  batcher R requests submitted from R / 8 threads (at most 16) and waited for: wall time of the round (median).
Records the card's name and power limit from the same run and the bytes of predictions staged per call
(32 per entry + 12 per request).
Subset leg (endpoint subsets on the chart engine, epp_schedule_subset_predicted): pools of 1024 and 4096 endpoints, a
batch of 64 requests, each restricted to S = 8, 64 or 1024 listed slots with a prediction for every listed slot:
  subset_kernel_ms    epp_stats.last_kernel_ms[6] of the device batch (k_subset_pick_lat, median), against
  pool_match_pick_ms  last_kernel_ms[3] of the same calls (the whole-pool match + pick kernel that runs first);
  host_ms_per_call    host clock around the synchronous host-batch call, packing both lists included (median).
Prints one JSON line (and writes it to --out)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    return [x.strip() for x in q.split(",")]


def med(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def engine(epp, kind, E):
    if kind == "default":
        return epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(2, 2.0), epp.ScorerSpec(1, 2.0), epp.ScorerSpec(0, 3.0)]),
                          tie_seed=0x5EED)
    spec = epp.ProfileSpec(0, [epp.ScorerSpec(10, 1.0)], epp.AffinityFilterSpec(0.80, 0.01, 5000.0), 2,
                           latency=dict(tier_filter=1, epsilon_explore_neg=0.01, a1_affinity_threshold=0.99,
                                        a1_exploration_probability=0.01, a1_max_ttft_penalty_ms=5000.0))
    return epp.Engine(E, spec, tie_seed=0x5EED)


def cell(epp, kind, E, R, reps, torch):
    rng = np.random.default_rng(E * 7 + R)
    L = 1024
    data = rng.integers(0, 256, R * L).astype(np.uint8)
    preds = None
    if kind == "chart":
        preds = []
        for _ in range(R):
            a = np.zeros(E, dtype=epp.PREDICTION_DTYPE)
            a["slot"] = np.arange(E)
            a["ttft"] = rng.integers(1, 500, E)
            a["ttft_headroom"] = rng.integers(-100, 200, E)
            a["tpot_headroom"] = rng.integers(-10, 30, E)
            a["dispatched"] = rng.integers(0, 3, E)
            preds.append(a)
    out = {}
    with engine(epp, kind, E) as eng:
        eng.register_model(b"m")
        eng.pool_set(np.arange(E, dtype=np.uint32), np.zeros(E, np.uint8), rng.random(E), rng.integers(0, 20, E),
                     rng.integers(0, 20, E))
        hashes, _ = eng.hash_prompts(data, uniform_len=L)
        for r in range(min(R, 256)):                # every prompt's first 8 blocks on 3 endpoints
            for e in (r % E, (r + 1) % E, (r + 7) % E):
                eng.index_add(e, np.asarray(hashes[r, :8], dtype=np.uint64))
        eng.index_commit()
        t = []
        for _ in range(reps + 2):
            t0 = time.perf_counter()
            eng.schedule(data, uniform_len=L, predictions=preds)
            t.append((time.perf_counter() - t0) * 1e3)
        out["host_ms"] = med(t[2:])
        dt = torch.from_numpy(data).cuda()
        k = []
        for _ in range(reps + 2):
            eng.schedule(dt, uniform_len=L, predictions=preds)
            k.append(eng.stats()["last_kernel_ms"][3])
        out["device_match_pick_ms"] = med(k[2:])
        b = epp.Batcher(eng, max_batch=min(R, 256), max_delay_us=50)
        try:
            nt = max(1, min(16, R // 8))
            rounds = []
            for _ in range(max(3, reps // 4) + 1):
                def worker(t):
                    for r in range(t, R, nt):
                        tk = b.submit(data[r * L:(r + 1) * L], predictions=preds[r] if preds else None)
                        b.wait(tk)
                th = [threading.Thread(target=worker, args=(i,)) for i in range(nt)]
                t0 = time.perf_counter()
                for x in th:
                    x.start()
                for x in th:
                    x.join()
                rounds.append((time.perf_counter() - t0) * 1e3)
            out["batcher_round_ms"] = med(rounds[1:])
            out["batcher_threads"] = nt
        finally:
            b.close()
    out["prediction_bytes_staged_per_call"] = (32 * E * R + 12 * R) if preds else 0
    return out


def subset_cell(epp, E, S, reps, torch):
    R, L = 64, 1024
    rng = np.random.default_rng(E * 11 + S)
    data = rng.integers(0, 256, R * L).astype(np.uint8)
    subsets, preds = [], []
    for _ in range(R):
        sl = np.sort(rng.choice(E, S, replace=False)).astype(np.uint32)
        a = np.zeros(S, dtype=epp.PREDICTION_DTYPE)
        a["slot"] = sl
        a["ttft"] = rng.integers(1, 500, S)
        a["ttft_headroom"] = rng.integers(-100, 200, S)
        a["tpot_headroom"] = rng.integers(-10, 30, S)
        a["dispatched"] = rng.integers(0, 3, S)
        subsets.append(sl)
        preds.append(a)
    out = {}
    with engine(epp, "chart", E) as eng:
        eng.register_model(b"m")
        eng.pool_set(np.arange(E, dtype=np.uint32), np.zeros(E, np.uint8), rng.random(E), rng.integers(0, 20, E),
                     rng.integers(0, 20, E))
        hashes, _ = eng.hash_prompts(data, uniform_len=L)
        for r in range(R):                          # every prompt's first 8 blocks on 3 listed endpoints
            for e in subsets[r][:3]:
                eng.index_add(int(e), np.asarray(hashes[r, :8], dtype=np.uint64))
        eng.index_commit()
        t = []
        for _ in range(reps + 2):
            t0 = time.perf_counter()
            eng.schedule(data, uniform_len=L, subsets=subsets, predictions=preds)
            t.append((time.perf_counter() - t0) * 1e3)
        out["host_ms_per_call"] = med(t[2:])
        dt = torch.from_numpy(data).cuda()
        ks, kp = [], []
        for _ in range(reps + 2):
            eng.schedule(dt, uniform_len=L, subsets=subsets, predictions=preds)
            st = eng.stats()["last_kernel_ms"]
            ks.append(st[6])
            kp.append(st[3])
        out["subset_kernel_ms"] = med(ks[2:])
        out["pool_match_pick_ms"] = med(kp[2:])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--leg", choices=("pool", "subset", "all"), default="all")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this probe measures the GPU path only")
    import epp_b200 as epp
    epp.build.build()
    name, power, clk = card()
    rec = {"probe": "predicted_latency", "card": name, "power_limit": power, "sm_clock_max": clk, "reps": a.reps,
           "prompt_bytes": 1024, "cells": []}
    if a.leg != "pool":
        rec["subset_cells"] = []
        for E in (1024, 4096):
            for S in (8, 64, 1024):
                c = subset_cell(epp, E, S, a.reps, torch)
                c.update(engine="chart", E=E, R=64, S=S)
                rec["subset_cells"].append(c)
                print(json.dumps(c), file=sys.stderr, flush=True)
    for E in ((64, 1024) if a.leg != "subset" else ()):
        for R in (1, 64, 1024):
            for kind in ("chart", "chart_no_predictions", "default"):
                c = cell(epp, "chart" if kind == "chart" else ("default" if kind == "default" else "chart_np"), E, R,
                         a.reps, torch)
                c.update(engine=kind, E=E, R=R)
                rec["cells"].append(c)
                print(json.dumps(c), file=sys.stderr, flush=True)
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
