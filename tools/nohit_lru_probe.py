"""What the no-hit-lru scorer costs per scheduling call, and whether consecutive device batches still decide what the CPU
restatement (tools/nohit_lru_model.py) decides.

    python tools/nohit_lru_probe.py [--steps K] [--reps N] [--out FILE]

Config 3 with a no-hit-lru scorer (weight 1) appended to its profile, and config 4 with it in decode and prefill, each
against the same config without the scorer.  In one process the two engines alternate over `reps` rounds of K async
device batches enqueued back to back (the pipelined two-chunk path) and timed with CUDA events on the engine's stream,
like bench.py's `value`.  Per engine it reports the step time, the match + pick time and the update's own CUDA-event
time of a synchronous batch (epp_stats.last_kernel_ms[3] / [4]) and the cold requests of a batch.  Parity: three
consecutive pipelined batches of a scaled workload (E = 256, R = 8192) against the restatement, decisions and
epp_nohit_lru_get after every batch.  Prints one JSON line (and writes it to --out)."""
from __future__ import annotations

import argparse
import dataclasses
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

NO_HIT = (9, 1.0, 0.0)


def with_scorer(w):
    w = dataclasses.replace(w, primary_scorers=tuple(w.primary_scorers) + (NO_HIT,))
    if w.prefill_scorers is not None:
        w = dataclasses.replace(w, prefill_scorers=tuple(w.prefill_scorers) + (NO_HIT,))
    return w


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in q.split(",")]
    return name, power


def cold_count(eng, tokens, w, chunk=4096):
    """Requests of the batch no endpoint holds a block of (epp_prefix_match): cold for every profile."""
    n = 0
    for r0 in range(0, tokens.shape[0], chunk):
        match, _ = eng.prefix_match(tokens[r0:r0 + chunk], uniform_len=w.prompt_bytes)
        n += int(((match > 0).sum(axis=1) == 0).sum())
    return n


def time_steps(eng, dev_tokens, w, steps):
    eng.event_record(0)
    for _ in range(steps):
        eng.schedule(dev_tokens, uniform_len=w.prompt_bytes, detail=False, asynchronous=True)
    eng.event_record(1)
    eng.synchronize()
    return eng.event_elapsed_ms() / steps


def parity(epp, orc, tg, helpers, M, name):
    import torch
    w = with_scorer(tg.baseline_configs()[name].scaled(E=256, R=8192, T=512))
    trace = tg.Trace(w)
    role, kv, waiting, running = trace.pool()
    profiles = [(w.primary_filter, list(w.primary_scorers))]
    if w.prefill_scorers is not None:
        profiles.append((tg.FILTER_PREFILL, list(w.prefill_scorers)))
    model = M.Model(orc, orc.PoolState(role, kv, waiting, running), w.E, profiles, 0, nct=w.non_cached_tokens,
                    block_size_tokens=w.block_size_tokens)
    ok = True
    with helpers.make_engine(w) as eng:
        helpers.setup_engine(eng, w, trace)
        for b in range(3):
            tokens, _, _ = trace.requests(b * w.R, w.R)
            match, total = eng.prefix_match(tokens, uniform_len=w.prompt_bytes)
            want = model.schedule(match, total, np.full(w.R, w.prompt_bytes, np.int64))
            dec, _ = eng.schedule(torch.from_numpy(tokens.view(np.int32)).cuda(), uniform_len=w.prompt_bytes,
                                  asynchronous=True)
            eng.synchronize()
            d = epp.decisions_from_torch(dec)
            st = np.array([x[0] for x in want])
            ok &= bool((d["status"] == st).all())
            ok &= bool((d["pick"][st == 0] == np.array([x[1] for x in want])[st == 0]).all())
            ok &= bool((d["score"][st == 0] == np.array([x[2] for x in want])[st == 0]).all())
            ok &= bool((d["prefill_pick"] == np.array([x[3] for x in want], dtype=np.uint32)).all())
            ok &= eng.nohit_lru_get() == model.lru.keys()
    return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch

    import epp_b200 as epp
    from oracle import pyoracle as orc
    from tools import nohit_lru_model as M
    from tools import tracegen as tg
    from tools import workload_setup as helpers
    if not torch.cuda.is_available():
        raise SystemExit("nohit_lru_probe needs a CUDA device")
    orc.build()
    gpu, power = card()
    result = {"what": "no-hit-lru scorer cost per scheduling call (async device batches, pipelined)", "gpu": gpu,
              "power_limit": power, "steps": args.steps, "reps": args.reps}
    for name in ("config3", "config4"):
        base_w = tg.baseline_configs()[name]
        trace = tg.Trace(base_w)
        tokens, _, _ = trace.requests(0, base_w.R)
        dev_tokens = torch.from_numpy(tokens.view(np.int32)).cuda()
        engines = {}
        for label, w in (("without", base_w), ("with", with_scorer(base_w))):
            eng = helpers.make_engine(w)
            helpers.setup_engine(eng, w, trace)
            for _ in range(2):
                eng.schedule(dev_tokens, uniform_len=w.prompt_bytes, detail=False)
            engines[label] = (eng, w)
        steps = {"without": [], "with": []}
        for _ in range(args.reps):                      # alternate the two engines
            for label, (eng, w) in engines.items():
                steps[label].append(time_steps(eng, dev_tokens, w, args.steps))
        out = {}
        for label, (eng, w) in engines.items():
            eng.schedule(dev_tokens, uniform_len=w.prompt_bytes, detail=False)     # synchronous: per-kernel events
            st = eng.stats()
            out[label] = {"step_ms": steps[label], "step_ms_min": min(steps[label]),
                          "match_pick_ms": st["last_kernel_ms"][3], "update_ms": st["last_kernel_ms"][4]}
        out["with"]["cold_requests_per_batch"] = cold_count(engines["with"][0], tokens, base_w)
        out["R"] = base_w.R
        out["E"] = base_w.E
        out["parity_3_batches_vs_restatement"] = parity(epp, orc, tg, helpers, M, name)
        for eng, _ in engines.values():
            eng.close()
        del dev_tokens
        torch.cuda.empty_cache()
        result[name] = out
    line = json.dumps(result)
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
