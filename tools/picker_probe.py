"""What the random pickers cost per scheduling call, and how much they spread a batch's picks.

    python tools/picker_probe.py [--steps K] [--reps N] [--out FILE]

Config 3 and config 4 (P/D), each with three engines that differ only in the picker of every profile: max-score (with
the random tie rule, tie_seed != 0), random and weighted-random.  In one process the engines alternate over `reps`
rounds of K async device batches enqueued back to back, timed with CUDA events on the engine's stream like bench.py's
`value`.  Per engine: the step time, the match + pick time of a synchronous batch (epp_stats.last_kernel_ms[3]), and the
hot-spotting of one batch -- the most picks on one endpoint and the distinct endpoints picked.  The card's name and
power limit are read in the same run.  Prints one JSON line (and writes it to --out)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PICKERS = {"max_score": 0, "random": 1, "weighted_random": 2}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in q.split(",")]
    return name, power


def make_engine(epp, tg, w, picker):
    primary = epp.ProfileSpec(w.primary_filter, [epp.ScorerSpec(*s) for s in w.primary_scorers], picker=picker)
    prefill = None
    if w.prefill_scorers is not None:
        prefill = epp.ProfileSpec(tg.FILTER_PREFILL, [epp.ScorerSpec(*s) for s in w.prefill_scorers], picker=picker)
    return epp.Engine(w.E, primary, prefill, block_size_tokens=w.block_size_tokens, max_prefix_blocks=w.max_prefix_blocks,
                      non_cached_tokens=w.non_cached_tokens, tie_seed=0x9E3779B97F4A7C15)


def time_steps(eng, dev_tokens, w, steps):
    eng.event_record(0)
    for _ in range(steps):
        eng.schedule(dev_tokens, uniform_len=w.prompt_bytes, detail=False, asynchronous=True)
    eng.event_record(1)
    eng.synchronize()
    return eng.event_elapsed_ms() / steps


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
        raise SystemExit("picker_probe needs a CUDA device")
    gpu, power = card()
    result = {"what": "random pickers: cost per scheduling call (async device batches, pipelined) and pick spread",
              "gpu": gpu, "power_limit": power, "steps": args.steps, "reps": args.reps}
    for name in ("config3", "config4"):
        w = tg.baseline_configs()[name]
        trace = tg.Trace(w)
        tokens, _, _ = trace.requests(0, w.R)
        dev_tokens = torch.from_numpy(tokens.view(np.int32)).cuda()
        engines = {}
        for label, pk in PICKERS.items():
            eng = make_engine(epp, tg, w, pk)
            helpers.setup_engine(eng, w, trace)
            for _ in range(2):
                eng.schedule(dev_tokens, uniform_len=w.prompt_bytes, detail=False)
            engines[label] = eng
        steps = {k: [] for k in engines}
        for _ in range(args.reps):                      # alternate the engines
            for label, eng in engines.items():
                steps[label].append(time_steps(eng, dev_tokens, w, args.steps))
        out = {"R": w.R, "E": w.E}
        for label, eng in engines.items():
            dec, _ = eng.schedule(dev_tokens, uniform_len=w.prompt_bytes, detail=False)     # synchronous: per-kernel events
            st = eng.stats()
            d = epp.decisions_from_torch(dec)
            picks = d["pick"][d["status"] == 0].astype(np.int64)
            counts = np.bincount(picks, minlength=w.E)
            out[label] = {"step_ms": steps[label], "step_ms_min": min(steps[label]),
                          "match_pick_ms": st["last_kernel_ms"][3], "max_picks_one_endpoint": int(counts.max()),
                          "distinct_endpoints_picked": int((counts > 0).sum())}
        for eng in engines.values():
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
