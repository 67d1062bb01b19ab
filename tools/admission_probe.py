"""Cost of admission on a config-3 batch (4 096 endpoints, 65 536 requests of 16 KiB, the populated config-3 index, the
config-3 profile), as synchronous device-pointer batches through epp_schedule_admit:
  none           no admission inputs (the engine has both admitters)
  prob_all       every request sheddable, whole pool, probabilistic-admitter only
  lat8 / lat64   latency-slo-admitter only, every request sheddable with an SLO and 8 / 64 invalid entries, on the
                 config-3 pool with every endpoint made busy (running >= 1) and warm (kv >= 0.02), so that every entry is read
  sub64 / sub1024  probabilistic-admitter only, every request sheddable with an endpoint subset of 64 / 1 024 slots
For each: the admission kernel's device time (epp_stats.last_kernel_ms[7]) and the step time (CUDA events on the
engine's stream around the call; the host arrays are packed beforehand), medians of --reps timed rounds after two warm-up
rounds, the variants alternating, with the card name, power limit and SM clock read in the same run.

    python tools/admission_probe.py [--reps 10] > profiles/h100_admission_probe.json
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
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
    eng_mod = sys.modules[epp.Engine.__module__]
    capi = epp.capi
    w = tg.baseline_configs()["config3"]
    trace = tg.Trace(w)
    tokens, _, _ = trace.requests(0, w.R)
    data = torch.from_numpy(tokens.view(np.int32)).cuda()
    R, E = w.R, w.E
    rng = np.random.default_rng(1)

    def engine(**acfg):
        eng = epp.Engine(E, epp.ProfileSpec(w.primary_filter, [epp.ScorerSpec(*s) for s in w.primary_scorers]),
                         block_size_tokens=w.block_size_tokens, max_prefix_blocks=w.max_prefix_blocks)
        eng.admission_set(**acfg)
        helpers.setup_engine(eng, w, trace)
        return eng

    engines = {"both": engine(latency_slo=True, probabilistic=True), "prob": engine(probabilistic=True),
               "lat": engine(latency_slo=True)}
    # the latency-slo-admitter reads the entries only when no candidate is idle or cold: a pool where every endpoint is busy
    role, kv, waiting, running = trace.pool()
    engines["lat"].pool_set(np.arange(E, dtype=np.uint32), role, np.maximum(kv, 0.02), waiting, np.maximum(running, 1))

    def spread(n):
        """[R][n] distinct ascending slots per request, at a random offset."""
        return np.sort((rng.integers(0, E, (R, 1)) + np.arange(n) * (E // n)) % E, axis=1).astype(np.uint32)

    prio = np.full(R, -1, np.int32)
    slo = np.full(R, 100.0)
    variants = {}                                       # name -> (engine, subsets, predictions, admission)
    variants["none"] = ("both", None, None, None)
    variants["prob_all"] = ("prob", None, None, dict(priority=prio))
    for n in (8, 64):
        slots = spread(n)
        ent = np.zeros((R, n), dtype=eng_mod.PREDICTION_DTYPE)
        ent["slot"] = slots
        counts = np.full(R, n, np.uint32)
        offsets = (np.arange(R, dtype=np.uint64) * n)
        packed = (counts, offsets, np.ascontiguousarray(ent.reshape(-1)))
        valid = np.zeros(R * n, np.uint8)
        variants[f"lat{n}"] = ("lat", None, packed, dict(priority=prio, ttft_slo=slo, tpot_slo=slo, pred_valid=valid))
    for n in (64, 1024):
        subs = spread(n)
        packed = (np.full(R, n, np.uint32), np.arange(R, dtype=np.uint64) * n, np.ascontiguousarray(subs.reshape(-1)))
        variants[f"sub{n}"] = ("prob", packed, None, dict(priority=prio))

    calls = {}
    for name, (en, subs, preds, adm) in variants.items():
        eng = engines[en]
        b, _, _, keep = eng._batch(data, None, w.prompt_bytes, None, None, None, None)
        dec = torch.empty((R, 32), dtype=torch.uint8, device=data.device)
        sub = pr = ad = None
        hold = [b, keep, dec]
        if subs is not None:
            sub = capi.Subset()
            sub.struct_size = C.sizeof(capi.Subset)
            sub.counts, sub.offsets, sub.slots = (a.ctypes.data for a in subs)
            hold += [sub, subs]
        if preds is not None:
            pr = eng_mod._predictions_struct(preds)
            hold += [pr, preds]
        if adm is not None:
            a = capi.Admission()
            a.struct_size = C.sizeof(capi.Admission)
            arrs = {k: np.ascontiguousarray(v) for k, v in adm.items()}
            for k, v in arrs.items():
                setattr(a, k, v.ctypes.data)
            ad = a
            hold += [a, arrs]
        calls[name] = (eng, b, sub, pr, ad, dec, hold)

    times = {n: [] for n in calls}
    kms = {n: [] for n in calls}
    rejected = {}
    for rep in range(args.reps + 2):
        for name, (eng, b, sub, pr, ad, dec, _) in calls.items():
            eng.event_record(0)
            rc = eng._lib.epp_schedule_admit(eng._h, C.byref(b), C.byref(sub) if sub is not None else None,
                                             C.byref(pr) if pr is not None else None,
                                             None, C.byref(ad) if ad is not None else None, C.c_void_p(dec.data_ptr()), None, 0, None)
            eng.event_record(1)
            assert rc == 0, eng._lib.epp_last_error()
            t = eng.event_elapsed_ms()
            st = eng.stats()
            if rep >= 2:
                times[name].append(t)
                kms[name].append(st["last_kernel_ms"][7])
            rejected[name] = int((epp.decisions_from_torch(dec)["status"] == capi.EPP_STATUS_REJECTED).sum())
    for eng in engines.values():
        eng.close()
    res = {n: dict(step_ms_median=float(np.median(times[n])), step_ms_min=float(np.min(times[n])),
                   step_ms_max=float(np.max(times[n])), admit_kernel_ms_median=float(np.median(kms[n])),
                   rejected=rejected[n]) for n in calls}
    print(json.dumps({"gpu": card(), "workload": f"config3: {E} endpoints, {R} requests of {w.prompt_bytes} B, synchronous "
                      f"device-pointer batches through epp_schedule_admit, {args.reps} timed rounds, variants alternating",
                      "results": res}))


if __name__ == "__main__":
    main()
