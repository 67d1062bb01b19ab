#!/usr/bin/env python
"""A/B probe: times the hot path of BASELINE config 3 (or another config) under several engine variants in ONE process
on ONE GPU and checks that every variant produces identical decisions / hashes.  The engine reads its EPP_* switches
at epp_engine_create, so each variant is a fresh engine with its own environment.

    python tools/ab_probe.py --variants 'base:;noskip:EPP_HASH_SKIP=0;notrim:EPP_HASH_TRIM=0' [--workload config3]

Prints one JSON line per variant: ms per step of K back-to-back async device batches (CUDA events on the engine's
stream), the synchronous per-kernel event times, and ms per hash-only pass.  Development tool (not the bench).
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variants", default="base:;noskip:EPP_HASH_SKIP=0")
    ap.add_argument("--workload", default="config3")
    ap.add_argument("--requests", type=int, default=0)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--index-fill", type=int, default=0)
    ap.add_argument("--hash-only", action="store_true")
    args = ap.parse_args()

    import torch

    import epp_b200 as epp
    from tools import workload_setup as helpers
    from tools import tracegen as tg

    epp.build.build()
    tg.build()
    w = tg.baseline_configs()[args.workload]
    if args.requests:
        w = w.scaled(R=args.requests, name=w.name)
    trace = tg.Trace(w)
    R = w.R
    host = np.empty((R, w.T), dtype=np.uint32)
    trace.requests(0, R, out=host)
    dev_tokens = torch.from_numpy(host.view(np.int32)).cuda()
    dev_dec = torch.empty((R, 32), dtype=torch.uint8, device="cuda")
    hbuf = (torch.empty((R, w.max_prefix_blocks), dtype=torch.int64, device="cuda"),
            torch.empty(R, dtype=torch.int32, device="cuda"))
    ref_dec = ref_hash = None
    known = [k for k in os.environ if k.startswith("EPP_")]
    for spec in args.variants.split(";"):
        name, _, envs = spec.partition(":")
        for k in list(os.environ):
            if k.startswith("EPP_") and k not in known:
                del os.environ[k]
        for kv in filter(None, envs.split(",")):
            k, _, v = kv.partition("=")
            os.environ[k] = v
        out = {"variant": name, "env": envs}
        try:
            eng = helpers.make_engine(w)
            helpers.setup_engine(eng, w, trace, filler_per_endpoint=args.index_fill)
            # hash only
            for _ in range(3):
                eng.hash_prompts(dev_tokens, uniform_len=w.prompt_bytes, out=hbuf)
            torch.cuda.synchronize()
            ms = []
            for _ in range(args.steps):
                eng.hash_prompts(dev_tokens, uniform_len=w.prompt_bytes, out=hbuf)
                st = eng.stats()
                ms.append(sum(st["last_kernel_ms"][:3]))
            out["hash_only_ms"] = float(np.median(ms))
            hh = hbuf[0].cpu().numpy()
            nb = hbuf[1].cpu().numpy()
            for r in range(R):          # rows are only defined up to nblocks
                hh[r, nb[r]:] = 0
            if ref_hash is None:
                ref_hash = (hh, nb)
                out["hash_equal_to_first"] = True
            else:
                out["hash_equal_to_first"] = bool((hh == ref_hash[0]).all() and (nb == ref_hash[1]).all())
            if not args.hash_only:
                for _ in range(3):
                    eng.schedule(dev_tokens, uniform_len=w.prompt_bytes, detail=False, out=dev_dec)
                torch.cuda.synchronize()
                eng.event_record(0)
                for _ in range(args.steps):
                    eng.schedule(dev_tokens, uniform_len=w.prompt_bytes, detail=False, out=dev_dec, asynchronous=True)
                eng.event_record(1)
                eng.synchronize()
                out["step_ms"] = eng.event_elapsed_ms() / args.steps
                out["decisions_per_s"] = R / (out["step_ms"] * 1e-3)
                dev_dec.zero_()
                eng.schedule(dev_tokens, uniform_len=w.prompt_bytes, detail=False, out=dev_dec)
                st = eng.stats()
                out["sync_kernel_ms"] = [round(x, 4) for x in st["last_kernel_ms"][:4]]
                out["launches"] = int(st["last_kernel_launches"])
                out["probes"], out["postings"] = int(st["last_probes"]), int(st["last_postings"])
                out["hash_bytes_stored"] = int(st["last_hash_bytes_stored"])
                out["prompt_bytes_read"] = int(st["last_prompt_bytes_read"])
                dec = epp.decisions_from_torch(dev_dec)
                if ref_dec is None:
                    ref_dec = dec.copy()
                    out["decisions_equal_to_first"] = True
                else:
                    out["decisions_equal_to_first"] = bool((dec.view(np.uint8) == ref_dec.view(np.uint8)).all())
            eng.close()
        except Exception as e:                              # keep going: the other variants still tell us something
            out["error"] = repr(e)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
