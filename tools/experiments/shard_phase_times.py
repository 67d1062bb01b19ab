"""Where the time of one endpoint-sharded step goes: two shard engines on ONE GPU, stepped phase by phase
(epp_shard_p2p_phase), each phase of rank 0 timed by the host clock around the call, which synchronises (rank 1 only
keeps the protocol moving).
    python tools/experiments/shard_phase_times.py [R] [config5|config4] [--seeded] [--out FILE.json]
config5 (default): the config-5 profile on a config-5 pool.  config4: three engine configurations on the same config-4
pool and batch -- the config-5 single profile, config 4's P/D handler (decode + prefill, S = 2 records per request) and
config 4 with the prefill profile removed (S = 1) -- so that the cost of scoring the prefill profile speculatively in
phase 1 is the difference of the last two.
--seeded: the config-5 profile on a config-5 pool, the lowest-slot engines (three phases) and the seeded ones
(epp_shard_set_seeded, tie_seed != 0: four phases) alternated round by round in the one call, and the share of requests
whose seeded member needed a select (its rank in its owner's local set >= 1), from one host-driven batch's records."""
import json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch
import epp_b200 as epp
from tools import tracegen as tg

PHASES = ("hash + presence masks + signal", "wait + OR + match over the shard + signal", "wait + gather + merge + check")
PHASES_SEEDED = PHASES[:2] + ("wait + gather + resolve + select + signal", "wait + gather + finish + check")


def engines_for(w, trace, primary, prefill, world, R_max, tie_seed=0):
    """`world` shard engines on one GPU wired by raw pointers; prefill None: the single-profile handler; tie_seed != 0:
    the seeded tie rule."""
    role, kv, waiting, running = trace.pool()
    fam = trace.family_tokens()
    engines, ptrs = [], []
    for g in range(world):
        eng = epp.Engine(w.E, epp.ProfileSpec(w.primary_filter, [epp.ScorerSpec(*s) for s in primary]),
                         None if prefill is None else epp.ProfileSpec(tg.FILTER_PREFILL, [epp.ScorerSpec(*s) for s in prefill]),
                         block_size_tokens=w.block_size_tokens, max_prefix_blocks=w.max_prefix_blocks,
                         non_cached_tokens=w.non_cached_tokens, tie_seed=tie_seed)
        eng.register_model(tg.MODEL)
        per = (w.E + world - 1) // world
        lo, hi = min(w.E, g * per), min(w.E, (g + 1) * per)
        stages = eng.shard_set_seeded(lo, hi) if tie_seed else eng.shard_set_staged(lo, hi)
        eng.pool_set(np.arange(w.E, dtype=np.uint32), role, kv, waiting, running)
        fh, _ = eng.hash_prompts(fam, uniform_len=w.prompt_bytes)
        hs, es = trace.index_pairs(fh)
        keep = (es >= lo) & (es < hi)
        eng.index_load_snapshot(hs[keep], es[keep])
        _, ptr = eng.shard_p2p_export(R_max)
        engines.append(eng)
        ptrs.append(ptr)
    for g, eng in enumerate(engines):
        eng.shard_p2p_connect(world, g, np.array(ptrs, dtype=np.uint64), ipc_handles=False)
    return engines, stages


def phase_times(engines, dt, w, iters=8, warm=2, n_phases=3):
    R = dt.shape[0]
    outs = [torch.zeros((R, 32), dtype=torch.uint8, device="cuda") for _ in engines]
    dets = [torch.zeros((R, 40), dtype=torch.uint8, device="cuda") for _ in engines]
    res = {p: [] for p in range(n_phases)}
    for it in range(iters):
        for phase in range(n_phases):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            engines[0].shard_p2p_phase(dt, outs[0], phase, uniform_len=w.prompt_bytes, out_detail=dets[0])
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            for e, o, d in zip(engines[1:], outs[1:], dets[1:]):
                e.shard_p2p_phase(dt, o, phase, uniform_len=w.prompt_bytes, out_detail=d)
            torch.cuda.synchronize()
            if it >= warm:
                res[phase].append((t1 - t0) * 1e3)
    dec = epp.decisions_from_torch(outs[0])
    det = dets[0].cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1)
    return {f"phase{p}_ms_median": float(np.median(res[p])) for p in range(n_phases)} | \
           {f"phase{p}_ms_all": [round(x, 4) for x in res[p]] for p in range(n_phases)} | \
           {"prefill_ran": int(det["prefill_ran"].sum()), "decided": int((dec["status"] == 0).sum()),
            "tied": int((dec["tie_count"] > 1).sum())}


def select_share(engines, dt, w, tie_seed):
    """One host-driven batch through the seeded engines' probe and pick: the share of requests whose seeded decode member
    is not its owner's lowest tied slot (a select ran for it), from sharded.resolve_records_host."""
    import importlib
    sh = importlib.import_module("llm-d-inference-scheduler_b200.sharded")
    R = dt.shape[0]
    W = (w.max_prefix_blocks + 31) // 32
    masks = []
    for eng in engines:
        m = torch.zeros((R, W), dtype=torch.int32, device="cuda")
        eng.shard_probe(dt, m, uniform_len=w.prompt_bytes)
        masks.append(m)
    gm = masks[0].clone()
    for m in masks[1:]:
        gm |= m
    torch.cuda.synchronize()
    bests = []
    for eng in engines:
        b = torch.zeros((R, 24 * eng.shard_stages), dtype=torch.uint8, device="cuda")
        eng.shard_pick(R, gm, b)
        bests.append(b.cpu().numpy().view(sh.SHARD_BEST_DTYPE).reshape(R, -1)[:, 0])
    _, owner, local = sh.resolve_records_host(np.stack(bests), tie_seed, engines[0].stats()["n_decisions"])
    return float((local >= 1).mean())


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    out = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    if out in args:
        args.remove(out)
    R = int(args[0]) if args else 65536
    workload = args[1] if len(args) > 1 else "config5"
    tg.build()
    if "--seeded" in sys.argv:
        return main_seeded(R, out)
    runs = []
    if workload == "config5":
        w = tg.baseline_configs()["config5"].scaled(E=8192, R=R, T=4096, name="config5")
        confs = [("config5 single profile", w.primary_scorers, None)]
    else:
        w = tg.baseline_configs()["config4"].scaled(E=2560, R=R, T=4096, name="config4")
        c5 = tg.baseline_configs()["config5"]
        confs = [("config5 single profile", c5.primary_scorers, None),
                 ("config4 P/D (S=2)", w.primary_scorers, w.prefill_scorers),
                 ("config4 prefill removed (S=1)", w.primary_scorers, None)]
    trace = tg.Trace(w)
    tokens, _, _ = trace.requests(0, R)
    dt = torch.from_numpy(tokens.view(np.int32)).cuda()
    info = gpu_info()
    for name, primary, prefill in confs:
        engines, stages = engines_for(w, trace, primary, prefill, 2, R)
        try:
            r = phase_times(engines, dt, w)
        finally:
            for e in engines:
                e.close()
        r.update(name=name, stages=stages)
        runs.append(r)
        print(f"{name}: " + ", ".join(f"phase {p} ({PHASES[p]}) {r[f'phase{p}_ms_median']:.3f} ms" for p in range(3)))
    rec = {"gpu (name, power limit, SM clock, max SM clock)": info, "info_read": "same run, before the timed loops",
           "workload": w.name, "E": w.E, "R": R, "T": w.T, "max_prefix_blocks": w.max_prefix_blocks, "world": 2,
           "ranks": "two shard engines on one GPU, stepped phase by phase", "timer": "host clock around each phase call of "
           "rank 0, which synchronises before it returns (launch + sync included); median of the timed iterations",
           "runs": runs}
    print(json.dumps({k: v for k, v in rec.items() if k != "runs"}))
    if out:
        with open(out, "w") as f:
            json.dump(rec, f, indent=1)


def main_seeded(R, out, rounds=3, tie_seed=0x5EED):
    w = tg.baseline_configs()["config5"].scaled(E=8192, R=R, T=4096, name="config5")
    trace = tg.Trace(w)
    tokens, _, _ = trace.requests(0, R)
    dt = torch.from_numpy(tokens.view(np.int32)).cuda()
    info = gpu_info()
    runs = []
    for rnd in range(rounds):
        for seed in (0, tie_seed):
            engines, stages = engines_for(w, trace, w.primary_scorers, None, 2, R, tie_seed=seed)
            try:
                r = phase_times(engines, dt, w, n_phases=4 if seed else 3)
                if seed and rnd == 0:
                    r["select_share"] = select_share(engines, dt, w, seed)
            finally:
                for e in engines:
                    e.close()
            r.update(name="seeded" if seed else "lowest slot", round=rnd, stages=stages)
            runs.append(r)
            names = PHASES_SEEDED if seed else PHASES
            print(f"round {rnd} {r['name']}: " + ", ".join(f"phase {p} ({names[p]}) {r[f'phase{p}_ms_median']:.3f} ms"
                                                          for p in range(len(names))))
    med = lambda name, p: float(np.median([x[f"phase{p}_ms_median"] for x in runs if x["name"] == name]))
    summary = {"lowest slot, phase medians over rounds (ms)": [med("lowest slot", p) for p in range(3)],
               "seeded, phase medians over rounds (ms)": [med("seeded", p) for p in range(4)],
               "extra phase (seeded phase 3, ms)": med("seeded", 3),
               "seeded phases 2 + 3 - lowest-slot phase 2 (ms)": med("seeded", 2) + med("seeded", 3) - med("lowest slot", 2),
               "select_share": next(x["select_share"] for x in runs if "select_share" in x)}
    rec = {"gpu (name, power limit, SM clock, max SM clock)": info, "info_read": "same run, before the timed loops",
           "workload": w.name, "E": w.E, "R": R, "T": w.T, "max_prefix_blocks": w.max_prefix_blocks, "world": 2,
           "tie_seed": tie_seed, "ranks": "two shard engines on one GPU, stepped phase by phase; lowest-slot and seeded "
           "engines alternated round by round", "timer": "host clock around each phase call of rank 0, which synchronises "
           "before it returns (launch + sync included); median of the timed iterations", "summary": summary, "runs": runs}
    print(json.dumps({k: v for k, v in rec.items() if k != "runs"}))
    if out:
        with open(out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
