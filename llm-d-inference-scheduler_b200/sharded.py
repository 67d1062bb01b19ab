"""Endpoint-sharded mode (SURVEY.md 8(e)): host-side protocol around the epp_shard_* entry points.

Rank g holds the postings of endpoints [begin_g, end_g) and the FULL pool state.  Because the reference's walk stops
at the first block NO server holds (approximateprefix/plugin.go:219-223), a shard cannot finish alone:

    phase 1  epp_shard_probe   local block-presence masks            [R][W] u32,  W = ceil(max_prefix_blocks / 32)
    exchange all-gather + bitwise OR of the masks (NCCL has no OR reduction)
    phase 2  epp_shard_pick    global stop applied to local counts -> local best records  [R][S] x 24 B
    exchange all-gather of the records
    phase 3  epp_shard_merge   per stage: max score, lowest slot id among equals, ties summed; then the deciders

S is the engine's number of stages (Engine.shard_set_staged): 1 for the single-profile handler, 2 for the disagg
handler's decode + prefill, 3 with its encode stage.

Seeded ties (Engine.shard_set_seeded, epp_engine.h "Seeded ties") add a third exchange: phase 3 becomes epp_shard_select,
which resolves the tie rule over the gathered records (resolve_records_host restates it) and selects the arg-max members
this rank owns; the 8-byte entries are all-gathered and epp_shard_finish builds the decisions from them.  The prefill and encode profiles do not depend on the decode pick,
only whether they run does: every rank publishes its best record of each stage (prefill whenever the P/D decider can
still say yes, encode for multimodal requests), and the merge applies the deciders to the merged decode pick -- still two
exchanges.

torch.distributed is the plumbing (NCCL on GPUs, gloo in the CPU tests); the Go shim uses ncclAllGather directly.
"""
from __future__ import annotations

import numpy as np

SHARD_BEST_DTYPE = np.dtype([("score", "<f8"), ("pick", "<u4"), ("tie_count", "<u4"), ("match_blocks", "<i4"),
                             ("status", "<i4")])
NO_ENDPOINT = 0xFFFFFFFF


def shard_range(rank: int, world: int, n_endpoints: int) -> tuple[int, int]:
    per = (n_endpoints + world - 1) // world
    return min(n_endpoints, rank * per), min(n_endpoints, (rank + 1) * per)


def or_allgather(local_masks, dist=None):
    """All-gather the per-rank masks and OR them.  local_masks: torch int32 tensor [R, W] (CPU or CUDA)."""
    import torch
    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        return local_masks.clone()
    world = dist.get_world_size()
    gathered = torch.empty((world,) + tuple(local_masks.shape), dtype=local_masks.dtype, device=local_masks.device)
    dist.all_gather_into_tensor(gathered.view(-1), local_masks.contiguous().view(-1))
    out = gathered[0].clone()
    for g in range(1, world):
        out |= gathered[g]
    return out


def allgather_records(local_best, dist=None):
    """All-gather the 24-byte best records (or the 8-byte selected entries).  local_best: torch uint8 tensor [R, X]
    -> [world, R, X]."""
    import torch
    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        return local_best.unsqueeze(0).clone()
    world = dist.get_world_size()
    gathered = torch.empty((world,) + tuple(local_best.shape), dtype=local_best.dtype, device=local_best.device)
    dist.all_gather_into_tensor(gathered.view(-1), local_best.contiguous().view(-1))
    return gathered


def merge_records_host(all_best: np.ndarray) -> np.ndarray:
    """Reference semantics of epp_shard_merge on the host (numpy), used by the CPU protocol tests only:
    all_best [world, R] of SHARD_BEST_DTYPE -> (status, pick, score, tie_count, match_blocks) arrays."""
    world, R = all_best.shape
    out = np.zeros(R, dtype=SHARD_BEST_DTYPE)
    out["status"] = -1
    out["pick"] = NO_ENDPOINT
    for g in range(world):
        rec = all_best[g]
        ok = rec["status"] == 0
        have = out["status"] == 0
        better = ok & (~have | (rec["score"] > out["score"]))
        equal = ok & have & (rec["score"] == out["score"])
        # ties: sum counts, keep the lowest slot id (and its match count)
        lower = equal & (rec["pick"] < out["pick"])
        out["tie_count"] = np.where(better, rec["tie_count"], np.where(equal, out["tie_count"] + rec["tie_count"], out["tie_count"]))
        take = better | lower
        out["pick"] = np.where(take, rec["pick"], out["pick"])
        out["match_blocks"] = np.where(take, rec["match_blocks"], out["match_blocks"])
        out["score"] = np.where(better, rec["score"], out["score"])
        out["status"] = np.where(ok, 0, out["status"])
    return out


SHARD_SEL_DTYPE = np.dtype([("pick", "<u4"), ("match_blocks", "<i4")])


def _mix64(z: int) -> int:
    m = (1 << 64) - 1
    z = (z + 0x9E3779B97F4A7C15) & m
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & m
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & m
    return z ^ (z >> 31)


def tie_rank_host(seed: int, key: int, n: int) -> int:
    """The tie rule's member rank (epp_engine.h, "Tie rule")."""
    return ((_mix64((seed ^ _mix64(key)) & ((1 << 64) - 1)) >> 32) * n) >> 32


def resolve_records_host(all_best: np.ndarray, tie_seed: int, tie_base: int, stage: int = 0):
    """The owner computation of epp_shard_select on the host: all_best [world, R] of SHARD_BEST_DTYPE (one stage) ->
    (merged records [R] as merge_records_host returns them, owner [R] (index in all_best, -1 when no rank has a
    candidate), rho_local [R]: the rank of member tie_rank(seed, 4 * (tie_base + r) + stage, N) in the owner's local
    set).  The shard ranges are disjoint, so the global arg-max set in ascending slot order is the local sets taken in
    the order of their records' picks."""
    world, R = all_best.shape
    merged = merge_records_host(all_best)
    owner = np.full(R, -1, np.int64)
    local = np.zeros(R, np.uint32)
    for r in range(R):
        if merged["status"][r] != 0:
            continue
        n = int(merged["tie_count"][r])
        rho = tie_rank_host(tie_seed, 4 * (tie_base + r) + stage, n) if n > 1 else 0
        at_max = [g for g in range(world) if all_best[g, r]["status"] == 0 and all_best[g, r]["score"] == merged["score"][r]]
        for g in sorted(at_max, key=lambda g: int(all_best[g, r]["pick"])):
            c = int(all_best[g, r]["tie_count"])
            if rho < c:
                owner[r], local[r] = g, rho
                break
            rho -= c
    return merged, owner, local


STAGE_DETAIL_DTYPE = np.dtype([("prefill_pick", "<u4"), ("prefill_score", "<f8"), ("prefill_tie_count", "<u4"),
                               ("prefill_ran", "<u4"), ("encode_pick", "<u4"), ("encode_score", "<f8"),
                               ("encode_tie_count", "<u4"), ("encode_ran", "<u4")])


def pd_decide_host(nct: int, in_len_bytes: int, match_blocks: int, block_size_tokens: int) -> bool:
    """PrefixBasedPDDecider.disaggregate (prefix_based_pd_decider.go:99-149), as score.cuh pd_decide."""
    if nct == 0:
        return False
    tokens = in_len_bytes // 4
    return tokens >= nct and tokens - match_blocks * block_size_tokens >= nct


def merge_stage_records_host(all_best: np.ndarray, in_len, multimodal=None, *, non_cached_tokens: int = 0,
                             always_disagg: bool = False, block_size_tokens: int = 16, encode_enabled: bool = False):
    """Reference semantics of the staged epp_shard_merge on the host, for the CPU tests: all_best [world, R, S] of
    SHARD_BEST_DTYPE, in_len [R] request bytes, multimodal [R] flags or None -> (decode records [R] as
    merge_records_host returns them, STAGE_DETAIL_DTYPE [R]).  Each stage is reduced by merge_records_host; the decode
    pick's match_blocks drives the P/D decider; no decode pick anywhere runs no other stage."""
    world, R, S = all_best.shape
    stages = [merge_records_host(all_best[:, :, s]) for s in range(S)]
    dec = stages[0]
    det = np.zeros(R, dtype=STAGE_DETAIL_DTYPE)
    det["prefill_pick"] = NO_ENDPOINT
    det["encode_pick"] = NO_ENDPOINT
    for r in range(R):
        if dec["status"][r] != 0:
            continue
        if S >= 3 and encode_enabled and multimodal is not None and multimodal[r]:
            det["encode_ran"][r] = 1
            e = stages[2][r]
            if e["status"] == 0:
                det["encode_pick"][r], det["encode_score"][r], det["encode_tie_count"][r] = e["pick"], e["score"], e["tie_count"]
        if S >= 2 and (always_disagg or pd_decide_host(non_cached_tokens, int(in_len[r]), int(dec["match_blocks"][r]),
                                                       block_size_tokens)):
            det["prefill_ran"][r] = 1
            p = stages[1][r]
            if p["status"] == 0:
                det["prefill_pick"][r], det["prefill_score"][r], det["prefill_tie_count"][r] = p["pick"], p["score"], p["tie_count"]
    return dec, det


def schedule_sharded(engine, tokens_dev, uniform_len: int, dist=None, detail=None, multimodal=None):
    """One batch through the sharded protocol on this rank's engine.  tokens_dev: torch CUDA tensor [R, T]; detail: a
    [R, 40] uint8 CUDA tensor for the epp_decision_detail records (the prefill and encode stages), or None; multimodal:
    [R] uint8 CUDA tensor or None.  Returns a [R, 32] uint8 CUDA tensor of epp_decision records (identical on every
    rank)."""
    import torch
    R = tokens_dev.shape[0]
    W = (engine.B + 31) // 32
    dev = tokens_dev.device
    masks = torch.empty((R, W), dtype=torch.int32, device=dev)
    engine.shard_probe(tokens_dev, masks, uniform_len=uniform_len, multimodal=multimodal)
    gmasks = or_allgather(masks, dist)
    best = torch.empty((R, 24 * engine.shard_stages), dtype=torch.uint8, device=dev)
    # The engine runs on its own streams and only guarantees that ITS outputs are complete on return; tensors produced
    # by torch / NCCL on the caller's stream must be complete before they are handed over (epp_engine.h, "streams").
    torch.cuda.current_stream(dev).synchronize()
    engine.shard_pick(R, gmasks, best)
    allb = allgather_records(best, dist)
    dec = torch.empty((R, 32), dtype=torch.uint8, device=dev)
    torch.cuda.current_stream(dev).synchronize()
    if not getattr(engine, "shard_seeded", False):
        engine.shard_merge(R, allb.shape[0], allb, dec, out_detail=detail)
        return dec
    # seeded ties: the third exchange carries the members each rank selected
    sel = torch.empty((R, 8 * engine.shard_stages), dtype=torch.uint8, device=dev)
    engine.shard_select(R, allb.shape[0], allb, sel)
    alls = allgather_records(sel, dist)
    torch.cuda.current_stream(dev).synchronize()
    engine.shard_finish(R, allb.shape[0], allb, alls, dec, out_detail=detail)
    return dec


# ---- the same protocol with the exchanges over NVLink peer memory (csrc/shard_p2p.cu): no NCCL on the data path ----
def connect_p2p(engine, max_requests: int, dist=None):
    """Export this rank's exchange buffer, all-gather the 64-byte CUDA IPC handles (the only collective, once) and open
    every peer's buffer."""
    import torch
    handle, _ = engine.shard_p2p_export(max_requests)
    if dist is None or not dist.is_initialized() or dist.get_world_size() == 1:
        engine.shard_p2p_connect(1, 0, handle.reshape(1, 64), ipc_handles=True)
        return
    world, rank = dist.get_world_size(), dist.get_rank()
    dev = torch.device("cuda", torch.cuda.current_device())
    mine = torch.from_numpy(handle).to(dev)
    allh = torch.empty((world, 64), dtype=torch.uint8, device=dev)
    dist.all_gather_into_tensor(allh.view(-1), mine)
    engine.shard_p2p_connect(world, rank, allh.cpu().numpy(), ipc_handles=True)


def schedule_sharded_p2p(engine, tokens_dev, uniform_len: int, out=None):
    """One batch; every rank calls it with the same tokens.  Returns a [R, 32] uint8 CUDA tensor of epp_decision."""
    import torch
    R = tokens_dev.shape[0]
    dec = out if out is not None else torch.empty((R, 32), dtype=torch.uint8, device=tokens_dev.device)
    engine.shard_schedule_p2p(tokens_dev, dec, uniform_len=uniform_len)
    return dec
