"""CPU-side checks of the drop-in boundary: libepp_engine.so builds for sm_90a, loads, exports every symbol
include/epp_engine.h declares, matches the ctypes struct layouts, and FAILS LOUDLY without a GPU (no CPU fallback).
No compute calls here."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "epp_engine.h")


@pytest.fixture(scope="module")
def epp():
    import epp_b200
    epp_b200.build.build()
    return epp_b200


def _declared_symbols():
    src = open(HEADER).read()
    return sorted(set(re.findall(r"^EPP_API [^;(]*?\b(epp_[a-z_0-9]+)\s*\(", src, flags=re.M)))


def test_every_declared_symbol_is_exported(epp):
    declared = _declared_symbols()
    assert len(declared) >= 25
    out = subprocess.check_output(["nm", "-D", "--defined-only", epp.capi.LIB_PATH], text=True)
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    missing = [s for s in declared if s not in exported]
    assert not missing, f"declared in include/epp_engine.h but not exported: {missing}"
    # and the ctypes table binds exactly the declared set
    assert sorted(epp.capi.SIGNATURES) == declared
    lib = epp.capi.load()
    assert lib.epp_abi_version() == 5


def test_library_contains_sm90a_code(epp):
    out = subprocess.run(["cuobjdump", "-lelf", epp.capi.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out, out[:400]


def test_struct_layouts_match_header(epp, tmp_path):
    """Compile a tiny C program against the header and compare sizeof/offsetof with the ctypes mirrors."""
    src = tmp_path / "layout.c"
    src.write_text(r'''
#include <stdio.h>
#include <stddef.h>
#include "epp_engine.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(epp_config), sizeof(epp_profile_cfg), sizeof(epp_scorer_cfg),
         sizeof(epp_decision), sizeof(epp_decision_detail), sizeof(epp_batch), sizeof(epp_stats), sizeof(epp_shard_best));
  printf("%zu %zu %zu %zu\n", offsetof(epp_config, non_cached_tokens), offsetof(epp_config, primary),
         offsetof(epp_config, prefill), offsetof(epp_decision, score));
  printf("%zu %zu %zu %zu %zu %zu\n", sizeof(epp_topk_out), sizeof(epp_batcher_cfg), sizeof(epp_batcher_stats_t),
         offsetof(epp_profile_cfg, affinity_threshold), offsetof(epp_config, tie_seed), offsetof(epp_config, index_commit_interval_us));
  return 0; }''')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    l1, l2, l3 = subprocess.check_output([str(exe)], text=True).splitlines()
    c = epp.capi
    assert [int(x) for x in l1.split()] == [C.sizeof(c.Config), C.sizeof(c.ProfileCfg), C.sizeof(c.ScorerCfg),
                                            C.sizeof(c.Decision), C.sizeof(c.DecisionDetail), C.sizeof(c.Batch),
                                            C.sizeof(c.Stats), C.sizeof(c.ShardBest)]
    assert [int(x) for x in l2.split()] == [c.Config.non_cached_tokens.offset, c.Config.primary.offset,
                                            c.Config.prefill.offset, c.Decision.score.offset]
    assert [int(x) for x in l3.split()] == [C.sizeof(c.TopkOut), C.sizeof(c.BatcherCfg), C.sizeof(c.BatcherStats),
                                            c.ProfileCfg.affinity_threshold.offset, c.Config.tie_seed.offset,
                                            c.Config.index_commit_interval_us.offset]
    assert epp.DECISION_DTYPE.itemsize == C.sizeof(c.Decision)


def test_default_config_is_the_reference_default(epp):
    cfg = epp.capi.Config()
    epp.capi.load().epp_config_default(C.byref(cfg))
    assert (cfg.block_size_tokens, cfg.max_prefix_blocks, cfg.lru_capacity_per_server) == (16, 256, 31250)  # types.go:92-110
    got = [(cfg.primary.scorers[i].kind, cfg.primary.scorers[i].weight) for i in range(cfg.primary.n_scorers)]
    assert got == [(epp.capi.SCORER_QUEUE, 2.0), (epp.capi.SCORER_KV_UTIL, 2.0), (epp.capi.SCORER_PREFIX, 3.0)]  # defaults.go:47-49,78-87


def test_no_gpu_means_loud_failure(epp):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(epp.EngineError) as ei:
        epp.Engine(64)
    assert ei.value.code == epp.capi.EPP_ERR_NO_DEVICE and "no CPU fallback" in ei.value.message


def test_product_never_imports_the_oracle():
    """The product package must not reference oracle/ (only tests, smoke() and bench's CPU legs may)."""
    pkg = os.path.join(ROOT, "llm-d-inference-scheduler_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "oracle" not in text.replace("no CPU fallback", ""), f"{f} mentions the oracle"


def test_tracegen_is_deterministic_and_thread_independent():
    from tools import tracegen as tg
    w = tg.baseline_configs()["config3"].scaled(E=256, R=64, T=512)
    a = tg.Trace(w, n_threads=1)
    b = tg.Trace(w, n_threads=7)
    ta, fa, sa = a.requests()
    tb, fb, sb = b.requests()
    np.testing.assert_array_equal(ta, tb)
    np.testing.assert_array_equal(fa, fb)
    tc, _, _ = b.requests(10, 20)
    np.testing.assert_array_equal(tc, ta[10:30])
    assert ta.max() < 128000
    hot = fa >= 0
    assert 0.5 < hot.mean() < 0.9
    fam = a.family_tokens()
    for r in np.flatnonzero(hot)[:10]:
        L = sa[r] * w.block_size_tokens
        np.testing.assert_array_equal(ta[r, :L], fam[fa[r], :L])
    role, kv, waiting, running = a.pool()
    assert set(role.tolist()) == {1} and kv.min() >= 0 and kv.max() <= 1 and (waiting == 0).mean() > 0.5
    n, ep, depth, hole = a.index_plan()
    assert set(n.tolist()) <= {1, 2, 3, 4, 5, 6, 7, 8} and (hole > 0).any()


def test_oracle_cycle_batch_matches_stepwise(orc):
    """orc_cycle_batch (the timed CPU baseline) == hash_prompt + match_longest_prefix + schedule, any thread count."""
    import helpers
    from tools import tracegen as tg
    for name, kw in (("config3", dict(E=128, R=96, T=512)), ("config4", dict(E=160, R=96, T=512))):
        w = tg.baseline_configs()[name].scaled(**kw)
        trace = tg.Trace(w)
        tokens, _, _ = trace.requests()
        pool, ix, primary, prefill, _ = helpers.setup_oracle(orc, w, trace)
        d1, t1 = helpers.oracle_decisions(orc, w, pool, ix, primary, prefill, tokens, n_threads=1)
        d3, t3 = helpers.oracle_decisions(orc, w, pool, ix, primary, prefill, tokens, n_threads=3)
        np.testing.assert_array_equal(d1, d3)
        for r in range(0, w.R, 7):
            h = orc.hash_prompt(tokens[r].tobytes(), tg.MODEL, w.block_size_tokens, w.max_prefix_blocks)
            m, _ = ix.match_longest_prefix(h, w.E)
            d = orc.schedule(primary, prefill, pool, m, len(h), w.block_size_tokens, w.prompt_bytes, w.non_cached_tokens)
            assert (d.status, d.pick, d.tie_count, d.prefill_pick, d.prefill_ran) == tuple(
                int(d1[k][r]) for k in ("status", "pick", "tie_count", "prefill_pick", "prefill_ran"))
            assert d.score == d1["score"][r] and t1[r] == len(h)


def test_every_switch_in_the_code_is_documented():
    """DESIGN.md section 12 lists every environment variable the library reads (and nothing else)."""
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    csrc = os.path.join(root, "llm-d-inference-scheduler_b200", "csrc")
    in_code = set()
    for f in os.listdir(csrc):
        if f.endswith((".cu", ".cuh", ".h")):
            in_code |= set(re.findall(r'getenv\("([A-Z0-9_]+)"\)', open(os.path.join(csrc, f)).read()))
    design = open(os.path.join(root, "DESIGN.md")).read()
    section = design[design.index("## 12. A/B switches"):]
    documented = set(re.findall(r"`(EPP_[A-Z0-9_]+)`", section))
    assert in_code == documented, (sorted(in_code - documented), sorted(documented - in_code))
