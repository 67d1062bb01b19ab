"""k_hash_fused looks up each window's leading block as soon as it is chained and examines the word at the end of the
same window (DESIGN.md section 4.1): a window proven absent is not stored, and a request closed at window c is done
once window c has been chained, so it reads at most one window past it.  With a bitmap of known size the bounds are
restated on the host: the stored rows are exactly [0, bound) (8 bytes per hash), and the bytes read lie between what
the bounds need and one window more.  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

from helpers import assert_decisions_equal
from test_hash_skip_gpu import ALL1, B, BB, BST, ENC, W, World, _engine, _oracle_profiles, _run

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


def _bounds(orc, world, prompts, model_idx, keys, log2bits):
    """Per request: bound (the first window start proven absent, else the partial block if it reads absent, else
    nblocks), the bytes a skipping read needs, and the most it may take (one window past the closing one)."""
    shift = 64 - log2bits
    bits = {int(k) >> shift for k in keys if int(k) != ALL1}

    def absent(h):
        return h != ALL1 and (h >> shift) not in bits

    bound = np.zeros(len(prompts), np.int64)
    lo = np.zeros(len(prompts), np.int64)
    hi = np.zeros(len(prompts), np.int64)
    for r, (p, i) in enumerate(zip(prompts, model_idx)):
        eff = 0 if len(p) < BB else min(len(p), BB * B)
        nfull = eff // BB
        h = orc.hash_prompt(p, world.models[i], BST, B) if nfull else []
        bound[r] = len(h)
        lo[r] = hi[r] = eff
        stop = next((b for b in range(0, nfull, W) if absent(h[b])), None)
        if stop is not None:
            c = stop // W
            bound[r] = stop
            lo[r] = min(nfull, (c + 1) * W) * BB
            hi[r] = min(nfull, (c + 2) * W) * BB
        elif len(h) > nfull and absent(h[nfull]):
            bound[r] = nfull
    return bound, lo, hi


@pytest.mark.parametrize("stages", [1, 3])
@pytest.mark.parametrize("seed", [5, 6])
def test_rows_end_at_the_bound_and_reads_one_window_past(epp, orc, monkeypatch, stages, seed):
    """Two models, 301 requests: holes at window starts, partial-block stops, cold prompts, prompts without a full
    block and past the block cap; one profile or the P/D + encode handler."""
    world = World(orc, seed, models=(b"m", b"other"))
    mm = (world.rng.random(len(world.prompts)) < 0.5).astype(np.uint8) if stages == 3 else None
    monkeypatch.setenv("EPP_PRESENCE_LOG2BITS", "20")
    monkeypatch.setenv("EPP_HASH_SKIP", "1")
    eng, mids = _engine(epp, world, stages)
    with eng:
        eng.index_load_snapshot(world.hs, world.es)
        dec, det = _run(epp, eng, mids, world.prompts, world.model_idx, mm)
        st = eng.stats()
    odec, ototal = world.oracle(orc, world.prompts, world.model_idx, _oracle_profiles(orc, stages), 4 if stages > 1 else 0,
                                0, mm, orc.make_profile(3, ENC) if stages == 3 else None)
    assert_decisions_equal(dec, det, odec, ototal, where=f"stages {stages} seed {seed}")
    bound, lo, hi = _bounds(orc, world, world.prompts, world.model_idx, world.hs, 20)
    assert st["last_hash_bytes_stored"] == 8 * bound.sum()
    assert lo.sum() <= st["last_prompt_bytes_read"] <= hi.sum(), (lo.sum(), st["last_prompt_bytes_read"], hi.sum())
    assert (bound < np.array([len(p) // BB for p in world.prompts])).sum() > 50       # most requests close early

