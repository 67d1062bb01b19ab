"""CPU checks of the no-hit-lru restatement (tools/nohit_lru_model.py): the reference's own tests
(scorer/nohitlru/no_hit_lru_test.go) re-encoded, and the device update's sequence-number algorithm against sequential
golang-lru Adds."""
import random

import numpy as np
import pytest

from tools import nohit_lru_model as M


# no_hit_lru_test.go:158-175 "cold request - all endpoints never used"
def test_score_table_cold_never_used():
    assert list(M.cold_column([0, 1, 2], [], 3)) == [1.0, 0.5, 0.0]


# no_hit_lru_test.go:176-194 "cache hit - neutral scores": one warm endpoint makes the request warm for every candidate
def test_score_table_cache_hit_is_warm():
    assert not M.is_cold([0, 1, 2], [3, 0, 0])
    assert M.is_cold([0, 1, 2], [0, 0, 0])


# no_hit_lru_test.go:195-208 "single endpoint - max score", and :396-402 (edge case)
def test_score_table_single_endpoint():
    assert list(M.cold_column([0], [], 1)) == [1.0]
    assert list(M.cold_column([0], [0], 1)) == [1.0]


# no_hit_lru_test.go:249-262: no prefix attribute at all counts as cold
def test_no_match_info_is_cold():
    assert M.is_cold([0], [0])


# no_hit_lru_test.go:378-394: an empty candidate list scores nobody
def test_empty_candidates():
    assert not M.cold_column([], [0, 1], 2).any()


# no_hit_lru_test.go:264-372 TestNoHitLRUPreferLeastRecentlyUsedAfterColdRequests
def test_prefer_least_recently_used_after_cold_requests():
    lru = M.GoLRU(1024)
    a, b, c = 0, 1, 2

    def best():
        col = M.cold_column([a, b, c], lru.keys(), 3)
        return int(np.argmax(col)), col

    assert best()[0] == a                   # :322-327 initial cold request seeds the cache
    lru.add(a)
    e, col = best()                         # :329-341 unused endpoints rank above existing ones
    assert e == b and col[b] == 1.0 and col[c] == 0.5 and col[b] > col[a]
    assert not M.is_cold([a, b, c], [1, 0, 0])     # :343-357 a warm request leaves the LRU untouched
    assert best()[0] == b
    lru.add(b)                              # :359-364 second cold request rotates to endpointB
    assert best()[0] == c
    lru.add(c)                              # :366-371 third cold request rotates back to endpointA
    assert best()[0] == a


# no_hit_lru_test.go:405-450 TestNoHitLRUPrefillDecodeTracking (P/D: decode and prefill targets both Added)
def test_prefill_decode_tracking():
    pa, pb, da, db = 0, 1, 2, 3
    lru = M.GoLRU(0)
    lru.add(da)                              # primary target first, then the "prefill" target (:307-312)
    lru.add(pa)
    assert lru.keys() == [da, pa]
    pre = M.cold_column([pa, pb], lru.keys(), 4)
    dec = M.cold_column([da, db], lru.keys(), 4)
    assert pre[pb] > pre[pa] and dec[db] > dec[da]
    lru2 = M.GoLRU(0)                        # :452-470 non-P/D: only the primary target
    lru2.add(da)
    dec = M.cold_column([da, db], lru2.keys(), 4)
    assert dec[db] > dec[da]


def test_clamp_for_members_outside_the_candidates():
    """lruPos counts every LRU member, candidates or not (:211-229), so used candidates can clamp to 0."""
    col = M.cold_column([4, 5, 6], [0, 1, 2, 3, 4, 5], 8)
    assert col[6] == 1.0 and col[4] == 0.0 and col[5] == 0.0


def test_golang_lru_capacity():
    lru = M.GoLRU(2)
    for k in (1, 2, 1, 3):
        lru.add(k)
    assert lru.keys() == [1, 3]


@pytest.mark.parametrize("lru_size", [1, 3, 8, 1024])
@pytest.mark.parametrize("seed", range(4))
def test_sequence_number_update_equals_sequential_adds(lru_size, seed):
    """The device update (atomicMax of seq0 + 2r + k, then keep the lru_size newest) equals golang-lru Adds in request
    order, call after call."""
    rnd = random.Random(seed)
    E = 12
    calls = []
    for _ in range(20):
        R = rnd.randint(1, 10)
        adds = []
        for r in range(R):
            if rnd.random() < 0.6:
                adds.append((r, 0, rnd.randrange(E)))
                if rnd.random() < 0.5:
                    adds.append((r, 1, rnd.randrange(E)))
        calls.append(adds)
    got = M.device_update([0] * E, calls, lru_size)
    lru = M.GoLRU(lru_size)
    for adds, g in zip(calls, got):
        for _, _, e in sorted(adds):
            lru.add(e)
        assert g == lru.keys()
