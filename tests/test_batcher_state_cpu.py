"""The flush replay of tests/batcher_replay.py on synthetic ticket lists, and the sensitivity guard of the batcher state
tests on the models alone: on each landscape those tests use, two different groupings of the same rows give different
decisions, so a batcher that grouped, ordered or ordinal-numbered its flushes wrongly cannot pass them."""
import numpy as np
import pytest

import batcher_replay as BR


def T(seq, idx):
    return (seq << 20) | idx


def test_grouping_follows_seq_then_idx():
    tickets = {"a": T(3, 1), "b": T(2, 0), "c": T(3, 0), "d": T(4, 0), "e": T(2, 1), "f": T(2, 2)}
    fl = BR.flushes(tickets)
    assert fl == [(2, ["b", "e", "f"]), (3, ["c", "a"]), (4, ["d"])]
    assert BR.sizes(fl) == [3, 2, 1]
    assert BR.with_bases(fl, 100) == [(2, ["b", "e", "f"], 100), (3, ["c", "a"], 103), (4, ["d"], 105)]


def test_a_failed_flush_takes_no_ordinals():
    fl = BR.flushes([T(0, 0), T(0, 1), T(1, 0), T(1, 1), T(1, 2), T(2, 0)])
    assert BR.with_bases(fl, 7, failed={1}) == [(0, [0, 1], 7), (1, [2, 3, 4], 9), (2, [5], 9)]
    assert BR.with_bases(fl, 7, failed={0, 2}) == [(0, [0, 1], 7), (1, [2, 3, 4], 7), (2, [5], 10)]


def test_a_refused_submit_reserves_no_row():
    # row 2's submit was refused (no ticket): row 3 took the next index of the same flush
    fl = BR.flushes([T(5, 0), T(5, 1), None, T(5, 2), T(6, 0)])
    assert fl == [(5, [0, 1, 3]), (6, [4])]
    assert BR.with_bases(fl, 0) == [(5, [0, 1, 3], 0), (6, [4], 3)]


def test_gaps_and_duplicates_are_refused():
    with pytest.raises(AssertionError):
        BR.flushes([T(0, 0), T(0, 2)])                    # row 1 reserved but its ticket missing
    with pytest.raises(AssertionError):
        BR.flushes([T(0, 0), T(0, 0)])                    # one ticket for two rows
    with pytest.raises(AssertionError):
        BR.flushes([T(0, 0), T(2, 0)])                    # flush 1 missing
    assert BR.flushes([T(0, 0), T(2, 0)], contiguous=False) == [(0, [0]), (2, [1])]


def test_single_is_request_order_at_the_first_ordinal():
    assert BR.single([4, 1, 3], 11) == [(0, [1, 3, 4], 11)]


def _groupings(R, first, step, seed):
    """The rows in a shuffled order cut into flushes of 1 .. step rows (what concurrent submitters produce), and the
    same rows as one flush in request order."""
    rng = np.random.default_rng(seed)
    order = [int(x) for x in rng.permutation(R)]
    plan, i, b = [], 0, first
    while i < R:
        n = int(rng.integers(1, step + 1))
        plan.append((len(plan), order[i:i + n], b))
        b += len(order[i:i + n])
        i += n
    return plan, BR.single(range(R), first)


@pytest.fixture(scope="module")
def tg():
    from tools import tracegen
    tracegen.build()
    return tracegen


def test_guard_pd_seeded_ties_with_prerequest(orc, tg):
    """Scenario 1's landscape: PreRequest between flushes and the seeded tie rule change picks with the grouping."""
    w, tokens, pool = BR.pd_landscape(tg, R=640)
    R = tokens.shape[0]
    plan, one = _groupings(R, 0, 48, 1)
    a, ixa = BR.pd_replay(orc, tg, w, tokens, pool, plan)
    b, ixb = BR.pd_replay(orc, tg, w, tokens, pool, one)
    picks = lambda d: np.array([(int(d[r][0]["pick"]), int(d[r][0]["prefill_pick"]), d[r][2]) for r in range(R)])  # noqa: E731
    pa, pb = picks(a), picks(b)
    assert (pa != pb).any(axis=1).sum() > R // 20
    assert sum(a[r][2] > 0 for r in range(R)) > R // 10            # later flushes match what earlier ones indexed
    assert sum(int(a[r][0]["tie_count"]) > 1 for r in range(R)) > R // 4
    # the same grouping without PreRequest: only the tie rule's keys stay the same
    c, _ = BR.pd_replay(orc, tg, w, tokens, pool, plan, index_picks=False)
    assert (picks(c) != pa).any(axis=1).sum() > R // 20
    # PreRequest indexed other picks: the two indexes differ in their (hash, endpoint) pairs
    pairs = lambda ix: set(zip(*(a.tolist() for a in ix.export())))      # noqa: E731
    assert pairs(ixa) != pairs(ixb)


@pytest.mark.parametrize("picker", [1, 2])
def test_guard_random_pickers(orc, picker):
    """Scenario 2's landscape: each draw is keyed by the row's ordinal, so an order other than the flushes' moves
    picks (the pickers keep no other state)."""
    from tools import picker_model as PM
    assert picker in (PM.RANDOM, PM.WEIGHTED_RANDOM)
    world = BR.PickerWorld(orc, R=300)
    plan, one = _groupings(world.R, 5, 12, 2)
    a, b = BR.picker_replay(world, picker, plan), BR.picker_replay(world, picker, one)
    diff = sum(a[r][0] != b[r][0] or a[r][4] != b[r][4] for r in range(world.R))
    assert diff > world.R // 4
    assert any(a[r][3] > 0 for r in range(world.R))


def test_guard_inflight_counters(orc, tg):
    """Scenario 4's landscape: each flush reads the counters every earlier flush left."""
    import helpers
    from tools import inflight_model as M
    w, trace = BR.inflight_landscape(tg, R=320)
    tokens = trace.requests()[0]
    _, ix, _, _, _ = helpers.setup_oracle(orc, w, trace)
    plan, one = _groupings(w.R, 0, 32, 3)
    ca, cb = M.Counters(w.E), M.Counters(w.E)
    a = BR.inflight_replay(orc, tg, w, trace, ix, ca, plan, tokens)
    b = BR.inflight_replay(orc, tg, w, trace, ix, cb, one, tokens)
    diff = sum(int(a[r][0]["pick"]) != int(b[r][0]["pick"]) for r in range(w.R))
    assert diff > w.R // 10
    # every row added once whatever the grouping: the same totals, spread over other endpoints
    assert ca.req.sum() == cb.req.sum() == w.R and ca.tok.sum() == cb.tok.sum()
    assert (ca.req != cb.req).any()


@pytest.mark.parametrize("picker", [0, 2])
def test_guard_nohit_lru(orc, picker):
    """Scenario 3's landscape: cold rows read the LRU every earlier flush left (and max-score's seeded ties and the
    weighted draw read the ordinal); the LRU evicts between flushes."""
    world = BR.PickerWorld(orc, E=96, R=480)
    plan, one = _groupings(world.R, 0, 16, 4)
    ma, mb = BR.nohit_model(orc, world, picker), BR.nohit_model(orc, world, picker)
    a, b = BR.nohit_replay(ma, world, plan), BR.nohit_replay(mb, world, one)
    cold = sum(a[r][5] for r in range(world.R))
    assert cold > 3 * BR.NOHIT_LRU                                  # far more cold picks than the LRU holds
    assert sum(a[r][1] != b[r][1] or a[r][2] != b[r][2] for r in range(world.R)) > world.R // 20
    # the same order cut into other flushes: only the LRU state each flush starts from differs
    c = BR.nohit_replay(BR.nohit_model(orc, world, picker), world, [(0, rows, base) for _, rows, base in plan[:len(plan) // 2]] +
                        [(1, [r for _, rows, _ in plan[len(plan) // 2:] for r in rows], plan[len(plan) // 2][2])])
    assert any(a[r][1] != c[r][1] or a[r][2] != c[r][2] for r in c)


def test_guard_admitters(orc, tg):
    """Scenario 5's landscape: the probabilistic draws follow each row's ordinal, and the index only holds the picks of
    admitted rows of earlier flushes."""
    from tools import admission_model as am
    w, tokens, pool, cfg, rows = BR.admit_landscape(tg, orc)
    plan, one = _groupings(w.R, 0, 16, 5)
    a, ixa, ca = BR.admit_replay(orc, tg, am, w, tokens, pool, cfg, rows, plan)
    b, ixb, cb = BR.admit_replay(orc, tg, am, w, tokens, pool, cfg, rows, one)
    st = lambda d: np.array([int(d[r][0]["status"]) for r in range(w.R)])     # noqa: E731
    sa, sb = st(a), st(b)
    rej = sa == am.STATUS_REJECTED
    assert w.R // 8 < rej.sum() < w.R // 2
    assert (sa != sb).sum() > w.R // 20                            # other ordinals, other draws
    assert ca.req.sum() == (sa == 0).sum() and cb.req.sum() == (sb == 0).sum()
    # a row the latency-slo-admitter rejects whatever its draw: sheddable, an SLO, predictions none of them valid
    assert any(rows["priority"][r] < 0 and rows["preds"][r] is not None and not any(v == 3 for v in rows["valid"][r])
               and (rows["ttft"][r] > 0 or rows["tpot"][r] > 0) and sa[r] == am.STATUS_REJECTED for r in range(w.R))
    picks = lambda d: [int(d[r][0]["pick"]) for r in range(w.R) if sa[r] == 0 and sb[r] == 0]   # noqa: E731
    assert picks(a) != picks(b) or len(ixa.export()[0]) != len(ixb.export()[0])
