"""The engine's random-picker and weighted-random-picker draw (include/epp_engine.h "Random pickers", DESIGN §4.10), as
restated in tools/picker_model.py: the reference's own known-answer tests re-encoded with request ordinals in place of
iterations, a second restatement written independently (item list built first, gaps searched linearly) compared pick
for pick on random landscapes and every rounding edge, and chi-square tests with fixed seeds against s_i / W and against
a literal A-Res restatement of weightedrandom/picker.go:121-154.  No GPU needed."""
import math

import numpy as np
import pytest

from tools import picker_model as PM

N_DRAWS = 10000
SEED = 0x1234_5678_9ABC_DEF1


def _flat(scores, picker, n_draws=N_DRAWS, seed=SEED):
    """Endpoints 0..n-1, no match anywhere: every candidate sits in one gap (the common cold request)."""
    cands = list(range(len(scores)))
    base = dict(enumerate(scores))
    return [PM.draw(picker, cands, base, base, set(), seed, 4 * i, [1.0])[0] for i in range(n_draws)]


# weightedrandom/picker_test.go:51-84 (cases) and :92-107 (expected probability s_i / sum, tolerance 5 %)
@pytest.mark.parametrize("scores", [[10, 90], [100, 100, 100], [30, 0], [100, 90, 50, 30, 20]])
def test_weighted_reference_kats(scores):
    picks = _flat([float(s) for s in scores], PM.WEIGHTED_RANDOM)
    total = float(sum(scores))
    for i, s in enumerate(scores):
        got = picks.count(i) / N_DRAWS
        assert abs(got - s / total) <= 0.05, (scores, i, got)


# random/picker_test.go:47-85: one endpoint out of the candidates, every candidate reachable, uniform
@pytest.mark.parametrize("n", [1, 2, 3, 7])
def test_random_reference_kats(n):
    picks = _flat([10.0 * (i + 1) for i in range(n)], PM.RANDOM)
    for i in range(n):
        assert abs(picks.count(i) / N_DRAWS - 1.0 / n) <= 0.05


def test_every_tie_seed_draws():
    """tie_seed 0 is not a deterministic mode for a configured random picker."""
    picks = _flat([1.0] * 8, PM.RANDOM, n_draws=400, seed=0)
    assert len(set(picks)) == 8


# ------------------------------------------------------------------------------------------------
# an independent restatement
# ------------------------------------------------------------------------------------------------
def _splitmix(x):
    x = (x + 0x9E3779B97F4A7C15) % 2 ** 64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) % 2 ** 64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) % 2 ** 64
    return x ^ (x >> 31)


def restated(picker, cands, base, score, explicit, seed, key, weights, out=()):
    pop = [c for c in cands if c not in out]
    n = len(pop)
    u = (_splitmix((seed ^ 0xE7037ED1A0B428DB) ^ _splitmix(key)) >> 11) / 2.0 ** 53
    sw = 0.0
    for w in weights:
        sw += abs(w)
    sigma = 2.0 ** -128 if sw > 2.0 ** 960 else 1.0

    def mass(s):
        return s * sigma if 0.0 < s < math.inf else 0.0

    def rank(m):
        return min(int(u * m), m - 1)

    def xmass(i):
        return 0.0 if cands[i] in out else mass(score[cands[i]])

    if picker == PM.RANDOM:
        return pop[rank(n)]
    wc = [0.0]
    for c in cands:
        wc.append(wc[-1] + mass(base[c]))
    seq, a = [], 0                                      # ("gap", a, b) / ("x", i)
    for i, c in enumerate(cands):
        if c in explicit or c in out:
            if i > a:
                seq.append(("gap", a, i))
            seq.append(("x", i))
            a = i + 1
    if a < len(cands):
        seq.append(("gap", a, len(cands)))
    infs = [i for i, c in enumerate(cands) if c not in out and (score[c] if c in explicit else base[c]) == math.inf]
    if infs:
        return cands[infs[rank(len(infs))]]
    W = 0.0
    for it in seq:
        W = W + (wc[it[2]] - wc[it[1]] if it[0] == "gap" else xmass(it[1]))
    if W == 0.0:
        return pop[rank(n)]
    t = u * W
    if t >= W:
        t = math.nextafter(W, 0.0)
    S = 0.0
    for it in seq:
        if it[0] == "x":
            if S + xmass(it[1]) > t:
                return cands[it[1]]
            S = S + xmass(it[1])
            continue
        _, ga, gb = it
        for i in range(ga, gb):                          # linear, where the model searches
            if S + (wc[i + 1] - wc[ga]) > t:
                return cands[i]
        S = S + (wc[gb] - wc[ga])
    raise AssertionError("the draw ran off the sequence")


def _landscape(rng, E, kind):
    cands = sorted(rng.choice(E, size=int(rng.integers(1, E + 1)), replace=False).tolist())
    base, score = {}, {}
    for c in cands:
        b = float(rng.choice([0.0, -1.0, rng.random() * 7.0, rng.random() * 1e-3]))
        if kind == "subnormal":
            b = float(rng.integers(0, 5)) * 5e-324
        if kind == "huge":
            b = float(rng.random()) * 1.5e308
        base[c] = b
        score[c] = b
    explicit = set()
    if kind == "all_explicit":
        explicit = set(cands)
    else:
        for c in cands:
            if rng.random() < 0.2:
                explicit.add(c)
    for pos in (0, len(cands) - 1):
        if rng.random() < 0.5:
            explicit.add(cands[pos])
    for c in explicit:
        s = float(rng.choice([rng.random() * 9.0, 0.0, -2.0, base[c]]))
        if kind == "inf" and rng.random() < 0.3:
            s = math.inf
        if kind == "huge":
            s = float(rng.random()) * 1.7e308
        score[c] = s
    if kind == "zero":
        base = {c: 0.0 for c in cands}
        score = {c: -1.0 if c in explicit else 0.0 for c in cands}
    if kind == "single":
        base = {c: 0.0 for c in cands}
        score = dict(base)
        one = cands[int(rng.integers(0, len(cands)))]
        base[one] = score[one] = 2.5
        explicit.discard(one)
    weights = [1.5e308, 1.5e308] if kind == "huge" else [2.0, 3.0]
    return cands, base, score, explicit, weights


@pytest.mark.parametrize("kind", ["plain", "inf", "zero", "single", "all_explicit", "subnormal", "huge"])
@pytest.mark.parametrize("E", [1, 31, 33, 70, 200])
def test_model_matches_the_restatement(kind, E):
    rng = np.random.default_rng(E * 101 + len(kind))
    for trial in range(60):
        cands, base, score, explicit, weights = _landscape(rng, E, kind)
        for picker in (PM.RANDOM, PM.WEIGHTED_RANDOM):
            for key in range(0, 40, 4):
                seed = int(rng.integers(0, 2 ** 63))
                got = PM.draw(picker, cands, base, score, explicit, seed, key, weights)
                want = restated(picker, cands, base, score, explicit, seed, key, weights)
                assert got[0] == want, (kind, E, trial, picker, key)
                assert got[2] == len(cands)
                if picker == PM.WEIGHTED_RANDOM and any(0.0 < score[c] for c in cands):
                    assert score[got[0]] > 0.0               # nothing of weight 0 is ever picked while W > 0


def test_t_rounding_to_w_stays_inside():
    """u close to 1: t = u * W rounds up to W; the pick must be the last positive item, not past the end."""
    cands = list(range(5))
    base = {0: 1.0, 1: 0.0, 2: 3.0, 3: 0.0, 4: 0.0}
    wcum, _ = PM.prefix(cands, base, 1.0)
    S, _, _ = PM._walk([], 5, wcum, [0] * 6, cands, True, 0)
    t = math.nextafter(S, 0.0)
    _, _, pick = PM._walk([], 5, wcum, [0] * 6, cands, True, 1, t=t)
    assert pick == 2


def test_chi_square_against_weights_and_a_res():
    """Pick counts of the CDF draw follow s_i / W; so do those of a literal A-Res (largest u^(1/s)) with a numpy RNG."""
    from scipy.stats import chisquare
    rng = np.random.default_rng(7)
    scores = [0.0, 4.0, 1.0, 0.5, 2.5, -1.0, 7.0, 3.0]
    pos = [i for i, s in enumerate(scores) if s > 0]
    p = np.array([scores[i] for i in pos]) / sum(scores[i] for i in pos)
    n = 40000
    picks = _flat(scores, PM.WEIGHTED_RANDOM, n_draws=n, seed=99)
    counts = np.bincount(picks, minlength=len(scores))
    assert counts[[i for i in range(len(scores)) if i not in pos]].sum() == 0
    assert chisquare(counts[pos], n * p).pvalue > 1e-3
    ares = np.zeros(len(scores), np.int64)
    for _ in range(n):                                     # weightedrandom/picker.go:121-154 with k = 1
        best, key_best = None, -1.0
        for i, s in enumerate(scores):
            if s <= 0:
                k = 0.0
            else:
                u = rng.random()
                k = (u if u != 0 else 1e-10) ** (1.0 / s)
            if k > key_best:
                best, key_best = i, k
        ares[best] += 1
    assert chisquare(ares[pos], n * p).pvalue > 1e-3
    # the two samplers agree with each other as well (two-sample chi-square on the positive endpoints)
    table = np.stack([counts[pos], ares[pos]])
    from scipy.stats import chi2_contingency
    assert chi2_contingency(table).pvalue > 1e-3


@pytest.mark.parametrize("kind", ["plain", "inf", "zero", "single", "all_explicit"])
@pytest.mark.parametrize("E", [33, 70])
def test_first_k_matches_the_restatement(kind, E):
    """Successive draws without replacement, up to 64 and past the positive set: draw j = the restatement with seed
    tie_seed + j * golden and the emitted endpoints out; pick 0 = the one-endpoint pick; no repeats; under the weighted
    picker every positive candidate comes before every candidate of mass 0."""
    rng = np.random.default_rng(E * 7 + len(kind))
    for trial in range(12):
        cands, base, score, explicit, weights = _landscape(rng, E, kind)
        for picker in (PM.RANDOM, PM.WEIGHTED_RANDOM):
            seed, key = int(rng.integers(0, 2 ** 63)), 4 * trial + 1
            got = PM.draw_k(picker, cands, base, score, explicit, seed, key, weights, 64)
            picks = [p for p, _ in got]
            assert len(picks) == min(64, len(cands)) and len(set(picks)) == len(picks)
            assert picks[0] == PM.draw(picker, cands, base, score, explicit, seed, key, weights)[0]
            for j, p in enumerate(picks):
                want = restated(picker, cands, base, score, explicit, (seed + j * 0x9E3779B97F4A7C15) % 2 ** 64, key,
                                weights, out=set(picks[:j]))
                assert p == want, (kind, E, trial, picker, j)
            if picker == PM.WEIGHTED_RANDOM and not any(score[c] == math.inf for c in cands):
                pos = [score[p] > 0.0 for p in picks]
                assert pos == sorted(pos, reverse=True)
