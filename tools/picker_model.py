"""CPU restatement of the engine's random pickers (include/epp_engine.h, "Random pickers"; DESIGN §4.10).

Python floats are IEEE binary64 with round-to-nearest-even, so every sum below is the double the kernels compute: the
model is bit-exact, not approximate.  The engine's pick for one profile of one request is

    draw(picker, cands, base, score, explicit, seed, key, weights)

cands     the profile's candidates in ascending slot order (after an affinity filter that narrowed nothing)
base      slot -> weighted score with no match (what the pool kernels precompute; the gaps' masses come from it)
score     slot -> the request's weighted score
explicit  slots whose score depends on the request (matchBlocks > 0, or the request's LoRA adapter resident there)
gaps      False when the affinity filter narrowed the set: every candidate is explicit
"""
from __future__ import annotations

import math

M64 = (1 << 64) - 1
PICK_DOMAIN = 0xE7037ED1A0B428DB
MAX_SCORE, RANDOM, WEIGHTED_RANDOM = 0, 1, 2


def mix64(z: int) -> int:
    z = (z + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def pick_u(seed: int, key: int) -> float:
    return (mix64((seed ^ PICK_DOMAIN) ^ mix64(key)) >> 11) * 2.0 ** -53


def pick_rank(u: float, n: int) -> int:
    return min(int(u * n), n - 1)


def mass_scale(weights) -> float:
    s = 0.0
    for w in weights:
        s = s + abs(w)
    return 2.0 ** -128 if s > 2.0 ** 960 else 1.0


def mass_of(s: float, sigma: float) -> float:
    return s * sigma if (s > 0.0 and s != math.inf) else 0.0


def prefix(cands, base, sigma):
    """wcum / icum of k_pool_cum: left folds over the candidates' bases."""
    wcum, icum = [0.0], [0]
    acc, ic = 0.0, 0
    for c in cands:
        acc = acc + mass_of(base[c], sigma)
        ic += 1 if base[c] == math.inf else 0
        wcum.append(acc)
        icum.append(ic)
    return wcum, icum


def _walk(items, n, wcum, icum, cands, gaps, mode, t=0.0, k=0):
    """items: (position, mass, is_inf, slot) in ascending slot order.  Returns (S, ninf, pick)."""
    S, ninf, a = 0.0, 0, 0

    def gap(b):
        nonlocal S, ninf, k
        if not gaps or b <= a:
            return None
        if mode == 2:
            c = icum[b] - icum[a]
            if k < c:
                lo, hi = a, b - 1
                while lo < hi:
                    mid = (lo + hi) >> 1
                    if icum[mid + 1] - icum[a] > k:
                        hi = mid
                    else:
                        lo = mid + 1
                return cands[lo]
            k -= c
            return None
        wa = wcum[a]
        ns = S + (wcum[b] - wa)
        if mode == 1 and ns > t:
            lo, hi = a, b - 1
            while lo < hi:
                mid = (lo + hi) >> 1
                if S + (wcum[mid + 1] - wa) > t:
                    hi = mid
                else:
                    lo = mid + 1
            return cands[lo]
        S = ns
        if mode == 0:
            ninf += icum[b] - icum[a]
        return None

    for pos, m, inf, e in items:
        p = gap(pos)
        if p is not None:
            return S, ninf, p
        a = pos + 1
        if mode == 2:
            if inf:
                if k == 0:
                    return S, ninf, e
                k -= 1
            continue
        ns = S + m
        if mode == 1 and ns > t:
            return S, ninf, e
        S = ns
        if mode == 0:
            ninf += 1 if inf else 0
    p = gap(n)
    return S, ninf, p


def draw(picker, cands, base, score, explicit, seed, key, weights, gaps=True, out=()):
    """(pick, pick's score, population size) of one profile, or (None, 0.0, 0) without candidates.  out: endpoints
    already emitted into the request's first-k list -- explicit items of mass 0, outside the population."""
    out = set(out)
    pop = [c for c in cands if c not in out]
    n = len(pop)
    if n == 0:
        return None, 0.0, 0
    u = pick_u(seed, key)
    if picker == RANDOM:
        pick = pop[pick_rank(u, n)]
        return pick, score[pick], n
    sigma = mass_scale(weights)
    wcum, icum = prefix(cands, base, sigma) if gaps else ([0.0], [0])
    items = [(i, 0.0 if c in out else mass_of(score[c], sigma), c not in out and score[c] == math.inf, c)
             for i, c in enumerate(cands) if (not gaps or c in explicit or c in out)]
    W, ninf, _ = _walk(items, len(cands), wcum, icum, cands, gaps, 0)
    if ninf:
        _, _, pick = _walk(items, len(cands), wcum, icum, cands, gaps, 2, k=pick_rank(u, ninf))
    elif not W > 0.0:
        pick = pop[pick_rank(u, n)]
    else:
        t = u * W
        if t >= W:
            t = math.nextafter(W, 0.0)
        _, _, pick = _walk(items, len(cands), wcum, icum, cands, gaps, 1, t=t)
    return pick, score[pick], n


GOLDEN = 0x9E3779B97F4A7C15


def draw_k(picker, cands, base, score, explicit, seed, key, weights, k, gaps=True):
    """The first k endpoints (epp_config.pick_k > 1): successive draws without replacement, draw j with the seed
    seed + j * 0x9E3779B97F4A7C15.  Returns [(pick, score)] of min(k, len(cands)) entries; entry 0 is draw()'s pick."""
    picks = []
    for j in range(min(k, len(cands))):
        p, s, _ = draw(picker, cands, base, score, explicit, (seed + j * GOLDEN) & M64, key, weights, gaps,
                       out=[q for q, _ in picks])
        picks.append((p, s))
    return picks
