"""The device matcher's tie-break (crit_match_kernel, csrc/criterion.cu) against scipy.optimize.linear_sum_assignment, on an
emulation of the kernel's loop: one warp's 32 lanes, each scanning its positions of `remaining`, then the shuffle reduction.

When reduced costs tie, several assignments are optimal and the gradients go to whichever queries the solver returns, so the
kernel must return scipy's.  scipy transposes the (query x target) matrix only when it has more rows than columns, scans the
unvisited columns in the order of its `remaining` array (reversed at first, a picked column replaced by the last entry), and
lets a later tied column displace the current pick only if it is free.  These tests require the same assignment on
tie-heavy problems -- integer costs, duplicated queries, duplicated targets, square and transposed -- and show that the rule
the kernel used before (free column first, then the lowest index; targets as rows when nt == nq) fails them.
"""
import numpy as np
import pytest
from scipy.optimize import linear_sum_assignment

INF = 1e300


def _pick_scipy(s, fr, k):
    """Lane-local scan (positions k rising): scipy's rule.  Returns the index into the lane's arrays or -1."""
    best, bi = INF, -1
    for n in range(len(k)):
        if s[n] < best or (s[n] == best and fr[n]):
            best, bi = s[n], n
    return bi


def _take_scipy(a, b):
    """Butterfly step: does candidate b = (cost, free, pos) replace a?"""
    if b[2] < 0:
        return False
    if a[2] < 0 or b[0] < a[0]:
        return True
    if b[0] != a[0]:
        return False
    if a[1] or b[1]:
        return bool(b[1] and (not a[1] or b[2] > a[2]))
    return b[2] < a[2]


def _take_old(a, b):
    if b[2] < 0:
        return False
    return a[2] < 0 or b[0] < a[0] or (b[0] == a[0] and (b[1] > a[1] or (b[1] == a[1] and b[2] < a[2])))


def emulate(cost, rule="scipy"):
    """cost: (nq, nt) fp32 matrix of one (image, group).  Returns match[target] = query, as the kernel writes it."""
    nq, nt = cost.shape
    rows_are_targets = nt < nq if rule == "scipy" else nt <= nq
    c = (cost.T if rows_are_targets else cost).astype(np.float64)
    R, Cn = c.shape
    u, v = np.zeros(R), np.zeros(Cn)
    col4row, row4col = np.full(R, -1), np.full(Cn, -1)
    path = np.full(Cn, -1)
    for cur in range(R):
        spc = np.full(Cn, INF)
        SR, SC = np.zeros(R, bool), np.zeros(Cn, bool)
        remaining = list(range(Cn - 1, -1, -1))
        minval, i, sink = 0.0, cur, -1
        while sink < 0:
            SR[i] = True
            # the scan order: positions of `remaining` (scipy) or the unvisited columns by index (old)
            order = remaining if rule == "scipy" else [j for j in range(Cn) if not SC[j]]
            for j in order:
                r = minval + c[i, j] - u[i] - v[j]
                if r < spc[j]:
                    spc[j], path[j] = r, i
            cands = []
            for lane in range(32):
                ks = list(range(lane, len(order), 32))
                s = [spc[order[k]] for k in ks]
                fr = [row4col[order[k]] < 0 for k in ks]
                if rule == "scipy":
                    n = _pick_scipy(s, fr, ks)
                    cands.append((s[n], fr[n], ks[n]) if n >= 0 else (INF, False, -1))
                else:                                   # lane-local: free first, then lowest j (scanned rising)
                    best, bf, bj = INF, False, -1
                    for sv, f, k in zip(s, fr, ks):
                        if sv < best or (sv == best and f > bf):
                            best, bf, bj = sv, f, k
                    cands.append((best, bf, bj))
            take = _take_scipy if rule == "scipy" else _take_old
            for o in (16, 8, 4, 2, 1):
                cands = [cands[l ^ o] if take(cands[l], cands[l ^ o]) else cands[l] for l in range(32)]
            best, _, k = cands[0]
            assert all(cd == cands[0] for cd in cands)          # every lane agrees
            assert k >= 0 and best < INF
            j = order[k]
            minval = best
            SC[j] = True
            if rule == "scipy":
                remaining[k] = remaining[-1]
                remaining.pop()
            if row4col[j] < 0:
                sink = j
            else:
                i = row4col[j]
        for r in range(R):
            if SR[r]:
                u[r] += minval if r == cur else minval - spc[col4row[r]]
        for j in range(Cn):
            if SC[j]:
                v[j] -= minval - spc[j]
        j = sink
        while True:
            r = path[j]
            row4col[j] = r
            j, col4row[r] = col4row[r], j
            if r == cur:
                break
    match = np.full(nt, -1)
    if rows_are_targets:
        for t in range(nt):
            match[t] = col4row[t]
    else:
        for t in range(nt):
            match[t] = row4col[t]
    return match


def scipy_match(cost):
    q, t = linear_sum_assignment(cost)
    match = np.full(cost.shape[1], -1)
    match[t] = q
    return match


def tie_problem(rng, nq, nt, kind):
    """A (nq, nt) fp32 cost matrix with exact ties by construction."""
    if kind == "int":
        c = rng.integers(0, 4, (nq, nt)).astype(np.float32)
    elif kind == "dup_rows":                            # duplicated queries
        base = rng.integers(0, 6, (max(1, nq // 2), nt)).astype(np.float32)
        c = base[rng.integers(0, base.shape[0], nq)]
    elif kind == "dup_cols":                            # duplicated targets
        base = rng.integers(0, 6, (nq, max(1, nt // 2))).astype(np.float32)
        c = base[:, rng.integers(0, base.shape[1], nt)]
    else:                                               # dyadic reals, duplicated both ways
        base = (rng.integers(0, 16, (max(1, nq // 2), max(1, nt // 2))) * 0.125).astype(np.float32)
        c = base[rng.integers(0, base.shape[0], nq)][:, rng.integers(0, base.shape[1], nt)]
    return np.ascontiguousarray(c)


def _problems(n, seed, max_side=12):
    rng = np.random.default_rng(seed)
    kinds = ("int", "dup_rows", "dup_cols", "dyadic")
    for e in range(n):
        nq = int(rng.integers(1, max_side + 1))
        shape = e % 3                                   # square, more targets than queries, more queries than targets
        nt = nq if shape == 0 else int(rng.integers(nq, max_side + 1)) if shape == 1 else int(rng.integers(1, nq + 1))
        yield tie_problem(rng, nq, nt, kinds[e % 4])


def _total(cost, match):
    return sum(float(cost[q, t]) for t, q in enumerate(match) if q >= 0)


def test_emulation_matches_scipy_on_ties():
    for cost in _problems(3000, 1):
        got, ref = emulate(cost), scipy_match(cost)
        assert np.array_equal(got, ref), (cost.shape, got, ref)


def test_emulation_matches_scipy_large():
    rng = np.random.default_rng(2)
    for kind, (nq, nt) in [("dup_rows", (300, 64)), ("dup_cols", (300, 64)), ("int", (64, 64)), ("dyadic", (50, 50))]:
        cost = tie_problem(rng, nq, nt, kind)
        assert np.array_equal(emulate(cost), scipy_match(cost)), kind


def test_old_rule_fails_on_ties():
    """Sharpness: the previous tie-break gives optimal but different assignments on the same problems."""
    n_diff = n = 0
    for cost in _problems(1000, 1):
        got, ref = emulate(cost, rule="old"), scipy_match(cost)
        assert _total(cost, got) == pytest.approx(_total(cost, ref))            # still an optimal assignment
        n_diff += not np.array_equal(got, ref)
        n += 1
    assert n_diff > n // 20, (n_diff, n)


def test_tie_free_problems_agree():
    """Without ties the rule is never consulted: both rules give scipy's (unique) assignment."""
    rng = np.random.default_rng(3)
    for e in range(60):
        nq, nt = int(rng.integers(1, 13)), int(rng.integers(1, 13))
        cost = rng.random((nq, nt)).astype(np.float32)
        ref = scipy_match(cost)
        assert np.array_equal(emulate(cost), ref) and np.array_equal(emulate(cost, rule="old"), ref)
