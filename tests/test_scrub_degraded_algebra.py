"""CPU: the scrub of a degraded stripe (fastecc_b200_rs_scrub_degraded, csrc/scrub.cu, api.cu, DESIGN 3j) restated in Python
integers on the helpers of test_scrub_algebra.py.  f blocks are known lost: their rows are never read (they hold garbage here),
the syndrome is weighted by the erasure locator cs_j = -l_E(y_j) / 2 of the repair pattern, the clean test and the locator check
start at f and f + L, and the roots at lost points do not count.  Checked: the four guarantees with M - f in place of M, and that
f = 0 is the plain scrub."""
import numpy as np
import pytest

from test_repair_algebra import pattern
from test_scrub_algebra import (CLEAN, DETECTED, LOCATED, ORDERS, P, berlekamp_massey, corrupt, divisors, dft, encode, fold, root, scrub,
                                stripe)


def erasure_scale(N, M, lost_data, lost_parity):
    """cs_j = -l_E(y_j) / 2, y_j = rho^(2Dj + 1), l_E = prod (x - rho^e) over E in the 2N-row numbering (what the pattern's d_cs
    holds): zero exactly on the lost parity rows"""
    rho, D = root(2 * N), N // M
    pts = [pow(rho, 2 * e, P) for e in lost_data] + [pow(rho, 2 * D * j + 1, P) for j in lost_parity]
    inv2 = pow(2, P - 2, P)
    out = []
    for j in range(M):
        y, l = pow(rho, 2 * D * j + 1, P), 1
        for z in pts:
            l = l * (y - z) % P
        out.append((P - l) * inv2 % P)
    return out


def scrub_degraded(data, parity, lost_data, lost_parity, max_bad, seed, size=None):
    """data: N rows, parity: M rows (the lost ones never read) -> (status, bad data blocks, bad parity blocks), survivors only"""
    N, M = len(data), len(parity)
    f = len(lost_data) + len(lost_parity)
    ld, lp = set(lost_data), set(lost_parity)
    cs = erasure_scale(N, M, lost_data, lost_parity)
    width = len(data[0]) if size is None else size
    live_d = [[0] * width if i in ld else row for i, row in enumerate(data)]            # a row that is never loaded folds to 0
    live_p = [[0] * width if j in lp else row for j, row in enumerate(parity)]
    zeta = root(M)
    zinv = pow(zeta, P - 2, P)
    u, U = [], []
    for fo in (0, 1):
        a, b = fold(live_d, seed, fo, size), fold(live_p, seed, fo, size)
        G = encode(a, M)
        u.append([(b[j] - G[j]) * cs[j] % P for j in range(M)])
        U.append(dft(u[fo], zinv))                                           # M * INTT_M(u)
    if not any(U[0][f:]) and not any(U[1][f:]):
        return CLEAN, [], []
    if max_bad == 0:
        return DETECTED, [], []
    Cz, L = berlekamp_massey(U[0][f:f + 2 * max_bad])
    if L > max_bad or len(Cz) - 1 != L:
        return DETECTED, [], []
    Chat = dft(Cz, zeta, M)                                                  # C(zeta^j)
    for fo in (0, 1):
        if any(dft([Chat[j] * u[fo][j] % P for j in range(M)], zinv)[f + L:]):
            return DETECTED, [], []
    bad_p = [j for j in range(M) if Chat[j] == 0 and cs[j]]
    rinv = pow(root(2 * N), P - 2, P)
    twisted = [c * pow(rinv, k, P) % P for k, c in enumerate(Cz)]
    bad_d = [i for i, v in enumerate(dft(twisted, root(N), N)) if v == 0 and i not in ld]
    if len(bad_d) + len(bad_p) != L:
        return DETECTED, [], []
    return LOCATED, bad_d, bad_p


def lose(N, M, f, kind, rng):
    """f lost blocks: data only, parity only (when f fits) or mixed"""
    if kind == "data" or (kind == "parity" and f > M):
        nd = f
    elif kind == "parity":
        nd = 0
    else:
        nd = int(rng.integers(max(0, f - M), f + 1))
    return sorted(rng.choice(N, size=nd, replace=False).tolist()), sorted(rng.choice(M, size=f - nd, replace=False).tolist())


def garble(data, parity, lost_data, lost_parity, rng):
    """Copies with random 32-bit garbage, different in every word, in the lost rows"""
    data, parity = [list(r) for r in data], [list(r) for r in parity]
    for rows, lost in ((data, lost_data), (parity, lost_parity)):
        for i in lost:
            rows[i] = [int(x) for x in rng.integers(0, 1 << 32, size=len(rows[i]))]
    return data, parity


def survivors_bad(N, M, lost_data, lost_parity, t, rng):
    """t corrupted blocks among the survivors, data and parity mixed"""
    sd = [i for i in range(N) if i not in set(lost_data)]
    sp = [j for j in range(M) if j not in set(lost_parity)]
    nd = int(rng.integers(max(0, t - len(sp)), min(t, len(sd)) + 1))
    return sorted(rng.choice(sd, size=nd, replace=False).tolist()), sorted(rng.choice(sp, size=t - nd, replace=False).tolist())


def f_values(M):
    """every f < M for small M, else the ends, the quarters and random ones"""
    if M <= 18:
        return list(range(M))
    return sorted({0, 1, 2, M // 4, M // 2, M - 3, M - 2, M - 1} | set(range(3, M - 3, max(1, M // 6))))


@pytest.mark.parametrize("N", ORDERS)
def test_the_four_guarantees_with_m_minus_f(N):
    rng = np.random.default_rng(400 + N)
    kinds = ("data", "parity", "mixed")
    cases = 0
    for M in divisors(N):
        data, parity = stripe(N, M, 2, rng)
        for f in f_values(M):
            kind = kinds[f % 3]
            lost_d, lost_p = lose(N, M, f, kind, rng)
            gd, gp = garble(data, parity, lost_d, lost_p, rng)
            room = M - f
            for max_bad in sorted({0, 1, room // 2} & set(range(room // 2 + 1))):
                for t in sorted({0, 1, max_bad, max_bad + 1, room - max_bad, room} & set(range(room + 1))):
                    bd, bp = survivors_bad(N, M, lost_d, lost_p, t, rng)
                    cd, cp = corrupt(gd, gp, bd, bp, rng, one_word=t % 2 == 1)
                    seed = int(rng.integers(1 << 63))
                    got = scrub_degraded(cd, cp, lost_d, lost_p, max_bad, seed)
                    why = (N, M, f, kind, lost_d, lost_p, max_bad, t, bd, bp, got)
                    cases += 1
                    if t == 0:
                        assert got == (CLEAN, [], []), why
                    else:
                        assert got[0] != CLEAN, why
                    if 1 <= t <= max_bad:
                        assert got == (LOCATED, bd, bp), why
                    elif max_bad < t <= room - max_bad:
                        assert got == (DETECTED, [], []), why
                    assert not set(got[1]) & set(lost_d) and not set(got[2]) & set(lost_p), why
                    if f == 0:
                        assert got == scrub(cd, cp, max_bad, seed), why
    assert cases > 0


@pytest.mark.parametrize("N,M", [(4, 4), (8, 4), (12, 6), (24, 8), (18, 9)])
def test_the_erasure_scale_is_the_repair_patterns(N, M):
    """cs_j here equals the d_cs that the repair pattern stores (test_repair_algebra.pattern), zero exactly on the lost parity"""
    rng = np.random.default_rng(N + M)
    for f in range(M + 1):
        lost_d, lost_p = lose(N, M, f, "mixed", rng)
        cs = erasure_scale(N, M, lost_d, lost_p)
        assert cs == [t[0] for t in pattern(N, M, lost_d, lost_p)[0]]
        assert [j for j in range(M) if cs[j] == 0] == lost_p


def test_the_lost_rows_are_never_read():
    """Two different garbage fillings of the lost rows, and all ones, give the same result"""
    rng = np.random.default_rng(7)
    N, M = 24, 12
    data, parity = stripe(N, M, 3, rng)
    lost_d, lost_p = [3, 17, 20], [0, 5]
    cd, cp = corrupt(data, parity, [9], [7], rng)
    fillings = [garble(cd, cp, lost_d, lost_p, rng) for _ in range(2)]
    fillings.append(([[(1 << 32) - 1] * 3 if i in lost_d else r for i, r in enumerate(cd)],
                     [[(1 << 32) - 1] * 3 if j in lost_p else r for j, r in enumerate(cp)]))
    for gd, gp in fillings:
        assert scrub_degraded(gd, gp, lost_d, lost_p, 2, 11) == (LOCATED, [9], [7])


def test_a_degraded_stripe_the_plain_scrub_cannot_handle():
    """M = 4 with f = 2 lost and one corrupted survivor: located here.  The plain scrub sees three bad blocks, more than its
    largest max_bad of M / 2 = 2, and cannot name them; with one check symbol left (f = 3) a bad survivor is still detected."""
    rng = np.random.default_rng(8)
    N, M = 8, 4
    data, parity = stripe(N, M, 4, rng)
    lost_d, lost_p = [2], [1]
    gd, gp = garble(data, parity, lost_d, lost_p, rng)
    cd, cp = corrupt(gd, gp, [6], [], rng)
    assert scrub_degraded(cd, cp, lost_d, lost_p, 1, 3) == (LOCATED, [6], [])
    plain = scrub(cd, cp, 2, 3)
    assert plain != (LOCATED, [2, 6], [1]) and len(plain[1]) + len(plain[2]) < 3
    assert scrub_degraded(gd, gp, lost_d, lost_p, 1, 3) == (CLEAN, [], [])
    lost_d3 = [2, 5]
    gd3, gp3 = garble(data, parity, lost_d3, lost_p, rng)
    assert scrub_degraded(gd3, gp3, lost_d3, lost_p, 0, 4) == (CLEAN, [], [])
    cd3, cp3 = corrupt(gd3, gp3, [], [3], rng)
    assert scrub_degraded(cd3, cp3, lost_d3, lost_p, 0, 4) == (DETECTED, [], [])


def test_pad_words_are_not_folded():
    """Rows of 5 words padded to 8 with garbage: scrubbed as their 5 words; the same rows over all 8 words are not clean"""
    rng = np.random.default_rng(10)
    N, M = 18, 6
    data, parity = stripe(N, M, 5, rng)
    pad_d = [r + [int(x) for x in rng.integers(0, 1 << 32, size=3)] for r in data]
    pad_p = [r + [int(x) for x in rng.integers(0, 1 << 32, size=3)] for r in parity]
    lost_d, lost_p = [4], [2, 3]
    gd, gp = garble(pad_d, pad_p, lost_d, lost_p, rng)
    assert scrub_degraded(gd, gp, lost_d, lost_p, 1, 1, size=5) == (CLEAN, [], [])
    cd = [list(r) for r in gd]
    cd[11][4] = (cd[11][4] + 5) % P
    assert scrub_degraded(cd, gp, lost_d, lost_p, 1, 2, size=5) == (LOCATED, [11], [])
    assert scrub_degraded(gd, gp, lost_d, lost_p, 1, 1)[0] != CLEAN
