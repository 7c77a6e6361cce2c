"""CPU: the scrub of a stored stripe (fastecc_b200_rs_scrub, csrc/scrub.cu, DESIGN 3i) restated in Python integers, against the
encode by definition.  The fold weights are the header's: splitmix64 of the counter seed + (2c + f + 1) * golden, mod P.  The
steps are the library's: fold the columns of every row, syndromes against the encode of the folded data, Berlekamp-Massey on
the inverse order-M transform of fold 0, the check of C * S^ mod (z^M - 1) in both folds, and the roots of C at the parity
points (order-M transform) and the data points (order-N transform of C_k rho^-k)."""
import functools

import numpy as np
import pytest

from test_repair_algebra import P, C, root, encode_by_definition

M64 = (1 << 64) - 1
CLEAN, LOCATED, DETECTED = 0, 1, 2


def weight(seed, f, c):
    """r_f,c: the splitmix64 output for the counter seed + (2c + f + 1) * 0x9E3779B97F4A7C15, reduced mod P (include/fastecc_b200.h)"""
    z = (seed + (2 * c + f + 1) * 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return (z ^ (z >> 31)) % P


def fold(rows, seed, f, size=None):
    """a_m = sum_c r_f,c * row_m[c] mod P over the first SIZE words of every row (raw words taken mod P; words past SIZE are
    not read; SIZE = the row length by default)"""
    size = (len(rows[0]) if rows else 0) if size is None else size
    r = [weight(seed, f, c) for c in range(size)]
    return [sum(w * (x % P) for w, x in zip(r, row[:size])) % P for row in rows]


@functools.lru_cache(maxsize=None)
def lagrange(N):
    """T[d] = -2 / (N (rho^(2d+1) - 1)): parity j of the N -> N encode is sum_i data_i T[(j - i) mod N] (DESIGN 3h)"""
    rho = root(2 * N)
    return [(P - 2) * pow(N * (pow(rho, 2 * d + 1, P) - 1) % P, P - 2, P) % P for d in range(N)]


def encode(data, M):
    """The M parity words of the stripe's encode of one column (parity j' = row (N/M) j' of the N -> N encode)"""
    N = len(data)
    T, D = lagrange(N), N // M
    return [sum(x * T[(D * j - i) % N] for i, x in enumerate(data)) % P for j in range(M)]


def dft(x, z, n=None):
    """X_j = sum_k x_k z^(jk), j < n (n = len(x) by default; x zero-padded to n)"""
    n = n or len(x)
    pw = [1] * n
    for i in range(1, n):
        pw[i] = pw[i - 1] * z % P
    return [sum(x[k] * pw[j * k % n] for k in range(len(x))) % P for j in range(n)]


def berlekamp_massey(s):
    """The shortest C = 1 + c_1 z + ... + c_L z^L with sum_i c_i s_(k-i) = 0 for k in [L, len(s)): (C, L)"""
    Cz, B, L, m, b = [1], [1], 0, 1, 1
    for n in range(len(s)):
        d = s[n]
        for i in range(1, L + 1):
            d = (d + Cz[i] * s[n - i]) % P
        if d == 0:
            m += 1
            continue
        coef = d * pow(b, P - 2, P) % P
        T = list(Cz)
        Cz += [0] * max(0, len(B) + m - len(Cz))
        for i, v in enumerate(B):
            Cz[i + m] = (Cz[i + m] - coef * v) % P
        if 2 * L <= n:
            L, B, b, m = n + 1 - L, T, d, 1
        else:
            m += 1
    while len(Cz) > 1 and Cz[-1] == 0:
        Cz.pop()
    return Cz, L


def scrub(data, parity, max_bad, seed, size=None):
    """data: N rows, parity: M rows of at least SIZE raw words each -> (status, bad data blocks, bad parity blocks)"""
    N, M = len(data), len(parity)
    s = []
    for f in (0, 1):
        a, b = fold(data, seed, f, size), fold(parity, seed, f, size)
        G = encode(a, M)
        s.append([(b[j] - G[j]) % P for j in range(M)])
    if not any(s[0]) and not any(s[1]):
        return CLEAN, [], []
    if max_bad == 0:
        return DETECTED, [], []
    zeta = root(M)
    zinv = pow(zeta, P - 2, P)
    S = dft(s[0], zinv)[:2 * max_bad]                    # M * S^: the scale of the sequence does not change C
    Cz, L = berlekamp_massey(S)
    if L > max_bad or len(Cz) - 1 != L:
        return DETECTED, [], []
    Chat = dft(Cz, zeta, M)                              # C(zeta^j)
    for f in (0, 1):
        back = dft([Chat[j] * s[f][j] % P for j in range(M)], zinv)       # M * (C * S^ mod z^M - 1)
        if any(back[L:]):
            return DETECTED, [], []
    bad_p = [j for j in range(M) if Chat[j] == 0]
    rinv = pow(root(2 * N), P - 2, P)
    twisted = [c * pow(rinv, k, P) % P for k, c in enumerate(Cz)]
    bad_d = [i for i, v in enumerate(dft(twisted, root(N), N)) if v == 0]   # C(rho^-1 omega^i)
    if len(bad_d) + len(bad_p) != L:
        return DETECTED, [], []
    return LOCATED, bad_d, bad_p


def stripe(N, M, S, rng):
    """N data rows of S random words and the M parity rows of their encode, column by column"""
    data = [[int(x) for x in rng.integers(0, P, size=S)] for _ in range(N)]
    cols = [encode([row[c] for row in data], M) for c in range(S)]
    return data, [[cols[c][j] for c in range(S)] for j in range(M)]


def corrupt(data, parity, bad_d, bad_p, rng, one_word=False):
    """Copies with every word (or one word) of the listed blocks changed mod P"""
    data, parity = [list(r) for r in data], [list(r) for r in parity]
    for rows, bad in ((data, bad_d), (parity, bad_p)):
        for i in bad:
            cols = [int(rng.integers(len(rows[i])))] if one_word else range(len(rows[i]))
            for c in cols:
                rows[i][c] = (rows[i][c] + int(rng.integers(1, P))) % P
    return data, parity


def split_bad(N, M, t, rng, kind):
    """t corrupted blocks: data only, parity only or mixed"""
    if kind == "data" or (kind == "mixed" and M == 1):
        nd = min(t, N)
    elif kind == "parity":
        nd = max(0, t - M)
    else:
        nd = int(rng.integers(max(0, t - M), min(t, N) + 1))
    return sorted(rng.choice(N, size=nd, replace=False).tolist()), sorted(rng.choice(M, size=t - nd, replace=False).tolist())


ORDERS = [1, 2, 4, 8, 16, 3, 6, 12, 24, 48, 9, 18, 36, 72]


def divisors(N):
    return [m for m in range(1, N + 1) if N % m == 0]


@pytest.mark.parametrize("N", ORDERS)
def test_clean_stripes_are_clean(N):
    rng = np.random.default_rng(N)
    for M in divisors(N):
        data, parity = stripe(N, M, 3, rng)
        assert scrub(data, parity, M // 2, 7) == (CLEAN, [], [])
        raw_d = [[x + P if x < C else x for x in r] for r in data]       # raw words >= P congruent to the stored ones
        raw_p = [[x + P if x < C else x for x in r] for r in parity]
        assert scrub(raw_d, raw_p, 0, 8) == (CLEAN, [], [])


@pytest.mark.parametrize("N", ORDERS)
def test_up_to_max_bad_corrupted_blocks_are_located(N):
    rng = np.random.default_rng(100 + N)
    for M in divisors(N):
        data, parity = stripe(N, M, 3, rng)
        for max_bad in sorted({M // 2, min(1, M // 2)} - {0}):
            for t in range(1, max_bad + 1):
                for kind in ("data", "parity", "mixed"):
                    bad_d, bad_p = split_bad(N, M, t, rng, kind)
                    cd, cp = corrupt(data, parity, bad_d, bad_p, rng, one_word=kind == "mixed")
                    seed = int(rng.integers(1 << 63))
                    got = scrub(cd, cp, max_bad, seed)
                    assert got == (LOCATED, bad_d, bad_p), (N, M, max_bad, kind, bad_d, bad_p, got)


@pytest.mark.parametrize("N", ORDERS)
def test_beyond_max_bad_is_detected_and_never_clean(N):
    rng = np.random.default_rng(200 + N)
    for M in divisors(N):
        data, parity = stripe(N, M, 2, rng)
        for max_bad in sorted({0, M // 2, M // 4, 1} & set(range(M // 2 + 1))):
            for t in range(1, M + 1):
                bad_d, bad_p = split_bad(N, M, t, rng, "mixed")
                cd, cp = corrupt(data, parity, bad_d, bad_p, rng)
                status, gd, gp = scrub(cd, cp, max_bad, t)
                assert status != CLEAN, (N, M, t)
                if t <= max_bad:
                    assert (status, gd, gp) == (LOCATED, bad_d, bad_p), (N, M, max_bad, t)
                elif t <= M - max_bad:
                    assert status == DETECTED, (N, M, max_bad, t, bad_d, bad_p, gd, gp)


def test_the_same_seed_gives_the_same_result_and_weights_differ():
    rng = np.random.default_rng(5)
    data, parity = stripe(12, 6, 4, rng)
    cd, cp = corrupt(data, parity, [2, 7], [5], rng)
    assert scrub(cd, cp, 3, 99) == scrub(cd, cp, 3, 99) == (LOCATED, [2, 7], [5])
    w = [weight(s, f, c) for s in (0, 1, 1 << 63) for f in (0, 1) for c in range(64)]
    assert len(set(w)) == len(w) and all(0 <= x < P for x in w)


@pytest.mark.parametrize("N", [1, 2, 3, 6, 8, 9, 12, 18, 24])
def test_the_circulant_encode_is_the_encode_by_definition(N):
    rng = np.random.default_rng(300 + N)
    data = [int(x) for x in rng.integers(0, P, size=N)]
    full = encode_by_definition(data)
    for M in divisors(N):
        assert encode(data, M) == full[::N // M], (N, M)


def test_weights_match_splitmix64():
    """weight(seed, f, c) is the (2c + f + 1)-th output of a splitmix64 generator started at `seed`, reduced mod P"""
    def splitmix64(state):
        while True:
            state = (state + 0x9E3779B97F4A7C15) & M64
            z = state
            z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
            z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
            yield z ^ (z >> 31)
    for seed in (0, 12345, M64):
        g = splitmix64(seed)
        outs = [next(g) % P for _ in range(10)]
        assert outs == [weight(seed, i % 2, i // 2) for i in range(10)]


def test_pad_words_and_single_words_in_one_column():
    """A word changed in one column of one block is located; rows padded to 8 words with random garbage in the 3 pad words (a
    partial last 16-byte group) are scrubbed as their 5 words alone, and the garbage would change the result if it were read."""
    rng = np.random.default_rng(9)
    data, parity = stripe(18, 6, 5, rng)
    for col in range(5):
        cd = [list(r) for r in data]
        cd[11][col] = (cd[11][col] + 1) % P
        assert scrub(cd, parity, 3, col) == (LOCATED, [11], [])
        cp = [list(r) for r in parity]
        cp[4][col] ^= 1
        assert scrub(data, cp, 1, col) == (LOCATED, [], [4])
    pad_d = [r + [int(x) for x in rng.integers(0, 1 << 32, size=3)] for r in data]
    pad_p = [r + [int(x) for x in rng.integers(0, 1 << 32, size=3)] for r in parity]
    assert scrub(pad_d, pad_p, 3, 1, size=5) == (CLEAN, [], [])
    cd = [list(r) for r in pad_d]
    cd[2][4] = (cd[2][4] + 5) % P
    assert scrub(cd, pad_p, 3, 2, size=5) == (LOCATED, [2], [])
    assert scrub(pad_d, pad_p, 3, 1) != (CLEAN, [], [])             # the same rows folded over all 8 words
