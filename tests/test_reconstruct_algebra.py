"""CPU: the degraded read of a stored stripe (csrc/reconstruct.cu, api.cu, DESIGN 3k) restated in Python integers, against every
D-th parity of the encode by definition.  The pass over the surviving data rows uses T as update_table_kernel builds it (the CRT
split of LeafRoots, Barrett triples) with the kernels' gf::mul and lazy gf::addl; the combination B is built as api.cu builds it
(GF_Root powers, a Gauss-Jordan inverse mod P) and applied with Barrett products.  The pipeline reads the stripe only through the
rows the header names (the surviving data rows and the parity rows J), which the tests check by filling every other row with
garbage."""
import itertools

import numpy as np
import pytest

from test_repair_algebra import MASK, P, root, triple
from test_update_algebra import addl, canon, encode_by_definition, mul, raw, table

MAX_K = 32                                         # FASTECC_B200_RECONSTRUCT_MAX


def rows_J(M, a, lost_parity):
    """the a lowest-numbered parity blocks not lost"""
    gone = set(lost_parity)
    return [j for j in range(M) if j not in gone][:a]


def host_entries(N, M, pos, E):
    """T(j, e) = T[(D j - e) mod N] = -2 / (N (y_j z_e - 1)), y_j = rho^(2Dj+1), z_e = rho^-2e, as api.cu computes them"""
    D, rho = N // M, root(2 * N)
    return [[(P - 2) * pow(N * (pow(rho, 2 * D * j + 1, P) * pow(rho, (2 * N - 2 * e) % (2 * N), P) - 1) % P, P - 2, P) % P for e in E] for j in pos]


def inverse(A):
    """Gauss-Jordan mod P"""
    a = len(A)
    A = [list(r) for r in A]
    X = [[int(i == j) for j in range(a)] for i in range(a)]
    for col in range(a):
        p = next(r for r in range(col, a) if A[r][col])
        A[col], A[p], X[col], X[p] = A[p], A[col], X[p], X[col]
        f = pow(A[col][col], P - 2, P)
        A[col] = [v * f % P for v in A[col]]
        X[col] = [v * f % P for v in X[col]]
        for r in range(a):
            m = A[r][col]
            if r != col and m:
                A[r] = [(x - m * y) % P for x, y in zip(A[r], A[col])]
                X[r] = [(x - m * y) % P for x, y in zip(X[r], X[col])]
    return X


def combination(N, M, E, J, want_d, want_p):
    """B: one row of a coefficients per output, the wanted data blocks first"""
    a = len(E)
    Tv = host_entries(N, M, J + list(want_p), E)
    X = inverse(Tv[:a])
    rows = [X[E.index(e)] for e in want_d]
    rows += [[sum(Tv[a + m][k] * X[k][j] for k in range(a)) % P for j in range(a)] for m in range(len(want_p))]
    return rows


def reconstruct(N, M, data, parity, lost_d, lost_p, want_d, want_p, T=None):
    """data: N rows, parity: M rows of raw words (lists); the wanted blocks, data first, canonical"""
    T, D, a = T or table(N), N // M, len(lost_d)
    S = len(data[0]) if data else len(parity[0])
    J = rows_J(M, a, lost_p)
    pos, lost = J + list(want_p), set(lost_d)
    r = []
    for j in pos:                                  # reconstruct_sum_kernel
        row = []
        for w in range(S):
            acc = 0
            for i in range(N):
                if i not in lost:
                    acc = addl(acc, mul(data[i][w], T[(D * j + N - i) % N]))
            row.append(canon(acc))
        r.append(row)
    B = combination(N, M, list(lost_d), J, want_d, want_p)
    out = []
    for q in range(len(want_d) + len(want_p)):     # reconstruct_combine_kernel
        row = []
        for w in range(S):
            acc = r[a + q - len(want_d)][w] if q >= len(want_d) else 0
            for j in range(a):
                acc = addl(acc, mul((canon(parity[J[j]][w]) - r[j][w]) % P, triple(B[q][j])))
            row.append(canon(acc))
        out.append(row)
    return out


def stripe(N, M, S, rng):
    """data rows and the M stored parity rows (canonical), by definition"""
    data = [[int(x) for x in rng.integers(0, P, size=S)] for _ in range(N)]
    cols = [encode_by_definition([data[i][w] for i in range(N)]) for w in range(S)]
    return data, [[cols[w][(N // M) * j] for w in range(S)] for j in range(M)]


def stored(data, parity, lost_d, lost_p, J, rng, fill):
    """raw copies: survivors with raw words >= P at random, lost rows and parity rows outside J overwritten by fill()"""
    d = [[raw(x, rng) for x in row] for row in data]
    p = [[raw(x, rng) for x in row] for row in parity]
    for e in lost_d:
        d[e] = [fill() for _ in d[e]]
    for j in range(len(p)):
        if j in lost_p or j not in J:
            p[j] = [fill() for _ in p[j]]
    return d, p


def check(N, M, data, parity, lost_d, lost_p, want_d, want_p, rng, T):
    J = rows_J(M, len(lost_d), lost_p)
    want = [data[e] for e in want_d] + [parity[j] for j in want_p]
    fills = (lambda: int(rng.integers(0, 1 << 32)), lambda: MASK)
    for fill in fills:
        d, p = stored(data, parity, lost_d, lost_p, J, rng, fill)
        got = reconstruct(N, M, d, p, lost_d, lost_p, want_d, want_p, T)
        assert got == want, (N, M, lost_d, lost_p, want_d, want_p)


def divisors(N):
    return [m for m in range(1, N + 1) if N % m == 0]


def subsets(xs, rng):
    """a random subset (possibly empty), ascending"""
    return sorted(x for x in xs if rng.integers(2))


@pytest.mark.parametrize("N", [1, 2, 3, 4, 6, 8, 9, 12, 16, 18])
def test_every_loss_of_up_to_two_data_and_two_parity_blocks(N):
    rng = np.random.default_rng(N)
    T = table(N)
    for M in divisors(N):
        data, parity = stripe(N, M, 2, rng)
        for a in range(min(2, M) + 1):
            for lost_d in itertools.combinations(range(N), a):
                for f in range(min(2, M - a) + 1):
                    for lost_p in itertools.combinations(range(M), f):
                        want_d, want_p = list(lost_d), list(lost_p)
                        if not want_d and not want_p:
                            continue
                        check(N, M, data, parity, list(lost_d), list(lost_p), want_d, want_p, rng, T)


@pytest.mark.parametrize("N", [24, 32, 36, 48, 64, 72])
def test_random_losses_and_wanted_subsets(N):
    rng = np.random.default_rng(100 + N)
    T = table(N)
    for M in divisors(N):
        data, parity = stripe(N, M, 2, rng)
        top = min(M, MAX_K)
        for _ in range(6):
            a = int(rng.integers(0, top + 1))
            lost_d = sorted(rng.choice(N, size=a, replace=False).tolist())
            lost_p = sorted(rng.choice(M, size=int(rng.integers(0, M - a + 1)), replace=False).tolist())
            want_d = subsets(lost_d, rng)
            want_p = subsets(lost_p, rng)[:MAX_K - a]
            if not want_d and not want_p:
                continue
            check(N, M, data, parity, lost_d, lost_p, want_d, want_p, rng, T)
        a = min(M, MAX_K) // 2                     # the cap: a + |W_p| = min(M, 32)
        lost_d = sorted(rng.choice(N, size=a, replace=False).tolist())
        lost_p = sorted(rng.choice(M, size=min(M, MAX_K) - a, replace=False).tolist())
        check(N, M, data, parity, lost_d, lost_p, lost_d, lost_p, rng, T)


def test_no_lost_data_gives_the_parity_of_the_current_data():
    rng = np.random.default_rng(7)
    for N, M in ((9, 3), (16, 16), (12, 1)):
        data, parity = stripe(N, M, 3, rng)
        lost_p = list(range(0, M, 2))
        d, _ = stored(data, parity, [], lost_p, [], rng, lambda: int(rng.integers(0, 1 << 32)))
        p = [[int(rng.integers(0, 1 << 32)) for _ in range(3)] for _ in range(M)]     # no parity row is read
        assert reconstruct(N, M, d, p, [], lost_p, [], lost_p, table(N)) == [parity[j] for j in lost_p]


def test_one_data_block_and_one_parity_block():
    """N = 1: the parity is a multiple of the one data block; M = 1: the single parity block rebuilds any one data block"""
    rng = np.random.default_rng(8)
    data, parity = stripe(1, 1, 4, rng)
    assert reconstruct(1, 1, [[0] * 4], parity, [0], [], [0], []) == data
    assert reconstruct(1, 1, data, [[5] * 4], [], [0], [], [0]) == parity
    data, parity = stripe(9, 1, 4, rng)
    for e in range(9):
        d = [row if i != e else [MASK] * 4 for i, row in enumerate(data)]
        assert reconstruct(9, 1, d, parity, [e], [], [e], []) == [data[e]]


def test_J_is_the_lowest_surviving_parity_blocks():
    assert rows_J(8, 3, [0, 2]) == [1, 3, 4]
    assert rows_J(8, 0, [1]) == []
    assert rows_J(4, 2, [0, 1]) == [2, 3]
    assert rows_J(6, 3, []) == [0, 1, 2]
    # changing a parity row in J changes the result, changing one outside J does not
    rng = np.random.default_rng(9)
    N, M = 12, 6
    data, parity = stripe(N, M, 1, rng)
    lost_d, lost_p = [2, 7], [1]
    base = reconstruct(N, M, data, parity, lost_d, lost_p, lost_d, [])
    for j in range(M):
        p = [list(r) for r in parity]
        p[j] = [(p[j][0] + 1) % P]
        changed = reconstruct(N, M, data, p, lost_d, lost_p, lost_d, []) != base
        assert changed == (j in rows_J(M, 2, lost_p)), j


@pytest.mark.parametrize("N", [1, 3, 8, 9, 18, 24, 72])
def test_host_entries_equal_the_device_table(N):
    """api.cu's T(j, e) from GF_Root powers equals update_table_kernel's canonical entry T[(D j - e) mod N]"""
    T = table(N)
    for M in divisors(N):
        D = N // M
        E = list(range(N))
        got = host_entries(N, M, list(range(M)), E)
        assert all(got[j][e] == T[(D * j - e) % N][0] for j in range(M) for e in E), (N, M)


@pytest.mark.parametrize("N", [8, 9, 24, 72])
def test_the_system_is_invertible_for_every_loss(N):
    """A = T(J, E) is Cauchy up to diagonal scalings: nonsingular for random J, E of every size up to min(M, 32)"""
    rng = np.random.default_rng(N)
    for M in divisors(N):
        for a in range(1, min(M, MAX_K) + 1):
            E = sorted(rng.choice(N, size=a, replace=False).tolist())
            J = sorted(rng.choice(M, size=a, replace=False).tolist())
            A = host_entries(N, M, J, E)
            X = inverse(A)
            assert all(sum(A[i][k] * X[k][j] for k in range(a)) % P == int(i == j) for i in range(a) for j in range(a))
