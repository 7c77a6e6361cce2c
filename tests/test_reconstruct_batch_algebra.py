"""CPU: the degraded read of a batch of stripes (csrc/batch.cu, api.cu, DESIGN 3m) restated in Python integers.  The host folds
the combination B of the single-stripe read (test_reconstruct_algebra.py) into one n_out x N matrix C over the source rows (the
surviving data rows, ascending, then J), with the N entries of update's table from one batch inversion; the kernel applies C
with gf::mul by Barrett triples, lazy gf::addl sums from 0 and one canon.  Checked against the encode by definition with garbage
in every row outside the source list, against the two-step result of the single-stripe read, and the host's T entries against
update's device table formula."""
import itertools

import numpy as np
import pytest

from test_reconstruct_algebra import combination, divisors, reconstruct as two_step, rows_J, stripe, subsets
from test_repair_algebra import MASK, P, root, triple
from test_update_algebra import addl, canon, mul, raw, table

ORDERS = [1, 2, 4, 8, 16, 32, 64, 3, 6, 12, 24, 48, 9, 18, 36]
MAX_K = 32                                         # FASTECC_B200_RECONSTRUCT_MAX, the two-step read's cap


def update_entries(N):
    """T[t] = -2 / (N (rho^(2t+1) - 1)), rho = GF_Root(2N), as api.cu's update_entries computes it"""
    rho = root(2 * N)
    return [(P - 2) * pow(N * (pow(rho, 2 * t + 1, P) - 1) % P, P - 2, P) % P for t in range(N)]


def fold(N, M, lost_d, lost_p, want_d, want_p):
    """(src, nd, C) as api.cu's reconstruct_batch builds them: source s is data row src[s] for s < nd, parity row src[s] after"""
    D, a = N // M, len(lost_d)
    J = rows_J(M, a, lost_p)
    B = combination(N, M, list(lost_d), J, want_d, want_p)
    T = update_entries(N)
    src = [i for i in range(N) if i not in set(lost_d)] + J
    nd, nwd = N - a, len(want_d)
    C = []
    for q in range(nwd + len(want_p)):
        row = []
        for i in src[:nd]:
            v = T[(D * want_p[q - nwd] - i) % N] if q >= nwd else 0
            v -= sum(B[q][j] * T[(D * J[j] - i) % N] for j in range(a))
            row.append(v % P)
        C.append(row + list(B[q]))
    return src, nd, C


def apply(src, nd, C, data, parity):
    """batch_reconstruct_kernel on one stripe: raw words straight into gf::mul by C's triples, lazy sums, one canon"""
    S = len(data[0]) if data else len(parity[0])
    rows = [data[r] if s < nd else parity[r] for s, r in enumerate(src)]
    trip = [[triple(c) for c in row] for row in C]
    out = []
    for q in range(len(C)):
        o = []
        for w in range(S):
            acc = 0
            for s, row in enumerate(rows):
                acc = addl(acc, mul(row[w], trip[q][s]))
            o.append(canon(acc))
        out.append(o)
    return out


def stored(data, parity, src, nd, rng, fill):
    """raw copies: the source rows with raw words >= P at random, every other row overwritten by fill()"""
    d = [[fill() for _ in row] for row in data]
    p = [[fill() for _ in row] for row in parity]
    for s, r in enumerate(src):
        if s < nd:
            d[r] = [raw(x, rng) for x in data[r]]
        else:
            p[r] = [raw(x, rng) for x in parity[r]]
    return d, p


def check(N, M, data, parity, lost_d, lost_p, want_d, want_p, rng, T):
    src, nd, C = fold(N, M, lost_d, lost_p, want_d, want_p)
    assert len(src) == N and len(set(src[:nd])) == nd and not set(src[:nd]) & set(lost_d)
    want = [data[e] for e in want_d] + [parity[j] for j in want_p]
    for k, fill in enumerate((lambda: int(rng.integers(0, 1 << 32)), lambda: MASK)):
        d, p = stored(data, parity, src, nd, rng, fill)
        got = apply(src, nd, C, d, p)
        assert got == want, (N, M, lost_d, lost_p, want_d, want_p)
        if not k and len(lost_d) + len(want_p) <= MAX_K:   # the single-stripe read of the same stored words
            assert got == two_step(N, M, d, p, lost_d, lost_p, want_d, want_p, T), (N, M, lost_d, lost_p)


@pytest.mark.parametrize("N", [1, 2, 3, 4, 6, 8, 9, 12, 16, 18])
def test_every_loss_of_up_to_two_data_and_two_parity_blocks(N):
    rng, T = np.random.default_rng(N), table(N)
    for M in divisors(N):
        data, parity = stripe(N, M, 2, rng)
        for a in range(min(2, M) + 1):
            for lost_d in itertools.combinations(range(N), a):
                for f in range(min(2, M - a) + 1):
                    for lost_p in itertools.combinations(range(M), f):
                        if not lost_d and not lost_p:
                            continue
                        check(N, M, data, parity, list(lost_d), list(lost_p), list(lost_d), list(lost_p), rng, T)


@pytest.mark.parametrize("N", [24, 32, 36, 48, 64])
def test_random_losses_and_wanted_subsets_up_to_M(N):
    rng, T = np.random.default_rng(200 + N), table(N)
    for M in divisors(N):
        data, parity = stripe(N, M, 2, rng)
        for k in range(5):
            a = M if k == 0 else int(rng.integers(0, M + 1))
            lost_d = sorted(rng.choice(N, size=a, replace=False).tolist())
            lost_p = sorted(rng.choice(M, size=int(rng.integers(0, M - a + 1)), replace=False).tolist())
            want_d, want_p = (lost_d, lost_p) if k == 0 else (subsets(lost_d, rng), subsets(lost_p, rng))
            if not want_d and not want_p:
                continue
            check(N, M, data, parity, lost_d, lost_p, want_d, want_p, rng, T)


@pytest.mark.parametrize("N", ORDERS)
def test_fold_equals_the_two_step_combination(N):
    """C as a matrix: applied to unit rows it gives the single-stripe read's result on those rows (sums of T, then B)"""
    rng = np.random.default_rng(300 + N)
    for M in divisors(N):
        a = int(rng.integers(0, min(M, MAX_K) + 1))
        lost_d = sorted(rng.choice(N, size=a, replace=False).tolist())
        lost_p = sorted(rng.choice(M, size=int(rng.integers(0, min(M - a, MAX_K - a) + 1)), replace=False).tolist())
        want_d, want_p = lost_d, lost_p
        if not want_d and not want_p:
            continue
        src, nd, C = fold(N, M, lost_d, lost_p, want_d, want_p)
        T = table(N)
        for s in range(N):                             # source row s = 1, every other row 0: column s of C
            data = [[int(s < nd and r == src[s])] for r in range(N)]
            parity = [[int(s >= nd and r == src[s])] for r in range(M)]
            got = two_step(N, M, data, parity, lost_d, lost_p, want_d, want_p, T)
            assert [row[0] for row in got] == [C[q][s] for q in range(len(C))], (N, M, s)


@pytest.mark.parametrize("N", ORDERS)
def test_host_entries_equal_the_device_table(N):
    assert update_entries(N) == [t[0] for t in table(N)], N


def test_lazy_sums_of_64_terms_stay_below_two_to_the_32():
    """a source row's raw word 0xFFFFFFFF times the largest coefficient P - 1, 64 times: every partial sum fits 32 bits"""
    acc = 0
    for _ in range(64):
        v = mul(MASK, triple(P - 1))
        assert 0 <= v <= P
        acc = addl(acc, v)
        assert 0 <= acc < 1 << 32
    assert canon(acc) == 64 * (MASK % P) * (P - 1) % P
