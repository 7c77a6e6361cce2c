"""CPU: the batch update's arithmetic (csrc/batch.cu: batch_update_kernel, DESIGN 3n) restated in Python integers, against the
encode by definition of the updated data: delta = subl(new, canon(old)) with raw new words, gf::mul by update's table triple
T[(D j - e) mod N] as update_table_kernel builds it, lazy gf::addl onto the raw stored parity word, one canon.  Every N <= 64 of
the family and every divisor M; every changed subset up to N = 6 and random subsets beyond; stored and new words 0, P - 1, P,
P + 5, 0xFFFFFFFF and random ones; garbage in the unchanged data rows, which the kernel never reads."""
import itertools

import numpy as np
import pytest

from test_update_algebra import C, P, addl, canon, encode_by_definition, mul, table

ORDERS = [1, 2, 4, 8, 16, 32, 64, 3, 6, 12, 24, 48, 9, 18, 36]
SPECIAL = [0, P - 1, P, P + 5, 0xFFFFFFFF, 1]


def subl(a, v):                                    # gf::subl: a in [0, 2^32), v in [0, P]
    s = a - v
    return s + (1 << 32) - C if s < 0 else s


def batch_update(N, M, data, parity, changed, new):
    """One word column of one stripe as the kernel computes it: data (N raw words, only the changed ones read), parity (M raw
    words), new (k raw words); the updated data and the M canonical parity words"""
    T, D = table(N), N // M
    delta = [subl(v, canon(data[e])) for e, v in zip(changed, new)]
    out_d = list(data)
    for e, v in zip(changed, new):
        out_d[e] = canon(v)
    out_p = []
    for j in range(M):
        acc = parity[j]
        for e, d in zip(changed, delta):
            acc = addl(acc, mul(d, T[(D * j + N - e) % N]))
        out_p.append(canon(acc))
    return out_d, out_p


def stored(x, rng):
    """x as a stored word: x + P where that fits 32 bits, at random"""
    return x + P if x < C and rng.integers(2) else x


def subsets(N, rng):
    if N <= 6:
        return [list(c) for k in range(1, N + 1) for c in itertools.combinations(range(N), k)]
    out = [[0], [N - 1], list(range(N)), [0, N - 1]]
    for k in sorted({1, 2, N // 4, N // 2, N - 1, N} | {int(x) for x in rng.integers(1, N + 1, size=4)} - {0}):
        out.append(sorted(rng.choice(N, size=k, replace=False).tolist()))
    return out


@pytest.mark.parametrize("N", ORDERS)
def test_batch_update_equals_the_encode_of_the_updated_data(N):
    rng = np.random.default_rng(700 + N)
    for trial in range(3):
        data = [int(x) for x in rng.integers(0, P, size=N)]
        if trial == 1:
            data = [[0, P - 1, 5][i % 3] for i in range(N)]
        full = encode_by_definition(data)
        for M in [m for m in range(1, N + 1) if N % m == 0]:
            D = N // M
            for changed in subsets(N, rng):
                k = len(changed)
                new_raw = [SPECIAL[(i + trial) % len(SPECIAL)] if (i + trial) % 2 else int(rng.integers(0, 1 << 32)) for i in range(k)]
                want_data = list(data)
                for e, v in zip(changed, new_raw):
                    want_data[e] = v % P
                want = encode_by_definition(want_data)[::D]
                stored_d = [stored(x, rng) for x in data]
                for i in range(N):                                  # garbage in the rows the kernel must not read
                    if i not in changed:
                        stored_d[i] = [0xFFFFFFFF, P, int(rng.integers(0, 1 << 32))][i % 3]
                got_d, got_p = batch_update(N, M, stored_d, [stored(x, rng) for x in full[::D]], changed, new_raw)
                assert got_p == want, (N, M, changed)
                assert [got_d[e] for e in changed] == [v % P for v in new_raw], (N, M, changed)
                assert all(got_d[i] == stored_d[i] for i in range(N) if i not in changed), (N, M, changed)


@pytest.mark.parametrize("N", [4, 12, 18, 36, 64])
def test_special_words_in_the_stored_data_parity_and_new_rows(N):
    """Every stored and new word from {0, P - 1, P, P + 5, 0xFFFFFFFF, 1}, in every column position"""
    rng = np.random.default_rng(800 + N)
    for s in range(len(SPECIAL)):
        raw_d = [SPECIAL[(i + s) % len(SPECIAL)] for i in range(N)]
        data = [x % P for x in raw_d]
        full = encode_by_definition(data)
        for M in [m for m in range(1, N + 1) if N % m == 0]:
            D = N // M
            raw_p = [stored(x, rng) for x in full[::D]]
            changed = sorted(rng.choice(N, size=max(1, N // 3), replace=False).tolist())
            new_raw = [SPECIAL[(q + 2 * s) % len(SPECIAL)] for q in range(len(changed))]
            want_data = list(data)
            for e, v in zip(changed, new_raw):
                want_data[e] = v % P
            _, got_p = batch_update(N, M, raw_d, raw_p, changed, new_raw)
            assert got_p == encode_by_definition(want_data)[::D], (N, M, s)


def test_stored_parity_words_of_0xffffffff_are_their_residue():
    """The lazy sum starts from the raw stored parity word: parity words 0xFFFFFFFF (= 0xFFFFE mod P) come out as 0xFFFFE plus
    the change of the encode, whatever the data"""
    rng = np.random.default_rng(5)
    for N in (4, 9, 32):
        data = [int(x) for x in rng.integers(0, P, size=N)]
        for M in (1, N):
            D = N // M
            changed = sorted(rng.choice(N, size=N // 2, replace=False).tolist())
            new = [int(x) for x in rng.integers(0, 1 << 32, size=len(changed))]
            after = list(data)
            for e, v in zip(changed, new):
                after[e] = v % P
            change = [(y - x) % P for x, y in zip(encode_by_definition(data)[::D], encode_by_definition(after)[::D])]
            _, got = batch_update(N, M, data, [0xFFFFFFFF] * M, changed, new)
            assert got == [(0xFFFFE + c) % P for c in change], (N, M)


@pytest.mark.parametrize("N", [12, 16, 18, 48, 64])
def test_two_successive_updates_equal_one_combined_update(N):
    rng = np.random.default_rng(900 + N)
    data = [int(x) for x in rng.integers(0, P, size=N)]
    full = encode_by_definition(data)
    for M in (1, N // 4 if N % 4 == 0 else 1, N):
        parity = full[::N // M]
        a = sorted(rng.choice(N, size=N // 3, replace=False).tolist())
        b = sorted(rng.choice(N, size=N // 2, replace=False).tolist())
        va = {e: int(rng.integers(0, 1 << 32)) for e in a}
        vb = {e: int(rng.integers(0, 1 << 32)) for e in b}
        d1, p1 = batch_update(N, M, data, parity, a, [va[e] for e in a])
        d2, p2 = batch_update(N, M, d1, p1, b, [vb[e] for e in b])
        final = {**va, **vb}
        both = sorted(final)
        d3, p3 = batch_update(N, M, data, parity, both, [final[e] for e in both])
        assert (d2, p2) == (d3, p3), (N, M)


@pytest.mark.parametrize("N", [9, 24, 64])
def test_new_equal_to_old_leaves_the_parity_residues_unchanged(N):
    rng = np.random.default_rng(1000 + N)
    data = [int(x) for x in rng.integers(0, P, size=N)]
    for M in [m for m in range(1, N + 1) if N % m == 0]:
        parity = encode_by_definition(data)[::N // M]
        raw_p = [stored(x, rng) for x in parity]
        changed = sorted(rng.choice(N, size=max(1, N // 3), replace=False).tolist())
        got_d, got_p = batch_update(N, M, [stored(x, rng) for x in data], raw_p, changed, [stored(data[e], rng) for e in changed])
        assert got_p == parity, (N, M)
        assert [got_d[e] for e in changed] == [data[e] for e in changed], (N, M)


def test_deltas_and_lazy_sums_stay_below_two_to_the_32():
    """subl keeps delta in [0, 2^32) for any raw new word and canonical old word; 64 terms of the largest product onto the
    largest raw parity word stay below 2^32"""
    for v in (0, 1, P - 1, P, 0xFFFFFFFF):
        for o in (0, 1, P - 1):
            d = subl(v, o)
            assert 0 <= d < 1 << 32 and d % P == (v - o) % P
    acc = 0xFFFFFFFF
    for _ in range(64):
        acc = addl(acc, P)
        assert 0 <= acc < 1 << 32
    assert canon(acc) == (0xFFFFFFFF + 64 * P) % P
