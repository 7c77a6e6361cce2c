"""CPU: the update of a stored stripe (csrc/update.cu, DESIGN 3h) restated in Python integers, against the encode by definition.
T[t] = -2 / (N (rho^(2t+1) - 1)) is computed as update_table_kernel computes it (rho^e by the CRT split of LeafRoots, a Barrett
triple of gf::make_tw), and the parity update is the kernel's: canonical deltas, gf::mul by the triple, lazy gf::addl onto the
raw parity word, one canon at the end."""
import numpy as np
import pytest

from test_repair_algebra import C, MASK, P, root, rho_pow_crt, triple


def mul(b, t):                                     # gf::mul: b * w mod P in [0, P] for any 32-bit b
    w, whi, wlo = t
    q = ((b * whi + ((b * wlo) >> 32)) >> 32) & MASK
    return (q * C + b * w) & MASK


def addl(a, v):                                    # gf::addl: a in [0, 2^32), v in [0, P]
    s = a + v
    return s - (1 << 32) + C if s >> 32 else s


def canon(x):
    return x - P if x >= P else x


def table(N):
    """What update_table_kernel stores"""
    n2 = 2 * N
    return [triple((P - 2) * pow(N * (rho_pow_crt(n2, 2 * t + 1) - 1) % P, P - 2, P) % P) for t in range(N)]


def update(N, M, data, parity, changed, new):
    """One word column: data (N raw words), parity (M raw words), the changed rows and their new raw words; updated copies"""
    T, D = table(N), N // M
    data, parity = list(data), list(parity)
    delta = []
    for e, v in zip(changed, new):                 # update_delta_kernel
        delta.append((canon(v) - canon(data[e])) % P)
        data[e] = canon(v)
    for j in range(M):                             # update_parity_kernel
        acc = parity[j]
        for e, d in zip(changed, delta):
            acc = addl(acc, mul(d, T[(D * j + N - e) % N]))
        parity[j] = canon(acc)
    return data, parity


def encode_by_definition(data):
    """parity j = f(rho^(2j+1)), f of degree < N with f(rho^(2i)) = data i, rho = GF_Root(2N), from a table of rho's powers"""
    N = len(data)
    n2 = 2 * N
    rp = [1] * n2
    rho = root(n2)
    for m in range(1, n2):
        rp[m] = rp[m - 1] * rho % P
    inv_n = pow(N, P - 2, P)
    coef = [sum(data[i] * rp[(n2 - 2 * i * k % n2) % n2] for i in range(N)) * inv_n % P for k in range(N)]     # omega^-ik / N
    return [sum(coef[k] * rp[(2 * j + 1) * k % n2] for k in range(N)) % P for j in range(N)]


def raw(x, rng):
    """x as a stored word: x + P where that fits 32 bits, at random"""
    return x + P if x < C and rng.integers(2) else x


ORDERS = [1, 2, 4, 8, 16, 32, 64, 3, 6, 12, 24, 48, 9, 18, 36, 72]


@pytest.mark.parametrize("N", ORDERS)
def test_update_equals_the_encode_of_the_new_data(N):
    rng = np.random.default_rng(N)
    data = [int(x) for x in rng.integers(0, P, size=N)]
    full = encode_by_definition(data)
    ks = range(1, N + 1) if N <= 36 else sorted({1, 2, 3, 5, 8, N // 4, N // 2, N - 1, N} | {int(k) for k in rng.integers(1, N + 1, size=6)})
    for M in [m for m in range(1, N + 1) if N % m == 0]:
        D = N // M
        for k in ks:
            changed = sorted(rng.choice(N, size=k, replace=False).tolist())
            new = [int(x) for x in rng.integers(0, P, size=k)]
            want_data = list(data)
            for e, v in zip(changed, new):
                want_data[e] = v
            want = encode_by_definition(want_data)[::D]
            got_d, got_p = update(N, M, [raw(x, rng) for x in data], [raw(x, rng) for x in full[::D]], changed, [raw(x, rng) for x in new])
            assert got_p == want, (N, M, changed)
            assert got_d == want_data, (N, M, changed)


@pytest.mark.parametrize("N", [12, 16, 18, 72])
def test_two_updates_equal_one_combined_update(N):
    rng = np.random.default_rng(100 + N)
    data = [int(x) for x in rng.integers(0, P, size=N)]
    full = encode_by_definition(data)
    for M in (1, N // 2, N):
        parity = full[::N // M]
        a = sorted(rng.choice(N, size=N // 3, replace=False).tolist())
        b = sorted(rng.choice(N, size=N // 2, replace=False).tolist())
        va = {e: int(rng.integers(0, P)) for e in a}
        vb = {e: int(rng.integers(0, P)) for e in b}
        d1, p1 = update(N, M, data, parity, a, [va[e] for e in a])
        d2, p2 = update(N, M, d1, p1, b, [vb[e] for e in b])
        final = {**va, **vb}                                        # b's value wins where both changed a block
        both = sorted(final)
        d3, p3 = update(N, M, data, parity, both, [final[e] for e in both])
        assert (d2, p2) == (d3, p3), (N, M)


@pytest.mark.parametrize("N", [9, 24, 64])
def test_new_equal_to_old_leaves_the_parity_unchanged(N):
    rng = np.random.default_rng(200 + N)
    data = [int(x) for x in rng.integers(0, P, size=N)]
    for M in [m for m in range(1, N + 1) if N % m == 0]:
        parity = encode_by_definition(data)[::N // M]
        changed = sorted(rng.choice(N, size=max(1, N // 3), replace=False).tolist())
        got_d, got_p = update(N, M, data, parity, changed, [raw(data[e], rng) for e in changed])
        assert got_p == parity and got_d == data, (N, M)


def test_table_matches_the_lagrange_basis():
    """T[(D j' - i) mod N] is L_i at the parity point j': the encode of a unit vector e_i is column i of the table"""
    for N in (1, 2, 3, 6, 8, 9):
        T = [t[0] for t in table(N)]
        for i in range(N):
            unit = [1 if r == i else 0 for r in range(N)]
            assert encode_by_definition(unit) == [T[(j - i) % N] for j in range(N)], (N, i)
