"""CPU: the batch encode's arithmetic (csrc/batch.cu, DESIGN 3l) restated in Python integers, against the encode by definition:
raw 32-bit data words straight into gf::mul by update's table triple T[(D j - i) mod N], a lazy gf::addl of the N terms from 0,
one canon.  Every N <= 64 of the family and every divisor M, with the words 0, P - 1, P, 0xFFFFFFFF and random ones."""
import numpy as np
import pytest

from test_update_algebra import P, addl, canon, encode_by_definition, mul, table

ORDERS = [1, 2, 4, 8, 16, 32, 64, 3, 6, 12, 24, 48, 9, 18, 36]


def batch_parity(N, M, data):
    """One word column of one stripe as the kernel computes it: data = N raw 32-bit words; the M canonical parity words"""
    T, D = table(N), N // M
    out = []
    for j in range(M):
        acc = 0
        for i in range(N):
            acc = addl(acc, mul(data[i], T[(D * j + N - i) % N]))
        out.append(canon(acc))
    return out


@pytest.mark.parametrize("N", ORDERS)
def test_batch_parity_equals_the_encode_by_definition(N):
    rng = np.random.default_rng(300 + N)
    special = [0, P - 1, P, 0xFFFFFFFF, P + 5, 1]
    columns = [[special[(i + k) % len(special)] for i in range(N)] for k in range(len(special))]
    columns += [[0xFFFFFFFF] * N, [P] * N]
    columns += [[int(x) for x in rng.integers(0, 1 << 32, size=N, dtype=np.uint64)] for _ in range(3)]
    for col in columns:
        full = encode_by_definition([x % P for x in col])
        for M in [m for m in range(1, N + 1) if N % m == 0]:
            assert batch_parity(N, M, col) == full[::N // M], (N, M, col[:4])


def test_lazy_sums_stay_below_two_to_the_32():
    """addl keeps a lazy sum in [0, 2^32) whatever the number of terms: 64 terms of the largest product value P"""
    acc = 0
    for _ in range(64):
        acc = addl(acc, P)
        assert 0 <= acc < 1 << 32
    assert canon(acc) == 64 * P % P
