"""CPU: the encode of N = r * L data blocks (r in {3, 9}, L = 2^k) into M | N parity blocks (csrc/mixed_radix.cu
radix_fold_kernel between the power-of-two transforms, api.cu encode, DESIGN 3f) restated in plain Python
integers: the constants as launch_radix_fold computes them (the coset twist of the output twiddle and its CRT split, the
output rows d_u), the kernel's fold by 2^f <= 2^i in place, the r / s forward transforms of order L / 2^f and the gather of
every 2^(i-f)-th output -- checked against every (N/M)-th parity of the encode by definition, for every divisor M and every
fold the host may pick.  The GPU kernels are compared with the oracle in tests/test_asym_mixed_encode.py; asym_erasures (the
decoder's view of these code words) is checked here as well."""
import random

import pytest

from test_mixed_encode_algebra import dft_r, encode_by_definition, rho_pow
from test_mixed_radix_algebra import by_definition, root

P = 0xFFF00001


def odd_part(n):
    while n % 2 == 0:
        n //= 2
    return n


def divisors(n):
    return [m for m in range(1, n + 1) if n % m == 0]


def fold_consts(r, L, s, log_d2):
    """launch_radix_fold's host constants: tr[u], tm[u] (rho^(2*k2*J_u) = GF_Root(r)^(tr*k2 mod r) * GF_Root(2L)^(tm*k2 mod 2L))
    and the output row offsets d[u], u < r / s, with J_u = j1 + r * c_j1, j1 = s*u, c_j1 = -j1 * r^-1 mod 2^i"""
    d2 = 1 << log_d2
    D = s * d2
    a2, b2 = pow(2 * L, -1, r), pow(r, -1, 2 * L)
    rinv = pow(r, -1, d2) if d2 > 1 else 0
    tr, tm, d, J = [], [], [], []
    for u in range(r // s):
        j1 = s * u
        c = -j1 * rinv % d2
        Ju = j1 + r * c
        assert Ju % D == 0
        J.append(Ju); tr.append(2 * Ju % r * a2 % r); tm.append(2 * Ju % (2 * L) * b2 % (2 * L)); d.append(Ju // D)
    return tr, tm, d, J


def fold_kernel(buf, r, L, s, log_d2, log_fold):
    """radix_fold_kernel on rows r*k2 + n1, in place: w_{s*u}[t] goes to row r*t + d[u] (t < T = L / 2^f)"""
    N = r * L
    invn = pow(N, P - 2, P)
    tr, tm, d, _ = fold_consts(r, L, s, log_d2)
    T = L >> log_fold
    out = {}
    for t in range(T):
        acc = [0] * (r // s)
        for q in range(1 << log_fold):
            k2 = t + q * T
            u_in = [buf[r * k2 + n1] % P * rho_pow(k2 * (1 - 2 * n1) % (2 * N), r, L) % P * invn % P for n1 in range(r)]
            a = dft_r(u_in, r, True)
            a = [a[k1] * pow(root(2 * r), k1, P) % P for k1 in range(r)]
            v = dft_r(a, r, False)
            for u in range(r // s):
                er, em = tr[u] * (k2 % r) % r, (tm[u] * k2) % (1 << 32) & (2 * L - 1)     # 32-bit product, masked
                tw = pow(root(r), er, P) * pow(root(2 * L), em, P) % P
                acc[u] = (acc[u] + v[s * u] * tw) % P
        for u in range(r // s):
            out[r * t + d[u]] = acc[u]
    for row, val in out.items():                          # every row written is one its own thread read (q = 0)
        buf[row] = val


def asym_mixed_encode(x, r, L, M, log_fold):
    N = r * L
    D = N // M
    s = odd_part(D)
    log_d2 = (D // s).bit_length() - 1
    u, keep = r // s, (D // s) >> log_fold
    buf = list(x)
    for n1 in range(r):                                   # step 1: as the full encode
        col = by_definition([buf[n1 + r * n2] for n2 in range(L)], L, True)
        for k2 in range(L):
            buf[n1 + r * k2] = col[k2]
    fold_kernel(buf, r, L, s, log_d2, log_fold)
    T = L >> log_fold
    for dd in range(u):                                   # step 3: u forward transforms of order T on rows dd + r*t
        col = by_definition([buf[dd + r * t] for t in range(T)], T, False)
        for t in range(T):
            buf[dd + r * t] = col[t]
    return [buf[g * r * keep + dd] for g in range(M // u) for dd in range(u)]     # the gather: row dd + r*keep*j'' -> dd + u*j''


@pytest.mark.parametrize("r", [3, 9])
@pytest.mark.parametrize("L", [1, 2, 8, 64])
def test_asym_mixed_encode_equals_every_d_th_parity(r, L):
    random.seed(100 * r + L)
    N = r * L
    x = [random.randrange(P) for _ in range(N)]
    full = encode_by_definition(x, N)
    for M in divisors(N):
        D = N // M
        log_d2 = (D // odd_part(D)).bit_length() - 1
        for f in range(log_d2 + 1):
            assert asym_mixed_encode(x, r, L, M, f) == full[::D], (M, f)


@pytest.mark.parametrize("r", [3, 9])
@pytest.mark.parametrize("L", [1, 2, 8, 64, 1 << 19])
def test_coset_twist_and_output_rows(r, L):
    """J_u = D * d_u; u -> d_u is a bijection onto [0, r/s); the split output twiddle is rho^(2*k2*J_u) = (the twiddle of the full
    encode, rho^(2*k2*j1)) * GF_Root(L)^(k2*c_j1), with the kernel's 32-bit product"""
    N = r * L
    rho = root(2 * N)
    random.seed(N)
    for D in sorted({m for m in [1, 2, 3, 6, 9, 18, 4 * r, N // 3, N // 2, N] if m and N % m == 0}):
        s = odd_part(D)
        log_d2 = (D // s).bit_length() - 1
        tr, tm, d, J = fold_consts(r, L, s, log_d2)
        assert sorted(d) == list(range(r // s)), D
        for u in range(r // s):
            j1, c = s * u, (J[u] - s * u) // r
            assert J[u] == D * d[u] and 0 <= c < (D // s)
            for k2 in [0, 1, L - 1] + [random.randrange(L) for _ in range(10)]:
                er, em = tr[u] * (k2 % r) % r, (tm[u] * k2) % (1 << 32) & (2 * L - 1)
                tw = pow(root(r), er, P) * pow(root(2 * L), em, P) % P
                assert tw == pow(rho, 2 * k2 * J[u] % (2 * N), P)
                assert tw == pow(rho, 2 * k2 * j1, P) * pow(root(L), k2 * c % L, P) % P


# ---- asym_erasures ---------------------------------------------------------------------------------------------------
def test_asym_erasures_rows():
    from fastecc_b200.decoder import asym_erasures
    assert asym_erasures(3, 3, [], []) == []
    assert asym_erasures(3, 1, [], []) == [3, 5]                      # parity 1, 2 never produced
    assert asym_erasures(3, 1, [2], []) == [3, 4, 5]
    assert asym_erasures(3, 1, [], [0]) == [1, 3, 5]
    assert asym_erasures(6, 2, [0], [1]) == [0, 3, 5, 7, 9, 11]       # D = 3: parity j' = 0, 1 sit in rows 1, 7
    assert asym_erasures(12, 4, [11, 3], []) == sorted([6, 22] + [2 * j + 1 for j in range(12) if j % 3])
    for N, M in ((18, 6), (96, 32), (9 * 64, 9 * 8)):
        rows = asym_erasures(N, M, range(M // 2), range(M - M // 2))
        assert len(rows) == N and rows == sorted(set(rows))          # exactly N of the 2N rows: the most the decoder takes
        produced = set(range(1, 2 * N, 2 * (N // M)))                  # rows of the M parity blocks
        assert sorted(set(rows) & produced) == [2 * (N // M) * j + 1 for j in range(M - M // 2)]
        assert [r for r in rows if r % 2 == 0] == [2 * i for i in range(M // 2)]


def test_asym_erasures_rejects():
    from fastecc_b200.decoder import asym_erasures
    with pytest.raises(ValueError):
        asym_erasures(12, 4, [0, 1, 2], [0, 1])                      # 5 > M blocks lost
    with pytest.raises(ValueError):
        asym_erasures(3, 1, [0], [0])
    with pytest.raises(ValueError):
        asym_erasures(12, 5, [], [])                                 # M does not divide N
    with pytest.raises(ValueError):
        asym_erasures(12, 4, [12], [])
    with pytest.raises(ValueError):
        asym_erasures(12, 4, [], [4])
