"""CPU: the repair of a stored stripe (csrc/repair.cu, DESIGN 3g) restated in Python integers, against every D-th parity of the
encode by definition.  The per-row constants are computed as finish_repair_kernel computes them (the locator over the lost
points of the 2N-row numbering, l(rho^m) and D[m] = NTT_2N(t * l_t)[m], rho^-k by the CRT split of LeafRoots) and every
element-wise product is the kernels' Barrett product with the triple of gf::make_tw."""
import numpy as np
import pytest

P = 0xFFF00001
C = (1 << 32) - P
GEN = 19
MASK = (1 << 32) - 1


def root(n):
    return pow(GEN, (P - 1) // n, P)


def triple(w):                                     # gf::make_tw
    whi, rem = divmod(w << 32, P)
    return w, whi, (rem << 32) // P


def mulc(b, t):                                    # gf::canon(gf::mul(b, w, whi, wlo)) for any 32-bit b
    w, whi, wlo = t
    q = ((b * whi + ((b * wlo) >> 32)) >> 32) & MASK
    v = (q * C + b * w) & MASK
    return v - P if v >= P else v


def dft(x, z):                                     # sum_k x_k z^(jk), unnormalised
    n = len(x)
    return [sum(x[k] * pow(z, j * k, P) for k in range(n)) % P for j in range(n)]


def encode_by_definition(data):
    """parity j = f(rho^(2j+1)), f of degree < N with f(rho^(2i)) = data i, rho = GF_Root(2N)"""
    N = len(data)
    rho = root(2 * N)
    coef = [c * pow(N, P - 2, P) % P for c in dft(data, pow(rho, 2 * (2 * N - 1), P))]     # omega^-1 = rho^(2N-2)
    return [sum(coef[k] * pow(rho, (2 * j + 1) * k, P) for k in range(N)) % P for j in range(N)]


def split_order(n):
    t = 0
    while n % 2 == 0:
        n //= 2; t += 1
    return n, t


def rho_pow_crt(n2, e):                            # LeafRoots: GF_Root(r)^(a2 e mod r) * GF_Root(2^t)^(b2 e mod 2^t)
    r, t = split_order(n2)
    m = 1 << t
    a2 = next(a for a in range(r) if a * m % r == 1 % r) if r > 1 else 0
    b2 = pow(r, -1, m) if m > 1 else 0
    g20 = root(1 << 20)
    v = pow(g20, ((b2 * e) & (m - 1)) << (20 - t), P)
    return v * pow(root(r), (a2 * (e % r)) % r, P) % P if r > 1 else v


def pattern(N, M, lost_data, lost_parity):
    """What finish_repair_kernel stores: c'_j, rho^-k / M, k, N / D[2e], -2 / (M D[2Dj' + 1]) as triples"""
    n2, D = 2 * N, N // M
    rho = root(n2)
    E = sorted([2 * e for e in lost_data] + [2 * D * j + 1 for j in lost_parity])
    lc = [1]
    for e in E:                                    # prod (x - rho^e), coefficient k at index k
        z = rho_pow_crt(n2, e)
        lc = [((lc[k - 1] if k else 0) - z * (lc[k] if k < len(lc) else 0)) % P for k in range(len(lc) + 1)]
    lc += [0] * (n2 - len(lc))
    lv = dft(lc, rho)                                                       # l(rho^m)
    dl = dft([t * c % P for t, c in enumerate(lc)], rho)                    # D[m] = rho^m l'(rho^m)
    inv2, inv_m = pow(2, P - 2, P), pow(M, P - 2, P)
    cs = [triple((P - lv[2 * D * j + 1]) % P * inv2 % P) for j in range(M)]
    cr = [triple(rho_pow_crt(n2, (n2 - k) % n2) * inv_m % P) for k in range(M)]
    ck = [triple(k) for k in range(M)]
    cd = [triple(N * pow(dl[2 * e], P - 2, P) % P) for e in lost_data]
    cp = [triple((P - 2) * pow(M * dl[2 * D * j + 1] % P, P - 2, P) % P) for j in lost_parity]
    return cs, cr, ck, cd, cp


def repair(N, M, data, parity, lost_data, lost_parity):
    """One word column: data (N raw words), parity (M raw words), repaired copies returned"""
    cs, cr, ck, cd, cp = pattern(N, M, lost_data, lost_parity)
    data, parity = list(data), list(parity)
    if not lost_data and not lost_parity:
        return data, parity
    D, ld = N // M, set(lost_data)
    zeta = root(M)
    ws = [0 if i in ld else data[i] % P for i in range(N)]                 # load
    G = encode_by_definition(ws)[::D]                                      # the encode of Z into M parity blocks
    u = []
    for j in range(M):                                                     # syndrome
        if cs[j][0] == 0:
            parity[j] = G[j]
            u.append(0)
        else:
            u.append(mulc((parity[j] % P - G[j]) % P, cs[j]))
    Pk = dft(u, pow(zeta, M - 1, P))                                       # inverse order-M transform: M p_k rho^k
    kp = [mulc(Pk[k], ck[k]) for k in range(M)]                            # split
    a = [mulc(Pk[k], cr[k]) for k in range(M)] + [0] * (N - M)
    if lost_data:
        A = dft(a, root(N))
        for i, e in enumerate(lost_data):                                  # scatter
            data[e] = mulc(A[e], cd[i])
    if lost_parity:
        K = dft(kp, zeta)
        for i, j in enumerate(lost_parity):
            parity[j] = (parity[j] + mulc(K[j], cp[i])) % P
    return data, parity


def loss_sets(N, M, rng):
    """none; parity only; data only; all M as data; |E_d| + |E_p| = M (twice); a single lost block of each kind"""
    def pick(n, k):
        return sorted(rng.choice(n, size=k, replace=False).tolist())
    out = [([], []), ([], pick(M, M)), (pick(N, max(1, M // 2)), []), (pick(N, M), []), ([N - 1], []), ([], [M - 1])]
    for _ in range(2):
        nd = int(rng.integers(0, M + 1))
        out.append((pick(N, nd), pick(M, M - nd)))
    return out


ORDERS = [1, 2, 4, 8, 16, 32, 3, 6, 12, 24, 48, 9, 18, 36, 72]


@pytest.mark.parametrize("N", ORDERS)
def test_repair_algebra_recovers_data_and_parity(N):
    rng = np.random.default_rng(N)
    data = [int(x) for x in rng.integers(0, P, size=N)]
    full = encode_by_definition(data)
    for M in [m for m in range(1, N + 1) if N % m == 0]:
        D = N // M
        parity = full[::D]
        for lost_data, lost_parity in loss_sets(N, M, rng):
            raw_d = [x + P if x < C else x for x in data]                 # surviving words taken mod P
            raw_p = list(parity)
            for e in lost_data:
                raw_d[e] = int(rng.integers(P, 1 << 32))                    # garbage >= P in the lost rows
            for j in lost_parity:
                raw_p[j] = int(rng.integers(P, 1 << 32))
            got_d, got_p = repair(N, M, raw_d, raw_p, lost_data, lost_parity)
            for e in lost_data:
                assert got_d[e] == data[e], (N, M, lost_data, lost_parity, e)
            for j in lost_parity:
                assert got_p[j] == parity[j], (N, M, lost_data, lost_parity, j)
            assert [got_d[i] for i in range(N) if i not in lost_data] == [raw_d[i] for i in range(N) if i not in lost_data]
            assert [got_p[j] for j in range(M) if j not in lost_parity] == [raw_p[j] for j in range(M) if j not in lost_parity]


def test_small_data_words_keep_raw_values_above_p():
    """Words below 2^32 - P can be stored raw as x + P; the repair reads them mod P."""
    N, M = 12, 4
    data = [int(x) for x in np.random.default_rng(1).integers(0, C, size=N)]
    parity = encode_by_definition(data)[::N // M]
    got_d, got_p = repair(N, M, [x + P for x in data], parity, [0, 5], [1, 3])
    assert got_d[0] == data[0] and got_d[5] == data[5] and got_p[1] == parity[1] and got_p[3] == parity[3]


def test_crt_split_matches_the_root_powers():
    for n2 in (2, 6, 18, 24, 72, 1 << 11, 3 << 10, 9 << 9):
        rho = root(n2)
        for e in (0, 1, 2, n2 // 3, n2 - 1):
            assert rho_pow_crt(n2, e) == pow(rho, e, P), (n2, e)
