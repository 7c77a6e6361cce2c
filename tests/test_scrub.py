"""GPU: scrub of a stored stripe (fastecc_b200_rs_scrub, csrc/scrub.cu, DESIGN 3i).  Small stripes are compared with the Python
pipeline of test_scrub_algebra.py, the fold with the header's weights through corruptions that those weights, and only those,
cannot see; large ones with the set that was corrupted.  Every call is checked to leave both buffers byte-identical."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

from test_scrub_algebra import CLEAN, DETECTED, LOCATED, scrub as py_scrub, weight

P = 0xFFF00001
C = (1 << 32) - P
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0x5EED5EED


def i32(x):
    """int64 words in [0, 2^32) as the int32 tensor that stores them"""
    import torch
    return (x - (x >= 1 << 31).to(torch.int64) * (1 << 32)).to(torch.int32)


def u64(t):
    import torch
    return t.to(torch.int64) & 0xFFFFFFFF


def rand_words(n, S, gen):
    import torch
    return torch.randint(0, P, (n, S), device="cuda", generator=gen, dtype=torch.int64)


def garbage(shape, gen=None):
    """random words over the whole 32-bit range, different in every position"""
    import torch
    return torch.randint(-(1 << 31), 1 << 31, shape, dtype=torch.int32, device="cuda", generator=gen)


def padded(x):
    """x (n x S words) in rows of ceil4(S) words: the aligned layout a stripe is stored in.  The pad words of a partial last
    16-byte group hold random garbage, different in every row and column, so that a fold that let them into its sums would change
    the syndromes (a constant pad column would not: it is the code word of a constant polynomial)."""
    n, S = x.shape
    buf = garbage((n, (S + 3) // 4 * 4))
    buf[:, :S] = x
    return buf[:, :S]


def encode(fecc, data, M):
    buf = data.clone()
    fecc.rs_encode_asym_mixed_dev(buf, M)
    return padded(buf[:M])


def scrub_readonly(fecc, data, parity, max_bad=0, seed=0, mem=None):
    """rs_scrub_dev, asserting that the buffers (or the whole allocation `mem` they are views of) are unchanged"""
    import torch
    keep = [m.clone() for m in (mem if mem is not None else (data, parity))]
    out = fecc.rs_scrub_dev(data, parity, max_bad, seed)
    for a, b in zip(mem if mem is not None else (data, parity), keep):
        assert torch.equal(a, b), "scrub wrote into the stripe"
    return out


def corrupt_rows(t, rows, gen, one_word=False):
    """Adds a nonzero value mod P to every word (or one random word) of the listed rows, in place"""
    import torch
    if not len(rows):
        return
    idx = torch.as_tensor(rows, device="cuda")
    old = u64(t[idx])
    delta = torch.randint(1, P, old.shape, device="cuda", generator=gen, dtype=torch.int64)
    if one_word:
        col = torch.randint(0, t.shape[1], (len(rows), 1), device="cuda", generator=gen)
        delta = delta * (torch.arange(t.shape[1], device="cuda")[None, :] == col)
    t[idx] = i32((old % P + delta) % P)


def pick(rng, n, k):
    return sorted(rng.choice(n, size=k, replace=False).tolist())


def mixed(rng, N, M, t):
    nd = int(rng.integers(max(0, t - M), min(t, N) + 1))
    return pick(rng, N, nd), pick(rng, M, t - nd)


# ---- small stripes against the Python pipeline ------------------------------------------------------------------------
SMALL = [(N, M) for N in (1, 2, 4, 8, 12, 16, 18, 36, 48, 72) for M in range(1, N + 1) if N % M == 0 and (N <= 18 or M in (1, 2, N // 4, N // 2, N))]


@pytest.mark.gpu
@pytest.mark.parametrize("N,M", SMALL)
def test_small_stripes_equal_the_python_pipeline(fecc, N, M):
    import torch
    rng = np.random.default_rng(N * 100 + M)
    gen = torch.Generator(device="cuda"); gen.manual_seed(N * 100 + M)
    for S in (5, 8):
        data = padded(i32(rand_words(N, S, gen))); parity = encode(fecc, data, M)
        for t in sorted({0, 1, M // 2, M // 2 + 1, M} & set(range(0, M + 1))):
            for max_bad in sorted({0, M // 2, M // 4}):
                d, p = padded(data), padded(parity)
                bd, bp = mixed(rng, N, M, t)
                corrupt_rows(d, bd, gen, one_word=t % 2 == 1); corrupt_rows(p, bp, gen)
                seed = int(rng.integers(1 << 64, dtype=np.uint64))
                got = scrub_readonly(fecc, d, p, max_bad, seed)
                want = py_scrub(u64(d).tolist(), u64(p).tolist(), max_bad, seed)
                assert got == want, (N, M, S, t, max_bad, bd, bp, got, want)
                if t == 0:
                    assert got[0] == CLEAN
                elif t <= max_bad:
                    assert got == (LOCATED, bd, bp)


def torch_scrub(data, parity, max_bad, seed):
    """The five steps of test_scrub_algebra.scrub in torch int64 on the device, with gfp_ref's encode by definition and transforms
    (no library code), for stripes too large for pure Python: the same (status, bad data, bad parity)"""
    import torch
    import gfp_ref as g
    from test_scrub_algebra import berlekamp_massey
    N, S = data.shape
    M = parity.shape[0]
    dev = data.device
    s = []
    for f in (0, 1):
        w = torch.tensor([weight(seed, f, c) for c in range(S)], dtype=torch.int64, device=dev)
        a = g.mulmod(u64(data) % P, w[None, :]).sum(1) % P                       # the fold, the SIZE words only
        b = g.mulmod(u64(parity) % P, w[None, :]).sum(1) % P
        G = g.encode_rows(a[:, None], [(N // M) * j for j in range(M)])[:, 0]
        s.append((b - G) % P)
    if not bool(s[0].any()) and not bool(s[1].any()):
        return CLEAN, [], []
    if max_bad == 0:
        return DETECTED, [], []
    S_hat = g.ntt_rows(s[0][:, None], range(2 * max_bad), inverse=True)[:, 0].tolist()
    Cz, L = berlekamp_massey(S_hat)
    if L > max_bad or len(Cz) - 1 != L:
        return DETECTED, [], []

    def horner(x):                                                                 # C(x) for a tensor of points
        acc = torch.zeros_like(x)
        for c in reversed(Cz):
            acc = (g.mulmod(acc, x) + c) % P
        return acc
    j = torch.arange(M, dtype=torch.int64, device=dev)
    Chat = horner(g.powers(M, dev)(j))                                             # C(zeta^j)
    for f in (0, 1):
        back = g.ntt_rows(g.mulmod(Chat, s[f])[:, None], range(L, M), inverse=True)
        if bool(back.any()):
            return DETECTED, [], []
    i = torch.arange(N, dtype=torch.int64, device=dev)
    Cd = horner(g.powers(2 * N, dev)(2 * i - 1 + 2 * N))                           # C(rho^-1 omega^i)
    bad_d, bad_p = (Cd == 0).nonzero().flatten().tolist(), (Chat == 0).nonzero().flatten().tolist()
    if len(bad_d) + len(bad_p) != L:
        return DETECTED, [], []
    return LOCATED, bad_d, bad_p


@pytest.mark.gpu
@pytest.mark.parametrize("N,M,S", [(1024, 1024, 5), (3 << 10, 3 << 8, 8), (9 << 10, 1 << 10, 5), (9 << 10, 9 << 10, 8)])
def test_larger_stripes_equal_the_torch_pipeline(fecc, N, M, S):
    """Up to 9 * 1024 rows: every result equal to the torch restatement of the five steps, random garbage in the pad words"""
    import torch
    rng = np.random.default_rng(N + M + S)
    gen = torch.Generator(device="cuda"); gen.manual_seed(N + M + S)
    data = padded(i32(rand_words(N, S, gen))); parity = encode(fecc, data, M)
    for t, max_bad in ((0, 8), (1, 8), (3, 0), (8, 8), (9, 8), (M // 2 + 1, 1)):
        d, p = padded(data), padded(parity)
        bd, bp = mixed(rng, N, M, t)
        corrupt_rows(d, bd, gen, one_word=t == 1); corrupt_rows(p, bp, gen)
        seed = int(rng.integers(1 << 64, dtype=np.uint64))
        got = scrub_readonly(fecc, d, p, max_bad, seed)
        assert got == torch_scrub(d, p, max_bad, seed), (N, M, S, t, max_bad, got)
        if t <= max_bad:
            assert got == ((CLEAN, [], []) if t == 0 else (LOCATED, bd, bp))
        elif t <= M - max_bad:
            assert got == (DETECTED, [], [])


def null_space_error(seed, cols):
    """A nonzero error on three columns that both folds with the header's weights map to zero: the cross product of the weight
    vectors of fold 0 and fold 1 on those columns"""
    a = [weight(seed, 0, c) for c in cols]
    b = [weight(seed, 1, c) for c in cols]
    return [(a[1] * b[2] - a[2] * b[1]) % P, (a[2] * b[0] - a[0] * b[2]) % P, (a[0] * b[1] - a[1] * b[0]) % P]


@pytest.mark.gpu
@pytest.mark.parametrize("N,M,S", [(12, 4, 7), (9 << 10, 9 << 6, 5), (3 << 10, 3 << 10, 8), (1 << 12, 1 << 6, 1030), (16, 8, 5000)])
def test_the_fold_uses_the_header_weights(fecc, N, M, S):
    """An error in the null space of the header's weights for `seed` is invisible (CLEAN); under another seed it is located.
    Columns across 16-byte groups and column tiles, the last (partial) group included, in a data and in a parity row."""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(N + S)
    data = padded(i32(rand_words(N, S, gen))); parity = encode(fecc, data, M)
    for seed in (0, 0xDEADBEEF12345678):
        for target, row in ((data, N - 1), (parity, M // 2)):
            cols = [0, S // 2, S - 1] if S > 2 else [0, 1, 2]
            e = null_space_error(seed, cols)
            old = target.clone()
            w = u64(target[row])
            for c, v in zip(cols, e):
                w[c] = (w[c] + v) % P
            target[row] = i32(w)
            assert fecc.rs_scrub_dev(data, parity, 1, seed) == (CLEAN, [], [])
            want = (LOCATED, [row], []) if target is data else (LOCATED, [], [row])
            assert fecc.rs_scrub_dev(data, parity, 1, seed + 1) == want
            target.copy_(old)


# ---- full-size stripes ---------------------------------------------------------------------------------------------------
def full_size(fecc, N, M, S, seed):
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(seed)
    rng = np.random.default_rng(seed)
    pitch = (S + 3) // 4 * 4 + 4
    dbuf = torch.full((N, pitch), SENTINEL, dtype=torch.int32, device="cuda")
    pbuf = torch.full((M, pitch), SENTINEL, dtype=torch.int32, device="cuda")
    data, parity = dbuf[:, :S], pbuf[:, :S]
    data.copy_(i32(rand_words(N, S, gen)))
    tmp = data.clone(); fecc.rs_encode_asym_mixed_dev(tmp, M); parity.copy_(tmp[:M]); del tmp
    torch.cuda.empty_cache()
    max_bad = min(M // 2, 4096)
    mem = (dbuf, pbuf)
    assert scrub_readonly(fecc, data, parity, max_bad, 1, mem) == (CLEAN, [], [])
    dbuf[:, S:] = garbage((N, pitch - S), gen); pbuf[:, S:] = garbage((M, pitch - S), gen)     # random garbage in the pad words only
    assert scrub_readonly(fecc, data, parity, max_bad, 2, mem) == (CLEAN, [], [])
    small = (u64(data) < C) & (torch.rand(data.shape, device="cuda", generator=gen) < 0.5)
    raw = padded(data); raw[small] = i32(u64(data)[small] + P)         # raw words >= P congruent to the stored ones
    assert scrub_readonly(fecc, raw, parity, max_bad, 3, (raw, pbuf)) == (CLEAN, [], [])
    del raw, small
    torch.cuda.empty_cache()
    for t in sorted({1, 3, 17, max_bad} & set(range(1, max_bad + 1))):
        bd, bp = mixed(rng, N, M, t)
        d0, p0 = data[bd].clone() if bd else None, parity[bp].clone() if bp else None
        corrupt_rows(data, bd, gen, one_word=t == 1); corrupt_rows(parity, bp, gen, one_word=t == 3)
        assert scrub_readonly(fecc, data, parity, max_bad, t, mem) == (LOCATED, bd, bp), (N, M, t)
        if bd:
            data[bd] = d0
        if bp:
            parity[bp] = p0
    row, col = int(rng.integers(N)), S - 1                            # one word of one column, the last of the row
    data[row, col] = i32(torch.tensor([(int(u64(data[row, col])) + 1) % P], device="cuda"))[0]
    assert scrub_readonly(fecc, data, parity, 1 if max_bad else 0, 9, mem) == ((LOCATED, [row], []) if max_bad else (DETECTED, [], []))
    del dbuf, pbuf, data, parity
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("M_div", [1, 16])
def test_full_size_2p19_4k_blocks(fecc, M_div):
    full_size(fecc, 1 << 19, (1 << 19) // M_div, 1024, 11 + M_div)


@pytest.mark.gpu
def test_full_size_9x2p19(fecc):
    """SIZE 15: the pad word of every row's last 16-byte group is loaded with it and must stay out of the sums"""
    full_size(fecc, 9 << 19, 1 << 19, 15, 99)


# ---- life cycle: update, corruption, scrub, repair, scrub ------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N,M,S", [(1 << 13, 1 << 13, 64), (3 << 12, 1 << 12, 37), (9 << 10, 1 << 10, 16), (1 << 19, 1 << 19, 1024)])
def test_scrub_repair_scrub_gives_the_stripe_back(fecc, N, M, S):
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(N + S)
    rng = np.random.default_rng(N + S)
    data = padded(i32(rand_words(N, S, gen))); parity = encode(fecc, data, M)
    changed = pick(rng, N, 5)
    fecc.rs_update_dev(data, parity, changed, padded(i32(rand_words(5, S, gen))))
    want_d, want_p = data.clone(), parity.clone()
    max_bad = min(M // 2, 4096)
    for t in sorted({1, 2, max_bad // 3, max_bad} - {0}):
        bd, bp = mixed(rng, N, M, t)
        if bd and changed[0] not in bd:                             # an updated block among the corrupted ones
            bd = sorted(bd[1:] + [changed[0]])
        corrupt_rows(data, bd, gen); corrupt_rows(parity, bp, gen)
        status, gd, gp = fecc.rs_scrub_dev(data, parity, max_bad, t)
        assert (status, gd, gp) == (LOCATED, bd, bp), (N, M, t)
        fecc.rs_repair_dev(data, parity, gd, gp)
        assert fecc.rs_scrub_dev(data, parity, max_bad, t + 1) == (CLEAN, [], [])
        assert torch.equal(data, want_d) and torch.equal(parity, want_p), (N, M, t)
    del data, parity, want_d, want_p
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("N,M", [(1 << 12, 1 << 12), (3 << 10, 3 << 6), (9 << 8, 9), (64, 1), (4096, 1)])
def test_beyond_max_bad_is_detected(fecc, N, M):
    """max_bad < t <= M - max_bad gives DETECTED; M = 1 is detect only; never CLEAN for 1 <= t <= M"""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(N * M)
    rng = np.random.default_rng(N * M)
    S = 12
    data = padded(i32(rand_words(N, S, gen))); parity = encode(fecc, data, M)
    for max_bad in sorted({0, 1, M // 4, M // 2}):
        if max_bad > M // 2:
            continue
        for t in sorted({max_bad + 1, (M + 1) // 2, M - max_bad, M} & set(range(max_bad + 1, M + 1))):
            d, p = padded(data), padded(parity)
            bd, bp = mixed(rng, N, M, t)
            corrupt_rows(d, bd, gen); corrupt_rows(p, bp, gen)
            status, gd, gp = scrub_readonly(fecc, d, p, max_bad, t)
            assert status != CLEAN, (N, M, max_bad, t)
            if t <= M - max_bad:
                assert (status, gd, gp) == (DETECTED, [], []), (N, M, max_bad, t, bd, bp, gd, gp)


@pytest.mark.gpu
@pytest.mark.parametrize("S", [5, 6, 7, 13])
def test_pitches_parity_below_data_and_partial_groups(fecc, S):
    """Data and parity as views of one allocation, parity first, at three different pitches, with random garbage in every pad word
    (the partial last 16-byte group of every row included); CLEAN and the exact lists, the allocation byte-identical"""
    import torch
    N, M = 3 << 8, 3 << 5
    gen = torch.Generator(device="cuda"); gen.manual_seed(S)
    rng = np.random.default_rng(S)
    dpitch, ppitch = S + 12 - S % 4, S + 4 - S % 4
    poff = 4
    doff = poff + M * ppitch + 12
    mem = garbage((doff + N * dpitch + 4,), gen)
    pv = mem.as_strided((M, S), (ppitch, 1), poff)
    dv = mem.as_strided((N, S), (dpitch, 1), doff)
    src = i32(rand_words(N, S, gen))
    dv.copy_(src); pv.copy_(encode(fecc, src, M))
    assert scrub_readonly(fecc, dv, pv, M // 2, 1, (mem,)) == (CLEAN, [], [])
    for t in (1, 7, M // 2):
        bd, bp = mixed(rng, N, M, t)
        keep = mem.clone()
        corrupt_rows(dv, bd, gen, one_word=True); corrupt_rows(pv, bp, gen, one_word=True)
        assert scrub_readonly(fecc, dv, pv, M // 2, t, (mem,)) == (LOCATED, bd, bp), (S, t)
        mem.copy_(keep)
    # the same stripe read through data and parity views that overlap is legal: nothing is written
    assert fecc.rs_scrub_dev(dv, dv[:M], 0, 0)[0] in (CLEAN, DETECTED)


@pytest.mark.gpu
def test_scrub_repair_and_update_on_three_streams_from_two_threads(fecc):
    import torch
    from fastecc_b200 import decoder
    gen = torch.Generator(device="cuda"); gen.manual_seed(3)
    rng = np.random.default_rng(3)
    S = 64
    N1, M1 = 3 << 13, 3 << 9                                            # scrubbed
    d1 = padded(i32(rand_words(N1, S, gen))); p1 = encode(fecc, d1, M1)
    bd1, bp1 = mixed(rng, N1, M1, 9)
    corrupt_rows(d1, bd1, gen); corrupt_rows(p1, bp1, gen)
    N2, M2 = 1 << 14, 1 << 10                                           # repaired
    d2 = padded(i32(rand_words(N2, S, gen))); p2 = encode(fecc, d2, M2)
    want_d2, want_p2 = d2.clone(), p2.clone()
    lost_d, lost_p = pick(rng, N2, M2 // 2), pick(rng, M2, M2 // 2)
    d2[torch.as_tensor(lost_d, device="cuda")] = 1; p2[torch.as_tensor(lost_p, device="cuda")] = 2
    rep = decoder.Repair(N2, M2, lost_d, lost_p)
    N3, M3 = 9 << 11, 9 << 7                                            # updated
    d3 = padded(i32(rand_words(N3, S, gen))); p3 = encode(fecc, d3, M3)
    ch = pick(rng, N3, 6); nw = i32(rand_words(6, S, gen))
    want_d3 = d3.clone(); want_d3[torch.as_tensor(ch, device="cuda")] = nw
    want_p3 = encode(fecc, want_d3, M3)
    torch.cuda.synchronize()
    errors, results, streams = [], [], [torch.cuda.Stream() for _ in range(3)]

    def thread1():
        try:
            with torch.cuda.stream(streams[0]):
                results.append(fecc.rs_scrub_dev(d1, p1, 16, 5))
            with torch.cuda.stream(streams[2]):
                fecc.rs_update_dev(d3, p3, ch, nw)
        except Exception as e:                   # re-raised on the main thread
            errors.append(e)

    def thread2():
        try:
            with torch.cuda.stream(streams[1]):
                rep.repair(d2, p2)
        except Exception as e:
            errors.append(e)

    threads = [threading.Thread(target=thread1), threading.Thread(target=thread2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    torch.cuda.synchronize()
    rep.close()
    assert not errors, errors
    assert results == [(LOCATED, bd1, bp1)]
    assert torch.equal(d2, want_d2) and torch.equal(p2, want_p2)
    assert torch.equal(d3, want_d3) and torch.equal(p3, want_p3)


@pytest.mark.gpu
def test_scrub_argument_table(fecc):
    """Every rule of the validation broken on its own gives FASTECC_B200_EINVAL (-1), launches nothing and writes no output"""
    import ctypes
    import torch
    L = fecc.lib()
    st = torch.cuda.current_stream().cuda_stream
    buf = torch.zeros((64, 8), dtype=torch.int32, device="cuda")
    d, p = buf[:12].data_ptr(), buf[32:36].data_ptr()
    wrong = []

    def call(data=d, dpitch=8, N=12, parity=p, ppitch=8, M=4, S=8, max_bad=2, out=True, lists=True):
        status, nd, np_ = ctypes.c_int(-9), ctypes.c_size_t(99), ctypes.c_size_t(98)
        bd, bp = np.zeros(8, dtype=np.uint32), np.zeros(8, dtype=np.uint32)
        rc = L.fastecc_b200_rs_scrub(data, dpitch, N, parity, ppitch, M, S, max_bad, 1, st, ctypes.byref(status) if out else None,
                                     bd.ctypes.data if lists else None, ctypes.byref(nd), bp.ctypes.data if lists else None, ctypes.byref(np_))
        return rc, (status.value, nd.value, np_.value)

    cases = [({}, 0), (dict(S=5), 0), (dict(M=12, parity=buf[16:28].data_ptr(), max_bad=6), 0), (dict(M=1, max_bad=0), 0),
             (dict(parity=d), 0), (dict(max_bad=0, lists=False), 0),
             (dict(N=5), -1), (dict(N=27), -1), (dict(N=3 << 20, M=3, max_bad=1), -1), (dict(M=0), -1), (dict(M=5), -1), (dict(M=24), -1),
             (dict(S=0), -1), (dict(data=None), -1), (dict(parity=None), -1), (dict(out=False), -1), (dict(lists=False), -1),
             (dict(max_bad=3), -1), (dict(M=1, max_bad=1), -1), (dict(dpitch=6, S=6), -1), (dict(ppitch=6, S=6), -1),
             (dict(dpitch=4), -1), (dict(ppitch=4), -1), (dict(data=d + 4, S=4), -1), (dict(parity=p + 8, S=4), -1)]
    for kw, want in cases:
        n0 = fecc.kernel_launches()
        rc, outs = call(**kw)
        if rc != want or (want and (fecc.kernel_launches() != n0 or outs != (-9, 99, 98))):
            wrong.append((kw, rc, outs))
    status, nd, np_ = ctypes.c_int(), ctypes.c_size_t(), ctypes.c_size_t()
    big = np.zeros(1, dtype=np.uint32)
    huge = torch.zeros((1 << 14, 4), dtype=torch.int32, device="cuda")
    rc = L.fastecc_b200_rs_scrub(huge.data_ptr(), 4, 1 << 14, huge.data_ptr(), 4, 1 << 14, 4, 4097, 0, st, ctypes.byref(status),
                                 big.ctypes.data, ctypes.byref(nd), big.ctypes.data, ctypes.byref(np_))
    if rc != -1:
        wrong.append(("max_bad 4097", rc))
    torch.cuda.synchronize()
    assert not wrong, wrong


@pytest.mark.gpu
def test_scrub_before_init_is_enoinit():
    code = ("import sys; sys.path.insert(0, %r); import fastecc_b200 as fe; L = fe.lib(); "
            "print(L.fastecc_b200_rs_scrub(None, 4, 12, None, 4, 4, 4, 0, 0, None, None, None, None, None, None))") % ROOT
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.stdout.split() == ["-4"], out.stdout + out.stderr
