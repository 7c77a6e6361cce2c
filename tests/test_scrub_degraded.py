"""GPU: scrub of a degraded stripe (fastecc_b200_rs_scrub_degraded, decoder.Repair.scrub, csrc/scrub.cu, DESIGN 3j).  Small stripes
are compared with the Python pipeline of test_scrub_degraded_algebra.py, larger ones with a torch restatement on gfp_ref's encode
and transforms, full-size ones with the set that was corrupted.  The lost rows hold garbage in every test (they are never read),
the pad words of partial last groups hold random garbage, and every call is checked to leave both buffers byte-identical."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

from test_scrub import SENTINEL, corrupt_rows, encode, garbage, i32, padded, pick, rand_words, u64
from test_scrub_algebra import CLEAN, DETECTED, LOCATED, weight
from test_scrub_degraded_algebra import scrub_degraded as py_scrub_degraded

P = 0xFFF00001
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def scrub_readonly(rep, data, parity, max_bad=0, seed=0, mem=None):
    """Repair.scrub, asserting that the buffers (or the whole allocations `mem` they are views of) are unchanged"""
    import torch
    keep = [m.clone() for m in (mem if mem is not None else (data, parity))]
    out = rep.scrub(data, parity, max_bad, seed)
    for a, b in zip(mem if mem is not None else (data, parity), keep):
        assert torch.equal(a, b), "the degraded scrub wrote into the stripe"
    assert not set(out[1]) & set(rep.lost_data) and not set(out[2]) & set(rep.lost_parity), ("a lost block was named", out)
    return out


def lose(rng, N, M, f):
    """f lost blocks, data and parity mixed"""
    nd = int(rng.integers(max(0, f - M), min(f, N) + 1))
    return pick(rng, N, nd), pick(rng, M, f - nd)


def survivors(rng, N, M, lost_d, lost_p, t):
    """t corrupted blocks among the survivors, data and parity mixed"""
    sd, sp = np.setdiff1d(np.arange(N), lost_d), np.setdiff1d(np.arange(M), lost_p)
    nd = int(rng.integers(max(0, t - len(sp)), min(t, len(sd)) + 1))
    return sorted(rng.choice(sd, size=nd, replace=False).tolist()), sorted(rng.choice(sp, size=t - nd, replace=False).tolist())


def fill(t, rows, gen=None, value=None):
    """The listed rows overwritten with random 32-bit garbage, or with `value` in every word"""
    import torch
    if len(rows):
        idx = torch.as_tensor(rows, device="cuda")
        t[idx] = garbage((len(rows), t.shape[1]), gen) if value is None else torch.full((len(rows), t.shape[1]), value, dtype=torch.int32, device="cuda")


def status_for(t, max_bad, room, bd, bp, got):
    """The guarantees of the header with room = M - f"""
    if t == 0:
        assert got == (CLEAN, [], []), got
    else:
        assert got[0] != CLEAN, got
    if 1 <= t <= max_bad:
        assert got == (LOCATED, bd, bp), (bd, bp, got)
    elif max_bad < t <= room - max_bad:
        assert got == (DETECTED, [], []), got


# ---- small stripes against the Python pipeline ------------------------------------------------------------------------
SMALL = [(N, M) for N in (2, 4, 8, 12, 16, 18, 36, 48, 72) for M in range(2, N + 1) if N % M == 0 and (N <= 18 or M in (2, N // 4, N // 2, N))]


@pytest.mark.gpu
@pytest.mark.parametrize("N,M", SMALL)
def test_small_stripes_equal_the_python_pipeline(fecc, N, M):
    import torch
    from fastecc_b200.decoder import Repair
    rng = np.random.default_rng(N * 100 + M + 7)
    gen = torch.Generator(device="cuda"); gen.manual_seed(N * 100 + M + 7)
    for S in (5, 8):
        data = padded(i32(rand_words(N, S, gen))); parity = encode(fecc, data, M)
        for f in sorted({1, M // 4, M // 2, M - 1} & set(range(1, M))):
            lost_d, lost_p = lose(rng, N, M, f)
            rep = Repair(N, M, lost_d, lost_p)
            room = M - f
            for t in sorted({0, 1, room // 2, room // 2 + 1, room} & set(range(room + 1))):
                for max_bad in sorted({0, room // 2}):
                    d, p = padded(data), padded(parity)
                    bd, bp = survivors(rng, N, M, lost_d, lost_p, t)
                    corrupt_rows(d, bd, gen, one_word=t % 2 == 1); corrupt_rows(p, bp, gen)
                    fill(d, lost_d, gen); fill(p, lost_p, gen)
                    seed = int(rng.integers(1 << 64, dtype=np.uint64))
                    got = scrub_readonly(rep, d, p, max_bad, seed)
                    want = py_scrub_degraded(u64(d).tolist(), u64(p).tolist(), lost_d, lost_p, max_bad, seed)
                    assert got == want, (N, M, S, f, lost_d, lost_p, t, max_bad, bd, bp, got, want)
                    status_for(t, max_bad, room, bd, bp, got)
            rep.close()


def torch_scrub_degraded(data, parity, lost_d, lost_p, max_bad, seed):
    """The five steps of test_scrub_degraded_algebra.scrub_degraded in torch int64 on the device, with gfp_ref's encode by
    definition and transforms (no library code), for stripes too large for pure Python"""
    import torch
    import gfp_ref as g
    from test_scrub_algebra import berlekamp_massey
    N, S = data.shape
    M = parity.shape[0]
    dev, D = data.device, N // M
    f = len(lost_d) + len(lost_p)
    pw = g.powers(2 * N, dev)
    j = torch.arange(M, dtype=torch.int64, device=dev)
    y = pw(2 * D * j + 1)
    l = torch.ones_like(y)
    for z in pw(torch.tensor([2 * e for e in lost_d] + [2 * D * q + 1 for q in lost_p], dtype=torch.int64, device=dev)).tolist():
        l = g.mulmod(l, (y - z) % P)
    cs = g.mulmod((P - l) % P, torch.full_like(l, (P + 1) // 2))                   # -l_E(y_j) / 2
    dz, pz = u64(data) % P, u64(parity) % P
    if lost_d:
        dz[torch.as_tensor(lost_d, device=dev)] = 0                                # never loaded
    if lost_p:
        pz[torch.as_tensor(lost_p, device=dev)] = 0
    u, U = [], []
    for fo in (0, 1):
        w = torch.tensor([weight(seed, fo, c) for c in range(S)], dtype=torch.int64, device=dev)
        a = g.mulmod(dz, w[None, :]).sum(1) % P
        b = g.mulmod(pz, w[None, :]).sum(1) % P
        G = g.encode_rows(a[:, None], [D * q for q in range(M)])[:, 0]
        u.append(g.mulmod((b - G) % P, cs))
        U.append(g.ntt_rows(u[fo][:, None], range(f, M), inverse=True)[:, 0])
    if not bool(U[0].any()) and not bool(U[1].any()):
        return CLEAN, [], []
    if max_bad == 0:
        return DETECTED, [], []
    Cz, L = berlekamp_massey(U[0][:2 * max_bad].tolist())
    if L > max_bad or len(Cz) - 1 != L:
        return DETECTED, [], []

    def horner(x):
        acc = torch.zeros_like(x)
        for c in reversed(Cz):
            acc = (g.mulmod(acc, x) + c) % P
        return acc
    Chat = horner(g.powers(M, dev)(j))
    for fo in (0, 1):
        if bool(g.ntt_rows(g.mulmod(Chat, u[fo])[:, None], range(f + L, M), inverse=True).any()):
            return DETECTED, [], []
    i = torch.arange(N, dtype=torch.int64, device=dev)
    Cd = horner(pw(2 * i - 1 + 2 * N))                                             # C(rho^-1 omega^i)
    live = torch.ones(N, dtype=torch.bool, device=dev)
    if lost_d:
        live[torch.as_tensor(lost_d, device=dev)] = False
    bad_d = ((Cd == 0) & live).nonzero().flatten().tolist()
    bad_p = ((Chat == 0) & (cs != 0)).nonzero().flatten().tolist()
    if len(bad_d) + len(bad_p) != L:
        return DETECTED, [], []
    return LOCATED, bad_d, bad_p


@pytest.mark.gpu
@pytest.mark.parametrize("N,M,S", [(1024, 1024, 5), (3 << 10, 3 << 8, 8), (9 << 10, 1 << 10, 5), (3 << 10, 3 << 10, 8)])
def test_larger_stripes_equal_the_torch_pipeline(fecc, N, M, S):
    import torch
    from fastecc_b200.decoder import Repair
    rng = np.random.default_rng(N + M + S + 1)
    gen = torch.Generator(device="cuda"); gen.manual_seed(N + M + S + 1)
    data = padded(i32(rand_words(N, S, gen))); parity = encode(fecc, data, M)
    for f in (1, 17, M // 4):
        lost_d, lost_p = lose(rng, N, M, f)
        rep = Repair(N, M, lost_d, lost_p)
        room = M - f
        for t, max_bad in ((0, 8), (1, 8), (3, 0), (8, 8), (9, 8), (room // 2 + 1, 1)):
            d, p = padded(data), padded(parity)
            bd, bp = survivors(rng, N, M, lost_d, lost_p, t)
            corrupt_rows(d, bd, gen, one_word=t == 1); corrupt_rows(p, bp, gen)
            fill(d, lost_d, gen); fill(p, lost_p, gen)
            seed = int(rng.integers(1 << 64, dtype=np.uint64))
            got = scrub_readonly(rep, d, p, max_bad, seed)
            assert got == torch_scrub_degraded(d, p, lost_d, lost_p, max_bad, seed), (N, M, S, f, t, max_bad, got)
            status_for(t, max_bad, room, bd, bp, got)
        rep.close()


@pytest.mark.gpu
@pytest.mark.parametrize("N,M,S", [(3 << 10, 3 << 8, 7), (1 << 12, 1 << 12, 6), (9 << 8, 9 << 4, 1030)])
def test_the_lost_rows_are_never_read(fecc, N, M, S):
    """Two different random garbage fillings of the lost rows and 0xFFFFFFFF in every word give identical results"""
    import torch
    from fastecc_b200.decoder import Repair
    rng = np.random.default_rng(N + S)
    gen = torch.Generator(device="cuda"); gen.manual_seed(N + S)
    data = padded(i32(rand_words(N, S, gen))); parity = encode(fecc, data, M)
    for f in (1, 50, M // 2):
        lost_d, lost_p = lose(rng, N, M, f)
        rep = Repair(N, M, lost_d, lost_p)
        max_bad = min((M - f) // 2, 8)
        for t in (0, 1, 5):
            d, p = padded(data), padded(parity)
            bd, bp = survivors(rng, N, M, lost_d, lost_p, t)
            corrupt_rows(d, bd, gen); corrupt_rows(p, bp, gen, one_word=True)
            seen = []
            for value in (None, None, -1):
                fill(d, lost_d, gen, value); fill(p, lost_p, gen, value)
                seen.append(scrub_readonly(rep, d, p, max_bad, t))
            assert seen[0] == seen[1] == seen[2] == ((CLEAN, [], []) if t == 0 else (LOCATED, bd, bp)), (N, M, f, t, seen)
        rep.close()


@pytest.mark.gpu
@pytest.mark.parametrize("N,M,S", [(12, 4, 5), (1024, 256, 8), (9 << 10, 1 << 10, 13), (3 << 12, 3 << 12, 6), (64, 1, 7)])
def test_nothing_lost_is_the_plain_scrub(fecc, N, M, S):
    """A pattern with nothing lost gives what rs_scrub_dev gives, with as many kernel launches"""
    import torch
    from fastecc_b200.decoder import Repair
    rng = np.random.default_rng(N * M + S)
    gen = torch.Generator(device="cuda"); gen.manual_seed(N * M + S)
    data = padded(i32(rand_words(N, S, gen))); parity = encode(fecc, data, M)
    rep = Repair(N, M)
    top = min(M // 2, 4096)
    for t in sorted({0, 1, top, top + 1, M} & set(range(M + 1))):
        for max_bad in sorted({0, top}):
            d, p = padded(data), padded(parity)
            bd, bp = survivors(rng, N, M, [], [], t)
            corrupt_rows(d, bd, gen); corrupt_rows(p, bp, gen)
            for seed in (0, int(rng.integers(1 << 64, dtype=np.uint64))):
                n0 = fecc.kernel_launches()
                want = fecc.rs_scrub_dev(d, p, max_bad, seed)
                n1 = fecc.kernel_launches()
                got = scrub_readonly(rep, d, p, max_bad, seed)
                n2 = fecc.kernel_launches()
                assert got == want and n2 - n1 == n1 - n0, (N, M, t, max_bad, got, want, n1 - n0, n2 - n1)
                assert fecc.rs_scrub_degraded_dev(d, p, [], [], max_bad, seed) == want
    rep.close()


# ---- full-size stripes ---------------------------------------------------------------------------------------------------
def full_size(fecc, N, M, S, seed, fs):
    import torch
    from fastecc_b200.decoder import Repair
    gen = torch.Generator(device="cuda"); gen.manual_seed(seed)
    rng = np.random.default_rng(seed)
    pitch = (S + 3) // 4 * 4 + 4
    dbuf = torch.full((N, pitch), SENTINEL, dtype=torch.int32, device="cuda")
    pbuf = torch.full((M, pitch), SENTINEL, dtype=torch.int32, device="cuda")
    data, parity = dbuf[:, :S], pbuf[:, :S]
    data.copy_(i32(rand_words(N, S, gen)))
    tmp = data.clone(); fecc.rs_encode_asym_mixed_dev(tmp, M); parity.copy_(tmp[:M]); del tmp
    dbuf[:, S:] = garbage((N, pitch - S), gen); pbuf[:, S:] = garbage((M, pitch - S), gen)     # random garbage in the pad words
    torch.cuda.empty_cache()
    mem = (dbuf, pbuf)
    for f in fs:
        lost_d, lost_p = lose(rng, N, M, f)
        keep_d, keep_p = data[lost_d].clone(), parity[lost_p].clone()
        fill(data, lost_d, gen); fill(parity, lost_p, gen)
        rep = Repair(N, M, lost_d, lost_p)
        max_bad = min((M - f) // 2, 4096)
        for t in sorted({0, 1, 17, max_bad} & set(range(max_bad + 1))):
            bd, bp = survivors(rng, N, M, lost_d, lost_p, t)
            d0, p0 = data[bd].clone() if bd else None, parity[bp].clone() if bp else None
            corrupt_rows(data, bd, gen, one_word=t == 1); corrupt_rows(parity, bp, gen, one_word=t == 17)
            want = (CLEAN, [], []) if t == 0 else (LOCATED, bd, bp)
            assert scrub_readonly(rep, data, parity, max_bad, t, mem) == want, (N, M, f, t)
            if bd:
                data[bd] = d0
            if bp:
                parity[bp] = p0
        rep.close()
        if lost_d:
            data[lost_d] = keep_d
        if lost_p:
            parity[lost_p] = keep_p
        del keep_d, keep_p
    del dbuf, pbuf, data, parity
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("M_div", [1, 16])
def test_full_size_2p19_4k_blocks(fecc, M_div):
    M = (1 << 19) // M_div
    full_size(fecc, 1 << 19, M, 1024, 21 + M_div, (1, 64, M // 4))


@pytest.mark.gpu
def test_full_size_9x2p19(fecc):
    """SIZE 15: the pad word of every row's last 16-byte group is loaded with it and must stay out of the sums"""
    M = 1 << 19
    full_size(fecc, 9 << 19, M, 15, 98, (1, 64, M // 4))


# ---- life cycle: lose, corrupt, scrub the survivors, repair, scrub --------------------------------------------------------
def merged(a, b):
    return sorted(set(a) | set(b))


@pytest.mark.gpu
@pytest.mark.parametrize("N,M,S", [(1 << 13, 1 << 13, 64), (3 << 12, 1 << 12, 37), (9 << 10, 1 << 10, 16), (1 << 19, 1 << 19, 1024)])
def test_scrub_survivors_then_repair_gives_the_stripe_back(fecc, N, M, S):
    import torch
    from fastecc_b200.decoder import Repair
    gen = torch.Generator(device="cuda"); gen.manual_seed(N + S + 3)
    rng = np.random.default_rng(N + S + 3)
    data = padded(i32(rand_words(N, S, gen))); parity = encode(fecc, data, M)
    want_d, want_p = data.clone(), parity.clone()
    for f in sorted({1, 16, M // 4}):
        lost_d, lost_p = lose(rng, N, M, f)
        max_bad = min((M - f) // 2, 4096)
        rep = Repair(N, M, lost_d, lost_p)
        for t in sorted({0, 1, 2, max_bad // 3, max_bad}):
            bd, bp = survivors(rng, N, M, lost_d, lost_p, t)
            fill(data, lost_d, gen); fill(parity, lost_p, gen)
            corrupt_rows(data, bd, gen); corrupt_rows(parity, bp, gen)
            status, gd, gp = rep.scrub(data, parity, max_bad, t)
            if t == 0:
                assert (status, gd, gp) == (CLEAN, [], [])
                rep.repair(data, parity)                                      # the same pattern
            else:
                assert (status, gd, gp) == (LOCATED, bd, bp), (N, M, f, t)
                both = Repair(N, M, merged(lost_d, gd), merged(lost_p, gp))
                both.repair(data, parity)
                both.close()
            assert fecc.rs_scrub_dev(data, parity, min(M // 2, 4096), t + 1) == (CLEAN, [], [])
            assert torch.equal(data, want_d) and torch.equal(parity, want_p), (N, M, f, t)
        rep.close()
    del data, parity, want_d, want_p
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_repair_without_the_scrub_rebuilds_wrong_blocks(fecc):
    """The plain route: a repair from survivors of which one is corrupted leaves a stripe that differs from the original in the
    rebuilt blocks; the degraded scrub names the bad survivor, and the repair with it gives the original back"""
    import torch
    from fastecc_b200.decoder import Repair
    N, M, S = 3 << 10, 3 << 8, 24
    gen = torch.Generator(device="cuda"); gen.manual_seed(5)
    rng = np.random.default_rng(5)
    data = padded(i32(rand_words(N, S, gen))); parity = encode(fecc, data, M)
    want_d, want_p = data.clone(), parity.clone()
    lost_d, lost_p = lose(rng, N, M, 40)
    bd, bp = survivors(rng, N, M, lost_d, lost_p, 1)
    fill(data, lost_d, gen); fill(parity, lost_p, gen)
    corrupt_rows(data, bd, gen); corrupt_rows(parity, bp, gen)
    plain_d, plain_p = data.clone(), parity.clone()
    rep = Repair(N, M, lost_d, lost_p)
    rep.repair(plain_d, plain_p)
    assert not torch.equal(plain_d[lost_d], want_d[lost_d]) or not torch.equal(plain_p[lost_p], want_p[lost_p])
    assert rep.scrub(data, parity, 4, 1) == (LOCATED, bd, bp)
    both = Repair(N, M, merged(lost_d, bd), merged(lost_p, bp))
    both.repair(data, parity)
    assert torch.equal(data, want_d) and torch.equal(parity, want_p)
    rep.close(); both.close()


@pytest.mark.gpu
@pytest.mark.parametrize("N,M", [(1024, 16), (3 << 8, 3 << 4), (9 << 6, 9), (64, 2)])
def test_one_check_symbol_left_detects_a_bad_survivor(fecc, N, M):
    """f = M - 1: detect only; CLEAN on a clean stripe, DETECTED with one corrupted survivor (data or parity)"""
    import torch
    from fastecc_b200.decoder import Repair
    gen = torch.Generator(device="cuda"); gen.manual_seed(N + M)
    rng = np.random.default_rng(N + M)
    S = 9
    data = padded(i32(rand_words(N, S, gen))); parity = encode(fecc, data, M)
    for lost_d, lost_p in (lose(rng, N, M, M - 1), (pick(rng, N, M - 1), [])):
        rep = Repair(N, M, lost_d, lost_p)
        d, p = padded(data), padded(parity)
        fill(d, lost_d, gen); fill(p, lost_p, gen)
        assert scrub_readonly(rep, d, p, 0, 1) == (CLEAN, [], [])
        for bd, bp in (survivors(rng, N, M, lost_d, lost_p, 1), (pick(rng, N, 0), [j for j in range(M) if j not in lost_p][:1])):
            d2, p2 = padded(d), padded(p)
            corrupt_rows(d2, bd, gen, one_word=True); corrupt_rows(p2, bp, gen, one_word=True)
            assert scrub_readonly(rep, d2, p2, 0, 2) == (DETECTED, [], []), (N, M, lost_d, lost_p, bd, bp)
        rep.close()


@pytest.mark.gpu
@pytest.mark.parametrize("S", [5, 6, 7, 13])
def test_pitches_parity_below_data_and_partial_groups(fecc, S):
    """Data and parity as views of one allocation, parity first, at three different pitches, with random garbage in every pad word
    and in the lost rows; CLEAN and the exact lists, the allocation byte-identical"""
    import torch
    from fastecc_b200.decoder import Repair
    N, M = 3 << 8, 3 << 5
    gen = torch.Generator(device="cuda"); gen.manual_seed(S + 50)
    rng = np.random.default_rng(S + 50)
    dpitch, ppitch = S + 12 - S % 4, S + 4 - S % 4
    poff = 4
    doff = poff + M * ppitch + 12
    mem = garbage((doff + N * dpitch + 4,), gen)
    pv = mem.as_strided((M, S), (ppitch, 1), poff)
    dv = mem.as_strided((N, S), (dpitch, 1), doff)
    src = i32(rand_words(N, S, gen))
    dv.copy_(src); pv.copy_(encode(fecc, src, M))
    lost_d, lost_p = lose(rng, N, M, 20)
    fill(dv, lost_d, gen); fill(pv, lost_p, gen)
    rep = Repair(N, M, lost_d, lost_p)
    room = M - 20
    assert scrub_readonly(rep, dv, pv, room // 2, 1, (mem,)) == (CLEAN, [], [])
    for t in (1, 7, room // 2):
        bd, bp = survivors(rng, N, M, lost_d, lost_p, t)
        keep = mem.clone()
        corrupt_rows(dv, bd, gen, one_word=True); corrupt_rows(pv, bp, gen, one_word=True)
        assert scrub_readonly(rep, dv, pv, room // 2, t, (mem,)) == (LOCATED, bd, bp), (S, t)
        mem.copy_(keep)
    # the same stripe read through data and parity views that overlap is legal: nothing is written
    assert rep.scrub(dv, dv[:M], 0, 0)[0] in (CLEAN, DETECTED)
    rep.close()


@pytest.mark.gpu
def test_degraded_scrub_repair_and_update_on_three_streams_from_two_threads(fecc):
    import torch
    from fastecc_b200 import decoder
    gen = torch.Generator(device="cuda"); gen.manual_seed(4)
    rng = np.random.default_rng(4)
    S = 64
    N1, M1 = 3 << 13, 3 << 9                                            # scrubbed, degraded
    d1 = padded(i32(rand_words(N1, S, gen))); p1 = encode(fecc, d1, M1)
    ld1, lp1 = lose(rng, N1, M1, 100)
    bd1, bp1 = survivors(rng, N1, M1, ld1, lp1, 9)
    fill(d1, ld1, gen); fill(p1, lp1, gen)
    corrupt_rows(d1, bd1, gen); corrupt_rows(p1, bp1, gen)
    sc = decoder.Repair(N1, M1, ld1, lp1)
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
                results.append(sc.scrub(d1, p1, 16, 5))
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
    rep.close(); sc.close()
    assert not errors, errors
    assert results == [(LOCATED, bd1, bp1)]
    assert torch.equal(d2, want_d2) and torch.equal(p2, want_p2)
    assert torch.equal(d3, want_d3) and torch.equal(p3, want_p3)


@pytest.mark.gpu
def test_degraded_scrub_argument_table(fecc):
    """Every rule of the validation broken on its own gives FASTECC_B200_EINVAL (-1), launches nothing and writes no output"""
    import ctypes
    import torch
    from fastecc_b200.decoder import Repair
    L = fecc.lib()
    st = torch.cuda.current_stream().cuda_stream
    buf = torch.zeros((64, 8), dtype=torch.int32, device="cuda")
    d, p = buf[:12].data_ptr(), buf[32:36].data_ptr()
    one = Repair(12, 4, [1], [])                      # f = 1: max_bad <= 1
    two = Repair(12, 4, [3], [2])                     # f = 2: max_bad <= 1
    none = Repair(12, 4)                              # f = 0: the plain scrub, max_bad <= 2
    full = Repair(12, 4, [0, 5], [1, 3])              # f = M
    wide = Repair(12, 12, [], [4])                    # M = 12, f = 1: max_bad <= 5
    wrong = []

    def call(R=one, data=d, dpitch=8, parity=p, ppitch=8, S=8, max_bad=1, out=True, counts=True, lists=True):
        status, nd, np_ = ctypes.c_int(-9), ctypes.c_size_t(99), ctypes.c_size_t(98)
        bd, bp = np.zeros(8, dtype=np.uint32), np.zeros(8, dtype=np.uint32)
        rc = L.fastecc_b200_rs_scrub_degraded(R._h if R is not None else None, data, dpitch, parity, ppitch, S, max_bad, 1, st,
                                              ctypes.byref(status) if out else None, bd.ctypes.data if lists else None,
                                              ctypes.byref(nd) if counts else None, bp.ctypes.data if lists else None, ctypes.byref(np_))
        return rc, (status.value, nd.value, np_.value)

    cases = [({}, 0), (dict(S=5), 0), (dict(R=two), 0), (dict(R=none, max_bad=2), 0), (dict(R=wide, parity=buf[16:28].data_ptr(), max_bad=5), 0),
             (dict(parity=d), 0), (dict(max_bad=0, lists=False), 0),
             (dict(R=None), -1), (dict(out=False), -1), (dict(counts=False), -1), (dict(R=full, max_bad=0), -1),
             (dict(max_bad=2), -1), (dict(R=two, max_bad=2), -1), (dict(R=none, max_bad=3), -1),
             (dict(R=wide, parity=buf[16:28].data_ptr(), max_bad=6), -1), (dict(lists=False), -1),
             (dict(S=0), -1), (dict(data=None), -1), (dict(parity=None), -1), (dict(dpitch=6, S=6), -1), (dict(ppitch=6, S=6), -1),
             (dict(dpitch=4), -1), (dict(ppitch=4), -1), (dict(data=d + 4, S=4), -1), (dict(parity=p + 8, S=4), -1)]
    for kw, want in cases:
        n0 = fecc.kernel_launches()
        rc, outs = call(**kw)
        if rc != want or (want and (fecc.kernel_launches() != n0 or outs != (-9, 99, 98))):
            wrong.append((kw, rc, outs))
    status, nd, np_ = ctypes.c_int(), ctypes.c_size_t(), ctypes.c_size_t()
    big = np.zeros(1, dtype=np.uint32)
    huge = torch.zeros((1 << 14, 4), dtype=torch.int32, device="cuda")
    deep = Repair(1 << 14, 1 << 14, [7], [])                            # (M - f) / 2 = 8191: the cap of 4096 applies
    rc = L.fastecc_b200_rs_scrub_degraded(deep._h, huge.data_ptr(), 4, huge.data_ptr(), 4, 4, 4097, 0, st, ctypes.byref(status),
                                          big.ctypes.data, ctypes.byref(nd), big.ctypes.data, ctypes.byref(np_))
    if rc != -1:
        wrong.append(("max_bad 4097", rc))
    with pytest.raises(ValueError):
        one.scrub(buf[:11], buf[32:36])                                  # Python: rows that do not match the pattern
    torch.cuda.synchronize()
    for r in (one, two, none, full, wide, deep):
        r.close()
    assert not wrong, wrong


@pytest.mark.gpu
def test_degraded_scrub_before_init_is_enoinit():
    code = ("import sys; sys.path.insert(0, %r); import fastecc_b200 as fe; L = fe.lib(); "
            "print(L.fastecc_b200_rs_scrub_degraded(None, None, 4, None, 4, 4, 0, 0, None, None, None, None, None, None))") % ROOT
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.stdout.split() == ["-4"], out.stdout + out.stderr
