"""GPU: degraded read of a stored stripe (fastecc_b200_rs_reconstruct, csrc/reconstruct.cu, DESIGN 3k).  Every result is compared
bit for bit with the blocks as the encode by definition (tests/gfp_ref.py) or the library's encode defines them, with the Python
restatement of test_reconstruct_algebra.py on small stripes, and with rs_repair_dev of a copy of the stripe at full size.  The
rows the call must not read (lost rows, parity rows outside J) hold garbage throughout; the call writes nothing but words
[0, SIZE) of its output rows."""
import subprocess
import sys
import threading

import numpy as np
import pytest

import gfp_ref
from test_reconstruct_algebra import reconstruct as reconstruct_py, rows_J
from test_update import P, ROOT, SENTINEL, encode, i32, launches, rand_words, raw, sample_divisors

MAX_K = 32                                                         # FASTECC_B200_RECONSTRUCT_MAX


def padded(x):
    """x (int32 rows of SIZE words) copied into rows of ceil4(SIZE) words: the 16-byte aligned pitch of the stripe calls"""
    import torch
    S = x.shape[1]
    v = torch.empty((x.shape[0], (S + 3) // 4 * 4), dtype=torch.int32, device=x.device)[:, :S]
    v.copy_(x)
    return v


def garbage(shape, gen, kind):
    import torch
    if kind == "ones":
        return torch.full(shape, -1, dtype=torch.int32, device="cuda")
    return i32(torch.randint(0, 1 << 32, shape, device="cuda", generator=gen, dtype=torch.int64))


def spoil(data, parity, lost_d, lost_p, J, gen, kind="random"):
    """garbage into the lost rows and the parity rows outside J (words [0, SIZE) of the views)"""
    import torch
    if lost_d:
        data[torch.as_tensor(lost_d, device="cuda")] = garbage((len(lost_d), data.shape[1]), gen, kind)
    keep = set(J)
    other = [j for j in range(parity.shape[0]) if j not in keep]
    if other:
        parity[torch.as_tensor(other, device="cuda")] = garbage((len(other), parity.shape[1]), gen, kind)


def random_loss(N, M, rng, a=None, wp=None):
    """a lost data blocks, lost parity blocks within M - a, wanted subsets (at least one block) within the cap"""
    if a is None:
        a = int(rng.integers(0, min(M, MAX_K) + 1))
    lost_d = sorted(rng.choice(N, size=a, replace=False).tolist())
    lost_p = sorted(rng.choice(M, size=int(rng.integers(0, M - a + 1)) if wp is None else max(wp, 0), replace=False).tolist())
    want_d = sorted(e for e in lost_d if rng.integers(2))
    want_p = sorted(j for j in lost_p if rng.integers(2))[:MAX_K - a]
    if not want_d and not want_p:
        if lost_d:
            want_d = lost_d[:1]
        elif lost_p:
            want_p = lost_p[:1]
    return lost_d, lost_p, want_d, want_p


SMALL = [1, 2, 3, 4, 6, 8, 9, 12, 18, 32, 36, 96, 288, 1024, 3 * 1024, 9 * 1024]


@pytest.mark.gpu
@pytest.mark.parametrize("N,S", [(N, S) for N in SMALL for S in (5, 8)])
def test_small_stripes_against_the_encode_by_definition(fecc, N, S):
    """Only the rows J of the stored parity are the encode (gfp_ref, by definition); every other parity row and every lost data row
    is garbage.  Up to 36 rows the result also equals the Python pipeline on the same stored words."""
    import torch
    rng = np.random.default_rng(17 * N + S)
    gen = torch.Generator(device="cuda"); gen.manual_seed(17 * N + S)
    data64 = rand_words(N, S, gen)
    for M in sample_divisors(N):
        D = N // M
        for _ in range(3 if N > 1 else 1):
            lost_d, lost_p, want_d, want_p = random_loss(N, M, rng)
            if not want_d and not want_p:
                continue
            J = rows_J(M, len(lost_d), lost_p)
            data = padded(raw(data64, gen))
            parity = padded(garbage((M, S), gen, "random"))
            if J:
                parity[torch.as_tensor(J, device="cuda")] = raw(gfp_ref.encode_rows(data64, [D * j for j in J]), gen)
            spoil(data, parity, lost_d, lost_p, J, gen)
            out = fecc.rs_reconstruct_dev(data, parity, lost_d, lost_p, want_d, want_p)
            parts = []
            if want_d:
                parts.append(data64[torch.as_tensor(want_d, device="cuda")])
            if want_p:
                parts.append(gfp_ref.encode_rows(data64, [D * j for j in want_p]))
            want = torch.cat(parts)
            got = out.to(torch.int64) & 0xFFFFFFFF
            assert torch.equal(got, want), (N, M, lost_d, lost_p, want_d, want_p)
            if N <= 36:
                words = lambda t: (t.to(torch.int64) & 0xFFFFFFFF).tolist()
                assert got.tolist() == reconstruct_py(N, M, words(data), words(parity), lost_d, lost_p, want_d, want_p)


@pytest.fixture(scope="module")
def full_2p19(fecc):
    """2^19 x 1024-word data rows and the parity of M = N, kept for the full-size comparisons"""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(2)
    N, S = 1 << 19, 1024
    data = i32(rand_words(N, S, gen))
    buf = data.clone()
    fecc.rs_encode_asym_mixed_dev(buf, N)
    yield data, buf
    del data, buf
    torch.cuda.empty_cache()


def against_repair(fecc, data, parity, lost_d, lost_p, want_d, want_p, gen):
    """reconstruct from a copy with garbage in the lost rows, repair the copy, compare row for row (and with the original); the
    surviving parity rows outside J stay intact here, since the repair reads them"""
    import torch
    d2, p2 = padded(data), padded(parity)
    gone = set(lost_p)
    spoil(d2, p2, lost_d, lost_p, [j for j in range(parity.shape[0]) if j not in gone], gen)
    out = fecc.rs_reconstruct_dev(d2, p2, lost_d, lost_p, want_d, want_p)
    fecc.rs_repair_dev(d2, p2, lost_d, lost_p)
    torch.cuda.synchronize()
    parts = ([d2[torch.as_tensor(want_d, device="cuda")]] if want_d else []) + ([p2[torch.as_tensor(want_p, device="cuda")]] if want_p else [])
    assert torch.equal(out, torch.cat(parts)), (len(lost_d), len(lost_p))
    orig = ([data[torch.as_tensor(want_d, device="cuda")]] if want_d else []) + ([parity[torch.as_tensor(want_p, device="cuda")]] if want_p else [])
    assert torch.equal(out, torch.cat(orig))
    del d2, p2, out
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("M_div", [1, 16])
@pytest.mark.parametrize("a", [1, 2, 32])
@pytest.mark.parametrize("with_parity", [False, True])
def test_full_size_2p19_4k_blocks_against_repair(fecc, full_2p19, M_div, a, with_parity):
    import torch
    data, full = full_2p19
    N = data.shape[0]
    M = N // M_div
    parity = full[:M] if M_div == 1 else full[::M_div][:M]
    parity = parity.contiguous() if M_div > 1 else parity
    rng = np.random.default_rng(a + 7 * M_div + with_parity)
    gen = torch.Generator(device="cuda"); gen.manual_seed(a)
    lost_d = sorted(rng.choice(N, size=a, replace=False).tolist())
    lost_p = sorted(rng.choice(M, size=(MAX_K - a if a < MAX_K else 3) if with_parity else 0, replace=False).tolist())
    want_p = lost_p[:MAX_K - a]
    against_repair(fecc, data, parity, lost_d, lost_p, lost_d, want_p, gen)


@pytest.mark.gpu
def test_full_size_9x2p19_15_words_against_repair(fecc):
    import torch
    N, S = 9 << 19, 15
    M = N // 9
    gen = torch.Generator(device="cuda"); gen.manual_seed(9)
    rng = np.random.default_rng(9)
    data = padded(i32(rand_words(N, S, gen)))
    parity = padded(encode(fecc, data, M))
    for a, f in ((1, 0), (2, 5), (32, 0), (20, 12)):
        lost_d = sorted(rng.choice(N, size=a, replace=False).tolist())
        lost_p = sorted(rng.choice(M, size=f, replace=False).tolist())
        against_repair(fecc, data, parity, lost_d, lost_p, lost_d, lost_p, gen)


@pytest.mark.gpu
def test_rows_that_must_not_matter(fecc):
    """Lost data rows, lost parity rows and parity rows outside J filled with two random garbages and with all ones give the same
    output; data and parity are byte-identical after the call; the sentinels in the output's pad words and in the rows around it
    stay."""
    import torch
    N, M, S, opitch = 3 << 10, 3 << 7, 61, 72
    gen = torch.Generator(device="cuda"); gen.manual_seed(4)
    rng = np.random.default_rng(4)
    data = padded(i32(rand_words(N, S, gen)))
    parity = padded(encode(fecc, data, M))
    lost_d, lost_p = sorted(rng.choice(N, size=9, replace=False).tolist()), sorted(rng.choice(M, size=40, replace=False).tolist())
    want_d, want_p = lost_d[::2], lost_p[:20]
    J = rows_J(M, len(lost_d), lost_p)
    n = len(want_d) + len(want_p)
    results = []
    for kind in ("random", "random", "ones"):
        d, p = padded(data), padded(parity)
        spoil(d, p, lost_d, lost_p, J, gen, kind)
        before = (d.clone(), p.clone())
        mem = torch.full((n + 2, opitch), SENTINEL, dtype=torch.int32, device="cuda")
        out = mem[1:n + 1, :S]
        fecc.rs_reconstruct_dev(d, p, lost_d, lost_p, want_d, want_p, out=out)
        torch.cuda.synchronize()
        assert torch.equal(d, before[0]) and torch.equal(p, before[1]), "the stripe was written"
        assert bool((mem[0] == SENTINEL).all() and (mem[-1] == SENTINEL).all() and (mem[:, S:] == SENTINEL).all()), "words outside the output"
        results.append(out.clone())
    want = torch.cat([data[torch.as_tensor(want_d, device="cuda")], parity[torch.as_tensor(want_p, device="cuda")]])
    assert all(torch.equal(r, want) for r in results)


@pytest.mark.gpu
@pytest.mark.parametrize("S", [5, 6, 7])
def test_raw_words_pad_garbage_pitches_and_overlap(fecc, S):
    """SIZE % 4 in {1, 2, 3}: raw words >= P in the survivors, random garbage in every pad word, three different pitches with
    the parity buffer below the data in one allocation; then data and parity interleaved in one buffer (overlapping ranges)."""
    import torch
    N, M = 9 << 6, 9 << 3
    gen = torch.Generator(device="cuda"); gen.manual_seed(S)
    rng = np.random.default_rng(S)
    data64 = rand_words(N, S, gen)
    parity64 = encode(fecc, i32(data64), M).to(torch.int64) & 0xFFFFFFFF
    dpitch, ppitch, opitch = S + 12 - S % 4, S + 4 - S % 4, S + 20 - S % 4
    for layout in ("separate", "interleaved"):
        if layout == "separate":
            mem = garbage((M * ppitch + 8 + N * dpitch,), gen, "random")
            pv = mem.as_strided((M, S), (ppitch, 1), 0)
            dv = mem.as_strided((N, S), (dpitch, 1), M * ppitch + 8)
        else:
            pitch = 2 * dpitch                                      # data row i at 2i, parity row j at 2j + 1 (in dpitch units)
            mem = garbage((N * pitch,), gen, "random")
            dv = mem.as_strided((N, S), (pitch, 1), 0)
            pv = mem.as_strided((M, S), (pitch, 1), dpitch)
        for _ in range(3):
            lost_d, lost_p, want_d, want_p = random_loss(N, M, rng)
            dv.copy_(raw(data64, gen))
            pv.copy_(raw(parity64, gen))
            spoil(dv, pv, lost_d, lost_p, rows_J(M, len(lost_d), lost_p), gen)
            n = len(want_d) + len(want_p)
            obuf = torch.full((n, opitch), SENTINEL, dtype=torch.int32, device="cuda")
            before = mem.clone()
            fecc.rs_reconstruct_dev(dv, pv, lost_d, lost_p, want_d, want_p, out=obuf[:, :S])
            torch.cuda.synchronize()
            assert torch.equal(mem, before)
            want = torch.cat(([data64[torch.as_tensor(want_d, device="cuda")]] if want_d else []) +
                             ([parity64[torch.as_tensor(want_p, device="cuda")]] if want_p else []))
            assert torch.equal(obuf[:, :S], i32(want)), (layout, lost_d, lost_p)
            assert bool((obuf[:, S:] == SENTINEL).all())


@pytest.mark.gpu
def test_the_cap_and_the_loss_bound(fecc):
    """a + |W_p| = 32 is accepted and 33 rejected without a launch; a + n_lost_parity = M is accepted"""
    import torch
    N, M, S = 1 << 10, 1 << 6, 8
    gen = torch.Generator(device="cuda"); gen.manual_seed(3)
    data = i32(rand_words(N, S, gen))
    parity = encode(fecc, data, M)
    for a in (0, 1, 16, 32):
        lost_d, lost_p = list(range(3, 3 + 2 * a, 2)), list(range(M - (MAX_K - a), M))
        out = fecc.rs_reconstruct_dev(data, parity, lost_d, lost_p)
        assert torch.equal(out, torch.cat(([data[lost_d]] if lost_d else []) + ([parity[lost_p]] if lost_p else [])))
        over = lost_p + [M - (MAX_K - a) - 1] if a < MAX_K else lost_p
        over_d = lost_d if a < MAX_K else lost_d + [N - 1]
        n0 = fecc.kernel_launches()
        with pytest.raises(fecc.FastEccError) as e:
            fecc.rs_reconstruct_dev(data, parity, over_d, sorted(over))
        assert e.value.code == -1 and "fastecc_b200_rs_repair" in str(e.value) and fecc.kernel_launches() == n0
    M, a = 8, 5                                                     # every parity block used: J = the 8 - 3 survivors
    data = i32(rand_words(64, S, gen))
    parity = encode(fecc, data, M)
    lost_d, lost_p = [0, 9, 10, 40, 63], [1, 4, 6]
    out = fecc.rs_reconstruct_dev(data, parity, lost_d, lost_p)
    assert torch.equal(out, torch.cat([data[lost_d], parity[lost_p]]))


@pytest.mark.gpu
def test_launch_counts(fecc):
    """Two launches per call once the table of the order exists (one more at its first use); none for an empty want list."""
    import torch
    N, M, S = 9 << 7, 9 << 2, 16                                    # an order no other test of this module uses
    gen = torch.Generator(device="cuda"); gen.manual_seed(6)
    data = i32(rand_words(N, S, gen))
    parity = encode(fecc, data, M)
    first = launches(fecc, lambda: fecc.rs_reconstruct_dev(data, parity, [3], [], [3], []))
    assert first in (2, 3)
    for lost_d, lost_p in (([3], []), ([0, 5, 7], [2]), (list(range(32)), []), ([], [0, 35])):
        assert launches(fecc, lambda: fecc.rs_reconstruct_dev(data, parity, lost_d, lost_p)) == 2
    assert launches(fecc, lambda: fecc.rs_reconstruct_dev(data, parity, [1, 2], [4], [], [])) == 0


@pytest.mark.gpu
def test_encode_lose_reconstruct(fecc):
    """rs_encode_asym_mixed_dev, lose blocks (their rows overwritten), reconstruct them: the original blocks"""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(8)
    for N, M in ((3 << 12, 3 << 10), (1 << 13, 1 << 13), (9 << 10, 9), (1 << 12, 1)):
        data = i32(rand_words(N, 256, gen))
        buf = data.clone()
        fecc.rs_encode_asym_mixed_dev(buf, M)
        parity = buf[:M].clone()
        lost_d, lost_p = ([N // 3, N - 1][:M], [0] if M > 2 else [])
        keep = data.clone(), parity.clone()
        data[lost_d] = 0
        if lost_p:
            parity[lost_p] = 0
        out = fecc.rs_reconstruct_dev(data, parity, lost_d, lost_p)
        assert torch.equal(out, torch.cat([keep[0][lost_d]] + ([keep[1][lost_p]] if lost_p else []))), (N, M)


@pytest.mark.gpu
def test_column_chunks(fecc):
    """K = 32 sums of 2^24 + 2^22 + 5 words exceed the 4 GiB workspace: two column chunks, the last ending in a partial group"""
    import torch
    torch.cuda.empty_cache()
    if torch.cuda.mem_get_info()[0] < (24 << 30):
        pytest.skip("needs 24 GiB of free device memory")
    N = M = 32
    S = (1 << 24) + (1 << 22) + 5
    gen = torch.Generator(device="cuda"); gen.manual_seed(12)
    data = padded(i32(rand_words(N, S, gen)))
    parity = padded(encode(fecc, data, M))
    torch.cuda.empty_cache()
    lost_d, lost_p = list(range(0, 32, 2)), list(range(1, 32, 2))
    d, p = padded(data), padded(parity)
    spoil(d, p, lost_d, lost_p, rows_J(M, 16, lost_p), gen)
    out = fecc.rs_reconstruct_dev(d, p, lost_d, lost_p)
    assert launches(fecc, lambda: fecc.rs_reconstruct_dev(d, p, lost_d, lost_p, out=out)) == 4
    assert torch.equal(out, torch.cat([data[lost_d], parity[lost_p]]))
    del data, parity, d, p, out
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_reconstruct_does_not_synchronise_the_stream(fecc):
    """With the workspace already large enough, the call returns while a kernel ahead of it on the stream is still running, and
    the host lists may be overwritten right after the call."""
    import torch
    N, M, S = 1 << 12, 1 << 8, 64
    gen = torch.Generator(device="cuda"); gen.manual_seed(9)
    data = i32(rand_words(N, S, gen)); parity = encode(fecc, data, M)
    lost_d, lost_p = np.array([5, 77, 300], dtype=np.int64), np.array([0, 9], dtype=np.int64)
    want = torch.cat([data[lost_d.tolist()], parity[lost_p.tolist()]])
    out = fecc.rs_reconstruct_dev(data, parity, lost_d, lost_p)            # warm: workspace, table, page-locked buffer
    torch.cuda.synchronize()
    torch.cuda._sleep(1 << 30)
    fecc.rs_reconstruct_dev(data, parity, lost_d, lost_p, out=out)
    busy = not torch.cuda.current_stream().query()
    lost_d[:] = 1; lost_p[:] = 2                                           # the caller reuses its lists
    torch.cuda.synchronize()
    assert busy, "the reconstruct waited for the stream"
    assert torch.equal(out, want)


@pytest.mark.gpu
def test_reconstruct_repair_and_update_on_three_streams_from_two_threads(fecc):
    """Thread 1 reconstructs from a stripe of an order no call has used yet (its table is built on that stream), then updates
    another stripe on a second stream; thread 2 repairs a third stripe on a third stream at the same time."""
    import torch
    from fastecc_b200 import decoder
    gen = torch.Generator(device="cuda"); gen.manual_seed(10)
    rng = np.random.default_rng(10)
    S = 64
    N1, M1 = 3 << 14, 3 << 9
    d1 = i32(rand_words(N1, S, gen)); p1 = encode(fecc, d1, M1)
    jobs = [random_loss(N1, M1, rng, a=a, wp=w) for a, w in ((1, 0), (8, 1), (30, 2))]
    want1 = [torch.cat(([d1[wd]] if wd else []) + ([p1[wp]] if wp else [])) for _, _, wd, wp in jobs]
    N2, M2 = 1 << 14, 1 << 10
    d2 = i32(rand_words(N2, S, gen)); p2 = encode(fecc, d2, M2)
    changed = sorted(rng.choice(N2, size=5, replace=False).tolist())
    new = i32(rand_words(5, S, gen))
    want_d2 = d2.clone(); want_d2[changed] = new
    want_p2 = encode(fecc, want_d2, M2)
    N3, M3 = 1 << 15, 1 << 11
    d3 = i32(rand_words(N3, S, gen)); p3 = encode(fecc, d3, M3)
    lost_d = sorted(rng.choice(N3, size=M3 // 2, replace=False).tolist())
    lost_p = sorted(rng.choice(M3, size=M3 - M3 // 2, replace=False).tolist())
    want_d3, want_p3 = d3.clone(), p3.clone()
    d3[lost_d] = 1
    p3[lost_p] = 2
    rep = decoder.Repair(N3, M3, lost_d, lost_p)
    torch.cuda.synchronize()
    errors, streams, outs = [], [torch.cuda.Stream() for _ in range(3)], []

    def thread1():
        try:
            with torch.cuda.stream(streams[0]):
                for ld, lp, wd, wp in jobs:
                    outs.append(fecc.rs_reconstruct_dev(d1, p1, ld, lp, wd, wp))
            with torch.cuda.stream(streams[2]):
                fecc.rs_update_dev(d2, p2, changed, new)
        except Exception as e:                                      # re-raised on the main thread
            errors.append(e)

    def thread2():
        try:
            with torch.cuda.stream(streams[1]):
                rep.repair(d3, p3)
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
    assert all(torch.equal(o, w) for o, w in zip(outs, want1)) and len(outs) == 3
    assert torch.equal(d2, want_d2) and torch.equal(p2, want_p2)
    assert torch.equal(d3, want_d3) and torch.equal(p3, want_p3)


@pytest.mark.gpu
def test_reconstruct_argument_table(fecc):
    """Every rule of the validation broken on its own gives FASTECC_B200_EINVAL (-1) and launches nothing; the valid calls give 0."""
    import torch
    L = fecc.lib()
    st = torch.cuda.current_stream().cuda_stream
    buf = torch.zeros((80, 8), dtype=torch.int32, device="cuda")
    d, p, o = buf[:12].data_ptr(), buf[32:36].data_ptr(), buf[48:52].data_ptr()
    wrong = []

    def arr(x):
        return None if x is None else np.asarray(x, dtype=np.uint32)

    def call(data=d, dpitch=8, N=12, parity=p, ppitch=8, M=4, ld=(1, 5), nld=None, lp=(2,), nlp=None, wd=(5,), nwd=None, wp=(2,), nwp=None,
             out=o, opitch=8, S=8):
        lists = [arr(x) for x in (ld, lp, wd, wp)]
        ns = [(0 if x is None else x.size) if n is None else n for x, n in zip(lists, (nld, nlp, nwd, nwp))]
        ptrs = [None if x is None or not x.size else x.ctypes.data for x in lists]
        return L.fastecc_b200_rs_reconstruct(data, dpitch, N, parity, ppitch, M, ptrs[0], ns[0], ptrs[1], ns[1], ptrs[2], ns[2], ptrs[3], ns[3],
                                             out, opitch, S, st)

    cases = [({}, 0), (dict(S=5), 0), (dict(M=12, parity=buf[16:28].data_ptr()), 0), (dict(M=1, lp=(), wp=(), ld=(3,), wd=(3,)), 0),
             (dict(ld=(), wd=(), lp=(0, 1, 2, 3), wp=(0, 1, 2, 3)), 0), (dict(ld=(0, 1, 2), lp=(3,), wd=(1,), wp=(3,)), 0),
             (dict(data=p, parity=p + 16), 0), (dict(parity=d + 8 * 4 * 4), 0),
             (dict(N=5), -1), (dict(N=27), -1), (dict(N=3 << 20, M=3), -1), (dict(M=0), -1), (dict(M=5), -1), (dict(M=24), -1),
             (dict(S=0), -1), (dict(data=None), -1), (dict(parity=None), -1), (dict(out=None), -1),
             (dict(ld=None, nld=2), -1), (dict(lp=None, nlp=1), -1), (dict(wd=None, nwd=1), -1), (dict(wp=None, nwp=1), -1),
             (dict(dpitch=6, S=6), -1), (dict(ppitch=6, S=6), -1), (dict(opitch=6, S=6), -1), (dict(dpitch=4), -1), (dict(ppitch=4), -1),
             (dict(opitch=4), -1), (dict(data=d + 4, S=4), -1), (dict(parity=p + 8, S=4), -1), (dict(out=o + 4, S=4), -1),
             (dict(ld=(5, 1)), -1), (dict(ld=(1, 1), wd=(1,)), -1), (dict(ld=(1, 12)), -1), (dict(lp=(4,), wp=(4,)), -1),
             (dict(lp=(2, 2), wp=(2,)), -1), (dict(wd=(5, 1)), -1), (dict(wd=(3,)), -1), (dict(wp=(1,)), -1), (dict(wd=(1, 5, 6)), -1),
             (dict(ld=(0, 1, 2), lp=(0, 3), wd=(1,), wp=(3,)), -1), (dict(ld=(0, 1, 2, 3), lp=(1,), wd=(1,), wp=()), -1),
             (dict(out=d + 8 * 4 * 4), -1), (dict(out=p - 8 * 4), -1), (dict(out=p + 8 * 3 * 4), -1), (dict(out=d - 8 * 4), -1)]
    for kw, want in cases:
        n0 = fecc.kernel_launches()
        rc = call(**kw)
        if rc != want or (want and fecc.kernel_launches() != n0):
            wrong.append((kw, rc))
    big = buf.new_zeros((2048, 8))
    cap = dict(data=big[:1024].data_ptr(), N=1024, parity=big[1024:1088].data_ptr(), M=64, out=big[1100:1140].data_ptr())
    for kw, want in ((dict(ld=tuple(range(20)), lp=tuple(range(12)), wd=(), wp=tuple(range(12))), 0),
                     (dict(ld=tuple(range(20)), lp=tuple(range(13)), wd=(), wp=tuple(range(13))), -1),
                     (dict(ld=tuple(range(33)), lp=(), wd=(0,), wp=()), -1)):
        n0 = fecc.kernel_launches()
        rc = call(**cap, **kw)
        if rc != want or (want and fecc.kernel_launches() != n0):
            wrong.append(("cap", kw, rc))
        if want and "fastecc_b200_rs_repair" not in L.fastecc_b200_last_error().decode():
            wrong.append(("cap message", kw))
    for kw in (dict(wd=(), wp=()), dict(wd=(), wp=(), out=None)):                     # nothing wanted: 0, no launch
        n0 = fecc.kernel_launches()
        if call(**kw) != 0 or fecc.kernel_launches() != n0:
            wrong.append(("nothing wanted", kw))
    torch.cuda.synchronize()
    assert not wrong, wrong


@pytest.mark.gpu
def test_reconstruct_before_init_is_enoinit():
    """In a fresh process that never called fastecc_b200_init, the call fails with FASTECC_B200_ENOINIT (-4)."""
    code = ("import sys; sys.path.insert(0, %r); import fastecc_b200 as fe; L = fe.lib(); "
            "print(L.fastecc_b200_rs_reconstruct(None, 4, 12, None, 4, 4, None, 0, None, 0, None, 0, None, 0, None, 4, 4, None))") % ROOT
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.stdout.split() == ["-4"], out.stdout + out.stderr
