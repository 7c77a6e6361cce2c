"""GPU: degraded read of a batch of small stripes with one loss pattern (fastecc_b200_rs_reconstruct_batch, csrc/batch.cu,
DESIGN 3m).  Stripes are written by rs_encode_batch_dev; every result is compared with the original rows, with rs_reconstruct_dev
of the same stored words where its cap allows, and on samples with the encode by definition (tests/gfp_ref.py).  The rows the
call must not read hold garbage; everything around the output rows holds sentinels that must come back unchanged."""
import subprocess
import sys
import threading

import numpy as np
import pytest

import gfp_ref
from test_encode_batch import SHAPES, ceil4, words
from test_reconstruct import garbage, padded
from test_reconstruct_algebra import rows_J
from test_update import C, P, ROOT, SENTINEL, i32, launches, rand_words

MAX_K = 32                                                         # FASTECC_B200_RECONSTRUCT_MAX


def stripes(fecc, B, N, M, S, gen):
    """[B, N, S] data (rows of ceil4(S) words) and its batch-encoded [B, M, S] parity; the data as canonical int64 words"""
    import torch
    data64 = rand_words(B * N, S, gen).view(B, N, S)
    data = torch.empty((B, N, ceil4(S)), dtype=torch.int32, device="cuda")[..., :S]
    data.copy_(i32(data64))
    return data64, data, fecc.rs_encode_batch_dev(data, M=M)


def copy(x):
    """x [B, R, S] copied into rows of ceil4(S) words: 16-byte aligned rows, as the call needs"""
    import torch
    v = torch.empty((*x.shape[:2], ceil4(x.shape[2])), dtype=x.dtype, device=x.device)[..., :x.shape[2]]
    v.copy_(x)
    return v


def spoil(data, parity, lost_d, lost_p, gen, kind="random"):
    """garbage into every stripe's lost data rows and parity rows outside J"""
    B, _, S = data.shape
    if lost_d:
        data[:, lost_d] = garbage((B, len(lost_d), S), gen, kind)
    other = [j for j in range(parity.shape[1]) if j not in rows_J(parity.shape[1], len(lost_d), lost_p)]
    if other:
        parity[:, other] = garbage((B, len(other), S), gen, kind)


def per_stripe(fecc, data, parity, lost_d, lost_p, want_d, want_p):
    """rs_reconstruct_dev on the B stripes side by side as one stripe of B S word columns (the read works column by column)"""
    B, N, S = data.shape
    M = parity.shape[1]
    d = padded(data.permute(1, 0, 2).reshape(N, B * S))
    p = padded(parity.permute(1, 0, 2).reshape(M, B * S))
    out = fecc.rs_reconstruct_dev(d, p, lost_d, lost_p, want_d, want_p)
    return out.reshape(len(want_d) + len(want_p), B, S).permute(1, 0, 2)


def losses(N, M, rng):
    """(i) one lost data block, (ii) one lost parity block, (iii) two lost data blocks, (iv) M lost data blocks, and a random
    loss with random wanted subsets: (lost_d, lost_p, want_d, want_p)"""
    pick = lambda n, k: sorted(rng.choice(n, size=k, replace=False).tolist())
    out = [(pick(N, 1), [], None, None), ([], pick(M, 1), None, None)]
    if M >= 2:
        out.append((pick(N, 2), [], None, None))
    out.append((pick(N, M), [], None, None))
    a = int(rng.integers(0, M + 1))
    ld, lp = pick(N, a), pick(M, int(rng.integers(0, M - a + 1)))
    wd, wp = [e for e in ld if rng.integers(2)], [j for j in lp if rng.integers(2)]
    if wd or wp:
        out.append((ld, lp, wd, wp))
    return [(ld, lp, ld if wd is None else wd, lp if wp is None else wp) for ld, lp, wd, wp in out]


@pytest.mark.gpu
@pytest.mark.parametrize("N,M", SHAPES)
def test_every_shape_against_the_originals_and_the_per_stripe_read(fecc, N, M):
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(2000 * N + M)
    rng = np.random.default_rng(2000 * N + M)
    D = N // M
    for B in (1, 7, 300):
        for S in (1, 5, 1024):
            data64, data, parity = stripes(fecc, B, N, M, S, gen)
            orig_p = parity.clone()
            for ld, lp, wd, wp in losses(N, M, rng):
                d, p = copy(data), copy(parity)
                spoil(d, p, ld, lp, gen)
                keep = d.clone(), p.clone()
                out = fecc.rs_reconstruct_batch_dev(d, p, ld, lp, wd, wp)
                assert torch.equal(d, keep[0]) and torch.equal(p, keep[1]), (N, M, B, S, ld, lp)
                want = torch.cat([i32(data64[:, wd]), orig_p[:, wp]], dim=1)
                assert torch.equal(out, want), (N, M, B, S, ld, lp, wd, wp)
                if len(ld) + len(wp) <= MAX_K:
                    assert torch.equal(out, per_stripe(fecc, d, p, ld, lp, wd, wp)), (N, M, B, S, ld, lp, wd, wp)
                if B == 7:
                    for b in (0, 6):
                        assert torch.equal(words(out[b, :len(wd)]), data64[b, wd]), (N, M, S, b)
                        if wp:
                            assert torch.equal(words(out[b, len(wd):]), gfp_ref.encode_rows(data64[b], [D * j for j in wp])), (N, M, S, b)


@pytest.mark.gpu
def test_rows_that_must_not_be_read(fecc):
    """Lost rows and parity rows outside J hold random words, 0xFFFFFFFF or zeros: the output is the same each time"""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(3)
    for N, M, ld, lp in ((12, 4, [2, 7], [0]), (36, 12, [0, 5, 35], [1, 2, 11]), (64, 64, list(range(0, 64, 3)), [0, 63]), (9, 9, [], [4, 8])):
        data64, data, parity = stripes(fecc, 40, N, M, 33, gen)
        results = []
        for kind in ("random", "ones", "zeros"):
            d, p = copy(data), copy(parity)
            if kind == "zeros":
                d[:, ld] = 0
                other = [j for j in range(M) if j not in rows_J(M, len(ld), lp)]
                p[:, other] = 0
            else:
                spoil(d, p, ld, lp, gen, kind)
            results.append(fecc.rs_reconstruct_batch_dev(d, p, ld, lp))
        want = torch.cat([data[:, ld], parity[:, lp]], dim=1)
        assert all(torch.equal(r, want) for r in results), (N, M)


def sentinel_buffer(n_words):
    import torch
    return torch.full((n_words,), SENTINEL, dtype=torch.int32, device="cuda")


def run_layout(fecc, B, N, M, S, ld, lp, lay, shared, guard=64):
    """lay = {side: (offset, pitch, stride)} for data, parity and out, as views of sentinel buffers with `guard` sentinel words
    around them; shared = one buffer for all three.  True when the call wrote exactly the wanted rows and nothing else."""
    import torch
    from torch import as_strided
    gen = torch.Generator(device="cuda"); gen.manual_seed(B * 131 + N * 7 + S)
    n_out = len(ld) + len(lp)
    rows = {"data": N, "parity": M, "out": n_out}
    end = {k: o + (B - 1) * st + (rows[k] - 1) * pi + ceil4(S) for k, (o, pi, st) in lay.items()}
    if shared:
        buf = sentinel_buffer(2 * guard + max(end.values()))
        bufs = dict.fromkeys(lay, buf)
    else:
        bufs = {k: sentinel_buffer(2 * guard + e) for k, e in end.items()}
    view = lambda k, b: as_strided(b, (B, rows[k], S), (lay[k][2], lay[k][1], 1), guard + lay[k][0])
    data64, d0, p0 = stripes(fecc, B, N, M, S, gen)
    view("data", bufs["data"]).copy_(d0)
    view("parity", bufs["parity"]).copy_(p0)
    spoil(view("data", bufs["data"]), view("parity", bufs["parity"]), ld, lp, gen)
    expect = {k: b.clone() for k, b in bufs.items()}
    view("out", expect["out"]).copy_(torch.cat([d0[:, ld], p0[:, lp]], dim=1))
    fecc.rs_reconstruct_batch_dev(view("data", bufs["data"]), view("parity", bufs["parity"]), ld, lp, out=view("out", bufs["out"]))
    if shared:
        return torch.equal(buf, expect["out"])
    return all(torch.equal(bufs[k], expect[k]) for k in ("data", "parity")) and torch.equal(bufs["out"], expect["out"])


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 2, 3, 5, 6, 7, 64, 1021])
def test_layouts_sentinels_and_pad_words(fecc, S):
    """Stripe-major and block-major on all three sides in every combination, separate buffers; one [B][N + M + n_out][pitch]
    buffer; pitches with pad words and gaps between rows and stripes."""
    B = 5
    for N, M, ld, lp in ((4, 2, [1], [0]), (12, 4, [0, 11], [3]), (9, 9, [2, 4, 8], [0, 1]), (16, 1, [7], [])):
        n_out = len(ld) + len(lp)
        pitch = ceil4(S) + 4
        sm = lambda n: (0, pitch, n * pitch + 8)                     # stripe-major: a gap between stripes
        bm = lambda n: (0, B * ceil4(S) + 12, ceil4(S))              # block-major: the stripes of one block side by side, then a gap
        for fd in (sm, bm):
            for fp in (sm, bm):
                for fo in (sm, bm):
                    lay = {"data": fd(N), "parity": fp(M), "out": fo(n_out)}
                    assert run_layout(fecc, B, N, M, S, ld, lp, lay, False), (N, M, S, lay)
        stride = (N + M + n_out) * pitch + 4
        lay = {"data": (0, pitch, stride), "parity": (N * pitch, pitch, stride), "out": ((N + M) * pitch, pitch, stride)}
        assert run_layout(fecc, B, N, M, S, ld, lp, lay, True), ("one buffer", N, M, S)
        lay = {"out": (0, pitch, stride), "data": (n_out * pitch, pitch, stride), "parity": ((n_out + N) * pitch, pitch, stride)}
        assert run_layout(fecc, B, N, M, S, ld, lp, lay, True), ("one buffer, out first", N, M, S)


@pytest.mark.gpu
def test_raw_words_are_taken_mod_p(fecc):
    """Stored words >= P congruent to small values, and 0xFFFFFFFF, give the blocks of their residues"""
    import torch
    B, S = 6, 12
    for N, M, ld, lp in ((4, 2, [3], [0]), (36, 12, [1, 2, 30], [5]), (64, 64, [0, 9], [63])):
        small = torch.randint(0, C, (B, N, S), device="cuda", dtype=torch.int64)
        small[:, 0, :3] = 0xFFFFFFFF - P
        parity = fecc.rs_encode_batch_dev(i32(small), M=M)
        par64 = words(parity)
        stored_d = i32(small + P)
        stored_d[:, 0, :3] = -1                                         # 0xFFFFFFFF = P + 0xFFFFE
        stored_p = i32(torch.where(par64 < C, par64 + P, par64))
        d = torch.zeros((B, N, 16), dtype=torch.int32, device="cuda")[..., :S]
        p = torch.zeros((B, M, 16), dtype=torch.int32, device="cuda")[..., :S]
        d.copy_(stored_d); p.copy_(stored_p)
        got = fecc.rs_reconstruct_batch_dev(d, p, ld, lp)
        assert torch.equal(got, torch.cat([i32(small[:, ld]), parity[:, lp]], dim=1)), (N, M)


@pytest.mark.gpu
def test_large_offsets(fecc):
    """A data stripe stride of 2^31 + 16 words: the last of three stripes starts past 2^32 words from the base (16 GiB of data)"""
    import torch
    torch.cuda.empty_cache()
    if torch.cuda.mem_get_info()[0] < (20 << 30):
        pytest.skip("needs 20 GiB of free device memory")
    B, N, M, S = 3, 12, 4, 37
    stride = (1 << 31) + 16
    big = torch.empty((B - 1) * stride + N * 40, dtype=torch.int32, device="cuda")
    gen = torch.Generator(device="cuda"); gen.manual_seed(4)
    data = big.as_strided((B, N, S), (stride, 40, 1))
    data64 = rand_words(B * N, S, gen).view(B, N, S)
    data.copy_(i32(data64))
    assert data[B - 1].data_ptr() - big.data_ptr() >= 4 << 32
    parity = fecc.rs_encode_batch_dev(data, M=M)
    want = torch.cat([i32(data64[:, [3, 11]]), parity[:, [1]]], dim=1)
    data[:, [3, 11]] = 0
    out = fecc.rs_reconstruct_batch_dev(data, parity, [3, 11], [1])
    assert torch.equal(out, want)
    del big, data, parity, out
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_encode_lose_reconstruct_against_repair(fecc):
    """Batch-encode [B][N + M] stripes, lose blocks in all of them, batch-read them back; rs_repair_dev of a copy of a stripe
    rebuilds the same rows"""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(5)
    B, S = 50, 256
    for N, M, ld, lp in ((12, 4, [0, 7], [3]), (18, 3, [17], [0, 2]), (32, 8, [1, 2, 3, 30], [4, 7]), (64, 16, list(range(8, 24)), [])):
        buf = torch.zeros((B, N + M, S), dtype=torch.int32, device="cuda")
        buf[:, :N] = i32(rand_words(B * N, S, gen).view(B, N, S))
        fecc.rs_encode_batch_dev(buf[:, :N], buf[:, N:])
        good = buf.clone()
        buf[:, ld] = 7
        buf[:, [N + j for j in lp]] = 9
        out = fecc.rs_reconstruct_batch_dev(buf[:, :N], buf[:, N:], ld, lp)
        assert torch.equal(out, torch.cat([good[:, ld], good[:, [N + j for j in lp]]], dim=1)), (N, M)
        for b in (0, B // 2, B - 1):
            d, p = buf[b, :N].clone(), buf[b, N:].clone()
            fecc.rs_repair_dev(d, p, ld, lp)
            assert torch.equal(out[b], torch.cat([d[ld], p[lp]])), (N, M, b)


@pytest.mark.gpu
def test_launch_counts(fecc):
    """One launch per call (no table build); none for B = 0 or nothing wanted"""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(6)
    _, data, parity = stripes(fecc, 9, 24, 6, 8, gen)
    for ld, lp in (([3], []), ([0, 5, 7], [2]), ([], [0, 5]), (list(range(6)), [])):
        assert launches(fecc, lambda: fecc.rs_reconstruct_batch_dev(data, parity, ld, lp)) == 1, (ld, lp)
    out = torch.empty((0, 1, 8), dtype=torch.int32, device="cuda")
    assert launches(fecc, lambda: fecc.rs_reconstruct_batch_dev(data[:0], parity[:0], [3], [], out=out)) == 0
    assert launches(fecc, lambda: fecc.rs_reconstruct_batch_dev(data, parity, [1, 2], [4], [], [])) == 0


@pytest.mark.gpu
def test_reconstruct_batch_does_not_synchronise_the_stream(fecc):
    """The call returns while a kernel ahead of it on the stream is still running, and the host lists may be overwritten right
    after the call"""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(9)
    _, data, parity = stripes(fecc, 100, 16, 4, 64, gen)
    lost_d, lost_p = np.array([5, 9], dtype=np.int64), np.array([3], dtype=np.int64)
    want = torch.cat([data[:, [5, 9]], parity[:, [3]]], dim=1)
    out = fecc.rs_reconstruct_batch_dev(data, parity, lost_d, lost_p)      # warm: workspace, page-locked buffer
    torch.cuda.synchronize()
    out.zero_()
    torch.cuda._sleep(1 << 30)
    fecc.rs_reconstruct_batch_dev(data, parity, lost_d, lost_p, out=out)
    busy = not torch.cuda.current_stream().query()
    lost_d[:] = 1; lost_p[:] = 2
    torch.cuda.synchronize()
    assert busy, "the batched read waited for the stream"
    assert torch.equal(out, want)


@pytest.mark.gpu
def test_many_patterns_queued_behind_a_busy_stream(fecc):
    """Twelve calls with different loss patterns behind a long kernel: more than the eight page-locked upload buffers, all correct"""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(11)
    rng = np.random.default_rng(11)
    N, M = 32, 8
    _, data, parity = stripes(fecc, 64, N, M, 40, gen)
    jobs = []
    for k in range(12):
        a = k % (M + 1)
        ld = sorted(rng.choice(N, size=a, replace=False).tolist())
        lp = sorted(rng.choice(M, size=int(rng.integers(0, M - a + 1)), replace=False).tolist())
        if not ld and not lp:
            lp = [k % M]
        jobs.append((ld, lp))
    torch.cuda.synchronize()
    torch.cuda._sleep(1 << 28)
    outs = [fecc.rs_reconstruct_batch_dev(data, parity, ld, lp) for ld, lp in jobs]
    torch.cuda.synchronize()
    for (ld, lp), out in zip(jobs, outs):
        assert torch.equal(out, torch.cat([data[:, ld], parity[:, lp]], dim=1)), (ld, lp)


@pytest.mark.gpu
def test_two_threads_on_two_streams(fecc):
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(12)
    work = [stripes(fecc, 300, 36, 12, 64, gen), stripes(fecc, 200, 48, 16, 100, gen)]
    patterns = [[([0, 35], [1]), (list(range(12)), []), ([], [0, 11])], [([47], []), (list(range(0, 48, 6)), [1, 3]), ([2, 3], [0, 15])]]
    outs, errors, go = [[], []], [], threading.Barrier(2)
    streams = [torch.cuda.Stream() for _ in range(2)]
    torch.cuda.synchronize()

    def run(k):
        try:
            with torch.cuda.stream(streams[k]):
                go.wait()
                for ld, lp in patterns[k]:
                    outs[k].append(fecc.rs_reconstruct_batch_dev(work[k][1], work[k][2], ld, lp))
        except Exception as e:                                      # re-raised on the main thread
            errors.append(e)
    th = [threading.Thread(target=run, args=(k,)) for k in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    torch.cuda.synchronize()
    assert not errors, errors
    for k in range(2):
        _, data, parity = work[k]
        assert len(outs[k]) == 3
        for (ld, lp), out in zip(patterns[k], outs[k]):
            assert torch.equal(out, torch.cat([data[:, ld], parity[:, lp]], dim=1)), (k, ld, lp)


@pytest.mark.gpu
def test_reconstruct_batch_argument_table(fecc):
    """Every rule broken on its own gives FASTECC_B200_EINVAL (-1), writes nothing and launches nothing; the listed layouts and
    overlapping data and parity are accepted."""
    import torch
    L = fecc.lib()
    st = torch.cuda.current_stream().cuda_stream
    buf = torch.full((8192,), SENTINEL, dtype=torch.int32, device="cuda")
    a = buf.data_ptr()
    B, S = 3, 8
    wrong = []

    def arr(x):
        return None if x is None else np.asarray(x, dtype=np.uint32)

    def call(data=a, dpitch=8, dstride=96, N=12, parity=a + 4 * 2048, ppitch=8, pstride=32, M=4, ld=(1, 5), nld=None, lp=(2,), nlp=None,
             wd=(5,), nwd=None, wp=(2,), nwp=None, out=a + 4 * 4096, opitch=8, ostride=16, B=B, S=S):
        lists = [arr(x) for x in (ld, lp, wd, wp)]
        ns = [(0 if x is None else x.size) if n is None else n for x, n in zip(lists, (nld, nlp, nwd, nwp))]
        ptrs = [None if x is None or not x.size else x.ctypes.data for x in lists]
        return L.fastecc_b200_rs_reconstruct_batch(data, dpitch, dstride, N, parity, ppitch, pstride, M, ptrs[0], ns[0], ptrs[1], ns[1], ptrs[2], ns[2],
                                                   ptrs[3], ns[3], out, opitch, ostride, B, S, st)
    shared = dict(data=a, dstride=144, parity=a + 4 * 96, pstride=144, out=a + 4 * 128, ostride=144)   # [B][12 + 4 + 2][8]
    cases = [({}, 0), (dict(S=5), 0), (dict(opitch=24, ostride=8), 0), (shared, 0), (dict(parity=a, pstride=96), 0),
             (dict(ld=(), wd=(), lp=(0, 1, 2, 3), wp=(0, 1, 2, 3), ostride=32), 0), (dict(M=1, ld=(3,), wd=(3,), lp=(), wp=(), pstride=8), 0),
             (dict(N=5), -1), (dict(N=27), -1), (dict(N=128, M=4), -1), (dict(N=72, M=8), -1), (dict(M=0), -1), (dict(M=5), -1), (dict(M=24), -1),
             (dict(S=0), -1), (dict(data=None), -1), (dict(parity=None), -1), (dict(out=None), -1),
             (dict(dpitch=4), -1), (dict(ppitch=4), -1), (dict(opitch=4), -1),
             (dict(data=a + 4), -1), (dict(parity=a + 4 * 2048 + 8), -1), (dict(out=a + 4 * 4096 + 4), -1),
             (dict(dpitch=10, S=6), -1), (dict(ppitch=10, S=6), -1), (dict(opitch=10, S=6), -1),
             (dict(dstride=98), -1), (dict(pstride=34), -1), (dict(ostride=18), -1),
             (dict(ostride=8), -1), (dict(opitch=0), -1), (dict(out=a + 4 * 8), -1), (dict(out=a + 4 * 2048), -1), (dict(out=a + 4 * 2048 + 4 * 88), -1),
             (dict(shared, out=a + 4 * 8), -1), (dict(shared, ostride=128), -1),
             (dict(ld=None, nld=2), -1), (dict(lp=None, nlp=1), -1), (dict(wd=None, nwd=1), -1), (dict(wp=None, nwp=1), -1),
             (dict(ld=(5, 1)), -1), (dict(ld=(1, 1), wd=(1,)), -1), (dict(ld=(1, 12)), -1), (dict(lp=(4,), wp=(4,)), -1),
             (dict(lp=(2, 2), wp=(2,)), -1), (dict(wd=(5, 1)), -1), (dict(wd=(3,)), -1), (dict(wp=(1,)), -1),
             (dict(ld=(0, 1, 2), lp=(0, 3), wd=(1,), wp=(3,)), -1), (dict(ld=(0, 1, 2, 3), lp=(1,), wd=(1,), wp=()), -1),
             (dict(B=1 << 35), -1)]
    for kw, want in cases:
        torch.cuda.synchronize()
        before = buf.clone()
        n0 = fecc.kernel_launches()
        rc = call(**kw)
        torch.cuda.synchronize()
        if rc != want:
            wrong.append((kw, rc, L.fastecc_b200_last_error().decode()))
        if want and (fecc.kernel_launches() != n0 or not torch.equal(buf, before)):
            wrong.append(("wrote or launched", kw))
        buf.fill_(SENTINEL)
    call(N=128, M=4)
    if "fastecc_b200_rs_reconstruct" not in L.fastecc_b200_last_error().decode():
        wrong.append("cap message")
    n0 = fecc.kernel_launches()
    for kw in (dict(B=0), dict(B=0, data=None, parity=None, out=None), dict(wd=(), wp=()), dict(wd=(), wp=(), data=None, parity=None, out=None)):
        if call(**kw) != 0:
            wrong.append(("nothing to do", kw))
    if fecc.kernel_launches() != n0:
        wrong.append("launched with nothing to do")
    torch.cuda.synchronize()
    assert not wrong, wrong


@pytest.mark.gpu
def test_reconstruct_batch_before_init_is_enoinit():
    code = ("import sys; sys.path.insert(0, %r); import fastecc_b200 as fe; L = fe.lib(); "
            "print(L.fastecc_b200_rs_reconstruct_batch(None, 4, 48, 12, None, 4, 16, 4, None, 0, None, 0, None, 0, None, 0, None, 4, 4, 1, 4, None))") % ROOT
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.stdout.split() == ["-4"], out.stdout + out.stderr
