"""GPU: update of a batch of small stripes in place with one changed list (fastecc_b200_rs_update_batch, csrc/batch.cu,
DESIGN 3n).  Stripes are written by rs_encode_batch_dev; every result is compared with rs_encode_batch_dev of the updated data,
with per-stripe rs_update_dev, and on samples with the encode by definition (tests/gfp_ref.py).  The data rows the call must not
read hold garbage; everything around the rows it writes holds sentinels that must come back unchanged.  The launcher's rule is
restated here and checked against the profiler's kernel records, one witness per geometry class."""
import subprocess
import sys

import numpy as np
import pytest

import gfp_ref
import stripe_geometry as sg
from stripe_geometry import ORDERS, Launch, cdiv, divisors
from test_encode_batch import SHAPES, ceil4, words
from test_reconstruct import garbage
from test_reconstruct_batch import copy, sentinel_buffer, stripes
from test_update import C, P, ROOT, SENTINEL, i32, launches, rand_words


def raw_words(shape, gen):
    """random 32-bit words, with 0xFFFFFFFF, P and P + 5 sprinkled in: stored words whose residues are what counts"""
    import torch
    x = torch.randint(0, 1 << 32, shape, device="cuda", generator=gen, dtype=torch.int64)
    flat = x.view(-1)
    flat[0::7] = 0xFFFFFFFF
    flat[3::11] = P
    flat[5::13] = P + 5
    return x


def as_stored(x64, gen):
    """canonical int64 words as int32 stored words: x + P at random where that fits 32 bits"""
    import torch
    bump = (torch.randint(0, 2, x64.shape, device="cuda", generator=gen) == 1) & (x64 < C)
    return i32(torch.where(bump, x64 + P, x64))


def subsets(N, rng):
    ks = sorted({1, min(2, N), N})
    out = [sorted(rng.choice(N, size=k, replace=False).tolist()) for k in ks]
    out.append(sorted(rng.choice(N, size=int(rng.integers(1, N + 1)), replace=False).tolist()))
    return out


def per_stripe(fecc, data, parity, changed, new):
    """rs_update_dev on the B stripes side by side as one stripe of B S word columns (the update works column by column)"""
    import torch
    B, N, S = data.shape
    M = parity.shape[1]
    flat = lambda x: copy(x.permute(1, 0, 2).reshape(1, x.shape[1], B * S))[0]
    d, p, n = flat(data), flat(parity), flat(new)
    fecc.rs_update_dev(d, p, changed, n)
    return d.reshape(N, B, S).permute(1, 0, 2), p.reshape(M, B, S).permute(1, 0, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("N,M", SHAPES)
def test_every_shape_against_the_batch_encode_and_the_per_stripe_update(fecc, N, M):
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(3000 * N + M)
    rng = np.random.default_rng(3000 * N + M)
    D = N // M
    for B in (1, 7, 300):
        for S in (1, 5, 1024):
            data64, data, parity = stripes(fecc, B, N, M, S, gen)
            for changed in subsets(N, rng):
                k = len(changed)
                new64 = raw_words((B, k, S), gen)
                new = copy(i32(new64))
                after64 = data64.clone()
                after64[:, changed] = new64 % P
                want_p = fecc.rs_encode_batch_dev(copy(i32(after64)), M=M)
                ref_d, ref_p = per_stripe(fecc, data, parity, changed, new)
                d, p = copy(data), copy(as_stored(words(parity), gen))
                d[:, changed] = as_stored(data64[:, changed], gen)
                others = [i for i in range(N) if i not in changed]
                if others:
                    d[:, others] = garbage((B, len(others), S), gen, "random")
                keep_d, keep_n = d.clone(), new.clone()
                fecc.rs_update_batch_dev(d, p, changed, new)
                assert torch.equal(p, want_p), (N, M, B, S, changed)
                assert torch.equal(p, ref_p), (N, M, B, S, changed)
                assert torch.equal(d[:, changed], i32(new64 % P)), (N, M, B, S, changed)
                assert torch.equal(d[:, changed], ref_d[:, changed]), (N, M, B, S, changed)
                if others:
                    assert torch.equal(d[:, others], keep_d[:, others]), (N, M, B, S, changed)
                assert torch.equal(new, keep_n), (N, M, B, S, changed)
                if B == 7:
                    for b in (0, 6):
                        assert torch.equal(words(p[b]), gfp_ref.encode_rows(after64[b], [D * j for j in range(M)])), (N, M, S, b)


@pytest.mark.gpu
def test_rows_that_must_not_be_read(fecc):
    """Unchanged data rows hold random words, 0xFFFFFFFF or zeros: the result is the same each time"""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(3)
    for N, M, changed in ((12, 4, [2, 7]), (36, 12, [0, 5, 35]), (64, 64, list(range(0, 64, 3))), (9, 9, [4]), (64, 1, [63])):
        _, data, parity = stripes(fecc, 40, N, M, 33, gen)
        new = copy(i32(raw_words((40, len(changed), 33), gen)))
        others = [i for i in range(N) if i not in changed]
        results = []
        for kind in ("random", "ones", "zeros"):
            d, p = copy(data), copy(parity)
            d[:, others] = 0 if kind == "zeros" else garbage((40, len(others), 33), gen, kind)
            fecc.rs_update_batch_dev(d, p, changed, new)
            results.append((d[:, changed].clone(), p))
        assert all(torch.equal(r[0], results[0][0]) and torch.equal(r[1], results[0][1]) for r in results), (N, M)


def run_layout(fecc, B, N, M, S, changed, lay, shared, guard=64):
    """lay = {side: (offset, pitch, stride)} for data, parity and new, as views of sentinel buffers with `guard` sentinel words
    around them; shared = one buffer for all three.  True when the call wrote exactly the changed data rows and the parity rows,
    with the expected words, and nothing else."""
    import torch
    from torch import as_strided
    gen = torch.Generator(device="cuda"); gen.manual_seed(B * 131 + N * 7 + S)
    k = len(changed)
    rows = {"data": N, "parity": M, "new": k}
    end = {s: o + max(B - 1, 0) * st + (rows[s] - 1) * pi + ceil4(S) for s, (o, pi, st) in lay.items()}
    if shared:
        buf = sentinel_buffer(2 * guard + max(end.values()))
        bufs = dict.fromkeys(lay, buf)
    else:
        bufs = {s: sentinel_buffer(2 * guard + e) for s, e in end.items()}
    view = lambda s: as_strided(bufs[s], (B, rows[s], S), (lay[s][2], lay[s][1], 1), guard + lay[s][0])
    data64, d0, p0 = stripes(fecc, B, N, M, S, gen)
    new64 = raw_words((B, k, S), gen)
    if lay["new"][2] == 0:
        new64[1:] = new64[0]
    view("data").copy_(d0)
    view("parity").copy_(p0)
    if lay["new"][2] == 0:                                          # one set of new rows for every stripe
        as_strided(bufs["new"], (k, S), (lay["new"][1], 1), guard + lay["new"][0]).copy_(i32(new64[0]))
    else:
        view("new").copy_(i32(new64))
    others = [i for i in range(N) if i not in changed]
    if others:
        view("data")[:, others] = garbage((B, len(others), S), gen, "random")
    after64 = data64.clone()
    after64[:, changed] = new64 % P
    expect = dict.fromkeys(lay, buf.clone()) if shared else {s: b.clone() for s, b in bufs.items()}
    dv = as_strided(expect["data"], (B, N, S), (lay["data"][2], lay["data"][1], 1), guard + lay["data"][0])
    dv[:, changed] = i32(new64 % P)
    as_strided(expect["parity"], (B, M, S), (lay["parity"][2], lay["parity"][1], 1), guard + lay["parity"][0]).copy_(
        fecc.rs_encode_batch_dev(copy(i32(after64)), M=M))
    fecc.rs_update_batch_dev(view("data"), view("parity"), changed, view("new"))
    torch.cuda.synchronize()
    return all(torch.equal(bufs[s], expect[s]) for s in bufs)


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 2, 3, 5, 6, 7, 64, 1021])
def test_layouts_sentinels_and_pad_words(fecc, S):
    """Stripe-major and block-major on all three sides in every combination, separate buffers; one [B][N + M][pitch] buffer
    with the new rows apart, with new_stripe_words = 0; one [B][N + M + k][pitch] buffer; gaps between rows and stripes."""
    B = 5
    for N, M, changed in ((4, 2, [1]), (12, 4, [0, 11]), (9, 9, [2, 4, 8]), (16, 1, list(range(16))), (64, 16, [5, 6, 60])):
        k = len(changed)
        pitch = ceil4(S) + 4
        sm = lambda n: (0, pitch, n * pitch + 8)                     # stripe-major: a gap between stripes
        bm = lambda n: (0, B * ceil4(S) + 12, ceil4(S))              # block-major: the stripes of one block side by side, then a gap
        for fd in (sm, bm):
            for fp in (sm, bm):
                for fn in (sm, bm):
                    lay = {"data": fd(N), "parity": fp(M), "new": fn(k)}
                    assert run_layout(fecc, B, N, M, S, changed, lay, False), (N, M, S, lay)
        lay = {"data": (0, pitch, N * pitch + 4), "parity": (0, pitch, M * pitch), "new": (0, pitch, 0)}
        assert run_layout(fecc, B, N, M, S, changed, lay, False), ("new_stripe_words = 0", N, M, S)
        stride = (N + M) * pitch + 4
        lay = {"data": (0, pitch, stride), "parity": (N * pitch, pitch, stride), "new": (B * stride + 16, pitch, k * pitch)}
        assert run_layout(fecc, B, N, M, S, changed, lay, True), ("[B][N + M] buffer, new rows apart", N, M, S)
        stride = (N + M + k) * pitch + 4
        lay = {"data": (0, pitch, stride), "parity": (N * pitch, pitch, stride), "new": ((N + M) * pitch, pitch, stride)}
        assert run_layout(fecc, B, N, M, S, changed, lay, True), ("[B][N + M + k] buffer", N, M, S)
        lay = {"new": (0, pitch, stride), "parity": (k * pitch, pitch, stride), "data": ((k + M) * pitch, pitch, stride)}
        assert run_layout(fecc, B, N, M, S, changed, lay, True), ("[B][k + M + N] buffer", N, M, S)


@pytest.mark.gpu
def test_raw_words_are_taken_mod_p(fecc):
    """Stored data, stored parity and new words >= P congruent to small values, and 0xFFFFFFFF, count as their residues"""
    import torch
    B, S = 6, 12
    for N, M, changed in ((4, 2, [0, 3]), (36, 12, [1, 2, 30]), (64, 64, [0, 9]), (18, 1, list(range(18)))):
        small = torch.randint(0, C, (B, N, S), device="cuda", dtype=torch.int64)
        small[:, 0, :3] = 0xFFFFFFFF - P
        parity = fecc.rs_encode_batch_dev(copy(i32(small)), M=M)
        par64 = words(parity)
        new_small = torch.randint(0, C, (B, len(changed), S), device="cuda", dtype=torch.int64)
        new_small[:, 0, 1:4] = 0xFFFFFFFF - P
        after = small.clone()
        after[:, changed] = new_small
        want = fecc.rs_encode_batch_dev(copy(i32(after)), M=M)
        d = copy(i32(small + P))
        d[:, 0, :3] = -1                                            # 0xFFFFFFFF = P + 0xFFFFE
        p = copy(i32(torch.where(par64 < C, par64 + P, par64)))
        n = copy(i32(new_small + P))
        n[:, 0, 1:4] = -1
        fecc.rs_update_batch_dev(d, p, changed, n)
        assert torch.equal(p, want), (N, M)
        assert torch.equal(d[:, changed], i32(new_small)), (N, M)


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
    new64 = rand_words(B * 2, S, gen).view(B, 2, S)
    after = data64.clone()
    after[:, [3, 11]] = new64
    fecc.rs_update_batch_dev(data, parity, [3, 11], copy(i32(new64)))
    assert torch.equal(parity, fecc.rs_encode_batch_dev(copy(i32(after)), M=M))
    assert torch.equal(words(data), after)
    del big, data, parity
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_encode_update_scrub_lose_and_rebuild(fecc):
    """Batch-encode [B][N + M] stripes, batch-update them, scrub sampled stripes (CLEAN), then lose blocks, updated ones among
    them: rs_reconstruct_batch_dev and rs_repair_dev give back the updated blocks"""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(5)
    B, S = 50, 256
    for N, M, changed, ld, lp in ((12, 4, [0, 7], [0, 5], [3]), (18, 3, [17], [17], [0, 2]), (32, 8, [1, 2, 3, 30], [1, 2, 3, 30], [4, 7]),
                                  (64, 16, list(range(8, 40)), list(range(8, 24)), [])):
        buf = torch.zeros((B, N + M, S), dtype=torch.int32, device="cuda")
        buf[:, :N] = i32(rand_words(B * N, S, gen).view(B, N, S))
        fecc.rs_encode_batch_dev(buf[:, :N], buf[:, N:])
        new = copy(i32(raw_words((B, len(changed), S), gen)))
        fecc.rs_update_batch_dev(buf[:, :N], buf[:, N:], changed, new)
        for b in (0, B // 2, B - 1):
            assert fecc.rs_scrub_dev(buf[b, :N], buf[b, N:], 1)[0] == fecc.SCRUB_CLEAN, (N, M, b)
        good = buf.clone()
        buf[:, ld] = 7
        buf[:, [N + j for j in lp]] = 9
        out = fecc.rs_reconstruct_batch_dev(buf[:, :N], buf[:, N:], ld, lp)
        assert torch.equal(out, torch.cat([good[:, ld], good[:, [N + j for j in lp]]], dim=1)), (N, M)
        for b in (0, B - 1):
            d, p = buf[b, :N].clone(), buf[b, N:].clone()
            fecc.rs_repair_dev(d, p, ld, lp)
            assert torch.equal(d, good[b, :N]) and torch.equal(p, good[b, N:]), (N, M, b)


@pytest.mark.gpu
def test_launch_counts(fecc):
    """One launch per call (the table of the N is built); none for B = 0 or nothing changed"""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(6)
    _, data, parity = stripes(fecc, 9, 24, 6, 8, gen)
    for changed in ([3], [0, 5, 7], list(range(24))):
        new = copy(i32(rand_words(9 * len(changed), 8, gen).view(9, len(changed), 8)))
        assert launches(fecc, lambda: fecc.rs_update_batch_dev(data, parity, changed, new)) == 1, changed
    new = torch.zeros((0, 1, 8), dtype=torch.int32, device="cuda")
    assert launches(fecc, lambda: fecc.rs_update_batch_dev(data[:0], parity[:0], [3], new)) == 0
    new = torch.zeros((9, 0, 8), dtype=torch.int32, device="cuda")
    assert launches(fecc, lambda: fecc.rs_update_batch_dev(data, parity, [], new)) == 0


FRESH = r"""
import sys, threading
sys.path.insert(0, %r); sys.path.insert(0, %r)
import numpy as np, torch
import fastecc_b200 as fe
import gfp_ref
from test_update import i32, launches, rand_words
fe.init(0)
gen = torch.Generator(device="cuda"); gen.manual_seed(8)
def case(N, M, B, S, changed):
    # parity by definition: the library has not built the order's table yet
    d64 = rand_words(B * N, S, gen).view(B, N, S)
    p = gfp_ref.encode_rows(d64.permute(1, 0, 2).reshape(N, B * S), [N // M * j for j in range(M)]).reshape(M, B, S).permute(1, 0, 2)
    return i32(d64).contiguous(), i32(p).contiguous(), i32(rand_words(B * len(changed), S, gen).view(B, len(changed), S)), changed
# launches: the first update of an order whose table the process has not built is two launches, the next one
d, p, n, ch = case(48, 16, 5, 40, [1, 2, 47])
first = launches(fe, lambda: fe.rs_update_batch_dev(d, p, ch, n))
again = launches(fe, lambda: fe.rs_update_batch_dev(d, p, ch, n))
# two threads on two streams make the first call of the same order at once
work = [case(36, 12, 300, 64, [0, 35]), case(36, 4, 200, 100, list(range(0, 36, 4)))]
after = []
for d, p, n, ch in work:
    a = d.clone(); a[:, ch] = n; after.append(a)
streams = [torch.cuda.Stream() for _ in range(2)]
go, errors = threading.Barrier(2), []
torch.cuda.synchronize()
def run(i):
    try:
        with torch.cuda.stream(streams[i]):
            go.wait()
            d, p, n, ch = work[i]
            fe.rs_update_batch_dev(d, p, ch, n)
    except Exception as e:
        errors.append(e)
th = [threading.Thread(target=run, args=(i,)) for i in range(2)]
[t.start() for t in th]; [t.join() for t in th]
torch.cuda.synchronize()
ok = not errors and all(torch.equal(work[i][1], fe.rs_encode_batch_dev(after[i], M=work[i][1].shape[1])) for i in range(2))
print(first, again, ok)
"""


@pytest.mark.gpu
def test_table_build_and_first_calls_from_two_threads_in_a_fresh_process():
    import os
    code = FRESH % (ROOT, os.path.join(ROOT, "tests"))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert out.stdout.split() == ["2", "1", "True"], out.stdout + out.stderr


@pytest.mark.gpu
def test_update_batch_does_not_synchronise_the_stream(fecc):
    """The call returns while a kernel ahead of it on the stream is still running, and the host list may be overwritten right
    after the call"""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(9)
    data64, data, parity = stripes(fecc, 100, 16, 4, 64, gen)
    changed = np.array([5, 9], dtype=np.int64)
    new = copy(i32(rand_words(200, 64, gen).view(100, 2, 64)))
    after = data64.clone(); after[:, [5, 9]] = words(new)
    want = fecc.rs_encode_batch_dev(copy(i32(after)), M=4)
    fecc.rs_update_batch_dev(copy(data), copy(parity), changed, new)             # warm: the table
    torch.cuda.synchronize()
    torch.cuda._sleep(1 << 30)
    fecc.rs_update_batch_dev(data, parity, changed, new)
    busy = not torch.cuda.current_stream().query()
    changed[:] = 0
    torch.cuda.synchronize()
    assert busy, "the batch update waited for the stream"
    assert torch.equal(parity, want)


@pytest.mark.gpu
def test_update_batch_argument_table(fecc):
    """Every rule broken on its own gives FASTECC_B200_EINVAL (-1), writes nothing and launches nothing; the listed layouts are
    accepted."""
    import torch
    L = fecc.lib()
    st = torch.cuda.current_stream().cuda_stream
    buf = torch.full((8192,), SENTINEL, dtype=torch.int32, device="cuda")
    a = buf.data_ptr()
    B, S = 3, 8
    wrong = []

    def call(data=a, dpitch=8, dstride=96, N=12, parity=a + 4 * 2048, ppitch=8, pstride=32, M=4, ch=(1, 5), nch=None, new=a + 4 * 4096,
             npitch=8, nstride=16, B=B, S=S):
        lst = None if ch is None else np.asarray(ch, dtype=np.uint32)
        n = (0 if lst is None else lst.size) if nch is None else nch
        return L.fastecc_b200_rs_update_batch(data, dpitch, dstride, N, parity, ppitch, pstride, M, None if lst is None or not lst.size else lst.ctypes.data, n,
                                              new, npitch, nstride, B, S, st)
    shared = dict(data=a, dstride=144, parity=a + 4 * 96, pstride=144, new=a + 4 * 128, nstride=144)   # [B][12 + 4 + 2][8]
    cases = [({}, 0), (dict(S=5), 0), (dict(npitch=24, nstride=8), 0), (shared, 0), (dict(nstride=0), 0), (dict(ch=tuple(range(12)), nstride=96), 0),
             (dict(M=1, pstride=8), 0), (dict(M=12, pstride=96), 0),
             (dict(N=5), -1), (dict(N=27), -1), (dict(N=128, M=4), -1), (dict(N=72, M=8), -1), (dict(M=0), -1), (dict(M=5), -1), (dict(M=24), -1),
             (dict(S=0), -1), (dict(data=None), -1), (dict(parity=None), -1), (dict(new=None), -1),
             (dict(dpitch=4), -1), (dict(ppitch=4), -1), (dict(npitch=4), -1),
             (dict(data=a + 4), -1), (dict(parity=a + 4 * 2048 + 8), -1), (dict(new=a + 4 * 4096 + 4), -1),
             (dict(dpitch=10, S=6), -1), (dict(ppitch=10, S=6), -1), (dict(npitch=10, S=6), -1),
             (dict(dstride=98), -1), (dict(pstride=34), -1), (dict(nstride=18), -1),
             (dict(new=a + 4 * 8), -1), (dict(new=a + 4 * 2048), -1), (dict(parity=a + 4 * 88), -1), (dict(pstride=8), -1),
             (dict(dstride=0), -1), (dict(dstride=48), -1), (dict(shared, new=a + 4 * 8), -1), (dict(shared, new=a + 4 * 96), -1),
             (dict(shared, dstride=128, pstride=128, nstride=128), -1),
             (dict(ch=None, nch=2), -1), (dict(ch=(5, 1)), -1), (dict(ch=(1, 1)), -1), (dict(ch=(1, 12)), -1), (dict(B=1 << 35), -1)]
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
    if "fastecc_b200_rs_update" not in L.fastecc_b200_last_error().decode():
        wrong.append("cap message")
    n0 = fecc.kernel_launches()
    for kw in (dict(B=0), dict(B=0, data=None, parity=None, new=None), dict(ch=()), dict(ch=(), data=None, parity=None, new=None)):
        if call(**kw) != 0:
            wrong.append(("nothing to do", kw))
    if fecc.kernel_launches() != n0:
        wrong.append("launched with nothing to do")
    torch.cuda.synchronize()
    assert not wrong, wrong


@pytest.mark.gpu
def test_update_batch_before_init_is_enoinit():
    code = ("import sys; sys.path.insert(0, %r); import fastecc_b200 as fe; L = fe.lib(); "
            "print(L.fastecc_b200_rs_update_batch(None, 4, 48, 12, None, 4, 16, 4, None, 0, None, 4, 4, 1, 4, None))") % ROOT
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.stdout.split() == ["-4"], out.stdout + out.stderr


# ---- the launch rule of launch_batch_update (csrc/batch.cu), restated ----------------------------------------------------
kUpdateRingBudget = 108 << 10                                        # batch.cu, dynamic shared memory of one of two CTAs per SM
STATIC_SMEM = 64 * 16 + 64 * 4 + 7 * 32 * 16                         # stab[kMaxN] uint4, se[kMaxN], spart[7 * 32] uint4
SM_SHARED = 228 << 10                                                # shared memory of an H100 SM; the SM keeps 1 KiB per CTA


def batch_update(N, M, k, B=1, S=4):
    U = 1 if M <= 8 else 2 if M <= 16 else 3 if M <= 24 else 4 if M <= 32 else 6 if M <= 48 else 8
    W = cdiv(M, U)
    rows = 2 * k + M
    lg_items = 5
    while (rows << lg_items) < sg.kTileChunks:
        lg_items += 1
    items = 1 << lg_items
    units = items // 32 * W
    slices = min(8 // units, k) if U == 1 and units < 8 else 1
    tile = (rows << lg_items) * 16
    stages = min(4, kUpdateRingBudget // tile) if 2 * tile <= kUpdateRingBudget else 1
    s4 = cdiv(S, 4)
    n_items = B * s4
    per_sm = 2 if 2 * (stages * tile + STATIC_SMEM + 1024) <= SM_SHARED else 1
    return Launch("batch_update_kernel<%du>" % U, 256, stages * tile, (U, W, slices, stages), items=items, n_items=n_items,
                  n_tiles=cdiv(n_items, items), per_sm=per_sm)


def batch_update_classes():
    """{(U, W, slices, stages): [(N, M, k), ...]} over every N of the family up to 64, every divisor M, k from 1 to N"""
    out = {}
    for N in ORDERS:
        for M in divisors(N):
            for k in range(1, N + 1):
                out.setdefault(batch_update(N, M, k).key, []).append((N, M, k))
    return out


BATCH_UPDATE = {                                                     # class: (N, M, k, S), S with an odd number of chunks
    (1, 1, 1, 1): (3, 1, 3, 9), (1, 1, 1, 2): (1, 1, 1, 1), (1, 1, 1, 3): (4, 1, 4, 1019),
    (1, 1, 2, 1): (16, 1, 14, 59), (1, 1, 2, 2): (9, 1, 9, 11), (1, 1, 2, 3): (8, 1, 8, 2),
    (1, 1, 4, 1): (32, 1, 27, 130), (1, 1, 4, 2): (18, 1, 18, 3), (1, 1, 4, 3): (16, 1, 16, 18),
    (1, 1, 8, 1): (64, 1, 54, 9), (1, 1, 8, 2): (36, 1, 36, 1), (1, 1, 8, 3): (32, 1, 32, 1019),
    (1, 2, 1, 1): (6, 2, 6, 59), (1, 2, 1, 2): (2, 2, 2, 11), (1, 2, 1, 3): (2, 2, 1, 2),
    (1, 2, 2, 1): (32, 2, 27, 130), (1, 2, 2, 2): (18, 2, 18, 3), (1, 2, 2, 3): (16, 2, 15, 18),
    (1, 2, 4, 1): (64, 2, 54, 9), (1, 2, 4, 2): (36, 2, 36, 1), (1, 2, 4, 3): (32, 2, 31, 1019),
    (1, 3, 1, 1): (3, 3, 2, 59), (1, 3, 1, 2): (3, 3, 1, 11), (1, 3, 1, 3): (3, 3, 3, 2),
    (1, 3, 2, 2): (36, 3, 35, 130), (1, 3, 2, 3): (36, 3, 31, 3), (1, 4, 1, 1): (8, 4, 5, 18),
    (1, 4, 1, 2): (4, 4, 1, 9), (1, 4, 1, 3): (4, 4, 2, 1), (1, 4, 2, 1): (64, 4, 53, 1019),
    (1, 4, 2, 2): (36, 4, 35, 59), (1, 4, 2, 3): (32, 4, 30, 11), (1, 6, 1, 1): (6, 6, 4, 2),
    (1, 6, 1, 2): (6, 6, 2, 130), (1, 6, 1, 3): (6, 6, 1, 3), (1, 8, 1, 1): (8, 8, 3, 18),
    (1, 8, 1, 2): (8, 8, 1, 9), (1, 8, 1, 3): (8, 8, 4, 1), (2, 5, 1, 1): (9, 9, 3, 1019),
    (2, 5, 1, 2): (9, 9, 1, 59), (2, 5, 1, 3): (9, 9, 4, 11), (2, 6, 1, 1): (12, 12, 1, 2),
    (2, 6, 1, 2): (12, 12, 4, 130), (2, 6, 1, 3): (12, 12, 2, 3), (2, 8, 1, 1): (16, 16, 6, 18),
    (2, 8, 1, 2): (16, 16, 2, 9), (2, 8, 1, 3): (16, 16, 1, 1), (3, 6, 1, 1): (18, 18, 5, 1019),
    (3, 6, 1, 2): (18, 18, 1, 59), (3, 6, 1, 3): (18, 18, 7, 11), (3, 8, 1, 1): (24, 24, 2, 2),
    (3, 8, 1, 2): (24, 24, 1, 130), (3, 8, 1, 3): (24, 24, 4, 3), (4, 8, 1, 1): (32, 32, 12, 18),
    (4, 8, 1, 2): (32, 32, 3, 9), (4, 8, 1, 3): (32, 32, 1, 1), (6, 6, 1, 1): (36, 36, 10, 1019),
    (6, 6, 1, 2): (36, 36, 1, 59), (6, 6, 1, 3): (36, 36, 14, 11), (6, 8, 1, 1): (48, 48, 4, 2),
    (6, 8, 1, 2): (48, 48, 1, 130), (6, 8, 1, 3): (48, 48, 8, 3), (8, 8, 1, 1): (64, 64, 23, 18),
    (8, 8, 1, 2): (64, 64, 5, 9), (8, 8, 1, 3): (64, 64, 1, 1),
}


def test_every_update_class_has_a_witness():
    classes = batch_update_classes()
    assert set(classes) == set(BATCH_UPDATE), (set(classes) ^ set(BATCH_UPDATE))
    for cls, (N, M, k, S) in BATCH_UPDATE.items():
        assert batch_update(N, M, k).key == cls and N in ORDERS and N % M == 0 and 1 <= k <= N, cls
    assert {c[2] for c in classes} == {1, 2, 4, 8} and {c[3] for c in classes} == {1, 2, 3}    # row slices and ring depths
    assert all(cdiv(S, 4) % 2 for _, _, _, S in BATCH_UPDATE.values())                    # so that every witness ends on a partial tile


def by_definition(data64, M):
    """The M parity rows of every stripe of canonical data [B, N, S], by definition: [B, M, S]"""
    B, N, S = data64.shape
    out = gfp_ref.encode_rows(data64.permute(1, 0, 2).reshape(N, B * S), [N // M * j for j in range(M)])
    return out.reshape(M, B, S).permute(1, 0, 2)


def update_witness(fecc, N, M, k, S, seed):
    """A witness call over several tiles and a partial last one: adversarial stored words (x + P, 0xFFFFFFFF), garbage in
    unchanged rows and pad words, sentinels around; check() compares every word with the encode by definition"""
    import torch
    from test_stripe_geometry import GUARD, buffer, with_view
    gen = torch.Generator(device="cuda"); gen.manual_seed(seed)
    L = batch_update(N, M, k, 1, S)
    s4 = cdiv(S, 4)
    B = cdiv(3 * L.info["items"] + 5, s4) | 1                      # odd, as s4 is: three tiles and a partial fourth
    changed = [i * N // k for i in range(k)]
    data64 = rand_words(B * N, S, gen).view(B, N, S)
    data64[0::4] = P - 1
    new64 = raw_words((B, k, S), gen)
    after = data64.clone()
    after[:, changed] = new64 % P
    dflat, dview = buffer((B, N), S, gen)
    pflat, pview = buffer((B, M), S, gen)
    nflat, nview = buffer((B, k), S, gen)
    dview.copy_(as_stored(data64, gen))
    others = [i for i in range(N) if i not in changed]
    if others:
        dview[:, others] = garbage((B, len(others), S), gen, "ones")
    pview.copy_(as_stored(by_definition(data64, M), gen))
    nview.copy_(i32(new64))
    keep_d, keep_n, keep_p = dflat.clone(), nflat.clone(), pflat.clone()

    def call():
        fecc.rs_update_batch_dev(dview, pview, changed, nview)

    def check():
        torch.cuda.synchronize()
        want_p = by_definition(after, M)
        assert torch.equal(words(pview), want_p)
        assert torch.equal(pflat, with_view(keep_p, pview, want_p)), "a word outside the parity rows changed"
        want_d = keep_d.clone()
        want_d.as_strided(dview.shape, dview.stride(), dview.storage_offset() - dflat.storage_offset())[:, changed] = i32(new64 % P)
        assert torch.equal(dflat, want_d), "the changed rows are not the canonical new blocks, or another word changed"
        assert torch.equal(nflat, keep_n), "the call wrote into the new rows"
    return call, check, B


@pytest.mark.gpu
@pytest.mark.parametrize("cls", list(BATCH_UPDATE), ids=str)
def test_update_batch_launch_is_the_restated_rule(fecc, cls):
    """Instance, block and shared memory of the witness as predicted; the grid is the tile count capped at the CTAs that fit
    on the SMs"""
    from test_stripe_geometry import expect_launch, launch_of
    sms = fecc.lib().fastecc_b200_num_sms()
    sg.STATIC_SMEM.setdefault("batch_update_kernel", STATIC_SMEM)
    N, M, k, S = BATCH_UPDATE[cls]
    call, _, B = update_witness(fecc, N, M, k, S, 600 + list(BATCH_UPDATE).index(cls))
    L = batch_update(N, M, k, B, S)
    assert L.key == cls
    grid = expect_launch(launch_of(call, r"\b(batch_update_kernel<\d+u>)\(", cls), L, cls)
    assert grid == min(L.info["n_tiles"], L.info["per_sm"] * sms), (cls, grid, L)
    assert L.info["n_items"] % L.info["items"], cls


@pytest.mark.gpu
@pytest.mark.parametrize("cls", list(BATCH_UPDATE), ids=str)
def test_update_batch_witness(fecc, cls):
    N, M, k, S = BATCH_UPDATE[cls]
    call, check, _ = update_witness(fecc, N, M, k, S, 600 + list(BATCH_UPDATE).index(cls))
    call()
    check()
