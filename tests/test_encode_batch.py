"""GPU: the encode of a batch of small stripes (fastecc_b200_rs_encode_batch, csrc/batch.cu, DESIGN 3l).  Every parity row is
compared bit for bit with rs_encode_asym_mixed_dev of its stripe, and on samples with the encode by definition (tests/gfp_ref.py).
The data and everything around the parity rows hold sentinels that must come back unchanged."""
import subprocess
import sys

import numpy as np
import pytest

import gfp_ref
from test_update import C, P, ROOT, SENTINEL, encode, i32, launches, rand_words, raw

ORDERS = [1, 2, 4, 8, 16, 32, 64, 3, 6, 12, 24, 48, 9, 18, 36]
SHAPES = [(N, M) for N in ORDERS for M in range(1, N + 1) if N % M == 0]


def ceil4(x):
    return (x + 3) // 4 * 4


def reference(fecc, data, M):
    """Each stripe's parity through the per-stripe encode: the B stripes of [B, N, S] side by side as one stripe of B S word
    columns (the encode works column by column), [B, M, S]"""
    B, N, S = data.shape
    cols = data.permute(1, 0, 2).reshape(N, B * S).contiguous()
    return encode(fecc, cols, M).reshape(M, B, S).permute(1, 0, 2)


def words(t):
    import torch
    return t.to(torch.int64) & 0xFFFFFFFF


@pytest.mark.gpu
@pytest.mark.parametrize("N,M", SHAPES)
def test_every_shape_against_the_per_stripe_encode(fecc, N, M):
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(1000 * N + M)
    D = N // M
    for B in (1, 7, 300):
        for S in (1, 5, 1024):
            data64 = rand_words(B * N, S, gen).view(B, N, S)
            data = torch.full((B, N, ceil4(S) + 4), SENTINEL, dtype=torch.int32, device="cuda")
            data[..., :S] = raw(data64.reshape(B * N, S), gen).view(B, N, S)
            keep = data.clone()
            par = fecc.rs_encode_batch_dev(data[..., :S], M=M)
            assert torch.equal(data, keep), (N, M, B, S)
            assert torch.equal(par, reference(fecc, i32(data64), M)), (N, M, B, S)
            if B == 7:                                                  # literally one stripe at a time, and by definition
                for b in (0, 3, 6):
                    assert torch.equal(par[b], encode(fecc, i32(data64[b]), M)), (N, M, S, b)
                    assert torch.equal(words(par[b]), gfp_ref.encode_rows(data64[b], [D * j for j in range(M)])), (N, M, S, b)


def sentinel_buffer(n_words):
    import torch
    return torch.full((n_words,), SENTINEL, dtype=torch.int32, device="cuda")


def run_layout(fecc, B, N, M, S, d_off, d_pitch, d_stride, p_off, p_pitch, p_stride, shared, guard=64):
    """Data and parity rows as views of sentinel buffers with `guard` sentinel words around them; shared = one buffer for both.
    Returns whether the call wrote exactly the parity words and left every other word alone, and the parity."""
    import torch
    from torch import as_strided
    gen = torch.Generator(device="cuda"); gen.manual_seed(B * 131 + N * 7 + S)
    d_end = d_off + (B - 1) * d_stride + (N - 1) * d_pitch + ceil4(S)
    p_end = p_off + (B - 1) * p_stride + (M - 1) * p_pitch + ceil4(S)
    if shared:
        buf = sentinel_buffer(guard + max(d_end, p_end) + guard)
        dbuf = pbuf = buf
    else:
        dbuf, pbuf = sentinel_buffer(guard + d_end + guard), sentinel_buffer(guard + p_end + guard)
    data64 = rand_words(B * N, S, gen).view(B, N, S)
    data = as_strided(dbuf, (B, N, S), (d_stride, d_pitch, 1), guard + d_off)
    data.copy_(raw(data64.reshape(B * N, S), gen).view(B, N, S))
    parity = as_strided(pbuf, (B, M, S), (p_stride, p_pitch, 1), guard + p_off)
    want_d = dbuf.clone()
    want_p = pbuf.clone()
    expect = reference(fecc, i32(data64), M)
    as_strided(want_p, (B, M, S), (p_stride, p_pitch, 1), guard + p_off).copy_(expect)
    fecc.rs_encode_batch_dev(data, parity)
    if shared:
        return torch.equal(buf, want_p)
    return torch.equal(dbuf, want_d) and torch.equal(pbuf, want_p)


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 2, 3, 5, 6, 7, 64, 1021])
def test_layouts_sentinels_and_pad_words(fecc, S):
    """Stripe-major and block-major separate buffers in every combination, one [B][N + M][pitch] buffer with the parity below
    the data, one with parity rows interleaved between data rows; pitches with pad words and gaps between rows and stripes."""
    B = 5
    for N, M in ((4, 2), (12, 4), (9, 9), (16, 1)):
        pitch = ceil4(S) + 4
        sm = lambda n: (pitch, n * pitch + 8)                        # stripe-major: (pitch, stride) with a gap between stripes
        bm = lambda n: (B * ceil4(S) + 12, ceil4(S))                 # block-major: stripes of one block side by side, then a gap
        for (dp, ds), (pp, ps) in ((sm(N), sm(M)), (bm(N), bm(M)), (sm(N), bm(M)), (bm(N), sm(M))):
            d_end = (B - 1) * ds + (N - 1) * dp + ceil4(S)
            assert run_layout(fecc, B, N, M, S, 0, dp, ds, 0, pp, ps, False), (N, M, S, dp, ds, pp, ps)
            assert run_layout(fecc, B, N, M, S, 0, dp, ds, d_end + 16, pp, ps, True), ("one buffer, data first", N, M, S, dp, ds, pp, ps)
        stride = (N + M) * pitch + 4
        assert run_layout(fecc, B, N, M, S, M * pitch, pitch, stride, 0, pitch, stride, True), ("parity below", N, M, S)
        stride = 2 * N * pitch + 4                                      # parity row j between data rows j and j + 1
        assert run_layout(fecc, B, N, M, S, 0, 2 * pitch, stride, pitch, 2 * pitch, stride, True), ("interleaved", N, M, S)


@pytest.mark.gpu
def test_raw_words_are_taken_mod_p(fecc):
    """Stored words >= P congruent to small values, and 0xFFFFFFFF, give the parity of their residues"""
    import torch
    B, S = 6, 12
    for N, M in ((4, 2), (36, 12), (64, 64)):
        small = torch.randint(0, C, (B, N, S), device="cuda", dtype=torch.int64)
        stored = i32(small + P)
        stored[:, 0, :3] = -1                                           # 0xFFFFFFFF = P + 0xFFFFE
        residues = small.clone()
        residues[:, 0, :3] = 0xFFFFFFFF - P
        buf = torch.zeros((B, N, 16), dtype=torch.int32, device="cuda")
        buf[..., :S] = stored
        got = fecc.rs_encode_batch_dev(buf[..., :S], M=M)
        assert torch.equal(got, reference(fecc, i32(residues), M)), (N, M)


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
    par = fecc.rs_encode_batch_dev(data, M=M)
    assert torch.equal(par, reference(fecc, i32(data64), M))
    del big, data, par
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_interop_with_scrub_repair_reconstruct_and_update(fecc):
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(5)
    rng = np.random.default_rng(5)
    B, S = 40, 256
    for N, M in ((12, 4), (18, 3), (32, 8), (64, 16)):
        buf = torch.zeros((B, N + M, S), dtype=torch.int32, device="cuda")      # [B][N + M][pitch], parity below the data
        buf[:, M:] = i32(rand_words(B * N, S, gen).view(B, N, S))
        fecc.rs_encode_batch_dev(buf[:, M:], buf[:, :M])
        for b in (0, B // 2, B - 1):
            data, parity = buf[b, M:], buf[b, :M]
            assert fecc.rs_scrub_dev(data, parity, min(M // 2, 4))[0] == fecc.SCRUB_CLEAN, (N, M, b)
            lost_d = sorted(rng.choice(N, size=M // 2, replace=False).tolist())
            lost_p = sorted(rng.choice(M, size=M - M // 2, replace=False).tolist())
            out = fecc.rs_reconstruct_dev(data, parity, lost_d, lost_p)
            want = torch.cat([data[lost_d], parity[lost_p]])
            assert torch.equal(out, want), (N, M, b)
            d, p = data.clone(), parity.clone()
            d[lost_d] = 7; p[lost_p] = 9
            fecc.rs_repair_dev(d, p, lost_d, lost_p)
            assert torch.equal(d, data) and torch.equal(p, parity), (N, M, b)
            changed = sorted(rng.choice(N, size=3, replace=False).tolist())
            new = i32(rand_words(3, S, gen))
            d, p = data.clone(), parity.clone()
            fecc.rs_update_dev(d, p, changed, new)
            stripe = buf[b:b + 1, M:].clone()
            stripe[0, changed] = new
            assert torch.equal(p, fecc.rs_encode_batch_dev(stripe, M=M)[0]), (N, M, b)


@pytest.mark.gpu
def test_launch_counts(fecc):
    """One launch per call once the table of the order exists; none for B = 0"""
    import torch
    data = torch.zeros((9, 24, 8), dtype=torch.int32, device="cuda")
    par = torch.zeros((9, 6, 8), dtype=torch.int32, device="cuda")
    first = launches(fecc, lambda: fecc.rs_encode_batch_dev(data, par))
    assert first in (1, 2)
    assert launches(fecc, lambda: fecc.rs_encode_batch_dev(data, par)) == 1
    assert launches(fecc, lambda: fecc.rs_encode_batch_dev(data[:0], par[:0])) == 0


FRESH = r'''
import sys, threading
sys.path.insert(0, %r); sys.path.insert(0, %r)
import torch
import fastecc_b200 as fe
from test_update import encode
fe.init(0)
def count(fn):
    torch.cuda.synchronize(); n0 = fe.kernel_launches(); fn(); torch.cuda.synchronize(); return fe.kernel_launches() - n0
d = torch.randint(0, 1 << 20, (5, 48, 16), dtype=torch.int32, device="cuda")
p = torch.empty((5, 16, 16), dtype=torch.int32, device="cuda")
counts = [count(lambda: fe.rs_encode_batch_dev(d, p)), count(lambda: fe.rs_encode_batch_dev(d, p)), count(lambda: fe.rs_encode_batch_dev(d[:0], p[:0]))]
ok = [torch.equal(p[b], encode(fe, d[b], 16)) for b in range(5)]
# two threads on two streams, both making the first call of N = 36 at the same time
data = [torch.randint(0, 1 << 31, (300, 36, 64), dtype=torch.int32, device="cuda") for _ in range(2)]
outs, errors, go = [None, None], [], threading.Barrier(2)
streams = [torch.cuda.Stream() for _ in range(2)]
torch.cuda.synchronize()
def work(k):
    try:
        with torch.cuda.stream(streams[k]):
            go.wait()
            outs[k] = fe.rs_encode_batch_dev(data[k], M=(12, 36)[k])
    except Exception as e:
        errors.append(e)
th = [threading.Thread(target=work, args=(k,)) for k in range(2)]
[t.start() for t in th]; [t.join() for t in th]
torch.cuda.synchronize()
for k in range(2):
    M = (12, 36)[k]
    ok += [not errors] + [torch.equal(outs[k][b], encode(fe, data[k][b], M)) for b in (0, 150, 299)]
print(counts, all(ok))
'''


@pytest.mark.gpu
def test_table_launch_and_two_streams_in_a_fresh_process():
    """In a process that has used no order yet: two launches at the first call of an N (the table, then the batch), one after,
    none for B = 0; then two threads on two streams make the first call of another N at the same time."""
    code = FRESH % (ROOT, __import__("os").path.join(ROOT, "tests"))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert out.stdout.split("\n")[0] == "[2, 1, 0] True", out.stdout + out.stderr


@pytest.mark.gpu
def test_batch_does_not_synchronise_the_stream(fecc):
    import torch
    data = torch.randint(0, 1 << 30, (100, 16, 64), dtype=torch.int32, device="cuda")
    par = fecc.rs_encode_batch_dev(data, M=4)
    want = reference(fecc, data, 4)
    torch.cuda.synchronize()
    par.zero_()
    torch.cuda._sleep(1 << 30)
    fecc.rs_encode_batch_dev(data, par)
    busy = not torch.cuda.current_stream().query()
    torch.cuda.synchronize()
    assert busy, "the batch encode waited for the stream"
    assert torch.equal(par, want)


@pytest.mark.gpu
def test_batch_argument_table(fecc):
    """Every rule broken on its own gives FASTECC_B200_EINVAL (-1), writes nothing and launches nothing; every listed layout is
    accepted."""
    import torch
    L = fecc.lib()
    st = torch.cuda.current_stream().cuda_stream
    buf = torch.full((4096,), SENTINEL, dtype=torch.int32, device="cuda")
    a = buf.data_ptr()
    B, N, M, S = 3, 12, 4, 8
    wrong = []

    def call(data=a, dpitch=8, dstride=96, N=N, parity=a + 4 * 2048, ppitch=8, pstride=32, M=M, B=B, S=S):
        return L.fastecc_b200_rs_encode_batch(data, dpitch, dstride, N, parity, ppitch, pstride, M, B, S, st)
    blk = B * 8                                                          # a block-major pitch of 3 stripes x 8 words
    cases = [({}, 0), (dict(S=5), 0), (dict(S=1, dpitch=4, dstride=48, ppitch=4, pstride=16), 0),
             (dict(dpitch=blk, dstride=8), 0), (dict(ppitch=blk, pstride=8), 0), (dict(dpitch=blk, dstride=8, ppitch=blk, pstride=8), 0),
             (dict(parity=a, data=a + 4 * 32, dstride=128, pstride=128), 0),                       # [B][N + M][8], parity below
             (dict(data=a, parity=a + 4 * 96, dstride=128, pstride=128), 0),                       # parity above
             (dict(data=a, dpitch=16, parity=a + 4 * 8, ppitch=16, N=4, M=4, dstride=64, pstride=64), 0),   # interleaved
             (dict(parity=a + 4 * 96 * 3), 0),                                                     # parity right after the data
             (dict(data=None), -1), (dict(parity=None), -1),
             (dict(N=5), -1), (dict(N=27), -1), (dict(N=128, M=4), -1), (dict(N=72, M=8), -1),
             (dict(M=0), -1), (dict(M=5), -1), (dict(M=24), -1), (dict(S=0), -1),
             (dict(dpitch=4), -1), (dict(ppitch=4), -1),
             (dict(data=a + 4), -1), (dict(parity=a + 4 * 2048 + 8), -1),
             (dict(dpitch=10, S=6), -1), (dict(ppitch=10, S=6), -1), (dict(dstride=98), -1), (dict(pstride=34), -1),
             (dict(pstride=16), -1), (dict(ppitch=blk, pstride=4), -1), (dict(ppitch=0, M=4), -1), (dict(pstride=0), -1),
             (dict(parity=a + 4 * 96 * 2), -1), (dict(parity=a + 4 * 8), -1),
             (dict(parity=a + 4 * 32, data=a, dstride=128, pstride=128), -1),                     # parity on data rows 4 .. 7
             (dict(parity=a, data=a + 4 * 32, dstride=128, pstride=96), -1)]                     # one buffer, strides differ
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
    rc = call(N=128, M=4)
    if "fastecc_b200_rs_encode_asym_mixed_dev" not in L.fastecc_b200_last_error().decode():
        wrong.append(("cap message", rc))
    n0 = fecc.kernel_launches()
    if call(B=0) != 0 or call(B=0, data=a, parity=a) != 0 or fecc.kernel_launches() != n0:
        wrong.append("B = 0")
    torch.cuda.synchronize()
    assert not wrong, wrong


@pytest.mark.gpu
def test_batch_before_init_is_enoinit():
    code = ("import sys; sys.path.insert(0, %r); import fastecc_b200 as fe; L = fe.lib(); "
            "print(L.fastecc_b200_rs_encode_batch(None, 4, 16, 4, None, 4, 8, 2, 1, 4, None))") % ROOT
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.stdout.split() == ["-4"], out.stdout + out.stderr
