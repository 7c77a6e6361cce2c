"""GPU parity tests (-m gpu): every call goes through the C ABI (include/fastecc_b200.h) and is compared bit for bit
with the CPU oracle, the committed reference vectors, the golden hashes of SURVEY.md 8c and -- at the full
BASELINE sizes -- golden hashes plus size-independent properties (round trip, linearity)."""
import json
import os

import numpy as np
import pytest

import oracle_lib as ol

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
G = json.load(open(os.path.join(HERE, "golden", "survey_8c.json")))
V = np.load(os.path.join(HERE, "golden", "vectors.npz"))
P = 0xFFF00001


def to_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).cuda()


def to_host(t):
    return t.cpu().numpy().view(np.uint32)


def dev_ntt(fecc, a, inverse):
    t = to_dev(a); fecc.ntt_dev(t, inverse); return to_host(t)


def dev_encode(fecc, a):
    t = to_dev(a); fecc.rs_encode_dev(t); return to_host(t)


SHAPES = [(0, 4), (1, 4), (2, 8), (3, 8), (4, 16), (5, 8), (6, 1024), (7, 1024), (8, 20), (9, 36), (10, 16), (10, 100),
          (11, 16), (11, 1024), (12, 40), (13, 64), (14, 12), (15, 32), (16, 16), (17, 8), (18, 4)]


@pytest.mark.parametrize("L,S", SHAPES)
def test_dev_ntt_and_encode_match_oracle(fecc, oracle, L, S):
    N = 1 << L
    a = ol.fill_B(oracle, N, S)
    assert np.array_equal(dev_ntt(fecc, a, False), ol.o_ntt(oracle, a, False))
    assert np.array_equal(dev_ntt(fecc, a, True), ol.o_ntt(oracle, a, True))
    assert np.array_equal(dev_encode(fecc, a), ol.o_encode(oracle, a))


@pytest.mark.parametrize("L,S", [(3, 1), (7, 513), (9, 5), (10, 17), (12, 3), (4, 1023)])
def test_dev_unaligned_sizes_repack_path(fecc, oracle, L, S):
    """SIZE not a multiple of 4 words (the reference default is 2052 bytes = 513 words, RS.cpp:74)."""
    N = 1 << L
    a = ol.fill_B(oracle, N, S)
    assert np.array_equal(dev_ntt(fecc, a, False), ol.o_ntt(oracle, a, False))
    assert np.array_equal(dev_encode(fecc, a), ol.o_encode(oracle, a))


def test_dev_padded_pitch_leaves_layout_intact(fecc, oracle):
    import torch
    N, S, pitch = 256, 24, 40
    a = ol.fill_B(oracle, N, S)
    buf = torch.full((N, pitch), 7, dtype=torch.int32, device="cuda")
    view = buf[:, :S]
    view.copy_(to_dev(a))
    fecc.rs_encode_dev(view)
    assert np.array_equal(to_host(view.contiguous()), ol.o_encode(oracle, a))
    assert bool((buf[:, S + (-S % 4):] == 7).all())          # only the 4-word-aligned data columns are touched


@pytest.mark.parametrize("L,S", [(0, 3), (2, 1), (4, 16), (7, 1024), (7, 513), (10, 24), (11, 1024), (13, 8)])
def test_host_pointer_table_api(fecc, oracle, L, S):
    """MFA_NTT / EncodeReedSolomon body through the reference's T** call surface (ntt.cpp:382, RS.cpp:41-63)."""
    N = 1 << L
    a = ol.fill_B(oracle, N, S)
    b = a.copy(); fecc.MFA_NTT(b, N, S, False); assert np.array_equal(b, ol.o_ntt(oracle, a, False))
    b = a.copy(); fecc.MFA_NTT(b, N, S, True);  assert np.array_equal(b, ol.o_ntt(oracle, a, True))
    b = a.copy(); fecc.EncodeReedSolomon_body(b, N, S); assert np.array_equal(b, ol.o_encode(oracle, a))


@pytest.mark.parametrize("pin", [False, True])
def test_host_api_at_pipelined_sizes(fecc, oracle, pin):
    """The host T** path above its pipelining threshold (32 MiB: column chunks on three streams, csrc/api.cu run_host) --
    what bench.py's e2e times -- from pageable memory, with and without in-place page-locking of the caller's array:
    2^16 x 4 KiB against the oracle word for word, then the headline 2^19 x 4 KiB against the reference's golden hashes."""
    fecc.pin_host_buffers(pin)
    keep = []                                  # the contract of pin_host_buffers: arrays stay alive while it is enabled
    try:
        N, S = 1 << 16, 1024
        a = ol.fill_B(oracle, N, S)
        b = a.copy(); keep.append(b); fecc.EncodeReedSolomon_body(b, N, S); assert np.array_equal(b, ol.o_encode(oracle, a))
        b = a.copy(); keep.append(b); fecc.MFA_NTT(b, N, S, False); assert np.array_equal(b, ol.o_ntt(oracle, a, False))
        b = a.copy(); keep.append(b); fecc.MFA_NTT(b, N, S, True); assert np.array_equal(b, ol.o_ntt(oracle, a, True))
        N = 1 << 19
        _, _, h0, h1 = [g for g in G["encode_fillA"] if g[0] == 19][0]
        a = ol.fill_A(oracle, N, S); keep.append(a)
        assert fecc.reference_hash(a) == h0
        fecc.EncodeReedSolomon_body(a, N, S)
        assert fecc.reference_hash(a) == h1
        oracle.oracle_fill_A(a.ctypes.data, N * S)                       # same array again: the second call finds it page-locked
        fecc.MFA_NTT(a, N, S, False)
        assert fecc.reference_hash(a) == G["ntt_fillA_4096B"]["19"][1]
    finally:
        fecc.pin_host_buffers(False)               # also releases every registration
        del keep


def test_elementwise_entry_points_match_oracle(fecc, oracle):
    """fastecc_b200_gf_mul_dev / _gf_inv_dev / _row_scale_dev directly against GF_Mul / GF_Inv of the oracle (GF(p).cpp:110-127,
    293-297), including non-canonical operands, 0, 1, P-1 and the values around P."""
    import torch
    rng = np.random.default_rng(3)
    edge = np.array([0, 1, 2, P - 2, P - 1, P, P + 1, 0xFFFFFFFF, 0x80000000, 0xFFF00000, 0x000FFFFF], dtype=np.uint32)
    a = np.concatenate([np.repeat(edge, len(edge)), rng.integers(0, 1 << 32, size=5000, dtype=np.uint64).astype(np.uint32)])
    b = np.concatenate([np.tile(edge, len(edge)), rng.integers(0, 1 << 32, size=5000, dtype=np.uint64).astype(np.uint32)])
    L = fecc.lib()
    st = torch.cuda.current_stream().cuda_stream
    ta, tb = to_dev(a), to_dev(b)
    out = torch.empty_like(ta)
    fecc._check(L.fastecc_b200_gf_mul_dev(ta.data_ptr(), tb.data_ptr(), out.data_ptr(), ta.numel(), st))
    want = np.array([oracle.oracle_gf_mul(int(x) % P, int(y) % P) for x, y in zip(a, b)], dtype=np.uint32)
    assert np.array_equal(to_host(out), want)
    fecc._check(L.fastecc_b200_gf_inv_dev(ta.data_ptr(), out.data_ptr(), ta.numel(), st))
    got = to_host(out)
    want = np.array([oracle.oracle_gf_inv(int(x) % P) if int(x) % P else 0 for x in a], dtype=np.uint32)
    assert np.array_equal(got, want)
    assert all(oracle.oracle_gf_mul(int(g), int(x) % P) == 1 for g, x in zip(got[:300], a[:300]) if int(x) % P)
    rows, S, pitch = 77, 36, 40                                            # row i *= c[i]  (the shape of RS.cpp:51-59)
    blk = rng.integers(0, 1 << 32, size=(rows, pitch), dtype=np.uint64).astype(np.uint32)
    c = rng.integers(0, 1 << 32, size=rows, dtype=np.uint64).astype(np.uint32)
    c[:len(edge)] = edge
    tblk, tc = to_dev(blk), to_dev(c)
    fecc._check(L.fastecc_b200_row_scale_dev(tblk.data_ptr(), rows, S, pitch, tc.data_ptr(), st))
    got = to_host(tblk)
    want = ((blk[:, :S].astype(np.uint64) % P) * (c.astype(np.uint64)[:, None] % P) % P).astype(np.uint32)
    assert np.array_equal(got[:, :S], want) and np.array_equal(got[:, S:], blk[:, S:])


@pytest.mark.parametrize("N,S", [(3, 4), (9, 8), (6, 5), (18, 4), (12, 16), (36, 3), (96, 8), (288, 4), (3 * 64, 1024), (9 * 32, 40),
                                 (3 * 1024, 8), (9 * 1024, 4), (3 * 2048, 4)])
def test_orders_3_and_9_times_a_power_of_two(fecc, oracle, N, S):
    """N = 3 * 2^k and 9 * 2^k (csrc/mixed_radix.cu on top of the power-of-two kernels) against the transform by definition
    with GF_Root(N) (Slow_NTT, ntt.cpp:451-483, restated in the oracle), both directions, device and host entry points."""
    a = ol.fill_B(oracle, N, S)
    for inverse in (False, True):
        want = a.copy()
        oracle.oracle_slow_ntt(want.ctypes.data, N, S, 1 if inverse else 0)
        assert np.array_equal(dev_ntt(fecc, a, inverse), want)
        b = a.copy(); fecc.MFA_NTT(b, N, S, inverse); assert np.array_equal(b, want)


@pytest.mark.parametrize("N", [3 << 16, 9 << 15, 3 << 18])
def test_large_mixed_orders_round_trip(fecc, N):
    """inverse(forward(x)) == N * x (mod P) on the device for orders too large for the O(N^2) oracle (S = 64 words)."""
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(N)
    x = torch.randint(0, P, (N, 64), device="cuda", generator=g, dtype=torch.int64)
    t = x.to(torch.int32)
    fecc.ntt_dev(t, False)
    assert int((t.long() & 0xFFFFFFFF).max()) < P
    fecc.ntt_dev(t, True)
    assert bool(((t.long() & 0xFFFFFFFF) == x * N % P).all())


def test_dev_calls_on_two_streams_share_scratch_safely(fecc, oracle):
    """Two-pass NTTs (which ping-pong through the context's ONE scratch buffer) and first-use table builds issued back to back
    on two different streams: the library orders them with events (csrc/api.cu Lease / TableSlot), results must be exact."""
    import torch
    N, S = 1 << 13, 256
    a = ol.fill_B(oracle, N, S)
    b = (a[::-1] ^ np.uint32(0x5A5A5A5A)) % np.uint32(P)
    want_a, want_b = ol.o_ntt(oracle, a, False), ol.o_ntt(oracle, np.ascontiguousarray(b), True)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for _ in range(5):
        ta, tb = to_dev(a), to_dev(np.ascontiguousarray(b))
        torch.cuda.synchronize()
        with torch.cuda.stream(s1):
            fecc.ntt_dev(ta, False)
        with torch.cuda.stream(s2):
            fecc.ntt_dev(tb, True)
        torch.cuda.synchronize()
        assert np.array_equal(to_host(ta), want_a) and np.array_equal(to_host(tb), want_b)
    N = 1 << 14                                                 # a fresh order: the tables built on s1 are used on s2 right away
    c = ol.fill_B(oracle, N, 64)
    want_c = ol.o_ntt(oracle, c, False)
    t1, t2 = to_dev(c), to_dev(c)
    torch.cuda.synchronize()
    with torch.cuda.stream(s1):
        fecc.ntt_dev(t1, False)
    with torch.cuda.stream(s2):
        fecc.ntt_dev(t2, False)
    torch.cuda.synchronize()
    assert np.array_equal(to_host(t1), want_c) and np.array_equal(to_host(t2), want_c)


def test_host_scattered_blocks(fecc, oracle):
    """Blocks at arbitrary addresses, in permuted order (the reference leaves its own table permuted)."""
    N, S = 64, 12
    a = ol.fill_B(oracle, N, S)
    rng = np.random.default_rng(5)
    pool = np.zeros((N * 3, S), dtype=np.uint32)
    rows = rng.permutation(N * 3)[:N]
    blocks = []
    for i in range(N):
        pool[rows[i]] = a[i]; blocks.append(pool[rows[i]])
    fecc.EncodeReedSolomon_body(blocks, N, S)
    want = ol.o_encode(oracle, a)
    for i in range(N):
        assert np.array_equal(blocks[i], want[i])


def test_reference_vectors(fecc):
    for key in V.files:
        if not key.startswith("in_"):
            continue
        L, S = map(int, key.split("_")[1:])
        x = V[key]
        assert np.array_equal(dev_ntt(fecc, x, False), V["ntt0_%d_%d" % (L, S)]), key
        assert np.array_equal(dev_ntt(fecc, x, True), V["ntt1_%d_%d" % (L, S)]), key
        assert np.array_equal(dev_encode(fecc, x), V["enc_%d_%d" % (L, S)]), key


def test_tiny_known_answers(fecc):
    a = np.array([[1], [2], [3], [4]], dtype=np.uint32)
    assert dev_ntt(fecc, a, False).ravel().tolist() == G["ntt4_fwd"]
    assert dev_ntt(fecc, a, True).ravel().tolist() == G["ntt4_inv"]
    a = np.arange(1, 9, dtype=np.uint32).reshape(8, 1)
    assert dev_ntt(fecc, a, False).ravel().tolist() == G["ntt8_fwd"]


def test_non_canonical_inputs_are_taken_mod_p(fecc, oracle):
    """Inputs >= P (the reference requires < P, GF(p).cpp:47): we reduce them, outputs stay canonical."""
    N, S = 512, 8
    rng = np.random.default_rng(11)
    raw = rng.integers(0, 1 << 32, size=(N, S), dtype=np.uint64).astype(np.uint32)
    raw[0, 0] = 0xFFFFFFFF; raw[1, 0] = P; raw[2, 0] = P + 1
    red = (raw.astype(np.uint64) % P).astype(np.uint32)
    out = dev_encode(fecc, raw)
    assert np.array_equal(out, ol.o_encode(oracle, red)) and int(out.max()) < P


@pytest.mark.parametrize("L", [7, 10, 11, 12, 16])
def test_hash_goldens_4096_byte_blocks(fecc, oracle, L):
    """`ntt n L 4096` and `rs L 4096` hashes recorded from the unmodified reference (SURVEY 8c)."""
    N = 1 << L
    a = ol.fill_A(oracle, N, 1024)
    h0, h1 = G["ntt_fillA_4096B"][str(L)]
    assert ol.ohash(oracle, a) == h0
    assert ol.ohash(oracle, dev_ntt(fecc, a, False)) == h1
    for l, s, e0, e1 in G["encode_fillA"]:
        if l == L and s == 1024:
            assert ol.ohash(oracle, dev_encode(fecc, a)) == e1


def test_published_hash_pair(fecc, oracle):
    """Benchmarks.md:491-507."""
    a = ol.fill_A(oracle, 1 << 20, 8)
    assert ol.ohash(oracle, a) == G["published_ntt_2p20_32B"][0]
    assert ol.ohash(oracle, dev_ntt(fecc, a, False)) == G["published_ntt_2p20_32B"][1]


def test_headline_config_encode_goldens(fecc, oracle):
    """BASELINE configs[1]: (n,k)=(2^20,2^19), 4096-byte blocks.  Parity hash must equal the reference's."""
    import torch
    N, S = 1 << 19, 1024
    for fill, key in ((ol.fill_A, "encode_fillA"), (ol.fill_B, "encode_fillB")):
        _, _, h0, h1 = [g for g in G[key] if g[0] == 19][0]
        a = fill(oracle, N, S)
        assert ol.ohash(oracle, a) == h0
        t = to_dev(a); del a
        fecc.rs_encode_dev(t)
        out = to_host(t)
        assert int(out.max()) < P
        assert ol.ohash(oracle, out) == h1
        del t, out
        torch.cuda.empty_cache()


@pytest.mark.parametrize("L", [19, 20])
def test_full_size_ntt_goldens_and_roundtrip(fecc, oracle, L):
    """BASELINE configs[4] end points; iNTT(NTT(x)) == N*x mod P checked on the device for all 2^(L+10) words."""
    import torch
    N, S = 1 << L, 1024
    h0, h1 = G["ntt_fillA_4096B"][str(L)]
    a = ol.fill_A(oracle, N, S)
    assert ol.ohash(oracle, a) == h0
    t = to_dev(a); del a
    orig = t.clone()
    fecc.ntt_dev(t, False)
    assert ol.ohash(oracle, to_host(t)) == h1
    fecc.ntt_dev(t, True)
    for lo in range(0, N, 1 << 16):                            # chunked to bound temporary memory
        want = (orig[lo:lo + (1 << 16)].long() & 0xFFFFFFFF) * N % P
        got = t[lo:lo + (1 << 16)].long() & 0xFFFFFFFF
        assert bool((want == got).all())
    del t, orig
    torch.cuda.empty_cache()


def test_full_size_encode_linearity(fecc, oracle):
    """encode(a + b) == encode(a) + encode(b) (mod P) at N = 2^19 x 4096 B."""
    import torch
    N, S = 1 << 19, 1024
    g = torch.Generator(device="cuda"); g.manual_seed(7)
    a = torch.randint(0, P, (N, S), device="cuda", generator=g, dtype=torch.int64)
    b = torch.randint(0, P, (N, S), device="cuda", generator=g, dtype=torch.int64)
    s = ((a + b) % P).to(torch.int32); a = a.to(torch.int32); b = b.to(torch.int32)
    for t in (a, b, s):
        fecc.rs_encode_dev(t)
    ok = True
    for lo in range(0, N, 1 << 16):
        sl = slice(lo, lo + (1 << 16))
        ok &= bool(((((a[sl].long() & 0xFFFFFFFF) + (b[sl].long() & 0xFFFFFFFF)) % P) == (s[sl].long() & 0xFFFFFFFF)).all())
    assert ok


@pytest.mark.parametrize("L,S", [(11, 16384), (12, 8192), (13, 4096), (14, 2048), (15, 1024), (16, 512), (17, 256), (18, 128), (19, 64), (20, 32)])
def test_many_tiles_column_sample(fecc, oracle, L, S):
    """128 MiB of blocks at every two-pass order: many tiles per CTA, every set-table hand-over and strip shape of the
    persistent tile loop.  The transform is independent per word column, so a sample of columns of
    the device result is compared with the oracle run on just those columns."""
    import torch
    N = 1 << L
    rng = np.random.default_rng(1000 + L)
    a = rng.integers(0, P, size=(N, S), dtype=np.uint64).astype(np.uint32)
    cols = np.r_[0:8, S // 2 - 4:S // 2 + 4, S - 8:S]
    sub = np.ascontiguousarray(a[:, cols])
    ops = [("ntt", False), ("intt", True)] + ([("encode", None)] if L <= 19 else [])
    for name, inv in ops:
        t = to_dev(a)
        if name == "encode":
            fecc.rs_encode_dev(t); want = ol.o_encode(oracle, sub)
        else:
            fecc.ntt_dev(t, inv); want = ol.o_ntt(oracle, sub, inv)
        got = to_host(t[:, torch.from_numpy(cols).cuda()].contiguous())
        assert np.array_equal(got, want), name
        del t
    torch.cuda.empty_cache()


@pytest.mark.parametrize("L,K,S", [(3, 1, 4), (4, 4, 8), (7, 2, 16), (10, 1, 24), (11, 1, 16), (12, 2, 40), (12, 8, 8), (13, 13, 4), (14, 3, 12), (16, 1, 16)])
def test_dev_asymmetric_encode_is_a_subset_of_the_full_encode(fecc, oracle, L, K, S):
    """N data -> M = N/2^K parity blocks (SURVEY 8f rank 2; RS.cpp:65-66): block j' must equal block 2^K * j' of the
    oracle's full encode.  Covers the native path (D on a subset of row sets), the gather path (M < N1, N <= 1024)."""
    N, M = 1 << L, 1 << (L - K)
    a = ol.fill_B(oracle, N, S)
    want = ol.o_encode(oracle, a)[::N // M]
    t = to_dev(a)
    fecc.rs_encode_asym_dev(t, M)
    assert np.array_equal(to_host(t[:M]), want)


@pytest.mark.parametrize("L,K,S", [(5, 2, 3), (9, 1, 513), (12, 1, 64), (13, 2, 1024)])
def test_host_asymmetric_encode(fecc, oracle, L, K, S):
    N, M = 1 << L, 1 << (L - K)
    a = ol.fill_B(oracle, N, S)
    want = ol.o_encode(oracle, a)[::N // M]
    blocks = a.copy()
    fecc.EncodeReedSolomon_asym(blocks, N, M, S)
    assert np.array_equal(blocks[:M], want)
    assert np.array_equal(blocks[M:], a[M:])                  # blocks M..N-1 are not written back


def test_full_size_asymmetric_encode(fecc, oracle):
    """2^19 data blocks -> 2^18 and 2^16 parity blocks of 4096 bytes == every 2nd / 8th block of the full encode, whose
    hash is pinned to the reference's (test_headline_config_encode_goldens)."""
    import torch
    N, S = 1 << 19, 1024
    a = torch.from_numpy(ol.fill_A(oracle, N, S).view(np.int32)).cuda()
    full = a.clone()
    fecc.rs_encode_dev(full)
    assert ol.ohash(oracle, to_host(full)) == [g for g in G["encode_fillA"] if g[0] == 19][0][3]
    for K in (1, 3):
        M = N >> K
        t = a.clone()
        fecc.rs_encode_asym_dev(t, M)
        assert bool((t[:M] == full[::1 << K]).all())
        del t
    del a, full
    torch.cuda.empty_cache()


def test_asymmetric_argument_validation(fecc):
    import torch
    t = torch.zeros((64, 8), dtype=torch.int32, device="cuda")
    for M in (0, 3, 128):
        with pytest.raises(Exception):
            fecc.rs_encode_asym_dev(t, M)


def test_argument_validation(fecc):
    for bad in (5, 7, 15, 27, 3 * 5, 9 * 3 * 4):                # neither 2^k nor 3 * 2^k nor 9 * 2^k
        a = np.zeros((bad, 4), dtype=np.uint32)
        with pytest.raises(fecc.FastEccError) as e:
            fecc.MFA_NTT(a, bad, 4, False)
        assert e.value.code == -1
    a = np.zeros((6, 4), dtype=np.uint32)
    with pytest.raises(fecc.FastEccError) as e:                 # the encoder is defined for powers of two only
        fecc.EncodeReedSolomon_body(a, 6, 4)
    assert e.value.code == -1
    import torch
    t = torch.zeros((1 << 20, 4), dtype=torch.int32, device="cuda")
    with pytest.raises(fecc.FastEccError) as e:                 # rs 20: rejected (the reference computes garbage, GF(p).cpp:274)
        fecc.rs_encode_dev(t)
    assert e.value.code == -1
    fecc.ntt_dev(t, False)                                      # but a 2^20 NTT is legal


def test_failed_allocation_is_not_reported_again(fecc, oracle):
    """A host entry point whose staging buffer cannot be allocated -- 2^10 blocks of 2^31 words would take 8 TiB -- returns
    ENOMEM (-3) before it reads a block or launches anything.  The failure is not charged to the next calls on the same thread:
    an encode on the small-DFT path and one on the pass path right after it succeed and match the oracle."""
    L = fecc.lib()
    blk = np.zeros(16, dtype=np.uint32)
    table = np.full(1 << 10, blk.ctypes.data, dtype=np.uint64)        # 1024 pointers into one small buffer, never read
    launches = fecc.kernel_launches()
    assert L.fastecc_b200_rs_encode(table.ctypes.data, 1 << 10, 1 << 31) == -3
    assert fecc.kernel_launches() == launches
    for N, S in ((16, 8), (1 << 12, 64)):
        a = ol.fill_B(oracle, N, S)
        assert np.array_equal(dev_encode(fecc, a), ol.o_encode(oracle, a))


def test_device_entry_point_argument_tables(fecc):
    """One table of argument tuples per device entry point that takes a row buffer: every rule of its validation, broken on
    its own, must give FASTECC_B200_EINVAL (-1) before anything is launched (kernel_launches() does not move), and the valid
    calls must give 0.  Every pointer lies in ONE device allocation that covers rows x pitch of every tuple (the largest, at
    the 32-bit chunk-count limit, span 2^36 bytes and a little more), so a tuple accepted by mistake stays inside it.  Not
    listed: the shard passes' upper pitch bound (their smallest buffer at that pitch is 64 rows of 16 GiB) and the ENOINIT
    check (the session is initialised)."""
    import ctypes
    import torch
    L = fecc.lib()
    torch.cuda.empty_cache()
    buf = torch.empty((1 << 34) + (1 << 24), dtype=torch.int32, device="cuda")     # 64 GiB + 64 MiB, never initialised
    B = buf.data_ptr()
    C = B + (1 << 36)                                                              # row constants of row_scale: past every row
    D = B + (1 << 30)                                                              # byte blocks of bytes_to_gfp
    X0, X1, Y0, Y1 = (B + k * (64 << 20) for k in range(4))                        # the shard passes' X and Y of ranks 0 and 1
    st = torch.cuda.current_stream().cuda_stream
    MAXP, BIG = 0xFFFFFFF0, 0xFFFFFFF4                                             # largest pitch / a pitch beyond it

    def peers(*p):
        return (ctypes.c_void_p * len(p))(*p)

    bad, good = "bad", "good"
    tables = {
        "ntt_u32_dev": (L.fastecc_b200_ntt_u32_dev, [        # (d, N, SIZE, pitch, inverse)
            (bad, 0, 16, 4, 4, 0), (bad, B, 16, 0, 4, 0),
            (bad, B, 0, 4, 4, 0), (bad, B, 5, 4, 4, 0), (bad, B, 27, 4, 4, 0), (bad, B, 1 << 21, 4, 4, 0), (bad, B, 3 << 21, 4, 4, 0),
            (bad, B, 1, MAXP + 1, BIG, 0), (bad, B, 3, MAXP + 1, BIG, 1),
            (bad, B, 16, 8, 4, 0), (bad, B, 1, 4, BIG, 0), (bad, B, 1, 4, MAXP + 1, 0),
            (bad, B, 1 << 20, 4, 1 << 14, 0), (bad, B, 1 << 20, 4, (1 << 14) - 3, 0),      # 2^20 x ceil(pitch / 4) = 2^32 chunks
            (bad, B, 3, 4, MAXP, 0),                                                  # 3 rows of the largest pitch: r * pitch overflows
            (bad, B + 4, 3, 1 << 31, (1 << 31) + 1, 0),                               # the same at the repacked pitch 2^31
            (good, B, 1 << 12, 64, 64, 0), (good, B, 1 << 12, 64, 64, 1), (good, B, 1 << 20, 4, 4, 0), (good, B, 48, 4, 4, 1),
            (good, B, 16, 5, 7, 0), (good, B + 4, 16, 4, 4, 0),                       # unaligned layouts are repacked
        ]),
        "rs_encode_dev": (L.fastecc_b200_rs_encode_dev, [    # (d, N, SIZE, pitch)
            (bad, 0, 16, 4, 4), (bad, B, 16, 0, 4),
            (bad, B, 0, 4, 4), (bad, B, 5, 4, 4), (bad, B, 3, 4, 4), (bad, B, 48, 4, 4), (bad, B, 1 << 20, 4, 4),
            (bad, B, 1, MAXP + 1, BIG), (bad, B, 16, 8, 4), (bad, B, 1, 4, BIG), (bad, B, 1, 4, MAXP + 1),
            (bad, B, 1 << 19, 4, 1 << 15), (bad, B, 1 << 19, 4, (1 << 15) - 3),
            (good, B, 1 << 12, 64, 64), (good, B, 1 << 19, 4, 4), (good, B, 16, 5, 7), (good, B + 4, 16, 4, 4),
        ]),
        "rs_encode_asym_dev": (L.fastecc_b200_rs_encode_asym_dev, [      # (d, N, M, SIZE, pitch)
            (bad, 0, 16, 4, 4, 4), (bad, B, 16, 4, 0, 4),
            (bad, B, 5, 1, 4, 4), (bad, B, 3, 1, 4, 4), (bad, B, 1 << 20, 1, 4, 4), (bad, B, 1, 1, MAXP + 1, BIG),
            (bad, B, 16, 0, 4, 4), (bad, B, 16, 3, 4, 4), (bad, B, 16, 32, 4, 4),
            (bad, B, 16, 4, 8, 4), (bad, B, 1, 1, 4, BIG), (bad, B, 16, 4, 4, 6), (bad, B + 4, 16, 4, 4, 4),
            (bad, B, 1 << 19, 1, 4, 1 << 15),
            (good, B, 1 << 12, 1 << 10, 64, 64), (good, B, 16, 4, 4, 4), (good, B, 1 << 19, 1 << 18, 4, 4),
        ]),
        "rs_encode_mixed_dev": (L.fastecc_b200_rs_encode_mixed_dev, [    # (d, N, SIZE, pitch)
            *[(bad, B, N, 4, 4) for N in (0, 5, 15, 27, 45, 1 << 20, 3 << 20, 9 << 20)],
            (bad, 0, 48, 4, 4), (bad, B, 48, 0, 4), (bad, B, 48, 8, 4), (bad, B, 3, 4, BIG), (bad, B, 3, MAXP + 1, BIG),
            (bad, B, 3, 4, MAXP),                                                     # 3 rows of the largest pitch: r * pitch overflows
            (bad, B + 4, 3, 1 << 31, (1 << 31) + 1),                                  # the same at the repacked pitch 2^31
            (bad, B, 9 << 19, 4, 3644),                                               # 2^32 16-byte chunks or more
            (good, B, 3, 4, 4), (good, B, 9, 1, 4), (good, B, 3 << 10, 8, 8), (good, B, 9 << 10, 64, 64), (good, B, 1 << 12, 16, 16),
            (good, B, 3 << 19, 4, 4), (good, B, 9 << 19, 4, 4), (good, B, 48, 5, 7), (good, B + 4, 48, 4, 4),
        ]),
        "rs_encode_asym_mixed_dev": (L.fastecc_b200_rs_encode_asym_mixed_dev, [      # (d, N, M, SIZE, pitch)
            *[(bad, B, N, 1, 4, 4) for N in (0, 5, 15, 27, 45, 1 << 20, 3 << 20, 9 << 20)],
            (bad, B, 48, 0, 4, 4), (bad, B, 48, 49, 4, 4), (bad, B, 48, 96, 4, 4), (bad, B, 48, 5, 4, 4), (bad, B, 48, 9, 4, 4),
            (bad, B, 3, 2, 4, 4), (bad, B, 9 << 19, 7, 4, 4), (bad, B, 1 << 10, 3, 4, 4),
            (bad, 0, 48, 16, 4, 4), (bad, B, 48, 16, 0, 4), (bad, B, 48, 16, 8, 4), (bad, B, 3, 1, 4, BIG), (bad, B, 3, 1, MAXP + 1, BIG),
            (bad, B, 3, 1, 4, MAXP),                                                  # 3 rows of the largest pitch: r * pitch overflows
            (bad, B, 9 << 19, 9, 4, 3644),                                            # 2^32 16-byte chunks or more
            (good, B, 3, 1, 4, 4), (good, B, 3, 3, 4, 4), (good, B, 9, 3, 1, 4), (good, B, 3 << 10, 1 << 10, 8, 8), (good, B, 9 << 10, 9, 64, 64),
            (good, B, 1 << 12, 1 << 9, 16, 16), (good, B, 3 << 19, 1 << 10, 4, 4), (good, B, 9 << 19, 1, 4, 4), (good, B, 9 << 19, 9 << 19, 4, 4),
            (good, B, 48, 12, 5, 7), (good, B + 4, 48, 6, 4, 4),
        ]),
        "row_scale_dev": (L.fastecc_b200_row_scale_dev, [    # (d, rows, SIZE, pitch, consts)
            (bad, 0, 16, 4, 4, C), (bad, B, 16, 4, 4, 0), (bad, B, 16, 0, 4, C),
            (bad, B, 16, 8, 4, C), (bad, B, 1, 4, BIG, C), (bad, B, 16, 4, 6, C), (bad, B + 4, 16, 4, 4, C),
            (good, B, 77, 36, 40, C), (good, B, 1 << 20, 4, 1 << 14, C),             # no chunk-count limit here
        ]),
        "bytes_to_gfp_dev": (L.fastecc_b200_bytes_to_gfp_dev, [          # (bytes, words, n_blocks, W, pitch)
            (bad, 0, B, 64, 16, 20), (bad, D, 0, 64, 16, 20),
            (bad, D, B, 64, 0, 4), (bad, D, B, 64, 1028, 1032), (bad, D, B, 64, 6, 8),
            (bad, D, B, 64, 16, 16), (bad, D, B, 64, 16, 18), (bad, D + 4, B, 64, 16, 20), (bad, D, B + 4, 64, 16, 20),
            (bad, B, B, 1 << 31, 4, 8),
            (good, D, B, 64, 16, 20),
        ]),
        "rs_encode_shard_pass": (L.fastecc_b200_rs_encode_shard_pass, [  # (d, N, ranks, rank, SIZE, pitch, which)
            (bad, 0, 1 << 12, 2, 0, 4, 4, 0), (bad, B, 1 << 12, 2, 0, 4, 4, -1), (bad, B, 1 << 12, 2, 0, 4, 4, 3),
            (bad, B, 1 << 12, 2, -1, 4, 4, 0), (bad, B, 1 << 12, 2, 2, 4, 4, 0), (bad, B, 1 << 12, 0, 0, 4, 4, 0),
            (bad, B, 1 << 12, 1, 0, 4, 4, 0), (bad, B, 1 << 12, 3, 0, 4, 4, 0), (bad, B, 1 << 10, 2, 0, 4, 4, 0),
            (bad, B, 1 << 20, 2, 0, 4, 4, 0), (bad, B, 3 << 11, 2, 0, 4, 4, 0), (bad, B, 1 << 11, 64, 0, 4, 4, 0),
            (bad, B, 1 << 12, 2, 0, 0, 4, 0), (bad, B, 1 << 12, 2, 0, 8, 4, 0), (bad, B, 1 << 12, 2, 0, 4, 6, 0),
            (bad, B + 4, 1 << 12, 2, 0, 4, 4, 0), (bad, B, 1 << 19, 2, 0, 4, 1 << 16, 0),
            (bad, B, 1 << 19, 1024, 0, 4, 4, 1),                                   # N2 = 1024 ranks, but N1 = 512 row sets for pass 1
            *[(good, B, 1 << 12, 2, r, 4, 4, w) for r in (0, 1) for w in (0, 1, 2)], (good, B, 1 << 11, 2, 0, 4, 4, 0),
        ]),
        "rs_encode_shard_pass_p2p": (L.fastecc_b200_rs_encode_shard_pass_p2p, [      # (src, peers, N, ranks, rank, SIZE, pitch, which)
            (bad, 0, peers(Y0, Y1), 1 << 12, 2, 0, 4, 4, 0), (bad, X0, None, 1 << 12, 2, 0, 4, 4, 0),
            (bad, X0, peers(Y0, 0), 1 << 12, 2, 0, 4, 4, 0), (bad, X0, peers(Y0, Y1 + 4), 1 << 12, 2, 0, 4, 4, 0),
            (bad, X0, peers(Y0 + 4, Y1), 1 << 12, 2, 0, 4, 4, 0),
            (bad, X0, peers(Y0, Y1), 1 << 12, 2, 0, 4, 4, -1), (bad, X0, peers(Y0, Y1), 1 << 12, 2, 0, 4, 4, 3),
            (bad, X0, peers(Y0, Y1), 1 << 12, 2, -1, 4, 4, 0), (bad, X0, peers(Y0, Y1), 1 << 12, 2, 2, 4, 4, 0),
            (bad, X0, peers(Y0), 1 << 12, 1, 0, 4, 4, 0), (bad, X0, peers(Y0, Y1, Y1), 1 << 12, 3, 0, 4, 4, 0),
            (bad, X0, peers(Y0, Y1), 1 << 11, 2, 0, 4, 4, 0), (bad, X0, peers(Y0, Y1), 1 << 20, 2, 0, 4, 4, 0),
            (bad, X0, peers(*[Y0] * 16), 1 << 19, 16, 0, 4, 4, 0),
            (bad, X0, peers(Y0, Y1), 1 << 12, 2, 0, 0, 4, 0), (bad, X0, peers(Y0, Y1), 1 << 12, 2, 0, 8, 4, 0),
            (bad, X0, peers(Y0, Y1), 1 << 12, 2, 0, 4, 6, 0), (bad, X0 + 4, peers(Y0, Y1), 1 << 12, 2, 0, 4, 4, 0),
            (bad, B, peers(B, B), 1 << 19, 2, 0, 4, 1 << 16, 0),
            *[c for r, (x, y) in enumerate(((X0, Y0), (X1, Y1))) for c in (
                (good, x, peers(Y0, Y1), 1 << 12, 2, r, 4, 4, 0), (good, y, peers(X0, X1), 1 << 12, 2, r, 4, 4, 1),
                (good, x, peers(X0, X1), 1 << 12, 2, r, 4, 4, 2))],
        ]),
        "ntt_shard_pass_p2p": (L.fastecc_b200_ntt_shard_pass_p2p, [      # (src, peers, N, ranks, rank, SIZE, pitch, inverse, which)
            (bad, 0, peers(Y0, Y1), 1 << 12, 2, 0, 4, 4, 0, 0), (bad, X0, None, 1 << 12, 2, 0, 4, 4, 0, 0),
            (bad, X0, peers(Y0, 0), 1 << 12, 2, 0, 4, 4, 0, 0), (bad, X0, peers(Y0, Y1 + 4), 1 << 12, 2, 0, 4, 4, 0, 0),
            (bad, X0, peers(Y0 + 4, Y1), 1 << 12, 2, 0, 4, 4, 0, 0),
            (bad, X0, peers(Y0, Y1), 1 << 12, 2, 0, 4, 4, 0, -1), (bad, X0, peers(Y0, Y1), 1 << 12, 2, 0, 4, 4, 0, 2),
            (bad, X0, peers(Y0, Y1), 1 << 12, 2, -1, 4, 4, 0, 0), (bad, X0, peers(Y0, Y1), 1 << 12, 2, 2, 4, 4, 0, 0),
            (bad, X0, peers(Y0), 1 << 12, 1, 0, 4, 4, 0, 0), (bad, X0, peers(Y0, Y1, Y1), 1 << 12, 3, 0, 4, 4, 0, 0),
            (bad, X0, peers(Y0, Y1), 1 << 10, 2, 0, 4, 4, 0, 0), (bad, X0, peers(Y0, Y1), 1 << 21, 2, 0, 4, 4, 0, 0),
            (bad, X0, peers(*[Y0] * 16), 1 << 20, 16, 0, 4, 4, 0, 0),
            (bad, X0, peers(Y0, Y1), 1 << 12, 2, 0, 0, 4, 0, 0), (bad, X0, peers(Y0, Y1), 1 << 12, 2, 0, 8, 4, 0, 0),
            (bad, X0, peers(Y0, Y1), 1 << 12, 2, 0, 4, 6, 0, 0), (bad, X0 + 4, peers(Y0, Y1), 1 << 12, 2, 0, 4, 4, 0, 0),
            (bad, B, peers(B, B), 1 << 20, 2, 0, 4, 1 << 15, 0, 0),
            *[c for r, (x, y) in enumerate(((X0, Y0), (X1, Y1))) for n in (1 << 11, 1 << 12, 1 << 20) for c in (
                (good, x, peers(Y0, Y1), n, 2, r, 4, 4, r, 0), (good, y, peers(X0, X1), n, 2, r, 4, 4, r, 1))],
        ]),
    }
    wrong = []
    for name, (fn, cases) in tables.items():
        for kind, *args in cases:
            launches = L.fastecc_b200_kernel_launches()
            rc = fn(*args, st)
            if rc != (0 if kind == good else -1):
                wrong.append((name, args, rc, L.fastecc_b200_last_error().decode()))
            if kind == bad and L.fastecc_b200_kernel_launches() != launches:           # rejected before anything is launched
                wrong.append((name, args, "launched", L.fastecc_b200_kernel_launches() - launches))
    torch.cuda.synchronize()
    del buf
    torch.cuda.empty_cache()
    assert not wrong, wrong


def test_dev_calls_from_two_host_threads(fecc, oracle):
    """Two host threads, each on its own stream, run NTTs and encodes of two different two-pass orders (2^12 x 64 and
    2^15 x 256 words) at the same time; the NTTs of both need the context's one Y buffer, which the larger may have to grow
    while the other is using it.  Scratch leases (csrc/api.cu) serialise them on the buffer: every result must equal the
    single-threaded result of the same input, computed afterwards so that the threads meet a buffer that has not grown yet."""
    import threading
    import torch
    inputs = [to_dev(ol.fill_B(oracle, N, S)) for N, S in ((1 << 12, 64), (1 << 15, 256))]
    ops = [lambda t: fecc.ntt_dev(t, False), lambda t: fecc.ntt_dev(t, True), fecc.rs_encode_dev]
    torch.cuda.synchronize()
    results, errors = [[], []], []

    def worker(k):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for i in range(10):
                    t = inputs[k].clone()
                    ops[i % len(ops)](t)
                    results[k].append(t)
            s.synchronize()
        except Exception as e:                       # re-raised on the main thread
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(k,)) for k in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for k, x in enumerate(inputs):
        want = []
        for op in ops:
            t = x.clone(); op(t); want.append(t)
        torch.cuda.synchronize()
        for i, t in enumerate(results[k]):
            assert torch.equal(t, want[i % len(ops)]), (k, i)
