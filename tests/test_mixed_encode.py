"""Reed-Solomon code words of N = 3 * 2^k and 9 * 2^k data blocks: fastecc_b200_rs_encode_mixed[_dev] (csrc/mixed_radix.cu
radix_encode_kernel between the power-of-two transforms, DESIGN 3e) and their erasure decoding through
fastecc_b200_rs_decode_pattern_mixed.  CPU: rs_code_order (the kernel's SASS: test_sass_evidence.py).  GPU: the encode
against the encode by definition (oracle), against the power-of-two encode and the reference's golden hash at N = 2^19, against
the composition inverse NTT -> row scaling by rho^m / N -> forward NTT at large orders, the argument tables of the host entry
point and of the pattern builder (the device entry point's: test_gpu_parity.py), and encode -> erase -> decode round trips up
to N = 9 * 2^19."""
import os
import sys

import numpy as np
import pytest

import oracle_lib as ol

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import decode_oracle                                    # noqa: E402

P = 0xFFF00001
HERE = os.path.dirname(os.path.abspath(__file__))


# ---- CPU ---------------------------------------------------------------------------------------------------------------
def test_rs_code_order_boundaries():
    import fastecc_b200 as fe
    for K, N in ((1, 1), (2, 2), (3, 3), (4, 4), (5, 6), (7, 8), (10, 12), (17, 18), (1 << 19, 1 << 19), ((1 << 19) + 1, 9 << 16),
                 (9 << 16, 9 << 16), ((9 << 16) + 1, 3 << 18), (9 << 19, 9 << 19)):
        assert fe.rs_code_order(K) == N, K
    for K in (0, -1, (9 << 19) + 1):
        with pytest.raises(ValueError):
            fe.rs_code_order(K)
    allowed = sorted(r << k for r in (1, 3, 9) for k in range(20))
    for K in list(range(1, 5000)) + [(1 << 19) - 1, (3 << 18) + 1, (9 << 18) + 7]:
        N = fe.rs_code_order(K)
        assert N == min(n for n in allowed if n >= K)
        assert 3 * N <= 4 * K if K <= 1 << 19 else N < 2 * K        # overhead of rounding up: at most 4/3, beyond 2^19 below 2


# ---- GPU ---------------------------------------------------------------------------------------------------------------
def to_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).cuda()


def to_host(t):
    return t.cpu().numpy().view(np.uint32)


def by_definition(oracle, a):
    a = np.ascontiguousarray(a, dtype=np.uint32)
    out = np.empty_like(a)
    oracle.oracle_rs_encode_by_definition(a.ctypes.data, out.ctypes.data, a.shape[0], a.shape[1])
    return out


def rho_powers_over_n(N):
    """rho^m / N for m < N, rho = GF_Root(2N), as uint32 (the scaling of RS.cpp:51-59 at this order)"""
    rho, inv, B = pow(19, (P - 1) // (2 * N), P), pow(N, P - 2, P), 4096
    lo, v = np.empty(B, dtype=np.uint64), inv
    for i in range(B):
        lo[i] = v; v = v * rho % P
    nb, step = (N + B - 1) // B, pow(rho, B, P)
    hi, v = np.empty(nb, dtype=np.uint64), 1
    for i in range(nb):
        hi[i] = v; v = v * step % P
    return ((hi[:, None] * lo[None, :]) % np.uint64(P)).ravel()[:N].astype(np.uint32)


def random_words(N, S, seed):
    return np.random.default_rng(seed).integers(0, P, size=(N, S), dtype=np.uint64).astype(np.uint32)


SMALL = [3, 6, 9, 12, 18, 36, 96, 288, 3 * 64, 9 * 32]


@pytest.mark.gpu
@pytest.mark.parametrize("N,S", [(N, S) for N in SMALL for S in (5, 8)] + [(3 * 1024, 3), (3 * 1024, 4), (9 * 1024, 1), (9 * 1024, 4)])
def test_mixed_encode_equals_the_encode_by_definition(fecc, oracle, N, S):
    a = random_words(N, S, 17 * N + S)
    want = by_definition(oracle, a)
    t = to_dev(a); fecc.rs_encode_mixed_dev(t)
    assert np.array_equal(to_host(t), want)
    b = a.copy(); fecc.EncodeReedSolomon_mixed(b, N, S)
    assert np.array_equal(b, want)
    b = [row.copy() for row in a]; fecc.EncodeReedSolomon_mixed(b, N, S)        # scattered blocks
    assert np.array_equal(np.stack(b), want)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [3, 9, 48, 9 * 64])
def test_mixed_encode_takes_raw_words_mod_p(fecc, oracle, N):
    """M = 1 (N = 3, 9): step 2 reads the caller's words directly."""
    raw = np.random.default_rng(N).integers(0, 1 << 32, size=(N, 8), dtype=np.uint64).astype(np.uint32)
    raw[0, :4] = [P, P + 1, 0xFFFFFFFF, P - 1]
    t = to_dev(raw); fecc.rs_encode_mixed_dev(t)
    assert np.array_equal(to_host(t), by_definition(oracle, raw % np.uint32(P)))


@pytest.mark.gpu
def test_mixed_encode_unaligned_pitch_repack_path(fecc, oracle):
    import torch
    N, S, pitch = 96, 5, 7
    a = random_words(N, S, 5)
    buf = torch.full((N, pitch), 7, dtype=torch.int32, device="cuda")
    view = buf[:, :S]
    view.copy_(to_dev(a))
    fecc.rs_encode_mixed_dev(view)
    assert np.array_equal(to_host(view.contiguous()), by_definition(oracle, a))
    assert bool((buf[:, S:] == 7).all())


@pytest.mark.gpu
def test_mixed_encode_at_a_power_of_two_is_the_encode(fecc, oracle):
    """N = 2^19 x 4 KiB through the mixed entry points: the reference's golden parity hash, bit-identical to rs_encode_dev."""
    import json
    import torch
    G = json.load(open(os.path.join(HERE, "golden", "survey_8c.json")))
    _, S, h0, h1 = [g for g in G["encode_fillA"] if g[0] == 19][0]
    N = 1 << 19
    a = ol.fill_A(oracle, N, S)
    assert ol.ohash(oracle, a) == h0
    t = to_dev(a)
    u = t.clone()
    fecc.rs_encode_mixed_dev(t)
    fecc.rs_encode_dev(u)
    assert torch.equal(t, u)
    assert ol.ohash(oracle, to_host(t)) == h1
    del t, u
    for L, S2 in ((10, 16), (4, 3)):                                              # and the host variant, small
        b = ol.fill_B(oracle, 1 << L, S2)
        c = b.copy(); fecc.EncodeReedSolomon_mixed(c, 1 << L, S2)
        assert np.array_equal(c, ol.o_encode(oracle, b))


@pytest.mark.gpu
@pytest.mark.parametrize("N", [3 << 16, 9 << 17, 3 << 19, 9 << 19])
def test_large_mixed_orders_equal_the_composition(fecc, N):
    """inverse mixed NTT -> row_scale_dev(rho^m / N) -> forward mixed NTT (the encode composed from existing entry points)."""
    import torch
    S = 64
    g = torch.Generator(device="cuda"); g.manual_seed(N)
    x = torch.randint(0, P, (N, S), device="cuda", generator=g, dtype=torch.int64).to(torch.int32)
    want = x.clone()
    consts = to_dev(rho_powers_over_n(N))
    fecc.ntt_dev(want, True)
    fecc._check(fecc.lib().fastecc_b200_row_scale_dev(want.data_ptr(), N, S, want.stride(0), consts.data_ptr(),
                                                      torch.cuda.current_stream().cuda_stream))
    fecc.ntt_dev(want, False)
    fecc.rs_encode_mixed_dev(x)
    assert torch.equal(x, want)


@pytest.mark.gpu
def test_mixed_entry_point_argument_tables(fecc):
    """Every rule of the host entry point's and the pattern builder's validation broken on its own gives FASTECC_B200_EINVAL
    (-1); the valid calls give 0.  The device entry point's table is in test_gpu_parity.py."""
    import ctypes
    import torch
    L = fecc.lib()
    st = torch.cuda.current_stream().cuda_stream
    bad, good = "bad", "good"
    wrong = []
    for N in (0, 5, 27, 1 << 20, 3 << 20):                                        # host variant: the shape rule of the device one
        a = np.zeros((max(N, 1), 4), dtype=np.uint32) if N < 64 else None
        tab = (ctypes.c_void_p * 1)(a.ctypes.data if a is not None else 0)
        rc = L.fastecc_b200_rs_encode_mixed(tab, N, 4)
        if rc != -1:
            wrong.append(("rs_encode_mixed", N, rc))
    pattern = [(bad, n, [1]) for n in (3, 9, 10, 27, 3 << 21, 0, 1)] + [
        (bad, 6, [0, 1, 2, 3]), (bad, 18, list(range(10))), (bad, 6, [2, 1]), (bad, 6, [1, 1]), (bad, 6, [6]),
        (good, 6, [1]), (good, 6, [0, 3, 5]), (good, 18, []), (good, 36, list(range(0, 36, 2))), (good, 9 << 20, [0, (9 << 20) - 1]),
    ]
    for kind, n2, pos in pattern:
        arr = np.asarray(pos, dtype=np.uint32)
        h = ctypes.c_void_p()
        rc = L.fastecc_b200_rs_decode_pattern_mixed(n2, arr.ctypes.data if arr.size else None, arr.size, st, ctypes.byref(h))
        if rc != (0 if kind == good else -1) or (rc == 0) != bool(h.value):
            wrong.append(("rs_decode_pattern_mixed", n2, pos, rc, L.fastecc_b200_last_error().decode()))
        L.fastecc_b200_rs_decode_free(h)
    torch.cuda.synchronize()
    assert not wrong, wrong


def _codeword(fecc, data):
    """the 2N-row code word of the mixed encode: row 2i = data block i, row 2j + 1 = parity block j"""
    import torch
    par = data.clone()
    fecc.rs_encode_mixed_dev(par)
    code = torch.empty((2 * data.shape[0], data.shape[1]), dtype=data.dtype, device=data.device)
    code[0::2] = data
    code[1::2] = par
    return code


@pytest.mark.gpu
@pytest.mark.parametrize("N,n_erased", [(3, 3), (6, 2), (9, 9), (12, 7), (18, 18), (48, 48), (288, 200), (3 << 12, 3 << 12), (9 << 12, 5000)])
def test_mixed_code_words_are_decoded(fecc, N, n_erased):
    """CErasurePattern(2N, E, mixed=True) on code words of the mixed encode: by definition (Lagrange, oracle/decode_oracle.py)
    for N <= 18, by round trip beyond; one pattern serves two code words."""
    import torch
    from fastecc_b200 import decoder
    S = 8
    rng = np.random.default_rng(N + n_erased)
    erased = sorted(rng.choice(2 * N, size=n_erased, replace=False).tolist())
    pat = decoder.CErasurePattern(2 * N, erased, mixed=True)
    for k in range(2):
        code = _codeword(fecc, to_dev(random_words(N, S, 100 * N + k)))
        want = to_host(code)[erased]
        damaged = code.clone()
        damaged[erased] = -1
        rec = to_host(pat.recover(damaged))
        assert np.array_equal(rec, want), k
        if N <= 18:
            rows = [[int(v) for v in r] for r in to_host(code)]
            ref = decode_oracle.recover(rows, erased)
            assert all([int(v) for v in rec[i]] == ref[e] for i, e in enumerate(erased))
    pat.close()
    with pytest.raises(fecc.FastEccError):                                       # the power-of-two pattern keeps rejecting these orders
        decoder.CErasurePattern(2 * N, erased)


@pytest.mark.gpu
@pytest.mark.parametrize("N,S", [(3 << 18, 64), (9 << 19, 16)])
def test_large_mixed_code_words_round_trip(fecc, N, S):
    """Encode, erase a random set of exactly N of the 2N rows, recover: the locator's product tree needs transform orders
    beyond 2^20 here (2^20 at the top level for 3 * 2^18, 9 * 2^20 for 9 * 2^19)."""
    import torch
    from fastecc_b200 import decoder
    g = torch.Generator(device="cuda"); g.manual_seed(N)
    data = torch.randint(0, P, (N, S), device="cuda", generator=g, dtype=torch.int64).to(torch.int32)
    code = _codeword(fecc, data)
    del data
    erased = torch.sort(torch.randperm(2 * N, device="cuda", generator=g)[:N]).values
    want = code[erased].clone()
    code[erased] = -1
    pat = decoder.CErasurePattern(2 * N, erased.cpu().numpy(), mixed=True)
    rec = pat.recover(code)
    assert torch.equal(rec, want)
    pat.close()
