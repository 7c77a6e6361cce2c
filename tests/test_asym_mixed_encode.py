"""Fewer parity blocks than data blocks for code words of N = 3 * 2^k and 9 * 2^k data blocks:
fastecc_b200_rs_encode_asym_mixed[_dev] (csrc/mixed_radix.cu radix_fold_kernel between the power-of-two transforms, DESIGN 3f).
GPU: the encode against every (N/M)-th parity of the encode by definition (oracle) for every divisor M at small orders, in all
three layouts; bit-identity with rs_encode_asym_dev at a power of two and with rs_encode_mixed_dev at M = N; every (N/M)-th row
of rs_encode_mixed_dev up to 9 * 2^19; the host entry point's argument table (the device one's: test_gpu_parity.py); two host
threads; encode -> scatter into the 2N-row code word -> lose M blocks -> decode with asym_erasures + CErasurePattern(mixed=True).
The kernel's SASS is checked in test_sass_evidence.py."""
import numpy as np
import pytest

P = 0xFFF00001


def divisors(n):
    return [m for m in range(1, n + 1) if n % m == 0]


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


def random_words(N, S, seed):
    return np.random.default_rng(seed).integers(0, P, size=(N, S), dtype=np.uint64).astype(np.uint32)


def rand_dev(N, S, seed):
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    return torch.randint(0, P, (N, S), device="cuda", generator=g, dtype=torch.int64).to(torch.int32)


SMALL = [3, 6, 9, 12, 18, 36, 96, 288, 3 * 1024, 9 * 1024]


@pytest.mark.gpu
@pytest.mark.parametrize("N,S", [(N, S) for N in SMALL for S in (5, 8)])
def test_asym_mixed_encode_equals_the_encode_by_definition(fecc, oracle, N, S):
    import torch
    a = random_words(N, S, 31 * N + S)
    full = by_definition(oracle, a)
    Ms = divisors(N)
    if N > 1000:
        Ms = [1, 2, 3, 9 if N % 9 == 0 else 6, 64, N // 1024, N // 64, N // 9 if N % 9 == 0 else N // 3, N // 8, N // 2, N]
    for M in sorted(set(Ms)):
        want = full[::N // M]
        t = to_dev(a); fecc.rs_encode_asym_mixed_dev(t, M)
        assert np.array_equal(to_host(t)[:M], want), ("dev", M)
        b = a.copy(); fecc.EncodeReedSolomon_asym_mixed(b, N, M, S)
        assert np.array_equal(b[:M], want) and np.array_equal(b[M:], a[M:]), ("host", M)
        b = [row.copy() for row in a]; fecc.EncodeReedSolomon_asym_mixed(b, N, M, S)      # scattered blocks
        assert np.array_equal(np.stack(b), np.concatenate([want, a[M:]])), ("scattered", M)
        pitch = S + 3 if (S + 3) % 4 else S + 2                                         # unaligned pitch: the repack path
        buf = torch.full((N, pitch), 7, dtype=torch.int32, device="cuda")
        view = buf[:, :S]
        view.copy_(to_dev(a))
        fecc.rs_encode_asym_mixed_dev(view, M)
        assert np.array_equal(to_host(view.contiguous())[:M], want), ("repack", M)
        assert bool((buf[:, S:] == 7).all())


@pytest.mark.gpu
@pytest.mark.parametrize("N", [3, 9])
def test_asym_mixed_encode_takes_raw_words_mod_p(fecc, oracle, N):
    """L = 1: step 2 reads the caller's words directly."""
    raw = np.random.default_rng(N).integers(0, 1 << 32, size=(N, 8), dtype=np.uint64).astype(np.uint32)
    raw[0, :4] = [P, P + 1, 0xFFFFFFFF, P - 1]
    full = by_definition(oracle, raw % np.uint32(P))
    for M in divisors(N):
        t = to_dev(raw); fecc.rs_encode_asym_mixed_dev(t, M)
        assert np.array_equal(to_host(t)[:M], full[::N // M]), M


@pytest.mark.gpu
def test_asym_mixed_encode_identity_cases(fecc):
    """A power of two runs rs_encode_asym_dev, M = N runs rs_encode_mixed_dev: bit for bit."""
    import torch
    N, M = 1 << 19, 1 << 16
    x = rand_dev(N, 1024, 1)
    y = x.clone()
    fecc.rs_encode_asym_mixed_dev(x, M)
    fecc.rs_encode_asym_dev(y, M)
    assert torch.equal(x[:M], y[:M])
    del x, y
    torch.cuda.empty_cache()
    for N in (3 << 12, 9 << 12):
        x = rand_dev(N, 64, N)
        y = x.clone()
        fecc.rs_encode_asym_mixed_dev(x, N)
        fecc.rs_encode_mixed_dev(y)
        assert torch.equal(x, y), N


@pytest.mark.gpu
@pytest.mark.parametrize("N,S", [(3 << 18, 64), (9 << 17, 16), (3 << 19, 32), (9 << 19, 16)])
def test_large_asym_mixed_orders_equal_the_full_encode(fecc, N, S):
    import torch
    x = rand_dev(N, S, N + S)
    full = x.clone()
    fecc.rs_encode_mixed_dev(full)
    r = 3 if N % 9 else 9
    for M in (N // 2, N // 8, N // r, 1 << 10, 1):
        t = x.clone()
        fecc.rs_encode_asym_mixed_dev(t, M)
        assert torch.equal(t[:M], full[::N // M]), M
        del t


@pytest.mark.gpu
def test_asym_mixed_encode_4k_blocks(fecc):
    import torch
    N = 3 << 17
    M = N // 8
    x = rand_dev(N, 1024, 7)
    full = x.clone()
    fecc.rs_encode_mixed_dev(full)
    fecc.rs_encode_asym_mixed_dev(x, M)
    assert torch.equal(x[:M], full[::8])


@pytest.mark.gpu
def test_asym_mixed_entry_point_argument_tables(fecc):
    """Every rule of the host entry point's validation broken on its own gives FASTECC_B200_EINVAL (-1); the valid calls give 0.
    The device entry point's table is in test_gpu_parity.py."""
    import ctypes
    import torch
    L = fecc.lib()
    wrong = []
    for N, M in ((0, 1), (5, 1), (27, 3), (12, 0), (12, 5), (12, 24), (1 << 20, 1), (3 << 20, 3)):   # host variant: the same shape rules
        a = np.zeros((max(N, 1), 4), dtype=np.uint32) if N < 64 else None
        tab = (ctypes.c_void_p * max(N, 1))(*([a.ctypes.data + 16 * i for i in range(max(N, 1))] if a is not None else [0]))
        rc = L.fastecc_b200_rs_encode_asym_mixed(tab, N, M, 4)
        if rc != -1:
            wrong.append(("rs_encode_asym_mixed", N, M, rc))
    a = np.zeros((12, 4), dtype=np.uint32)
    tab = (ctypes.c_void_p * 12)(*[a.ctypes.data + 16 * i for i in range(12)])
    for M, S, want in ((4, 0, -1), (4, 4, 0), (12, 4, 0)):
        rc = L.fastecc_b200_rs_encode_asym_mixed(tab, 12, M, S)
        if rc != want:
            wrong.append(("rs_encode_asym_mixed", 12, M, S, rc))
    if L.fastecc_b200_rs_encode_asym_mixed(None, 12, 4, 4) != -1:
        wrong.append(("rs_encode_asym_mixed", "null table"))
    torch.cuda.synchronize()
    assert not wrong, wrong


@pytest.mark.gpu
def test_asym_mixed_dev_calls_from_two_host_threads(fecc):
    """Two host threads, each on its own stream, run encodes of two different (N, M) at the same time (both need the
    context's scratch buffer, for the sub-transforms and the gather); every result equals the single-threaded one."""
    import threading
    import torch
    shapes = [(3 << 14, (3 << 14) // 8, 64), (9 << 13, 1 << 10, 256)]
    inputs = [rand_dev(N, S, N) for N, _, S in shapes]
    torch.cuda.synchronize()
    results, errors = [[], []], []

    def worker(k):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for _ in range(8):
                    t = inputs[k].clone()
                    fecc.rs_encode_asym_mixed_dev(t, shapes[k][1])
                    results[k].append(t[:shapes[k][1]])
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
        N, M, _ = shapes[k]
        want = x.clone()
        fecc.rs_encode_mixed_dev(want)
        torch.cuda.synchronize()
        for i, t in enumerate(results[k]):
            assert torch.equal(t, want[::N // M]), (k, i)


def _round_trip(fecc, data, M, rng):
    """encode M parity blocks, scatter into the 2N-row code word, lose exactly M blocks mixed between data and parity, decode"""
    import torch
    from fastecc_b200 import decoder
    N, S = data.shape
    par = data.clone()
    fecc.rs_encode_asym_mixed_dev(par, M)
    code = torch.zeros((2 * N, S), dtype=data.dtype, device=data.device)
    code[0::2] = data
    code[1::2 * (N // M)] = par[:M]
    n_data = int(rng.integers(0, M + 1))
    lost_data = sorted(rng.choice(N, size=n_data, replace=False).tolist())
    lost_parity = sorted(rng.choice(M, size=M - n_data, replace=False).tolist())
    rows = decoder.asym_erasures(N, M, lost_data, lost_parity)
    assert len(rows) == N
    pat = decoder.CErasurePattern(2 * N, rows, mixed=True)
    damaged = code.clone()
    damaged[torch.as_tensor(rows, device=code.device)] = -1
    rec = pat.recover(damaged)
    pat.close()
    pos = {e: i for i, e in enumerate(rows)}
    for i in lost_data:
        assert torch.equal(rec[pos[2 * i]], data[i]), i
    for j in lost_parity:
        assert torch.equal(rec[pos[2 * (N // M) * j + 1]], par[j]), j


@pytest.mark.gpu
@pytest.mark.parametrize("N", [3, 12, 18, 96, 9 * 64, 3 << 12])
def test_asym_mixed_code_words_are_decoded(fecc, N):
    rng = np.random.default_rng(N)
    for M in sorted({1, N // 3, N // 2 if N % 2 == 0 else 1, N // 8 if N % 8 == 0 else 1, N}):
        for k in range(2):
            _round_trip(fecc, to_dev(random_words(N, 8, 10 * N + M + k)), M, rng)


@pytest.mark.gpu
def test_large_asym_mixed_code_word_round_trip(fecc):
    N = 9 << 17
    _round_trip(fecc, rand_dev(N, 16, 5), N // 8, np.random.default_rng(5))
