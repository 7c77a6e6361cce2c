"""GPU: repair of a stored stripe in place (fastecc_b200_rs_repair_pattern / _repair, csrc/repair.cu, DESIGN 3g).
Small orders against every (N/M)-th parity of the encode by definition (oracle), with garbage in the lost rows, raw words >= P
in the surviving rows and a sentinel in the pad columns; large orders as library encode -> lose -> repair -> bitwise equal,
including several column chunks; one pattern over several stripes and SIZEs; two host threads on two streams; the argument
table.  The algebra is restated on the CPU in test_repair_algebra.py, the kernels' SASS is checked in test_repair_abi.py."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

P = 0xFFF00001
C = (1 << 32) - P
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0x5EED5EED


def divisors(n):
    return [m for m in range(1, n + 1) if n % m == 0]


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


def rand_dev(N, S, seed):
    import torch
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    return torch.randint(0, P, (N, S), device="cuda", generator=g, dtype=torch.int64).to(torch.int32)


def loss_sets(N, M, rng):
    """none; parity only; data only; all M losses as data; |E_d| + |E_p| = M; one block of each kind"""
    def pick(n, k):
        return sorted(rng.choice(n, size=k, replace=False).tolist())
    nd = int(rng.integers(0, M + 1))
    return [([], []), ([], pick(M, M)), (pick(N, max(1, M // 2)), []), (pick(N, M), []), (pick(N, nd), pick(M, M - nd)),
            ([N - 1], []), ([], [M - 1])]


def padded(rows, S, pitch):
    """rows (uint32 [n, S]) in a [n, pitch] buffer with the sentinel in the pad columns"""
    buf = np.full((rows.shape[0], pitch), SENTINEL, dtype=np.uint32)
    buf[:, :rows.shape[1]] = rows
    return buf


SMALL = [1, 2, 3, 4, 6, 8, 9, 12, 18, 32, 36, 96, 288, 1024, 3 * 1024, 9 * 1024]


def sample_divisors(N):
    Ms = divisors(N)
    if N < 1000:
        return Ms
    return sorted({m for m in (1, 2, 3, 4, 9, 64, N // 1024, N // 64, N // 9, N // 8, N // 3, N // 2, N) if m >= 1 and N % m == 0})


@pytest.mark.gpu
@pytest.mark.parametrize("N,S", [(N, S) for N in SMALL for S in (5, 8)])
def test_repair_against_the_encode_by_definition(fecc, oracle, N, S):
    from fastecc_b200 import decoder
    rng = np.random.default_rng(17 * N + S)
    data = rng.integers(0, P, size=(N, S), dtype=np.uint64).astype(np.uint32)
    data[:, 0] = rng.integers(0, C, size=N)                                  # words that can be stored raw as x + P
    raw_data = data.copy()
    raw_data[:, 0] += np.uint32(P)
    full = by_definition(oracle, data)
    pitch = S + 4 - S % 4                                                    # at least one pad word per row
    for M in sample_divisors(N):
        parity = full[::N // M]
        for lost_data, lost_parity in loss_sets(N, M, rng):
            d = padded(raw_data, S, pitch)
            p = padded(parity, S, pitch)
            if lost_data:
                d[lost_data, :S] = rng.integers(P, 1 << 32, size=(len(lost_data), S), dtype=np.uint64).astype(np.uint32)
            if lost_parity:
                p[lost_parity, :S] = rng.integers(P, 1 << 32, size=(len(lost_parity), S), dtype=np.uint64).astype(np.uint32)
            want_d, want_p = d.copy(), p.copy()
            want_d[lost_data, :S] = data[lost_data]
            want_p[lost_parity, :S] = parity[lost_parity]
            td, tp = to_dev(d), to_dev(p)
            r = decoder.Repair(N, M, lost_data, lost_parity)
            r.repair(td[:, :S], tp[:, :S])
            r.close()
            assert np.array_equal(to_host(td), want_d), (M, lost_data, lost_parity)
            assert np.array_equal(to_host(tp), want_p), (M, lost_data, lost_parity)


def _encode(fecc, data, M):
    import torch
    buf = data.clone()
    fecc.rs_encode_asym_mixed_dev(buf, M)
    par = buf[:M].clone() if M < data.shape[0] else buf
    torch.cuda.synchronize()
    return par


def _lose_and_repair(fecc, data, parity, n_lost, rng, S=None):
    """lose n_lost blocks split at random between data and parity (garbage in their rows), repair, compare bitwise"""
    import torch
    N, M = data.shape[0], parity.shape[0]
    nd = int(rng.integers(0, n_lost + 1))
    lost_d = sorted(rng.choice(N, size=nd, replace=False).tolist())
    lost_p = sorted(rng.choice(M, size=n_lost - nd, replace=False).tolist())
    want_d, want_p = data.clone(), parity.clone()
    S = S or data.shape[1]
    if lost_d:
        data[:, :S][torch.as_tensor(lost_d, device=data.device)] = -1
    if lost_p:
        parity[:, :S][torch.as_tensor(lost_p, device=data.device)] = -7
    fecc.rs_repair_dev(data[:, :S], parity[:, :S], lost_d, lost_p)
    torch.cuda.synchronize()
    assert torch.equal(data, want_d), (N, M, len(lost_d), len(lost_p))
    assert torch.equal(parity, want_p), (N, M, len(lost_d), len(lost_p))


@pytest.mark.gpu
@pytest.mark.parametrize("M_div", [1, 16])
def test_large_repair_2p19_4k_blocks(fecc, M_div):
    import torch
    N = 1 << 19
    data = rand_dev(N, 1024, 3 + M_div)
    parity = _encode(fecc, data, N // M_div)
    _lose_and_repair(fecc, data, parity, N // M_div, np.random.default_rng(M_div))
    del data, parity
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("M_div", [9, 1])
def test_large_repair_9x2p19(fecc, M_div):
    import torch
    N = 9 << 19
    data = rand_dev(N, 16, 9 + M_div)
    parity = _encode(fecc, data, N // M_div)
    _lose_and_repair(fecc, data, parity, N // M_div, np.random.default_rng(90 + M_div))
    del data, parity
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_repair_in_column_chunks_keeps_the_pad_words(fecc):
    """3 * 2^19 rows of SIZE 1022 in a 1024-word pitch, M = N / 3: the (N + M)-row workspace of the whole row would be 8 GiB, so
    the repair runs in two column chunks, the second one ending in a partial 16-byte group."""
    import torch
    N, S = 3 << 19, 1022
    M = N // 3
    data = rand_dev(N, 1024, 33)
    data[:, S:] = SENTINEL
    buf = data.clone()
    fecc.rs_encode_asym_mixed_dev(buf[:, :S], M)                            # parity of the first S words, in the same pitch
    parity = buf[:M].clone()
    del buf
    torch.cuda.empty_cache()
    parity[:, S:] = SENTINEL
    _lose_and_repair(fecc, data, parity, M, np.random.default_rng(3), S=S)
    del data, parity
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_one_pattern_repairs_several_stripes_and_sizes(fecc):
    import torch
    from fastecc_b200 import decoder
    N, M = 3 << 10, 3 << 6
    rng = np.random.default_rng(8)
    lost_d = sorted(rng.choice(N, size=M // 2, replace=False).tolist())
    lost_p = sorted(rng.choice(M, size=M - M // 2, replace=False).tolist())
    r = decoder.Repair(N, M, lost_d, lost_p)
    for seed, S in ((1, 64), (2, 64), (3, 1000), (4, 8)):
        data = rand_dev(N, S, seed)
        parity = _encode(fecc, data, M)
        want_d, want_p = data.clone(), parity.clone()
        data[lost_d] = 5
        parity[lost_p] = 6
        r.repair(data, parity)
        torch.cuda.synchronize()
        assert torch.equal(data, want_d) and torch.equal(parity, want_p), (seed, S)
    r.close()


@pytest.mark.gpu
def test_repairs_from_two_host_threads(fecc):
    """Two host threads, each on its own stream, repair stripes of two different shapes at the same time (both use the
    context's repair workspace and the encode's scratch buffer); every result is correct."""
    import threading
    import torch
    from fastecc_b200 import decoder
    shapes = [(3 << 14, (3 << 14) // 8, 64), (1 << 15, 1 << 11, 256)]
    cases = []
    for k, (N, M, S) in enumerate(shapes):
        rng = np.random.default_rng(k)
        data = rand_dev(N, S, 70 + k)
        parity = _encode(fecc, data, M)
        lost_d = sorted(rng.choice(N, size=M // 3, replace=False).tolist())
        lost_p = sorted(rng.choice(M, size=M - M // 3, replace=False).tolist())
        cases.append((data, parity, lost_d, lost_p, decoder.Repair(N, M, lost_d, lost_p)))
    torch.cuda.synchronize()
    results, errors = [[], []], []

    def worker(k):
        try:
            data, parity, lost_d, lost_p, r = cases[k]
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for i in range(6):
                    d, p = data.clone(), parity.clone()
                    d[lost_d] = i
                    p[lost_p] = -i
                    r.repair(d, p)
                    results[k].append((d, p))
            s.synchronize()
        except Exception as e:                       # re-raised on the main thread
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(k,)) for k in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for k, (data, parity, _, _, r) in enumerate(cases):
        r.close()
        for i, (d, p) in enumerate(results[k]):
            assert torch.equal(d, data) and torch.equal(p, parity), (k, i)


@pytest.mark.gpu
def test_repair_argument_table(fecc):
    """Every rule of the validation broken on its own gives FASTECC_B200_EINVAL (-1); the valid calls give 0."""
    import torch
    L = fecc.lib()
    st = torch.cuda.current_stream().cuda_stream
    wrong = []

    def pattern(N, M, ld, lp, out=True):
        a = np.asarray(ld, dtype=np.uint32); b = np.asarray(lp, dtype=np.uint32)
        h = ctypes.c_void_p()
        rc = L.fastecc_b200_rs_repair_pattern(N, M, a.ctypes.data if a.size else None, a.size, b.ctypes.data if b.size else None, b.size,
                                              st, ctypes.byref(h) if out else None)
        return rc, h

    for args, want in ((((12, 4, [1], [2])), 0), ((0, 1, [], []), -1), ((5, 1, [], []), -1), ((27, 3, [], []), -1), ((1 << 20, 1, [], []), -1),
                       ((3 << 20, 3, [], []), -1), ((12, 0, [], []), -1), ((12, 5, [], []), -1), ((12, 24, [], []), -1),
                       ((12, 4, [12], []), -1), ((12, 4, [], [4]), -1), ((12, 4, [3, 1], []), -1), ((12, 4, [], [2, 2]), -1),
                       ((12, 4, [0, 1, 2], [0, 1]), -1), ((12, 4, [0, 1, 2, 3, 4], []), -1), ((12, 4, [0, 1], [0, 1]), 0), ((9 << 19, 9, [], []), 0)):
        rc, h = pattern(*args)
        if rc != want:
            wrong.append(("pattern", args, rc))
        L.fastecc_b200_rs_repair_free(h)
    if L.fastecc_b200_rs_repair_pattern(12, 4, None, 1, None, 0, st, ctypes.byref(ctypes.c_void_p())) != -1:
        wrong.append("null lost_data")
    if L.fastecc_b200_rs_repair_pattern(12, 4, None, 0, None, 1, st, ctypes.byref(ctypes.c_void_p())) != -1:
        wrong.append("null lost_parity")
    if pattern(12, 4, [1], [], out=False)[0] != -1:
        wrong.append("null output")
    rc, h = pattern(12, 4, [1], [2])
    assert rc == 0
    buf = torch.zeros((16 * 3, 8), dtype=torch.int32, device="cuda")
    data, par = buf[:12], buf[32:36]
    d, p = data.data_ptr(), par.data_ptr()
    for args, want in (((d, 8, p, 8, 8), 0), ((d, 8, p, 8, 5), 0), ((None, 8, p, 8, 8), -1), ((d, 8, None, 8, 8), -1), ((d, 8, p, 8, 0), -1),
                       ((d, 6, p, 8, 6), -1), ((d, 8, p, 6, 6), -1), ((d, 4, p, 8, 8), -1), ((d + 4, 8, p, 8, 4), -1), ((d, 8, p + 8, 8, 4), -1),
                       ((d, 8, d + 8 * 11 * 4, 8, 8), -1), ((d + 64, 8, d, 8, 8), -1)):
        rc = L.fastecc_b200_rs_repair(h, *args, st)
        if rc != want:
            wrong.append(("repair", args, rc))
    if L.fastecc_b200_rs_repair(None, d, 8, p, 8, 8, st) != -1:
        wrong.append("null pattern")
    L.fastecc_b200_rs_repair_free(h)
    torch.cuda.synchronize()
    assert not wrong, wrong


@pytest.mark.gpu
def test_repair_before_init_is_enoinit():
    """In a fresh process that never called fastecc_b200_init, both entry points fail with FASTECC_B200_ENOINIT (-4)."""
    code = ("import ctypes, sys; sys.path.insert(0, %r); import fastecc_b200 as fe; L = fe.lib(); h = ctypes.c_void_p(); "
            "a = (ctypes.c_uint32 * 1)(0); "
            "print(L.fastecc_b200_rs_repair_pattern(12, 4, a, 1, None, 0, None, ctypes.byref(h)), "
            "L.fastecc_b200_rs_repair(None, None, 4, None, 4, 4, None))") % ROOT
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.stdout.split() == ["-4", "-4"], out.stdout + out.stderr
