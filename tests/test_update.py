"""GPU: update of a stored stripe in place (fastecc_b200_rs_update, csrc/update.cu, DESIGN 3h).  Every result is compared, bit
for bit and over whole buffers (data, parity and the new rows, sentinels in every pad word), with rs_encode_asym_mixed_dev of the
updated data.  Both paths are run on either side of the library's choice, each confirmed by its launch count: the direct path
is the delta and parity kernels (plus one table build at the first update of an N), the re-encode at least four launches.
The algebra is restated on the CPU in test_update_algebra.py, the kernels' SASS is checked in test_update_abi.py."""
import ctypes
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

P = 0xFFF00001
C = (1 << 32) - P
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0x5EED5EED
UPDATE_DIRECT, UPDATE_ROW_LANES, UPDATE_FIXED = 20, 400000, 50000000     # kUpdateDirect, kUpdateRowLanes, kUpdateFixed in csrc/api.cu
MAX_WORKSPACE = 4 << 30                                            # kMaxRepairBytes


def lanes(M, S):
    """update_parity_kernel's grid: 32-row x 32-chunk tiles of 16-byte chunks, padding included"""
    s4 = (S + 3) // 4
    return -(-M // 32) * 32 * (-(-s4 // 32) * 32)


def crossover(N, M, S):
    """the largest k of the direct path (update_direct in csrc/api.cu)"""
    s4 = (S + 3) // 4
    return min((UPDATE_DIRECT * N * s4 + UPDATE_FIXED) // (lanes(M, S) + UPDATE_ROW_LANES), MAX_WORKSPACE // (16 * s4))


def direct(N, M, k, S):
    return k <= crossover(N, M, S)


def i32(x):
    """int64 words in [0, 2^32) as the int32 tensor that stores them"""
    import torch
    return (x - (x >= 1 << 31).to(torch.int64) * (1 << 32)).to(torch.int32)


def rand_words(n, S, gen):
    import torch
    return torch.randint(0, P, (n, S), device="cuda", generator=gen, dtype=torch.int64)


def raw(x, gen):
    """canonical int64 words as stored words: x + P at random where that fits 32 bits"""
    import torch
    up = (torch.rand(x.shape, device=x.device, generator=gen) < 0.5) & (x < C)
    return i32(x + up.to(torch.int64) * P)


def encode(fecc, data, M):
    buf = data.clone()
    fecc.rs_encode_asym_mixed_dev(buf, M)
    return buf[:M].clone()


def launches(fecc, fn):
    import torch
    torch.cuda.synchronize()
    n0 = fecc.kernel_launches()
    fn()
    torch.cuda.synchronize()
    return fecc.kernel_launches() - n0


def check_path(N, M, k, S, n):
    if direct(N, M, k, S):
        assert n in (2, 3), ("direct path expected", N, M, k, n)
    else:
        assert n >= 4, ("re-encode path expected", N, M, k, n)


def update_case(fecc, N, M, S, changed, seed, dpitch=None, ppitch=None, npitch=None):
    """Data and parity as strided views of one buffer (parity first, then data), at their own pitches, sentinels in every
    pad word, raw words >= P in the stored data, parity and new rows; update; compare whole buffers."""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(seed)
    k = len(changed)
    dpitch, ppitch, npitch = dpitch or (S + 4 - S % 4), ppitch or (S + 8 - S % 4), npitch or (S + 4 - S % 4)
    data = rand_words(N, S, gen)
    parity = encode(fecc, i32(data), M).to(torch.int64) & 0xFFFFFFFF
    new = rand_words(k, S, gen)
    poff = 4
    doff = poff + M * ppitch + 12
    mem = torch.full((doff + N * dpitch + 4,), SENTINEL, dtype=torch.int32, device="cuda")
    pv = mem.as_strided((M, S), (ppitch, 1), poff)
    dv = mem.as_strided((N, S), (dpitch, 1), doff)
    stored_parity, stored_data = raw(parity, gen), raw(data, gen)
    pv.copy_(stored_parity)
    dv.copy_(stored_data)
    nbuf = torch.full((max(k, 1), npitch), SENTINEL, dtype=torch.int32, device="cuda")
    nv = nbuf[:k, :S]
    nv.copy_(raw(new, gen))
    new_data = data.clone()
    want = mem.clone()
    if k:                                       # unchanged data rows keep their raw words; the parity is rewritten canonical
        rows = torch.as_tensor(changed, device="cuda")
        new_data[rows] = new
        stored_data[rows] = i32(new)
        want.as_strided((M, S), (ppitch, 1), poff).copy_(encode(fecc, i32(new_data), M))
    want.as_strided((N, S), (dpitch, 1), doff).copy_(stored_data)
    want_new = nbuf.clone()
    n = launches(fecc, lambda: fecc.rs_update_dev(dv, pv, changed, nv))
    if k == 0:
        assert n == 0
    else:
        check_path(N, M, k, S, n)
    assert torch.equal(nbuf, want_new), "the new rows were written"
    if not torch.equal(mem, want):
        bad = (mem != want).nonzero().flatten()
        pytest.fail("N=%d M=%d S=%d k=%d: %d words differ, first at flat word %d (parity from %d, data from %d)"
                    % (N, M, S, k, bad.numel(), int(bad[0]), poff, doff))
    return n


SMALL = [1, 2, 3, 4, 6, 8, 9, 12, 18, 32, 36, 96, 288, 1024, 3 * 1024, 9 * 1024]


def sample_divisors(N):
    Ms = [m for m in range(1, N + 1) if N % m == 0]
    if len(Ms) <= 8:
        return Ms
    return sorted({m for m in (1, 2, 3, 4, 9, 64, N // 1024, N // 64, N // 9, N // 8, N // 3, N // 2, N) if m >= 1 and N % m == 0})


@pytest.mark.gpu
@pytest.mark.parametrize("N,S", [(N, S) for N in SMALL for S in (5, 8)])
def test_small_stripes_on_both_paths(fecc, N, S):
    rng = np.random.default_rng(31 * N + S)
    for M in sample_divisors(N):
        kc = crossover(N, M, S)
        for k in sorted({0, 1, 2, kc - 1, kc, kc + 1, N} & set(range(0, N + 1))):
            changed = sorted(rng.choice(N, size=k, replace=False).tolist())
            update_case(fecc, N, M, S, changed, int(rng.integers(1 << 30)))


@pytest.mark.gpu
@pytest.mark.parametrize("S", [5, 6, 7, 13])
def test_layouts_and_partial_groups(fecc, S):
    """SIZE % 4 in {1, 2, 3}, three different pitches with room to spare, on both paths"""
    N, M = 3 << 8, 3 << 5
    rng = np.random.default_rng(S)
    for k in (1, crossover(N, M, S), crossover(N, M, S) + 1, N):
        changed = sorted(rng.choice(N, size=min(k, N), replace=False).tolist())
        update_case(fecc, N, M, S, changed, 40 + k, dpitch=S + 12 - S % 4, ppitch=S + 4 - S % 4, npitch=S + 20 - S % 4)


def big_case(fecc, N, M, S, ks, seed):
    """library encode -> update of k random blocks -> equal to the encode of the updated data, bit for bit"""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(seed)
    rng = np.random.default_rng(seed)
    data = i32(rand_words(N, S, gen))
    parity = encode(fecc, data, M)
    for k in ks:
        changed = sorted(rng.choice(N, size=k, replace=False).tolist())
        new = i32(rand_words(k, S, gen))
        want_data = data.clone()
        want_data[torch.as_tensor(changed, device="cuda")] = new
        want_parity = encode(fecc, want_data, M)
        n = launches(fecc, lambda: fecc.rs_update_dev(data, parity, changed, new))
        check_path(N, M, k, S, n)
        assert torch.equal(data, want_data), (N, M, k)
        assert torch.equal(parity, want_parity), (N, M, k, int((parity != want_parity).sum()))
        del want_data, want_parity
    del data, parity
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("M_div", [1, 16])
def test_full_size_2p19_4k_blocks(fecc, M_div):
    N = 1 << 19
    kc = crossover(N, N // M_div, 1024)
    big_case(fecc, N, N // M_div, 1024, [1, max(kc, 1), kc + 1], 5 + M_div)


@pytest.mark.gpu
@pytest.mark.parametrize("M,S", [(1, 1024), (16, 1024), (256, 1024), (1, 16), (256, 16), (1 << 10, 16)])
def test_few_parity_rows_and_short_rows_on_both_paths(fecc, M, S):
    """Parity grids too small to fill the GPU and rows shorter than a 32-chunk tile: the switch follows the padded lanes and the
    per-row term of the rule, not k * M alone; both sides of it."""
    N = 1 << 14
    kc = crossover(N, M, S)
    big_case(fecc, N, M, S, sorted({1, max(kc, 1), kc + 1} & set(range(1, N + 1))), M + S)


@pytest.mark.gpu
def test_full_size_9x2p19(fecc):
    N = 9 << 19
    kc = crossover(N, N // 9, 16)
    big_case(fecc, N, N // 9, 16, [1, max(kc, 1), kc + 1], 99)


@pytest.mark.gpu
def test_reencode_in_three_column_chunks(fecc):
    """9 * 2^18 blocks, M = N, SIZE 502 in a 504-word pitch: the re-encode runs in chunks of 224 + 224 + 54 words, the last one
    ending in a partial 16-byte group; the pad words keep their sentinel."""
    import torch
    torch.cuda.empty_cache()
    if torch.cuda.mem_get_info()[0] < (30 << 30):
        pytest.skip("needs 30 GiB of free device memory")
    N, S, pitch = 9 << 18, 502, 504
    gen = torch.Generator(device="cuda"); gen.manual_seed(7)
    rng = np.random.default_rng(7)
    data = torch.full((N, pitch), SENTINEL, dtype=torch.int32, device="cuda")
    data[:, :S] = i32(rand_words(N, S, gen))
    buf = data.clone()
    fecc.rs_encode_asym_mixed_dev(buf[:, :S], N)
    parity = buf
    parity[:, S:] = SENTINEL
    k = 3 * crossover(N, N, S)
    changed = sorted(rng.choice(N, size=k, replace=False).tolist())
    new = torch.full((k, pitch), SENTINEL, dtype=torch.int32, device="cuda")
    new[:, :S] = i32(rand_words(k, S, gen))
    want_data = data.clone()
    want_data[torch.as_tensor(changed, device="cuda"), :S] = new[:, :S]
    n = launches(fecc, lambda: fecc.rs_update_dev(data[:, :S], parity[:, :S], changed, new[:, :S]))
    check_path(N, N, k, S, n)
    assert torch.equal(data, want_data)
    del data
    torch.cuda.empty_cache()
    want_parity = want_data
    fecc.rs_encode_asym_mixed_dev(want_parity[:, :S], N)
    assert torch.equal(parity, want_parity)
    del parity, want_parity, want_data, buf
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("N,M", [(3 << 12, 1 << 12), (1 << 13, 1 << 13), (9 << 10, 1 << 10)])
def test_update_then_lose_then_repair(fecc, N, M):
    """After an update, losing up to M blocks (updated ones among them) and repairing brings the new data back."""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(N + M)
    rng = np.random.default_rng(N + M)
    S = 64
    data = i32(rand_words(N, S, gen))
    parity = encode(fecc, data, M)
    for k in (1, crossover(N, M, S) + 1):
        changed = sorted(rng.choice(N, size=min(k, N), replace=False).tolist())
        new = i32(rand_words(len(changed), S, gen))
        fecc.rs_update_dev(data, parity, changed, new)
        want_d, want_p = data.clone(), parity.clone()
        nd = min(M // 2, len(changed))
        lost_d = sorted(set(changed[:nd]) | set(rng.choice(N, size=M // 2 - nd, replace=False).tolist()) if M > 1 else changed[:1])
        lost_d = lost_d[:M]
        lost_p = sorted(rng.choice(M, size=M - len(lost_d), replace=False).tolist())
        data[torch.as_tensor(lost_d, device="cuda")] = -3
        if lost_p:
            parity[torch.as_tensor(lost_p, device="cuda")] = 11
        fecc.rs_repair_dev(data, parity, lost_d, lost_p)
        torch.cuda.synchronize()
        assert torch.equal(data, want_d) and torch.equal(parity, want_p), (N, M, k)


@pytest.mark.gpu
def test_update_repair_and_encode_on_three_streams_from_two_threads(fecc):
    """Thread 1 updates a stripe of an order no update has used yet (its table is built on that stream) and then runs a mixed
    encode on a second stream; thread 2 repairs a stripe on a third stream at the same time.  No host sync between them."""
    import torch
    from fastecc_b200 import decoder
    gen = torch.Generator(device="cuda"); gen.manual_seed(5)
    rng = np.random.default_rng(5)
    N1, M1, S = 3 << 15, 3 << 11, 64
    d1 = i32(rand_words(N1, S, gen)); p1 = encode(fecc, d1, M1)
    ks = [1, crossover(N1, M1, S) + 7]
    jobs = []
    for k in ks:
        changed = sorted(rng.choice(N1, size=k, replace=False).tolist())
        new = i32(rand_words(k, S, gen))
        jobs.append((changed, new))
    want_d1 = d1.clone()
    for changed, new in jobs:
        want_d1[torch.as_tensor(changed, device="cuda")] = new
    want_p1 = encode(fecc, want_d1, M1)
    N3 = 9 << 13
    x3 = i32(rand_words(N3, S, gen))
    want_x3 = x3.clone(); fecc.rs_encode_mixed_dev(want_x3)
    N2, M2 = 1 << 15, 1 << 11
    d2 = i32(rand_words(N2, S, gen)); p2 = encode(fecc, d2, M2)
    lost_d = sorted(rng.choice(N2, size=M2 // 2, replace=False).tolist())
    lost_p = sorted(rng.choice(M2, size=M2 - M2 // 2, replace=False).tolist())
    want_d2, want_p2 = d2.clone(), p2.clone()
    d2[torch.as_tensor(lost_d, device="cuda")] = 1
    p2[torch.as_tensor(lost_p, device="cuda")] = 2
    rep = decoder.Repair(N2, M2, lost_d, lost_p)
    torch.cuda.synchronize()
    errors, streams = [], [torch.cuda.Stream() for _ in range(3)]

    def thread1():
        try:
            with torch.cuda.stream(streams[0]):
                for changed, new in jobs:
                    fecc.rs_update_dev(d1, p1, changed, new)
            with torch.cuda.stream(streams[2]):
                fecc.rs_encode_mixed_dev(x3)
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
    assert torch.equal(d1, want_d1) and torch.equal(p1, want_p1)
    assert torch.equal(d2, want_d2) and torch.equal(p2, want_p2)
    assert torch.equal(x3, want_x3)


@pytest.mark.gpu
def test_update_does_not_synchronise_the_stream(fecc):
    """With the workspace already large enough, the call returns while a kernel ahead of it on the stream is still running, and
    the host list may be overwritten right after the call."""
    import torch
    N, M, S = 1 << 12, 1 << 8, 64
    gen = torch.Generator(device="cuda"); gen.manual_seed(9)
    data = i32(rand_words(N, S, gen)); parity = encode(fecc, data, M)
    for k in (3, crossover(N, M, S) + 1):
        changed = np.arange(0, 2 * k, 2, dtype=np.int64)
        new = i32(rand_words(k, S, gen))
        fecc.rs_update_dev(data, parity, changed, new)           # warm: workspace, table, page-locked list
        want_d = data.clone(); want_d[torch.as_tensor(changed, device="cuda")] = new
        want_p = encode(fecc, want_d, M)
        torch.cuda.synchronize()
        torch.cuda._sleep(1 << 30)
        fecc.rs_update_dev(data, parity, changed, new)
        busy = not torch.cuda.current_stream().query()
        changed[:] = 1                                          # the caller reuses its list
        torch.cuda.synchronize()
        assert busy, "the update waited for the stream"
        assert torch.equal(data, want_d) and torch.equal(parity, want_p), k


@pytest.mark.gpu
def test_update_argument_table(fecc):
    """Every rule of the validation broken on its own gives FASTECC_B200_EINVAL (-1) and launches nothing; the valid calls give 0."""
    import torch
    L = fecc.lib()
    st = torch.cuda.current_stream().cuda_stream
    buf = torch.zeros((64, 8), dtype=torch.int32, device="cuda")
    d, p, nw = buf[:12].data_ptr(), buf[32:36].data_ptr(), buf[48:50].data_ptr()
    two = np.array([1, 5], dtype=np.uint32)
    wrong = []

    def call(data=d, dpitch=8, N=12, parity=p, ppitch=8, M=4, changed=two, k=None, new=nw, npitch=8, S=8):
        arr = None if changed is None else np.asarray(changed, dtype=np.uint32)
        k = (0 if arr is None else arr.size) if k is None else k
        return L.fastecc_b200_rs_update(data, dpitch, N, parity, ppitch, M, None if arr is None or not arr.size else arr.ctypes.data, k, new, npitch, S, st)

    cases = [({}, 0), (dict(S=5), 0), (dict(M=12, parity=buf[16:28].data_ptr()), 0), (dict(M=1), 0),
             (dict(N=5), -1), (dict(N=27), -1), (dict(N=3 << 20, M=3), -1), (dict(M=0), -1), (dict(M=5), -1), (dict(M=24), -1),
             (dict(S=0), -1), (dict(data=None), -1), (dict(parity=None), -1), (dict(new=None), -1), (dict(changed=None, k=2), -1),
             (dict(dpitch=6, S=6), -1), (dict(ppitch=6, S=6), -1), (dict(npitch=6, S=6), -1), (dict(dpitch=4), -1), (dict(ppitch=4), -1), (dict(npitch=4), -1),
             (dict(data=d + 4, S=4), -1), (dict(parity=p + 8, S=4), -1), (dict(new=nw + 4, S=4), -1),
             (dict(changed=[5, 1]), -1), (dict(changed=[2, 2]), -1), (dict(changed=[3, 12]), -1),
             (dict(parity=d + 8 * 11 * 4), -1), (dict(data=p - 64, parity=p), -1), (dict(new=d + 8 * 4), -1), (dict(new=p + 8 * 3 * 4), -1),
             (dict(new=p - 8 * 4), -1)]
    for kw, want in cases:
        n0 = fecc.kernel_launches()
        rc = call(**kw)
        if rc != want or (want and fecc.kernel_launches() != n0):
            wrong.append((kw, rc))
    for kw in (dict(changed=[]), dict(changed=None, new=None)):                    # nothing changed: 0, no launch
        n0 = fecc.kernel_launches()
        if call(**kw) != 0 or fecc.kernel_launches() != n0:
            wrong.append(("n_changed = 0", kw))
    torch.cuda.synchronize()
    assert not wrong, wrong


@pytest.mark.gpu
def test_update_before_init_is_enoinit():
    """In a fresh process that never called fastecc_b200_init, the update fails with FASTECC_B200_ENOINIT (-4)."""
    code = ("import sys; sys.path.insert(0, %r); import fastecc_b200 as fe; L = fe.lib(); "
            "print(L.fastecc_b200_rs_update(None, 4, 12, None, 4, 4, None, 0, None, 4, 4, None))") % ROOT
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.stdout.split() == ["-4"], out.stdout + out.stderr
