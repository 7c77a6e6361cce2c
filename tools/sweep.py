#!/usr/bin/env python
"""Device-resident timing sweep over the BASELINE parity configs (SURVEY 8d: configs 1, 3 and the NTT sweep 5):
encode at N = 2^7 .. 2^19 and forward NTT at N = 2^10 .. 2^20, 4096-byte blocks, CUDA events around `reps` back-to-back
calls.  Arrays below ~100 MB stay in the 126 MB L2 between calls (marked); the small orders are launch-latency bound.
Then recoding, decoding, the asymmetric encode, the encode of 3 * 2^k / 9 * 2^k blocks (`encode_mixed`, DESIGN 3e) and
their encode into fewer parity blocks (`encode_asym_mixed`, DESIGN 3f; `--asym-mixed`: only these).  `--repair`: only the repair
of a stored stripe against the 2N-row decoder (DESIGN 3g); `--update`, `--scrub`, `--scrub-degraded`, `--reconstruct`: only the update (3h),
the scrub (3i), the degraded scrub (3j) or the degraded read (3k) lines; `--batch`: only the batch encode of small stripes (3l);
`--reconstruct-batch`: only the degraded read of a batch of small stripes (3m); `--update-batch`: only the update of a batch of
small stripes in place (3n).
Prints one JSON line per point."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

import fastecc_b200 as fe

P = 0xFFF00001


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    fe.init(0)
    S = 1024
    if "--asym-mixed" in sys.argv:                            # only the encode_asym_mixed lines
        asym_mixed_encode(S)
        return 0
    only_extras = "--extras" in sys.argv
    for op, Ls in (() if only_extras else (("encode", range(7, 20)), ("ntt", range(10, 21)))):
        for L in Ls:
            N = 1 << L
            x = (torch.arange(N * S, device="cuda", dtype=torch.int64) % P).to(torch.int32).view(N, S)
            reps = max(5, min(200, int(2e9 // (N * S * 4))))
            ms = timed((lambda: fe.rs_encode_dev(x)) if op == "encode" else (lambda: fe.ntt_dev(x, False)), reps)
            nbytes = N * S * 4
            print(json.dumps({"op": op, "log_n": L, "block_bytes": 4096, "array_MiB": nbytes / 2**20, "ms": round(ms, 5), "reps": reps,
                              "GBps_read_plus_write": round(2 * nbytes / ms / 1e6, 1),
                              "MiBps_reference_convention": round((2 if op == "encode" else 1) * nbytes / 2**20 / ms * 1e3),
                              "l2_resident": nbytes < 100e6}), flush=True)
            del x
            torch.cuda.empty_cache()
    n, W = 1 << 19, 1024                                      # byte <-> GF(p) recoding, 2 GiB of random bytes (22 % of the blocks need recoding)
    raw = torch.randint(0, 256, (n, 4 * W), dtype=torch.uint8, device="cuda")
    words = torch.zeros((n, W + 4), dtype=torch.int32, device="cuda")
    ms = timed(lambda: fe.bytes_to_gfp_dev(raw, words), 10)
    print(json.dumps({"op": "bytes_to_gfp", "blocks": n, "block_bytes": 4 * W, "ms": round(ms, 5), "GBps_read_plus_write": round((n * 4 * W + n * 4 * (W + 1)) / ms / 1e6, 1)}), flush=True)
    back = torch.empty_like(raw)
    ms = timed(lambda: fe._check(fe.lib().fastecc_b200_gfp_to_bytes_dev(words.data_ptr(), back.data_ptr(), n, W, W + 4, torch.cuda.current_stream().cuda_stream)), 10)
    print(json.dumps({"op": "gfp_to_bytes", "blocks": n, "block_bytes": 4 * W, "ms": round(ms, 5), "GBps_read_plus_write": round((n * 4 * W + n * 4 * (W + 1)) / ms / 1e6, 1),
                      "roundtrip_ok": bool((back == raw).all())}), flush=True)
    del raw, words, back
    torch.cuda.empty_cache()
    from fastecc_b200 import decoder                          # erasure decoding at the headline order: 2^19 data + 2^19 parity blocks of 4 KiB
    N2 = 1 << 20
    code = (torch.arange(N2 * S, device="cuda", dtype=torch.int64) % P).to(torch.int32).view(N2, S)
    g = torch.Generator(device="cuda"); g.manual_seed(1)
    erased = torch.sort(torch.randperm(N2, device="cuda", generator=g)[:N2 // 2]).values.cpu().tolist()
    torch.cuda.synchronize()
    import time
    t0 = time.perf_counter()
    pat = decoder.ErasurePattern(N2, erased, code.device)
    torch.cuda.synchronize()
    t_pat = (time.perf_counter() - t0) * 1e3
    ms = timed(lambda: pat.recover(code), 3)                 # (timing only: the workspace is not a code word after the first call)
    print(json.dumps({"op": "decode", "log_n": 19, "erased": N2 // 2, "block_bytes": 4096, "pattern_setup_ms_wall": round(t_pat, 1), "recover_ms": round(ms, 4),
                      "GBps_codeword_bytes": round(N2 * S * 4 / ms / 1e6, 1)}), flush=True)
    del code, pat
    torch.cuda.empty_cache()
    N = 1 << 19
    for K in (1, 2, 3, 6):
        x = (torch.arange(N * S, device="cuda", dtype=torch.int64) % P).to(torch.int32).view(N, S)
        ms = timed(lambda: fe.rs_encode_asym_dev(x, N >> K), 5)
        print(json.dumps({"op": "encode_asym", "log_n": 19, "log_m": 19 - K, "block_bytes": 4096, "ms": round(ms, 5),
                          "GBps_data_plus_parity": round((N + (N >> K)) * S * 4 / ms / 1e6, 1)}), flush=True)
        del x
        torch.cuda.empty_cache()
    mixed_encode(S)
    asym_mixed_encode(S)
    return 0


def rho_powers_over_n(N):
    """rho^m / N for m < N, rho = GF_Root(2N) (the scaling of RS.cpp:51-59 at this order), as an int32 device tensor"""
    rho, inv, B = pow(19, (P - 1) // (2 * N), P), pow(N, P - 2, P), 4096
    lo, v = np.empty(B, dtype=np.uint64), inv
    for i in range(B):
        lo[i] = v; v = v * rho % P
    nb, step = (N + B - 1) // B, pow(rho, B, P)
    hi, v = np.empty(nb, dtype=np.uint64), 1
    for i in range(nb):
        hi[i] = v; v = v * step % P
    c = ((hi[:, None] * lo[None, :]) % np.uint64(P)).ravel()[:N].astype(np.uint32)
    return torch.from_numpy(c.view(np.int32)).cuda()


def mixed_encode(S):
    """Encode of N = 3 * 2^k / 9 * 2^k blocks (fastecc_b200_rs_encode_mixed_dev, 5 passes over the array) against the same
    encode composed from existing entry points (inverse mixed NTT, row scaling by rho^m / N, forward mixed NTT: 9 passes) on
    the same array, the power-of-two encode at the next power of two where one exists, and radix_encode_kernel alone
    (torch.profiler, in a profiled loop of its own after the timed ones)."""
    lib, stream = fe.lib(), torch.cuda.current_stream().cuda_stream
    for N in (3 << 16, 9 << 15, 3 << 17, 9 << 16, 3 << 18, 9 << 17, 3 << 19, 9 << 18):
        x = (torch.arange(N * S, device="cuda", dtype=torch.int64) % P).to(torch.int32).view(N, S)
        consts = rho_powers_over_n(N)
        reps = max(5, min(50, int(4e9 // (N * S * 4))))

        def composed():
            fe.ntt_dev(x, True)
            fe._check(lib.fastecc_b200_row_scale_dev(x.data_ptr(), N, S, S, consts.data_ptr(), stream))
            fe.ntt_dev(x, False)
        ms_mixed = timed(lambda: fe.rs_encode_mixed_dev(x), reps)
        ms_composed = timed(composed, reps)
        ms_mixed_again = timed(lambda: fe.rs_encode_mixed_dev(x), reps)       # alternated: the spread of the first figure
        N2 = 1 << (N - 1).bit_length()
        ms_pow2 = None
        if N2 <= 1 << 19:
            y = (torch.arange(N2 * S, device="cuda", dtype=torch.int64) % P).to(torch.int32).view(N2, S)
            ms_pow2 = round(timed(lambda: fe.rs_encode_dev(y), reps), 5)
            del y
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fe.rs_encode_mixed_dev(x)
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if "radix_encode_kernel" in e.key]
        us = sum(getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0) for e in ev)
        n = sum(e.count for e in ev)
        nbytes = N * S * 4
        print(json.dumps({"op": "encode_mixed", "N": N, "r": 3 if N % 9 else 9, "block_bytes": 4 * S, "array_MiB": nbytes / 2**20, "reps": reps,
                          "ms": round(min(ms_mixed, ms_mixed_again), 5), "ms_runs": [round(ms_mixed, 5), round(ms_mixed_again, 5)],
                          "ms_composed_9_pass": round(ms_composed, 5), "next_pow2": N2, "ms_pow2_encode_next_pow2": ms_pow2,
                          "ms_radix_encode_kernel": round(us / 1e3 / n, 5) if n else None,
                          "GBps_kernel_read_plus_write": round(2 * nbytes / (us / n) / 1e3, 1) if n else None,
                          "MiBps_reference_convention": round(2 * nbytes / 2**20 / min(ms_mixed, ms_mixed_again) * 1e3)}), flush=True)
        del x, consts
        torch.cuda.empty_cache()


def asym_mixed_encode(S):
    """N = 3 * 2^k / 9 * 2^k data blocks into M = N/2, N/r, N/8, N/64 parity blocks (fastecc_b200_rs_encode_asym_mixed_dev,
    DESIGN 3f) against the full encode of the same array (rs_encode_mixed_dev), timed alternately, twice each; the lower
    figures.  Every line carries the card's name and power limit, read in the same run."""
    from bench import gpu_identity
    card = gpu_identity(torch.cuda.current_device())
    for N in (3 << 16, 9 << 15, 3 << 17, 9 << 16, 3 << 18, 9 << 17, 3 << 19, 9 << 18):
        r = 3 if N % 9 else 9
        x = (torch.arange(N * S, device="cuda", dtype=torch.int64) % P).to(torch.int32).view(N, S)
        reps = max(5, min(50, int(4e9 // (N * S * 4))))
        for M in (N // 2, N // r, N // 8, N // 64):
            runs_asym, runs_full = [], []
            for _ in range(2):
                runs_full.append(timed(lambda: fe.rs_encode_mixed_dev(x), reps))
                runs_asym.append(timed(lambda: fe.rs_encode_asym_mixed_dev(x, M), reps))
            ms, ms_full = min(runs_asym), min(runs_full)
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:               # a profiled loop of its own, after the timed ones
                for _ in range(reps):
                    fe.rs_encode_asym_mixed_dev(x, M)
                torch.cuda.synchronize()
            dev_ms = {}
            for e in prof.key_averages():
                us = getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
                if us:
                    k = "radix_fold_kernel" if "radix_fold_kernel" in e.key else "memcpy" if "emcpy" in e.key else "transforms"
                    dev_ms[k] = dev_ms.get(k, 0) + us / 1e3 / reps
            print(json.dumps({"op": "encode_asym_mixed", "N": N, "M": M, "r": r, "block_bytes": 4 * S, "reps": reps,
                              "ms": round(ms, 5), "ms_runs": [round(v, 5) for v in runs_asym],
                              "ms_full_mixed_encode": round(ms_full, 5), "ms_full_runs": [round(v, 5) for v in runs_full],
                              "ratio": round(ms / ms_full, 3), "profiled_ms": {k: round(v, 4) for k, v in sorted(dev_ms.items())},
                              "gpu": card["name"], "power_limit_w": card["power_limit_w"]}), flush=True)
        del x
        torch.cuda.empty_cache()


def repair_sweep(S):
    """Repair of a stored stripe in place (fastecc_b200_rs_repair, DESIGN 3g) with M and M/8 blocks lost, half of them data, half
    parity, against the same losses through the 2N-row decoder: assemble the code word (data in the even rows, parity in every
    2(N/M)-th odd row), asym_erasures + CErasurePattern(mixed=True), recover.  Pattern builds are wall-clock times; the repair
    and the recover are CUDA-event times, two runs each, alternated (the lower figures).  Each line names the card and its
    power limit, read in the same run."""
    import time
    from bench import gpu_identity
    from fastecc_b200 import decoder
    card = gpu_identity(torch.cuda.current_device())
    rng = np.random.default_rng(1)
    points = [(1 << 19, m) for m in (1 << 19, 1 << 18, 1 << 15, 1 << 13)] + [(3 << 19, 1 << 19), (9 << 18, 1 << 18)]
    for N, M in points:
        data = (torch.arange(N * S, device="cuda", dtype=torch.int64) % P).to(torch.int32).view(N, S)
        torch.cuda.empty_cache()                              # so that no block below lands in (and pins) a cached int64 temporary
        buf = data.clone()
        fe.rs_encode_asym_mixed_dev(buf, M)
        parity = torch.empty((M, S), dtype=torch.int32, device="cuda")
        parity.copy_(buf[:M])
        del buf
        torch.cuda.empty_cache()
        for lost in (M, M // 8):
            lost_d = sorted(rng.choice(N, size=lost // 2, replace=False).tolist())
            lost_p = sorted(rng.choice(M, size=lost - lost // 2, replace=False).tolist())
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rep = decoder.Repair(N, M, lost_d, lost_p)
            t_pat = (time.perf_counter() - t0) * 1e3
            torch.cuda.empty_cache()                          # the 2N-row code word of 9 * 2^18 blocks takes 18 GiB in one piece
            line = {"op": "repair", "N": N, "M": M, "lost_data": len(lost_d), "lost_parity": len(lost_p), "block_bytes": 4 * S,
                    "pattern_ms_wall": round(t_pat, 1), "gpu": card["name"], "power_limit_w": card["power_limit_w"]}
            code = old = None
            try:
                t0 = time.perf_counter()
                code = torch.zeros((2 * N, S), dtype=torch.int32, device="cuda")
                code[0::2] = data
                code[1::2 * (N // M)] = parity
                torch.cuda.synchronize()
                line["old_assemble_ms_wall"] = round((time.perf_counter() - t0) * 1e3, 1)
                t0 = time.perf_counter()
                old = decoder.CErasurePattern(2 * N, decoder.asym_erasures(N, M, lost_d, lost_p), mixed=True)
                torch.cuda.synchronize()
                line["old_pattern_ms_wall"] = round((time.perf_counter() - t0) * 1e3, 1)
            except (torch.OutOfMemoryError, fe.FastEccError) as e:          # the 2N-row route needs about twice the memory
                line["old_route"] = "out of device memory: %s" % str(e).splitlines()[0][:120]
                code = old = None
                torch.cuda.empty_cache()
            runs, runs_old = [], []
            for _ in range(2):
                runs.append(timed(lambda: rep.repair(data, parity), 5))
                if old is not None:
                    runs_old.append(timed(lambda: old.recover(code), 3))  # (timing only: the workspace is not a code word after the first call)
            rep.close()
            if old is not None:
                old.close()
                line.update(old_recover_ms=round(min(runs_old), 4), old_recover_runs=[round(v, 4) for v in runs_old])
            line.update(ms=round(min(runs), 4), ms_runs=[round(v, 4) for v in runs])
            print(json.dumps(line), flush=True)
            del code, old, rep
            torch.cuda.empty_cache()
        del data, parity
        torch.cuda.empty_cache()


def update_sweep():
    """Update of k data blocks of a stored stripe (fastecc_b200_rs_update, DESIGN 3h) on each of its two paths.  The library picks
    the path itself, so builds of it that differ only in -DFECC_UPDATE_PATH=1 (always direct) and =2 (always re-encode), and a
    third that is always direct with the quotient of its products on the FP64 unit (-DFECC_UPDATE_MUL_H, gf::mul_h), are compiled
    into a temporary directory and loaded side by side.  CUDA events around `reps` back-to-back calls, the builds alternated twice
    (the lower figures); at k = 1 also an in-place torch op over the same parity tensor (parity.add_(1), one read and one write of
    the same bytes).  k runs over powers of 4 and 100 (a count whose index list is not a multiple of 64 words) until the direct
    path takes more than twice the re-encode.  Each line names the card and its power limit, read in the same run."""
    import ctypes
    import shutil
    import subprocess
    import tempfile
    from bench import gpu_identity
    from fastecc_b200 import build as b
    card = gpu_identity(torch.cuda.current_device())
    tmp = tempfile.mkdtemp(prefix="fastecc_update_")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    builds = []
    for name, flags in (("direct", ["-DFECC_UPDATE_PATH=1"]), ("reencode", ["-DFECC_UPDATE_PATH=2"]), ("direct_mul_h", ["-DFECC_UPDATE_PATH=1", "-DFECC_UPDATE_MUL_H"])):
        out = os.path.join(tmp, "libfastecc_b200_%s.so" % name)
        cmd = [nvcc] + b.NVCC_FLAGS + flags + ["-o", out] + [os.path.join(b.CSRC, s) for s in b.SOURCES]
        builds.append((name, subprocess.Popen(cmd), out))
    libs = {}
    for name, proc, out in builds:
        if proc.wait() != 0:
            raise RuntimeError("nvcc failed building %s" % out)
        L = ctypes.CDLL(out)
        sz, vp = ctypes.c_size_t, ctypes.c_void_p
        L.fastecc_b200_rs_update.argtypes = [vp, sz, sz, vp, sz, sz, vp, sz, vp, sz, sz, vp]
        L.fastecc_b200_rs_encode_asym_mixed_dev.argtypes = [vp, sz, sz, sz, sz, vp]
        L.fastecc_b200_last_error.restype = ctypes.c_char_p
        if L.fastecc_b200_init(0):
            raise RuntimeError(L.fastecc_b200_last_error().decode())
        libs[name] = L

    def call(L, rc):
        if rc:
            raise RuntimeError(L.fastecc_b200_last_error().decode())

    rng = np.random.default_rng(1)
    points = [(1 << 19, m, 1024) for m in (1 << 19, 1 << 18, 1 << 15, 1 << 13, 1 << 11, 1 << 8, 1 << 4, 1)]
    points += [(3 << 19, 1 << 19, 1024), (9 << 18, 1 << 18, 1024), (1 << 19, 1 << 15, 16)]
    for N, M, S in points:
        stream = torch.cuda.current_stream().cuda_stream
        data = (torch.arange(N * S, device="cuda", dtype=torch.int64) % P).to(torch.int32).view(N, S)
        buf = data.clone()
        call(libs["reencode"], libs["reencode"].fastecc_b200_rs_encode_asym_mixed_dev(buf.data_ptr(), N, M, S, S, stream))
        parity = buf[:M].clone()
        del buf
        torch.cuda.empty_cache()
        ks = sorted({4 ** i for i in range(12) if 4 ** i <= N} | ({100} if N >= 100 else set()))
        for k in ks:
            changed = np.sort(rng.choice(N, size=k, replace=False)).astype(np.uint32)
            new = torch.randint(0, P, (k, S), device="cuda", dtype=torch.int64).to(torch.int32)
            reps = 5

            def run(L):
                return lambda: call(L, L.fastecc_b200_rs_update(data.data_ptr(), S, N, parity.data_ptr(), S, M, changed.ctypes.data, k,
                                                                 new.data_ptr(), S, S, stream))
            runs = {name: [] for name in libs}
            for _ in range(2):
                for name, L in libs.items():
                    runs[name].append(timed(run(L), reps))
            line = {"op": "update", "N": N, "M": M, "k": k, "block_bytes": 4 * S, "reps": reps}
            for name in libs:
                line[name + "_ms"] = round(min(runs[name]), 4)
                line[name + "_runs"] = [round(v, 4) for v in runs[name]]
            line.update(faster="direct" if min(runs["direct"]) < min(runs["reencode"]) else "reencode", gpu=card["name"], power_limit_w=card["power_limit_w"])
            if k == 1:                                        # (the parity is stale afterwards; no timing depends on its content)
                line["torch_add_on_parity_ms"] = round(timed(lambda: parity.add_(1), 10), 4)
            print(json.dumps(line), flush=True)
            del new
            if min(runs["direct"]) > 2 * min(runs["reencode"]):
                break
        del data, parity
        torch.cuda.empty_cache()
    for L in libs.values():
        L.fastecc_b200_shutdown()
    shutil.rmtree(tmp, ignore_errors=True)


def scrub_sweep():
    """Scrub of a stored stripe (fastecc_b200_rs_scrub, DESIGN 3i), shipped build against one whose fold takes the products'
    quotient on the FP64 unit (-DFECC_SCRUB_MUL_H, gf::mul_h), compiled into a temporary directory and loaded side by side.  The
    whole call: CUDA events around `reps` back-to-back calls (each synchronises the stream itself).  The fold kernel alone: its
    device time in a torch.profiler trace of the same calls.  The two builds alternated twice (the lower figures).  For the fold,
    the fraction of its memory floor ((N + M) * SIZE * 4 bytes at the data sheet's 3.35 TB/s) and of update's measured product
    rate (2 (N + M) SIZE products at 1.7e12 per second, DESIGN 3h).  Beside it, today's detect-only route: copy the data into a
    preallocated buffer, rs_encode_asym_mixed_dev, torch.equal against the parity.  t corrupted blocks, half data and half
    parity, max_bad = min(M / 2, 4096); the host's Berlekamp-Massey time is scrub - (its time at t = 0) roughly.  Each line
    names the card and its power limit, read in the same run."""
    import ctypes
    import shutil
    import subprocess
    import tempfile
    from torch.profiler import ProfilerActivity, profile
    from bench import gpu_identity
    from fastecc_b200 import build as b
    fe.init(0)
    card = gpu_identity(torch.cuda.current_device())
    tmp = tempfile.mkdtemp(prefix="fastecc_scrub_")
    out = os.path.join(tmp, "libfastecc_b200_mul_h.so")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.run([nvcc] + b.NVCC_FLAGS + ["-DFECC_SCRUB_MUL_H", "-o", out] + [os.path.join(b.CSRC, src) for src in b.SOURCES], check=True)
    libs = {"mul": fe.lib(), "mul_h": ctypes.CDLL(out)}
    sz, vp = ctypes.c_size_t, ctypes.c_void_p
    for L in libs.values():
        L.fastecc_b200_rs_scrub.argtypes = [vp, sz, sz, vp, sz, sz, sz, sz, ctypes.c_uint64, vp, vp, vp, vp, vp, vp]
        L.fastecc_b200_last_error.restype = ctypes.c_char_p
    if libs["mul_h"].fastecc_b200_init(0):
        raise RuntimeError(libs["mul_h"].fastecc_b200_last_error().decode())

    def scrub(L, data, parity, max_bad):
        cap = max(max_bad, 1)
        bd, bp = np.zeros(cap, dtype=np.uint32), np.zeros(cap, dtype=np.uint32)
        st, nd, npar = ctypes.c_int(), ctypes.c_size_t(), ctypes.c_size_t()
        rc = L.fastecc_b200_rs_scrub(data.data_ptr(), data.stride(0), data.shape[0], parity.data_ptr(), parity.stride(0), parity.shape[0], data.shape[1],
                                     max_bad, 7, torch.cuda.current_stream().cuda_stream, ctypes.byref(st), bd.ctypes.data, ctypes.byref(nd),
                                     bp.ctypes.data, ctypes.byref(npar))
        if rc:
            raise RuntimeError(L.fastecc_b200_last_error().decode())
        return st.value

    def fold_ms(L, data, parity, max_bad, reps):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                scrub(L, data, parity, max_bad)
            torch.cuda.synchronize()
        us = [e.device_time_total for e in prof.key_averages() if "scrub_fold_kernel" in e.key]
        return us[0] / 1000 / reps if us else float("nan")

    S, reps = 1024, 5
    points = [(1 << 19, m) for m in (1 << 19, 1 << 18, 1 << 15, 1 << 13, 16, 1)] + [(3 << 19, 1 << 19), (9 << 18, 1 << 18)]
    rng = np.random.default_rng(1)
    for N, M in points:
        data = (torch.arange(N * S, device="cuda", dtype=torch.int64) * 2654435761 % P).to(torch.int32).view(N, S)
        buf = data.clone()
        fe.rs_encode_asym_mixed_dev(buf, M)
        parity = buf[:M].clone()
        torch.cuda.synchronize()
        max_bad = min(M // 2, 4096)

        def reencode():
            buf.copy_(data)
            fe.rs_encode_asym_mixed_dev(buf, M)
            return torch.equal(buf[:M], parity)
        reencode_ms = timed(reencode, 3)
        for t in sorted({0, 1, 16, max_bad} & set(range(0, max_bad + 1))):
            nd = t // 2
            bd = np.sort(rng.choice(N, size=nd, replace=False)); bp = np.sort(rng.choice(M, size=t - nd, replace=False))
            keep_d, keep_p = data[bd].clone(), parity[bp].clone()
            data[bd] ^= 1; parity[bp] ^= 2
            statuses = {name: scrub(L, data, parity, max_bad) for name, L in libs.items()}
            ms = {name: [] for name in libs}
            fold = {name: [] for name in libs}
            for _ in range(2):
                for name, L in libs.items():
                    ms[name].append(timed(lambda: scrub(L, data, parity, max_bad), reps if t < 4096 else 2))
                    fold[name].append(fold_ms(L, data, parity, max_bad, reps if t < 4096 else 2))
            rows = N + M
            mem_ms, prod_ms = rows * S * 4 / 3.35e12 * 1e3, 2 * rows * S / 1.7e12 * 1e3
            line = {"op": "scrub", "N": N, "M": M, "t": t, "max_bad": max_bad, "block_bytes": 4 * S, "status": statuses["mul"],
                    "status_mul_h": statuses["mul_h"], "fold_memory_floor_ms": round(mem_ms, 4), "fold_product_ms_at_1.7e12": round(prod_ms, 4),
                    "reencode_compare_ms": round(reencode_ms, 4), "gpu": card["name"], "power_limit_w": card["power_limit_w"]}
            for name in libs:
                f = min(fold[name])
                line.update({"scrub_ms_" + name: round(min(ms[name]), 4), "fold_ms_" + name: round(f, 4),
                             "fold_of_memory_floor_" + name: round(mem_ms / f, 3), "fold_of_product_rate_" + name: round(prod_ms / f, 3)})
            print(json.dumps(line), flush=True)
            data[bd] = keep_d; parity[bp] = keep_p
        del data, buf, parity
        torch.cuda.empty_cache()
    libs["mul_h"].fastecc_b200_shutdown()
    shutil.rmtree(tmp, ignore_errors=True)


def scrub_degraded_sweep():
    """Scrub of a degraded stripe (fastecc_b200_rs_scrub_degraded through decoder.Repair.scrub, DESIGN 3j) against the plain
    rs_scrub_dev of the same stripe with its lost rows intact, the two alternated twice in one session (the lower figures).  The
    whole call: CUDA events around `reps` back-to-back calls (each synchronises the stream itself).  The fold alone: the device
    time of degraded_fold_kernel / scrub_fold_kernel in a torch.profiler trace of the same calls.  f lost blocks (half data, half
    parity), t corrupted survivors (half data, half parity), max_bad = min((M - f) / 2, 4096) for the degraded scrub and
    min(M / 2, 4096) for the plain one; the fold's expected share of the plain fold's bytes is (N + M - f) / (N + M).  Each line
    names the card and its power limit, read in the same run."""
    from torch.profiler import ProfilerActivity, profile
    from bench import gpu_identity
    from fastecc_b200.decoder import Repair
    fe.init(0)
    card = gpu_identity(torch.cuda.current_device())

    def fold_ms(fn, kernel, reps):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
        us = [e.device_time_total for e in prof.key_averages() if kernel in e.key]
        return us[0] / 1000 / reps if us else float("nan")

    S, reps = 1024, 5
    rng = np.random.default_rng(2)
    for N, M in ((1 << 19, 1 << 19), (1 << 19, 1 << 15), (3 << 19, 1 << 19)):
        data = (torch.arange(N * S, device="cuda", dtype=torch.int64) * 2654435761 % P).to(torch.int32).view(N, S)
        buf = data.clone()
        fe.rs_encode_asym_mixed_dev(buf, M)
        parity = buf[:M].clone()
        del buf
        torch.cuda.empty_cache()
        for f in (1, 16, M // 4):
            fd = f // 2
            lost_d = np.sort(rng.choice(N, size=fd, replace=False)); lost_p = np.sort(rng.choice(M, size=f - fd, replace=False))
            rep = Repair(N, M, lost_d, lost_p)
            max_bad, plain_bad = min((M - f) // 2, 4096), min(M // 2, 4096)
            sd, sp = np.setdiff1d(np.arange(N), lost_d), np.setdiff1d(np.arange(M), lost_p)
            for t in (0, 1, 16):
                nd = t // 2
                bd = np.sort(rng.choice(sd, size=nd, replace=False)); bp = np.sort(rng.choice(sp, size=t - nd, replace=False))
                keep_d, keep_p = data[bd].clone(), parity[bp].clone()
                data[bd] ^= 1; parity[bp] ^= 2
                calls = {"degraded": (lambda: rep.scrub(data, parity, max_bad, 7), "degraded_fold_kernel"),
                         "plain": (lambda: fe.rs_scrub_dev(data, parity, plain_bad, 7), "scrub_fold_kernel")}
                status = {name: fn()[0] for name, (fn, _) in calls.items()}
                ms = {name: [] for name in calls}
                fold = {name: [] for name in calls}
                for _ in range(2):
                    for name, (fn, kernel) in calls.items():
                        ms[name].append(timed(fn, reps))
                        fold[name].append(fold_ms(fn, kernel, reps))
                line = {"op": "scrub_degraded", "N": N, "M": M, "f": f, "t": t, "max_bad": max_bad, "block_bytes": 4 * S,
                        "status": status["degraded"], "status_plain": status["plain"], "expected_fold_share": round((N + M - f) / (N + M), 4),
                        "gpu": card["name"], "power_limit_w": card["power_limit_w"]}
                for name in calls:
                    line.update({"scrub_ms_" + name: round(min(ms[name]), 4), "fold_ms_" + name: round(min(fold[name]), 4)})
                line["call_ratio"] = round(line["scrub_ms_degraded"] / line["scrub_ms_plain"], 3)
                line["fold_ratio"] = round(line["fold_ms_degraded"] / line["fold_ms_plain"], 3)
                print(json.dumps(line), flush=True)
                data[bd] = keep_d; parity[bp] = keep_p
            rep.close()
        del data, parity
        torch.cuda.empty_cache()


def reconstruct_sweep():
    """Degraded read (fastecc_b200_rs_reconstruct, DESIGN 3k) against rs_repair_dev of the same stripe and losses (its pattern
    built once, outside the timing), the two alternated twice in one session (the lower figures).  The call: CUDA events around
    `reps` back-to-back calls.  The sum kernel: its device time in a torch.profiler trace of the same calls, and that time over
    two floors: the memory floor (N * SIZE * 4 bytes at the data sheet's 3.35 TB/s) and the product floor (K * N * SIZE products at
    the 1.7e12 products/s that update_parity_kernel measured, DESIGN 3h).  a lost data blocks, all wanted; "+p": one lost parity
    block wanted as well (K = a + 1).  Each line names the card and its power limit, read in the same run."""
    from torch.profiler import ProfilerActivity, profile
    from bench import gpu_identity
    from fastecc_b200.decoder import Repair
    fe.init(0)
    card = gpu_identity(torch.cuda.current_device())

    def kernel_ms(fn, kernel, reps):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
        us = [e.device_time_total for e in prof.key_averages() if kernel in e.key]
        return sum(us) / 1000 / reps if us else float("nan")

    S, reps = 1024, 5
    rng = np.random.default_rng(3)
    for N, M in ((1 << 19, 1 << 19), (1 << 19, 1 << 15), (3 << 19, 1 << 19), (9 << 18, 1 << 18)):
        data = (torch.arange(N * S, device="cuda", dtype=torch.int64) * 2654435761 % P).to(torch.int32).view(N, S)
        buf = data.clone()
        fe.rs_encode_asym_mixed_dev(buf, M)
        parity = buf[:M].clone()
        del buf
        torch.cuda.empty_cache()
        for a in (1, 2, 4, 8, 16, 32):
            for with_p in ((False, True) if a < 32 else (False,)):
                lost_d = np.sort(rng.choice(N, size=a, replace=False))
                lost_p = np.sort(rng.choice(M, size=1, replace=False)) if with_p else np.zeros(0, dtype=np.int64)
                K = a + len(lost_p)
                want = torch.cat([data[torch.as_tensor(lost_d, device="cuda")], parity[torch.as_tensor(lost_p, device="cuda")]])
                out = fe.rs_reconstruct_dev(data, parity, lost_d, lost_p)
                ok = bool(torch.equal(out, want))
                rep = Repair(N, M, lost_d, lost_p)
                calls = {"reconstruct": lambda: fe.rs_reconstruct_dev(data, parity, lost_d, lost_p, out=out),
                         "repair": lambda: rep.repair(data, parity)}
                ms = {name: [] for name in calls}
                sum_ms = []
                for _ in range(2):
                    for name, fn in calls.items():
                        ms[name].append(timed(fn, reps))
                    sum_ms.append(kernel_ms(calls["reconstruct"], "reconstruct_sum_kernel", reps))
                rep.close()
                mem_floor = N * S * 4 / 3.35e12 * 1e3
                prod_floor = K * N * S / 1.7e12 * 1e3
                t = min(sum_ms)
                print(json.dumps({"op": "reconstruct", "N": N, "M": M, "a": a, "want_parity": int(with_p), "K": K, "block_bytes": 4 * S, "ok": ok,
                                  "call_ms": round(min(ms["reconstruct"]), 4), "sum_kernel_ms": round(t, 4),
                                  "memory_floor_frac": round(mem_floor / t, 3), "product_floor_frac_at_update_rate": round(prod_floor / t, 3),
                                  "repair_ms": round(min(ms["repair"]), 4), "speedup_vs_repair": round(min(ms["repair"]) / min(ms["reconstruct"]), 2),
                                  "gpu": card["name"], "power_limit_w": card["power_limit_w"]}), flush=True)
                del out, want
        del data, parity
        torch.cuda.empty_cache()


def batch_sweep():
    """Encode of a batch of small stripes (fastecc_b200_rs_encode_batch, DESIGN 3l) at the common storage shapes, 4 KiB blocks, B
    stripes of about 1 GiB of data in all, data and parity in separate stripe-major buffers.  The batch call: CUDA events around
    `reps` back-to-back calls.  Its floors: memory, (N + M) * B * 4096 bytes at the data sheet's 3.35 TB/s; products, M * N * B *
    1024 at the 1.7e12 products/s that update_parity_kernel measured (DESIGN 3h); the larger one binds.  Beside it, the
    per-stripe path on the first `few` stripes: clone the stripe, rs_encode_asym_mixed_dev, copy the M parity rows out; timed
    with events around the loop and scaled to B.  The two alternated twice (the lower figures).  Each line names the card and
    its power limit, read in the same run."""
    from bench import gpu_identity
    fe.init(0)
    card = gpu_identity(torch.cuda.current_device())
    S, few = 1024, 300
    for N, M in ((4, 2), (6, 3), (8, 4), (9, 3), (12, 4), (16, 4), (18, 3), (32, 8), (48, 16), (64, 16), (64, 64)):
        B = (1 << 30) // (N * S * 4)
        data = (torch.arange(B * N * S, device="cuda", dtype=torch.int64) * 2654435761 % P).to(torch.int32).view(B, N, S)
        parity = torch.empty((B, M, S), dtype=torch.int32, device="cuda")
        fe.rs_encode_batch_dev(data, parity)
        torch.cuda.synchronize()
        ok = all(torch.equal(parity[b], _encode_one(data[b], M)) for b in (0, B // 2, B - 1))
        scratch = torch.empty((N, S), dtype=torch.int32, device="cuda")
        out = torch.empty((few, M, S), dtype=torch.int32, device="cuda")

        def per_stripe():
            for b in range(few):
                scratch.copy_(data[b])
                fe.rs_encode_asym_mixed_dev(scratch, M)
                out[b].copy_(scratch[:M])
        runs, runs_per = [], []
        for _ in range(2):
            runs.append(timed(lambda: fe.rs_encode_batch_dev(data, parity), 10))
            runs_per.append(timed(per_stripe, 2) * B / few)
        ms, ms_per = min(runs), min(runs_per)
        mem_ms = (N + M) * B * S * 4 / 3.35e12 * 1e3
        prod_ms = M * N * B * S / 1.7e12 * 1e3
        print(json.dumps({"op": "encode_batch", "N": N, "M": M, "B": B, "block_bytes": 4 * S, "ok": ok, "ms": round(ms, 4), "ms_runs": [round(v, 4) for v in runs],
                          "memory_floor_ms": round(mem_ms, 4), "product_floor_ms_at_1.7e12": round(prod_ms, 4),
                          "binds": "memory" if mem_ms >= prod_ms else "products", "fraction_of_binding_floor": round(max(mem_ms, prod_ms) / ms, 3),
                          "GBps_data_plus_parity": round((N + M) * B * S * 4 / ms / 1e6, 1),
                          "per_stripe_ms_scaled_to_B": round(ms_per, 2), "per_stripe_stripes_timed": few, "speedup": round(ms_per / ms, 1),
                          "gpu": card["name"], "power_limit_w": card["power_limit_w"]}), flush=True)
        del data, parity, scratch, out
        torch.cuda.empty_cache()


def reconstruct_batch_sweep():
    """Degraded read of a batch of small stripes with one loss pattern (fastecc_b200_rs_reconstruct_batch, DESIGN 3m) at the shapes
    of --batch, 4 KiB blocks, B stripes of about 1 GiB of data in all, data, parity and output in separate stripe-major buffers.
    Loss cases: (i) one lost data block, (ii) one lost parity block, (iii) two lost data blocks, (iv) M lost data blocks, all
    wanted.  The call: CUDA events around `reps` back-to-back calls, alternated twice with rs_encode_batch_dev of the same
    stripes (the lower figures).  The kernel: its device time in a torch.profiler trace of the same calls, over the memory floor
    ((N + n_out) * B * 4096 bytes at the data sheet's 3.35 TB/s) and the product floor (n_out * N * B * 1024 products at the
    1.7e12 products/s of update_parity_kernel, DESIGN 3h); the larger one binds.  The per-stripe path: rs_reconstruct_dev of the
    first `few` stripes, events around the loop, scaled to B (n/a where a + n_want_parity > 32).  "ok": the output of three
    sampled stripes equals their original blocks.  Each line names the card and its power limit, read in the same run."""
    from torch.profiler import ProfilerActivity, profile
    from bench import gpu_identity
    fe.init(0)
    card = gpu_identity(torch.cuda.current_device())
    S, few, reps = 1024, 300, 10
    rng = np.random.default_rng(7)

    def kernel_ms(fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
        us = [e.device_time_total for e in prof.key_averages() if "batch_reconstruct_kernel" in e.key]
        return sum(us) / 1000 / reps if us else float("nan")

    for N, M in ((4, 2), (6, 3), (8, 4), (9, 3), (12, 4), (16, 4), (18, 3), (32, 8), (48, 16), (64, 16), (64, 64)):
        B = (1 << 30) // (N * S * 4)
        data = (torch.arange(B * N * S, device="cuda", dtype=torch.int64) * 2654435761 % P).to(torch.int32).view(B, N, S)
        parity = torch.empty((B, M, S), dtype=torch.int32, device="cuda")
        fe.rs_encode_batch_dev(data, parity)
        cases = [("i", sorted(rng.choice(N, size=1, replace=False).tolist()), []), ("ii", [], [M - 1])]
        if M >= 2:
            cases.append(("iii", sorted(rng.choice(N, size=2, replace=False).tolist()), []))
        cases.append(("iv", sorted(rng.choice(N, size=M, replace=False).tolist()), []))
        for case, ld, lp in cases:
            n_out = len(ld) + len(lp)
            out = torch.empty((B, n_out, S), dtype=torch.int32, device="cuda")
            fe.rs_reconstruct_batch_dev(data, parity, ld, lp, out=out)
            torch.cuda.synchronize()
            ok = all(torch.equal(out[b], torch.cat([data[b, ld], parity[b, lp]])) for b in (0, B // 2, B - 1))
            call = lambda: fe.rs_reconstruct_batch_dev(data, parity, ld, lp, out=out)
            runs, runs_enc = [], []
            for _ in range(2):
                runs.append(timed(call, reps))
                runs_enc.append(timed(lambda: fe.rs_encode_batch_dev(data, parity), reps))
            k_ms = min(kernel_ms(call) for _ in range(2))
            ms, ms_enc = min(runs), min(runs_enc)
            per = None
            if len(ld) + len(lp) <= 32:
                one = torch.empty((few, n_out, S), dtype=torch.int32, device="cuda")

                def per_stripe():
                    for b in range(few):
                        fe.rs_reconstruct_dev(data[b], parity[b], ld, lp, out=one[b])
                per = min(timed(per_stripe, 2) for _ in range(2)) * B / few
                del one
            mem_ms = (N + n_out) * B * S * 4 / 3.35e12 * 1e3
            prod_ms = n_out * N * B * S / 1.7e12 * 1e3
            print(json.dumps({"op": "reconstruct_batch", "N": N, "M": M, "B": B, "case": case, "a": len(ld), "n_out": n_out, "block_bytes": 4 * S,
                              "ok": ok, "call_ms": round(ms, 4), "call_ms_runs": [round(v, 4) for v in runs], "kernel_ms": round(k_ms, 4),
                              "memory_floor_ms": round(mem_ms, 4), "product_floor_ms_at_1.7e12": round(prod_ms, 4),
                              "binds": "memory" if mem_ms >= prod_ms else "products", "memory_floor_frac": round(mem_ms / k_ms, 3),
                              "fraction_of_binding_floor": round(max(mem_ms, prod_ms) / k_ms, 3),
                              "encode_batch_ms": round(ms_enc, 4), "vs_encode_batch": round(ms_enc / ms, 3),
                              "per_stripe_ms_scaled_to_B": "n/a" if per is None else round(per, 2), "per_stripe_stripes_timed": few,
                              "speedup_vs_per_stripe": "n/a" if per is None else round(per / ms, 1),
                              "gpu": card["name"], "power_limit_w": card["power_limit_w"]}), flush=True)
            del out
        del data, parity
        torch.cuda.empty_cache()


def update_batch_sweep():
    """Update of a batch of small stripes in place with one changed list (fastecc_b200_rs_update_batch, DESIGN 3n) at the shapes
    of --batch, 4 KiB blocks, B stripes of about 1 GiB of data in all, data, parity and new rows in separate stripe-major buffers;
    k changed blocks in {1, 2, N/4, N/2, N}.  The call: CUDA events around `reps` back-to-back calls (repeats write the same
    words, so each does the same work), alternated twice with two other paths, the lower figures: (a) the new rows written into
    the data with torch, then rs_encode_batch_dev of the stripes; (b) rs_update_dev stripe by stripe over the first `few`
    stripes, events around the loop, scaled to B.  Floors: memory, (3 k + 2 M) * B * 4096 bytes at the data sheet's 3.35 TB/s
    (k old rows read and written, k new rows read, M parity rows read and written); products, k * M * B * 1024 at the 1.7e12
    products/s of update_parity_kernel (DESIGN 3h); the larger one binds.  "ok": the parity of three sampled stripes equals
    rs_encode_asym_mixed_dev of their updated data.  Each line names the card and its power limit, read in the same run."""
    from bench import gpu_identity
    fe.init(0)
    card = gpu_identity(torch.cuda.current_device())
    S, few, reps = 1024, 300, 10
    rng = np.random.default_rng(13)
    for N, M in ((4, 2), (6, 3), (8, 4), (9, 3), (12, 4), (16, 4), (18, 3), (32, 8), (48, 16), (64, 16), (64, 64)):
        B = (1 << 30) // (N * S * 4)
        data = (torch.arange(B * N * S, device="cuda", dtype=torch.int64) * 2654435761 % P).to(torch.int32).view(B, N, S)
        parity = torch.empty((B, M, S), dtype=torch.int32, device="cuda")
        fe.rs_encode_batch_dev(data, parity)
        for k in sorted({1, 2, max(N // 4, 1), max(N // 2, 1), N}):
            changed = sorted(rng.choice(N, size=k, replace=False).tolist())
            new = (torch.arange(B * k * S, device="cuda", dtype=torch.int64) * 40503 % P).to(torch.int32).view(B, k, S)
            call = lambda: fe.rs_update_batch_dev(data, parity, changed, new)
            call()
            torch.cuda.synchronize()
            ok = all(torch.equal(parity[b], _encode_one(data[b], M)) and torch.equal(data[b, changed], new[b]) for b in (0, B // 2, B - 1))

            def overwrite_and_encode():
                data[:, changed] = new
                fe.rs_encode_batch_dev(data, parity)

            def per_stripe():
                for b in range(few):
                    fe.rs_update_dev(data[b], parity[b], changed, new[b])
            runs, runs_a, runs_b = [], [], []
            for _ in range(2):
                runs.append(timed(call, reps))
                runs_a.append(timed(overwrite_and_encode, reps))
                runs_b.append(timed(per_stripe, 2) * B / few)
            ms, ms_a, ms_b = min(runs), min(runs_a), min(runs_b)
            mem_ms = (3 * k + 2 * M) * B * S * 4 / 3.35e12 * 1e3
            prod_ms = k * M * B * S / 1.7e12 * 1e3
            print(json.dumps({"op": "update_batch", "N": N, "M": M, "B": B, "k": k, "block_bytes": 4 * S, "ok": ok, "call_ms": round(ms, 4),
                              "call_ms_runs": [round(v, 4) for v in runs], "memory_floor_ms": round(mem_ms, 4), "product_floor_ms_at_1.7e12": round(prod_ms, 4),
                              "binds": "memory" if mem_ms >= prod_ms else "products", "memory_floor_frac": round(mem_ms / ms, 3),
                              "fraction_of_binding_floor": round(max(mem_ms, prod_ms) / ms, 3),
                              "overwrite_encode_ms": round(ms_a, 4), "vs_overwrite_encode": round(ms_a / ms, 3),
                              "per_stripe_ms_scaled_to_B": round(ms_b, 2), "per_stripe_stripes_timed": few, "speedup_vs_per_stripe": round(ms_b / ms, 1),
                              "gpu": card["name"], "power_limit_w": card["power_limit_w"]}), flush=True)
            del new
        del data, parity
        torch.cuda.empty_cache()


def _encode_one(x, M):
    buf = x.clone()
    fe.rs_encode_asym_mixed_dev(buf, M)
    return buf[:M]


if __name__ == "__main__":
    if "--update-batch" in sys.argv:                          # only the batch update lines
        update_batch_sweep()
        sys.exit(0)
    if "--reconstruct-batch" in sys.argv:                     # only the batched degraded read lines
        reconstruct_batch_sweep()
        sys.exit(0)
    if "--batch" in sys.argv:                                 # only the batch encode lines
        batch_sweep()
        sys.exit(0)
    if "--reconstruct" in sys.argv:                           # only the degraded read lines
        reconstruct_sweep()
        sys.exit(0)
    if "--scrub-degraded" in sys.argv:                        # only the degraded scrub lines
        scrub_degraded_sweep()
        sys.exit(0)
    if "--scrub" in sys.argv:                                 # only the scrub lines
        scrub_sweep()
        sys.exit(0)
    if "--repair" in sys.argv:                                # only the repair lines
        fe.init(0)
        repair_sweep(1024)
        sys.exit(0)
    if "--update" in sys.argv:                                # only the update lines
        update_sweep()
        sys.exit(0)
    sys.exit(main())
