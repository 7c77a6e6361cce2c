"""fastecc_b200 -- H100 (sm_90a) NTT Reed-Solomon encoder behind FastECC's call surface.

Python host-side mirror of the reference interface for the one hot path (SURVEY.md section 8b):

    MFA_NTT(data, N, SIZE, InvNTT)          <->  template MFA_NTT<uint32_t,0xFFF00001>      ntt.cpp:382-383
    EncodeReedSolomon_body(data, N, SIZE)   <->  the timed body of EncodeReedSolomon        RS.cpp:41-63
    GF_Add / GF_Sub / GF_Mul / GF_Pow / GF_Root / GF_Inv  (host scalars, GF(p).cpp:37-48,110-127,254-297)

Everything that computes on blocks goes through the C ABI in include/fastecc_b200.h (ctypes); there is no CPU
fallback: if libfastecc_b200.so is missing, or no sm_90 GPU is usable, the calls raise.  `data` mirrors the
reference's ``T** data``: either a C-contiguous numpy uint32 array of shape (N, SIZE) (block i = data[i]) or a
sequence of N 1-D uint32 arrays (arbitrary block addresses).  Results are written in place.
"""
from __future__ import annotations

import ctypes
import os
from typing import Sequence, Union

import numpy as np

P = 0xFFF00001
MAX_LOG_N = 20
MAX_LOG_N_ENCODE = 19

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("FASTECC_B200_LIB", os.path.join(_HERE, "libfastecc_b200.so"))   # override: A/B builds of the same ABI
_lib = None


class FastEccError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"fastecc_b200 error {code}: {msg}")
        self.code = code


def lib() -> ctypes.CDLL:
    """Load the CUDA library (built by fastecc_b200.build / __graft_entry__.build). Never falls back."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(f"{LIB_PATH} is missing: run `python -m fastecc_b200.build` (no CPU fallback exists)")
        L = ctypes.CDLL(LIB_PATH)
        sz, vp, ci = ctypes.c_size_t, ctypes.c_void_p, ctypes.c_int
        L.fastecc_b200_init.argtypes = [ci]; L.fastecc_b200_init.restype = ci
        L.fastecc_b200_shutdown.argtypes = []; L.fastecc_b200_shutdown.restype = None
        L.fastecc_b200_last_error.argtypes = []; L.fastecc_b200_last_error.restype = ctypes.c_char_p
        L.fastecc_b200_device.argtypes = []; L.fastecc_b200_device.restype = ci
        L.fastecc_b200_num_sms.argtypes = []; L.fastecc_b200_num_sms.restype = ci
        L.fastecc_b200_ntt_u32.argtypes = [vp, sz, sz, ci]; L.fastecc_b200_ntt_u32.restype = ci
        L.fastecc_b200_rs_encode.argtypes = [vp, sz, sz]; L.fastecc_b200_rs_encode.restype = ci
        L.fastecc_b200_ntt_u32_dev.argtypes = [vp, sz, sz, sz, ci, vp]; L.fastecc_b200_ntt_u32_dev.restype = ci
        L.fastecc_b200_rs_encode_dev.argtypes = [vp, sz, sz, sz, vp]; L.fastecc_b200_rs_encode_dev.restype = ci
        L.fastecc_b200_rs_encode_asym.argtypes = [vp, sz, sz, sz]; L.fastecc_b200_rs_encode_asym.restype = ci
        L.fastecc_b200_rs_encode_asym_dev.argtypes = [vp, sz, sz, sz, sz, vp]; L.fastecc_b200_rs_encode_asym_dev.restype = ci
        L.fastecc_b200_rs_encode_mixed.argtypes = [vp, sz, sz]; L.fastecc_b200_rs_encode_mixed.restype = ci
        L.fastecc_b200_rs_encode_mixed_dev.argtypes = [vp, sz, sz, sz, vp]; L.fastecc_b200_rs_encode_mixed_dev.restype = ci
        L.fastecc_b200_rs_encode_asym_mixed.argtypes = [vp, sz, sz, sz]; L.fastecc_b200_rs_encode_asym_mixed.restype = ci
        L.fastecc_b200_rs_encode_asym_mixed_dev.argtypes = [vp, sz, sz, sz, sz, vp]; L.fastecc_b200_rs_encode_asym_mixed_dev.restype = ci
        L.fastecc_b200_bytes_to_gfp_dev.argtypes = [vp, vp, sz, sz, sz, vp]; L.fastecc_b200_bytes_to_gfp_dev.restype = ci
        L.fastecc_b200_gfp_to_bytes_dev.argtypes = [vp, vp, sz, sz, sz, vp]; L.fastecc_b200_gfp_to_bytes_dev.restype = ci
        L.fastecc_b200_gf_mul_dev.argtypes = [vp, vp, vp, sz, vp]; L.fastecc_b200_gf_mul_dev.restype = ci
        L.fastecc_b200_gf_inv_dev.argtypes = [vp, vp, sz, vp]; L.fastecc_b200_gf_inv_dev.restype = ci
        L.fastecc_b200_row_scale_dev.argtypes = [vp, sz, sz, sz, vp, vp]; L.fastecc_b200_row_scale_dev.restype = ci
        L.fastecc_b200_rs_decode_pattern.argtypes = [sz, vp, sz, vp, ctypes.POINTER(vp)]; L.fastecc_b200_rs_decode_pattern.restype = ci
        L.fastecc_b200_rs_decode_pattern_mixed.argtypes = [sz, vp, sz, vp, ctypes.POINTER(vp)]; L.fastecc_b200_rs_decode_pattern_mixed.restype = ci
        L.fastecc_b200_rs_decode_recover.argtypes = [vp, vp, sz, sz, vp, sz, vp]; L.fastecc_b200_rs_decode_recover.restype = ci
        L.fastecc_b200_rs_decode_count.argtypes = [vp]; L.fastecc_b200_rs_decode_count.restype = sz
        L.fastecc_b200_rs_decode_free.argtypes = [vp]; L.fastecc_b200_rs_decode_free.restype = None
        L.fastecc_b200_rs_repair_pattern.argtypes = [sz, sz, vp, sz, vp, sz, vp, ctypes.POINTER(vp)]; L.fastecc_b200_rs_repair_pattern.restype = ci
        L.fastecc_b200_rs_repair.argtypes = [vp, vp, sz, vp, sz, sz, vp]; L.fastecc_b200_rs_repair.restype = ci
        L.fastecc_b200_rs_repair_free.argtypes = [vp]; L.fastecc_b200_rs_repair_free.restype = None
        L.fastecc_b200_rs_update.argtypes = [vp, sz, sz, vp, sz, sz, vp, sz, vp, sz, sz, vp]; L.fastecc_b200_rs_update.restype = ci
        L.fastecc_b200_rs_scrub.argtypes = [vp, sz, sz, vp, sz, sz, sz, sz, ctypes.c_uint64, vp, vp, vp, vp, vp, vp]; L.fastecc_b200_rs_scrub.restype = ci
        L.fastecc_b200_rs_scrub_degraded.argtypes = [vp, vp, sz, vp, sz, sz, sz, ctypes.c_uint64, vp, vp, vp, vp, vp, vp]; L.fastecc_b200_rs_scrub_degraded.restype = ci
        L.fastecc_b200_rs_reconstruct.argtypes = [vp, sz, sz, vp, sz, sz, vp, sz, vp, sz, vp, sz, vp, sz, vp, sz, sz, vp]; L.fastecc_b200_rs_reconstruct.restype = ci
        L.fastecc_b200_rs_encode_batch.argtypes = [vp, sz, sz, sz, vp, sz, sz, sz, sz, sz, vp]; L.fastecc_b200_rs_encode_batch.restype = ci
        L.fastecc_b200_rs_reconstruct_batch.argtypes = [vp, sz, sz, sz, vp, sz, sz, sz, vp, sz, vp, sz, vp, sz, vp, sz, vp, sz, sz, sz, sz, vp]
        L.fastecc_b200_rs_reconstruct_batch.restype = ci
        L.fastecc_b200_rs_update_batch.argtypes = [vp, sz, sz, sz, vp, sz, sz, sz, vp, sz, vp, sz, sz, sz, sz, vp]; L.fastecc_b200_rs_update_batch.restype = ci
        L.fastecc_b200_rs_encode_shard_pass.argtypes = [vp, sz, ci, ci, sz, sz, ci, vp]; L.fastecc_b200_rs_encode_shard_pass.restype = ci
        L.fastecc_b200_rs_encode_shard_pass_p2p.argtypes = [vp, vp, sz, ci, ci, sz, sz, ci, vp]; L.fastecc_b200_rs_encode_shard_pass_p2p.restype = ci
        L.fastecc_b200_ntt_shard_pass_p2p.argtypes = [vp, vp, sz, ci, ci, sz, sz, ci, ci, vp]; L.fastecc_b200_ntt_shard_pass_p2p.restype = ci
        L.fastecc_b200_rs_encode_shard_p2p.argtypes = [vp, vp, vp, vp, sz, ci, ci, sz, sz, vp]; L.fastecc_b200_rs_encode_shard_p2p.restype = ci
        L.fastecc_b200_ntt_shard_p2p.argtypes = [vp, vp, vp, vp, sz, ci, ci, sz, sz, ci, vp]; L.fastecc_b200_ntt_shard_p2p.restype = ci
        L.fastecc_b200_shard_barrier.argtypes = [vp, ci, ci, ctypes.c_uint32, vp]; L.fastecc_b200_shard_barrier.restype = ci
        L.fastecc_b200_dev_alloc.argtypes = [sz]; L.fastecc_b200_dev_alloc.restype = vp
        L.fastecc_b200_dev_free.argtypes = [vp]; L.fastecc_b200_dev_free.restype = None
        L.fastecc_b200_ipc_export.argtypes = [vp, vp]; L.fastecc_b200_ipc_export.restype = ci
        L.fastecc_b200_ipc_open.argtypes = [vp, ctypes.POINTER(vp)]; L.fastecc_b200_ipc_open.restype = ci
        L.fastecc_b200_ipc_close.argtypes = [vp]; L.fastecc_b200_ipc_close.restype = ci
        L.fastecc_b200_kernel_launches.argtypes = []; L.fastecc_b200_kernel_launches.restype = ctypes.c_ulonglong
        L.fastecc_b200_rs_encode_dev_timed.argtypes = [vp, sz, sz, sz, vp, vp, vp, vp]; L.fastecc_b200_rs_encode_dev_timed.restype = ci
        L.fastecc_b200_shard_geometry.argtypes = [sz, ci, vp, vp, vp]; L.fastecc_b200_shard_geometry.restype = ci
        L.fastecc_b200_copy2d_async.argtypes = [vp, sz, vp, sz, sz, sz, ci, vp]; L.fastecc_b200_copy2d_async.restype = ci
        L.fastecc_b200_pin_host_buffers.argtypes = [ci]; L.fastecc_b200_pin_host_buffers.restype = ci
        L.fastecc_b200_hash_u32.argtypes = [vp, sz, sz]; L.fastecc_b200_hash_u32.restype = ctypes.c_uint32
        L.fastecc_b200_host_alloc.argtypes = [sz]; L.fastecc_b200_host_alloc.restype = vp
        L.fastecc_b200_host_free.argtypes = [vp]; L.fastecc_b200_host_free.restype = None
        _lib = L
    return _lib


def _check(rc: int) -> None:
    if rc != 0:
        raise FastEccError(rc, lib().fastecc_b200_last_error().decode())


def init(device: int = 0) -> None:
    _check(lib().fastecc_b200_init(int(device)))


def shutdown() -> None:
    lib().fastecc_b200_shutdown()


def pin_host_buffers(enable: bool = True) -> None:
    """Opt in to page-locking large pageable arrays passed to MFA_NTT / EncodeReedSolomon_body in place (see the header)."""
    _check(lib().fastecc_b200_pin_host_buffers(1 if enable else 0))


def kernel_launches() -> int:
    return int(lib().fastecc_b200_kernel_launches())


# ---- host scalars of the reference call surface (pure Python ints; used by callers such as RS.cpp:51-57) ----------
def GF_Sub(x: int, y: int) -> int:            # GF(p).cpp:37-42
    return (x - y) % P


def GF_Add(x: int, y: int) -> int:            # GF(p).cpp:44-48
    return (x + y) % P


def GF_Mul(x: int, y: int) -> int:            # GF(p).cpp:110-127
    return (x * y) % P


def GF_Pow(x: int, n: int) -> int:            # GF(p).cpp:254-264
    return pow(x, n, P)


def GF_Root(n: int) -> int:                   # GF(p).cpp:267-276
    return pow(19, (P - 1) // n, P)


def GF_Inv(x: int) -> int:                    # GF(p).cpp:293-297
    return pow(x, P - 2, P)


Blocks = Union[np.ndarray, Sequence[np.ndarray]]


def _pointer_table(data: Blocks, N: int, SIZE: int):
    """Build the reference's ``T** data`` (RS.cpp:31-33) for a 2-D array or a sequence of block arrays."""
    if isinstance(data, np.ndarray):
        if data.dtype != np.uint32 or data.ndim != 2 or data.shape != (N, SIZE) or not data.flags.c_contiguous or not data.flags.writeable:
            raise ValueError("data must be a writeable C-contiguous uint32 array of shape (N, SIZE)")
        tab = data.ctypes.data + np.arange(N, dtype=np.uint64) * np.uint64(SIZE * 4)      # data[i] = data0 + i*SIZE
        return tab, data
    if len(data) != N:
        raise ValueError("len(data) != N")
    tab = np.empty(N, dtype=np.uint64)
    for i, blk in enumerate(data):
        if blk.dtype != np.uint32 or blk.ndim != 1 or blk.shape[0] < SIZE or not blk.flags.c_contiguous or not blk.flags.writeable:
            raise ValueError(f"block {i} must be a writeable contiguous uint32 vector of >= SIZE words")
        tab[i] = blk.ctypes.data
    return tab, data


def MFA_NTT(data: Blocks, N: int, SIZE: int, InvNTT: bool) -> None:
    """In-place length-N NTT of every word column (unnormalised inverse), bit-exact with ntt.cpp:382-447."""
    tab, keep = _pointer_table(data, N, SIZE)
    _check(lib().fastecc_b200_ntt_u32(tab.ctypes.data, N, SIZE, 1 if InvNTT else 0))
    del keep


def EncodeReedSolomon_body(data: Blocks, N: int, SIZE: int) -> None:
    """N data blocks -> N parity blocks in place: MFA_NTT(inv); x[i] *= root_2N^i/N; MFA_NTT(fwd)  (RS.cpp:41-63)."""
    tab, keep = _pointer_table(data, N, SIZE)
    _check(lib().fastecc_b200_rs_encode(tab.ctypes.data, N, SIZE))
    del keep


def EncodeReedSolomon_asym(data: Blocks, N: int, M: int, SIZE: int) -> None:
    """N data blocks -> M = N/2^k parity blocks in data[0..M): parity block j' = block (N/M)*j' of the full encode
    (the even points of the second transform, RS.cpp:65-66)."""
    tab, keep = _pointer_table(data, N, SIZE)
    _check(lib().fastecc_b200_rs_encode_asym(tab.ctypes.data, N, M, SIZE))
    del keep


def EncodeReedSolomon_mixed(data: Blocks, N: int, SIZE: int) -> None:
    """N = 2^k, 3 * 2^k or 9 * 2^k data blocks (2^k <= 2^19) -> N parity blocks in place: parity j = f(rho^(2j+1)),
    rho = GF_Root(2N), f(rho^(2i)) = data block i.  Powers of two give exactly EncodeReedSolomon_body's result."""
    tab, keep = _pointer_table(data, N, SIZE)
    _check(lib().fastecc_b200_rs_encode_mixed(tab.ctypes.data, N, SIZE))
    del keep


def EncodeReedSolomon_asym_mixed(data: Blocks, N: int, M: int, SIZE: int) -> None:
    """N data blocks (as EncodeReedSolomon_mixed takes them) -> M parity blocks in data[0..M), M any divisor of N: parity
    block j' = block (N/M)*j' of EncodeReedSolomon_mixed.  Blocks M .. N-1 are left untouched."""
    tab, keep = _pointer_table(data, N, SIZE)
    _check(lib().fastecc_b200_rs_encode_asym_mixed(tab.ctypes.data, N, M, SIZE))
    del keep


def rs_code_order(K: int) -> int:
    """The smallest N >= K that EncodeReedSolomon_mixed / rs_encode_mixed_dev accept (2^k, 3 * 2^k or 9 * 2^k, 2^k <= 2^19):
    the number of data blocks to pad K blocks to instead of the next power of two (at most 4/3 K up to K = 2^19, at most 2 K
    beyond).  ValueError for K < 1 or K > 9 * 2^19."""
    K = int(K)
    if K < 1 or K > 9 << MAX_LOG_N_ENCODE:
        raise ValueError("no code of %d data blocks: 1 <= K <= 9 * 2^19" % K)
    best = None
    for r in (1, 3, 9):
        n = r
        while n < K:
            n *= 2
        if n // r <= 1 << MAX_LOG_N_ENCODE and (best is None or n < best):
            best = n
    return best


# ---- device-resident entry points (torch tensors are used only as owners of device memory) -----------------------
def _dev_args(t):
    import torch
    if not (t.is_cuda and t.dim() == 2 and t.dtype in (torch.int32, torch.uint32) and t.stride(1) == 1):
        raise ValueError("expected a 2-D CUDA int32/uint32 tensor with unit stride along the word dimension")
    return t.data_ptr(), t.shape[0], t.shape[1], t.stride(0), torch.cuda.current_stream(t.device).cuda_stream


def ntt_dev(t, inverse: bool = False) -> None:
    ptr, N, size, pitch, stream = _dev_args(t)
    _check(lib().fastecc_b200_ntt_u32_dev(ptr, N, size, pitch, 1 if inverse else 0, stream))


def rs_encode_dev(t) -> None:
    ptr, N, size, pitch, stream = _dev_args(t)
    _check(lib().fastecc_b200_rs_encode_dev(ptr, N, size, pitch, stream))


def rs_encode_dev_timed(t):
    """One encode with an event between the passes: [(kernel instantiation, ms), ...] (synchronises the stream)."""
    ptr, N, size, pitch, stream = _dev_args(t)
    cap = 8
    ms = (ctypes.c_float * cap)(); names = (ctypes.c_char_p * cap)(); n = ctypes.c_int(cap)
    _check(lib().fastecc_b200_rs_encode_dev_timed(ptr, N, size, pitch, stream, ms, names, ctypes.byref(n)))
    return [((names[i] or b"?").decode(), float(ms[i])) for i in range(n.value)]


def rs_encode_mixed_dev(t) -> None:
    """EncodeReedSolomon_mixed on the rows of a device tensor (N = t.shape[0] = 2^k, 3 * 2^k or 9 * 2^k)."""
    ptr, N, size, pitch, stream = _dev_args(t)
    _check(lib().fastecc_b200_rs_encode_mixed_dev(ptr, N, size, pitch, stream))


def rs_encode_asym_dev(t, M: int) -> None:
    """Rows [0, M) of t receive the M parity blocks; the other rows are undefined afterwards."""
    ptr, N, size, pitch, stream = _dev_args(t)
    _check(lib().fastecc_b200_rs_encode_asym_dev(ptr, N, M, size, pitch, stream))


def rs_encode_asym_mixed_dev(t, M: int) -> None:
    """EncodeReedSolomon_asym_mixed on the rows of a device tensor: rows [0, M) of t receive the M parity blocks (M divides
    N = t.shape[0]); the other rows are undefined afterwards."""
    ptr, N, size, pitch, stream = _dev_args(t)
    _check(lib().fastecc_b200_rs_encode_asym_mixed_dev(ptr, N, M, size, pitch, stream))


def rs_repair_dev(data, parity, lost_data, lost_parity) -> None:
    """Repair a stored stripe in place: data = the N data rows, parity = the M parity rows of rs_encode_asym_mixed_dev (int32
    CUDA tensors, 16-byte aligned rows with pitches that are multiples of 4 words); lost_data / lost_parity = the lost block
    numbers (at most M in all).  The lost rows receive their canonical blocks, nothing else is written.  One-shot form of
    decoder.Repair (which builds the pattern once for any number of stripes)."""
    from .decoder import Repair
    r = Repair(data.shape[0], parity.shape[0], lost_data, lost_parity)
    try:
        r.repair(data, parity)
    finally:
        r.close()


def rs_update_dev(data, parity, changed, new) -> None:
    """Update a stored stripe in place (fastecc_b200_rs_update, DESIGN 3h): data = the N data rows, parity = the M parity rows
    of rs_encode_asym_mixed_dev (int32 CUDA tensors, 16-byte aligned rows with pitches that are multiples of 4 words); changed =
    ascending distinct block numbers below N; row i of `new` is the new content of data block changed[i].  The changed data rows
    receive their canonical new blocks and the parity becomes the encode of the updated data; the stored parity must be the
    encode of the stored data.  Asynchronous on the current stream."""
    from .decoder import _CPattern
    (dp, N, S, dpitch, stream), (pp, M, ps, ppitch, _), (nptr, k, ns, npitch, _) = _dev_args(data), _dev_args(parity), _dev_args(new)
    idx = _CPattern._u32(changed, "changed: block numbers in [0, 2^32)")
    if k != idx.size:
        raise ValueError("new has %d rows for %d changed blocks" % (k, idx.size))
    if not S == ps == ns:
        raise ValueError("data, parity and new rows differ in length: %d, %d and %d words" % (S, ps, ns))
    _check(lib().fastecc_b200_rs_update(dp, dpitch, N, pp, ppitch, M, idx.ctypes.data, idx.size, nptr, npitch, S, stream))


SCRUB_CLEAN, SCRUB_LOCATED, SCRUB_DETECTED = 0, 1, 2


def rs_scrub_dev(data, parity, max_bad: int = 0, seed: int = 0):
    """Scrub a stored stripe (fastecc_b200_rs_scrub, DESIGN 3i): data = the N data rows, parity = the M parity rows of
    rs_encode_asym_mixed_dev (int32 CUDA tensors, 16-byte aligned rows with pitches that are multiples of 4 words), read only.
    Returns (status, bad_data, bad_parity): SCRUB_CLEAN if the parity is the encode of the data; SCRUB_LOCATED with the ascending
    lists of corrupted data and parity blocks (at most max_bad in all, ready for rs_repair_dev); SCRUB_DETECTED if corrupted but
    not located within max_bad (0 = detect only; at most min(M // 2, 4096)).  `seed` picks the fold weights (the header states
    them).  Synchronises the current stream."""
    (dp, N, S, dpitch, stream), (pp, M, ps, ppitch, _) = _dev_args(data), _dev_args(parity)
    if S != ps:
        raise ValueError("data and parity rows differ in length: %d and %d words" % (S, ps))
    cap = max(int(max_bad), 1)
    bd, bp = np.zeros(cap, dtype=np.uint32), np.zeros(cap, dtype=np.uint32)
    status, nd, npar = ctypes.c_int(-1), ctypes.c_size_t(0), ctypes.c_size_t(0)
    _check(lib().fastecc_b200_rs_scrub(dp, dpitch, N, pp, ppitch, M, S, int(max_bad), int(seed) & ((1 << 64) - 1), stream, ctypes.byref(status),
                                       bd.ctypes.data, ctypes.byref(nd), bp.ctypes.data, ctypes.byref(npar)))
    return status.value, [int(x) for x in bd[:nd.value]], [int(x) for x in bp[:npar.value]]


def rs_scrub_degraded_dev(data, parity, lost_data, lost_parity, max_bad: int = 0, seed: int = 0):
    """Scrub a degraded stripe (fastecc_b200_rs_scrub_degraded, DESIGN 3j): rs_scrub_dev with the blocks lost_data / lost_parity
    known lost (fewer than M in all; their rows are never read).  The survivors are checked: (status, bad_data, bad_parity) with
    the corrupted survivors when LOCATED (max_bad at most min((M - f) // 2, 4096), f lost blocks).  Repair with lost + located
    blocks afterwards.  One-shot form of decoder.Repair(...).scrub (which builds the pattern once)."""
    from .decoder import Repair
    r = Repair(data.shape[0], parity.shape[0], lost_data, lost_parity)
    try:
        return r.scrub(data, parity, max_bad, seed)
    finally:
        r.close()


def rs_reconstruct_dev(data, parity, lost_data, lost_parity, want_data=None, want_parity=None, out=None):
    """Degraded read of a stored stripe (fastecc_b200_rs_reconstruct, DESIGN 3k): data = the N data rows, parity = the M parity
    rows of rs_encode_asym_mixed_dev (int32 CUDA tensors, 16-byte aligned rows with pitches that are multiples of 4 words), read
    only; lost_data / lost_parity = the unavailable blocks (at most M in all); want_data / want_parity = the lost blocks to produce
    (default: all of them; len(lost_data) + len(want_parity) <= 32).  Reads the surviving data rows and the len(lost_data) lowest
    surviving parity rows only.  Row q of `out` receives want_data[q], then the wanted parity blocks; `out` defaults to a new
    int32 tensor with rows of ceil4(SIZE) words.  Returns `out`.  Asynchronous on the current stream."""
    import torch
    from .decoder import _CPattern
    (dp, N, S, dpitch, stream), (pp, M, ps, ppitch, _) = _dev_args(data), _dev_args(parity)
    if S != ps:
        raise ValueError("data and parity rows differ in length: %d and %d words" % (S, ps))
    u32 = lambda v: _CPattern._u32(v, "block numbers in [0, 2^32)")
    ld, lp = u32(lost_data), u32(lost_parity)
    wd = ld if want_data is None else u32(want_data)
    wp = lp if want_parity is None else u32(want_parity)
    n = wd.size + wp.size
    if out is None:
        out = torch.empty((n, (S + 3) // 4 * 4), dtype=torch.int32, device=data.device)[:, :S]
    optr, on, osz, opitch, _ = _dev_args(out)
    if (on, osz) != (n, S):
        raise ValueError("out is %d x %d words for %d wanted blocks of %d words" % (on, osz, n, S))
    arr = lambda a: a.ctypes.data if a.size else None
    _check(lib().fastecc_b200_rs_reconstruct(dp, dpitch, N, pp, ppitch, M, arr(ld), ld.size, arr(lp), lp.size, arr(wd), wd.size, arr(wp), wp.size,
                                             optr, opitch, S, stream))
    return out


def _batch_args(t, name):
    """(pointer, B, rows, S, pitch, stripe stride) of a [B, rows, S] batch view"""
    import torch
    if not (t.is_cuda and t.dim() == 3 and t.dtype in (torch.int32, torch.uint32) and t.stride(2) == 1):
        raise ValueError("%s: expected a 3-D CUDA int32/uint32 tensor with unit stride along the word dimension" % name)
    return t.data_ptr(), t.shape[0], t.shape[1], t.shape[2], t.stride(1), t.stride(0)


def rs_encode_batch_dev(data, parity=None, M=None):
    """Encode a batch of small stripes in one launch (fastecc_b200_rs_encode_batch, DESIGN 3l): data = [B, N, S] CUDA int32/uint32
    tensor with unit word stride (a view such as buf[:, :N, :S] of a [B, N + M, pitch] buffer is fine), read only; N <= 64 in the
    family rs_encode_asym_mixed_dev accepts.  parity = [B, M, S] receives each stripe's M parity blocks, bit for bit those of
    rs_encode_asym_mixed_dev on that stripe; when it is None, M must be given and a new int32 tensor with rows of ceil4(S) words is
    allocated.  Rows 16-byte aligned with pitches and stripe strides that are multiples of 4 words; the parity may not overlap
    itself or the data.  Returns `parity`.  Asynchronous on the current stream."""
    import torch
    args = _batch_args
    dp, B, N, S, dpitch, dstride = args(data, "data")
    if parity is None:
        if M is None:
            raise ValueError("give the number of parity blocks M or a parity tensor")
        parity = torch.empty((B, int(M), (S + 3) // 4 * 4), dtype=torch.int32, device=data.device)[..., :S]
    pp, pB, pM, pS, ppitch, pstride = args(parity, "parity")
    if (pB, pS) != (B, S) or (M is not None and pM != int(M)):
        raise ValueError("parity is %d x %d x %d words for %d stripes of %s x %d-word blocks" % (pB, pM, pS, B, "M" if M is None else int(M), S))
    _check(lib().fastecc_b200_rs_encode_batch(dp, dpitch, dstride, N, pp, ppitch, pstride, pM, B, S, torch.cuda.current_stream(data.device).cuda_stream))
    return parity


def rs_reconstruct_batch_dev(data, parity, lost_data, lost_parity, want_data=None, want_parity=None, out=None):
    """Degraded read of a batch of small stripes with one loss pattern (fastecc_b200_rs_reconstruct_batch, DESIGN 3m): data =
    [B, N, S], parity = [B, M, S] CUDA int32/uint32 tensors with unit word stride (views such as buf[:, :N, :S] are fine), read
    only; N <= 64 in the family rs_encode_asym_mixed_dev accepts.  lost_data / lost_parity = the blocks every stripe lost (at most
    M in all); want_data / want_parity = the lost blocks to produce (default: all of them).  Reads each stripe's surviving data
    rows and its len(lost_data) lowest surviving parity rows only.  out = [B, n_out, S] receives each stripe's wanted data blocks,
    then its wanted parity blocks, bit for bit what rs_reconstruct_dev gives for that stripe; when it is None, a new int32 tensor
    with rows of ceil4(S) words is allocated.  Rows 16-byte aligned with pitches and stripe strides that are multiples of 4 words;
    `out` may not overlap itself, the data or the parity.  Returns `out`.  Asynchronous on the current stream."""
    import torch
    from .decoder import _CPattern
    dp, B, N, S, dpitch, dstride = _batch_args(data, "data")
    pp, pB, M, pS, ppitch, pstride = _batch_args(parity, "parity")
    if (pB, pS) != (B, S):
        raise ValueError("parity is %d x %d x %d words for %d stripes of %d-word blocks" % (pB, M, pS, B, S))
    u32 = lambda v: _CPattern._u32(v, "block numbers in [0, 2^32)")
    ld, lp = u32(lost_data), u32(lost_parity)
    wd = ld if want_data is None else u32(want_data)
    wp = lp if want_parity is None else u32(want_parity)
    n = wd.size + wp.size
    if out is None:
        out = torch.empty((B, n, (S + 3) // 4 * 4), dtype=torch.int32, device=data.device)[..., :S]
    op, oB, on, oS, opitch, ostride = _batch_args(out, "out")
    if (oB, on, oS) != (B, n, S):
        raise ValueError("out is %d x %d x %d words for %d stripes of %d wanted blocks of %d words" % (oB, on, oS, B, n, S))
    arr = lambda a: a.ctypes.data if a.size else None
    _check(lib().fastecc_b200_rs_reconstruct_batch(dp, dpitch, dstride, N, pp, ppitch, pstride, M, arr(ld), ld.size, arr(lp), lp.size, arr(wd), wd.size,
                                                   arr(wp), wp.size, op, opitch, ostride, B, S, torch.cuda.current_stream(data.device).cuda_stream))
    return out


def rs_update_batch_dev(data, parity, changed, new) -> None:
    """Update a batch of small stripes in place with one changed list (fastecc_b200_rs_update_batch, DESIGN 3n): data = [B, N, S],
    parity = [B, M, S] and new = [B, k, S] CUDA int32/uint32 tensors with unit word stride (views such as buf[:, :N, :S] are
    fine; new may be expanded over B with stride 0); N <= 64 in the family rs_encode_asym_mixed_dev accepts.  changed = k
    ascending distinct block numbers below N, the same for every stripe; row q of new[b] is the new content of data block
    changed[q] of stripe b.  The changed data rows receive their canonical new blocks and the parity becomes the batch encode of
    the updated data; the stored parity must be the encode of the stored data.  Data rows outside `changed` are never read.  All
    N + M rows of all stripes must be pairwise disjoint and apart from the new rows.  Asynchronous on the current stream."""
    import torch
    from .decoder import _CPattern
    dp, B, N, S, dpitch, dstride = _batch_args(data, "data")
    pp, pB, M, pS, ppitch, pstride = _batch_args(parity, "parity")
    nptr, nB, k, nS, npitch, nstride = _batch_args(new, "new")
    idx = _CPattern._u32(changed, "changed: block numbers in [0, 2^32)")
    if k != idx.size:
        raise ValueError("new has %d rows for %d changed blocks" % (k, idx.size))
    if not (B == pB == nB and S == pS == nS):
        raise ValueError("data, parity and new are %d x %d, %d x %d and %d x %d (stripes x words)" % (B, S, pB, pS, nB, nS))
    _check(lib().fastecc_b200_rs_update_batch(dp, dpitch, dstride, N, pp, ppitch, pstride, M, idx.ctypes.data if idx.size else None, idx.size, nptr,
                                              npitch, nstride, B, S, torch.cuda.current_stream(data.device).cuda_stream))


def bytes_to_gfp_dev(raw, words=None):
    """raw: 2-D CUDA uint8 tensor [n_blocks, 4*W] (contiguous) -> int32 tensor [n_blocks, pitch] with words 0..W of every row
    set (GF.md:72-104 recoding: all of them < P).  pitch = W + 4 keeps rows 16-byte aligned."""
    import torch
    n, nbytes = raw.shape
    W = nbytes // 4
    if words is None:
        words = torch.zeros((n, W + 4), dtype=torch.int32, device=raw.device)
    _check(lib().fastecc_b200_bytes_to_gfp_dev(raw.data_ptr(), words.data_ptr(), n, W, words.stride(0), torch.cuda.current_stream(raw.device).cuda_stream))
    return words


def gfp_to_bytes_dev(words, W: int):
    import torch
    n = words.shape[0]
    raw = torch.empty((n, 4 * W), dtype=torch.uint8, device=words.device)
    _check(lib().fastecc_b200_gfp_to_bytes_dev(words.data_ptr(), raw.data_ptr(), n, W, words.stride(0), torch.cuda.current_stream(words.device).cuda_stream))
    return raw


def reference_hash(data: Blocks) -> int:
    """main.cpp:203-212 rolling hash over blocks in data[i] order (verification only; sequential by construction)."""
    if isinstance(data, np.ndarray):
        data = np.ascontiguousarray(data, dtype=np.uint32)
        if data.ndim == 1:
            data = data.reshape(1, -1)
        N, SIZE = data.shape
    else:
        N, SIZE = len(data), min(int(b.shape[0]) for b in data)
    tab = (data.ctypes.data + np.arange(N, dtype=np.uint64) * np.uint64(SIZE * 4)) if isinstance(data, np.ndarray) \
        else np.array([b.ctypes.data for b in data], dtype=np.uint64)
    return int(lib().fastecc_b200_hash_u32(tab.ctypes.data, N, SIZE))
