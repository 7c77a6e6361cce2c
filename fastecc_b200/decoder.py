"""Erasure decoding for the systematic code of the encoder (SURVEY 8f rank 4).

The reference describes the algorithm and does not implement it (README.md:88-119 "Fastest", RS.md:42-79, roadmap
README.md:173).  Code word: c[m] = f(rho^m), m = 0 .. 2N-1, rho = GF_Root(2N), deg f < N; the encoder's layout is
c[2i] = data block i, c[2j+1] = parity block j (RS.cpp:22-68).  Given any set E of at most N erased positions:

    l(x)  = prod_{e in E} (x - rho^e)                      erasure locator, built ONCE per erasure pattern
    p(x)  = f(x) * l(x)                                    known everywhere: p(rho^m) = c[m] * l(rho^m), 0 on E
    f(rho^e) = p'(rho^e) / l'(rho^e)                       because l(rho^e) = 0

Per word column that is: scale row m by l(rho^m), inverse NTT of order 2N (coefficients of p, times 2N), scale row t by
t (formal derivative, up to the shift x^-1), forward NTT of order 2N, and scale the erased rows by 1 / (2N * D[e]) with
D = NTT(m * l_m) -- the shift factors rho^-e of p' and l' cancel.  Two order-2N transforms of the whole code word
(the hot-path kernels) plus three row scalings.  The locator is a product tree over the erased points whose level
with polynomials of degree d is ONE batched order-4d transform with the polynomials as word columns.

`Backend` supplies the five primitives; `CudaBackend` is the product (C ABI on CUDA tensors).  The CPU tests plug in
the oracle instead (tests/test_decoder.py) -- nothing here falls back to the CPU by itself."""
from __future__ import annotations

P = 0xFFF00001
GEN = 19                                                    # GF(p).cpp:267-276: GF_Root(n) = 19^((P-1)/n)


class CudaBackend:
    """The primitives on CUDA int32 tensors through libfastecc_b200.so (fails loudly without it)."""

    def __init__(self):
        import torch
        import fastecc_b200 as fe
        self.torch, self.fe, self.lib = torch, fe, fe.lib()
        fe.init(torch.cuda.current_device())

    def _stream(self, t):
        return self.torch.cuda.current_stream(t.device).cuda_stream

    def ntt(self, t, inverse):                              # in place along dim 0, every column
        self.fe.ntt_dev(t, inverse)

    def gf_mul(self, a, b):
        a, b = a.contiguous(), b.contiguous()
        out = self.torch.empty_like(a)
        self.fe._check(self.lib.fastecc_b200_gf_mul_dev(a.data_ptr(), b.data_ptr(), out.data_ptr(), a.numel(), self._stream(a)))
        return out

    def gf_inv(self, a):
        a = a.contiguous()
        out = self.torch.empty_like(a)
        self.fe._check(self.lib.fastecc_b200_gf_inv_dev(a.data_ptr(), out.data_ptr(), a.numel(), self._stream(a)))
        return out

    def row_scale(self, t, consts):                         # t[i, :] *= consts[i], in place
        consts = consts.contiguous()
        if t.stride(1) == 1 and t.stride(0) % 4 == 0 and t.data_ptr() % 16 == 0:
            self.fe._check(self.lib.fastecc_b200_row_scale_dev(t.data_ptr(), t.shape[0], t.shape[1], t.stride(0), consts.data_ptr(), self._stream(t)))
        else:                                               # short helper arrays of the locator tree
            t.copy_(self.gf_mul(t, consts.view(-1, 1).expand_as(t)))


def _const_i32(torch, value: int, n: int, device):
    """n copies of the 32-bit pattern `value` (an int in [0, 2^32)) as an int32 tensor"""
    return torch.full((n,), value - (1 << 32) if value >= (1 << 31) else value, dtype=torch.int32, device=device)


def _positions(torch, erased, n2: int, device):
    """erased positions (list or tensor) -> validated sorted int64 tensor on `device`"""
    idx = torch.as_tensor(erased, dtype=torch.long).to(device).view(-1)
    me = idx.numel()
    if me > n2 // 2:
        raise ValueError("at most N = %d of the 2N symbols can be erased, got %d" % (n2 // 2, me))
    if me and (int(idx.min()) < 0 or int(idx.max()) >= n2 or (me > 1 and not bool((idx[1:] > idx[:-1]).all()))):
        raise ValueError("erased: sorted distinct positions in [0, 2N)")
    return idx


def root_powers(n2: int, device, be):
    """[rho^m for m < n2] as the forward transform of the unit impulse at index 1."""
    import torch
    x = torch.zeros((n2, 1), dtype=torch.int32, device=device)
    if n2 > 1:
        x[1, 0] = 1
    else:
        x[0, 0] = 1
    be.ntt(x, False)
    return x.view(-1)


def locator_coefficients(erased, n2: int, device, be):
    """Coefficients l_0 .. l_{n2-1} (zero padded) of prod (x - rho^e), e in `erased` (sorted, distinct, at most n2/2)."""
    import torch
    idx = _positions(torch, erased, n2, device)
    me = idx.numel()
    lc = torch.zeros(n2, dtype=torch.int32, device=device)
    if me == 0:
        lc[0] = 1
        return lc
    mp = 1
    while mp < me:
        mp *= 2
    pw = root_powers(n2, device, be)
    minus = be.gf_mul(pw[idx], _const_i32(torch, P - 1, me, device))           # -rho^e
    polys = torch.zeros((2, mp), dtype=torch.int32, device=device)             # column = one factor: [-rho^e, 1]; padding: [1, 0]
    polys[0, :me] = minus
    polys[1, :me] = 1
    polys[0, me:] = 1
    d = 1
    while polys.shape[1] > 1:
        cnt = polys.shape[1]
        a = torch.zeros((4 * d, cnt), dtype=torch.int32, device=device)        # degree <= d each; the product needs 2d+1 <= 4d coefficients
        a[:d + 1] = polys
        be.ntt(a, False)
        b = be.gf_mul(a[:, 0::2], a[:, 1::2])
        be.ntt(b, True)
        inv = pow(4 * d, P - 2, P)
        be.row_scale(b, _const_i32(torch, inv, 4 * d, device))
        polys = b[:2 * d + 1].contiguous()
        d *= 2
    lc[:mp + 1] = polys[:, 0]
    return lc


class ErasurePattern:
    """Everything that depends only on WHICH rows are lost (built once, reused for any number of code words / columns):
    l(rho^m) for every row, and 1 / (2N * D[e]) for the erased rows.  Power-of-two code words only (2N = 2 .. 2^20); the code
    words of 3 * 2^k and 9 * 2^k data blocks are decoded by CErasurePattern(..., mixed=True)."""

    def __init__(self, n2: int, erased, device, be=None):
        import torch
        self.be = be or CudaBackend()
        if n2 < 2 or n2 & (n2 - 1) or n2 > (1 << 20):
            raise ValueError("the code word must have 2N = 2 .. 2^20 rows (a power of two)")
        self.idx = _positions(torch, erased, n2, device)
        me = self.idx.numel()
        self.n2, self.me = n2, me
        if me == 0:
            return
        be = self.be
        self.pos = torch.arange(n2, dtype=torch.int32, device=device)
        lc = locator_coefficients(self.idx, n2, device, be)
        lv = lc.clone().view(n2, 1)
        be.ntt(lv, False)                                                      # l(rho^m): zero exactly on the erased rows
        self.lv = lv.view(-1).contiguous()
        dl = be.gf_mul(lc, self.pos).view(n2, 1)
        be.ntt(dl, False)                                                      # D[j] = rho^j * l'(rho^j)
        self.ce = be.gf_inv(be.gf_mul(dl.view(-1)[self.idx], _const_i32(torch, n2, me, device)))   # 1 / (2N * D[e])

    def recover(self, code):
        """code: [2N, S] int32 tensor, arbitrary content in the erased rows; DESTROYED (it is the workspace of the two
        transforms).  Returns the [len(erased), S] tensor of recovered rows, in the order of `erased`."""
        if code.shape[0] != self.n2:
            raise ValueError("code word has %d rows, the pattern was built for %d" % (code.shape[0], self.n2))
        if self.me == 0:
            return code[:0].clone()
        be = self.be
        code[self.idx] = 0                                                     # whatever was there: p vanishes on E
        be.row_scale(code, self.lv)                                            # p(rho^m) = c[m] * l(rho^m)
        be.ntt(code, True)                                                     # 2N * coefficients of p
        be.row_scale(code, self.pos)                                           # t * p_t: x * p'(x)
        be.ntt(code, False)                                                    # 2N * rho^j * p'(rho^j)
        rec = code[self.idx].contiguous()
        be.row_scale(rec, self.ce)
        return rec


def asym_erasures(N: int, M: int, lost_data, lost_parity):
    """Erased rows of the 2N-row code word (row 2i = data block i, row 2j + 1 = parity block j of the full encode) for the
    M parity blocks of EncodeReedSolomon_asym_mixed / rs_encode_asym_mixed_dev: 2i for every lost data block i,
    2*(N/M)*j' + 1 for every lost parity block j', and every odd row that was never produced.  Sorted.  Place the parity with
    code[1::2*(N//M)] = parity[:M] and decode with CErasurePattern(2N, rows, mixed=True).  ValueError when more than M blocks
    are lost."""
    N, M = int(N), int(M)
    if N < 1 or M < 1 or M > N or N % M:
        raise ValueError("M = %d must divide N = %d" % (M, N))
    data, par = sorted({int(i) for i in lost_data}), sorted({int(j) for j in lost_parity})
    if (data and (data[0] < 0 or data[-1] >= N)) or (par and (par[0] < 0 or par[-1] >= M)):
        raise ValueError("lost data blocks must lie in [0, N), lost parity blocks in [0, M)")
    if len(data) + len(par) > M:
        raise ValueError("%d blocks lost; M = %d parity blocks recover at most %d" % (len(data) + len(par), M, M))
    D, lost = N // M, set(par)
    rows = [2 * i for i in data] + [2 * j + 1 for j in range(N) if j % D or j // D in lost]
    return sorted(rows)


class _CPattern:
    """A pattern built on the device through the C ABI: owns the handle, which close() (or garbage collection) frees with the
    library function named by _free."""
    _free = None

    def __init__(self):
        import torch
        import fastecc_b200 as fe
        self._fe, self._lib, self._h = fe, fe.lib(), None
        fe.init(torch.cuda.current_device())

    @staticmethod
    def _u32(values, error: str):
        """`values` (a list, array or tensor of block or row numbers) as a contiguous uint32 array; ValueError(error) if one
        of them is negative or does not fit 32 bits."""
        import numpy as np
        a = np.ascontiguousarray(np.asarray(values, dtype=np.int64).reshape(-1))
        if a.size and (a.min() < 0 or a.max() >= (1 << 32)):
            raise ValueError(error)
        return a.astype(np.uint32)

    def close(self):
        if self._h:
            getattr(self._lib, self._free)(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:            # noqa: BLE001 -- interpreter shutdown
            pass


class CErasurePattern(_CPattern):
    """The same decoder through the C ABI (fastecc_b200_rs_decode_pattern / _recover: csrc/decode.cu): what a C++ host uses.
    Locator, its values and derivative values are built on the device in one call; recover() is asynchronous.
    mixed=True: fastecc_b200_rs_decode_pattern_mixed, for the code words of EncodeReedSolomon_mixed / rs_encode_mixed_dev
    (n2 = 2N with N = 2^k, 3 * 2^k or 9 * 2^k, 2^k <= 2^19)."""
    _free = "fastecc_b200_rs_decode_free"

    def __init__(self, n2: int, erased, mixed: bool = False):
        import ctypes
        import torch
        super().__init__()
        pos = self._u32(erased, "erased: positions in [0, 2N)")
        h = ctypes.c_void_p()
        build = self._lib.fastecc_b200_rs_decode_pattern_mixed if mixed else self._lib.fastecc_b200_rs_decode_pattern
        self._fe._check(build(n2, pos.ctypes.data, pos.size, torch.cuda.current_stream().cuda_stream, ctypes.byref(h)))
        self._h, self.n2, self.me = h, n2, int(pos.size)

    def recover(self, code):
        """code: [2N, S] int32 CUDA tensor (S % 4 == 0 or padded rows), DESTROYED.  Returns the [len(erased), S] recovered rows."""
        import torch
        if code.shape[0] != self.n2:
            raise ValueError("code word has %d rows, the pattern was built for %d" % (code.shape[0], self.n2))
        S = code.shape[1]
        out = torch.empty((self.me, (S + 3) // 4 * 4), dtype=torch.int32, device=code.device)
        if self.me:
            self._fe._check(self._lib.fastecc_b200_rs_decode_recover(self._h, code.data_ptr(), S, code.stride(0), out.data_ptr(), out.stride(0),
                                                                    torch.cuda.current_stream(code.device).cuda_stream))
        return out[:, :S]


class Repair(_CPattern):
    """Repair of a stored stripe in place through the C ABI (fastecc_b200_rs_repair_pattern / _repair: csrc/repair.cu, DESIGN 3g):
    the N data rows and M parity rows of EncodeReedSolomon_asym_mixed / rs_encode_asym_mixed_dev (M divides N, M = N included),
    with the blocks `lost_data` (< N) and `lost_parity` (< M) lost, at most M in all.  The pattern is built on the device once;
    repair() serves any number of stripes of any SIZE and is asynchronous on the current stream."""
    _free = "fastecc_b200_rs_repair_free"

    def __init__(self, N: int, M: int, lost_data=(), lost_parity=()):
        import ctypes
        import torch
        super().__init__()
        d, p = (self._u32(lost, "%s: block numbers in [0, 2^32)" % name) for name, lost in (("lost_data", lost_data), ("lost_parity", lost_parity)))
        h = ctypes.c_void_p()
        self._fe._check(self._lib.fastecc_b200_rs_repair_pattern(int(N), int(M), d.ctypes.data, d.size, p.ctypes.data, p.size,
                                                                 torch.cuda.current_stream().cuda_stream, ctypes.byref(h)))
        self._h, self.N, self.M = h, int(N), int(M)
        self.lost_data, self.lost_parity = d.tolist(), p.tolist()

    def _stripe(self, data, parity):
        if self._h is None:
            raise ValueError("the pattern was closed")
        (dp, dn, S, dpitch, stream), (pp, pn, ps, ppitch, _) = self._fe._dev_args(data), self._fe._dev_args(parity)
        for rows, want, name in ((dn, self.N, "data"), (pn, self.M, "parity")):
            if rows != want:
                raise ValueError("%s has %d rows, the pattern was built for %d" % (name, rows, want))
        if S != ps:
            raise ValueError("data and parity rows differ in length: %d and %d words" % (S, ps))
        return dp, dpitch, pp, ppitch, S, stream

    def repair(self, data, parity):
        """data: [N, S] and parity: [M, S] int32 CUDA tensors (unit word stride), repaired in place."""
        dp, dpitch, pp, ppitch, S, stream = self._stripe(data, parity)
        self._fe._check(self._lib.fastecc_b200_rs_repair(self._h, dp, dpitch, pp, ppitch, S, stream))

    def scrub(self, data, parity, max_bad: int = 0, seed: int = 0):
        """Check the surviving blocks of the stripe before repair() trusts them (fastecc_b200_rs_scrub_degraded, DESIGN 3j): the
        lost rows are never read.  Returns (status, bad_data, bad_parity) as rs_scrub_dev does, the lists naming corrupted survivors
        only (max_bad at most min((M - f) // 2, 4096), f = the lost blocks).  LOCATED: repair with Repair(N, M, lost + located);
        CLEAN: repair with this pattern.  Synchronises the current stream."""
        import ctypes
        import numpy as np
        dp, dpitch, pp, ppitch, S, stream = self._stripe(data, parity)
        cap = max(int(max_bad), 1)
        bd, bp = np.zeros(cap, dtype=np.uint32), np.zeros(cap, dtype=np.uint32)
        status, nd, npar = ctypes.c_int(-1), ctypes.c_size_t(0), ctypes.c_size_t(0)
        self._fe._check(self._lib.fastecc_b200_rs_scrub_degraded(self._h, dp, dpitch, pp, ppitch, S, int(max_bad), int(seed) & ((1 << 64) - 1), stream,
                                                                 ctypes.byref(status), bd.ctypes.data, ctypes.byref(nd), bp.ctypes.data, ctypes.byref(npar)))
        return status.value, [int(x) for x in bd[:nd.value]], [int(x) for x in bp[:npar.value]]


def decode(code, erased, be=None):
    """One-shot form: build the pattern, recover the erased rows of `code` (destroyed)."""
    return ErasurePattern(code.shape[0], erased, code.device, be).recover(code)
