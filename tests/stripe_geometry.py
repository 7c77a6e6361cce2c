"""The launch rules of the stripe kernels restated in Python, and the geometry classes they select (test-only, no library code).

Each function maps the shape of one call to the launch the library makes: the kernel's template instance, block and dynamic
shared memory, and the geometry class, the tuple of launch parameters that selects different code plus the edge flags that the
launch meets.  The constants are copied from the sources named beside them; tests/test_stripe_geometry.py checks on the GPU that
the restatement is the library's rule (through the profiler's kernel records) and that every class computes the encode by
definition.

  batch_read    launch_batch_reconstruct   csrc/batch.cu    (U, W, slices, stages)
  single_read   launch_reconstruct_sum     csrc/reconstruct.cu (U, G) + one slice or several, partial last slice, partial column block
  fold          launch_degraded_fold       csrc/scrub.cu    (log_w, slices > 1) + rows not a multiple of 4 rw
  batch_encode  launch_batch_encode        csrc/batch.cu    (U, W, G) + several row tiles, partial last row tile
  update        launch_update_parity       csrc/update.cu   several row blocks, partial row block, partial column block, several
                                                            delta groups, partial last group"""

ORDERS = [1, 2, 3, 4, 6, 8, 9, 12, 16, 18, 24, 32, 36, 48, 64]      # the batch calls' N (FASTECC_B200_BATCH_MAX_N = 64)
H100_SMS = 132                                                       # fastecc_b200_num_sms() on an H100 SXM

# csrc/batch.cu
kTileChunks = 2048                                                   # batch.cu:18, staged 16-byte chunks per CTA
kRingBudget = 109 << 10                                              # batch.cu:297, shared memory of one of two CTAs per SM
# csrc/reconstruct.cu
kTile = 32                                                           # reconstruct.cu:15, rows per tile and chunks per CTA
# csrc/scrub.cu
kFoldUnroll = 4                                                      # scrub.cu:38, rows loaded per lane before any is used
# csrc/update.cu
kRows, kCols, kGroup = 32, 32, 32                                    # update.cu:51

# Static shared memory of each kernel (the profiler reports static + dynamic)
STATIC_SMEM = {
    "batch_reconstruct_kernel": 64 * 8 + 7 * 32 * 16,                # batch.cu:159-160, srow[kMaxN] pointers, spart[7 * 32] uint4
    "batch_encode_kernel": 64 * 16,                                  # batch.cu:44, stab[kMaxN] uint4
    "reconstruct_sum_kernel": 2 * 32 * 4,                            # reconstruct.cu:34, sbase[kMaxK], slost[kMaxK]
    "scrub_fold_kernel": 0,
    "degraded_fold_kernel": 0,
    "update_parity_kernel": kGroup * kCols * 16 + kGroup * 4,        # update.cu:57-58, sd[kGroup][kCols] uint4, se[kGroup]
}


def cdiv(a, b):
    return -(-a // b)


def divisors(N):
    return [M for M in range(1, N + 1) if N % M == 0]


def family(limit):
    """The stripe orders 2^k, 3 * 2^k and 9 * 2^k up to limit, ascending"""
    out = set()
    for base in (1, 3, 9):
        n = base
        while n <= limit:
            out.add(n)
            n *= 2
    return sorted(out)


class Launch:
    """One predicted launch: kernel name (with the template instance), block, dynamic shared memory, the geometry class
    (`key`: the tuple of code-selecting parameters and the edge flags), and whatever else a test needs (`info`)."""

    def __init__(self, kernel, block, smem, key, **info):
        self.kernel, self.block, self.smem, self.key, self.info = kernel, block, smem, key, info

    def __repr__(self):
        return "Launch(%s, block=%d, smem=%d, %r, %r)" % (self.kernel, self.block, self.smem, self.key, self.info)


# ---- launch_batch_reconstruct (csrc/batch.cu:287-322) ------------------------------------------------------------------
def batch_read(N, n_out, B=1, S=4):
    U = 1 if n_out <= 8 else 2 if n_out <= 16 else 3 if n_out <= 24 else 4 if n_out <= 32 else 6 if n_out <= 48 else 8
    W = cdiv(n_out, U)
    lg_items = 5
    while (N << lg_items) < kTileChunks:
        lg_items += 1
    items = 1 << lg_items
    units = items // 32 * W
    slices = 8 // units if U == 1 and units < 8 else 1
    tile, coef = (N << lg_items) * 16, n_out * N * 16
    stages = min(4, (kRingBudget - coef) // tile) if coef + 2 * tile <= kRingBudget else 1
    s4 = cdiv(S, 4)
    n_items = B * s4
    n_tiles = cdiv(n_items, items)
    return Launch("batch_reconstruct_kernel<%du>" % U, 256, coef + stages * tile, (U, W, slices, stages),
                  lg_items=lg_items, items=items, n_items=n_items, n_tiles=n_tiles, s4=s4)


def batch_read_classes():
    """{(U, W, slices, stages): [(N, M, n_out), ...]} over every N of the family up to 64, every divisor M, n_out from 1 to M"""
    out = {}
    for N in ORDERS:
        for M in divisors(N):
            for n_out in range(1, M + 1):
                out.setdefault(batch_read(N, n_out).key, []).append((N, M, n_out))
    return out


# ---- launch_reconstruct_sum (csrc/reconstruct.cu:141-161) --------------------------------------------------------------
def single_read(N, K, S, num_sms=H100_SMS):
    s4 = cdiv(S, 4)
    col_blocks = cdiv(s4, kTile)
    G = 1 if K <= 8 else 2 if K <= 16 else 4
    U = 1 if K <= 1 else 2 if K <= 2 else 4 if K <= 4 else 8
    tiles = cdiv(N, kTile)
    slices = num_sms * 8 // col_blocks
    slices = 1 if slices < 1 else tiles if slices > tiles else slices
    slice_rows = cdiv(tiles, slices) * kTile
    slices = cdiv(N, slice_rows)
    key = (U, G, slices > 1, N % slice_rows != 0, s4 % kTile != 0)
    return Launch("reconstruct_sum_kernel<%du>" % U, 256, (kTile + K) * kTile * 16, key, grid=slices * col_blocks, slices=slices,
                  slice_rows=slice_rows, col_blocks=col_blocks)


def single_read_classes(num_sms=H100_SMS):
    """{class: [(N, K, S), ...]}: K from 1 to 32, N of the family from K to 2^19, and per N one S for every distinct number of
    slices the SM count allows (the smallest column-block count giving it), each as whole and as partial 32-chunk blocks"""
    cbs, seen = [], set()
    for cb in range(1, num_sms * 8 + 2):
        q = max(1, num_sms * 8 // cb)
        if q not in seen:
            seen.add(q)
            cbs.append(cb)
    out = {}
    for N in family(1 << 19):
        for K in range(1, min(N, 32) + 1):
            for cb in cbs:
                for S in (128 * cb, 128 * cb - 5):
                    out.setdefault(single_read(N, K, S, num_sms).key, []).append((N, K, S))
    return out


# ---- launch_degraded_fold (csrc/scrub.cu:202-224), the plain and the degraded scrub -------------------------------------
def fold(rows, S, num_sms=H100_SMS, degraded=False):
    s4 = cdiv(S, 4)
    log_w = 0
    while log_w < 5 and (1 << log_w) < s4:
        log_w += 1
    W = 1 << log_w
    rw, tiles = 32 // W, cdiv(s4, W)
    max_blocks = num_sms * 4
    groups = cdiv(rows, rw)
    slices = max_blocks * 8 // tiles
    slices = 1 if slices < 1 else groups if slices > groups else slices
    slice_rows = cdiv(groups, slices) * rw
    slices = cdiv(rows, slice_rows)
    items = tiles * slices
    blocks = min(cdiv(items, 8), max_blocks)
    key = (log_w, slices > 1, rows % (kFoldUnroll * rw) != 0)
    return Launch("degraded_fold_kernel" if degraded else "scrub_fold_kernel", 256, 0, key, grid=blocks, slices=slices, slice_rows=slice_rows)


def fold_rows_domain():
    """Every N + M of the accepted stripes (N of the family, M a divisor of N) from 2 to 2^20 rows"""
    rows = set()
    for N in family(1 << 19):
        for M in (m for m in divisors(N) if N + m <= 1 << 20) if N <= 1 << 12 else {N, N // 2, N // 3, N // 4, N // 9, 1} & set(divisors(N)):
            rows.add(N + M)
    return sorted(r for r in rows if r >= 2)


def fold_classes(num_sms=H100_SMS):
    """{class: [(rows, S), ...]}: s4 from 1 to 40 and around every change of the slice count, rows over fold_rows_domain()"""
    s4s = set(range(1, 41))
    for q in range(1, num_sms * 32 + 1):                              # tiles = num_sms 32 // q: the last s4 of each slice count
        t = num_sms * 32 // q
        s4s.update({32 * t, 32 * t + 1, 32 * t + 31})
    out = {}
    rows_domain = fold_rows_domain()
    for s4 in sorted(s4s):
        S = 4 * s4 - 1 if s4 > 1 else 3
        for rows in rows_domain:
            out.setdefault(fold(rows, S, num_sms).key, []).append((rows, S))
    return out


# ---- launch_batch_encode (csrc/batch.cu:261-285) -----------------------------------------------------------------------
def batch_encode(N, M, B=1, S=4):
    U = 1
    while M % U or M // U > 8:
        U += 1
    W = M // U
    G = 8 if 8 // W >= 8 else 4 if 8 // W >= 4 else 2 if 8 // W >= 2 else 1
    items = 32 * G
    rows = kTileChunks // items
    s4 = cdiv(S, 4)
    n_items = B * s4
    key = (U, W, G, N > rows, N % rows != 0)
    return Launch("batch_encode_kernel<%du>" % U, 32 * W * G, min(N, rows) * items * 16, key, grid=cdiv(n_items, items), items=items, rows=rows)


def batch_encode_classes():
    out = {}
    for N in ORDERS:
        for M in divisors(N):
            out.setdefault(batch_encode(N, M).key, []).append((N, M))
    return out


# ---- launch_update_parity (csrc/update.cu:127-135) ---------------------------------------------------------------------
def update(M, k, S):
    s4 = cdiv(S, 4)
    col_blocks = cdiv(s4, kCols)
    key = (M > kRows, M % kRows != 0, s4 % kCols != 0, k > kGroup, k % kGroup != 0)
    return Launch("update_parity_kernel", 256, 0, key, grid=cdiv(M, kRows) * col_blocks)


def update_classes():
    """{class: [(N, M, k), ...]}: N of the family up to 2^12, every divisor M, k changed rows from 1 to N; both column flags"""
    out = {}
    for N in family(1 << 12):
        for M in divisors(N):
            for k in range(1, min(N, 3 * kGroup + 1) + 1):
                for S in (4 * kCols, 4 * kCols - 5):
                    out.setdefault(update(M, k, S).key, []).append((N, M, k, S))
    return out


# ---- one concrete call per class (tests/test_stripe_geometry.py checks that each maps to its class) ---------------------
BATCH_READ = {                                                       # class: (N, M, n_out, S)
    (1, 1, 1, 2): (12, 1, 1, 9),
    (1, 1, 1, 3): (9, 1, 1, 10),
    (1, 1, 2, 2): (24, 1, 1, 11),
    (1, 1, 2, 3): (18, 1, 1, 9),
    (1, 1, 4, 2): (48, 1, 1, 10),
    (1, 1, 4, 3): (36, 1, 1, 11),
    (1, 1, 8, 3): (64, 1, 1, 9),
    (1, 2, 1, 2): (24, 2, 2, 10),
    (1, 2, 1, 3): (18, 2, 2, 11),
    (1, 2, 2, 2): (48, 2, 2, 9),
    (1, 2, 2, 3): (32, 2, 2, 10),
    (1, 2, 4, 3): (64, 2, 2, 11),
    (1, 3, 1, 2): (48, 3, 3, 9),
    (1, 3, 1, 3): (32, 4, 3, 10),
    (1, 3, 2, 3): (64, 4, 3, 11),
    (1, 4, 1, 2): (48, 4, 4, 9),
    (1, 4, 1, 3): (32, 4, 4, 10),
    (1, 4, 2, 3): (64, 4, 4, 11),
    (1, 5, 1, 2): (48, 6, 5, 9),
    (1, 5, 1, 3): (64, 8, 5, 10),
    (1, 6, 1, 2): (48, 6, 6, 11),
    (1, 6, 1, 3): (64, 8, 6, 9),
    (1, 7, 1, 2): (48, 8, 7, 10),
    (1, 7, 1, 3): (64, 8, 7, 11),
    (1, 8, 1, 2): (48, 8, 8, 9),
    (1, 8, 1, 3): (64, 8, 8, 10),
    (2, 5, 1, 2): (48, 12, 9, 11),
    (2, 5, 1, 3): (64, 16, 9, 9),
    (2, 6, 1, 2): (48, 12, 11, 10),
    (2, 6, 1, 3): (64, 16, 11, 11),
    (2, 7, 1, 2): (48, 16, 13, 9),
    (2, 7, 1, 3): (64, 16, 13, 10),
    (2, 8, 1, 2): (64, 16, 15, 11),
    (2, 8, 1, 3): (32, 16, 15, 9),
    (3, 6, 1, 1): (48, 24, 18, 10),
    (3, 6, 1, 2): (64, 32, 17, 11),
    (3, 6, 1, 3): (32, 32, 17, 9),
    (3, 7, 1, 1): (48, 24, 19, 10),
    (3, 7, 1, 2): (64, 32, 19, 11),
    (3, 7, 1, 3): (32, 32, 19, 9),
    (3, 8, 1, 1): (48, 24, 22, 10),
    (3, 8, 1, 2): (64, 32, 22, 11),
    (3, 8, 1, 3): (32, 32, 22, 9),
    (4, 7, 1, 1): (48, 48, 25, 10),
    (4, 7, 1, 2): (64, 32, 25, 11),
    (4, 7, 1, 3): (32, 32, 25, 9),
    (4, 8, 1, 1): (48, 48, 29, 10),
    (4, 8, 1, 2): (64, 32, 29, 11),
    (6, 6, 1, 1): (48, 48, 33, 9),
    (6, 6, 1, 2): (64, 64, 33, 10),
    (6, 7, 1, 1): (48, 48, 37, 11),
    (6, 7, 1, 2): (64, 64, 37, 9),
    (6, 8, 1, 1): (48, 48, 43, 10),
    (6, 8, 1, 2): (64, 64, 43, 11),
    (8, 7, 1, 1): (64, 64, 49, 9),
    (8, 8, 1, 1): (64, 64, 57, 10),
}
SINGLE_READ = {                                                      # class: (N, M, K, S)
    (1, 1, False, False, False): (32, 16, 1, 127),
    (1, 1, False, False, True): (32, 16, 1, 122),
    (1, 1, False, True, False): (24, 12, 1, 125),
    (1, 1, False, True, True): (24, 12, 1, 123),
    (1, 1, True, False, False): (96, 48, 1, 126),
    (1, 1, True, False, True): (96, 48, 1, 121),
    (1, 1, True, True, False): (72, 36, 1, 127),
    (1, 1, True, True, True): (72, 36, 1, 122),
    (2, 1, False, False, False): (32, 16, 2, 125),
    (2, 1, False, False, True): (32, 16, 2, 123),
    (2, 1, False, True, False): (24, 12, 2, 126),
    (2, 1, False, True, True): (24, 12, 2, 121),
    (2, 1, True, False, False): (96, 48, 2, 127),
    (2, 1, True, False, True): (96, 48, 2, 122),
    (2, 1, True, True, False): (72, 36, 2, 125),
    (2, 1, True, True, True): (72, 36, 2, 123),
    (4, 1, False, False, False): (32, 16, 3, 126),
    (4, 1, False, False, True): (32, 16, 3, 121),
    (4, 1, False, True, False): (24, 12, 3, 127),
    (4, 1, False, True, True): (24, 12, 3, 122),
    (4, 1, True, False, False): (96, 48, 3, 125),
    (4, 1, True, False, True): (96, 48, 3, 123),
    (4, 1, True, True, False): (72, 36, 3, 126),
    (4, 1, True, True, True): (72, 36, 3, 121),
    (8, 1, False, False, False): (32, 16, 5, 127),
    (8, 1, False, False, True): (32, 16, 5, 122),
    (8, 1, False, True, False): (24, 12, 5, 125),
    (8, 1, False, True, True): (24, 12, 5, 123),
    (8, 1, True, False, False): (96, 48, 5, 126),
    (8, 1, True, False, True): (96, 48, 5, 121),
    (8, 1, True, True, False): (72, 36, 5, 127),
    (8, 1, True, True, True): (72, 36, 5, 122),
    (8, 2, False, False, False): (32, 16, 9, 125),
    (8, 2, False, False, True): (32, 16, 9, 123),
    (8, 2, False, True, False): (24, 12, 9, 126),
    (8, 2, False, True, True): (24, 12, 9, 121),
    (8, 2, True, False, False): (96, 48, 9, 127),
    (8, 2, True, False, True): (96, 48, 9, 122),
    (8, 2, True, True, False): (72, 36, 9, 125),
    (8, 2, True, True, True): (72, 36, 9, 123),
    (8, 4, False, False, False): (32, 32, 17, 126),
    (8, 4, False, False, True): (32, 32, 17, 121),
    (8, 4, False, True, False): (24, 24, 17, 127),
    (8, 4, False, True, True): (24, 24, 17, 122),
    (8, 4, True, False, False): (96, 48, 17, 125),
    (8, 4, True, False, True): (96, 48, 17, 123),
    (8, 4, True, True, False): (72, 36, 17, 126),
    (8, 4, True, True, True): (72, 36, 17, 121),
}
FOLD = {                                                             # class: (N, M, S)
    (0, False, True): (6, 6, 3),
    (0, True, False): (96, 32, 2),
    (0, True, True): (24, 12, 1),
    (1, False, True): (6, 6, 7),
    (1, True, False): (48, 16, 6),
    (1, True, True): (12, 6, 5),
    (2, False, True): (4, 4, 11),
    (2, True, False): (24, 8, 10),
    (2, True, True): (6, 6, 9),
    (3, False, True): (2, 2, 19),
    (3, True, False): (8, 8, 18),
    (3, True, True): (6, 6, 17),
    (4, False, True): (1, 1, 35),
    (4, True, False): (8, 8, 34),
    (4, True, True): (6, 6, 33),
    (5, False, False): (6, 6, 270339),
    (5, False, True): (12, 6, 270338),
    (5, True, False): (6, 6, 65),
    (5, True, True): (12, 6, 67),
}
BATCH_ENCODE = {                                                     # class: (N, M, S)
    (1, 1, 8, False, False): (8, 1, 13),
    (1, 1, 8, False, True): (6, 1, 14),
    (1, 1, 8, True, False): (64, 1, 15),
    (1, 1, 8, True, True): (36, 1, 13),
    (1, 2, 4, False, False): (16, 2, 14),
    (1, 2, 4, False, True): (12, 2, 15),
    (1, 2, 4, True, False): (64, 2, 13),
    (1, 2, 4, True, True): (36, 2, 14),
    (1, 3, 2, False, True): (24, 3, 15),
    (1, 3, 2, True, True): (48, 3, 13),
    (1, 4, 2, False, False): (32, 4, 14),
    (1, 4, 2, False, True): (24, 4, 15),
    (1, 4, 2, True, False): (64, 4, 13),
    (1, 4, 2, True, True): (48, 4, 14),
    (1, 6, 1, False, True): (48, 6, 15),
    (1, 8, 1, False, False): (64, 8, 13),
    (1, 8, 1, False, True): (48, 8, 14),
    (2, 6, 1, False, True): (48, 12, 15),
    (2, 8, 1, False, False): (64, 16, 13),
    (2, 8, 1, False, True): (48, 16, 14),
    (3, 3, 2, False, True): (18, 9, 15),
    (3, 3, 2, True, True): (36, 9, 13),
    (3, 6, 1, False, True): (36, 18, 14),
    (3, 8, 1, False, True): (48, 24, 15),
    (4, 8, 1, False, False): (64, 32, 13),
    (4, 8, 1, False, True): (32, 32, 14),
    (6, 6, 1, False, True): (36, 36, 15),
    (6, 8, 1, False, True): (48, 48, 13),
    (8, 8, 1, False, False): (64, 64, 14),
}
UPDATE = {                                                           # class: (N, M, k, S)
    (False, False, False, False, False): (32, 32, 32, 127),
    (False, False, False, False, True): (32, 32, 1, 126),
    (False, False, False, True, False): (64, 32, 64, 125),
    (False, False, False, True, True): (64, 32, 33, 127),
    (False, False, True, False, False): (32, 32, 32, 122),
    (False, False, True, False, True): (32, 32, 1, 121),
    (False, False, True, True, False): (64, 32, 64, 123),
    (False, False, True, True, True): (64, 32, 33, 122),
    (False, True, False, False, False): (32, 16, 32, 125),
    (False, True, False, False, True): (1, 1, 1, 127),
    (False, True, False, True, False): (64, 16, 64, 126),
    (False, True, False, True, True): (36, 18, 33, 125),
    (False, True, True, False, False): (32, 16, 32, 123),
    (False, True, True, False, True): (1, 1, 1, 122),
    (False, True, True, True, False): (64, 16, 64, 121),
    (False, True, True, True, True): (36, 18, 33, 123),
    (True, False, False, False, False): (64, 64, 32, 126),
    (True, False, False, False, True): (64, 64, 1, 125),
    (True, False, False, True, False): (64, 64, 64, 127),
    (True, False, False, True, True): (64, 64, 33, 126),
    (True, False, True, False, False): (64, 64, 32, 121),
    (True, False, True, False, True): (64, 64, 1, 123),
    (True, False, True, True, False): (64, 64, 64, 122),
    (True, False, True, True, True): (64, 64, 33, 121),
    (True, True, False, False, False): (36, 36, 32, 127),
    (True, True, False, False, True): (36, 36, 1, 126),
    (True, True, False, True, False): (72, 72, 64, 125),
    (True, True, False, True, True): (36, 36, 33, 127),
    (True, True, True, False, False): (36, 36, 32, 122),
    (True, True, True, False, True): (36, 36, 1, 121),
    (True, True, True, True, False): (72, 72, 64, 123),
    (True, True, True, True, True): (36, 36, 33, 122),
}
