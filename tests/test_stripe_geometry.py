"""Every launch geometry of the stripe kernels against the encode by definition.

The launchers of the batched and the single degraded read, the scrub's fold, the batch encode and update's parity kernel each
switch on the shape of the call: template instance, warps per group, slices, ring stages, lanes per row.  tests/stripe_geometry.py
restates each rule and enumerates the geometry classes it reaches over the whole accepted domain, with one concrete call (a
witness) per class.
  CPU: every enumerated class has a witness and every witness maps to its class.
  GPU: the profiler's kernel records (template instance, grid, block, shared memory) of every witness are the ones predicted, so
       the restatement is the library's rule; and every witness computes, word for word, what tests/gfp_ref.py gives by
       definition, on adversarial stored words (x + P, 0xFFFFFFFF, all-P stripes that must come out all zero, all P - 1), with
       garbage in every row the call must not read and in every input pad word, and sentinels around every output."""
import json
import os
import re
import tempfile

import numpy as np
import pytest

import gfp_ref
import stripe_geometry as sg
from stripe_geometry import BATCH_ENCODE, BATCH_READ, FOLD, SINGLE_READ, UPDATE, cdiv
from test_update import C, P, SENTINEL, direct, i32


def ceil4(x):
    return (x + 3) // 4 * 4


# ---- CPU: the witnesses cover every class --------------------------------------------------------------------------------
def _in_family(N, limit):
    return N in sg.family(limit)


def _check_batch_read(cls, w):
    N, M, n_out, S = w
    return N in sg.ORDERS and N % M == 0 and 1 <= n_out <= M and S % 4 and sg.batch_read(N, n_out, 1, S).key == cls


def _check_single_read(cls, w):
    N, M, K, S = w
    return _in_family(N, 1 << 19) and N % M == 0 and 1 <= K <= min(M, 32) and S % 4 and sg.single_read(N, K, S).key == cls


def _check_fold(cls, w):
    N, M, S = w
    return _in_family(N, 1 << 19) and N % M == 0 and sg.fold(N + M, S).key == cls


def _check_batch_encode(cls, w):
    N, M, S = w
    return N in sg.ORDERS and N % M == 0 and S % 4 and sg.batch_encode(N, M, 1, S).key == cls


def _check_update(cls, w):
    N, M, k, S = w
    return _in_family(N, 1 << 19) and N % M == 0 and 1 <= k <= N and S % 4 and direct(N, M, k, S) and sg.update(M, k, S).key == cls


LAUNCHERS = {                                  # name: (witnesses, classes over the domain, witness check, expected class count)
    "batch_read": (BATCH_READ, sg.batch_read_classes, _check_batch_read, 56),
    "single_read": (SINGLE_READ, sg.single_read_classes, _check_single_read, 48),
    "fold": (FOLD, sg.fold_classes, _check_fold, 19),
    "batch_encode": (BATCH_ENCODE, sg.batch_encode_classes, _check_batch_encode, 29),
    "update": (UPDATE, sg.update_classes, _check_update, 32),
}


@pytest.mark.parametrize("name", list(LAUNCHERS), ids=["%s: %d of %d classes" % (k, len(v[0]), v[3]) for k, v in LAUNCHERS.items()])
def test_witnesses_cover_every_class(name):
    """The witness table names exactly the classes the launcher reaches over the accepted domain, one call each, and each call is
    in the domain (S % 4 != 0 wherever the class allows it) and maps to the class it claims"""
    witnesses, classes, check, count = LAUNCHERS[name]
    reached = classes()
    assert len(reached) == count, (name, len(reached), sorted(reached))
    assert sorted(witnesses) == sorted(reached), (name, set(reached) ^ set(witnesses))
    wrong = [(cls, w) for cls, w in witnesses.items() if not check(cls, w)]
    assert not wrong, (name, wrong)


def test_batch_read_classes_include_the_partial_warp_groups_and_single_slot_rings():
    """The classes where W U > n_out skips outputs in the last warp (U = 6 and 8 among them) and every single-slot ring are
    witnessed with such calls"""
    guarded = {cls: w for cls, w in BATCH_READ.items() if cls[0] * cls[1] > w[2]}
    assert {cls[0] for cls in guarded} >= {2, 3, 4, 6, 8}, sorted(guarded)
    assert sum(1 for cls in BATCH_READ if cls[3] == 1) == 10


SM_SHARED = 228 << 10                                               # shared memory of one H100 SM


def ctas_per_sm(L):
    """An upper bound on the CTAs of launch L resident on one SM: 8 of 256 threads, or as many as their shared memory allows
    (1 KiB per CTA reserved by the runtime)"""
    return min(2048 // L.block, SM_SHARED // (L.smem + sg.STATIC_SMEM[L.kernel.split("<")[0]] + 1024))


def batch_read_size(N, n_out, S, num_sms):
    """B for a witness of the batched read: however many CTAs share an SM, every CTA runs at least stages + 2 tiles, so each ring
    slot is refilled while the others are in flight, and the last tile is partial"""
    L = sg.batch_read(N, n_out, 1, S)
    items, stages, s4 = L.info["items"], L.key[3], cdiv(S, 4)
    n_tiles = ctas_per_sm(L) * num_sms * (stages + 2) + 1
    B = cdiv((n_tiles - 1) * items + items // 2, s4)
    while B * s4 % items == 0:
        B += 1
    return B


def test_batch_read_cases_wrap_the_ring_and_end_on_a_partial_tile():
    for (U, W, slices, stages), (N, M, n_out, S) in BATCH_READ.items():
        B = batch_read_size(N, n_out, S, sg.H100_SMS)
        L = sg.batch_read(N, n_out, B, S)
        assert L.info["n_items"] % L.info["items"] and L.info["n_tiles"] // (ctas_per_sm(L) * sg.H100_SMS) >= stages + 2, (N, M, n_out, S, B)


# ---- GPU: adversarial stripes, layouts with garbage and sentinels -------------------------------------------------------
def adversarial(R, B, S, gen):
    """Canonical words [R, B, S]: stripe b % 4 = 0 all zero, 1 all P - 1, 2 words below 2^32 - P (every 7th one 2^32 - P - 1),
    3 random"""
    import torch
    x = torch.randint(0, P, (R, B, S), device="cuda", generator=gen, dtype=torch.int64)
    small = torch.randint(0, C, (R, B, S), device="cuda", generator=gen, dtype=torch.int64)
    small[..., ::7] = C - 1
    kind = (torch.arange(B, device="cuda") % 4)[None, :, None]
    return torch.where(kind == 0, 0, torch.where(kind == 1, P - 1, torch.where(kind == 2, small, x)))


def stored(x, gen):
    """Canonical words as stored: x + P where that fits in 32 bits, always for 0 (an all-zero stripe is stored as all P) and for
    2^32 - P - 1 (stored as 0xFFFFFFFF), at random elsewhere"""
    import torch
    up = (x < C) & ((x == 0) | (x == C - 1) | (torch.rand(x.shape, device="cuda", generator=gen) < 0.5))
    return i32(x + up.to(torch.int64) * P)


def columns(R, S, gen):
    """Canonical words [R, S] of one stripe whose column quarters are the four kinds of adversarial()"""
    q = cdiv(S, 4)
    return adversarial(R, 4, q, gen).reshape(R, 4 * q)[:, :S].contiguous()


def encode_by_definition(data, rows, D):
    """Parity blocks `rows` of canonical data [N, ...] (every trailing index a column), by definition: [len(rows), ...]"""
    N = data.shape[0]
    if not len(rows):
        return data[:0]
    out = gfp_ref.encode_rows(data.reshape(N, -1), [D * j for j in rows])
    return out.reshape(len(rows), *data.shape[1:])


def garbage(shape, gen):
    import torch
    return torch.randint(-(1 << 31), 1 << 31, shape, dtype=torch.int32, device="cuda", generator=gen)


def words(t):
    import torch
    return t.to(torch.int64) & 0xFFFFFFFF


GUARD = 64


def buffer(shape, S, gen=None):
    """A flat buffer and a view of it: [B, R, S] (or [R, S]) rows of ceil4(S) + 4 words, 4 more words between stripes, GUARD words
    before and after.  Every word outside the view holds random garbage (an input: a read of a pad word would change the result)
    or, without gen, the sentinel (an output: a write outside the rows would show)."""
    import torch
    pitch = ceil4(S) + 4
    B, R = shape if len(shape) == 2 else (1, shape[0])
    stride = R * pitch + 4
    n = 2 * GUARD + B * stride
    flat = garbage((n,), gen) if gen is not None else torch.full((n,), SENTINEL, dtype=torch.int32, device="cuda")
    size, strides = ((B, R, S), (stride, pitch, 1)) if len(shape) == 2 else ((R, S), (pitch, 1))
    return flat, flat.as_strided(size, strides, GUARD)


def with_view(flat, view, value):
    """A copy of flat with `value` (canonical int64 words) in the words of `view`"""
    out = flat.clone()
    out.as_strided(view.shape, view.stride(), view.storage_offset() - flat.storage_offset()).copy_(i32(value))
    return out


def read_pattern(N, M, n_out):
    """(lost data, lost parity, wanted parity) of n_out wanted blocks: ceil(n_out / 2) lost data blocks spread over the stripe,
    the rest wanted parity blocks; the lowest parity blocks are lost (one more, unwanted, where M allows), so J skips them"""
    a = (n_out + 1) // 2
    nwp = n_out - a
    extra = 1 if a + nwp < M else 0
    lost_p = list(range(nwp + extra))
    return [i * N // a for i in range(a)], lost_p, lost_p[extra:]


def rows_J(M, a, lost_p):
    return [j for j in range(M) if j not in lost_p][:a]


# -- the batched read
def batch_read_case(fecc, N, M, n_out, S, seed):
    """(call, check) of one witness of the batched read"""
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(seed)
    B = batch_read_size(N, n_out, S, fecc.lib().fastecc_b200_num_sms())
    lost_d, lost_p, want_p = read_pattern(N, M, n_out)
    J = rows_J(M, len(lost_d), lost_p)
    data = adversarial(N, B, S, gen)
    par = encode_by_definition(data, J, N // M)
    dflat, dview = buffer((B, N), S, gen)
    pflat, pview = buffer((B, M), S, gen)
    oflat, oview = buffer((B, n_out), S)
    dview.copy_(stored(data, gen).permute(1, 0, 2))
    for lost in lost_d:                                                   # garbage stays in the lost rows
        dview[:, lost] = garbage((B, S), gen)
    for k, j in enumerate(J):                                             # and in every parity row outside J
        pview[:, j] = stored(par[k], gen)
    keep = dflat.clone(), pflat.clone()
    del par

    def call():
        fecc.rs_reconstruct_batch_dev(dview, pview, lost_d, lost_p, lost_d, want_p, out=oview)

    def check():
        torch.cuda.synchronize()
        assert torch.equal(dflat, keep[0]) and torch.equal(pflat, keep[1]), "the batched read wrote into its input"
        want = torch.cat([data[lost_d], encode_by_definition(data, want_p, N // M)]).permute(1, 0, 2)
        got = words(oview)
        bad = (got != want).nonzero()
        assert not len(bad), ("wrong words", len(bad), bad[:4].tolist(), got[tuple(bad[0])].item(), want[tuple(bad[0])].item())
        assert torch.equal(oflat, with_view(torch.full_like(oflat, SENTINEL), oview, want)), "a word outside the output rows changed"
        assert not bool(got[0::4].any()), "an all-zero stripe must come out all zero"
    return call, check, B


# -- the single read
def single_read_case(fecc, N, M, K, S, seed):
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(seed)
    lost_d, lost_p, want_p = read_pattern(N, M, K)
    J = rows_J(M, len(lost_d), lost_p)
    data = columns(N, S, gen)
    dflat, dview = buffer((N,), S, gen)
    pflat, pview = buffer((M,), S, gen)
    oflat, oview = buffer((K,), S)
    dview.copy_(stored(data, gen))
    for lost in lost_d:
        dview[lost] = garbage((S,), gen)
    if J:
        pview[J] = stored(encode_by_definition(data, J, N // M), gen)
    keep = dflat.clone(), pflat.clone()

    def call():
        fecc.rs_reconstruct_dev(dview, pview, lost_d, lost_p, lost_d, want_p, out=oview)

    def check():
        torch.cuda.synchronize()
        assert torch.equal(dflat, keep[0]) and torch.equal(pflat, keep[1]), "the read wrote into its input"
        want = torch.cat([data[lost_d], encode_by_definition(data, want_p, N // M)])
        assert torch.equal(words(oview), want)
        assert torch.equal(oflat, with_view(torch.full_like(oflat, SENTINEL), oview, want)), "a word outside the output rows changed"
        assert not bool(words(oview)[:, :cdiv(S, 4)].any()), "the all-zero columns must come out all zero"
    return call, check


# -- the batch encode
def batch_encode_case(fecc, N, M, S, seed):
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(seed)
    L = sg.batch_encode(N, M, 1, S)
    s4 = cdiv(S, 4)
    B = cdiv(3 * L.info["items"] + 5, s4) | 1                           # three CTAs and a partial fourth
    while B * s4 % L.info["items"] == 0:
        B += 2
    data = adversarial(N, B, S, gen)
    dflat, dview = buffer((B, N), S, gen)
    pflat, pview = buffer((B, M), S)
    dview.copy_(stored(data, gen).permute(1, 0, 2))
    keep = dflat.clone()

    def call():
        fecc.rs_encode_batch_dev(dview, pview)

    def check():
        torch.cuda.synchronize()
        assert torch.equal(dflat, keep), "the batch encode wrote into the data"
        want = encode_by_definition(data, range(M), N // M).permute(1, 0, 2)
        assert torch.equal(words(pview), want)
        assert torch.equal(pflat, with_view(torch.full_like(pflat, SENTINEL), pview, want)), "a word outside the parity rows changed"
        assert not bool(want[0::4].any()) and not bool(words(pview)[0::4].any())
    return call, check, B


# -- update
def update_case(fecc, N, M, k, S, seed):
    import torch
    gen = torch.Generator(device="cuda"); gen.manual_seed(seed)
    changed = [i * N // k for i in range(k)]
    data, new = columns(N, S, gen), columns(k, S, gen).flip(1).contiguous()
    dflat, dview = buffer((N,), S, gen)
    pflat, pview = buffer((M,), S, gen)
    nflat, nview = buffer((k,), S, gen)
    dview.copy_(stored(data, gen))
    pview.copy_(stored(encode_by_definition(data, range(M), N // M), gen))
    nview.copy_(stored(new, gen))
    after = data.clone()
    after[changed] = new
    keep_d, keep_n, keep_p = dflat.clone(), nflat.clone(), pflat.clone()

    def call():
        fecc.rs_update_dev(dview, pview, changed, nview)

    def check():
        torch.cuda.synchronize()
        want_d, pitch = keep_d.clone(), dview.stride(0)
        for r, i in enumerate(changed):
            want_d[GUARD + i * pitch:GUARD + i * pitch + S] = i32(new[r])
        assert torch.equal(dflat, want_d), "the changed rows are not the canonical new blocks, or another word changed"
        assert torch.equal(nflat, keep_n), "update wrote into the new rows"
        want_p = encode_by_definition(after, range(M), N // M)
        assert torch.equal(words(pview), want_p)
        assert torch.equal(pflat, with_view(keep_p, pview, want_p)), "a word outside the parity rows changed"
    return call, check


# ---- GPU: the profiler's kernel records are the predicted launches ------------------------------------------------------
def kernel_records(fn, pattern):
    """(kernel, grid, block, shared memory) of every kernel whose name matches `pattern` that fn() launches, in launch order,
    from the profiler's trace; None when the trace holds no kernel records at all"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    kernels = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    if not kernels:
        return None
    out = []
    for e in kernels:
        m = re.search(pattern, e["name"])
        if m:
            a = e["args"]
            out.append((m.group(1), tuple(a["grid"]), tuple(a["block"]), a["shared memory"]))
    return out


def launch_of(call, pattern, what, tries=3):
    """The one kernel record matching `pattern` of call() (which may be repeated), profiled on its own.  The activity buffers
    occasionally come back without a record, so a call is profiled up to `tries` times; a trace that never holds any kernel
    record skips the test with that reason."""
    recs = None
    for _ in range(tries):
        recs = kernel_records(call, pattern)
        if recs is not None and len(recs) == 1:
            return recs[0]
    if recs is None:
        pytest.skip("the profiler trace holds no kernel records on this machine")
    assert len(recs) == 1, (what, recs)


def base(kernel):
    return kernel.split("<")[0]


def expect_launch(rec, L, what):
    kernel, grid, block, smem = rec
    assert kernel == L.kernel, (what, rec, L)
    assert block == (L.block, 1, 1), (what, rec, L)
    assert smem == L.smem + sg.STATIC_SMEM[base(L.kernel)], (what, rec, L)
    assert grid[1:] == (1, 1), (what, rec)
    return grid[0]


@pytest.mark.gpu
def test_batch_read_launches_are_the_restated_rule(fecc):
    """Instance, block and shared memory of every witness as predicted; the grid is capped at a multiple of the SM count, and
    every CTA runs at least stages + 2 tiles"""
    sms = fecc.lib().fastecc_b200_num_sms()
    for i, (cls, (N, M, n_out, S)) in enumerate(BATCH_READ.items()):
        call, _, B = batch_read_case(fecc, N, M, n_out, S, 100 + i)
        L = sg.batch_read(N, n_out, B, S)
        assert L.key == cls
        grid = expect_launch(launch_of(call, r"\b(batch_reconstruct_kernel<\d+u>)\(", cls), L, cls)
        n_tiles, stages = L.info["n_tiles"], cls[3]
        assert grid <= n_tiles and grid % sms == 0, (cls, grid, n_tiles)
        assert n_tiles // grid >= stages + 2, ("a CTA runs fewer than stages + 2 tiles", cls, grid, n_tiles)
        assert L.info["n_items"] % L.info["items"], cls


@pytest.mark.gpu
def test_single_read_launches_are_the_restated_rule(fecc):
    sms = fecc.lib().fastecc_b200_num_sms()
    for i, (cls, (N, M, K, S)) in enumerate(SINGLE_READ.items()):
        call, _ = single_read_case(fecc, N, M, K, S, 200 + i)
        L = sg.single_read(N, K, S, sms)
        assert L.key == cls, ("the witness falls into another class on %d SMs" % sms, cls, L.key)
        rec = launch_of(call, r"\b(reconstruct_sum_kernel<\d+u>)\(", cls)
        assert expect_launch(rec, L, cls) == L.info["grid"], (cls, rec, L)


@pytest.mark.gpu
def test_fold_launches_are_the_restated_rule(fecc):
    """The plain and the degraded scrub of every witness"""
    from fastecc_b200.decoder import Repair
    sms = fecc.lib().fastecc_b200_num_sms()
    for i, (cls, (N, M, S)) in enumerate(FOLD.items()):
        d, p, _ = scrub_stripe(fecc, N, M, S, 300 + i)
        L = sg.fold(N + M, S, sms)
        assert L.key == cls, ("the witness falls into another class on %d SMs" % sms, cls, L.key)
        rec = launch_of(lambda: fecc.rs_scrub_dev(d, p), r"\b(scrub_fold_kernel)\(", cls)
        assert expect_launch(rec, L, cls) == L.info["grid"], (cls, rec, L)
        if M >= 2:
            rep = Repair(N, M, [N // 2], [])
            try:
                rec = launch_of(lambda: rep.scrub(d, p), r"\b(degraded_fold_kernel)\(", cls)
            finally:
                rep.close()
            L = sg.fold(N + M, S, sms, degraded=True)
            assert expect_launch(rec, L, cls) == L.info["grid"], (cls, rec, L)


@pytest.mark.gpu
def test_batch_encode_launches_are_the_restated_rule(fecc):
    for i, (cls, (N, M, S)) in enumerate(BATCH_ENCODE.items()):
        call, _, B = batch_encode_case(fecc, N, M, S, 400 + i)
        L = sg.batch_encode(N, M, B, S)
        assert L.key == cls
        rec = launch_of(call, r"\b(batch_encode_kernel<\d+u>)\(", cls)
        assert expect_launch(rec, L, cls) == L.info["grid"], (cls, rec, L)


@pytest.mark.gpu
def test_update_launches_are_the_restated_rule(fecc):
    for i, (cls, (N, M, k, S)) in enumerate(UPDATE.items()):
        call, _ = update_case(fecc, N, M, k, S, 500 + i)
        L = sg.update(M, k, S)
        rec = launch_of(call, r"\b(update_parity_kernel)\(", cls)
        assert expect_launch(rec, L, cls) == L.info["grid"], (cls, rec, L)


# ---- GPU: every witness against the encode by definition ----------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cls", list(BATCH_READ), ids=str)
def test_batch_read_witness(fecc, cls):
    N, M, n_out, S = BATCH_READ[cls]
    call, check, _ = batch_read_case(fecc, N, M, n_out, S, 100 + list(BATCH_READ).index(cls))
    call()
    check()


@pytest.mark.gpu
@pytest.mark.parametrize("cls", list(SINGLE_READ), ids=str)
def test_single_read_witness(fecc, cls):
    N, M, K, S = SINGLE_READ[cls]
    call, check = single_read_case(fecc, N, M, K, S, 200 + list(SINGLE_READ).index(cls))
    call()
    check()


@pytest.mark.gpu
@pytest.mark.parametrize("cls", list(BATCH_ENCODE), ids=str)
def test_batch_encode_witness(fecc, cls):
    N, M, S = BATCH_ENCODE[cls]
    call, check, _ = batch_encode_case(fecc, N, M, S, 400 + list(BATCH_ENCODE).index(cls))
    call()
    check()


@pytest.mark.gpu
@pytest.mark.parametrize("cls", list(UPDATE), ids=str)
def test_update_witness(fecc, cls):
    N, M, k, S = UPDATE[cls]
    call, check = update_case(fecc, N, M, k, S, 500 + list(UPDATE).index(cls))
    call()
    check()


# -- the fold: the plain and the degraded scrub
def scrub_stripe(fecc, N, M, S, seed):
    """A clean stripe of raw words (x + P where that fits) in rows whose pad words hold garbage, its parity by definition"""
    import torch
    from test_scrub import padded
    gen = torch.Generator(device="cuda"); gen.manual_seed(seed)
    data = columns(N, S, gen)
    par = encode_by_definition(data, range(M), N // M)
    return padded(stored(data, gen)), padded(stored(par, gen)), gen


@pytest.mark.gpu
@pytest.mark.parametrize("cls", list(FOLD), ids=str)
def test_fold_witness(fecc, cls):
    """Clean; max_bad corrupted blocks located exactly; one more compared with the torch restatement of the scrub"""
    from fastecc_b200.decoder import Repair
    from test_scrub import CLEAN, LOCATED, corrupt_rows, mixed, padded, torch_scrub
    from test_scrub_degraded import survivors, torch_scrub_degraded
    N, M, S = FOLD[cls]
    seed = 300 + list(FOLD).index(cls)
    rng = np.random.default_rng(seed)
    data, parity, gen = scrub_stripe(fecc, N, M, S, seed)
    s = int(rng.integers(1 << 63))
    assert fecc.rs_scrub_dev(data, parity, min(M // 2, 2), s) == (CLEAN, [], [])
    max_bad = min(M // 2, 2)
    for t in sorted({max_bad, max_bad + 1} - {0}):
        d, p = padded(data), padded(parity)
        bd, bp = mixed(rng, N, M, t)
        corrupt_rows(d, bd, gen); corrupt_rows(p, bp, gen)
        got = fecc.rs_scrub_dev(d, p, max_bad, s)
        if t <= max_bad:
            assert got == (LOCATED, bd, bp), (t, bd, bp, got)
        else:
            assert got == torch_scrub(d, p, max_bad, s), (t, bd, bp, got)
    if M < 2:
        return
    lost_d = [N // 2]
    d = padded(data)
    d[lost_d[0]] = garbage((S,), gen)
    rep = Repair(N, M, lost_d, [])
    try:
        max_bad = min((M - 1) // 2, 2)
        assert rep.scrub(d, parity, max_bad, s) == (CLEAN, [], [])
        for t in sorted({max_bad, max_bad + 1} - {0}):
            if t > N + M - 1:
                continue
            dd, pp = padded(d), padded(parity)
            bd, bp = survivors(rng, N, M, lost_d, [], t)
            corrupt_rows(dd, bd, gen); corrupt_rows(pp, bp, gen)
            got = rep.scrub(dd, pp, max_bad, s)
            if t <= max_bad:
                assert got == (LOCATED, bd, bp), ("degraded", t, bd, bp, got)
            else:
                assert got == torch_scrub_degraded(dd, pp, lost_d, [], max_bad, s), ("degraded", t, bd, bp, got)
    finally:
        rep.close()
