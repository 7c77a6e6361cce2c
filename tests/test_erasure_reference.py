"""Erasure decoding (csrc/decode.cu) and stripe repair (csrc/repair.cu) against closed-form code words, without the library's
encoder.  Column c of a stripe is the polynomial z^m_c (m_c < N from special_values), so row x of its 2N-row code word is
rho^(x*m_c), rho = GF_Root(2N): data i is rho^(2*i*m_c) and parity j' of an M-block stripe is rho^((2*(N/M)*j'+1)*m_c)
(tests/gfp_ref.py).  Every recovered word is compared, chunk by chunk.

  CPU   the locator tree's transform orders restated from erasure_locator: leaves of 32 points, order 4d up to 2^20, beyond
        that the smallest order above the largest product degree min(2d, |E|).  The erasure counts of TREE reach each of the
        nine orders the rule can pick above 2^20, with |E| = L - 1 (the tightest product that does not alias) and |E| = L
        (one order up) for each.  codeword_rows against the encode by definition.
  GPU   decode: every band of TREE; structured loss sets (all data, all parity, halves, cosets, the rows an asymmetric encode
        never produced, runs across leaf boundaries, single rows, the empty set, counts at the leaf boundaries) from 2N = 2 to
        9 * 2^20, where the torch-level ErasurePattern must equal the C ABI pattern at powers of two; padded pitches, an out
        pitch above the code pitch, raw words x + P, one pattern on two streams.
        repair: 2^19, 3 * 2^19 and 9 * 2^19 data blocks at M from 1 to N, structured losses, data and parity at different
        pitches (parity below data), sentinels in every pad word, raw words >= P in the surviving rows (whole buffers compared).
        The storage pipeline: bytes -> words -> asymmetric encode -> loss -> repair and 2N-row decode -> bytes.
        In a child process each: a repair in three column chunks (15 GiB of tensors beside the library's 4 GiB workspace and
        its encode buffers; skipped with the reason printed below 24 GiB free), and a repair, a decode and
        a mixed encode enqueued on three streams with no host synchronisation in between.
The run as a script (`python tests/test_erasure_reference.py chunks|streams`) is the child process of the last two."""
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if __name__ == "__main__":
    sys.path[:0] = [ROOT, HERE]

import gfp_ref as R                           # noqa: E402
import test_full_size_reference as F          # noqa: E402   buffer, fill, check, values (closed-form degrees)

P = R.P
C = (1 << 32) - P                             # words below C can be stored raw as x + P
DEV = "cuda"
SENT = 0x5EED5EED
LEAF = 32                                     # points per leaf polynomial of the locator tree
MAX_ORDER = 1 << 20                           # largest power-of-two transform order


# ==== the locator tree's transform orders ==================================================================================
def order_above(t):
    """The smallest transform order of the library (2^a, 3 * 2^a or 9 * 2^a, 2^a <= 2^20) above t."""
    return min(r << a for r in (1, 3, 9) for a in range(21) if r << a > t)


def tree_orders(me):
    """The transform order of every level of the product tree over me erased points: the leaves hold 32 points each (their
    count rounded up to a power of two), a level multiplies pairs of degree <= d at order 4d while 4d <= 2^20, beyond that
    at the smallest order above the largest product degree min(2d, me)."""
    groups = 1
    while groups * LEAF < me:
        groups *= 2
    d, out = LEAF, []
    while groups > 1:
        out.append(4 * d if 4 * d <= MAX_ORDER else order_above(min(2 * d, me)))
        groups //= 2
        d *= 2
    return out


# (code word N, |E|, the orders of the levels with 4d > 2^20)
TREE = [(9 << 16, (1 << 19) + 1, [9 << 16]), (9 << 16, 589823, [9 << 16]), (9 << 16, 589824, [3 << 18]),
        (3 << 18, 786431, [3 << 18]), (3 << 18, 786432, [1 << 20]),
        (9 << 17, (1 << 20) - 1, [1 << 20]), (9 << 17, 1 << 20, [9 << 17]),
        (9 << 17, 1179647, [9 << 17, 9 << 17]), (9 << 17, 1179648, [9 << 17, 3 << 19]),
        (3 << 19, 1572863, [9 << 17, 3 << 19]), (3 << 19, 1572864, [9 << 17, 9 << 18]),
        (9 << 18, 2359295, [9 << 17, 9 << 18, 9 << 18]), (9 << 18, 2359296, [9 << 17, 9 << 18, 3 << 20]),
        (9 << 19, 3145727, [9 << 17, 9 << 18, 3 << 20]), (9 << 19, 3145728, [9 << 17, 9 << 18, 9 << 19]),
        (9 << 19, 4718591, [9 << 17, 9 << 18, 9 << 19, 9 << 19]), (9 << 19, 4718592, [9 << 17, 9 << 18, 9 << 19, 9 << 20])]
ABOVE_2P20 = [9 << 16, 3 << 18, 1 << 20, 9 << 17, 3 << 19, 9 << 18, 3 << 20, 9 << 19, 9 << 20]


def levels_above(me):
    return [o for k, o in enumerate(tree_orders(me)) if 4 * (LEAF << k) > MAX_ORDER]


def test_tree_orders_confirm_the_table():
    for N, me, top in TREE:
        assert me <= N and F.order_parts(N)[0] > 1, (N, me)
        assert levels_above(me) == top, (N, me, tree_orders(me))
        assert all(o > min(2 * (LEAF << k), me) for k, o in enumerate(tree_orders(me))), (N, me)      # no product aliases
    assert all(not levels_above(me) for me in (1, 32, 33, 1 << 18, (1 << 19) - 1, 1 << 19))             # every code word 2N <= 2^20


def test_tree_cases_reach_every_order_above_2p20():
    # the rule picks order_above(t) for 2^19 < t <= 9 * 2^19: exactly these nine orders
    picks = sorted({order_above(t) for t in [(1 << 19) + 1] + [L + e for L in ABOVE_2P20 for e in (-1, 0)] if (1 << 19) < t <= 9 << 19})
    assert picks == sorted(ABOVE_2P20)
    assert {o for _, me, _ in TREE for o in levels_above(me)} == set(ABOVE_2P20)
    counts = {me for _, me, _ in TREE}
    for L in ABOVE_2P20:
        if L > 9 << 19:
            continue
        assert L - 1 in counts and L in counts, L
        assert tree_orders(L - 1)[-1] == L                       # product degree L - 1 at order L
        assert tree_orders(L)[-1] == order_above(L) > L          # degree L moves one order up


@pytest.mark.parametrize("N", [1, 2, 4, 8, 32, 256, 3, 6, 12, 96, 9, 18, 72, 288])
def test_codeword_rows_equal_the_encode_by_definition(N):
    degs = F.values(N, 8, seed=3)
    cw = R.codeword_rows(N, degs)
    data = R.monomial_data(N, degs)
    assert cw.shape == (2 * N, 8)
    assert torch.equal(cw[0::2], data)
    assert torch.equal(cw[1::2], R.encode_rows(data, range(N)))
    rows = [0, N, 2 * N - 1]
    assert torch.equal(R.codeword_rows(N, degs, rows), cw[rows])


# ==== GPU helpers =========================================================================================================
def raw(x):
    """x + P wherever that still fits 32 bits"""
    return torch.where(x < C, x + P, x)


def code_word(N, degs, pitch=None):
    """The 2N-row code word of the monomial stripe as a [2N, S] view of a buffer at `pitch` with the sentinel in its pads."""
    t = F.buffer(2 * N, len(degs), pitch, fill=SENT)
    F.fill(t, lambda x: R.codeword_rows(N, degs, x, DEV))
    return t


def garbage(n, S, seed):
    g = torch.Generator(device=DEV); g.manual_seed(seed)
    return torch.randint(-(1 << 31), 1 << 31, (n, S), device=DEV, generator=g, dtype=torch.int64).to(torch.int32)


def decode_case(N, degs, pristine, erased, what, torch_level=False, seed=0):
    """Garbage in the erased rows of a copy of `pristine`, recover them through the C ABI pattern (and the torch-level
    ErasurePattern), every recovered word against the closed form."""
    from fastecc_b200 import decoder
    n2, S = 2 * N, len(degs)
    E = np.asarray(erased, dtype=np.int64)
    Ed = torch.from_numpy(E).to(DEV)
    code = pristine.clone()
    if E.size:
        code[Ed] = garbage(E.size, S, seed)
    pat = decoder.CErasurePattern(n2, E, mixed=True)
    rec = pat.recover(code)
    pat.close()
    assert rec.shape == (E.size, S), what
    F.check(rec, lambda i: R.codeword_rows(N, degs, Ed[i], DEV), what)
    if torch_level:
        code = pristine.clone()
        if E.size:
            code[Ed] = -1
        rec2 = decoder.ErasurePattern(n2, Ed, DEV).recover(code)
        assert torch.equal(rec2, rec), what + ": the torch-level ErasurePattern differs from the C ABI pattern"


def order_divisors(n):
    r, L = F.order_parts(n)
    return sorted(q << a for q in (1, 3, 9) if r % q == 0 for a in range(L.bit_length()))


def structured_losses(N, seed):
    """(name, ascending rows of the 2N-row code word) for the structured loss sets of a code word of N data blocks."""
    from fastecc_b200 import decoder
    n2, ar = 2 * N, np.arange
    rng = np.random.default_rng(seed)
    sets = [("all data rows", ar(0, n2, 2)), ("all parity rows", ar(1, n2, 2)), ("the first N rows", ar(N)),
            ("the last N rows", ar(N, n2)), ("row 0", ar(1)), ("row 2N-1", ar(n2 - 1, n2)), ("no row", ar(0))]
    for s in order_divisors(n2):
        if s >= 2:
            sets += [("coset %d + %d k" % (a, s), ar(a, n2, s)) for a in sorted({0, s - 1})]
    for M in sorted({m for m in (1, 3, 9, N // 8, N // 3, N) if m >= 1 and N % m == 0}):
        ld = np.sort(rng.choice(N, M // 2, replace=False))
        lp = np.sort(rng.choice(M, M - M // 2, replace=False))
        sets.append(("never produced by the encode into M=%d" % M, np.asarray(decoder.asym_erasures(N, M, ld, lp))))
    for n in sorted({33, 65, 1025, (LEAF << max(0, ((N - 1) // LEAF).bit_length() - 1)) + 1}):
        if n <= N:                                               # a run across leaf boundaries around row N
            s0 = max(0, min(n2 - n, N - 16))
            sets.append(("run of %d from %d" % (n, s0), ar(s0, s0 + n)))
    for n in [1, 31, 32, 33] + [(LEAF << k) + e for k in range(1, 20) for e in (-1, 1)]:
        if n <= N:
            sets.append(("%d random rows" % n, np.sort(rng.choice(n2, n, replace=False))))
    return sets


def recover_into(pat, code, S, pitch, out, out_pitch):
    """fastecc_b200_rs_decode_recover on raw pointers: code rows at `pitch`, out rows at `out_pitch`."""
    import fastecc_b200 as fe
    fe._check(fe.lib().fastecc_b200_rs_decode_recover(pat._h, code.data_ptr(), S, pitch, out.data_ptr(), out_pitch,
                                                      torch.cuda.current_stream().cuda_stream))


def stripe(N, M, S, dpitch, ppitch, degs):
    """The monomial stripe in one allocation, the M parity rows (at ppitch) below the N data rows (at dpitch); every word
    below C stored raw as x + P, the sentinel in every pad word.  Returns (flat buffer, [N, dpitch] data, [M, ppitch] parity)."""
    flat = torch.full((M * ppitch + N * dpitch,), SENT, dtype=torch.int32, device=DEV)
    parity, data = flat[:M * ppitch].view(M, ppitch), flat[M * ppitch:].view(N, dpitch)
    F.fill(data[:, :S], lambda i: raw(R.monomial_data(N, degs, i, DEV)))
    F.fill(parity[:, :S], lambda j: raw(R.monomial_parity(N, degs, j, DEV, N // M)))
    return flat, data, parity


def check_rows(buf, S, gen, lost, what):
    """Every word of buf's rows: gen(rows) in words [0, S) -- canonical in the rows where `lost` is set, raw (x + P where x < C)
    in the others -- and the sentinel in the pad words."""
    n, pitch = buf.shape
    for r0, r1 in F.row_chunks(n, pitch):
        i = torch.arange(r0, r1, dtype=torch.int64, device=DEV)
        x = gen(i)
        want = torch.full((r1 - r0, pitch), SENT, dtype=torch.int64, device=DEV)
        want[:, :S] = torch.where(lost[i, None], x, raw(x))
        got = R.as_words(buf[r0:r1])
        bad = got != want
        if bool(bad.any()):
            idx = bad.nonzero()[:4].tolist()
            detail = ["row %d word %d: got %d want %d" % (r0 + a, b, int(got[a, b]), int(want[a, b])) for a, b in idx]
            raise AssertionError("%s: %d of %d words differ in rows [%d, %d); %s" % (what, int(bad.sum()), bad.numel(), r0, r1, "; ".join(detail)))


def repair_case(N, M, S, degs, pristine, views, ld, lp, what):
    """Reset the stripe, garbage in the lost rows, repair, compare both whole buffers."""
    from fastecc_b200 import decoder
    flat, data, parity = views
    flat.copy_(pristine)
    ld, lp = np.asarray(ld, dtype=np.int64), np.asarray(lp, dtype=np.int64)
    lost_d = torch.zeros(N, dtype=torch.bool, device=DEV)
    lost_p = torch.zeros(M, dtype=torch.bool, device=DEV)
    if ld.size:
        lost_d[torch.from_numpy(ld).to(DEV)] = True
        data[torch.from_numpy(ld).to(DEV), :S] = -1
    if lp.size:
        lost_p[torch.from_numpy(lp).to(DEV)] = True
        parity[torch.from_numpy(lp).to(DEV), :S] = 0x7EADBEEF
    r = decoder.Repair(N, M, ld, lp)
    r.repair(data[:, :S], parity[:, :S])
    r.close()
    what = "%s (N=%d M=%d S=%d, %d data + %d parity lost)" % (what, N, M, S, ld.size, lp.size)
    check_rows(data, S, lambda i: R.monomial_data(N, degs, i, DEV), lost_d, what + ": data")
    check_rows(parity, S, lambda j: R.monomial_parity(N, degs, j, DEV, N // M), lost_p, what + ": parity")


def repair_losses(N, M, seed):
    """(name, lost data, lost parity): data [0, M); all parity; one residue class of the data mod N/M; data (N/M) j' with
    parity j' (adjacent rows 2i, 2i + 1 of the code word); at M = N the erasure counts of TREE that fit."""
    rng = np.random.default_rng(seed)
    D = N // M
    sets = [("data [0, M)", np.arange(M), []), ("all parity", [], np.arange(M)), ("data = %d mod %d" % (D - 1, D), np.arange(D - 1, N, D), [])]
    if M >= 2:
        j = np.sort(rng.choice(M, M // 2, replace=False))
        sets.append(("data D j' with parity j'", D * j, j))
    if M == N:
        for n in ((1 << 19) + 1, 1 << 20, 3145727, 4718591):
            if n <= N:
                sets.append(("%d blocks" % n, np.sort(rng.choice(N, n // 2, replace=False)), np.sort(rng.choice(N, n - n // 2, replace=False))))
    return sets


def child(mode, timeout=1800):
    torch.cuda.empty_cache()
    t0 = time.time()
    p = subprocess.run([sys.executable, os.path.abspath(__file__), mode], cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=timeout)
    print(p.stdout)
    print("child %s: %.1f s" % (mode, time.time() - t0))
    if p.returncode == 3:
        pytest.skip(p.stdout.strip().splitlines()[-1])
    assert p.returncode == 0, p.stdout[-6000:]
    return p.stdout


# ==== GPU: decode ===========================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("N,me,top", TREE, ids=["N=%d-E=%d" % (N, me) for N, me, _ in TREE])
def test_decode_every_band_of_the_locator_tree(fecc, N, me, top):
    """|E| random rows of the code word at the orders of TREE: the levels above 2^20 run at the orders `top`."""
    from fastecc_b200 import decoder
    S = 4 if N >= 9 << 18 else 8
    degs = F.values(N, S, seed=me)
    code = code_word(N, degs)
    g = torch.Generator(device=DEV); g.manual_seed(me)
    Ed = torch.sort(torch.randperm(2 * N, device=DEV, generator=g)[:me]).values
    code[Ed] = garbage(me, S, me)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    pat = decoder.CErasurePattern(2 * N, Ed.cpu().numpy(), mixed=True)
    torch.cuda.synchronize(); t1 = time.perf_counter()
    rec = pat.recover(code)
    torch.cuda.synchronize(); t2 = time.perf_counter()
    pat.close()
    print("N=%d |E|=%d tree orders above 2^20 %s: pattern %.0f ms, recover %.1f ms" % (N, me, top, 1e3 * (t1 - t0), 1e3 * (t2 - t1)))
    F.check(rec, lambda i: R.codeword_rows(N, degs, Ed[i], DEV), "decode N=%d |E|=%d" % (N, me))


STRUCT_N2 = [2, 4, 64, 1 << 11, 1 << 16, 1 << 20, 6, 18, 3 << 5, 9 << 10, 3 << 15, 9 << 16, 3 << 20, 9 << 20]


@pytest.mark.gpu
@pytest.mark.parametrize("n2", STRUCT_N2)
def test_decode_structured_losses(fecc, n2):
    N, S = n2 // 2, 4
    degs = F.values(N, S, seed=n2)
    pristine = code_word(N, degs)
    pow2 = n2 & (n2 - 1) == 0
    for k, (name, E) in enumerate(structured_losses(N, n2)):
        decode_case(N, degs, pristine, E, "decode 2N=%d, %s" % (n2, name), torch_level=pow2, seed=k)


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 5, 1021])
@pytest.mark.parametrize("N", [1 << 11, 3 << 10])
def test_decode_pitches_and_raw_words(fecc, N, S):
    """Code rows at ceil4(S) + 8 words, out rows at ceil4(S) + 20 (sentinels past ceil4(S) survive).  Every surviving word
    below C is stored raw as x + P -- all of column 0, the constant 1 of degree 0 -- and decodes as x; random words below C
    in the surviving rows decode alike with and without + P."""
    from fastecc_b200 import decoder
    n2, s4 = 2 * N, (S + 3) // 4 * 4
    pitch, out_pitch = s4 + 8, s4 + 20
    degs = F.values(N, S, seed=S)
    assert degs[0] == 0
    rng = np.random.default_rng(N + S)
    E = np.array(sorted(set(rng.choice(n2, N // 2, replace=False).tolist()) | {0, n2 - 1}), dtype=np.int64)
    Ed = torch.from_numpy(E).to(DEV)
    surv = torch.ones(n2, dtype=torch.bool, device=DEV)
    surv[Ed] = False
    code = F.buffer(n2, S, pitch, fill=SENT)
    F.fill(code, lambda i: torch.where(surv[i, None], raw(R.codeword_rows(N, degs, i, DEV)), torch.full((len(i), S), 0xFFFFFFFF, dtype=torch.int64, device=DEV)))
    assert bool((R.as_words(code[surv][:, 0]) == P + 1).all())
    pat = decoder.CErasurePattern(n2, E, mixed=True)
    out = torch.full((E.size, out_pitch), SENT, dtype=torch.int32, device=DEV)
    recover_into(pat, code, S, pitch, out, out_pitch)
    what = "decode N=%d S=%d pitch %d out pitch %d" % (N, S, pitch, out_pitch)
    F.check(out[:, :S], lambda i: R.codeword_rows(N, degs, Ed[i], DEV), what)
    assert bool((out[:, s4:] == SENT).all()), what + ": words past ceil4(S) of the out rows were written"
    g = torch.Generator(device=DEV); g.manual_seed(S)
    x = torch.randint(0, C, (n2, S), device=DEV, generator=g, dtype=torch.int64)
    outs = []
    for add in (0, P):
        t = F.buffer(n2, S, pitch, fill=SENT)
        t.copy_(F.to_i32(x + add))
        o = torch.full((E.size, out_pitch), SENT, dtype=torch.int32, device=DEV)
        recover_into(pat, t, S, pitch, o, out_pitch)
        outs.append(R.as_words(o[:, :S]))
    pat.close()
    assert bool((outs[0] < P).all()) and torch.equal(outs[0], outs[1]), what + ": raw surviving words x + P decode unlike x"


@pytest.mark.gpu
def test_one_decode_pattern_on_two_streams(fecc):
    from fastecc_b200 import decoder
    N, S = 3 << 14, 16
    g = torch.Generator(device=DEV); g.manual_seed(21)
    Ed = torch.sort(torch.randperm(2 * N, device=DEV, generator=g)[:N]).values
    pat = decoder.CErasurePattern(2 * N, Ed.cpu().numpy(), mixed=True)
    degs = [F.values(N, S, seed=k) for k in range(2)]
    codes = [code_word(N, d).clone() for d in degs]
    for k, c in enumerate(codes):
        c[Ed] = garbage(N, S, k)
    streams = [torch.cuda.Stream() for _ in range(2)]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    recs = []
    for s, c in zip(streams, codes):
        with torch.cuda.stream(s):
            recs.append(pat.recover(c))
    torch.cuda.synchronize()
    pat.close()
    for k in range(2):
        F.check(recs[k], lambda i: R.codeword_rows(N, degs[k], Ed[i], DEV), "decode on stream %d" % k)


# ==== GPU: repair ===========================================================================================================
def repair_shapes():
    out = []
    for N, S in ((1 << 19, 5), (3 << 19, 6), (9 << 19, 3)):
        out += [(N, M, S) for M in sorted({m for m in (1, 2, 3, 9, N // 1024, N // 9, N // 8, N) if N % m == 0})]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("N,M,S", repair_shapes())
def test_repair_closed_form_stripes(fecc, N, M, S):
    """Data rows at ceil4(S) + 4 words, parity rows at ceil4(S) + 8, the parity below the data."""
    s4 = (S + 3) // 4 * 4
    degs = F.values(N, S, seed=M)
    views = stripe(N, M, S, s4 + 4, s4 + 8, degs)
    pristine = views[0].clone()
    for name, ld, lp in repair_losses(N, M, N + M):
        repair_case(N, M, S, degs, pristine, views, ld, lp, name)
    del views, pristine
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1021, 1022, 1023])
@pytest.mark.parametrize("N,M", [(9 << 9, 512), (3 << 10, 3 << 10)])
def test_repair_distinct_pitches(fecc, N, M, S):
    """Data rows at 1028 words, parity rows at 1040, the parity buffer below the data buffer."""
    degs = F.values(N, S, seed=S)
    views = stripe(N, M, S, 1028, 1040, degs)
    pristine = views[0].clone()
    rng = np.random.default_rng(S + M)
    nd = M // 3
    cases = repair_losses(N, M, S) + [("random", np.sort(rng.choice(N, nd, replace=False)), np.sort(rng.choice(M, M - nd, replace=False)))]
    for name, ld, lp in cases:
        repair_case(N, M, S, degs, pristine, views, ld, lp, name)


@pytest.mark.gpu
def test_repair_in_three_column_chunks(fecc):
    out = child("chunks")
    assert "ok chunks" in out, out


# ==== GPU: three operation families on three streams ========================================================================
@pytest.mark.gpu
def test_repair_decode_and_encode_on_three_streams(fecc):
    out = child("streams")
    assert out.count("ok streams") == 2, out


# ==== GPU: the storage pipeline, bytes to bytes =============================================================================
@pytest.mark.gpu
def test_byte_pipeline_through_repair_and_decode(fecc):
    """4 KiB blocks (random, and the adversarial blocks of the recoding) -> 1025-word blocks at a 1028-word pitch -> M parity
    blocks, sampled rows against the encode by definition -> M blocks lost -> repair, and the 2N-row decode -> the bytes."""
    import test_byte_recode as TB
    from fastecc_b200 import decoder
    N, M, W = 3 << 9, 3 << 5, 1024
    D, SZ, pitch = N // M, W + 1, W + 4
    rng = np.random.default_rng(12)
    x = rng.integers(0, 1 << 32, size=(N, W), dtype=np.uint64).astype(np.uint32)
    adv = TB._cases(W, rng)
    x[:len(adv)] = adv
    raw_bytes = torch.from_numpy(x.view(np.uint8).reshape(N, 4 * W)).to(DEV)
    words = torch.full((N, pitch), SENT, dtype=torch.int32, device=DEV)
    fecc.bytes_to_gfp_dev(raw_bytes, words)
    assert bool((words[:, SZ:] == SENT).all()), "the recoding wrote past word W"
    enc = words.clone()
    fecc.rs_encode_asym_mixed_dev(enc[:, :SZ], M)
    parity = torch.full((M, pitch), SENT, dtype=torch.int32, device=DEV)
    parity[:, :SZ] = enc[:M, :SZ]
    del enc
    js = sorted({0, 1, M // 2, M - 1} | set(rng.choice(M, 4, replace=False).tolist()))
    want = R.encode_rows(R.as_words(words[:, :SZ]), [D * j for j in js])
    assert torch.equal(R.as_words(parity[js, :SZ]), want), "sampled parity rows differ from the encode by definition"
    # lose the adversarial blocks 7 .. 12 (all 0xFFF digits, a P - 1 word, ...) and others: M blocks in all
    ld = sorted(list(range(7, 13)) + rng.choice(np.arange(13, N), M // 2 - 6, replace=False).tolist())
    lp = sorted(rng.choice(M, M - len(ld), replace=False).tolist())
    dmg_d, dmg_p = words.clone(), parity.clone()
    dmg_d[ld, :SZ] = -1
    dmg_p[lp, :SZ] = 12345
    data, par = dmg_d.clone(), dmg_p.clone()
    fecc.rs_repair_dev(data[:, :SZ], par[:, :SZ], ld, lp)
    assert torch.equal(data, words), "repaired data (pad words 1025 - 1027 included)"
    assert torch.equal(par, parity), "repaired parity (pad words 1025 - 1027 included)"
    assert bool((fecc.gfp_to_bytes_dev(data, W) == raw_bytes).all()), "bytes after repair"
    code = torch.full((2 * N, pitch), SENT, dtype=torch.int32, device=DEV)
    code[0::2] = dmg_d
    code[1::2 * D] = dmg_p
    rows = decoder.asym_erasures(N, M, ld, lp)
    at = {r: k for k, r in enumerate(rows)}
    pat = decoder.CErasurePattern(2 * N, rows, mixed=True)
    rec = pat.recover(code[:, :SZ])
    pat.close()
    got = dmg_d.clone()
    got[ld, :SZ] = rec[[at[2 * i] for i in ld]]
    assert torch.equal(got, words), "data decoded from the 2N-row code word"
    assert torch.equal(rec[[at[2 * D * j + 1] for j in lp]], parity[lp, :SZ]), "parity decoded from the 2N-row code word"
    assert bool((fecc.gfp_to_bytes_dev(got, W) == raw_bytes).all()), "bytes after the 2N-row decode"


# ==== child processes =======================================================================================================
def _chunks(fe):
    """N = 9 * 2^18, M = N, SIZE = 502: the 4 GiB workspace holds 224 words of the N + M rows, so the repair runs in chunks of
    224 + 224 + 54 words, the last one ending in a partial 16-byte group."""
    GiB = 1 << 30
    free, total = torch.cuda.mem_get_info()
    print("device %s: %.1f GiB free of %.1f GiB" % (torch.cuda.get_device_name(), free / GiB, total / GiB), flush=True)
    if free < 24 * GiB:
        print("SKIP: %.1f GiB free on the device, the three-chunk repair needs 24 GiB" % (free / GiB))
        sys.exit(3)
    N = M = 9 << 18
    S = 502
    cap = (4 << 30) // 4 // (N + M) // 4 * 4
    assert cap == 224 and S - 2 * cap == 54
    degs = F.values(N, S, seed=7)
    views = stripe(N, M, S, 508, 512, degs)
    t0 = time.time()
    ld, lp = np.arange(1, N, 2), np.arange(N // 2)             # the odd data rows and the first half of the parity
    lost_d = torch.zeros(N, dtype=torch.bool, device=DEV)
    lost_p = torch.zeros(M, dtype=torch.bool, device=DEV)
    lost_d[1::2] = True
    lost_p[:N // 2] = True
    views[1][1::2, :S] = -1
    views[2][:N // 2, :S] = 0x7EADBEEF
    from fastecc_b200 import decoder
    r = decoder.Repair(N, M, ld, lp)
    torch.cuda.synchronize(); t1 = time.time()
    r.repair(views[1][:, :S], views[2][:, :S])
    torch.cuda.synchronize(); t2 = time.time()
    r.close()
    print("pattern %.1f s, repair %.1f s" % (t1 - t0, t2 - t1), flush=True)
    check_rows(views[1], S, lambda i: R.monomial_data(N, degs, i, DEV), lost_d, "three-chunk repair: data")
    check_rows(views[2], S, lambda j: R.monomial_parity(N, degs, j, DEV, 1), lost_p, "three-chunk repair: parity")
    del views
    free2, _ = torch.cuda.mem_get_info()
    print("ok chunks: peak %.1f GiB allocated by torch, %.1f GiB in use on the device at the end" % (torch.cuda.max_memory_allocated() / GiB, (total - free2) / GiB))


def _streams(fe):
    """A repair, a mixed-order decode and a mixed encode of an order not used before in the process, enqueued back to back on
    three streams (they share the context's scratch buffers), twice."""
    from fastecc_b200 import decoder
    S = 64
    Nr, Mr = 3 << 16, 3 << 14
    degs_r = F.values(Nr, S, seed=1)
    rviews = stripe(Nr, Mr, S, S + 4, S + 8, degs_r)
    rpristine = rviews[0].clone()
    rng = np.random.default_rng(5)
    ld = np.sort(rng.choice(Nr, Mr // 2, replace=False))
    lp = np.sort(rng.choice(Mr, Mr - Mr // 2, replace=False))
    lost_d = torch.zeros(Nr, dtype=torch.bool, device=DEV)
    lost_p = torch.zeros(Mr, dtype=torch.bool, device=DEV)
    lost_d[torch.from_numpy(ld).to(DEV)] = True
    lost_p[torch.from_numpy(lp).to(DEV)] = True
    rep = decoder.Repair(Nr, Mr, ld, lp)
    Nd = 9 << 14
    degs_d = F.values(Nd, S, seed=2)
    dpristine = code_word(Nd, degs_d).clone()
    g = torch.Generator(device=DEV); g.manual_seed(6)
    Ed = torch.sort(torch.randperm(2 * Nd, device=DEV, generator=g)[:Nd]).values
    dpristine[Ed] = garbage(Nd, S, 6)
    pat = decoder.CErasurePattern(2 * Nd, Ed.cpu().numpy(), mixed=True)
    Ne = 9 << 16
    degs_e = F.values(Ne, S, seed=3)
    for k in range(2):
        rviews[0].copy_(rpristine)
        rviews[1][torch.from_numpy(ld).to(DEV), :S] = -1
        rviews[2][torch.from_numpy(lp).to(DEV), :S] = 77
        code = dpristine.clone()
        enc = F.buffer(Ne, S)
        F.fill(enc, lambda i: R.monomial_data(Ne, degs_e, i, DEV))
        streams = [torch.cuda.Stream() for _ in range(3)]
        for s in streams:
            s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(streams[0]):
            rep.repair(rviews[1][:, :S], rviews[2][:, :S])
        with torch.cuda.stream(streams[1]):
            rec = pat.recover(code)
        with torch.cuda.stream(streams[2]):
            fe.rs_encode_mixed_dev(enc)
        torch.cuda.synchronize()
        check_rows(rviews[1], S, lambda i: R.monomial_data(Nr, degs_r, i, DEV), lost_d, "repair on stream 0: data")
        check_rows(rviews[2], S, lambda j: R.monomial_parity(Nr, degs_r, j, DEV, Nr // Mr), lost_p, "repair on stream 0: parity")
        F.check(rec, lambda i: R.codeword_rows(Nd, degs_d, Ed[i], DEV), "decode on stream 1")
        F.check(enc, lambda j: R.monomial_parity(Ne, degs_e, j, DEV), "mixed encode on stream 2")
        print("ok streams round %d" % k, flush=True)
    rep.close()
    pat.close()


if __name__ == "__main__":
    import fastecc_b200
    fastecc_b200.init(0)
    {"chunks": _chunks, "streams": _streams}[sys.argv[1]](fastecc_b200)
