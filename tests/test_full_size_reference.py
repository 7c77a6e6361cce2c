"""Every transform and encode against something other than the library: closed forms that fix every output word, and rows by
definition (tests/gfp_ref.py, plain torch int64, no library code) where the oracle's O(N^2) loops cannot reach.

  CPU   gfp_ref against the oracle (Slow_NTT both ways, the encode by definition, the power-of-two encode) and the closed forms
        against gfp_ref's rows by definition.
  GPU   closed forms, every word: the transform at every order the ABI accepts (2^0 .. 9 * 2^20, both directions), the encodes
        at every order (2^0 .. 9 * 2^19), the asymmetric encodes at a spread of M, the host (T**) entry points, wide shapes and
        the repack path; random data against rows by definition at the mixed orders 3 * 2^k, 9 * 2^k, k >= 11, where the
        order-2^k sub-transforms run on every r-th row; raw 32-bit inputs against their residues for one shape per plan class.
        In a child process each (the library's context keeps its scratch buffers, and reads the launcher's settings once per
        process): buffers past 2^32 words, and the launcher's settings FASTECC_B200_NO_TMA, _SPLIT=lo|hi, _CTAS_PER_SM.

Closed forms (rho = GF_Root(2N), omega = GF_Root(N)): column c of a monomial stripe holds data_i = rho^(2*i*m_c), its parity is
parity_j = rho^((2j+1)*m_c) and its asymmetric parity j' = rho^((2*(N/M)*j'+1)*m_c); a delta at n_c transforms to
omega^(n_c*k), the geometric column omega^(-m_c*n) to N at k = m_c and 0 elsewhere (omega inverted for the inverse transform).
The run as a script (`python tests/test_full_size_reference.py large|knobs`) is the child process of the last two groups."""
import json
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

import gfp_ref as R                  # noqa: E402
import oracle_lib as ol              # noqa: E402

P = R.P
CHUNK = 1 << 26                      # int64 elements per row chunk of a fill or a comparison (512 MiB)
DEV = "cuda"


# ---- shapes ------------------------------------------------------------------------------------------------------------
def order_parts(N):
    """N = r * L, r in {1, 3, 9}, L a power of two"""
    r = 9 if N % 9 == 0 else 3 if N % 3 == 0 else 1
    return r, N // r


def plan_boundaries(N):
    """Indices where the plan changes digit: the seams k1 * L of N = r * L and the N1 (and N2) of L's two-level split."""
    r, L = order_parts(N)
    b = [L] if r > 1 else []
    lg = L.bit_length() - 1
    if lg > 9:
        n1 = 1 << ((lg + 1) // 2)
        b += [n1, L // n1, r * n1]
    return b + [k * L for k in range(2, r)]


def values(N, count, seed=0):
    vals = R.special_values(N, plan_boundaries(N), count=count, seed=seed)
    return (vals * count)[:count]


POW2 = [1 << k for k in range(21)]
MIXED_NTT = [r << k for r in (3, 9) for k in range(21)]
MIXED_ENC = [r << k for r in (3, 9) for k in range(20)]


# ---- device buffers -----------------------------------------------------------------------------------------------------
def to_i32(t):
    """int64 words in [0, 2^32) -> int32 with the same bits"""
    return torch.where(t >= 1 << 31, t - (1 << 32), t).to(torch.int32)


def buffer(N, S, pitch=None, fill=-1):
    """N rows of S words at `pitch` (default S rounded up to 4; a pitch that is not a multiple of 4 takes the repack path),
    pad words set to `fill`; returns the [N, S] view."""
    pitch = pitch or (S + 3) // 4 * 4
    return torch.full((N, pitch), fill, dtype=torch.int32, device=DEV)[:, :S]


def row_chunks(n, S):
    step = max(1, CHUNK // max(S, 1))
    for r0 in range(0, n, step):
        yield r0, min(n, r0 + step)


def fill(t, gen):
    """t[rows] = gen(rows) chunk by chunk (gen returns int64 words)"""
    for r0, r1 in row_chunks(t.shape[0], t.shape[1]):
        t[r0:r1] = to_i32(gen(torch.arange(r0, r1, dtype=torch.int64, device=t.device)))


def check(got, want_fn, what, rows=None):
    """Every word of got (int32 view) equals want_fn(row indices) (int64), compared chunk by chunk."""
    n, S = got.shape[0] if rows is None else rows, got.shape[1]
    for r0, r1 in row_chunks(n, S):
        g = R.as_words(got[r0:r1])
        w = want_fn(torch.arange(r0, r1, dtype=torch.int64, device=got.device))
        bad = g != w
        if bool(bad.any()):
            idx = bad.nonzero()[:4].tolist()
            detail = ["row %d col %d: got %d want %d" % (r0 + i, c, int(g[i, c]), int(w[i, c])) for i, c in idx]
            raise AssertionError("%s: %d of %d words differ in rows [%d, %d); %s" % (what, int(bad.sum()), bad.numel(), r0, r1, "; ".join(detail)))


# ---- the operations, device and host entry points -------------------------------------------------------------------------
ENCODES = ("encode", "mixed", "asym", "asym_mixed", "host_encode", "host_mixed", "host_asym", "host_asym_mixed")


def run(fe, kind, t, M=None):
    """`kind` in place on the [N, S] device view t; the output rows are t[:M] for the asymmetric encodes, else all of t."""
    N, S = t.shape
    if kind == "ntt":
        fe.ntt_dev(t, False)
    elif kind == "intt":
        fe.ntt_dev(t, True)
    elif kind == "encode":
        fe.rs_encode_dev(t)
    elif kind == "mixed":
        fe.rs_encode_mixed_dev(t)
    elif kind == "asym":
        fe.rs_encode_asym_dev(t, M)
    elif kind == "asym_mixed":
        fe.rs_encode_asym_mixed_dev(t, M)
    else:
        a = np.ascontiguousarray(t.cpu().numpy()).view(np.uint32)
        {"host_ntt": lambda: fe.MFA_NTT(a, N, S, False),
         "host_intt": lambda: fe.MFA_NTT(a, N, S, True),
         "host_encode": lambda: fe.EncodeReedSolomon_body(a, N, S),
         "host_mixed": lambda: fe.EncodeReedSolomon_mixed(a, N, S),
         "host_asym": lambda: fe.EncodeReedSolomon_asym(a, N, M, S),
         "host_asym_mixed": lambda: fe.EncodeReedSolomon_asym_mixed(a, N, M, S)}[kind]()
        t.copy_(torch.from_numpy(a.view(np.int32)))
    return t[:M] if M else t


def closed_form(fe, kind, N, S=16, M=None, pitch=None, seed=0):
    """Run `kind` on the closed-form input of N x S words and compare every output word with the closed form."""
    dev = DEV
    vals = values(N, S, seed)
    shown = lambda v: str(v if len(v) <= 8 else v[:8] + ["..."])
    t = buffer(N, S, pitch)
    if kind.endswith(ENCODES):
        dec = N // M if M else 1
        fill(t, lambda i: R.monomial_data(N, vals, i, dev))
        out = run(fe, kind, t, M)
        check(out, lambda j: R.monomial_parity(N, vals, j, dev, dec), "%s N=%d S=%d M=%s degrees %s" % (kind, N, S, M, shown(vals)))
        return
    inverse = kind.endswith("intt")
    h = S // 2                                       # columns [0, h): deltas at vals[:h]; [h, S): geometric columns of vals[h:]
    pos, freq = vals[:h], vals[h:]
    pos_t = torch.tensor(pos, dtype=torch.int64, device=dev)
    fill(t[:, :h], lambda i: (i[:, None] == pos_t[None, :]).to(torch.int64))
    fill(t[:, h:], lambda i: R.geometric_ntt_input(N, freq, i, dev, inverse))
    out = run(fe, kind, t)
    what = "%s N=%d S=%d" % (kind, N, S)
    check(out[:, :h], lambda k: R.delta_ntt_columns(N, pos, k, dev, inverse), what + " deltas at %s" % shown(pos))
    check(out[:, h:], lambda k: R.ntt_spike(N, freq, k, dev), what + " geometric columns of %s" % shown(freq))


# ==== CPU: the reference against the oracle ===============================================================================
REF_ORDERS = [1 << k for k in range(11)] + [r << k for r in (3, 9) for k in range(6) if r << k <= 288]


def rand_words(N, S, seed):
    return np.random.default_rng(seed).integers(0, P, size=(N, S), dtype=np.uint64).astype(np.uint32)


def t64(a):
    return torch.from_numpy(np.ascontiguousarray(a).astype(np.int64))


def test_mulmod_and_powers_on_edge_words():
    vals = [0, 1, 2, 0xFFFF, 0x10000, P - 2, P - 1, 1 << 31, 0xFFF00000, 123456789]
    a = torch.tensor([x for x in vals for _ in vals], dtype=torch.int64)
    b = torch.tensor([y for _ in vals for y in vals], dtype=torch.int64)
    assert R.mulmod(a, b).tolist() == [x * y % P for x in vals for y in vals]
    assert R.inv(torch.tensor(vals[1:], dtype=torch.int64)).tolist() == [pow(x, P - 2, P) for x in vals[1:]]
    for n in (2, 3, 4096, 9 << 12, 9 << 20):
        e = torch.tensor([0, 1, 4095, 4096, 4097, n - 1, n, 3 * n + 5], dtype=torch.int64)
        w = R.root(n)
        assert R.RootPowers(n)(e).tolist() == [pow(w, int(x) % n, P) for x in e]
        assert R.RootPowers(n, sign=-1)(e).tolist() == [pow(w, (-int(x)) % n, P) for x in e]
        assert pow(w, n, P) == 1 and (n == 1 or pow(w, n // 2, P) != 1)


@pytest.mark.parametrize("N", REF_ORDERS)
def test_reference_transform_equals_slow_ntt(oracle, N):
    S = 3
    a = rand_words(N, S, N)
    for inverse in (0, 1):
        want = a.copy()
        oracle.oracle_slow_ntt(want.ctypes.data, N, S, inverse)
        got = R.ntt_rows(t64(a), range(N), inverse=bool(inverse))
        assert torch.equal(got, t64(want)), (N, inverse)


@pytest.mark.parametrize("N", REF_ORDERS)
def test_reference_encode_equals_the_oracle(oracle, N):
    S = 3
    a = rand_words(N, S, 7 * N)
    want = np.empty_like(a)
    oracle.oracle_rs_encode_by_definition(a.ctypes.data, want.ctypes.data, N, S)
    got = R.encode_rows(t64(a), range(N))
    assert torch.equal(got, t64(want))
    if N & (N - 1) == 0:
        assert torch.equal(got, t64(ol.o_encode(oracle, a)))


@pytest.mark.parametrize("N", [1, 2, 3, 4, 6, 8, 9, 12, 18, 32, 36, 96, 288, 1024])
def test_closed_forms_equal_the_definitions(N):
    """monomial stripes (full and every asymmetric M dividing N), deltas and geometric columns against the rows by definition"""
    degs = values(N, 8, seed=1)
    data = R.monomial_data(N, degs)
    assert torch.equal(R.encode_rows(data, range(N)), R.monomial_parity(N, degs))
    for M in [m for m in range(1, N) if N % m == 0][-4:]:
        assert torch.equal(R.encode_rows(data, range(0, N, N // M)), R.monomial_parity(N, degs, decimation=N // M)), M
    for inverse in (False, True):
        delta = torch.zeros((N, len(degs)), dtype=torch.int64)
        delta[degs, torch.arange(len(degs))] = 1
        assert torch.equal(R.ntt_rows(delta, range(N), inverse), R.delta_ntt_columns(N, degs, inverse=inverse))
        geo = R.geometric_ntt_input(N, degs, inverse=inverse)
        assert torch.equal(R.ntt_rows(geo, range(N), inverse), R.ntt_spike(N, degs))


def test_plan_boundaries_name_the_seams():
    assert plan_boundaries(1 << 19) == [1024, 512, 1024]
    assert plan_boundaries(3 << 12) == [4096, 64, 64, 192, 8192]
    assert plan_boundaries(9 << 9) == [512] + [k * 512 for k in range(2, 9)]
    v = values(9 << 20, 16)
    assert v[:7] == [0, 1, (9 << 20) - 1, 9 << 19, (1 << 20) - 1, 1 << 20, (1 << 20) + 1]


# ==== GPU: closed forms, every output word ================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("N", POW2 + MIXED_NTT)
def test_transform_closed_forms_at_every_order(fecc, N):
    closed_form(fecc, "ntt", N)
    closed_form(fecc, "intt", N, seed=1)


@pytest.mark.gpu
@pytest.mark.parametrize("N", POW2[:20])
def test_encode_closed_form_at_every_power_of_two(fecc, N):
    closed_form(fecc, "encode", N)


@pytest.mark.gpu
@pytest.mark.parametrize("N", MIXED_ENC)
def test_mixed_encode_closed_form_at_every_order(fecc, N):
    closed_form(fecc, "mixed", N)


def asym_cases():
    """(N, M): M = 1, M below and at the split's N1 (gather and native paths for powers of two), N/r, N/2."""
    out = []
    for N in (1 << 5, 1 << 10, 1 << 11, 1 << 14, 1 << 16, 1 << 19):
        lg = N.bit_length() - 1
        n1 = 1 << ((lg + 1) // 2)
        out += sorted({(N, M) for M in (1, 2, n1 // 2, n1, 2 * n1, N // 2) if 1 <= M < N})
    for N in (3, 9, 3 << 6, 9 << 10, 3 << 13, 9 << 16, 3 << 19, 9 << 19):
        r, L = order_parts(N)
        out += sorted({(N, M) for M in (1, 3, L // 4, L, 3 * L, N // 2, N // 3) if M >= 1 and N % M == 0 and M < N})
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("N,M", asym_cases())
def test_asym_encode_closed_form(fecc, N, M):
    closed_form(fecc, "asym_mixed" if N & (N - 1) else "asym", N, 8, M)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,N,M", [("ntt", 1 << 19, None), ("intt", 3 << 18, None), ("encode", 1 << 19, None),
                                      ("mixed", 3 << 18, None), ("asym", 1 << 19, 1 << 13), ("asym_mixed", 3 << 18, 1 << 16)])
def test_wide_closed_forms(fecc, kind, N, M):
    """1024 words: many strips of the wide 512-thread geometry per row set"""
    closed_form(fecc, kind, N, 1024, M)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,N,M", [("ntt", 1 << 12, None), ("intt", 9 << 11, None), ("encode", 1 << 12, None), ("encode", 1 << 19, None),
                                      ("mixed", 3 << 12, None), ("asym_mixed", 9 << 11, 1 << 9)])
def test_repacked_layout_closed_forms(fecc, kind, N, M):
    """SIZE = 13 words at a pitch of 15: the unaligned layout goes through the internal repack"""
    closed_form(fecc, kind, N, 13, M, pitch=15)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,N,M", [("host_ntt", 1 << 10, None), ("host_intt", 3 << 11, None), ("host_encode", 1 << 12, None),
                                      ("host_mixed", 9 << 8, None), ("host_asym", 1 << 13, 1 << 5), ("host_asym_mixed", 3 << 12, 3 << 8),
                                      ("host_encode", 1 << 15, None), ("host_ntt", 1 << 15, None)])
def test_host_entry_point_closed_forms(fecc, kind, N, M):
    """T** entry points; 2^15 x 300 words takes the pipelined column-chunk path of large arrays (a partial last chunk)"""
    closed_form(fecc, kind, N, 300 if N == 1 << 15 else 16, M)


# ==== GPU: random data against rows by definition at the large mixed orders ================================================
def sample_rows(N, seed):
    r, L = order_parts(N)
    rows = [0, 1, N - 1] + [k * L + d for k in range(1, r) for d in (-1, 0, 1)]
    g = torch.Generator().manual_seed(seed)
    rows += torch.randint(0, N, (16,), generator=g).tolist()
    return sorted(set(rows))


def sample_cols(S, seed):
    g = torch.Generator().manual_seed(seed + 1)
    return sorted(set([0, 1, 2, 3, S - 4, S - 3, S - 2, S - 1] + torch.randint(4, S - 4, (2,), generator=g).tolist()))


def random_buffer(N, S, seed):
    g = torch.Generator(device=DEV); g.manual_seed(seed)
    t = buffer(N, S)
    t.copy_(to_i32(torch.randint(0, P, (N, S), device=DEV, generator=g, dtype=torch.int64)))
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("N", [r << k for r in (3, 9) for k in range(11, 21)])
@pytest.mark.parametrize("inverse", [False, True])
def test_large_mixed_transforms_by_definition(fecc, N, inverse):
    S = 30                                                   # pitch 32: the last chunk of 4 words is partial
    t = random_buffer(N, S, N + inverse)
    rows, cols = sample_rows(N, N), sample_cols(S, N)
    x = R.as_words(t[:, cols])
    fecc.ntt_dev(t, inverse)
    want = R.ntt_rows(x, rows, inverse)
    got = R.as_words(t[rows][:, cols])
    assert torch.equal(got, want), [(rows[i], cols[c]) for i, c in (got != want).nonzero()[:8].tolist()]


@pytest.mark.gpu
@pytest.mark.parametrize("N", [r << k for r in (3, 9) for k in range(11, 20)])
def test_large_mixed_encodes_by_definition(fecc, N):
    S = 30
    t = random_buffer(N, S, 3 * N)
    rows, cols = sample_rows(N, 2 * N), sample_cols(S, 2 * N)
    x = R.as_words(t[:, cols])
    fecc.rs_encode_mixed_dev(t)
    want = R.encode_rows(x, rows)
    got = R.as_words(t[rows][:, cols])
    assert torch.equal(got, want), [(rows[i], cols[c]) for i, c in (got != want).nonzero()[:8].tolist()]


# ==== GPU: raw 32-bit words are taken mod P ================================================================================
RAW_SHAPES = [                         # (kind, N, S, M, pitch): one per plan class
    ("ntt", 16, 8, None, None), ("encode", 8, 8, None, None),                   # small DFT
    ("intt", 256, 8, None, None), ("encode", 512, 8, None, None),               # single pass; the fused one is the narrow twin <9,2,1>
    ("ntt", 1 << 12, 8, None, None), ("encode", 1 << 12, 8, None, None),        # two-pass NTT, three-pass encode
    ("ntt", 1 << 20, 64, None, None), ("encode", 1 << 19, 64, None, None),      # wide 1024-row passes and the wide fused pass
    ("intt", 9 << 11, 8, None, None), ("mixed", 3 << 12, 8, None, None),        # mixed step 2 (transform, encode)
    ("ntt", 9, 8, None, None), ("intt", 3, 8, None, None),                      # ... reading the caller's words (order L = 1)
    ("asym_mixed", 9 << 12, 8, 1 << 10, None), ("asym_mixed", 3, 8, 1, None),   # the fold
    ("asym", 1 << 16, 8, 1 << 9, None), ("asym", 1 << 16, 8, 1 << 4, None),     # asymmetric native and gather
    ("encode", 1 << 12, 5, None, 7), ("ntt", 3 << 10, 5, None, 7),              # repack
    ("host_encode", 1 << 11, 8, None, None), ("host_ntt", 9 << 6, 8, None, None), ("host_asym_mixed", 3 << 10, 8, 3 << 4, None),
]
RAW_FILLS = ["ones", "p", "p_plus_col", "alt_rows", "alt_cols", "random"]


def raw_words(fill_kind, N, S, seed):
    i = torch.arange(N, dtype=torch.int64, device=DEV)[:, None]
    c = torch.arange(S, dtype=torch.int64, device=DEV)[None, :]
    if fill_kind == "ones":
        return torch.full((N, S), 0xFFFFFFFF, dtype=torch.int64, device=DEV)
    if fill_kind == "p":
        return torch.full((N, S), P, dtype=torch.int64, device=DEV)
    if fill_kind == "p_plus_col":
        return (P + c).expand(N, S).clone()
    if fill_kind == "alt_rows":
        return ((i % 2) * 0xFFFFFFFF).expand(N, S).clone()
    if fill_kind == "alt_cols":
        return ((c % 2) * 0xFFFFFFFF).expand(N, S).clone()
    g = torch.Generator(device=DEV); g.manual_seed(seed)
    return torch.randint(0, 1 << 32, (N, S), device=DEV, generator=g, dtype=torch.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("fill_kind", RAW_FILLS)
@pytest.mark.parametrize("kind,N,S,M,pitch", RAW_SHAPES)
def test_raw_words_equal_their_residues(fecc, kind, N, S, M, pitch, fill_kind):
    raw = raw_words(fill_kind, N, S, N * S)
    outs = []
    for x in (raw, raw % P):
        t = buffer(N, S, pitch)
        t.copy_(to_i32(x))
        outs.append(R.as_words(run(fecc, kind, t, M)).clone())
    assert bool((outs[0] < P).all()), "non-canonical output words"
    bad = (outs[0] != outs[1]).nonzero()[:8].tolist()
    assert not bad, bad


# ==== child processes: buffers past 2^32 words, the launcher's settings ======================================================
KNOBS = ("FASTECC_B200_NO_TMA", "FASTECC_B200_SPLIT", "FASTECC_B200_CTAS_PER_SM")
WIDE_2P19 = ["ntt_pass_kernel<10,1,1,512>", "ntt_pass_kernel<9,2,1,512>", "ntt_pass_kernel<10,1,1,512>"]


@pytest.mark.gpu
def test_timed_encode_names_each_geometry(fecc):
    """rs_encode_dev_timed names the instantiation every pass ran as, whichever geometry of <9,2,1> ran first in the process:
    the single-pass encode of 2^9 blocks takes the narrow twin, the fused pass of the 2^19 x 1024-word encode the wide one."""
    if any(k in os.environ for k in KNOBS):
        pytest.skip("a launcher setting is in the environment")
    assert [n for n, _ in fecc.rs_encode_dev_timed(buffer(512, 8))] == ["ntt_pass_kernel<9,2,1>"]
    assert [n for n, _ in fecc.rs_encode_dev_timed(buffer(1 << 19, 1024))] == WIDE_2P19
    assert [n for n, _ in fecc.rs_encode_dev_timed(buffer(512, 8))] == ["ntt_pass_kernel<9,2,1>"]


def child(mode, env_extra=None, timeout=1200):
    torch.cuda.empty_cache()
    env = {k: v for k, v in os.environ.items() if k not in KNOBS}
    env.update(env_extra or {})
    t0 = time.time()
    p = subprocess.Popen([sys.executable, os.path.abspath(__file__), mode], cwd=ROOT, env=env,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        out, _ = p.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        p.kill()
        out, _ = p.communicate()
        pytest.fail("child %s %s timed out after %d s:\n%s" % (mode, env_extra, timeout, out[-4000:]))
    print(out)
    print("child %s %s: %.1f s" % (mode, env_extra, time.time() - t0))
    if p.returncode == 3:
        pytest.skip(out.strip().splitlines()[-1])
    assert p.returncode == 0, out[-6000:]
    return out


@pytest.mark.gpu
def test_buffers_past_2_to_the_32_words(fecc):
    out = child("large")
    assert out.count("ok ") == 6, out


@pytest.mark.gpu
@pytest.mark.parametrize("env", [{"FASTECC_B200_NO_TMA": "1"}, {"FASTECC_B200_SPLIT": "lo"}, {"FASTECC_B200_SPLIT": "hi"},
                                 {"FASTECC_B200_CTAS_PER_SM": "1"}], ids=["no_tma", "split_lo", "split_hi", "ctas_per_sm_1"])
def test_launcher_settings(fecc, env):
    out = child("knobs", env)
    assert "knobs ok" in out, out


def _large(fe):
    """Every word past 2^31 and 2^32 of five entry points, against the closed forms."""
    GiB = 1 << 30
    free, total = torch.cuda.mem_get_info()
    print("device %s: %.1f GiB free of %.1f GiB" % (torch.cuda.get_device_name(), free / GiB, total / GiB), flush=True)
    if free < 40 * GiB:
        print("SKIP: %.1f GiB free on the device, these cases need 40 GiB" % (free / GiB))
        sys.exit(3)
    dev = DEV

    def step(name, f):
        t0 = time.time()
        f()
        torch.cuda.synchronize()
        print("ok %s (%.1f s)" % (name, time.time() - t0), flush=True)
        fe.shutdown(); fe.init(0)                           # drop the context's scratch buffers between cases
        torch.cuda.empty_cache()

    step("rs_encode_dev 2^19 x 8200", lambda: closed_form(fe, "encode", 1 << 19, 8200))

    def ntt_round_trip():
        N, S = 1 << 20, 4100
        vals = values(N, S)
        h = S // 2
        pos, freq = vals[:h], vals[h:]
        pos_t = torch.tensor(pos, dtype=torch.int64, device=dev)
        t = buffer(N, S)
        gen_d = lambda i: (i[:, None] == pos_t[None, :]).to(torch.int64)
        gen_g = lambda i: R.geometric_ntt_input(N, freq, i, dev)
        fill(t[:, :h], gen_d)
        fill(t[:, h:], gen_g)
        fe.ntt_dev(t, False)
        check(t[:, :h], lambda k: R.delta_ntt_columns(N, pos, k, dev), "ntt 2^20 x 4100 deltas")
        check(t[:, h:], lambda k: R.ntt_spike(N, freq, k, dev), "ntt 2^20 x 4100 geometric columns")
        fe.ntt_dev(t, True)
        check(t[:, :h], lambda i: gen_d(i) * N, "inverse(forward) 2^20 x 4100 deltas")
        check(t[:, h:], lambda i: R.mulmod(gen_g(i), N), "inverse(forward) 2^20 x 4100 geometric columns")
    step("ntt_dev forward and inverse 2^20 x 4100", ntt_round_trip)

    N, S = 9 << 19, 1024
    step("rs_encode_mixed_dev 9*2^19 x 1024", lambda: closed_form(fe, "mixed", N, S))
    step("rs_encode_asym_mixed_dev 9*2^19 x 1024, M = N/9", lambda: closed_form(fe, "asym_mixed", N, S, N // 9))

    def repair():
        M = N // 9
        vals = values(N, S, seed=2)
        data, parity = buffer(N, S), buffer(M, S)
        fill(data, lambda i: R.monomial_data(N, vals, i, dev))
        fill(parity, lambda j: R.monomial_parity(N, vals, j, dev, 9))
        g = torch.Generator(device=dev); g.manual_seed(9)
        lost_d = torch.sort(torch.randperm(N, device=dev, generator=g)[:M // 2]).values
        lost_p = torch.sort(torch.randperm(M, device=dev, generator=g)[:M - M // 2]).values
        data[lost_d] = -1
        parity[lost_p] = 12345
        fe.rs_repair_dev(data, parity, lost_d.cpu().numpy(), lost_p.cpu().numpy())
        check(data, lambda i: R.monomial_data(N, vals, i, dev), "repaired data 9*2^19 x 1024")
        check(parity, lambda j: R.monomial_parity(N, vals, j, dev, 9), "repaired parity 9*2^19 x 1024")
    step("rs_repair_dev 9*2^19 x 1024, M = N/9, M losses", repair)
    print("ok large: peak %.1f GiB allocated by torch" % (torch.cuda.max_memory_allocated() / GiB))


def _knobs(fe):
    """A compact matrix under the launcher settings in the environment, and the pass names they select."""
    env = {k: v for k, v in os.environ.items() if k.startswith("FASTECC_B200_")}
    print("settings", env, flush=True)
    for k in range(5, 21):
        closed_form(fe, "ntt", 1 << k)
        closed_form(fe, "intt", 1 << k, seed=1)
        if k < 20:
            closed_form(fe, "encode", 1 << k)
    for N in (3 << 12, 9 << 16, 3 << 19):
        closed_form(fe, "ntt", N)
        closed_form(fe, "intt", N, seed=1)
        closed_form(fe, "mixed", N)
    for M in (512, 1 << 16):
        closed_form(fe, "asym", 1 << 19, 8, M)
    G = json.load(open(os.path.join(HERE, "golden", "survey_8c.json")))
    _, S, h0, h1 = [g for g in G["encode_fillA"] if g[0] == 19][0]
    o = ol.load_oracle()
    a = ol.fill_A(o, 1 << 19, S)
    assert ol.ohash(o, a) == h0
    t = torch.from_numpy(a.view(np.int32)).cuda()
    del a
    names = [n for n, _ in fe.rs_encode_dev_timed(t)]
    assert ol.ohash(o, t.cpu().numpy().view(np.uint32)) == h1, "fill_A 2^19 x %d encode hash" % S
    print("2^19 passes:", names, flush=True)
    if env.get("FASTECC_B200_SPLIT") == "lo":
        assert names == ["ntt_pass_kernel<9,1,1>", "ntt_pass_kernel<10,2,1,512>", "ntt_pass_kernel<9,1,1>"], names
    elif env.get("FASTECC_B200_NO_TMA"):
        for N in (1 << 11, 1 << 16):
            u = buffer(N, 64)
            names += [n for n, _ in fe.rs_encode_dev_timed(u)]
        print("NO_TMA passes:", names, flush=True)
        assert all(n.split("<")[1].rstrip(">").split(",")[2] == "0" for n in names), names
    else:                                                   # the matrix above ran the narrow twin <9,2,1> first (2^9)
        assert names == WIDE_2P19, names
    print("knobs ok", flush=True)


if __name__ == "__main__":
    import fastecc_b200
    fastecc_b200.init(0)
    {"large": _large, "knobs": _knobs}[sys.argv[1]](fastecc_b200)
