"""The sharded encode and transform on ONE GPU: every rank of a G-rank run lives in this process, on this device.

A "peer" of the sharded entry points is just a device pointer, so rank r's X and Y buffers are rows of two device tensors here,
and every rank's pass k is enqueued on one stream before any rank's pass k + 1: stream order does the barrier's job.  That runs
the kernels only the sharded paths use -- the instantiations ntt_pass_kernel<LR, NXF, 2> whose stores pick a destination buffer
from the peers, launch_pass's handling of log_g, the exchange-by-caller passes with their rank-dependent tables, the column-chunk
pointers P2PShardedEncoder.encode_host passes, and the barrier kernel (only where its wait is already satisfied) -- and compares
every output word with the oracle (small and mid orders), closed forms from tests/gfp_ref.py evaluated on the device (full size),
or the golden hashes of the reference (the headline shapes).

Layout: rank r's buffer of one role is [guard | N/G rows | guard] at a pitch with pad words; the guard rows and the pad words past
ceil4(SIZE) hold a sentinel above every canonical word, and every run ends by checking that none of them changed.  Blocks are
dealt cyclically: global block l*G + r is row l of rank r, for the data going in and the parity (or transform) coming out.  The
exchanges of the caller-exchange encode are written here from the ownership formulas:
  after pass 0:  (rank r, row k1*(N2/G) + n2')  ->  (rank k1 mod G, row (k1/G)*N2 + n2'*G + r)
  after pass 1:  (rank s, row k1'*N2 + j2)      ->  (rank j2 mod G, row (k1'*G + s)*(N2/G) + j2/G)
Launcher settings are read once per process, so those cases run this file as a script in a child process
(`python tests/test_sharded_one_gpu.py no_tma|split_lo`)."""
import ctypes
import functools
import json
import os
import subprocess
import sys
import threading
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
DEV = "cuda"
SENT = -1                            # 0xFFFFFFFF: above every canonical word
GUARD = 2                            # sentinel rows before and after every rank's rows
CHUNK = 1 << 25                      # int64 elements per fill / comparison step
ECUDA = -2
KNOBS = ("FASTECC_B200_NO_TMA", "FASTECC_B200_SPLIT", "FASTECC_B200_CTAS_PER_SM")
LIB = os.path.join(ROOT, "fastecc_b200", "libfastecc_b200.so")


# ---- which shapes shard (csrc/plan.h, default split), checked against the library by test_support_rules_match_the_library ----
def split(LN):
    """(L1, L2) of the sharded plans: L1 = ceil(LN/2) capped at 9, within [5, 10] for both factors"""
    L1 = max(min((LN + 1) // 2, 9), 5)
    if LN - L1 > 10:
        L1 = LN - 10
    return L1, LN - L1


def lg(G):
    return G.bit_length() - 1


def shard_ok(LN, G):
    """the exchange-by-caller passes: G divides both factors"""
    L1, L2 = split(LN)
    return 11 <= LN <= 19 and G >= 2 and lg(G) <= min(L1, L2)


def p2p_encode_ok(LN, G):
    L1, L2 = split(LN)
    return shard_ok(LN, G) and G <= 8 and min(L1, L2) >= 5 + lg(G)


def p2p_ntt_ok(LN, G):
    L1, L2 = split(LN)
    return 11 <= LN <= 20 and 2 <= G <= 8 and L1 >= 5 + lg(G) and L2 >= lg(G)


GS = (2, 4, 8)
P2P_ENCODES = [(LN, G) for LN in range(12, 20) for G in GS if p2p_encode_ok(LN, G)]
P2P_NTTS = [(LN, G) for LN in range(11, 21) for G in GS if p2p_ntt_ok(LN, G)]
SHAPES = [(5, 12), (36, 40), (64, 64)]                 # (SIZE, pitch): a partial chunk, two strips of a narrow 512-row tile, full


def shape(LN, G):
    return SHAPES[(LN + lg(G)) % len(SHAPES)]


def exchange_cases():
    """G = 2, 4, 8, 16 and the largest G at every order; at 2^18 a SIZE whose wide fused tiles are fewer than the SMs for some G
    (5 words: one strip per row set) and one with more (300 words: five strips)"""
    out = []
    for LN in range(11, 20):
        top = 1 << min(split(LN))
        for G in sorted({2, 4, 8, 16, top}):
            if not shard_ok(LN, G):
                continue
            for S, pitch in ([(5, 12), (300, 304)] if LN == 18 else [shape(LN, G)]):
                out.append((LN, G, S, pitch))
    return out


EXCHANGE_CASES = exchange_cases()


# ---- buffers --------------------------------------------------------------------------------------------------------------
def to_i32(t):
    return torch.where(t >= 1 << 31, t - (1 << 32), t).to(torch.int32)


def ceil4(n):
    return (n + 3) // 4 * 4


class Shards:
    """One role (X or Y) of G ranks: [G, GUARD + rows + GUARD, pitch] int32, every word the sentinel to begin with."""

    def __init__(self, G, rows, size, pitch):
        self.G, self.rows, self.size, self.pitch = G, rows, size, pitch
        self.full = torch.full((G, rows + 2 * GUARD, pitch), SENT, dtype=torch.int32, device=DEV)
        self.data = self.full[:, GUARD:GUARD + rows]

    def ptr(self, r, col=0):
        return self.full[r, GUARD].data_ptr() + 4 * col

    def peers(self, col=0):
        return (ctypes.c_void_p * self.G)(*[self.ptr(r, col) for r in range(self.G)])

    def reset(self):
        self.full.fill_(SENT)

    def check_untouched(self, what):
        """no guard row and no pad word past ceil4(SIZE) changed"""
        for name, part in (("leading guard", self.full[:, :GUARD]), ("trailing guard", self.full[:, GUARD + self.rows:]),
                           ("pad past ceil4(SIZE)", self.data[:, :, ceil4(self.size):])):
            bad = part != SENT
            if bool(bad.any()):
                idx = bad.nonzero()[:4].tolist()
                raise AssertionError("%s: %d words of the %s changed, first at (rank, row, col) %s" % (what, int(bad.sum()), name, idx))


def spans(sh):
    """(rank index, first row, end row, global blocks) steps over every rank's rows: global block of row l of rank r = l*G + r"""
    per = max(1, CHUNK // max(sh.size, 1))
    if sh.G * sh.rows <= per:
        g = torch.arange(sh.rows, dtype=torch.int64, device=DEV)[None, :] * sh.G + torch.arange(sh.G, dtype=torch.int64, device=DEV)[:, None]
        yield slice(None), 0, sh.rows, g.reshape(-1)
        return
    for r in range(sh.G):
        for l0 in range(0, sh.rows, per):
            l1 = min(sh.rows, l0 + per)
            yield r, l0, l1, torch.arange(l0, l1, dtype=torch.int64, device=DEV) * sh.G + r


def fill(sh, gen):
    """words [0, SIZE) of global block b = gen(b) (int64 words)"""
    for r, l0, l1, g in spans(sh):
        v = to_i32(gen(g))
        sh.data[r, l0:l1, :sh.size] = v.view(sh.G, l1 - l0, sh.size) if isinstance(r, slice) else v


def expect(sh, gen, what):
    """every word [0, SIZE) of global block b equals gen(b) (canonical), and sentinels are intact"""
    for r, l0, l1, g in spans(sh):
        got = R.as_words(sh.data[r, l0:l1, :sh.size]).reshape(-1, sh.size)
        want = gen(g)
        bad = got != want
        if bool(bad.any()):
            idx = bad.nonzero()[:4].tolist()
            detail = ["block %d col %d: got %d want %d" % (int(g[i]), c, int(got[i, c]), int(want[i, c])) for i, c in idx]
            raise AssertionError("%s: %d of %d words differ; %s" % (what, int(bad.sum()), bad.numel(), "; ".join(detail)))
    sh.check_untouched(what)


def below_p(sh, what):
    bad = R.as_words(sh.data[:, :, :sh.size]) >= P
    assert not bool(bad.any()), "%s: %d output words >= P, first at %s" % (what, int(bad.sum()), bad.nonzero()[:4].tolist())


# ---- the library --------------------------------------------------------------------------------------------------------------
def fe():
    import fastecc_b200
    return fastecc_b200


def call(rc):
    fe()._check(rc)


def stream():
    return torch.cuda.current_stream().cuda_stream


def geometry(N, G):
    n1, n2, ok = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_int()
    rc = fe().lib().fastecc_b200_shard_geometry(N, G, ctypes.byref(n1), ctypes.byref(n2), ctypes.byref(ok))
    return rc, n1.value, n2.value, ok.value


# ---- the all-ranks-in-one-process drivers ----------------------------------------------------------------------------------------
def encode_p2p(N, X, Y, col=0, width=None):
    """the exchange fused into the stores: pass 0 of every rank (X_r -> the Ys), pass 1 (Y_r -> the Xs), pass 2 (in place on X_r).
    Words [col, col + width) of every row (column-chunk pointers, SIZE = width, the full pitch).  Before pass 1 the chunk of every
    X is overwritten with the sentinel: pass 1 has to store every word of it."""
    L, st, G = fe().lib(), stream(), X.G
    w = X.size if width is None else width
    yp, xp = Y.peers(col), X.peers(col)
    for r in range(G):
        call(L.fastecc_b200_rs_encode_shard_pass_p2p(X.ptr(r, col), yp, N, G, r, w, X.pitch, 0, st))
    X.data[:, :, col:col + ceil4(w)] = SENT
    for r in range(G):
        call(L.fastecc_b200_rs_encode_shard_pass_p2p(Y.ptr(r, col), xp, N, G, r, w, X.pitch, 1, st))
    for r in range(G):
        call(L.fastecc_b200_rs_encode_shard_pass_p2p(X.ptr(r, col), xp, N, G, r, w, X.pitch, 2, st))


def ntt_p2p(N, X, Y, inverse):
    """pass A' of every rank (X_r -> the Ys), then pass B' (Y_r -> X_r); X is overwritten with the sentinel in between"""
    L, st, G = fe().lib(), stream(), X.G
    yp, xp = Y.peers(), X.peers()
    for r in range(G):
        call(L.fastecc_b200_ntt_shard_pass_p2p(X.ptr(r), yp, N, G, r, X.size, X.pitch, int(inverse), 0, st))
    X.data[:, :, :ceil4(X.size)] = SENT
    for r in range(G):
        call(L.fastecc_b200_ntt_shard_pass_p2p(Y.ptr(r), xp, N, G, r, X.size, X.pitch, int(inverse), 1, st))


def route(kind, N, G, N1, N2, r, device=None):
    """(source row, destination rank, destination row) of every row rank r's pass sends away, from the ownership formulas:
    "a" / "bc" the encode's exchanges after pass 0 / pass 1; "ntt" the store targets of the transform's pass A' (element k1 of
    the transform over n1 of local set n2' goes to rank k1 mod G, row (n2'*G + r)*(N1/G) + k1/G)."""
    l = torch.arange(N // G, dtype=torch.int64, device=device or DEV)
    if kind == "a":
        k1, n2p = l // (N2 // G), l % (N2 // G)
        return l, k1 % G, (k1 // G) * N2 + n2p * G + r
    if kind == "bc":
        k1p, j2 = l // N2, l % N2
        return l, j2 % G, (k1p * G + r) * (N2 // G) + j2 // G
    n2p, k1 = l // N1, l % N1
    return None, k1 % G, (n2p * G + r) * (N1 // G) + k1 // G


def exchange(src, dst, kind, N, N1, N2):
    """the caller's all-to-all of whole blocks (words [0, SIZE)) between two sets of shards"""
    G = src.G
    rr = torch.arange(G, dtype=torch.int64, device=DEV)[:, None]
    s_row, d_rank, d_row = route(kind, N, G, N1, N2, rr)
    s_row = s_row[None, :].expand(G, -1)
    assert torch.unique(d_rank * (N // G) + d_row).numel() == N            # a permutation of the blocks
    dst.data[d_rank, d_row, :src.size] = src.data[rr.expand(G, N // G), s_row, :src.size]


def encode_shard(N, X):
    """exchange by the caller: pass 0 in place on every X_r, exchange into fresh shards, pass 1, exchange, pass 2; returns the
    shards holding the parity (X and the intermediate shards are checked for untouched sentinels)."""
    L, st, G = fe().lib(), stream(), X.G
    rc, N1, N2, _ = geometry(N, G)
    assert rc == 0
    bufs = [X, Shards(G, X.rows, X.size, X.pitch), Shards(G, X.rows, X.size, X.pitch)]
    for which in range(3):
        cur = bufs[which]
        for r in range(G):
            call(L.fastecc_b200_rs_encode_shard_pass(cur.ptr(r), N, G, r, cur.size, cur.pitch, which, st))
        if which < 2:
            exchange(cur, bufs[which + 1], "a" if which == 0 else "bc", N, N1, N2)
    for k, b in enumerate(bufs[:2]):
        b.check_untouched("encode_shard N=%d G=%d, shards after pass %d" % (N, G, k))
    return bufs[2]


# ---- references ------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=4)
def oracle_pair(kind, N, S):
    """(fill_B of N x S, its oracle encode / forward / inverse transform) as device int64 tensors indexed by global block"""
    o = ol.load_oracle()
    a = ol.fill_B(o, N, S)
    out = ol.o_encode(o, a) if kind == "encode" else ol.o_ntt(o, a, kind == "intt")
    dev = lambda x: torch.from_numpy(x.astype(np.int64)).to(DEV)
    return dev(a), dev(out)


def boundaries(N, G):
    L1, L2 = split(N.bit_length() - 1)
    return (1 << L1, 1 << L2, G << L1, G << L2, (1 << L2) // G, (1 << L1) // G)


def encode_reference(N, G, S, seed=0):
    """(input generator, expected parity generator) over global blocks: the oracle below 2^17, monomial stripes from there"""
    if N < 1 << 17:
        a, want = oracle_pair("encode", N, S)
        return (lambda b: a[b]), (lambda b: want[b]), "oracle fill_B"
    degs = R.special_values(N, boundaries(N, G), count=S, seed=seed)[:S]
    return (lambda b: R.monomial_data(N, degs, b, DEV)), (lambda b: R.monomial_parity(N, degs, b, DEV)), "monomials %s" % degs[:6]


def ntt_reference(N, G, S, inverse, seed=0):
    if N < 1 << 17:
        a, want = oracle_pair("intt" if inverse else "ntt", N, S)
        return (lambda b: a[b]), (lambda b: want[b]), "oracle fill_B"
    vals = R.special_values(N, boundaries(N, G), count=S, seed=seed)[:S]
    h = S // 2                                                # columns [0, h): deltas; [h, S): geometric columns
    pos = torch.tensor(vals[:h], dtype=torch.int64, device=DEV)
    freq = vals[h:]

    def data(b):
        return torch.cat([(b[:, None] == pos[None, :]).to(torch.int64), R.geometric_ntt_input(N, freq, b, DEV, inverse)], 1)

    def want(b):
        return torch.cat([R.delta_ntt_columns(N, vals[:h], b, DEV, inverse), R.ntt_spike(N, freq, b, DEV)], 1)
    return data, want, "deltas at %s, geometric columns of %s" % (vals[:min(h, 4)], freq[:4])


def run_encode_p2p(N, G, S, pitch, seed=0):
    data, want, what = encode_reference(N, G, S, seed)
    X, Y = Shards(G, N // G, S, pitch), Shards(G, N // G, S, pitch)
    fill(X, data)
    encode_p2p(N, X, Y)
    desc = "fused-exchange encode N=2^%d G=%d SIZE=%d pitch=%d (%s)" % (N.bit_length() - 1, G, S, pitch, what)
    expect(X, want, desc)
    Y.check_untouched(desc + ", Y")
    return X, Y


# ==== CPU: the support rules and the exchange formulas ==========================================================================
def _lib_or_skip():
    if not os.path.exists(LIB):
        pytest.skip("needs the built library")
    if any(k in os.environ for k in KNOBS):
        pytest.skip("a launcher setting is in the environment")
    return fe()


def test_support_rules_match_the_library():
    """The rules the matrix below is drawn from are the library's: for every N = 2^1 .. 2^21 and G = 1 .. 2048, the shard
    geometry's N1 / N2, its fused-exchange bits and its verdict.  In particular G must divide N1 as well as N2."""
    _lib_or_skip()
    for LN in range(1, 22):
        for G in [1 << k for k in range(12)]:
            rc, n1, n2, ok = geometry(1 << LN, G)
            if LN > 10:
                assert (n1, n2) == tuple(1 << x for x in split(LN)), (LN, G)
            want_ok = (p2p_encode_ok(LN, G) and 1) | (p2p_ntt_ok(LN, G) and 2)
            assert ok == want_ok, (LN, G, ok)
            assert (rc == 0) == (G == 1 or shard_ok(LN, G) or p2p_ntt_ok(LN, G)), (LN, G, rc)
    assert geometry(1 << 19, 1024)[0] == -1 and geometry(1 << 19, 512)[0] == 0


def test_matrix_reaches_every_sharded_instantiation():
    """The fused-exchange encodes and transforms below run every <LR, NXF, 2> instantiation: LR 6 .. 10 with NXF 1 (pass A' of the
    transform, pass 0 of the encode) and NXF 2 (pass 1 of the encode)."""
    reached = set()
    for LN, G in P2P_ENCODES:
        L1, L2 = split(LN)
        reached |= {(L1, 1), (L2, 2)}
    for LN, G in P2P_NTTS:
        reached.add((split(LN)[0], 1))
    assert reached == {(lr, nxf) for lr in range(6, 11) for nxf in (1, 2)}, sorted(reached)
    assert (19, 8) in P2P_ENCODES and (20, 8) in P2P_NTTS and (12, 2) in P2P_ENCODES
    assert any(ceil4(S) != S for _, _, S, _ in EXCHANGE_CASES) and all(p > ceil4(S) for S, p in SHAPES[:2])


def test_exchange_formulas_equal_the_python_orchestration(monkeypatch):
    """The test-local exchanges (from the ownership formulas) move every block where fastecc_b200/sharded.py's do, with a
    simulated all-to-all on CPU tensors."""
    _lib_or_skip()
    from fastecc_b200 import sharded

    class Sent(Exception):
        pass
    for LN, G in ((11, 2), (13, 4), (16, 8), (19, 16), (19, 512)):
        N = 1 << LN
        _, N1, N2, _ = geometry(N, G)
        block = torch.arange(N, dtype=torch.int32)[:, None].repeat(1, 2)      # its global block number in every word
        shards = [block[r::G].contiguous() for r in range(G)]
        for kind, fn in (("a", sharded.exchange_after_a), ("bc", sharded.exchange_after_bc)):
            sends = {}

            def deposit(send, group):
                sends[group] = send
                raise Sent
            monkeypatch.setattr(sharded, "_all_to_all", deposit)
            for r in range(G):
                with pytest.raises(Sent):
                    fn(shards[r], N, G, group=r)
            recv = [torch.stack([sends[s][r] for s in range(G)]) for r in range(G)]
            monkeypatch.setattr(sharded, "_all_to_all", lambda send, group: recv[group])
            got = torch.stack([fn(shards[r], N, G, group=r)[:, 0] for r in range(G)])
            rr = torch.arange(G, dtype=torch.int64)[:, None]
            s_row, d_rank, d_row = route(kind, N, G, N1, N2, rr, device="cpu")
            mine = torch.full((G, N // G), -1, dtype=torch.int32)
            mine[d_rank, d_row] = torch.stack(shards)[rr.expand(G, N // G), s_row[None, :].expand(G, -1), 0]
            assert torch.equal(got, mine), (LN, G, kind)


# ==== GPU: the fused-exchange encode and transform against the oracle and closed forms ===========================================
@pytest.mark.gpu
@pytest.mark.parametrize("LN,G", P2P_ENCODES)
def test_fused_exchange_encode(fecc, LN, G):
    assert geometry(1 << LN, G)[3] & 1
    S, pitch = shape(LN, G)
    run_encode_p2p(1 << LN, G, S, pitch, seed=LN)
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("LN,G", P2P_NTTS)
def test_fused_exchange_transform(fecc, LN, G):
    assert geometry(1 << LN, G)[3] & 2
    N = 1 << LN
    S, pitch = shape(LN, G)
    for inverse in (False, True):
        data, want, what = ntt_reference(N, G, S, inverse, seed=LN)
        X, Y = Shards(G, N // G, S, pitch), Shards(G, N // G, S, pitch)
        fill(X, data)
        ntt_p2p(N, X, Y, inverse)
        desc = "fused-exchange %s transform N=2^%d G=%d SIZE=%d pitch=%d (%s)" % ("inverse" if inverse else "forward", LN, G, S, pitch, what)
        expect(X, want, desc)
        Y.check_untouched(desc + ", Y")
    torch.cuda.empty_cache()


# ==== GPU: exchange by the caller ==================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("LN,G,S,pitch", EXCHANGE_CASES)
def test_exchange_by_caller_encode(fecc, LN, G, S, pitch):
    N = 1 << LN
    data, want, what = encode_reference(N, G, S, seed=LN + G)
    X = Shards(G, N // G, S, pitch)
    fill(X, data)
    out = encode_shard(N, X)
    expect(out, want, "exchange-by-caller encode N=2^%d G=%d SIZE=%d pitch=%d (%s)" % (LN, G, S, pitch, what))
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_2_to_the_18_runs_the_fused_pass_narrow_and_wide(fecc):
    """launch_pass runs pass 1 of a 2^18 exchange-by-caller encode (<9,2,1>, 512-row tiles) on the narrow twin when the wide
    geometry would have fewer tiles than SMs: the cases above include both sides of that line for some G."""
    sms = fecc.lib().fastecc_b200_num_sms()
    narrow = set()
    for LN, G, S, _ in EXCHANGE_CASES:
        if LN == 18:
            tiles = (512 // G) * -(-ceil4(S) // 64)          # row sets x strips of 64 words (a wide 512-row tile)
            narrow.add(tiles < sms)
    assert narrow == {True, False}, (sms, narrow)


# ==== GPU: where the peer stores land ================================================================================================
def written_rows(sh, what):
    """[G, rows] masks: rows with any word changed, rows with every word of [0, ceil4(SIZE)) changed"""
    any_ = (sh.data != SENT).any(-1)
    all_ = (sh.data[:, :, :ceil4(sh.size)] != SENT).all(-1)
    sh.check_untouched(what)
    return any_, all_


@pytest.mark.gpu
@pytest.mark.parametrize("G", GS)
@pytest.mark.parametrize("kind", ["a", "bc", "ntt"])
def test_peer_stores_land_on_their_owner_rows(fecc, G, kind):
    """Rank r's pass alone, into freshly sentinelled peers: on every peer it writes exactly the rows the ownership formula gives
    (all words of them, nothing else), it leaves its source alone, and over all r these row sets partition every peer's rows."""
    N, S, pitch = 1 << 16, 5, 12
    rc, N1, N2, ok = geometry(N, G)
    assert rc == 0 and ok == 3
    L, st = fecc.lib(), stream()
    src, dst = Shards(G, N // G, S, pitch), Shards(G, N // G, S, pitch)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(G)
    src.data[:, :, :S] = to_i32(torch.randint(0, P, (G, N // G, S), device=DEV, generator=gen, dtype=torch.int64))
    before = src.full.clone()
    cover = torch.zeros((G, N // G), dtype=torch.int32, device=DEV)
    for r in range(G):
        dst.reset()
        if kind == "ntt":
            call(L.fastecc_b200_ntt_shard_pass_p2p(src.ptr(r), dst.peers(), N, G, r, S, pitch, 0, 0, st))
        else:
            call(L.fastecc_b200_rs_encode_shard_pass_p2p(src.ptr(r), dst.peers(), N, G, r, S, pitch, 0 if kind == "a" else 1, st))
        what = "%s stores of rank %d of %d" % (kind, r, G)
        any_, all_ = written_rows(dst, what)
        _, d_rank, d_row = route(kind, N, G, N1, N2, r)
        want = torch.zeros((G, N // G), dtype=torch.bool, device=DEV)
        want[d_rank, d_row] = True
        for name, got in (("rows written at all", any_), ("rows written in full", all_)):
            bad = got != want
            assert not bool(bad.any()), "%s: %s differ from the formula at %d rows, first (peer, row) %s" % (
                what, name, int(bad.sum()), bad.nonzero()[:4].tolist())
        assert torch.equal(src.full, before), what + ": the source changed"
        cover += want.to(torch.int32)
    assert bool((cover == 1).all())


# ==== GPU: inputs and layouts ==========================================================================================================
def raw_words(G, rows, S, seed):
    gen = torch.Generator(device=DEV)
    gen.manual_seed(seed)
    x = torch.randint(0, 1 << 32, (G, rows, S), device=DEV, generator=gen, dtype=torch.int64)
    x[:, ::7] = 0xFFFFFFFF
    x[:, 1::7] = P + torch.arange(S, device=DEV)
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("op,LN,G", [("encode_p2p", 14, 2), ("encode_p2p", 19, 8), ("ntt_p2p", 16, 4), ("intt_p2p", 20, 8), ("encode_shard", 13, 4)])
def test_raw_words_equal_their_residues(fecc, op, LN, G):
    """32-bit words >= P in X give bit for bit the output of their residues"""
    N, S, pitch = 1 << LN, 5, 12
    raw = raw_words(G, N // G, S, LN)
    outs = []
    for x in (raw, raw % P):
        X, Y = Shards(G, N // G, S, pitch), Shards(G, N // G, S, pitch)
        X.data[:, :, :S] = to_i32(x)
        if op == "encode_shard":
            X = encode_shard(N, X)
        elif op == "encode_p2p":
            encode_p2p(N, X, Y)
        else:
            ntt_p2p(N, X, Y, op == "intt_p2p")
        what = "%s N=2^%d G=%d" % (op, LN, G)
        X.check_untouched(what)
        Y.check_untouched(what)
        below_p(X, what)
        outs.append(X.data[:, :, :S].clone())
    bad = (outs[0] != outs[1]).nonzero()[:8].tolist()
    assert not bad, bad


@pytest.mark.gpu
def test_column_chunks_equal_the_whole_rows(fecc):
    """The passes on column chunks the way P2PShardedEncoder.encode_host runs them: pointers offset by c0 words, SIZE = the chunk
    width, the full pitch, chunks of 256 words and a partial last one; the parity equals the whole-row encode and the oracle."""
    N, G, S, pitch, cw = 1 << 15, 4, 1000, 1008, 256
    data, want, _ = encode_reference(N, G, S)
    whole, _ = run_encode_p2p(N, G, S, pitch)
    X, Y = Shards(G, N // G, S, pitch), Shards(G, N // G, S, pitch)
    fill(X, data)
    for c0 in range(0, S, cw):
        encode_p2p(N, X, Y, c0, min(cw, S - c0))
    expect(X, want, "fused-exchange encode in column chunks of %d words" % cw)
    Y.check_untouched("column chunks, Y")
    assert torch.equal(X.full, whole.full)


# ==== GPU: the headline shapes against the reference's golden hashes ====================================================================
def gather_hash(X):
    """the reference's hash (main.cpp:203-212) of the cyclic shards reassembled in global block order"""
    G, rows, S = X.G, X.rows, X.size
    full = np.empty((G * rows, S), dtype=np.uint32)
    for r in range(G):
        full[r::G] = X.data[r, :, :S].cpu().numpy().view(np.uint32)
    return fe().reference_hash(full)


def fill_a(N, S):
    return lambda b: (b[:, None] * S + torch.arange(S, dtype=torch.int64, device=DEV)[None, :]) % P      # data0[i] = i % P


def golden():
    return json.load(open(os.path.join(HERE, "golden", "survey_8c.json")))


@pytest.mark.gpu
def test_fused_exchange_encode_headline_hash(fecc):
    """2^19 x 1024 words of fill A over 8 ranks: the parity hashes to the reference's 4272226309"""
    N, G, S = 1 << 19, 8, 1024
    _, _, h0, h1 = [g for g in golden()["encode_fillA"] if g[0] == 19 and g[1] == S][0]
    X, Y = Shards(G, N // G, S, S), Shards(G, N // G, S, S)
    fill(X, fill_a(N, S))
    assert gather_hash(X) == h0
    encode_p2p(N, X, Y)
    X.check_untouched("headline encode")
    Y.check_untouched("headline encode, Y")
    below_p(X, "headline encode")
    assert gather_hash(X) == h1 == 4272226309
    del X, Y
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("LN,G", [(19, 4), (20, 8)])
def test_fused_exchange_transform_headline_hash(fecc, LN, G):
    """ntt of 2^19 and 2^20 blocks of 4096 bytes of fill A: the reference's golden hashes of the input and the transform"""
    N, S = 1 << LN, 1024
    h0, h1 = golden()["ntt_fillA_4096B"][str(LN)]
    X, Y = Shards(G, N // G, S, S), Shards(G, N // G, S, S)
    fill(X, fill_a(N, S))
    assert gather_hash(X) == h0
    ntt_p2p(N, X, Y, False)
    X.check_untouched("headline transform")
    Y.check_untouched("headline transform, Y")
    below_p(X, "headline transform")
    assert gather_hash(X) == h1
    del X, Y
    torch.cuda.empty_cache()


# ==== GPU: buffers past 2^32 bytes ====================================================================================================
@pytest.mark.gpu
def test_fused_exchange_encode_past_2_to_the_32_bytes(fecc):
    """G = 2, N = 2^19, SIZE = 4100: each rank's X and Y hold 2^18 rows of 16400 bytes, 4.3 GB; every word by closed form"""
    GiB = 1 << 30
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < 24 * GiB:
        pytest.skip("%.1f GiB free on the device; this case needs about 24 GiB" % (free / GiB))
    N, G, S = 1 << 19, 2, 4100
    assert (N // G) * S * 4 > 1 << 32
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    run_encode_p2p(N, G, S, S, seed=3)
    torch.cuda.synchronize()
    print("2^19 x 4100 over 2 ranks: %.1f s, peak %.1f GiB allocated by torch" % (time.time() - t0, torch.cuda.max_memory_allocated() / GiB))
    torch.cuda.empty_cache()


# ==== GPU: the barrier kernel, only where its wait is already satisfied ===============================================================
BARRIER_FILL = 0x5A5A5A5A


def u32(x):
    return x - (1 << 32) if x >= 1 << 31 else x


def run_barrier(F, n, rank, epoch):
    """rank's barrier over the flag arrays F[0 .. n) (16 words each); returns the host time to completion"""
    arr = (ctypes.c_void_p * n)(*[F[p].data_ptr() for p in range(n)])
    torch.cuda.synchronize()
    t0 = time.time()
    call(fe().lib().fastecc_b200_shard_barrier(arr, n, rank, epoch, stream()))
    torch.cuda.synchronize()
    return time.time() - t0


def barrier_flags(n, rank, epoch, others, previous):
    """flag arrays before rank's barrier: the other ranks' words of rank's own array at `others` (arrived), every other word
    [0, n) at `previous`, word [8] (the error word) 0, the rest a fill pattern"""
    F = torch.full((n, 16), u32(BARRIER_FILL), dtype=torch.int32, device=DEV)
    F[:, :n] = u32(previous)
    F[:, 8] = 0
    for p in range(n):
        if p != rank:
            F[rank, p] = u32(others)
    return F


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 8])
def test_barrier_publishes_its_epoch(fecc, n):
    """Word [rank] of every peer's array becomes the epoch; the error word [8] stays 0; words [n, 8) and [9, 16) and the other
    ranks' words are untouched."""
    for rank in range(n):
        epoch = 5 + 3 * rank
        F = barrier_flags(n, rank, epoch, epoch, epoch - 1)
        want = F.clone()
        want[:, rank] = epoch
        dt = run_barrier(F, n, rank, epoch)
        assert torch.equal(F, want), (n, rank, F.tolist())
        assert dt < 2.0, dt


@pytest.mark.gpu
@pytest.mark.parametrize("epoch,others,previous", [(0, 0, 0xFFFFFFFF), (5, 6, 4), (0xFFFFFFFF, 0, 0xFFFFFFFE), (7, 0x80000006, 6)],
                         ids=["epoch_0_after_wrap", "flag_ahead", "flag_ahead_across_wrap", "flag_half_ahead"])
def test_barrier_wraps_around(fecc, epoch, others, previous):
    """The flags compare as a signed difference: epoch 0 after 0xFFFFFFFF, and a flag ahead of the epoch (a rank already at its
    next barrier), both return at once."""
    n, rank = 2, 0
    F = barrier_flags(n, rank, epoch, others, previous)
    want = F.clone()
    want[:, rank] = u32(epoch)
    dt = run_barrier(F, n, rank, epoch)
    assert torch.equal(F, want), F.tolist()
    assert dt < 2.0, dt


# ==== GPU: the Python orchestration on CUDA tensors ====================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("LN,G,S", [(16, 2, 64), (16, 4, 64), (16, 8, 64), (19, 8, 1024)])
def test_rs_encode_sharded_with_one_thread_per_rank(fecc, monkeypatch, LN, G, S):
    """sharded.rs_encode_sharded with gpu_pass_runner, one host thread per rank; the all-to-all is an in-process rendezvous
    (each rank deposits its send, waits for all, takes recv[src] = sends[src][rank], waits again), `group` is the rank"""
    from fastecc_b200 import sharded
    N = 1 << LN
    rows = N // G
    sends = [None] * G
    bar = threading.Barrier(G, timeout=120)

    def all_to_all(send, group):
        sends[group] = send
        bar.wait()
        recv = torch.stack([sends[s][group] for s in range(G)])
        bar.wait()
        return recv
    monkeypatch.setattr(sharded, "_all_to_all", all_to_all)
    if LN == 19:
        gen, want = fill_a(N, S), None
        h1 = [g for g in golden()["encode_fillA"] if g[0] == 19 and g[1] == S][0][3]
    else:
        gen, want, _ = encode_reference(N, G, S)
    X = Shards(G, rows, S, S)
    fill(X, gen)
    local = [X.data[r].contiguous() for r in range(G)]
    del X
    outs, errors = [None] * G, []

    def worker(r):
        try:
            outs[r] = sharded.rs_encode_sharded(local[r], N, G, sharded.gpu_pass_runner(N, G, r), group=r)
        except BaseException as e:                     # noqa: BLE001 -- re-raised below
            errors.append(e)
            bar.abort()
    threads = [threading.Thread(target=worker, args=(r,)) for r in range(G)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    torch.cuda.synchronize()
    out = Shards(G, rows, S, S)
    out.data.copy_(torch.stack(outs))
    if want is None:
        below_p(out, "rs_encode_sharded 2^19")
        assert gather_hash(out) == h1
    else:
        expect(out, want, "rs_encode_sharded N=2^%d G=%d" % (LN, G))
    del out, outs, local
    torch.cuda.empty_cache()


# ==== child processes: the launcher's settings ===========================================================================================
def child(mode, env_extra, timeout=600):
    torch.cuda.empty_cache()
    env = {k: v for k, v in os.environ.items() if k not in KNOBS}
    env.update(env_extra)
    t0 = time.time()
    p = subprocess.Popen([sys.executable, os.path.abspath(__file__), mode], cwd=ROOT, env=env,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        out, _ = p.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        p.kill()
        out, _ = p.communicate()
        pytest.fail("child %s timed out after %d s:\n%s" % (mode, timeout, out[-4000:]))
    print(out)
    print("child %s: %.1f s" % (mode, time.time() - t0))
    assert p.returncode == 0, out[-6000:]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("mode,env", [("no_tma", {"FASTECC_B200_NO_TMA": "1"}), ("split_lo", {"FASTECC_B200_SPLIT": "lo"})])
def test_launcher_settings(fecc, mode, env):
    assert "sharded %s ok" % mode in child(mode, env)


def _rejects_without_launch(fn, *args):
    L = fe().lib()
    before = L.fastecc_b200_kernel_launches()
    rc = fn(*args)
    assert rc == -1, (args, rc)
    assert L.fastecc_b200_kernel_launches() == before, args


def _no_tma():
    """The peer-store passes exist only as TMA instantiations: without TMA each fails with ECUDA and X and Y stay as they were.
    The local passes (encode pass 2, transform pass B') and the exchange-by-caller encode run on cp.async loads."""
    L, st = fe().lib(), stream()
    N, G, S, pitch = 1 << 16, 4, 5, 12
    X, Y = Shards(G, N // G, S, pitch), Shards(G, N // G, S, pitch)
    for A in (X, Y):
        A.data[:, :, :S] = to_i32(torch.randint(0, P, (G, N // G, S), device=DEV, dtype=torch.int64))
    x0, y0 = X.full.clone(), Y.full.clone()
    for name, f, args in (("encode pass 0", L.fastecc_b200_rs_encode_shard_pass_p2p, (X.ptr(1), Y.peers(), N, G, 1, S, pitch, 0)),
                          ("encode pass 1", L.fastecc_b200_rs_encode_shard_pass_p2p, (Y.ptr(1), X.peers(), N, G, 1, S, pitch, 1)),
                          ("transform pass A'", L.fastecc_b200_ntt_shard_pass_p2p, (X.ptr(1), Y.peers(), N, G, 1, S, pitch, 1, 0))):
        rc = f(*args, st)
        torch.cuda.synchronize()
        assert rc == ECUDA, (name, rc)
        assert torch.equal(X.full, x0) and torch.equal(Y.full, y0), name + " touched X or Y"
        print("ok %s: %s" % (name, L.fastecc_b200_last_error().decode()), flush=True)
    call(L.fastecc_b200_rs_encode_shard_pass_p2p(X.ptr(1), X.peers(), N, G, 1, S, pitch, 2, st))
    call(L.fastecc_b200_ntt_shard_pass_p2p(Y.ptr(1), X.peers(), N, G, 1, S, pitch, 0, 1, st))
    torch.cuda.synchronize()
    for LN, G, S, pitch in ((11, 2, 5, 12), (14, 8, 36, 40), (16, 16, 5, 12), (18, 4, 300, 304), (19, 8, 5, 12)):
        N = 1 << LN
        data, want, what = encode_reference(N, G, S, seed=LN)
        X = Shards(G, N // G, S, pitch)
        fill(X, data)
        expect(encode_shard(N, X), want, "no_tma exchange-by-caller encode N=2^%d G=%d (%s)" % (LN, G, what))
        print("ok exchange-by-caller encode 2^%d over %d ranks" % (LN, G), flush=True)


def _split_lo():
    """FASTECC_B200_SPLIT=lo: 2^11 = 32 x 64 cannot go to 64 ranks (pass 1 would have no row set), 2^19 not to 1024; the sharded
    passes follow the lower split (2^13 = 64 x 128 here, 128 x 64 by default)."""
    L = fe().lib()
    assert geometry(1 << 11, 64)[:3] == (-1, 32, 64)
    assert geometry(1 << 19, 1024)[0] == -1
    assert geometry(1 << 13, 4)[:3] == (0, 64, 128)
    x = torch.zeros((1 << 10, 4), dtype=torch.int32, device=DEV)
    for which in (0, 1, 2):
        _rejects_without_launch(L.fastecc_b200_rs_encode_shard_pass, x.data_ptr(), 1 << 11, 64, 0, 4, 4, which, stream())
        _rejects_without_launch(L.fastecc_b200_rs_encode_shard_pass, x.data_ptr(), 1 << 19, 1024, 0, 4, 4, which, stream())
    print("ok rejections", flush=True)
    for LN, G, S, pitch in ((11, 2, 5, 12), (11, 32, 5, 12), (13, 4, 36, 40), (19, 8, 5, 12)):
        N = 1 << LN
        data, want, what = encode_reference(N, G, S, seed=LN)
        X = Shards(G, N // G, S, pitch)
        fill(X, data)
        expect(encode_shard(N, X), want, "split lo exchange-by-caller encode N=2^%d G=%d (%s)" % (LN, G, what))
        print("ok exchange-by-caller encode 2^%d over %d ranks" % (LN, G), flush=True)
    for LN, G in ((13, 2), (16, 4), (19, 8)):
        assert geometry(1 << LN, G)[3] & 1
        run_encode_p2p(1 << LN, G, 5, 12, seed=LN)
        print("ok fused-exchange encode 2^%d over %d ranks" % (LN, G), flush=True)
    for LN, G in ((15, 4), (20, 8)):
        N = 1 << LN
        for inverse in (False, True):
            data, want, what = ntt_reference(N, G, 5, inverse, seed=LN)
            X, Y = Shards(G, N // G, 5, 12), Shards(G, N // G, 5, 12)
            fill(X, data)
            ntt_p2p(N, X, Y, inverse)
            expect(X, want, "split lo fused-exchange transform N=2^%d G=%d inverse=%d (%s)" % (LN, G, inverse, what))
            Y.check_untouched("split lo transform, Y")
        print("ok fused-exchange transform 2^%d over %d ranks" % (LN, G), flush=True)


if __name__ == "__main__":
    import fastecc_b200
    fastecc_b200.init(0)
    print("settings", {k: v for k, v in os.environ.items() if k.startswith("FASTECC_B200_")}, flush=True)
    {"no_tma": _no_tma, "split_lo": _split_lo}[sys.argv[1]]()
    print("sharded %s ok" % sys.argv[1], flush=True)
