"""CPU: the layout rule of the batch update (csrc/batch.h: batch_update_layout_disjoint), compiled for the host with nvcc as
test_encode_batch_layout.py compiles the batch encode's.  The call writes into the stripes it reads, so every layout the rule
accepts must keep each written word (of the N data rows, which hold the changed ones, and of the M parity rows) apart from every
other written word and from every new word; that is checked by brute force on word sets over thousands of random three-sided
lattices.  The layouts the header promises must be accepted."""
import ctypes
import itertools
import os
import subprocess

import numpy as np
import pytest

from test_encode_batch_layout import block_major, ceil4, extent, rows, stripe_major

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

HARNESS = r'''
#include "batch.h"
typedef unsigned long long u64;
extern "C" int layout_ok(u64 db, u64 dp, u64 ds, u64 n, u64 pb, u64 pp, u64 ps, u64 m, u64 nb, u64 np, u64 ns, u64 k, u64 b, u64 size)
{
    return fecc::batch_update_layout_disjoint(fecc::BatchRows{db, dp, ds, n}, fecc::BatchRows{pb, pp, ps, m}, fecc::BatchRows{nb, np, ns, k}, b, size);
}
'''


@pytest.fixture(scope="module")
def rule(tmp_path_factory):
    d = tmp_path_factory.mktemp("update_layout")
    src, out = d / "harness.cu", str(d / "liblayout.so")
    src.write_text(HARNESS)
    cmd = ["/usr/local/cuda/bin/nvcc", "-Wno-deprecated-gpu-targets", "-O1", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-o", out, str(src),
           "-I" + os.path.join(ROOT, "fastecc_b200", "csrc")]
    subprocess.run(cmd, check=True, capture_output=True)
    L = ctypes.CDLL(out)
    L.layout_ok.argtypes = [ctypes.c_ulonglong] * 14
    L.layout_ok.restype = ctypes.c_int
    return lambda d, p, n, B, size: bool(L.layout_ok(*d, *p, *n, B, size))


def safe(d, p, n, B, size):
    """No written word (data or parity) is another written word or a new word; new rows may overlap each other"""
    seen = set()
    for r in rows(d, B) + rows(p, B):
        words = set(range(r, r + size))
        if words & seen:
            return False
        seen |= words
    new = set()
    for r in rows(n, B):
        new.update(range(r, r + size))
    return not (seen & new)


def shift(side, by):
    return (side[0] + by,) + side[1:]


def test_random_three_sided_lattices_accepted_only_when_safe(rule):
    rng = np.random.default_rng(17)
    accepted = 0
    mk = [stripe_major, block_major]
    for case in range(8000):
        B = int(rng.integers(1, 6))
        N = int(rng.integers(1, 8))
        M = int(rng.integers(1, 8))
        k = int(rng.integers(1, N + 1))
        size = int(rng.integers(1, 11))
        kind = case % 4
        if kind == 0:                                                    # three spans, each stripe- or block-major, shifted about
            sides = [mk[rng.integers(2)](0, r, B, size, int(rng.integers(0, 2)), int(rng.integers(0, 2))) for r in (N, M, k)]
            if rng.integers(3) == 0:
                sides[2] = (0, sides[2][1], 0, k)                        # every stripe the same new rows
            at = 0
            for i in rng.permutation(3):
                sides[i] = shift(sides[i], at + 4 * int(rng.integers(-3, 2)) if at else 0)
                at = (extent(sides[i], B, size) + 3) // 4 * 4
            d, p, n = sides
            d, p, n = [(max(s[0], 0),) + s[1:] for s in (d, p, n)]
        elif kind == 1:                                                  # one buffer [B][rows][pitch] in some row order, slack or not
            pitch = ceil4(size) + 4 * int(rng.integers(0, 2))
            order = rng.permutation(3)
            counts = (N, M, k)
            starts, at = [0, 0, 0], 0
            for i in order:
                starts[i] = max(at + 4 * int(rng.integers(-1, 2)) * int(rng.integers(0, 2)), 0)
                at += counts[i] * pitch
            stride = at + 4 * int(rng.integers(-2, 3))
            d, p, n = [(starts[i], pitch, max(stride, 0), counts[i]) for i in range(3)]
            if rng.integers(3) == 0:                                     # the new rows in a buffer of their own
                n = (at * B + 64, pitch, int(rng.integers(0, 2)) * k * pitch, k)
        elif kind == 2:                                                  # interleaved rows of one buffer
            pitch = ceil4(size)
            stride = 3 * max(N, M, k) * pitch + 4 * int(rng.integers(-2, 3))
            d, p, n = (0, 3 * pitch, stride, N), (pitch + 4 * int(rng.integers(-1, 2)), 3 * pitch, stride, M), (2 * pitch, 3 * pitch, stride, k)
            p = (max(p[0], 0),) + p[1:]
        else:                                                            # anything: random pitches, strides and bases in 4-word steps
            d, p, n = [(4 * int(rng.integers(0, 30)), ceil4(size) + 4 * int(rng.integers(0, 8)), 4 * int(rng.integers(0, 40)), r) for r in (N, M, k)]
        ok = rule(d, p, n, B, size)
        assert safe(d, p, n, B, size) or not ok, (d, p, n, B, size)
        accepted += ok
    assert accepted > 1500, accepted                                     # the rule is not vacuous


@pytest.mark.parametrize("B,N,M,k,size", [(1, 1, 1, 1, 1), (5, 4, 2, 1, 5), (6, 9, 3, 9, 12), (3, 6, 6, 2, 7), (2, 8, 4, 3, 4), (4, 3, 1, 2, 2)])
def test_separate_spans_in_every_combination_are_accepted(rule, B, N, M, k, size):
    for fd, fp, fn in itertools.product((stripe_major, block_major), repeat=3):
        for sp, ss in ((0, 0), (1, 0), (0, 2), (3, 1)):
            d = fd(0, N, B, size, sp, ss)
            p = shift(fp(0, M, B, size, ss, sp), (extent(d, B, size) + 3) // 4 * 4 + 4 * sp)
            n = shift(fn(0, k, B, size, sp, ss), (extent(p, B, size) + 3) // 4 * 4)
            assert rule(d, p, n, B, size), (fd.__name__, fp.__name__, fn.__name__, sp, ss)
            assert rule(shift(d, 4096), shift(p, 4096), (0,) + n[1:], B, size)                 # the new rows below the stripes
            assert rule(d, p, (n[0], n[1], 0, k), B, size)                                      # new_stripe_words = 0


@pytest.mark.parametrize("B,N,M,k,size", [(1, 4, 2, 1, 3), (5, 4, 2, 4, 5), (6, 9, 3, 2, 12), (3, 6, 6, 6, 7), (2, 8, 4, 1, 4), (3, 1, 1, 1, 1)])
def test_one_stripe_buffer_with_the_new_rows_apart_or_inside_is_accepted(rule, B, N, M, k, size):
    for slack in (0, 1, 3):
        pitch = ceil4(size) + 4 * slack
        stride = (N + M) * pitch
        d, p = (0, pitch, stride, N), (N * pitch, pitch, stride, M)
        apart = B * stride + 8
        assert rule(d, p, (apart, pitch, k * pitch, k), B, size)                               # [B][N + M][pitch], new rows apart
        assert rule(d, p, (apart, pitch, 0, k), B, size)
        stride = (N + M + k) * pitch                                                            # [B][N + M + k][pitch]
        assert rule((0, pitch, stride, N), (N * pitch, pitch, stride, M), ((N + M) * pitch, pitch, stride, k), B, size)
        assert rule((k * pitch, pitch, stride, N), ((k + N) * pitch, pitch, stride, M), (0, pitch, stride, k), B, size)


def test_unsafe_layouts_are_rejected(rule):
    size, B, N, M, k = 8, 3, 4, 2, 2
    d, p, n = (0, 8, 32, N), (1000, 8, 16, M), (2000, 8, 16, k)
    assert rule(d, p, n, B, size)
    assert not rule(d, p, (16, 8, 32, k), B, size)                     # new rows on data rows 2 and 3
    assert not rule(d, p, (1008, 8, 16, k), B, size)                   # new rows on parity rows
    assert not rule(d, (1000, 8, 8, M), n, B, size)                    # parity stripes overlap each other
    assert not rule((0, 8, 0, N), p, n, B, size)                       # every stripe the same data rows: written by all of them
    assert not rule((0, 8, 16, N), p, n, B, size)                      # data stripes overlap each other
    assert not rule(d, (24, 8, 32, M), n, B, size)                     # parity on the last data row
    assert not rule((0, 4, 32, N), p, n, B, size)                      # data rows overlap within a stripe
