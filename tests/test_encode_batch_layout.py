"""CPU: the layout rule of the batch encode (csrc/batch.h: batch_layout_disjoint), compiled for the host with nvcc.  Every layout
it accepts must really keep each parity word apart from every other parity word and every data word, which is checked by brute
force on word sets over thousands of small random lattices; and the layouts the header promises must be accepted."""
import ctypes
import itertools
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

HARNESS = r'''
#include "batch.h"
extern "C" int layout_ok(unsigned long long db, unsigned long long dp, unsigned long long ds, unsigned long long n,
                         unsigned long long pb, unsigned long long pp, unsigned long long ps, unsigned long long m,
                         unsigned long long b, unsigned long long size)
{
    return fecc::batch_layout_disjoint(fecc::BatchRows{db, dp, ds, n}, fecc::BatchRows{pb, pp, ps, m}, b, size);
}
'''


@pytest.fixture(scope="module")
def rule(tmp_path_factory):
    d = tmp_path_factory.mktemp("batch_layout")
    src, out = d / "harness.cu", str(d / "liblayout.so")
    src.write_text(HARNESS)
    cmd = ["/usr/local/cuda/bin/nvcc", "-Wno-deprecated-gpu-targets", "-O1", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-o", out, str(src),
           "-I" + os.path.join(ROOT, "fastecc_b200", "csrc")]
    subprocess.run(cmd, check=True, capture_output=True)
    L = ctypes.CDLL(out)
    L.layout_ok.argtypes = [ctypes.c_ulonglong] * 10
    L.layout_ok.restype = ctypes.c_int
    return lambda d, p, B, size: bool(L.layout_ok(*d, *p, B, size))


def rows(side, B):
    base, pitch, stride, n = side
    return [base + b * stride + i * pitch for b in range(B) for i in range(n)]


def disjoint(d, p, B, size):
    """No parity word is another parity word or a data word (data rows may overlap each other)"""
    seen = set()
    for r in rows(p, B):
        words = set(range(r, r + size))
        if words & seen:
            return False
        seen |= words
    data = set()
    for r in rows(d, B):
        data.update(range(r, r + size))
    return not (seen & data)


def ceil4(x):
    return (x + 3) // 4 * 4


def stripe_major(base, n, B, size, slack_pitch=0, slack_stride=0):
    pitch = ceil4(size) + 4 * slack_pitch
    return (base, pitch, (n - 1) * pitch + ceil4(size) + 4 * slack_stride if B > 1 else 4 * slack_stride, n)


def block_major(base, n, B, size, slack_pitch=0, slack_stride=0):
    stride = ceil4(size) + 4 * slack_stride
    return (base, (B - 1) * stride + ceil4(size) + 4 * slack_pitch, stride, n)


def extent(side, B, size):
    base, pitch, stride, n = side
    return base + (B - 1) * stride + (n - 1) * pitch + size


def test_random_lattices_accepted_only_when_disjoint(rule):
    rng = np.random.default_rng(11)
    accepted = 0
    for case in range(6000):
        B = int(rng.integers(1, 7))
        N = int(rng.integers(1, 11))
        M = int(rng.integers(1, 13 - N))
        size = int(rng.integers(1, 13))
        kind = case % 4
        if kind == 0:                                                    # separate buffers, each side stripe- or block-major
            mk = [stripe_major, block_major]
            d = mk[rng.integers(2)](0, N, B, size, int(rng.integers(0, 2)), int(rng.integers(0, 2)))
            p = mk[rng.integers(2)](0, M, B, size, int(rng.integers(0, 2)), int(rng.integers(0, 2)))
            shift = 4 * int(rng.integers(-4, 5)) + (extent(d, B, size) + 3) // 4 * 4 * int(rng.integers(0, 2))
            if shift >= 0:
                p = (p[0] + shift,) + p[1:]
            else:
                d = (d[0] - shift,) + d[1:]
        elif kind == 1:                                                  # one buffer: data progression, parity progression, common stride
            pitch = ceil4(size) + 4 * int(rng.integers(0, 2))
            below = bool(rng.integers(2))
            d0, p0 = (0, N * pitch) if below else (M * pitch, 0)
            d0 += 4 * int(rng.integers(-1, 2)) if d0 else 0
            p0 += 4 * int(rng.integers(-1, 2)) if p0 else 0
            stride = (N + M) * pitch + 4 * int(rng.integers(-2, 3))
            d, p = (d0, pitch, max(stride, 0), N), (p0, pitch, max(stride, 0), M)
        elif kind == 2:                                                  # one buffer, data in the even row slots, parity in the odd ones
            pitch = ceil4(size) + 4 * int(rng.integers(0, 2))
            stride = 2 * max(N, M) * pitch + 4 * int(rng.integers(-2, 3))
            d, p = (0, 2 * pitch, stride, N), (pitch + 4 * int(rng.integers(-1, 2)), 2 * pitch, stride, M)
        else:                                                            # anything: random pitches, strides and bases in 4-word steps
            d = (4 * int(rng.integers(0, 30)), ceil4(size) + 4 * int(rng.integers(0, 8)), 4 * int(rng.integers(0, 40)), N)
            p = (4 * int(rng.integers(0, 30)), ceil4(size) + 4 * int(rng.integers(0, 8)), 4 * int(rng.integers(0, 40)), M)
        ok = rule(d, p, B, size)
        truth = disjoint(d, p, B, size)
        assert truth or not ok, (d, p, B, size)
        accepted += ok
    assert accepted > 1500, accepted                                     # the rule is not vacuous


@pytest.mark.parametrize("B,N,M,size", [(1, 1, 1, 1), (5, 4, 2, 5), (6, 9, 3, 12), (3, 6, 6, 7), (2, 8, 4, 4), (4, 3, 1, 2)])
def test_separate_buffers_in_every_combination_are_accepted(rule, B, N, M, size):
    for dm, pm in itertools.product((stripe_major, block_major), repeat=2):
        for sp, ss in ((0, 0), (1, 0), (0, 2), (3, 1)):
            d = dm(0, N, B, size, sp, ss)
            p = pm(0, M, B, size, ss, sp)
            after = (extent(d, B, size) + 3) // 4 * 4 + 4 * sp
            assert rule(d, (after,) + p[1:], B, size), (dm.__name__, pm.__name__, sp, ss)
            before = (extent(p, B, size) + 3) // 4 * 4
            assert rule((before,) + d[1:], p, B, size), (dm.__name__, pm.__name__, sp, ss)


@pytest.mark.parametrize("B,N,M,size", [(1, 4, 2, 3), (5, 4, 2, 5), (6, 9, 3, 12), (3, 6, 6, 7), (2, 8, 4, 4), (4, 3, 1, 2), (3, 1, 1, 1)])
def test_one_buffer_with_the_parity_below_or_above_the_data_is_accepted(rule, B, N, M, size):
    for slack in (0, 1, 3):
        pitch = ceil4(size) + 4 * slack
        stride = (N + M) * pitch
        assert rule((M * pitch, pitch, stride, N), (0, pitch, stride, M), B, size)              # [B][N + M][pitch], parity below
        assert rule((0, pitch, stride, N), (N * pitch, pitch, stride, M), B, size)              # parity above
        assert rule((0, pitch, stride + 8, N), (N * pitch, pitch, stride + 8, M), B, size)      # slack between stripes


def test_one_buffer_in_any_row_order_is_accepted_when_the_sides_are_progressions(rule):
    """Stripe 0's rows in any order that keeps each side an arithmetic progression: interleaved D P D P .., blocks of data and
    parity in either order, and gaps between rows"""
    for B, N, M, size in ((4, 4, 4, 5), (3, 6, 3, 8), (2, 8, 8, 1), (5, 2, 1, 12)):
        pitch = ceil4(size)
        if M == N:
            d, p = (0, 2 * pitch, 2 * N * pitch, N), (pitch, 2 * pitch, 2 * N * pitch, M)
            assert rule(d, p, B, size)
            assert disjoint(d, p, B, size)
        d, p = (0, pitch + 4, (N + M) * (pitch + 4) + 4, N), (N * (pitch + 4), pitch + 4, (N + M) * (pitch + 4) + 4, M)
        assert rule(d, p, B, size) and disjoint(d, p, B, size)


def test_overlapping_parity_is_rejected(rule):
    size, B, N, M = 8, 3, 4, 2
    assert not rule((0, 8, 32, N), (1000, 8, 8, M), B, size)            # parity stripes overlap each other
    assert not rule((0, 8, 32, N), (1000, 4, 16, M), B, size)           # parity rows overlap within a stripe
    assert not rule((0, 8, 48, N), (24, 8, 48, M), B, size)             # parity on the last data row
    assert not rule((0, 8, 32, N), (16, 8, 32, M), 1, size)             # B = 1, parity on data rows 2 and 3
    assert rule((0, 8, 0, N), (1000, 8, 16, M), B, size)                # all stripes share the same data rows: allowed
