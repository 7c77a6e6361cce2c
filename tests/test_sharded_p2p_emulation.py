"""CPU: the sharded encoder with the exchange fused into the stores (csrc/plan.h plan_encode_shard_p2p,
fastecc_b200_rs_encode_shard_pass_p2p).  All G ranks are simulated in one process: each rank's X / Y buffers are numpy
arrays, "peer memory" is simply the other ranks' arrays, and the pass descriptors the GPU path would launch are run on
the CPU emulation of the kernel (tests/emulate_lib.cu) -- so the store addressing (owner = element mod G, row on the
owner) is the production code.  Parity, reassembled from the cyclic shards, must equal the oracle bit for bit."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_lib as ol                                   # noqa: E402
from test_sharded_gloo import EMU, _build_emulator        # noqa: E402


def _ptr_array(arrs):
    return (ctypes.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])


@pytest.mark.parametrize("G,L,S", [(2, 12, 8), (2, 15, 12), (4, 14, 4), (8, 16, 4), (4, 17, 4), (8, 19, 4)])
def test_p2p_sharded_passes_match_oracle(G, L, S):
    _build_emulator()
    emu = ctypes.CDLL(EMU)
    f = emu.emu_rs_encode_shard_pass_p2p
    f.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int]
    N = 1 << L
    o = ol.load_oracle()
    full = ol.fill_B(o, N, S)
    X = [np.ascontiguousarray(full[r::G]) for r in range(G)]               # cyclic ownership: block l*G + r is row l on rank r
    Y = [np.full_like(X[0], 0xDEADBEEF) for _ in range(G)]
    yp, xp = _ptr_array(Y), _ptr_array(X)
    for r in range(G):                                                      # pass A: local X -> everybody's Y
        assert f(X[r].ctypes.data, yp, N, G, r, S, S, 0) == 0
    for x in X:
        x[:] = 0xDEADBEEF                                                   # every word of X must be rewritten by pass BC
    for r in range(G):                                                      # pass BC: local Y -> everybody's X
        assert f(Y[r].ctypes.data, xp, N, G, r, S, S, 1) == 0
    for r in range(G):                                                      # pass D: local, in place
        assert f(X[r].ctypes.data, xp, N, G, r, S, S, 2) == 0
    par = np.empty_like(full)
    for r in range(G):
        par[r::G] = X[r]
    assert np.array_equal(par, ol.o_encode(o, full))


@pytest.mark.parametrize("G,L,S,inverse", [(2, 11, 8, 0), (2, 15, 12, 1), (4, 14, 4, 0), (8, 16, 4, 1), (8, 19, 4, 0), (8, 20, 4, 0), (4, 20, 4, 1)])
def test_p2p_sharded_ntt_passes_match_oracle(G, L, S, inverse):
    """Standalone transform (plan_ntt_shard_p2p): pass A' scatters into the owners' Y, pass B' is local; output cyclic again."""
    _build_emulator()
    emu = ctypes.CDLL(EMU)
    f = emu.emu_ntt_shard_pass_p2p
    f.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int, ctypes.c_int]
    N = 1 << L
    o = ol.load_oracle()
    full = ol.fill_B(o, N, S)
    X = [np.ascontiguousarray(full[r::G]) for r in range(G)]
    Y = [np.full_like(X[0], 0xDEADBEEF) for _ in range(G)]
    yp, xp = _ptr_array(Y), _ptr_array(X)
    for r in range(G):
        assert f(X[r].ctypes.data, yp, N, G, r, S, S, inverse, 0) == 0
    for x in X:
        x[:] = 0xDEADBEEF
    for r in range(G):
        assert f(Y[r].ctypes.data, xp, N, G, r, S, S, inverse, 1) == 0
    out = np.empty_like(full)
    for r in range(G):
        out[r::G] = X[r]
    assert np.array_equal(out, ol.o_ntt(o, full, bool(inverse)))


def test_p2p_rejects_unsupported_shapes():
    _build_emulator()
    emu = ctypes.CDLL(EMU)
    f = emu.emu_rs_encode_shard_pass_p2p
    f.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int]
    x = np.zeros((1 << 10, 4), dtype=np.uint32)
    p = _ptr_array([x, x])
    assert f(x.ctypes.data, p, 1 << 11, 2, 0, 4, 4, 0) == -1               # 2^11 = 64 x 32: the 32-row tiles cannot split their outputs
    assert f(x.ctypes.data, p, 1 << 12, 16, 0, 4, 4, 0) == -1              # more than 8 peers
    g = emu.emu_rs_encode_shard_pass
    g.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int]
    for which in (0, 1, 2):                                                 # 2^19 = 512 x 1024 over 1024 ranks: no row set of pass 1 anywhere
        assert g(x.ctypes.data, 1 << 19, 1024, 0, 4, 4, which) == -1
