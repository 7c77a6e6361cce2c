"""CPU: the single-GPU plans split 2^19 as 1024 x 512 (csrc/plan.h split_l1): the strided passes A, D and A' run on 1024-row tiles
and the fused pass BC on 512-row tiles, both in the wide geometry (512 threads, 128 KiB tiles; pass_threads() in ntt_tile.cuh).
The sharded plans keep 512 x 1024, and so does the asymmetric encode to fewer parity blocks than 1024.  Checked on the built
library's SASS, on the plans and the geometry the launcher picks for each pass (tests/emulate_split.cu), and by emulating the
transforms of 2^19 and 2^20 thread by thread in that geometry against the oracle."""
import ctypes
import os
import subprocess

import pytest

import oracle_lib as ol
import sass_lib

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB = os.path.join(ROOT, "fastecc_b200", "libfastecc_b200.so")


@pytest.fixture(scope="module")
def sass():
    return sass_lib.kernels()


@pytest.mark.parametrize("lr,nxf", [(10, 1), (9, 2)])
def test_wide_passes_of_the_split(sass, lr, nxf):
    wide = "ntt_pass_kernelILi%dELi%dELi1ELi512E" % (lr, nxf)
    hits = [k for k in sass if wide in k]
    assert len(hits) == 1, hits
    body = sass[hits[0]]
    text = "\n".join(body)
    assert "UTMALDG" in text and "UBLKCP" in text                         # TMA tile + table loads
    assert not any("LDL" in l or "STL" in l for l in body)
    narrow = [k for k in sass if "ntt_pass_kernelILi%dELi%dELi1ELi256E" % (lr, nxf) in k]
    if lr == 10:
        assert not narrow                                                 # no narrow twin left
    else:                                                                 # the twin for passes with fewer wide tiles than SMs
        assert len(narrow) == 1 and not any("LDL" in l or "STL" in l for l in sass[narrow[0]])
    assert [k for k in sass if "ntt_pass_kernelILi%dELi%dELi2ELi256E" % (lr, nxf) in k]       # the sharded one stays narrow


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    ol.load_oracle()
    out = str(tmp_path_factory.mktemp("split") / "emulate_split")
    cmd = ["/usr/local/cuda/bin/nvcc", "-Wno-deprecated-gpu-targets", "-O2", "-o", out, os.path.join(HERE, "emulate_split.cu"),
           "-I" + os.path.join(ROOT, "fastecc_b200", "csrc"), "-I" + os.path.join(ROOT, "oracle"),
           os.path.join(ROOT, "oracle", "liboracle.so"), "-Xlinker", "-rpath=" + os.path.join(ROOT, "oracle")]
    subprocess.run(cmd, check=True, capture_output=True)
    return out


def _env():
    return {k: v for k, v in os.environ.items() if k != "FASTECC_B200_SPLIT"}


@pytest.fixture(scope="module")
def plans(exe):
    r = subprocess.run([exe, "plans"], capture_output=True, text=True, check=True, env=_env())
    out = {}
    for line in r.stdout.splitlines():
        head, passes = line.split(" : ")
        what, ln, g = head.split()
        out[(what, int(ln), int(g))] = passes.split()
    return out


def test_single_gpu_plans_split_19_as_1024_x_512(plans):
    assert plans[("encode", 19, 1)] == ["10/1/512", "9/2/512", "10/1/512"]
    assert plans[("ntt", 19, 1)] == plans[("ntt-inv", 19, 1)] == ["10/1/512", "9/1/256"]
    assert plans[("asym1", 19, 1)] == ["10/1/512", "9/2/512", "10/1/512"]
    assert plans[("asym9", 19, 1)] == ["10/1/512", "9/2/512", "10/1/512"]     # M = 1024 = N1
    assert plans[("asym10", 19, 1)] == ["9/1/256", "10/2/512", "9/1/256"]     # M = 512 < N1: the 512 x 1024 split keeps it native


def test_other_orders_keep_their_split(plans):
    assert plans[("ntt", 20, 1)] == plans[("ntt-inv", 20, 1)] == ["10/1/512", "10/1/512"]
    assert plans[("encode", 18, 1)] == ["9/1/256", "9/2/512", "9/1/256"]
    assert plans[("encode", 16, 1)] == ["8/1/256", "8/2/256", "8/1/256"]
    assert plans[("encode", 11, 1)] == ["6/1/256", "5/2/256", "6/1/256"]


@pytest.mark.parametrize("G", [2, 4, 8])
def test_sharded_plans_keep_512_x_1024(plans, G):
    assert plans[("encode-shard-p2p", 19, G)] == ["9/1/256", "10/2/256", "9/1/256"]
    assert plans[("ntt-shard-p2p", 19, G)] == ["9/1/256", "10/1/512"]      # B' is local: a single-GPU pass


@pytest.mark.parametrize("G", [2, 4, 8])
def test_shard_geometry_keeps_512_x_1024(G):
    if not os.path.exists(LIB):
        pytest.skip("needs the built library")
    if os.environ.get("FASTECC_B200_SPLIT"):
        pytest.skip("FASTECC_B200_SPLIT overrides the split")
    lib = ctypes.CDLL(LIB)
    f = lib.fastecc_b200_shard_geometry
    f.argtypes = [ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    f.restype = ctypes.c_int
    n1, n2, ok = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_int()
    assert f(1 << 19, G, ctypes.byref(n1), ctypes.byref(n2), ctypes.byref(ok)) == 0
    assert (n1.value, n2.value) == (512, 1024)


def test_shard_geometry_rejects_1024_ranks_at_2_to_the_19():
    """Pass 1 of the sharded encode works on N1 / G row sets, passes 0 and 2 on N2 / G: 2^19 = 512 x 1024 cannot be dealt to 1024
    ranks although N2 is a multiple of 1024 (every rank would get no row set of pass 1)."""
    if not os.path.exists(LIB):
        pytest.skip("needs the built library")
    lib = ctypes.CDLL(LIB)
    f = lib.fastecc_b200_shard_geometry
    f.argtypes = [ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    f.restype = ctypes.c_int
    ok = ctypes.c_int(-1)
    assert f(1 << 19, 1024, None, None, ctypes.byref(ok)) == -1
    assert ok.value == 0
    assert f(1 << 19, 512, None, None, None) == 0


def test_ntt_19_20_as_launched_matches_oracle(exe):
    r = subprocess.run([exe], capture_output=True, text=True, cwd=HERE, env=_env())
    assert r.returncode == 0, r.stdout[-3000:]
    assert "EMULATION OK" in r.stdout
    assert r.stdout.count(": ok") == 12
    assert "ntt-fwd  N=2^19 S=1   passes=10/512 9/256 " in r.stdout
    assert "ntt-inv  N=2^20 S=33  passes=10/512 10/512 " in r.stdout
