"""CPU-only: the C-ABI library builds for sm_90a, loads, and exports every symbol include/fastecc_b200.h declares;
argument validation and the "no GPU -> loud failure, never a CPU fallback" behaviour."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from fastecc_b200 import build as b
    b.build()
    import fastecc_b200
    return fastecc_b200


def test_exports_match_header(lib):
    hdr = open(os.path.join(ROOT, "include", "fastecc_b200.h")).read()
    names = sorted(set(re.findall(r"\b(fastecc_b200_[a-z0-9_]+)\s*\(", hdr)))
    assert len(names) >= 12
    L = ctypes.CDLL(lib.LIB_PATH)
    for n in names:
        assert hasattr(L, n), n


def test_library_is_sm90a_only(lib):
    import subprocess
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-lelf", lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out and not re.search(r"sm_(?!90a)\d+", out)


def test_no_gpu_means_error_not_fallback(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(lib.FastEccError):
        lib.init(0)
    a = np.zeros((16, 4), dtype=np.uint32)
    with pytest.raises(lib.FastEccError) as e:
        lib.MFA_NTT(a, 16, 4, False)
    assert e.value.code == -4          # ENOINIT: nothing was computed on the CPU
    with pytest.raises(lib.FastEccError):
        lib.EncodeReedSolomon_body(a, 16, 4)


def test_product_never_references_oracle():
    """The product path must not include, link or import anything under oracle/ (tier rule 3)."""
    bad = []
    for d, _, files in os.walk(os.path.join(ROOT, "fastecc_b200")):
        for f in files:
            if f.endswith((".cu", ".cuh", ".h", ".cpp", ".py")):
                txt = open(os.path.join(d, f), errors="ignore").read()
                if re.search(r"oracle[/_]|liboracle|gfp_oracle|_ref/", txt):
                    bad.append(f)
    assert not bad, bad


def test_host_scalars_match_reference_constants(lib):
    assert lib.GF_Root(2) == lib.P - 1                     # main.cpp:314
    assert lib.GF_Root(1 << 20) == 3156611342 and lib.GF_Inv(1 << 19) == 4293910531
    assert lib.GF_Mul(123456789, 987654321) == 3168667484
    assert lib.GF_Add(lib.P - 1, 1) == 0 and lib.GF_Sub(0, 1) == lib.P - 1
