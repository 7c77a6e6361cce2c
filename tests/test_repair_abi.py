"""CPU: the repair entry points (csrc/repair.cu, api.cu) without a GPU fail with ENOINIT and compute nothing; their four
element-wise kernels are in the library and do not spill (cuobjdump, as test_sass_evidence.py does)."""
import ctypes

import numpy as np
import pytest

import sass_lib

KERNELS = ("repair_load_kernel", "repair_syndrome_kernel", "repair_split_kernel", "repair_scatter_kernel")


@pytest.fixture(scope="module")
def lib():
    from fastecc_b200 import build as b
    b.build()
    import fastecc_b200
    return fastecc_b200


def test_repair_without_a_gpu_is_enoinit(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    L = lib.lib()
    lost = np.array([0, 3], dtype=np.uint32)
    h = ctypes.c_void_p()
    assert L.fastecc_b200_rs_repair_pattern(12, 4, lost.ctypes.data, 2, None, 0, None, ctypes.byref(h)) == -4
    assert not h.value
    buf = np.zeros((12, 4), dtype=np.uint32)
    assert L.fastecc_b200_rs_repair(None, buf.ctypes.data, 4, buf.ctypes.data, 4, 4, None) == -4
    assert "fastecc_b200_init" in L.fastecc_b200_last_error().decode()
    L.fastecc_b200_rs_repair_free(None)                      # a null pattern is a no-op
    with pytest.raises(lib.FastEccError) as e:
        lib._check(L.fastecc_b200_rs_repair_pattern(12, 4, None, 0, lost.ctypes.data, 2, None, ctypes.byref(h)))
    assert e.value.code == -4


@pytest.fixture(scope="module")
def sass():
    return sass_lib.kernels()


@pytest.mark.parametrize("kernel", KERNELS)
def test_repair_kernel_is_in_the_library_and_does_not_spill(sass, kernel):
    hits = [k for k in sass if kernel in k]
    assert len(hits) == 1, hits
    body = sass[hits[0]]
    assert body and not any("LDL" in l or "STL" in l for l in body), kernel
    text = "\n".join(body)
    assert "LDG.E.128" in text and "STG.E.128" in text, kernel        # 16-byte accesses


def test_repair_kernels_use_barrett_triples_not_division(sass):
    """The products are gf::mul with a precomputed triple: IMAD.HI, and no call to a 64-bit remainder routine."""
    for kernel in KERNELS[1:]:
        body = "\n".join(sass[[k for k in sass if kernel in k][0]])
        assert "IMAD.HI" in body and "CALL" not in body, kernel
