"""CPU: the degraded scrub entry point (fastecc_b200_rs_scrub_degraded, csrc/scrub.cu, api.cu) without a GPU fails with ENOINIT and
writes none of its outputs; its kernels are in the library and do not spill, and its fold (the pass over the surviving rows) uses
16-byte loads and Barrett products with no call to a division routine (cuobjdump, as test_scrub_abi.py does)."""
import ctypes

import numpy as np
import pytest

import sass_lib

FOLD = "degraded_fold_kernel"
KERNELS = (FOLD, "degraded_syndrome_kernel", "degraded_roots_kernel")


@pytest.fixture(scope="module")
def lib():
    from fastecc_b200 import build as b
    b.build()
    import fastecc_b200
    return fastecc_b200


@pytest.mark.parametrize("max_bad", [0, 1])
def test_degraded_scrub_without_a_gpu_is_enoinit(lib, max_bad):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    L = lib.lib()
    N, M, S = 12, 4, 4
    data = np.arange(N * S, dtype=np.uint32).reshape(N, S)
    parity = data[:M] + 7
    before = (data.copy(), parity.copy())
    status, nd, np_ = ctypes.c_int(-7), ctypes.c_size_t(77), ctypes.c_size_t(78)
    bd, bp = np.full(4, 9, dtype=np.uint32), np.full(4, 9, dtype=np.uint32)
    rc = L.fastecc_b200_rs_scrub_degraded(None, data.ctypes.data, S, parity.ctypes.data, S, S, max_bad, 5, None, ctypes.byref(status),
                                          bd.ctypes.data, ctypes.byref(nd), bp.ctypes.data, ctypes.byref(np_))
    assert rc == -4
    assert "fastecc_b200_init" in L.fastecc_b200_last_error().decode()
    assert (status.value, nd.value, np_.value) == (-7, 77, 78)
    assert (bd == 9).all() and (bp == 9).all()
    assert np.array_equal(data, before[0]) and np.array_equal(parity, before[1])


def test_python_degraded_scrub_without_a_gpu_raises(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises((ValueError, RuntimeError, AssertionError)):
        lib.rs_scrub_degraded_dev(torch.zeros((4, 4), dtype=torch.int32), torch.zeros((2, 4), dtype=torch.int32), [1], [])


@pytest.fixture(scope="module")
def sass():
    return sass_lib.kernels()


def body(sass, kernel):
    hits = [k for k in sass if kernel in k]
    assert len(hits) == 1, hits
    return sass[hits[0]]


@pytest.mark.parametrize("kernel", KERNELS)
def test_degraded_kernel_is_in_the_library_and_does_not_spill(sass, kernel):
    lines = body(sass, kernel)
    assert lines and not any("LDL" in l or "STL" in l for l in lines), kernel


def test_degraded_fold_uses_16_byte_loads_barrett_products_and_no_call(sass):
    text = "\n".join(body(sass, FOLD))
    assert "LDG.E.128" in text
    assert "IMAD.HI" in text
    assert "CALL" not in text
