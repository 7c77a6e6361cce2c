"""CPU: the update entry point (fastecc_b200_rs_update, csrc/update.cu, api.cu) without a GPU fails with ENOINIT on both of its
paths and computes nothing; its kernels are in the library, do not spill, use 16-byte accesses and Barrett triples (cuobjdump,
as test_repair_abi.py does)."""
import ctypes

import numpy as np
import pytest

import sass_lib

KERNELS = ("update_delta_kernel", "update_parity_kernel")


@pytest.fixture(scope="module")
def lib():
    from fastecc_b200 import build as b
    b.build()
    import fastecc_b200
    return fastecc_b200


@pytest.mark.parametrize("k", [1, 12])                          # few changed blocks (direct) and all of them (re-encode)
def test_update_without_a_gpu_is_enoinit(lib, k):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    L = lib.lib()
    N, M, S = 12, 12, 4
    data = np.arange(N * S, dtype=np.uint32).reshape(N, S)
    parity = data + 7
    new = np.full((k, S), 3, dtype=np.uint32)
    before = (data.copy(), parity.copy(), new.copy())
    changed = np.arange(k, dtype=np.uint32)
    rc = L.fastecc_b200_rs_update(data.ctypes.data, S, N, parity.ctypes.data, S, M, changed.ctypes.data, k, new.ctypes.data, S, S, None)
    assert rc == -4
    assert "fastecc_b200_init" in L.fastecc_b200_last_error().decode()
    assert all(np.array_equal(a, b) for a, b in zip((data, parity, new), before))
    with pytest.raises(lib.FastEccError) as e:
        lib._check(L.fastecc_b200_rs_update(data.ctypes.data, S, N, parity.ctypes.data, S, M, None, 0, None, S, S, None))
    assert e.value.code == -4


@pytest.fixture(scope="module")
def sass():
    return sass_lib.kernels()


@pytest.mark.parametrize("kernel", KERNELS + ("update_table_kernel",))
def test_update_kernel_is_in_the_library_and_does_not_spill(sass, kernel):
    hits = [k for k in sass if kernel in k]
    assert len(hits) == 1, hits
    body = sass[hits[0]]
    assert body and not any("LDL" in l or "STL" in l for l in body), kernel


@pytest.mark.parametrize("kernel", KERNELS)
def test_update_kernels_use_16_byte_accesses(sass, kernel):
    text = "\n".join(sass[[k for k in sass if kernel in k][0]])
    assert "LDG.E.128" in text and "STG.E.128" in text, kernel


def test_update_parity_kernel_uses_barrett_triples_not_division(sass):
    """The products are gf::mul with the table's triple: IMAD.HI, and no call to a 64-bit remainder routine."""
    for kernel in KERNELS:
        body = "\n".join(sass[[k for k in sass if kernel in k][0]])
        assert "CALL" not in body, kernel
    body = "\n".join(sass[[k for k in sass if "update_parity_kernel" in k][0]])
    assert "IMAD.HI" in body
