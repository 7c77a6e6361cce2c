"""CPU: the batch encode (fastecc_b200_rs_encode_batch, csrc/batch.cu, api.cu) without a GPU fails with ENOINIT and writes
nothing; its kernel is in the library, does not spill, calls no routine (no 64-bit division), reads the data with 16-byte loads
and multiplies by Barrett triples (cuobjdump, as test_reconstruct_abi.py does)."""
import numpy as np
import pytest

import sass_lib

KERNEL = "batch_encode_kernel"


@pytest.fixture(scope="module")
def lib():
    from fastecc_b200 import build as b
    b.build()
    import fastecc_b200
    return fastecc_b200


def test_encode_batch_without_a_gpu_is_enoinit(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    L = lib.lib()
    B, N, M, S = 3, 12, 4, 8
    data = np.arange(B * N * S, dtype=np.uint32).reshape(B, N, S)
    parity = np.full((B, M, S), 5, dtype=np.uint32)
    before = (data.copy(), parity.copy())
    rc = L.fastecc_b200_rs_encode_batch(data.ctypes.data, S, N * S, N, parity.ctypes.data, S, M * S, M, B, S, None)
    assert rc == -4
    assert "fastecc_b200_init" in L.fastecc_b200_last_error().decode()
    assert np.array_equal(data, before[0]) and np.array_equal(parity, before[1])
    with pytest.raises(lib.FastEccError) as e:
        lib._check(L.fastecc_b200_rs_encode_batch(None, S, N * S, N, None, S, M * S, M, 0, S, None))
    assert e.value.code == -4


@pytest.fixture(scope="module")
def sass():
    return sass_lib.kernels()


def test_batch_kernel_is_in_the_library_and_does_not_spill(sass):
    hits = [k for k in sass if KERNEL in k]
    assert len(hits) == 6, hits                                      # 1, 2, 3, 4, 6 and 8 outputs per warp
    for k in hits:
        t = "\n".join(sass[k])
        assert t and "LDL" not in t and "STL" not in t, k
        assert "CALL" not in t, k                                    # no 64-bit division or remainder routine


def test_batch_kernel_loads_16_bytes_and_uses_barrett_products(sass):
    for k in [k for k in sass if KERNEL in k]:
        t = "\n".join(sass[k])
        assert "LDG.E.128" in t, k
        assert "IMAD.HI" in t, k
        assert "STG.E.128" in t, k
