"""CPU: the batch update (fastecc_b200_rs_update_batch, csrc/batch.cu, api.cu) without a GPU fails with ENOINIT and writes
nothing; its kernel is in the library in all six widths, does not spill, calls no routine (no 64-bit division), copies every
stripe row to shared memory 16 bytes at a time (cp.async), stores 16 bytes and multiplies by Barrett triples.  It writes into
the stripes, so no stripe row may be read through the non-coherent path: the only .CONSTANT load left is the T table's."""
import numpy as np
import pytest

import sass_lib

KERNEL = "batch_update_kernel"


@pytest.fixture(scope="module")
def lib():
    from fastecc_b200 import build as b
    b.build()
    import fastecc_b200
    return fastecc_b200


def test_update_batch_without_a_gpu_is_enoinit(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    L = lib.lib()
    B, N, M, S = 3, 12, 4, 8
    data = np.arange(B * N * S, dtype=np.uint32).reshape(B, N, S)
    parity = np.arange(B * M * S, dtype=np.uint32).reshape(B, M, S)
    new = np.full((B, 2, S), 5, dtype=np.uint32)
    changed = np.array([1, 5], dtype=np.uint32)
    before = (data.copy(), parity.copy(), new.copy())
    rc = L.fastecc_b200_rs_update_batch(data.ctypes.data, S, N * S, N, parity.ctypes.data, S, M * S, M, changed.ctypes.data, 2, new.ctypes.data, S,
                                        2 * S, B, S, None)
    assert rc == -4
    assert "fastecc_b200_init" in L.fastecc_b200_last_error().decode()
    assert all(np.array_equal(x, y) for x, y in zip((data, parity, new), before))
    with pytest.raises(lib.FastEccError) as e:
        lib._check(L.fastecc_b200_rs_update_batch(None, S, N * S, N, None, S, M * S, M, None, 0, None, S, S, 0, S, None))
    assert e.value.code == -4


@pytest.fixture(scope="module")
def sass():
    return sass_lib.kernels()


def test_update_batch_kernel_is_in_the_library_and_does_not_spill(sass):
    hits = [k for k in sass if KERNEL in k]
    assert len(hits) == 6, hits                                      # 1, 2, 3, 4, 6 and 8 outputs per warp
    for k in hits:
        t = "\n".join(sass[k])
        assert t and "LDL" not in t and "STL" not in t, k
        assert "CALL" not in t, k                                    # no 64-bit division or remainder routine


def test_update_batch_kernel_copies_and_stores_16_bytes_and_uses_barrett_products(sass):
    for k in [k for k in sass if KERNEL in k]:
        t = "\n".join(sass[k])
        assert "LDGSTS.E.BYPASS.128" in t, k
        assert "STG.E.128" in t, k
        assert "IMAD.HI" in t, k


def test_update_batch_kernel_reads_no_stripe_row_through_the_non_coherent_path(sass):
    """Every stripe row goes through cp.async; the one .CONSTANT load is the staging of the T table"""
    for k in [k for k in sass if KERNEL in k]:
        loads = [l for l in sass[k] if "LDG" in l and "LDGSTS" not in l and "LDGDEPBAR" not in l]
        assert len(loads) == 1 and ".CONSTANT" in loads[0] and ".128" in loads[0], (k, loads)
