"""CPU: the degraded-read entry point (fastecc_b200_rs_reconstruct, csrc/reconstruct.cu, api.cu) without a GPU fails with ENOINIT
and writes nothing; its kernels are in the library, do not spill, read the data with 16-byte loads and multiply by Barrett triples
(cuobjdump, as test_update_abi.py does)."""
import numpy as np
import pytest

import sass_lib

KERNELS = ("reconstruct_sum_kernel", "reconstruct_combine_kernel")


@pytest.fixture(scope="module")
def lib():
    from fastecc_b200 import build as b
    b.build()
    import fastecc_b200
    return fastecc_b200


def test_reconstruct_without_a_gpu_is_enoinit(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    L = lib.lib()
    N, M, S = 12, 4, 4
    data = np.arange(N * S, dtype=np.uint32).reshape(N, S)
    parity = data[:M] + 7
    out = np.full((2, S), 3, dtype=np.uint32)
    before = (data.copy(), parity.copy(), out.copy())
    lost_d, lost_p = np.array([1, 5], dtype=np.uint32), np.array([0], dtype=np.uint32)
    rc = L.fastecc_b200_rs_reconstruct(data.ctypes.data, S, N, parity.ctypes.data, S, M, lost_d.ctypes.data, 2, lost_p.ctypes.data, 1,
                                       lost_d.ctypes.data, 1, lost_p.ctypes.data, 1, out.ctypes.data, S, S, None)
    assert rc == -4
    assert "fastecc_b200_init" in L.fastecc_b200_last_error().decode()
    assert all(np.array_equal(a, b) for a, b in zip((data, parity, out), before))
    with pytest.raises(lib.FastEccError) as e:
        lib._check(L.fastecc_b200_rs_reconstruct(None, S, N, None, S, M, None, 0, None, 0, None, 0, None, 0, None, S, S, None))
    assert e.value.code == -4


@pytest.fixture(scope="module")
def sass():
    return sass_lib.kernels()


def bodies(sass, kernel):
    hits = [k for k in sass if kernel in k]
    return hits, ["\n".join(sass[k]) for k in hits]


@pytest.mark.parametrize("kernel", KERNELS)
def test_reconstruct_kernels_are_in_the_library_and_do_not_spill(sass, kernel):
    hits, texts = bodies(sass, kernel)
    assert len(hits) == (4 if kernel == "reconstruct_sum_kernel" else 1), hits     # the sum kernel: 1, 2, 4 and 8 outputs per warp
    for t in texts:
        assert t and "LDL" not in t and "STL" not in t, kernel
        assert "CALL" not in t, kernel                                          # no 64-bit remainder routine


def test_reconstruct_sum_kernel_loads_16_bytes_and_uses_barrett_products(sass):
    _, texts = bodies(sass, "reconstruct_sum_kernel")
    for t in texts:
        assert "LDG.E.128" in t
        assert "IMAD.HI" in t
    _, (combine,) = bodies(sass, "reconstruct_combine_kernel")
    assert "IMAD.HI" in combine and "STG.E.128" in combine
