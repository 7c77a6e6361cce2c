"""CPU: the built library really contains what DESIGN.md says the kernels are made of.  cuobjdump -sass of
fastecc_b200/libfastecc_b200.so (sm_90a cubins only): the headline pass kernels take their quotient from the FP64 unit
(I2F.F64.U32 + DFMA.RM + VIADDMNMX.U32, one each per product, and no IMAD.HI in the butterflies), load their tiles and tables
with TMA (UTMALDG / UBLKCP + SYNCS mbarrier instructions) and do not spill."""
import re

import pytest

import sass_lib


@pytest.fixture(scope="module")
def sass():
    elf = sass_lib.dump("-lelf")
    assert "sm_90a" in elf and not re.search(r"sm_(?!90a)\d+", elf), elf
    return sass_lib.kernels()


def _kernel(sass, pattern):
    hits = [k for k in sass if pattern in k]
    assert len(hits) == 1, hits
    return sass[hits[0]]


@pytest.mark.parametrize("pattern", ["ntt_pass_kernelILi10ELi2ELi1E", "ntt_pass_kernelILi9ELi1ELi1E", "ntt_pass_kernelILi10ELi2ELi2E", "ntt_pass_kernelILi9ELi1ELi2E"])
def test_headline_kernels_use_the_fp64_quotient_and_tma(sass, pattern):
    body = _kernel(sass, pattern)
    text = "\n".join(body)
    n_cvt, n_fma, n_fix = text.count("I2F.F64.U32"), text.count("DFMA.RM"), text.count("VIADDMNMX.U32")
    assert n_cvt >= 300 and n_cvt == n_fma and n_fix >= n_cvt                  # one conversion, one DFMA, one add-min per product
    assert text.count("IMAD.HI") <= 16                                            # address arithmetic only: none in the butterflies
    assert "UTMALDG" in text and "UBLKCP" in text and "SYNCS" in text            # TMA tensor + bulk loads, mbarrier
    assert sum(1 for l in body if "LDL" in l or "STL" in l) <= 4                  # no spilling to speak of


def test_radix_encode_kernel_is_in_the_library_and_does_not_spill(sass):
    hits = {k: v for k, v in sass.items() if "radix_encode_kernel" in k}
    assert sorted(re.search(r"ILi(\d)E", k).group(1) for k in hits) == ["3", "9"], list(hits)
    for k, body in hits.items():
        assert body and not any("LDL" in l or "STL" in l for l in body), k


def test_radix_fold_kernel_is_in_the_library_and_does_not_spill(sass):
    hits = {k: v for k, v in sass.items() if "radix_fold_kernel" in k}
    assert sorted(re.search(r"ILi(\d)ELi(\d)E", k).groups() for k in hits) == [("3", "1"), ("3", "3"), ("9", "1"), ("9", "3"), ("9", "9")], list(hits)
    for k, body in hits.items():
        assert body and not any("LDL" in l or "STL" in l for l in body), k


def test_library_contains_every_kernel_family(sass):
    names = " ".join(sass)
    for k in ("ntt_pass_kernel", "build_tables_kernel", "small_dft_kernel", "radix_pass_kernel", "row_scale_kernel", "shard_barrier_kernel",
              "leaves_kernel", "pairmul_kernel", "gather_scale_kernel"):
        assert k in names, k
