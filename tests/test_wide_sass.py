"""CPU: the wide pass-kernel instantiations (512 threads, 128 KiB tiles; pass_threads() in ntt_tile.cuh) are in the built library,
replace their narrow twins, load by TMA and do not spill.  cuobjdump -sass of fastecc_b200/libfastecc_b200.so."""
import re

import pytest

import sass_lib

WIDE = ["ntt_pass_kernelILi10ELi2ELi1ELi512E"]                       # <LR, NXF, TMA, threads>


@pytest.fixture(scope="module")
def sass():
    return sass_lib.kernels()


@pytest.mark.parametrize("pattern", WIDE)
def test_wide_kernel_exists_and_does_not_spill(sass, pattern):
    hits = [k for k in sass if pattern in k]
    assert len(hits) == 1, hits
    body = sass[hits[0]]
    text = "\n".join(body)
    assert not any("LDL" in l or "STL" in l for l in body)
    assert "UTMALDG" in text and "UBLKCP" in text                         # TMA tile + table loads
    narrow = pattern[:-len("ELi512E")]                                     # the same <LR, NXF, TMA> exists in one geometry only
    assert [k for k in sass if narrow + "ELi" in k] == hits


def test_every_pass_kernel_carries_its_geometry(sass):
    names = [k for k in sass if "ntt_pass_kernel" in k]
    assert names and all(re.search(r"ntt_pass_kernelILi\d+ELi\dELi\dELi(256|512)E", k) for k in names), names
