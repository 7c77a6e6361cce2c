"""The reference's own drivers, UNMODIFIED, built against the H100 library through fastecc_b200/shim/ntt.cpp.

CPU part: the shim compiles and links (only where the reference tree exists).  GPU part: `ntt-b200 n L 4096` -- the
reference's integration test of MFA_NTT (main.cpp:239-300: forward, inverse, x N^-1, hashes) -- must print
"Verified!" with the golden hashes of SURVEY.md 8c, and `rs-b200` must run."""
import json
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DROPIN = os.path.join(ROOT, "oracle", "_ref", "dropin")
G = json.load(open(os.path.join(ROOT, "tests", "golden", "survey_8c.json")))


def test_shim_builds_against_unmodified_reference_sources():
    if not os.path.exists("/root/reference/ntt.cpp"):
        pytest.skip("no reference tree on this machine")
    r = subprocess.run([os.path.join(ROOT, "integration", "build_dropin.sh")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    for exe in ("rs-b200", "ntt-b200"):
        assert os.path.exists(os.path.join(DROPIN, exe))
    stage = os.path.join(DROPIN, "stage")
    for f in os.listdir(stage):                       # nothing copied: the staging directory holds symlinks only
        assert os.path.islink(os.path.join(stage, f)), f


@pytest.mark.gpu
@pytest.mark.parametrize("L", [7, 10, 12, 16, 19])
def test_reference_ntt_driver_verifies_on_gpu(L):
    exe = os.path.join(DROPIN, "ntt-b200")
    if not os.path.exists(exe):
        pytest.skip("drop-in binaries were not built (needs the reference tree at build time)")
    r = subprocess.run([exe, "n", str(L), "4096"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-1000:]
    m = re.search(r"Verified!\s+Original (\d+),\s+after NTT: (\d+)", r.stdout)
    assert m, r.stdout[-1000:]
    h0, h1 = G["ntt_fillA_4096B"][str(L)]
    assert (int(m.group(1)), int(m.group(2))) == (h0, h1)


@pytest.mark.gpu
def test_reference_rs_driver_runs_on_gpu():
    exe = os.path.join(DROPIN, "rs-b200")
    if not os.path.exists(exe):
        pytest.skip("drop-in binaries were not built (needs the reference tree at build time)")
    r = subprocess.run([exe, "16", "4096"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-1000:]
    assert re.search(r"Reed-Solomon encoding.*MiB/s", r.stdout), r.stdout[-1000:]
