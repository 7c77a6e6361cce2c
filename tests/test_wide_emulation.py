"""CPU-only: the encode plans with the pass kernels in the wide tile geometry (512 threads, 128 KiB tiles; the launcher runs
the fused 1024-row pass that way), thread by thread on the host (tests/emulate_wide.cu) against the oracle, at widths that
leave partial strips."""
import os
import subprocess

import pytest

import oracle_lib as ol

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    ol.load_oracle()
    out = str(tmp_path_factory.mktemp("wide") / "emulate_wide")
    cmd = ["/usr/local/cuda/bin/nvcc", "-Wno-deprecated-gpu-targets", "-O2", "-o", out, os.path.join(HERE, "emulate_wide.cu"),
           "-I" + os.path.join(ROOT, "fastecc_b200", "csrc"), "-I" + os.path.join(ROOT, "oracle"),
           os.path.join(ROOT, "oracle", "liboracle.so"), "-Xlinker", "-rpath=" + os.path.join(ROOT, "oracle")]
    subprocess.run(cmd, check=True, capture_output=True)
    return out


@pytest.mark.parametrize("mode", [[], ["all"]], ids=["as_launched", "every_pass_wide"])
def test_wide_geometry_emulation_matches_oracle(exe, mode):
    r = subprocess.run([exe] + mode, capture_output=True, text=True, cwd=HERE)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "EMULATION OK" in r.stdout
