"""cuobjdump of the built library for the CPU tests that check its machine code (test infrastructure only)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "fastecc_b200", "libfastecc_b200.so")


def dump(*args) -> str:
    """The output of `cuobjdump <args> LIB`; skips the test when cuobjdump or the built library is missing."""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(LIB):
        pytest.skip("needs cuobjdump and the built library")
    return subprocess.run([exe, *args, LIB], capture_output=True, text=True, check=True).stdout


def kernels() -> dict:
    """{mangled kernel name: [its SASS instruction lines]} of the library."""
    out, name = {}, None
    for line in dump("-sass").splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1); out[name] = []
        elif name and re.match(r"\s+/\*[0-9a-f]{4,5}\*/", line):
            out[name].append(line)
    return out
