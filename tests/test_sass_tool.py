"""tools/sass_by_line.py — the static-SASS instrument DESIGN.md §11a relies on — runs on the built library without a GPU."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(not (shutil.which("cuobjdump") and shutil.which("nvdisasm")), reason="CUDA binary utilities not installed")
def test_sass_by_line_lists_the_dp_loop_with_source_lines():
    from racon_b200 import build
    lib = build.build_cuda()
    tool = os.path.join(ROOT, "tools", "sass_by_line.py")
    out = subprocess.run([sys.executable, tool, "--lib", lib, "--grep", r"VIADDMNMX\.S16x2"], stdout=subprocess.PIPE,
                         text=True, check=True).stdout.splitlines()
    assert out[0].startswith("kernel rp_poa_kernelILi32ELi16ELi3E:")
    # the DPX row arithmetic of both copies of the row loop (with and without the chunk carry): 39 each, + the banded rows
    assert len(out) - 1 >= 2 * 39
    assert all(".hpp:" in l or ".cuh:" in l or ".cu:" in l for l in out[1:])
