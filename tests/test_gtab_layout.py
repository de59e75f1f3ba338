"""The combiner's global table layout (GtabLayout in csrc/mrhbm_kernels.h) on the CPU: the hash-to-bucket mapping, the
wrap at a bucket count that is not a power of two, the long-entry slots, and the byte count against what the
compaction reads, at every size a shuffle can grow to.  The driver tests/native/gtab_layout_check.cu is host-compiled
from the same header."""
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_gtab_layout(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path / "gtab_layout_check")
    subprocess.check_call([nvcc, "-O2", "-std=c++17", "-I", os.path.join(ROOT, "lua-mapreduce_b200", "csrc"),
                           "-o", exe, os.path.join(ROOT, "tests", "native", "gtab_layout_check.cu")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.splitlines()[-1] == "ok", out.stdout
