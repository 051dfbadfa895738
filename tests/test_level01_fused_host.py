"""The fused level-0/1 kernel of octave 0 (march_level01x2_kernel) on the host, no GPU needed: it ships in the library's
SASS with the byte-tile cp.async staging and the 64-bit plane stores of the level kernels, and ptxas gives it no spills
and few enough registers for the 4 resident CTAs per SM its launch partition (make_partition's default slots) assumes."""
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "popsift_b200", "csrc")
LIB = os.path.join(ROOT, "popsift_b200", "lib", "libpopsift_b200.so")
NF, CTAS_PER_SM, REGS_PER_SM = 160, 4, 65536     # the fused kernel's block size and residency


def test_fused_kernel_in_shipped_sass():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sass_hist
    k = sass_hist.histogram(LIB)
    fused = {n: c for n, c in k.items() if "march_level01x2_kernel" in n}
    assert len(fused) == 1, list(fused)
    c = next(iter(fused.values()))
    assert c["LDGSTS"] > 0                   # byte tiles staged with cp.async
    assert c["STG"] > 0 and c["LDS"] > 0 and c["STS"] > 0


def test_fused_kernel_no_spills_and_residency():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = os.path.join(os.environ.get("TMPDIR", "/tmp"), "k_pyramid_march_ptxas_%d.o" % os.getpid())
    r = subprocess.run([nvcc, "-std=c++17", "-O3", "--fmad=false", "-I" + os.path.join(ROOT, "include"), "-I" + CSRC,
                        "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c",
                        os.path.join(CSRC, "k_pyramid_march.cu"), "-o", out], capture_output=True, text=True, timeout=900)
    if os.path.exists(out):
        os.remove(out)
    assert r.returncode == 0, r.stderr[-2000:]
    m = re.search(r"Function properties for \S*march_level01x2_kernel\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\nptxas info\s*: Used (\d+) registers", r.stderr)
    assert m, "no ptxas report for march_level01x2_kernel"
    stack, spill_st, spill_ld, regs = map(int, m.groups())
    assert spill_st == 0 and spill_ld == 0 and stack == 0
    assert CTAS_PER_SM * NF * regs <= REGS_PER_SM, regs
