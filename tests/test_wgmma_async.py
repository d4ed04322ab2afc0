"""CPU guard: the tensor-core kernels keep their wgmma pipelines asynchronous.

ptxas silently serialises every wgmma.mma_async of a kernel (a wait after each MMA) when it cannot prove the
pipeline safe: a function call anywhere in the kernel (a device-side printf is one), or a non-wgmma instruction
defining accumulator registers inside a pipeline stage.  It says so only as an informational C75xx diagnostic under
-Xptxas -v, and the kernel still computes the same numbers, so nothing else would notice.  This compiles the three
tensor-core sources for sm_90a with the Makefile's flags plus -Xptxas -v and fails on any such diagnostic and on
register spills.
"""
import os
import re
import shlex
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "wild_visual_navigation_b200", "csrc")
SOURCES = ("gemm_wgmma.cu", "attention_wgmma.cu", "pixel_head.cu")

# Kernels that spill a few dozen bytes under their register caps, in epilogue code: the patch-embed GEMM at BN >= 192
# (168 registers for 384 threads) and the pixel head (128 registers, two CTAs per SM).  They are held to a bound
# instead of zero; every other kernel in these sources must not spill at all.
SPILL_ALLOWANCE = {r"gemm_bf16_kernelILi\d+ELi3ELi\d+E": 128, r"pixel_head_kernel": 64}


def _nvcc():
    found = shutil.which("nvcc")
    if found:
        return found
    for home in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if home and os.path.isfile(os.path.join(home, "bin", "nvcc")):
            return os.path.join(home, "bin", "nvcc")
    return None


def _makefile_flags():
    text = open(os.path.join(CSRC, "Makefile")).read()
    arch = re.search(r"^ARCH\s*:=\s*(.+)$", text, re.M).group(1)
    flags = re.search(r"^NVCCFLAGS\s*:=\s*(.+)$", text, re.M).group(1).replace("$(ARCH)", arch)
    return shlex.split(flags)


def _ptxas_reports(nvcc):
    flags = _makefile_flags() + ["-Xptxas", "-v"]
    with tempfile.TemporaryDirectory() as tmp:
        procs = {
            src: subprocess.Popen([nvcc] + flags + ["-c", os.path.join(CSRC, src), "-o", os.path.join(tmp, src + ".o")],
                                  cwd=CSRC, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
            for src in SOURCES
        }
        out = {src: p.communicate()[0] for src, p in procs.items()}
        for src, p in procs.items():
            assert p.returncode == 0, f"nvcc failed on {src}:\n{out[src][-4000:]}"
    return out


@pytest.fixture(scope="module")
def reports():
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    return _ptxas_reports(nvcc)


@pytest.mark.parametrize("src", SOURCES)
def test_no_serialised_wgmma(reports, src):
    bad = [l.strip() for l in reports[src].splitlines() if re.search(r"\(C75\d\d\)|wgmma\.mma_async instructions are serialized", l)]
    assert not bad, f"{src}: ptxas serialised wgmma ({len(bad)} diagnostics):\n" + "\n".join(bad[:10])


@pytest.mark.parametrize("src", SOURCES)
def test_no_register_spills(reports, src):
    kernel, seen, over = None, 0, []
    for line in reports[src].splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            kernel = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and kernel is not None:
            seen += 1
            spilled = max(int(m.group(1)), int(m.group(2)))
            allowed = next((b for pat, b in SPILL_ALLOWANCE.items() if re.search(pat, kernel)), 0)
            if spilled > allowed:
                over.append(f"{kernel}: {line.strip()} (allowed {allowed} bytes)")
            kernel = None
    assert seen > 0, f"{src}: no ptxas resource report found"
    assert not over, f"{src}: register spills:\n" + "\n".join(over)
