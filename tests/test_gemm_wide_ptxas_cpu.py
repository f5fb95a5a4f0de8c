"""What ptxas makes of the 128 x 256 f16f8 GEMM (gemm_wide_kernel; CPU only: nvcc cross-compiles for sm_90a without a GPU).

The kernel holds a 64 x 256 fp32 accumulator and a 64 x 256 fp16 one per consumer warpgroup (192 of its 232 registers), so a
spill or a serialised wgmma pipeline would be easy to introduce and would cost more than the wide tile saves.  This compiles
gemm_wide_f16f8.cu exactly as vima_b200/build.py does, plus -Xptxas -v, and checks for every instantiation

  * no "wgmma serialized" warning (C7510 / C7520),
  * no spill bytes,
  * the SASS has the 64x256x16 fp16 wgmma into fp32 and the 64x256x32 e4m3 wgmma into fp16.
"""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from vima_b200 import build as vbuild

SRC = "gemm_wide_f16f8.cu"
N_EPILOGUES = 13  # the rows of VIMA_GEMM_VARIANTS; no generic runtime-flag instantiation


def _tool(name):
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    path = os.path.join(os.path.dirname(nvcc), name)
    return path if os.path.isfile(path) else None


@pytest.fixture(scope="module")
def compiled():
    nvcc = _tool("nvcc")
    if nvcc is None:
        pytest.skip("nvcc not found")
    assert SRC in vbuild.SOURCES
    tmp = tempfile.mkdtemp(prefix="vima_ptxas_wide_")
    try:
        obj = os.path.join(tmp, "wide.o")
        r = subprocess.run([nvcc, *vbuild.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(vbuild.CSRC, SRC), "-o", obj],
                           capture_output=True, text=True)
        assert r.returncode == 0, f"nvcc failed for {SRC}:\n{r.stderr[-4000:]}"
        cuobjdump = _tool("cuobjdump")
        sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout if cuobjdump else None
        yield r.stderr, sass
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def _functions(log):
    """-> {mangled kernel name: (spill store bytes, spill load bytes)} from a ptxas -v log."""
    out = {}
    for m in re.finditer(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log):
        out[m.group(1)] = (int(m.group(2)), int(m.group(3)))
    return out


def test_wide_gemm_ptxas(compiled):
    log, _ = compiled
    bad = [ln.strip() for ln in log.splitlines() if re.search(r"C75[12]0|wgmma\.mma_async instructions are serialized", ln)]
    assert not bad, "\n".join(bad)
    fns = _functions(log)
    wide = {k: v for k, v in fns.items() if "gemm_wide_kernel" in k}
    assert len(wide) == N_EPILOGUES and len(fns) == N_EPILOGUES, sorted(fns)
    assert not any("EpiCfgILb1E" in k for k in wide), "a generic runtime-flag instantiation"
    spilled = {k: v for k, v in wide.items() if v != (0, 0)}
    assert not spilled, spilled


def test_wide_gemm_sass(compiled):
    _, sass = compiled
    if sass is None:
        pytest.skip("cuobjdump not found")
    assert len(re.findall(r"HGMMA\.64x256x16\.F32(?!\.BF16)", sass)) == 4 * N_EPILOGUES  # 4 per k block of 64
    assert len(re.findall(r"QGMMA\.64x256x32\.F16\.E4M3\.E4M3", sass)) == 4 * N_EPILOGUES  # 2 per cross term
    assert not re.search(r"[HQ]GMMA\.64x(?!256x)", sass), "a narrower wgmma in the wide kernel"
