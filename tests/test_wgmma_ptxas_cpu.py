"""What ptxas makes of the wgmma kernels (CPU only: nvcc cross-compiles for sm_90a without a GPU).

The GEMM and attention main loops only reach the tensor-core rate if ptxas keeps the wgmma pipeline asynchronous: a wgmma
under a run-time branch or a function call in the loop makes it serialise every wgmma of the kernel ("Potential Performance
Loss: wgmma.mma_async instructions are serialized"), and accumulators spilled to local memory stall it.  This compiles the
GEMM instantiation sources and the streaming attention kernel (attention_tc.cu) exactly as vima_b200/build.py does, plus
-Xptxas -v, and checks

  * no serialisation warning for gemm_tc_kernel or any attention instantiation,
  * no spill bytes in any epilogue-specialised gemm_tc_kernel (the generic runtime-flag variant is exempt) or attention instantiation,
  * the full-width instructions (64x128 fp16 and e4m3; attention's 64x64 and 64x32) are in the SASS.

About 35 s on 8 cores (the sources compile in parallel, like the library build).
"""
import os
import re
import shutil
import subprocess
import tempfile
from concurrent.futures import ThreadPoolExecutor

import pytest

from vima_b200 import build as vbuild

GEMM_SOURCES = sorted(s for s in vbuild.SOURCES if s.startswith("gemm_tc_"))
SOURCES = GEMM_SOURCES + ["attention_tc.cu"]


def _tool(name):
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    path = os.path.join(os.path.dirname(nvcc), name)
    return path if os.path.isfile(path) else None


@pytest.fixture(scope="module")
def compiled():
    nvcc = _tool("nvcc")
    if nvcc is None:
        pytest.skip("nvcc not found")
    tmp = tempfile.mkdtemp(prefix="vima_ptxas_")

    def one(src):
        obj = os.path.join(tmp, src.replace(".cu", ".o"))
        r = subprocess.run([nvcc, *vbuild.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(vbuild.CSRC, src), "-o", obj],
                           capture_output=True, text=True)
        assert r.returncode == 0, f"nvcc failed for {src}:\n{r.stderr[-4000:]}"
        return src, obj, r.stderr

    try:
        with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
            results = list(ex.map(one, SOURCES))
        sass = {}
        cuobjdump = _tool("cuobjdump")
        for src, obj, _ in results:
            if src in ("gemm_tc_f16.cu", "gemm_tc_f16f8.cu", "attention_tc.cu") and cuobjdump:
                sass[src] = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
        yield {src: log for src, _, log in results}, sass
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def _functions(log):
    """-> {mangled kernel name: (spill store bytes, spill load bytes)} from a ptxas -v log."""
    out = {}
    for m in re.finditer(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log):
        out[m.group(1)] = (int(m.group(2)), int(m.group(3)))
    return out


def test_no_serialised_wgmma(compiled):
    logs, _ = compiled
    bad = [ln.strip() for log in logs.values() for ln in log.splitlines()
           if "wgmma.mma_async instructions are serialized" in ln and ("gemm_tc_kernel" in ln or "attention_tc_kernel" in ln)]
    assert not bad, "\n".join(bad)
    assert any("attention_tc_kernel" in k for k in _functions(logs["attention_tc.cu"]))


def test_no_spills_in_specialised_gemms(compiled):
    logs, _ = compiled
    n_specialised, spilled = 0, []
    for src in GEMM_SOURCES:
        for name, spill in _functions(logs[src]).items():
            if "gemm_tc_kernel" not in name or "EpiCfgILb1E" in name:  # EpiCfg<GENERIC=true, ...>: the runtime-flag variant
                continue
            n_specialised += 1
            if spill != (0, 0):
                spilled.append(f"{src}: {name} spills {spill[0]} B stored / {spill[1]} B loaded")
    assert not spilled, "\n".join(spilled)
    # 5 precision modes x 13 epilogues x 4 tile widths, less 32 / 96 for the 2 GLU epilogues
    assert n_specialised == 5 * (13 * 4 - 2 * 2)


def test_full_width_wgmma_in_sass(compiled):
    _, sass = compiled
    if not sass:
        pytest.skip("cuobjdump not found")
    assert re.search(r"HGMMA\.64x128x16\.F32", sass["gemm_tc_f16.cu"])
    assert re.search(r"QGMMA\.64x128x32\.F32\.E4M3\.E4M3", sass["gemm_tc_f16f8.cu"])
    assert re.search(r"HGMMA\.64x128x16\.F32", sass["gemm_tc_f16f8.cu"])


def test_attention_tc_ptxas(compiled):
    """The one streaming attention body's six instantiations: the decoder entry point (attention_tc_kernel, f16 and bf16) and the
    T5 entry point (attention_bias_tc_kernel, {f16, bf16} x {split, single-pass}).  None has a wgmma serialisation warning (C7510 /
    C7520) or spills; the SASS has the M64 N64 K16 wgmmas (QK^T, and PV at head_dim 64) in fp16 and bf16 and the decoder's
    M64 N32 K16 PV wgmma."""
    logs, sass = compiled
    log = logs["attention_tc.cu"]
    bad = [ln.strip() for ln in log.splitlines() if re.search(r"C75[12]0|wgmma\.mma_async instructions are serialized", ln)]
    assert not bad, "\n".join(bad)
    fns = _functions(log)
    decoder = {k: v for k, v in fns.items() if "attention_tc_kernel" in k}
    t5 = {k: v for k, v in fns.items() if "attention_bias_tc_kernel" in k}
    assert len(decoder) == 2 and len(t5) == 4 and len(fns) == 6, fns
    spilled = {k: v for k, v in fns.items() if v != (0, 0)}
    assert not spilled, spilled
    if "attention_tc.cu" not in sass:
        pytest.skip("cuobjdump not found")
    assert re.search(r"HGMMA\.64x64x16\.F32(?!\.BF16)", sass["attention_tc.cu"])
    assert re.search(r"HGMMA\.64x64x16\.F32\.BF16", sass["attention_tc.cu"])
    assert re.search(r"HGMMA\.64x32x16\.F32", sass["attention_tc.cu"])
