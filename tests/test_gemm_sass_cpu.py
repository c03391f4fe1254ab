"""CPU: what the compiler made of the GEMM kernel (needs the CUDA toolkit's cuobjdump / nvcc, no GPU).

* No GPU-scope memory barrier inside any gemm_kernel's main loop (between its first and last wgmma): a consumer
  releases a shared-memory stage to the peer CTA of its cluster with a plain CTA-scope mbarrier arrive.  (The
  cluster barriers at kernel entry and exit keep their release semantics.)
* ptxas spills nothing in the instantiations on the training step's main-loop-bound kinds.  The QuickGELU'/GELU'
  (EPI_BF16_DACT) and cross-entropy statistics (EPI_CE_STATS) epilogues keep 128 accumulator registers live next to
  their own state and spill a few words in the epilogue; their spill bytes are capped so that growth is caught.
"""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from multimodal_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPI_BF16_DACT, EPI_CE_STATS = 2, 4
EPILOGUE_SPILL_CAP = 128   # bytes of spill stores per DACT / CE_STATS instantiation


def _tool(name):
    p = shutil.which(name)
    if p is None and os.path.exists(f"/usr/local/cuda/bin/{name}"):
        p = f"/usr/local/cuda/bin/{name}"
    return p


def _epilogue(fn):
    # gemm_kernel<A_MN, B_MN, EPI, ACT, CLU>: _ZN3mmb11gemm_kernelILb?ELb?ELi<EPI>ELi<ACT>ELb?E...
    m = re.search(r"gemm_kernelILb[01]ELb[01]ELi(\d+)E", fn)
    return int(m.group(1)) if m else None


@pytest.mark.skipif(_tool("cuobjdump") is None, reason="cuobjdump not installed")
def test_no_gpu_scope_membar_in_gemm_main_loop():
    if not _lib.LIB_PATH.exists():
        pytest.skip("library not built")
    sass = subprocess.run([_tool("cuobjdump"), "-sass", str(_lib.LIB_PATH)], capture_output=True, text=True,
                          check=True).stdout
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs.setdefault(cur, [])
        elif cur is not None:
            funcs[cur].append(line)
    gemm = {f: lines for f, lines in funcs.items() if "gemm_kernel" in f}
    assert len(gemm) >= 20, sorted(funcs)[:10]
    for f, lines in gemm.items():
        hg = [i for i, l in enumerate(lines) if "HGMMA" in l]
        assert hg, f"{f}: no wgmma"
        loop = lines[hg[0]:hg[-1] + 1]
        # the stage release follows the last wgmma of the k-block: include the few instructions after it
        loop += lines[hg[-1] + 1:hg[-1] + 40]
        bad = [l.strip() for l in loop if re.search(r"MEMBAR\.(ALL|SC)\.GPU", l)]
        assert not bad, f"{f}: GPU-scope barrier in the main loop: {bad[:2]}"


@pytest.mark.skipif(_tool("nvcc") is None, reason="nvcc not installed")
def test_gemm_ptxas_spills():
    nvcc = _tool("nvcc")
    src = os.path.join(ROOT, "multimodal_b200", "csrc", "gemm.cu")
    with tempfile.TemporaryDirectory() as td:
        cmd = [nvcc, *_lib.NVCC_FLAGS, "-Xptxas", "-v", "-I", os.path.join(ROOT, "multimodal_b200", "csrc"),
               "-I", os.path.join(ROOT, "include"), "-c", src, "-o", os.path.join(td, "gemm.o")]
        out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    log = out.stdout + out.stderr
    props = re.findall(r"Function properties for (\S+)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    kernels = [(f, int(s), int(l)) for f, s, l in props if "gemm_kernel" in f]
    assert len(kernels) >= 20
    for f, st, ld in kernels:
        if _epilogue(f) in (EPI_BF16_DACT, EPI_CE_STATS):
            assert st <= EPILOGUE_SPILL_CAP and ld <= EPILOGUE_SPILL_CAP, (f, st, ld)
        else:
            assert st == 0 and ld == 0, (f, st, ld)
