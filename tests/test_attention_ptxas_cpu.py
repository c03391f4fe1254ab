"""CPU: what ptxas made of the self-attention kernels (needs the CUDA toolkit's nvcc, no GPU).

* No attention kernel spills.
* The staged backward (attn_bwd_staged_kernel) runs one warp per 16-row tile, up to 14 warps in one CTA, and relies on
  that many warps being resident to hide mma.sync / ldmatrix / exp2 latency.  Warps are spread over the SM's four
  sub-partitions, each with a quarter of the 64K-register file, so 14 warps (four on some sub-partitions) need at most
  16384 / (4 * 32) = 128 registers per thread.  More registers and the CTA cannot launch at S = 209..224.
"""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from multimodal_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGED_MAX_WARPS = 224 // 16
REGS_PER_SUBPARTITION = 65536 // 4


def _nvcc():
    p = shutil.which("nvcc")
    if p is None and os.path.exists("/usr/local/cuda/bin/nvcc"):
        p = "/usr/local/cuda/bin/nvcc"
    return p


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not installed")
def test_attention_ptxas_spills_and_registers():
    src = os.path.join(ROOT, "multimodal_b200", "csrc", "attention.cu")
    with tempfile.TemporaryDirectory() as td:
        cmd = [_nvcc(), *_lib.NVCC_FLAGS, "-Xptxas", "-v", "-I", os.path.join(ROOT, "multimodal_b200", "csrc"),
               "-I", os.path.join(ROOT, "include"), "-c", src, "-o", os.path.join(td, "attention.o")]
        out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    log = out.stdout + out.stderr
    props = re.findall(r"Function properties for (\S+)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    regs = {}
    for block in log.split("Compiling entry function '")[1:]:
        m = re.search(r"Used (\d+) registers", block)
        regs[block.split("'", 1)[0]] = int(m.group(1))
    kernels = [(f, int(s), int(l)) for f, s, l in props if "attn_" in f]
    # forward, recompute backward and staged backward, causal and not
    assert len(kernels) == 6, kernels
    for f, st, ld in kernels:
        assert st == 0 and ld == 0, (f, st, ld)
    staged = {f: int(r) for f, r in regs.items() if "attn_bwd_staged_kernel" in f}
    assert len(staged) == 2, regs
    warps_per_subpartition = -(-STAGED_MAX_WARPS // 4)
    budget = REGS_PER_SUBPARTITION // (warps_per_subpartition * 32)
    for f, r in staged.items():
        assert r <= budget, (f, r, budget)
