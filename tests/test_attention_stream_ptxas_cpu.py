"""CPU: what ptxas made of the streamed self-attention kernels (attention_stream.cu; needs nvcc, no GPU).

* The forward, the dQ backward and the dK / dV backward, causal and not, compile for sm_90a without spilling.
* The launcher plans ST_CTAS_PER_SM CTAs of ST_THREADS threads per SM (constants read from the source): each kernel's
  register count must let that many CTAs share the SM's 64K-register file, or the streamed ring of one CTA has no
  second CTA to overlap its loads with.
"""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from multimodal_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "multimodal_b200", "csrc", "attention_stream.cu")
REGS_PER_SM = 65536


def _nvcc():
    p = shutil.which("nvcc")
    if p is None and os.path.exists("/usr/local/cuda/bin/nvcc"):
        p = "/usr/local/cuda/bin/nvcc"
    return p


def _constant(name):
    m = re.search(rf"constexpr int {name} = (\d+);", open(SRC).read())
    assert m, name
    return int(m.group(1))


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not installed")
def test_streamed_attention_no_spills_and_planned_occupancy():
    with tempfile.TemporaryDirectory() as td:
        cmd = [_nvcc(), *_lib.NVCC_FLAGS, "-Xptxas", "-v", "-I", os.path.join(ROOT, "multimodal_b200", "csrc"),
               "-I", os.path.join(ROOT, "include"), "-c", SRC, "-o", os.path.join(td, "attention_stream.o")]
        out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    log = out.stdout + out.stderr
    props = re.findall(r"Function properties for (\S+)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    kernels = [(f, int(s), int(l)) for f, s, l in props if "attn_" in f]
    names = ("attn_fwd_stream_kernel", "attn_bwd_stream_dq_kernel", "attn_bwd_stream_dkdv_kernel")
    assert len(kernels) == 6 and all(sum(n in f for f, _, _ in kernels) == 2 for n in names), kernels
    for f, st, ld in kernels:
        assert st == 0 and ld == 0, (f, st, ld)
    regs = {}
    for block in log.split("Compiling entry function '")[1:]:
        m = re.search(r"Used (\d+) registers", block)
        regs[block.split("'", 1)[0]] = int(m.group(1))
    threads, ctas = _constant("ST_THREADS"), _constant("ST_CTAS_PER_SM")
    budget = REGS_PER_SM // (threads * ctas)
    streamed = {f: r for f, r in regs.items() if any(n in f for n in names)}
    assert len(streamed) == 6, regs
    for f, r in streamed.items():
        assert r <= budget, (f, r, budget)
