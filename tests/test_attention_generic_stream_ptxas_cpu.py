"""CPU: what ptxas made of the streamed general attention kernels (attention_generic_stream.cu; needs nvcc, no GPU), and
which shapes the general entry points send to them.

* The forward, the dQ backward and the dK / dV backward, for head_dim 64 / 96 / 128, causal and not, compile for sm_90a
  without spilling.
* Each kernel's register count lets GS_*_CTAS_PER_SM_D<head_dim> CTAs of GS_THREADS threads (constants read from the
  source) share the SM's 64K-register file.
* mmb_attention_generic_streamed switches at the resident forward's shared-memory bound (the library loads without a
  GPU).
"""
import ctypes
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from multimodal_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "multimodal_b200", "csrc", "attention_generic_stream.cu")
REGS_PER_SM = 65536
KINDS = {"attn_fwd_gstream_kernel": "FWD", "attn_bwd_gstream_dq_kernel": "DQ", "attn_bwd_gstream_dkdv_kernel": "DKDV"}


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
def test_generic_streamed_attention_no_spills_and_planned_occupancy():
    with tempfile.TemporaryDirectory() as td:
        cmd = [_nvcc(), *_lib.NVCC_FLAGS, "-Xptxas", "-v", "-I", os.path.join(ROOT, "multimodal_b200", "csrc"),
               "-I", os.path.join(ROOT, "include"), "-c", SRC, "-o", os.path.join(td, "attention_generic_stream.o")]
        out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    log = out.stdout + out.stderr
    props = re.findall(r"Function properties for (\S+)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    assert props
    for f, st, ld in props:
        assert int(st) == 0 and int(ld) == 0, (f, st, ld)
    regs = {}
    for block in log.split("Compiling entry function '")[1:]:
        m = re.search(r"Used (\d+) registers", block)
        regs[block.split("'", 1)[0]] = int(m.group(1))
    threads = _constant("GS_THREADS")
    seen = set()
    for f, r in regs.items():
        kind = next((v for k, v in KINDS.items() if k in f), None)
        if kind is None:
            continue
        m = re.search(r"ILi(\d+)ELb([01])E", f)
        assert m, f
        D, causal = int(m.group(1)), int(m.group(2))
        seen.add((kind, D, causal))
        budget = REGS_PER_SM // (threads * _constant(f"GS_{kind}_CTAS_PER_SM_D{D}"))
        assert r <= min(budget, 255), (f, r, budget)
    assert seen == {(k, D, c) for k in KINDS.values() for D in (64, 96, 128) for c in (0, 1)}, sorted(seen)


def test_generic_streamed_switch_at_the_shared_memory_bound():
    lib = ctypes.CDLL(str(_lib.LIB_PATH))
    f = lib.mmb_attention_generic_streamed
    f.restype, f.argtypes = ctypes.c_int, [ctypes.c_int] * 3
    for D, S in ((64, 512), (96, 336), (128, 256)):   # largest self-attention the resident forward takes, and one more
        assert f(S, S, D) == 0 and f(S + 1, S + 1, D) == 1, D
    assert f(256, 256, 96) == 0                       # ViT-L/14 pooler at 224 px: unchanged path
    assert f(256, 576, 96) == 1 and f(257, 576, 96) == 1 and f(32, 576, 96) == 1
    assert f(76, 256, 64) == 0 and f(77, 1025, 64) == 1 and f(1, 1500, 128) == 1
    assert f(600, 600, 80) == 0 and f(0, 600, 64) == 0   # unsupported head_dim / empty shapes: not the streamed path


def test_generic_streamed_rejects_unaligned_outputs():
    """The streamed kernels move 16-byte row chunks: an output view that is not 16-byte aligned is refused with
    MMB_ERR_ARG before anything is launched (the addresses below are never dereferenced)."""
    lib = ctypes.CDLL(str(_lib.LIB_PATH))
    vp, ll, i32 = ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int
    fwd, bwd = lib.mmb_attention_fwd_generic, lib.mmb_attention_bwd_generic
    fwd.restype = bwd.restype = i32
    fwd.argtypes = [vp, ll, ll, vp, ll, ll, vp, ll, ll, vp, ll, ll, vp, ll, ll, i32, i32, i32, i32, i32, i32,
                    ctypes.c_float, vp]
    bwd.argtypes = [vp, ll, ll, vp, ll, ll, vp, ll, ll, vp, ll, ll, vp, ll, ll, vp, vp, ll, vp, vp, vp, i32, i32, i32,
                    i32, i32, i32, ctypes.c_float, vp]
    B, Sq, Skv, H, D = 2, 77, 1025, 2, 64   # streamed
    d = H * D
    q, k, v, dout, base = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000
    scratch = 0x60000
    for out in (base + 8, base + 2):
        assert fwd(q, d, Sq * d, k, 2 * d, Skv * 2 * d, v, 2 * d, Skv * 2 * d, out, d, Sq * d, None, 0, 0,
                   B, Sq, Skv, H, D, 0, 0.125, None) == -22
    for dq, dk, dv in ((base + 8, base, base + 0x1000), (base, base + 8, base + 0x1000), (None, base, base + 0x1008)):
        assert bwd(q, d, Sq * d, k, 2 * d, Skv * 2 * d, v, 2 * d, Skv * 2 * d, dout, d, Sq * d, None, 0, 0, dq, None, 0,
                   dk, dv, scratch, B, Sq, Skv, H, D, 0, 0.125, None) == -22
