"""Loader / builder for libmmb200.so, the C-ABI shared library holding every sm_90a kernel.

The library is built in-tree (``multimodal_b200/libmmb200.so``) with plain ``nvcc`` so that it travels
with the repository snapshot to the GPU box.  There is NO fallback: if the library is missing, or a
kernel returns a non-zero status, the caller gets an exception.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from pathlib import Path

_HERE = Path(__file__).resolve().parent
_CSRC = _HERE / "csrc"
LIB_PATH = _HERE / "libmmb200.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-diag-suppress", "177",
]


def sources() -> list[Path]:
    return sorted(_CSRC.glob("*.cu"))


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile csrc/*.cu -> libmmb200.so (cross-compiles without a GPU)."""
    srcs = sources()
    deps = srcs + sorted(_CSRC.glob("*.cuh")) + sorted(_CSRC.glob("*.h"))
    if not force and LIB_PATH.exists():
        newest = max(p.stat().st_mtime for p in deps)
        if LIB_PATH.stat().st_mtime >= newest:
            return LIB_PATH
    nvcc = os.environ.get("NVCC", "nvcc")
    objdir = _HERE / "build"
    objdir.mkdir(exist_ok=True)
    procs = []
    objs = []
    for s in srcs:
        o = objdir / (s.stem + ".o")
        objs.append(o)
        if not force and o.exists() and o.stat().st_mtime >= max(
            s.stat().st_mtime, *(p.stat().st_mtime for p in deps if p.suffix in (".cuh", ".h"))
        ):
            continue
        cmd = [nvcc, *NVCC_FLAGS, "-I", str(_CSRC), "-I", str(_HERE.parent / "include"), "-c", str(s), "-o", str(o)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed for {s}:\n{out}")
        if verbose and out:
            print(out)
    # link into a temporary name and rename: a concurrent reader (another rank importing the package, a snapshot of
    # the tree) never sees a half-written library
    tmp = LIB_PATH.with_name(LIB_PATH.name + f".tmp{os.getpid()}")
    link = [nvcc, "-shared", "-o", str(tmp), *map(str, objs), "-lcudart_static", "-ldl", "-lpthread", "-lrt"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        tmp.unlink(missing_ok=True)
        raise RuntimeError(f"link failed:\n{r.stdout}")
    os.replace(tmp, LIB_PATH)
    return LIB_PATH


_lib = None


class MMBError(RuntimeError):
    pass


def lib() -> ctypes.CDLL:
    """Return the loaded library; raise loudly if it has not been built."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise MMBError(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU / PyTorch fallback for the CUDA path)"
            )
        _lib = ctypes.CDLL(str(LIB_PATH))
        from . import _abi

        _abi.declare(_lib)
    return _lib


LAUNCHES = 0  # kernels launched through the C ABI (bench.py reports the count inside its timed region)


def check(rc: int, what: str) -> None:
    global LAUNCHES
    if rc != 0:
        raise MMBError(f"{what} failed with status {rc}")
    if what != "mmb_memset_async":
        LAUNCHES += 1   # ops.attention_bwd adds the second kernel of the two-pass backward itself
