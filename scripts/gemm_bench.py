"""Times every GEMM kind of the CLIP ViT-B/16 training step (512 pairs per GPU) at its exact shape, epilogue and
split count, next to torch.matmul (cuBLAS) on the same bf16 operands.

    python scripts/gemm_bench.py [--min-seconds 0.5] [--json OUT]

Each shape is warmed up, then launched until at least --min-seconds of GPU time has been timed with CUDA events.
The card's name, power limit and maximum SM clock are read in the same run and printed with the results.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from multimodal_b200 import ops  # noqa: E402

B = 512
IMG_M, IMG_D, IMG_FF = B * 197, 768, 3072      # image tower: 197 tokens per image
TXT_M, TXT_D, TXT_FF = B * 77, 512, 2048       # text tower: 77 tokens per caption
PATCH_M, PATCH_K = B * 196, 3 * 16 * 16


def kinds():
    """(name, M, N, K, a_mn, b_mn, epilogue, splits, launches per step)"""
    out = []
    for tower, M, d, ff in (("img", IMG_M, IMG_D, IMG_FF), ("txt", TXT_M, TXT_D, TXT_FF)):
        out += [
            (f"{tower} fwd qkv", M, 3 * d, d, 0, 0, ops.EPI_BF16, 1, 12),
            (f"{tower} fwd out-proj", M, d, d, 0, 0, ops.EPI_BF16, 1, 12),
            (f"{tower} fwd fc1+act", M, ff, d, 0, 0, ops.EPI_BF16_ACT, 1, 12),
            (f"{tower} fwd fc2", M, d, ff, 0, 0, ops.EPI_BF16, 1, 12),
            (f"{tower} dgrad qkv", M, d, 3 * d, 0, 1, ops.EPI_BF16, 1, 12),
            (f"{tower} dgrad out-proj", M, d, d, 0, 1, ops.EPI_BF16, 1, 12),
            (f"{tower} dgrad fc1", M, d, ff, 0, 1, ops.EPI_BF16, 1, 12),
            (f"{tower} dgrad fc2 x act'", M, ff, d, 0, 1, ops.EPI_BF16_DACT, 1, 12),
        ]
        for name, r, c in (("qkv", 3 * d, d), ("out-proj", d, d), ("fc1", ff, d), ("fc2", d, ff)):
            out.append((f"{tower} wgrad {name}", r, c, M, 1, 1, ops.EPI_F32, ops.wgrad_splits(r, c, M), 12))
    out.append(("img fwd patch", PATCH_M, IMG_D, PATCH_K, 0, 0, ops.EPI_BF16, 1, 1))
    return out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else "nvidia-smi unavailable"


def time_fn(fn, min_seconds):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n, total = 2, 0.0
    while True:
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        e1.synchronize()
        total = e0.elapsed_time(e1) * 1e-3
        if total >= min_seconds:
            return total / n
        n = max(2 * n, int(n * 1.2 * min_seconds / max(total, 1e-6)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_bench.py needs a CUDA GPU")
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    print(f"card: {card()}")
    print(f"{'kind':26s} {'M':>7s} {'N':>5s} {'K':>7s} {'split':>5s} {'mmb TF/s':>9s} {'cuBLAS TF/s':>11s} {'ms/step':>8s}")
    rows, tot_ms, tot_f = [], 0.0, 0.0
    for name, M, N, K, a_mn, b_mn, epi, splits, per_step in kinds():
        A = (torch.randn(K, M, device=dev) if a_mn else torch.randn(M, K, device=dev)).bfloat16()
        Bm = (torch.randn(K, N, device=dev) if b_mn else torch.randn(N, K, device=dev)).bfloat16()
        out = torch.empty(M, N, device=dev, dtype=torch.float32 if epi == ops.EPI_F32 else torch.bfloat16)
        out2 = torch.empty(M, N, device=dev, dtype=torch.bfloat16) if epi == ops.EPI_BF16_ACT else None
        aux = torch.randn(M, N, device=dev).bfloat16() if epi == ops.EPI_BF16_DACT else None
        bias = torch.zeros(N, device=dev) if epi in (ops.EPI_BF16, ops.EPI_BF16_ACT) else None
        colsum = torch.zeros(N, device=dev) if epi in (ops.EPI_BF16, ops.EPI_BF16_DACT) and b_mn else None
        t = time_fn(lambda: ops.gemm(A, Bm, a_mn=bool(a_mn), b_mn=bool(b_mn), epilogue=epi, out=out, out2=out2,
                                     bias=bias, aux=aux, splits=splits, colsum=colsum), args.min_seconds)
        # cuBLAS yardstick: the same contraction on the same bf16 operands, bf16 output, no fused epilogue
        ta = A.t() if a_mn else A
        tb = Bm if b_mn else Bm.t()
        tc = time_fn(lambda: torch.matmul(ta, tb), args.min_seconds)
        f = 2.0 * M * N * K
        tot_ms += t * 1e3 * per_step
        tot_f += f * per_step
        rows.append({"kind": name, "M": M, "N": N, "K": K, "splits": splits, "tflops": f / t / 1e12,
                     "cublas_tflops": f / tc / 1e12, "ms_per_step": t * 1e3 * per_step})
        r = rows[-1]
        print(f"{name:26s} {M:7d} {N:5d} {K:7d} {splits:5d} {r['tflops']:9.1f} {r['cublas_tflops']:11.1f} {r['ms_per_step']:8.2f}")
        del A, Bm, out, out2, aux
    print(f"{'all GEMMs of one step':26s} {'':29s} {tot_f / (tot_ms * 1e-3) / 1e12:9.1f} {'':11s} {tot_ms:8.2f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "rows": rows, "total_ms_per_step": tot_ms}, f, indent=1)


if __name__ == "__main__":
    main()
