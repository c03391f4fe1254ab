"""Times the fused self-attention kernels (mmb_attention_fwd / mmb_attention_bwd) at the shapes of the CLIP training
steps: ViT-B/16 image tower (S = 197), its causal text tower (S = 77) and the ViT-L/14 image tower (S = 257), and at
the lengths served by the streamed kernels (S > 384): ViT-L/14@336 (577), 512-token text, FLAVA's multimodal encoder
(710), S = 4096, and the 384 / 385 boundary between the resident and the streamed kernels.  For the streamed rows the
same bf16 operands also go through torch's scaled_dot_product_attention (flash backend), forward and backward, as a
reference point from the same run.

    python scripts/attn_bench.py [--min-seconds 0.5] [--json OUT]

Each shape is warmed up, then launched until at least --min-seconds of GPU time has been timed with CUDA events.
Work is the algorithmic FLOP count (4 S^2 64 per head forward, 2.5x that backward, halved when causal).  Bytes are
the least HBM traffic per token and head: forward reads q, k, v and writes O and the LSE (516 B); backward reads
q, k, v, O, dO and the LSE and writes dq, dk, dv (1028 B).  The card's name, power limit and maximum SM clock are
read in the same run and printed with the results.
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

# (name, B, S, H, causal)
SHAPES = [
    ("b16 image", 512, 197, 12, False),
    ("b16 text (causal)", 512, 77, 12, True),
    ("l14 image", 256, 257, 16, False),
    ("l14@336", 64, 577, 16, False),
    ("text 512", 64, 512, 12, False),
    ("flava mm", 32, 710, 12, False),
    ("long", 4, 4096, 16, False),
    ("long (causal)", 4, 4096, 16, True),
    ("boundary", 128, 384, 12, False),
    ("boundary", 128, 385, 12, False),
]
STREAMED_MIN_S = 385   # longer sequences take the streamed kernels
FWD_BYTES, BWD_BYTES = 516, 1028   # per token and head


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


def sdpa_fns(qkv, dout, B, S, H, causal):
    """forward and backward of F.scaled_dot_product_attention (flash backend) on the same bf16 operands"""
    from torch.nn.attention import SDPBackend, sdpa_kernel

    q, k, v = (t.detach().requires_grad_(True) for t in qkv.view(B, S, 3, H, 64).permute(2, 0, 3, 1, 4))
    do = dout.view(B, S, H, 64).transpose(1, 2)
    F = torch.nn.functional

    def fwd():
        with sdpa_kernel(SDPBackend.FLASH_ATTENTION), torch.no_grad():
            F.scaled_dot_product_attention(q, k, v, is_causal=causal, scale=0.125)

    with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
        o = F.scaled_dot_product_attention(q, k, v, is_causal=causal, scale=0.125)

    def bwd():
        torch.autograd.grad(o, (q, k, v), do, retain_graph=True)

    return fwd, bwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_bench.py needs a CUDA GPU")
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    print(f"card: {card()}")
    print(f"{'shape':20s} {'B':>4s} {'S':>4s} {'H':>3s} {'dir':>4s} {'ms':>8s} {'TFLOP/s':>8s} {'GB/s':>7s} {'HBM floor':>9s}")
    rows = []
    for name, B, S, H, causal in SHAPES:
        d = H * 64
        qkv = (torch.randn(B * S, 3 * d, device=dev) * 0.7).bfloat16()
        out = torch.empty(B * S, d, device=dev, dtype=torch.bfloat16)
        lse = torch.empty(B * H * S, device=dev)
        dout = (torch.randn(B * S, d, device=dev) * 0.5).bfloat16()
        dqkv = torch.empty_like(qkv)
        fwd = lambda: ops.attention_fwd(qkv, out, lse, B, S, H, causal, 0.125)  # noqa: E731
        bwd = lambda: ops.attention_bwd(qkv, out, dout, lse, dqkv, B, S, H, causal, 0.125)  # noqa: E731
        fwd()
        flop = 4.0 * S * S * 64 * H * B * (0.5 if causal else 1.0)
        for direction, fn, f, nbytes in (("fwd", fwd, flop, FWD_BYTES), ("bwd", bwd, 2.5 * flop, BWD_BYTES)):
            t = time_fn(fn, args.min_seconds)
            gbytes = B * S * H * nbytes / 1e9
            floor_ms = gbytes / 3350.0 * 1e3      # 3.35 TB/s: H100 SXM data sheet, not measured
            rows.append({"shape": name, "B": B, "S": S, "H": H, "causal": causal, "dir": direction, "ms": t * 1e3,
                         "tflops": f / t / 1e12, "gbps": gbytes / t, "hbm_floor_ms": floor_ms})
            r = rows[-1]
            print(f"{name:20s} {B:4d} {S:4d} {H:3d} {direction:>4s} {r['ms']:8.3f} {r['tflops']:8.1f} {r['gbps']:7.0f} "
                  f"{floor_ms:7.3f}ms")
        if S >= STREAMED_MIN_S:
            sfwd, sbwd = sdpa_fns(qkv, dout, B, S, H, causal)
            for direction, fn, f in (("fwd", sfwd, flop), ("bwd", sbwd, 2.5 * flop)):
                t = time_fn(fn, args.min_seconds)
                rows.append({"shape": name + " sdpa-flash", "B": B, "S": S, "H": H, "causal": causal, "dir": direction,
                             "ms": t * 1e3, "tflops": f / t / 1e12})
                print(f"{'  torch sdpa flash':20s} {B:4d} {S:4d} {H:3d} {direction:>4s} {t * 1e3:8.3f} {f / t / 1e12:8.1f}")
            del sfwd, sbwd
        del qkv, out, lse, dout, dqkv
    rate = {(r["shape"], r["dir"]): r["tflops"] for r in rows}
    for direction in ("fwd", "bwd"):
        a, b = rate[("l14@336", direction)], rate[("l14 image", direction)]
        print(f"{direction}: streamed S = 577 {a:.1f} TFLOP/s vs resident S = 257 {b:.1f} TFLOP/s "
              f"({'at least' if a >= b else 'BELOW'} the resident rate)")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
