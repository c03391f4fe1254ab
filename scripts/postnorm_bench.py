"""Times the post-norm TransformerEncoder at BERT-base shapes on one GPU.

    python scripts/postnorm_bench.py [--layers 12] [--tokens 16384] [--steps 10] [--warmup 3] [--repeats 3] [--json OUT]

1. A TransformerEncoder at the reference defaults and BERT-base shapes: 12 layers, d 768, 12 heads, ff 3072, ReLU,
   post-norm, layer_norm_eps 1e-12, with B * S = 16384 tokens at S = 128 and at S = 512.  Per case the training step
   (forward + backward of <upstream, output>) and the torch.no_grad() forward, for three runs:
     postnorm   this package's post-norm runtime;
     prenorm    this package's pre-norm runtime at the same shapes (the same GEMMs and attention kernels: the ceiling);
     eager      torch.nn.TransformerEncoder with norm_first=False and ReLU (the reference layer's arithmetic), eager
                under bf16 autocast with scaled_dot_product_attention.
2. The FC1 GEMM with the ReLU epilogue and the ReLU DACT GEMM against the erf-GELU ones at the FC1 shape of case 1
   (M = 16384, N = 3072, K = 768; the DACT GEMM: K = 768 -> N = 3072 from the [M, 768] gradient).
Every time is CUDA-event time after warm-up, the median of --repeats windows with their min and max.  The card's name,
power limit and SM clocks are read in the same run and printed with the results.

Extra traffic over pre-norm, from the shapes: the FC1 and QKV input gradients are fp32 GEMMs that read and write the
fp32 gradient they accumulate into, about 8 * M * d bytes each per layer (0.1 GB each at M = 16384, d = 768).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from multimodal_b200 import ops  # noqa: E402

D, H, FF = 768, 12, 3072


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else "nvidia-smi unavailable"


def timed(fn, warmup, steps, repeats):
    """(median, min, max) ms per call over `repeats` windows of `steps` calls, after `warmup` calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / steps)
    return round(statistics.median(out), 3), round(min(out), 3), round(max(out), 3)


def build(kind, n_layer, dev):
    torch.manual_seed(0)
    if kind == "eager":
        layer = nn.TransformerEncoderLayer(D, H, FF, dropout=0.0, activation="relu", layer_norm_eps=1e-12,
                                           batch_first=True, norm_first=False)
        return nn.TransformerEncoder(layer, n_layer, enable_nested_tensor=False).to(dev)
    from multimodal_b200.modules.layers.transformer import TransformerEncoder

    return TransformerEncoder(n_layer, D, H, FF, norm_first=kind == "prenorm").to(dev)


def encoder_cases(args, dev):
    rows = []
    for S in (128, 512):
        B = args.tokens // S
        g = torch.Generator(device=dev).manual_seed(S)
        x = torch.randn(B, S, D, device=dev, generator=g)
        up = torch.randn(B, S, D, device=dev, generator=g)
        for kind in ("postnorm", "prenorm", "eager"):
            m = build(kind, args.layers, dev).train()

            def run():
                if kind == "eager":
                    with torch.autocast("cuda", dtype=torch.bfloat16):
                        return m(x)
                return m(x).last_hidden_state

            def step():
                m.zero_grad(set_to_none=True)
                (run().float() * up).sum().backward()

            def infer():
                with torch.no_grad():
                    run()

            row = {"S": S, "B": B, "run": kind, "train_step_ms": timed(step, args.warmup, args.steps, args.repeats)}
            m.eval()
            row["no_grad_forward_ms"] = timed(infer, args.warmup, args.steps, args.repeats)
            rows.append(row)
            print(json.dumps(row), flush=True)
            del m
            torch.cuda.empty_cache()
    return rows


def gemm_cases(args, dev):
    M, N, K = args.tokens, FF, D
    g = torch.Generator(device=dev).manual_seed(3)
    bf = torch.bfloat16
    X = torch.randn(M, K, device=dev, generator=g).to(bf)
    W1 = torch.randn(N, K, device=dev, generator=g).to(bf)
    b1 = torch.randn(N, device=dev, generator=g)
    PRE, HACT = torch.empty(M, N, device=dev, dtype=bf), torch.empty(M, N, device=dev, dtype=bf)
    dY = torch.randn(M, K, device=dev, generator=g).to(bf)
    W2 = torch.randn(K, N, device=dev, generator=g).to(bf)       # FC2 weight [d, ff]: the DACT GEMM reads it [K, N]
    dPRE = torch.empty(M, N, device=dev, dtype=bf)
    cs = torch.zeros(N, device=dev)
    ops.gemm(X, W1, bias=b1, epilogue=ops.EPI_BF16_ACT, out=PRE, out2=HACT, act=ops.ACT_RELU)
    flops = 2.0 * M * N * K
    rows = []
    for name, act in (("relu", ops.ACT_RELU), ("gelu_erf", ops.ACT_GELU_ERF)):
        fwd = timed(lambda: ops.gemm(X, W1, bias=b1, epilogue=ops.EPI_BF16_ACT, out=PRE, out2=HACT, act=act),
                    args.warmup, 50, args.repeats)
        dact = timed(lambda: ops.gemm(dY, W2, b_mn=True, epilogue=ops.EPI_BF16_DACT, aux=PRE, out=dPRE, act=act,
                                      colsum=cs), args.warmup, 50, args.repeats)
        row = {"act": name, "fc1_act_ms": fwd, "fc1_act_TFLOPs": round(flops / fwd[0] / 1e9, 1), "dact_ms": dact,
               "dact_TFLOPs": round(flops / dact[0] / 1e9, 1), "M": M, "N": N, "K": K}
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=12)
    ap.add_argument("--tokens", type=int, default=16384)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("postnorm_bench: needs a CUDA device (nothing is timed on the CPU)")
    dev = torch.device("cuda:0")
    info = {"card": card(), "torch": torch.__version__}
    print(json.dumps(info), flush=True)
    res = {**info, "encoder": encoder_cases(args, dev), "gemm": gemm_cases(args, dev)}
    res["card_after"] = card()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
