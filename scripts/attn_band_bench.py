"""Times unmasked head_dim-64 self-attention forward at 385-512 tokens on the two kernels that can serve it: the fused
entry point (ops.attention_fwd, K/V-streamed above 384 tokens) and the general one (ops.attention_fwd_generic, which
keeps Q, K and V resident up to 512 tokens at head_dim 64).  The inference path of CoCa and the standalone layers used
the general kernel in this band until the single attention router sent it to the fused one, as training already did.

    python scripts/attn_band_bench.py [--min-seconds 0.5] [--json OUT]

Work is the algorithmic FLOP count (4 S^2 D per head, halved when causal).  The card's name, power limit and maximum
SM clock are read in the same run and printed with the results.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from attn_bench import card, time_fn  # noqa: E402
from multimodal_b200 import ops  # noqa: E402

B, H, D = 64, 12, 64


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_band_bench.py needs a CUDA GPU")
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    print(f"card: {card()}")
    print(f"{'S':>4s} {'causal':>6s} {'fused ms':>9s} {'TFLOP/s':>8s} {'general ms':>10s} {'TFLOP/s':>8s}")
    rows = []
    d = H * D
    for S in (400, 448, 512):
        for causal in (False, True):
            qkv = (torch.randn(B * S, 3 * d, device=dev) * 0.7).bfloat16()
            out = torch.empty(B * S, d, device=dev, dtype=torch.bfloat16)
            fused = lambda: ops.attention_fwd(qkv, out, None, B, S, H, causal, 0.125)  # noqa: E731
            general = lambda: ops.attention_fwd_generic(  # noqa: E731
                qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], out, B=B, Sq=S, Skv=S, H=H, head_dim=D, bsq=S * 3 * d,
                bsk=S * 3 * d, bsv=S * 3 * d, bso=S * d, scale=0.125, causal=causal)
            flop = 4.0 * S * S * D * H * B * (0.5 if causal else 1.0)
            tf, tg = time_fn(fused, args.min_seconds), time_fn(general, args.min_seconds)
            rows.append({"S": S, "causal": causal, "fused_ms": tf * 1e3, "fused_tflops": flop / tf / 1e12,
                         "general_ms": tg * 1e3, "general_tflops": flop / tg / 1e12})
            print(f"{S:4d} {str(causal):>6s} {tf * 1e3:9.3f} {flop / tf / 1e12:8.1f} {tg * 1e3:10.3f} "
                  f"{flop / tg / 1e12:8.1f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "B": B, "H": H, "head_dim": D, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
