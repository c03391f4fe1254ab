"""Times the general attention entry points (mmb_attention_fwd_generic / mmb_attention_bwd_generic) at shapes past the
resident kernel's shared-memory bound, where the streamed kernels serve them: the CoCa ViT-L/14@336 captioning pooler
(256 batch-shared queries over 576 keys, head_dim 96), the parallel pooler (257 queries), head_dim-64 causal
self-attention at S = 1024 with a [B, S, S] mask, and cross-attention 77 x 1024.  One shape just inside the bound
(ViT-L/14@224's pooler: 256 keys) shows the resident forward and SIMT backward on the other side of the switch.  Each
row names the path mmb_attention_generic_streamed reports, and the same bf16 operands also go through torch's
F.scaled_dot_product_attention (whichever backend torch picks for the mask), forward and backward.

    python scripts/attn_generic_bench.py [--min-seconds 0.5] [--json OUT]

Work is the algorithmic FLOP count (4 Sq Skv D per head forward, 2.5x that backward, halved when causal).  The card's
name, power limit and maximum SM clock are read in the same run and printed with the results.
"""
import argparse
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from attn_bench import card, time_fn  # noqa: E402
from multimodal_b200 import _lib, ops  # noqa: E402

# (name, B, Sq, Skv, H, D, shared queries, mask, causal)
SHAPES = [
    ("pooler l14@336", 64, 256, 576, 8, 96, True, None, False),
    ("parallel pooler", 64, 257, 576, 8, 96, True, None, False),
    ("masked causal 1024", 16, 1024, 1024, 12, 64, False, "full", True),
    ("cross 77x1024", 64, 77, 1024, 12, 64, False, None, False),
    ("pooler l14@224", 64, 256, 256, 8, 96, True, None, False),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_generic_bench.py needs a CUDA GPU")
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    F = torch.nn.functional
    print(f"card: {card()}")
    print(f"{'shape':22s} {'B':>3s} {'Sq':>4s} {'Skv':>4s} {'H':>3s} {'D':>3s} {'path':>8s} {'dir':>4s} {'ms':>8s} "
          f"{'TFLOP/s':>8s}")
    rows = []
    for name, B, Sq, Skv, H, D, shared, mask_kind, causal in SHAPES:
        d, scale = H * D, 1.0 / math.sqrt(D)
        path = "streamed" if _lib.lib().mmb_attention_generic_streamed(Sq, Skv, D) else "resident"
        q = (torch.randn((1 if shared else B) * Sq, d, device=dev) * 0.7).bfloat16()
        kv = (torch.randn(B * Skv, 2 * d, device=dev) * 0.7).bfloat16()
        dout = (torch.randn(B * Sq, d, device=dev) * 0.5).bfloat16()
        out = torch.empty(B * Sq, d, device=dev, dtype=torch.bfloat16)
        dkv = torch.empty_like(kv)
        mask = None
        if mask_kind == "full":
            mask = torch.rand(B, Sq, Skv, device=dev) < 0.9
            mask[:, :, 0] = True
        mu8 = mask.to(torch.uint8).contiguous() if mask is not None else None
        kw = dict(B=B, Sq=Sq, Skv=Skv, H=H, head_dim=D, bsq=0 if shared else Sq * d, bsk=Skv * 2 * d,
                  bsv=Skv * 2 * d, bso=Sq * d, scale=scale, mask=mu8, mask_bs=Sq * Skv if mask is not None else 0,
                  mask_qs=Skv if mask is not None else 0, causal=causal)
        dq = None if shared else torch.empty_like(q)
        dq32 = torch.zeros(Sq, d, device=dev) if shared else None
        fwd = lambda: ops.attention_fwd_generic(q, kv[:, :d], kv[:, d:], out, **kw)  # noqa: E731
        bwd = lambda: ops.attention_bwd_generic(q, kv[:, :d], kv[:, d:], dout, dkv[:, :d], dkv[:, d:], dq=dq,  # noqa: E731
                                                dq_f32=dq32, **kw)
        fwd()
        flop = 4.0 * Sq * Skv * D * H * B * (0.5 if causal else 1.0)
        for direction, fn, f in (("fwd", fwd, flop), ("bwd", bwd, 2.5 * flop)):
            t = time_fn(fn, args.min_seconds)
            rows.append({"shape": name, "B": B, "Sq": Sq, "Skv": Skv, "H": H, "D": D, "path": path, "dir": direction,
                         "ms": t * 1e3, "tflops": f / t / 1e12})
            print(f"{name:22s} {B:3d} {Sq:4d} {Skv:4d} {H:3d} {D:3d} {path:>8s} {direction:>4s} {t * 1e3:8.3f} "
                  f"{f / t / 1e12:8.1f}")
        # torch SDPA on the same operands (queries expanded over the batch for the pooler)
        qh = (q.view(1, Sq, H, D).expand(B, Sq, H, D) if shared else q.view(B, Sq, H, D)).transpose(1, 2)
        qh = qh.detach().requires_grad_(True)
        kh = kv[:, :d].reshape(B, Skv, H, D).transpose(1, 2).detach().requires_grad_(True)
        vh = kv[:, d:].reshape(B, Skv, H, D).transpose(1, 2).detach().requires_grad_(True)
        am = None
        if mask is not None:
            am = mask[:, None]
            if causal:
                am = am & torch.ones(Sq, Skv, device=dev, dtype=torch.bool).tril()
        sc = causal and am is None
        do = dout.view(B, Sq, H, D).transpose(1, 2)

        def sfwd():
            with torch.no_grad():
                F.scaled_dot_product_attention(qh, kh, vh, attn_mask=am, is_causal=sc, scale=scale)

        o = F.scaled_dot_product_attention(qh, kh, vh, attn_mask=am, is_causal=sc, scale=scale)

        def sbwd():
            torch.autograd.grad(o, (qh, kh, vh), do, retain_graph=True)

        for direction, fn, f in (("fwd", sfwd, flop), ("bwd", sbwd, 2.5 * flop)):
            t = time_fn(fn, args.min_seconds)
            rows.append({"shape": name + " sdpa", "B": B, "Sq": Sq, "Skv": Skv, "H": H, "D": D, "path": "torch",
                         "dir": direction, "ms": t * 1e3, "tflops": f / t / 1e12})
            print(f"{'  torch sdpa':22s} {B:3d} {Sq:4d} {Skv:4d} {H:3d} {D:3d} {'torch':>8s} {direction:>4s} "
                  f"{t * 1e3:8.3f} {f / t / 1e12:8.1f}")
        del o, sfwd, sbwd, qh, kh, vh, q, kv, dout, out, dkv, mask, mu8, dq, dq32
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
