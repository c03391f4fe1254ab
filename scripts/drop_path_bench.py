"""Times stochastic depth (`vision_drop_path_rate`) on one GPU.

    python scripts/drop_path_bench.py [--batch 128] [--steps 10] [--warmup 3] [--json OUT]

1. One CoCaForPretraining training step at CoCa-L/14 shapes (coca_vit_l_14: ViT-L/14 on 224 x 224 images, 256 patches,
   text and fusion decoders of 12 layers, vocabulary 49408): forward, contrastive + captioning losses and backward, for
   vision_drop_path_rate None, 0.1 and 0.4, each alone and with vision_patch_drop_rate 0.5.  The same weights serve
   every setting (neither rate adds a parameter: the layers' StochasticDepth / nn.Dropout modules and the embeddings'
   patch_drop_rate are swapped in place).  Random images and captions; the noise is drawn anew every step.
2. The residual-add + LayerNorm forward and the LayerNorm backward at ViT-L/14 shapes (M = 512 * 256 rows, d = 1024),
   unscaled and with a per-sample factor (256 rows per factor), in GB/s of the bytes each kernel has to move.
Every time is CUDA-event time after warm-up.  The card's name, power limit and SM clocks are read in the same run and
printed with the results.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from multimodal_b200 import ops  # noqa: E402
from multimodal_b200.modules.layers.stochastic_depth import StochasticDepth  # noqa: E402

SETTINGS = [(None, None), (0.1, None), (0.4, None), (None, 0.5), (0.1, 0.5), (0.4, 0.5)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else "nvidia-smi unavailable"


def event_ms(fn, warmup, steps):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def set_drop_path(layers, rate):
    """What TransformerEncoder(drop_path_rate=rate) builds, on existing layers."""
    rates = torch.linspace(0, rate, len(layers)).tolist() if rate is not None else [None] * len(layers)
    for layer, p in zip(layers, rates):
        if p is None:
            layer.attention_dropout, layer.feedforward_dropout = nn.Dropout(0.0), nn.Dropout(0.0)
        else:
            layer.attention_dropout = layer.feedforward_dropout = StochasticDepth(p, "row")


def train_steps(args, dev):
    from multimodal_b200.models.coca.coca_model import coca_for_pretraining

    kw = dict(vision_patch_size=14, vision_n_layer=24, vision_n_head=16, vision_dim_feedforward=4096,
              vision_include_cls_embed=False, vocab_size=49408, num_text_positions=77, text_hidden_dim=768,
              text_n_layer=12, text_n_head=12, text_dim_feedforward=3072, text_output_dim=768, fusion_n_layer=12,
              fusion_n_head=12, fusion_dim_feedforward=3072, multimodal_output_projection_dim=49408,
              pooler_input_embed_dim=1024, pooler_output_embed_dim=768, pooler_n_head=8, cascaded_pooler=True)
    torch.manual_seed(0)
    with torch.device(dev):
        m = coca_for_pretraining(**kw)
    m = m.to(dev).train()
    B = args.batch
    g = torch.Generator(device=dev).manual_seed(1)
    images = torch.randn(B, 3, 224, 224, device=dev, generator=g)
    texts = torch.randint(1, 49408, (B, 77), device=dev, generator=g)
    vis = m.model.vision_encoder
    rows = []
    for rate, patch_rate in SETTINGS:
        set_drop_path(vis.encoder.layer, rate)
        vis.train()
        vis.embeddings.patch_drop_rate = patch_rate

        def step():
            m.zero_grad(set_to_none=True)
            out = m(images, texts)
            (out["contrastive"] + out["captioning"]).backward()

        try:
            ms = event_ms(step, args.warmup, args.steps)
            peak = torch.cuda.max_memory_allocated() / 2 ** 30
            rows.append({"drop_path_rate": rate, "patch_drop_rate": patch_rate, "step_ms": round(ms, 2),
                         "images_per_s": round(B * 1e3 / ms, 1), "peak_GiB": round(peak, 1)})
        except torch.cuda.OutOfMemoryError:
            rows.append({"drop_path_rate": rate, "patch_drop_rate": patch_rate, "step_ms": None,
                         "note": f"out of memory at batch {B}"})
        m.zero_grad(set_to_none=True)
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        print(json.dumps(rows[-1]), flush=True)
    return rows


def kernels(args, dev):
    B, S, d = 512, 256, 1024
    M = B * S
    gen = torch.Generator(device=dev).manual_seed(2)
    x = torch.randn(M, d, device=dev, generator=gen)
    y = torch.randn(M, d, device=dev, generator=gen).to(torch.bfloat16)
    xo = torch.empty(M, d, device=dev)
    ln = torch.empty(M, d, device=dev, dtype=torch.bfloat16)
    mean, rstd = torch.empty(M, device=dev), torch.empty(M, device=dev)
    gamma, beta = torch.ones(d, device=dev), torch.zeros(d, device=dev)
    g = torch.randn(M, d, device=dev, generator=gen)
    gb = torch.empty(M, d, device=dev, dtype=torch.bfloat16)
    dg, db, gs = (torch.zeros(d, device=dev) for _ in range(3))
    scale = torch.empty(B, device=dev).bernoulli_(0.9, generator=gen).div_(0.9)
    ops.add_layernorm_fwd(x, None, None, None, None, gamma, beta, mean, rstd, M, d, 1e-5)   # LN statistics of x
    # bytes each kernel moves: fwd reads x fp32 + y bf16, writes x_out fp32 + LN bf16 (+ 8 B of statistics per row);
    # bwd reads x fp32 + dy bf16 + g_in fp32, writes g_out fp32 + g_bf16 (+ 8 B of statistics per row); + 4 B per factor
    fwd_b, bwd_b = M * d * 12 + M * 8, M * d * 16 + M * 8
    rows = []
    for scaled in (False, True):
        s = scale if scaled else None
        t_f = event_ms(lambda: ops.add_layernorm_fwd(x, y, xo, ln, None, gamma, beta, mean, rstd, M, d, 1e-5,
                                                     branch_scale=s, rows_per_scale=S), args.warmup, 30)
        t_b = event_ms(lambda: ops.layernorm_bwd(x, ln, None, mean, rstd, gamma, g, g, gb, dg, db, M, d, gsum=gs,
                                                 branch_scale=s, rows_per_scale=S), args.warmup, 30)
        extra = 4 * B if scaled else 0
        rec = {"scaled": scaled, "add_ln_fwd_us": round(t_f * 1e3, 1),
               "add_ln_fwd_GBps": round((fwd_b + extra) / (t_f * 1e-3) / 1e9, 0),
               "ln_bwd_us": round(t_b * 1e3, 1), "ln_bwd_GBps": round((bwd_b + extra) / (t_b * 1e-3) / 1e9, 0)}
        rows.append(rec)
        print(json.dumps(rec), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-train", action="store_true")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("drop_path_bench: no CUDA device")
    if args.steps < 10 or args.warmup < 3:
        raise SystemExit("drop_path_bench: at least 3 warm-up and 10 timed steps")
    dev = torch.device("cuda:0")
    info = card()
    print("card (name, power limit, SM clock, max SM clock):", info, flush=True)
    res = {"card": info, "kernels": kernels(args, dev)}
    if not args.skip_train:
        res["train_batch"] = args.batch
        res["train_step"] = train_steps(args, dev)
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
