"""Times random patch dropping (FLIP, `vision_patch_drop_rate`) on one GPU.

    python scripts/patch_drop_bench.py [--batch 128] [--steps 10] [--warmup 3] [--front-batch 512] [--json OUT]

1. One CoCaForPretraining training step at CoCa-L/14 shapes (coca_vit_l_14: ViT-L/14 on 224 x 224 images, 256 patches,
   text and fusion decoders of 12 layers, vocabulary 49408): forward, contrastive + captioning losses and backward,
   for vision_patch_drop_rate None, 0.5, 0.75 and (0.5, 0.5).  The same weights serve every rate (the rate is a
   PatchEmbeddings attribute that adds no parameter).  Random images and captions.
2. The patch front end alone at ViT-L/14 shapes (B = --front-batch, d = 1024): gathered im2col, gathered token assembly
   and its backward (dpatch, dpos, no CLS) at 128 and 64 kept patches, next to today's full-sequence kernels
   (im2col, vit_assemble_fwd, vit_assemble_bwd + batch_sum over 256 patches).
Every time is CUDA-event time after warm-up.  The card's name, power limit and SM clocks are read in the same run and
printed with the results.
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

RATES = [None, 0.5, 0.75, (0.5, 0.5)]


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
    emb = m.model.vision_encoder.embeddings
    rows = []
    for rate in RATES:
        emb.patch_drop_rate = rate

        def step():
            m.zero_grad(set_to_none=True)
            out = m(images, texts)
            (out["contrastive"] + out["captioning"]).backward()

        try:
            ms = event_ms(step, args.warmup, args.steps)
            peak = torch.cuda.max_memory_allocated() / 2 ** 30
            rows.append({"rate": rate, "step_ms": round(ms, 2), "images_per_s": round(B * 1e3 / ms, 1),
                         "peak_GiB": round(peak, 1)})
        except torch.cuda.OutOfMemoryError:
            rows.append({"rate": rate, "step_ms": None, "note": f"out of memory at batch {B}"})
        m.zero_grad(set_to_none=True)
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        print(json.dumps(rows[-1]), flush=True)
    base = rows[0]["step_ms"]
    for r in rows:
        if base and r["step_ms"]:
            r["vs_none"] = round(r["step_ms"] / base, 3)
    return rows


def front_end(args, dev):
    B, H, ps, d = args.front_batch, 224, 14, 1024
    P, K, Kp = (H // ps) ** 2, 3 * ps * ps, 592
    gen = torch.Generator(device=dev).manual_seed(2)
    img = torch.randn(B, 3, H, H, device=dev, generator=gen)
    pos = torch.randn(1, P, d, device=dev, generator=gen)
    rows = []
    for L in (P, 128, 64):
        full = L == P
        keep = torch.argsort(torch.rand(B, P, device=dev, generator=gen), 1)[:, :L].to(torch.int32).contiguous()
        patch = torch.empty(B * L, Kp, device=dev, dtype=torch.bfloat16)[:, :K]
        po = torch.randn(B * L, d, device=dev, generator=gen).to(torch.bfloat16)
        x = torch.empty(B * L, d, device=dev)
        gr = torch.randn(B * L, d, device=dev, generator=gen)
        dp = torch.empty(B * L, d, device=dev, dtype=torch.bfloat16)
        dpos = torch.zeros(P, d, device=dev)
        if full:
            t_im = event_ms(lambda: ops.im2col(img, ps, patch), args.warmup, 50)
            t_fwd = event_ms(lambda: ops.vit_assemble_fwd(po, None, pos, None, None, x, B, P, d), args.warmup, 50)

            def bwd():
                ops.batch_sum(gr, dpos, B, P * d, P * d)
                ops.vit_assemble_bwd(gr, None, dp, None, B, P, d, False)
        else:
            t_im = event_ms(lambda: ops._im2col_gather(img, keep, ps, patch), args.warmup, 50)
            t_fwd = event_ms(lambda: ops._vit_assemble_gather_fwd(po, None, pos, None, None, keep, x, P, d),
                             args.warmup, 50)

            def bwd():
                ops._vit_assemble_gather_bwd(gr, None, keep, dp, None, None, dpos, P, d, False)
        t_bwd = event_ms(bwd, args.warmup, 50)
        # bytes each kernel has to move: pixels read + bf16 rows written; bf16 rows + pos read, fp32 rows written;
        # fp32 gradient read (twice: dpatch and dpos), bf16 rows written
        gb = {"im2col": (B * L * K * (4 + 2)) / 1e9, "assemble_fwd": (B * L * d * (2 + 4) + P * d * 4) / 1e9,
              "assemble_bwd": (B * L * d * (4 * 2 + 2)) / 1e9}
        rec = {"kept": L, "kernels": "full (today)" if full else "gathered"}
        for k, t in (("im2col", t_im), ("assemble_fwd", t_fwd), ("assemble_bwd", t_bwd)):
            rec[f"{k}_us"] = round(t * 1e3, 1)
            rec[f"{k}_GBps"] = round(gb[k] / (t * 1e-3), 0)
        rows.append(rec)
        print(json.dumps(rec), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--front-batch", type=int, default=512)
    ap.add_argument("--skip-train", action="store_true")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("patch_drop_bench: no CUDA device")
    if args.steps < 10 or args.warmup < 3:
        raise SystemExit("patch_drop_bench: at least 3 warm-up and 10 timed steps")
    dev = torch.device("cuda:0")
    info = card()
    print("card (name, power limit, SM clock, max SM clock):", info, flush=True)
    res = {"card": info, "front_end": front_end(args, dev)}
    if not args.skip_train:
        res["train_batch"] = args.batch
        res["train_step"] = train_steps(args, dev)
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
