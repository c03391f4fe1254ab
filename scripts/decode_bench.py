"""Times autoregressive decoding with a key / value cache.

1. Attention kernels on the same bf16 operands: the split-KV decode kernel (mmb_attention_fwd_decode), the general
   kernel (mmb_attention_fwd_generic) and torch's F.scaled_dot_product_attention, at Sq 1 / 4 / 16 (and Sq 17 on the
   general path, the other side of the switch), Skv 77 / 512 / 4096 / 65536, (B, H) (1, 12) / (8, 12) / (64, 12),
   head_dim 64 / 128.  The kernels are bound by HBM: the figure of merit is the K / V bytes (4 Skv D per head) over the
   time, as GB/s and as a share of the H100 SXM data-sheet 3.35 TB/s.
2. Per-token latency of one step of a 12-layer d = 768 TransformerDecoder (12 heads, cross-attention over 256 image
   tokens, a cache of 76 tokens) at B = 1 and 32, against the reference formulation (F.linear, SDPA, LayerNorm in fp32,
   as torchmultimodal runs it) executed eagerly on the same GPU, and the step's GPU time split by kernel family
   (torch.profiler, a separate run), which shows the share of the projection GEMMs at M = B.

    python scripts/decode_bench.py [--min-seconds 0.2] [--json OUT] [--skip-kernels] [--skip-step]

The card's name, power limit and maximum SM clock are read in the same run and printed with the results.
"""
import argparse
import json
import math
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from attn_bench import card, time_fn  # noqa: E402
from multimodal_b200 import ops  # noqa: E402

HBM = 3.35e12


def kernel_table(min_seconds):
    dev = torch.device("cuda:0")
    rows = []
    print(f"{'D':>3s} {'B':>3s} {'H':>3s} {'Skv':>6s} {'Sq':>3s} {'splits':>6s} {'decode us':>10s} {'general us':>10s} "
          f"{'sdpa us':>9s} {'decode GB/s':>11s} {'%HBM':>5s} {'general GB/s':>12s} {'%HBM':>5s}")
    for D in (64, 128):
        for B, H in ((1, 12), (8, 12), (64, 12)):
            for Skv in (77, 512, 4096, 65536):
                d = H * D
                kv = torch.randn(B * Skv, 2 * d, device=dev).bfloat16()
                k, v = kv[:, :d], kv[:, d:]
                kh = kv.view(B, Skv, 2, H, D)[:, :, 0].transpose(1, 2)
                vh = kv.view(B, Skv, 2, H, D)[:, :, 1].transpose(1, 2)
                nbytes = 4.0 * B * H * Skv * D
                for Sq in (1, 4, 16, 17):
                    q = torch.randn(B * Sq, d, device=dev).bfloat16()
                    o1, o2 = (torch.empty(B * Sq, d, device=dev, dtype=torch.bfloat16) for _ in range(2))
                    kw = dict(B=B, Sq=Sq, Skv=Skv, H=H, head_dim=D, bsq=Sq * d, bsk=Skv * 2 * d, bsv=Skv * 2 * d,
                              bso=Sq * d, scale=1 / math.sqrt(D))
                    t_dec = None
                    if Sq <= ops.DECODE_MAX_SQ:
                        t_dec = time_fn(lambda: ops.attention_fwd_decode(q, k, v, o1, **kw), min_seconds)
                    t_gen = time_fn(lambda: ops.attention_fwd_generic(q, k, v, o2, **kw), min_seconds)
                    qh = q.view(B, Sq, H, D).transpose(1, 2)
                    try:
                        t_sdpa = time_fn(lambda: F.scaled_dot_product_attention(qh, kh, vh), min_seconds)
                    except RuntimeError:
                        t_sdpa = None
                    diff = None
                    if t_dec is not None:
                        diff = (o1.float() - o2.float()).abs().max().item()
                    r = dict(D=D, B=B, H=H, Skv=Skv, Sq=Sq, splits=ops.attention_decode_splits(B, H, Skv),
                             decode_us=t_dec and t_dec * 1e6, general_us=t_gen * 1e6, sdpa_us=t_sdpa and t_sdpa * 1e6,
                             decode_gbs=t_dec and nbytes / t_dec / 1e9, general_gbs=nbytes / t_gen / 1e9,
                             max_diff_decode_vs_general=diff)
                    rows.append(r)
                    f = lambda x, w, p=1: f"{x:{w}.{p}f}" if x is not None else f"{'-':>{w}s}"
                    print(f"{D:3d} {B:3d} {H:3d} {Skv:6d} {Sq:3d} {r['splits']:6d} {f(r['decode_us'], 10)} "
                          f"{f(r['general_us'], 10)} {f(r['sdpa_us'], 9)} {f(r['decode_gbs'], 11, 0)} "
                          f"{f(r['decode_gbs'] and 100 * r['decode_gbs'] * 1e9 / HBM, 5, 0)} "
                          f"{f(r['general_gbs'], 12, 0)} {f(100 * r['general_gbs'] * 1e9 / HBM, 5, 0)}", flush=True)
                del kv, k, v, kh, vh
                torch.cuda.empty_cache()
    return rows


# ---- one decoder step ------------------------------------------------------------------------------------------------
def _ref_layer(m, x, enc, past):
    """TransformerDecoderLayer._forward_prenorm (torchmultimodal/modules/layers/transformer.py:390-428) with
    MultiHeadAttentionWithCache.forward (multi_head_attention.py:141-180), eager fp32."""
    def mha(a, q, kv, past=None):
        B, Sq, d = q.shape
        H = a.num_heads
        hd = d // H
        Q = F.linear(q, a.q_proj.weight, a.q_proj.bias).view(B, -1, H, hd).transpose(1, 2)
        K = F.linear(kv, a.k_proj.weight, a.k_proj.bias).view(B, -1, H, hd).transpose(1, 2)
        V = F.linear(kv, a.v_proj.weight, a.v_proj.bias).view(B, -1, H, hd).transpose(1, 2)
        if past is not None:
            K, V = torch.cat([past[0], K], 2), torch.cat([past[1], V], 2)
        o = F.scaled_dot_product_attention(Q, K, V).transpose(1, 2).reshape(B, -1, d)
        return F.linear(o, a.output_proj.weight, a.output_proj.bias), (K, V)

    def ln(t, n):
        return F.layer_norm(t, n.normalized_shape, n.weight, n.bias, n.eps)

    h = ln(x, m.attention_layernorm)
    a, kv = mha(m.attention, h, h, past)
    h = a + x
    h = mha(m.cross_attention, ln(h, m.cross_attention_layernorm), enc)[0] + h
    seq = m.feedforward.model
    f = F.linear(F.gelu(F.linear(ln(h, m.feedforward_layernorm), seq[0].weight, seq[0].bias)), seq[-1].weight,
                 seq[-1].bias)
    return h + f, kv


def _family(name):
    n = name.lower()
    for key, fam in (("gemm", "GEMM (projections, MLP)"), ("attn_fwd_decode", "attention decode"),
                     ("attn_decode_combine", "attention decode"), ("attn", "attention general"),
                     ("kv_cache_append", "cache append"), ("layernorm", "add + LayerNorm"), ("ln", "add + LayerNorm"),
                     ("cast", "cast"), ("memcpy", "copies"), ("memset", "copies")):
        if key in n:
            return fam
    return "other"


def decoder_step(min_seconds):
    from multimodal_b200.modules.layers.transformer import TransformerDecoder

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    L, d, H, ff, S_img, Sp = 12, 768, 12, 3072, 256, 76
    dec = TransformerDecoder(L, d, H, ff, activation=torch.nn.GELU, norm_first=True, use_cross_attention=True,
                             dim_kv=d).to(dev).eval()
    rows = []
    for B in (1, 32):
        x = torch.randn(B, 1, d, device=dev)
        img = torch.randn(B, S_img, d, device=dev)
        with torch.no_grad():
            pre = dec(torch.randn(B, Sp, d, device=dev), img,
                      attention_mask=torch.ones(Sp, Sp, dtype=torch.bool, device=dev).tril(), use_cache=True)
            past = pre.current_key_values
            ours = lambda: dec(x, img, past_key_values=past, use_cache=True)

            def ref():
                h = x
                for i, layer in enumerate(dec.layer):
                    h, _ = _ref_layer(layer, h, img, past[i])
                return h

            t_ours = time_fn(ours, min_seconds)
            t_ref = time_fn(ref, min_seconds)
            err = (ours().last_hidden_state - ref()).abs().max().item()
            from torch.profiler import ProfilerActivity, profile

            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(20):
                    ours()
                torch.cuda.synchronize()
        fam = {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = e.cuda_time_total
            if t:
                fam[_family(e.key)] = fam.get(_family(e.key), 0.0) + t / 20.0
        total = sum(fam.values())
        r = dict(B=B, layers=L, d=d, cache=Sp, image_tokens=S_img, ours_ms=t_ours * 1e3, reference_eager_fp32_ms=t_ref * 1e3,
                 max_abs_diff=err, gpu_us_by_family={k: round(v, 1) for k, v in sorted(fam.items(), key=lambda kv: -kv[1])},
                 gpu_us_total=round(total, 1))
        rows.append(r)
        print(f"decoder step B={B}: ours {t_ours * 1e3:.3f} ms, reference eager fp32 {t_ref * 1e3:.3f} ms "
              f"(max |diff| {err:.3e}); GPU time {total:.0f} us: " +
              ", ".join(f"{k} {v:.0f} us ({100 * v / total:.0f} %)" for k, v in r["gpu_us_by_family"].items()),
              flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=0.2)
    ap.add_argument("--json", default=None)
    ap.add_argument("--skip-kernels", action="store_true")
    ap.add_argument("--skip-step", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decode_bench.py needs a CUDA GPU")
    c = card()
    print(f"card: {c}")
    res = {"card": c}
    if not args.skip_kernels:
        res["kernels"] = kernel_table(args.min_seconds)
    if not args.skip_step:
        res["decoder_step"] = decoder_step(args.min_seconds)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
