"""General attention past the shared-memory bound: the streamed kernels behind ops.attention_fwd_generic /
attention_bwd_generic (cross-attention, head_dim 64 / 96 / 128, batch-shared queries, boolean masks), and the modules
that now run at those lengths.

Kernel parity uses the formula and bars of test_gpu_coca_train.py::test_attention_bwd_generic (relative error < 1e-2
for out, dq / dq_f32, dk and dv against fp32 autograd).  Module tests use the bars of the existing CoCa and standalone
layer tests.  The pinned digests are recorded on an H100 by ``python tests/test_gpu_attention_generic_long.py``; the
resident-path digests were recorded with the kernels as they were before the streamed path existed, and must not move.
"""
import hashlib
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _rel(got, ref):
    got, ref = got.float(), ref.float()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-20)).item()


def _streamed(Sq, Skv, D):
    from multimodal_b200 import _lib

    return _lib.lib().mmb_attention_generic_streamed(Sq, Skv, D)


def _fits(Sq, Skv, D):
    """The resident forward's shared-memory formula: Q rows padded to 16, K and V rows to 64, 2*D + 16 bytes each."""
    return (-(-Sq // 16) * 16 + 2 * -(-Skv // 64) * 64) * (2 * D + 16) <= 227 * 1024


def _problem(B, Sq, Skv, H, D, kind, mask_kind=None, causal=False, seed=5):
    """Operands in the layouts the modules use.  kind: 'shared' (pooler queries [Sq, d], bsq = 0), 'cross' (q [B*Sq, d],
    packed kv [B*Skv, 2d]) or 'packed' (self-attention on column slices of a packed [B*S, 3d] buffer)."""
    gen = torch.Generator().manual_seed(seed)
    d = H * D
    bf = torch.bfloat16
    if kind == "packed":
        assert Sq == Skv
        qkv = (torch.randn(B * Sq, 3 * d, generator=gen) * 0.7).to(bf)
        q, k, v = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
        bsq = bsk = bsv = Sq * 3 * d
    else:
        q = (torch.randn((Sq if kind == "shared" else B * Sq), d, generator=gen) * 0.7).to(bf)
        kv = (torch.randn(B * Skv, 2 * d, generator=gen) * 0.7).to(bf)
        k, v = kv[:, :d], kv[:, d:]
        bsq = 0 if kind == "shared" else Sq * d
        bsk = bsv = Skv * 2 * d
    dout = (torch.randn(B * Sq, d, generator=gen) * 0.5).to(bf)
    mask, mask_bs, mask_qs = None, 0, 0
    if mask_kind == "key":
        mask = torch.rand(B, Skv, generator=gen) < 0.8
        mask[:, 0] = True
        mask[0, Skv // 2:] = False          # a long run of masked keys
        mask_bs = Skv
    elif mask_kind == "full":
        mask = torch.rand(B, Sq, Skv, generator=gen) < 0.6
        mask[:, :, 0] = True
        mask[B - 1, 3, :] = False           # a query row that sees no key
        mask_bs, mask_qs = Sq * Skv, Skv
    return dict(B=B, Sq=Sq, Skv=Skv, H=H, D=D, kind=kind, causal=causal, q=q, k=k, v=v, dout=dout, mask=mask,
                bsq=bsq, bsk=bsk, bsv=bsv, mask_bs=mask_bs, mask_qs=mask_qs)


def _run(pb, dev):
    """Forward and backward through ops on `dev`: out, dq (bf16; None for shared queries), dq32, dk, dv."""
    from multimodal_b200 import ops

    B, Sq, H, D = pb["B"], pb["Sq"], pb["H"], pb["D"]
    d = H * D
    q, k, v, dout = (pb[n].to(dev) for n in ("q", "k", "v", "dout"))
    if pb["kind"] == "packed":   # operands and gradients as column slices of one buffer each
        base = torch.cat([q, k, v], 1).contiguous()
        q, k, v = base[:, :d], base[:, d:2 * d], base[:, 2 * d:]
        g = torch.full_like(base, float("nan"))
        dq, dk, dv = g[:, :d], g[:, d:2 * d], g[:, 2 * d:]
    else:
        kvb = torch.cat([k, v], 1).contiguous()
        k, v = kvb[:, :d], kvb[:, d:]
        g = torch.full_like(kvb, float("nan"))
        dk, dv = g[:, :d], g[:, d:]
        dq = None if pb["kind"] == "shared" else torch.full_like(q, float("nan"))
    mu8 = pb["mask"].to(torch.uint8).contiguous().to(dev) if pb["mask"] is not None else None
    kw = dict(B=B, Sq=Sq, Skv=pb["Skv"], H=H, head_dim=D, bsq=pb["bsq"], bsk=pb["bsk"], bsv=pb["bsv"], bso=Sq * d,
              scale=1.0 / math.sqrt(D), mask=mu8, mask_bs=pb["mask_bs"], mask_qs=pb["mask_qs"], causal=pb["causal"])
    out = torch.full((B * Sq, d), float("nan"), device=dev, dtype=torch.bfloat16)
    ops.attention_fwd_generic(q, k, v, out, **kw)
    dq32 = torch.zeros(Sq, d, device=dev) if pb["kind"] == "shared" else None
    ops.attention_bwd_generic(q, k, v, dout.contiguous(), dk, dv, dq=dq, dq_f32=dq32, **kw)
    torch.cuda.synchronize()
    return dict(out=out, dq=dq, dq32=dq32, dk=dk, dv=dv)


def _reference(pb, dev):
    B, Sq, Skv, H, D = pb["B"], pb["Sq"], pb["Skv"], pb["H"], pb["D"]
    qf = pb["q"].float().to(dev).requires_grad_(True)
    kf = pb["k"].float().to(dev).requires_grad_(True)
    vf = pb["v"].float().to(dev).requires_grad_(True)
    qh = (qf.view(1, Sq, H, D).expand(B, Sq, H, D) if pb["kind"] == "shared" else qf.view(B, Sq, H, D)).transpose(1, 2)
    kh, vh = kf.view(B, Skv, H, D).transpose(1, 2), vf.view(B, Skv, H, D).transpose(1, 2)
    s = (qh @ kh.transpose(-1, -2)) / math.sqrt(D)
    if pb["causal"]:
        s = s + torch.full((Sq, Skv), float("-inf"), device=dev).triu(1)
    m = pb["mask"]
    if m is not None:
        m = m.to(dev)
        s = s.masked_fill(~(m[:, None, None, :] if m.dim() == 2 else m[:, None]), float("-inf"))
    p = torch.nan_to_num(torch.softmax(s, -1), nan=0.0)   # a row with no visible key -> zeros (the kernels' convention)
    ref = (p @ vh).transpose(1, 2).reshape(B * Sq, H * D)
    ref.backward(pb["dout"].float().to(dev))
    return ref.detach(), qf.grad, kf.grad, vf.grad


def _check(pb, got, dev):
    ref, gq, gk, gv = _reference(pb, dev)
    assert torch.isfinite(got["out"].float()).all()
    assert _rel(got["out"], ref) < 1e-2
    for t in (got["dk"], got["dv"]):
        assert torch.isfinite(t.float()).all()
    assert _rel(got["dk"], gk) < 1e-2 and _rel(got["dv"], gv) < 1e-2
    if got["dq32"] is not None:
        assert _rel(got["dq32"], gq) < 1e-2
    else:
        assert torch.isfinite(got["dq"].float()).all()
        assert _rel(got["dq"], gq) < 1e-2


KERNEL_CASES = [
    # name, (B, Sq, Skv, H, D, kind, mask_kind, causal)
    ("pooler_256x576_d96", (3, 256, 576, 8, 96, "shared", None, False)),        # CoCa ViT-L/14@336 captioning pooler
    ("single_query_1500_d128", (3, 1, 1500, 2, 128, "shared", None, False)),   # contrastive pooler, one query
    ("parallel_pooler_257x576_d96", (3, 257, 576, 8, 96, "shared", None, False)),
    ("cross_77x1025_keymask_d64", (2, 77, 1025, 2, 64, "cross", "key", False)),
    ("packed_600_mask_causal_d64", (2, 600, 600, 2, 64, "packed", "full", True)),
    ("causal_300x700_d128", (2, 300, 700, 2, 128, "cross", None, True)),
    ("packed_337_d96", (2, 337, 337, 2, 96, "packed", None, False)),
    ("packed_513_d64", (2, 513, 513, 2, 64, "packed", None, False)),
    ("cross_333x705_mask_d96", (2, 333, 705, 2, 96, "cross", "full", False)),
    # batch-shared queries with several batches per dQ CTA (see _dq_chunks): the ring carries over from batch to batch
    # and each chunk's dQ sum is accumulated in scratch; 21 batches make 11 chunks of 2, the last holding one
    ("pooler_21_batches_256x576_d96", (21, 256, 576, 8, 96, "shared", None, False)),
    ("shared_40_batches_200x700_keymask_d64", (40, 200, 700, 4, 64, "shared", "key", False)),
]


def _dq_chunks(B, Sq, H):
    """(batches per chunk, chunks) of the streamed dQ kernel for dq_f32: about 256 CTAs, from the shape alone
    (GS_DQ_TARGET_CTAS in attention_generic_stream.cu)."""
    cta = -(-Sq // 128) * H
    n = min(max(-(-256 // cta), 1), B)
    per = -(-B // n)
    return per, -(-B // per)


def test_shared_query_cases_cover_multi_batch_chunks():
    cases = dict(KERNEL_CASES)
    assert _dq_chunks(*[cases["pooler_21_batches_256x576_d96"][i] for i in (0, 1, 3)]) == (2, 11)   # last chunk: 1
    assert _dq_chunks(*[cases["shared_40_batches_200x700_keymask_d64"][i] for i in (0, 1, 3)])[0] > 1


@pytest.mark.parametrize("name,case", KERNEL_CASES, ids=[c[0] for c in KERNEL_CASES])
def test_streamed_generic_against_fp32_autograd(dev, name, case):
    B, Sq, Skv, H, D, kind, mk, causal = case
    assert _streamed(Sq, Skv, D) == 1
    pb = _problem(B, Sq, Skv, H, D, kind, mk, causal)
    _check(pb, _run(pb, dev), dev)


def _boundary(D):
    S = 16
    while _fits(S + 1, S + 1, D):
        S += 1
    return S


@pytest.mark.parametrize("D", [64, 96, 128])
def test_both_sides_of_the_switch(dev, D):
    S = _boundary(D)
    assert {64: 512, 96: 336, 128: 256}[D] == S
    for s, want in ((S, 0), (S + 1, 1)):
        assert _streamed(s, s, D) == want
        pb = _problem(2, s, s, 2, D, "packed", "key", False, seed=7)
        _check(pb, _run(pb, dev), dev)


def test_exact_zeros_for_masked_keys_and_rows_without_keys(dev):
    pb = _problem(2, 77, 1025, 2, 64, "cross", "key")
    got = _run(pb, dev)
    masked = ~pb["mask"].to(dev).reshape(-1)   # [B * Skv] rows of dk / dv
    assert masked.sum() > 500
    assert got["dk"][masked].abs().max().item() == 0 and got["dv"][masked].abs().max().item() == 0
    pb = _problem(2, 600, 600, 2, 64, "packed", "full", True)
    got = _run(pb, dev)
    row = (pb["B"] - 1) * pb["Sq"] + 3   # no visible key
    assert got["out"][row].abs().max().item() == 0 and got["dq"][row].abs().max().item() == 0
    for t in got.values():
        if t is not None:
            assert not torch.isnan(t.float()).any()


def _digest(t):
    return hashlib.sha256(t.detach().cpu().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()


@pytest.mark.parametrize("name", ["pooler_256x576_d96", "packed_600_mask_causal_d64", "causal_300x700_d128",
                                  "pooler_21_batches_256x576_d96", "shared_40_batches_200x700_keymask_d64"])
def test_streamed_generic_is_run_to_run_deterministic(dev, name):
    case = dict(KERNEL_CASES)[name]
    pb = _problem(*case)
    a, b = _run(pb, dev), _run(pb, dev)
    for k in a:
        if a[k] is not None:
            assert _digest(a[k]) == _digest(b[k]), k


# ---- pinned digests ---------------------------------------------------------------------------------------------
STREAMED_PIN_CASES = ["pooler_256x576_d96", "cross_77x1025_keymask_d64", "packed_600_mask_causal_d64",
                      "causal_300x700_d128", "pooler_21_batches_256x576_d96"]
# sha256 of out | dq or dq_f32 (deterministic on this path) | dk | dv, recorded on an H100 80GB HBM3
PINNED_STREAMED = {
    'pooler_256x576_d96': {
        'out': 'ea97f734d19d112d2a1d3d1d4f01ca50ab064801e537491a972b9bf8e80e9612',
        'dk': 'a29e35ce237360f2af4f3863c4e7c79e057529cd771ff81905eb04c32418d97e',
        'dv': 'f9c1e739f8c7e50ea48e4e6aa477109a68d68bf814edd24193baa7be13168b39',
        'dq32': 'f8d4c7c23fc4fa899aaa4499912b0d3ec6f318d945a18b9e7a0dbea5cbab377e',
    },
    'cross_77x1025_keymask_d64': {
        'out': 'ab63623544a980f97ca080afd20b5fda20cbad69d12d6e5417f96c1233f80e5f',
        'dq': '58dfdb57da8383a0aa1b29f441f0e4920fa9784f53723ecd9596fb54c5944fd7',
        'dk': 'ac089c82bc100a36d121ee74f637b2bf75157ccc1bb3778e2f8b69f926535ddb',
        'dv': '41ef3e04996fbf64e9b387b71ebc4627d80090ab465b9fed7b51c7627e9a56ff',
    },
    'packed_600_mask_causal_d64': {
        'out': 'c7bd90d1552c4241e338ecf9a4bcf84fe9e86e91007ce147387e99f59b61d6ed',
        'dq': 'd8dfd2e569a5c9ef8e7a80f09de36e0a6eababe917807ff723e30704a859d1d4',
        'dk': '507f782f6cb7fdaa16eb723079a737d3e8577bfefc80afcf54d1abd3c0c06f59',
        'dv': '7e973afc9a079ffb10cb74d3274958fb50b19f0931a6c145f921feaf349fdb4c',
    },
    'causal_300x700_d128': {
        'out': '5b2a293fe1e193514836bcbda6c67851dee997cfd8f5a7078c2dc74cdcfb999f',
        'dq': '3965e4e29508d5e2dd9a07b4946bb364ca727b2228d81c64dc3115ff4b791c75',
        'dk': '6ca837be1269a5f89ebbd111ef676d20f94e662c5f6d8421474ed26935e7946f',
        'dv': 'fb7add855add546eaa9d59d9ecba829c19954289176d4c90c892f27c95284eb7',
    },
    'pooler_21_batches_256x576_d96': {
        'out': 'f00b674b4444da3fa0f98fd779c45ea3a1d7879edbb54bef4dcc4452a999c2ce',
        'dk': '3783723e10f815807f128283cc308b71c430b0c9226650c2b54c57cfbb3d505a',
        'dv': 'd1d0a358a9a497112be30082d16ea690e6ee07a6258c9284ab73bcec5bab05b0',
        'dq32': 'f63df30beb0824b9cc90ae94f49ea4f884b5afc83ec7ed77cbc6e7ca2cdf9a51',
    },
}

RESIDENT_PIN_CASES = {
    "pooler_256x256_d96": (3, 256, 256, 8, 96, "shared", None, False),   # ViT-L/14 at 224 px
    "cross_76x256_d64": (2, 76, 256, 2, 64, "cross", "key", False),
    "packed_21_mask_d64": (3, 21, 21, 2, 64, "packed", "full", False),
}
# Recorded with the resident forward and the SIMT backward before the streamed kernels were added: out, dq, dk and dv
# by sha256; dq_f32 of shared queries (fp32 atomics) by its float64 sum and sum of squares
PINNED_RESIDENT = {
    'cross_76x256_d64': {
        'out': '10175e7af582f0d35173433abee6d7d8e125419890a8dcd061a785889573688c',
        'dq': 'a3b85417cc1f0241138578fe9ac80a24ed504b989eca76d89b2f644e9f0df145',
        'dk': '11471bd7d2063c82f5df147716f50c1ec9a4c430cc263a007e796eb8eacfebee',
        'dv': 'c9ba455ad001e70ec6f3239391c76fb0c3c368c8275302da49d9fbc3ecc55486',
    },
    'packed_21_mask_d64': {
        'out': 'd9d02b5456f117fec34dcaee1a3fa0c1d40e68ef679fbefab92cd84c34c323bb',
        'dq': 'b9616bea7f1fcde26d191479ef4adccb9fd99734caf1b0747e9a8acc4b880f77',
        'dk': '4337ef696fbe2147597654b28f976ed38d65c0438a0733d66eeb1904b8bedde1',
        'dv': '6ddd80626135c7a988a50fc4206c683275c3fa5228c32c168de073b4bd7b1291',
    },
    'pooler_256x256_d96': {
        'out': '78035cdd544198be110de28b5748e2c8bf83743eced26a669781eed50f74eb2f',
        'dk': 'f1e4944db1848bffb08d2bba622683ff460deb228de799428425a4c041c35031',
        'dv': '4b1ade2e9961cd7a529de9baa49414b0890447892bb142b26b20b7642584f8ee',
        'dq32': (-12.280703367971, 175.62155078914338),
    },
}


def _summaries(got, streamed=False):
    """sha256 digests; dq_f32 by digest on the streamed path, by its float64 sum and sum of squares on the resident one
    (fp32 atomics)"""
    dig = {k: _digest(got[k]) for k in ("out", "dq", "dk", "dv") if got[k] is not None}
    if got["dq32"] is not None:
        x = got["dq32"].double()
        dig["dq32"] = _digest(got["dq32"]) if streamed else (x.sum().item(), (x * x).sum().item())
    return dig


@pytest.mark.parametrize("name", STREAMED_PIN_CASES)
def test_streamed_generic_pinned(dev, name):
    got = _summaries(_run(_problem(*dict(KERNEL_CASES)[name]), dev), streamed=True)
    want = PINNED_STREAMED[name]
    assert set(got) == set(want)
    for k in want:
        assert got[k] == want[k], k


@pytest.mark.parametrize("name", sorted(RESIDENT_PIN_CASES))
def test_resident_generic_unchanged(dev, name):
    B, Sq, Skv, H, D = RESIDENT_PIN_CASES[name][:5]
    assert _streamed(Sq, Skv, D) == 0
    got = _summaries(_run(_problem(*RESIDENT_PIN_CASES[name]), dev))
    want = PINNED_RESIDENT[name]
    assert set(got) == set(want)
    for k in want:
        if k == "dq32":
            assert got[k] == pytest.approx(want[k], rel=1e-5), k
        else:
            assert got[k] == want[k], k


# ---- modules ----------------------------------------------------------------------------------------------------
def _coca_case(image_size):
    import coca_cases as CC

    c = {k: (dict(v) if isinstance(v, dict) else v) for k, v in CC.CASES["coca_small"].items()}
    c["kwargs"].update(image_size=image_size, vision_include_cls_embed=False)
    return c


def test_coca_576_image_tokens_inference_against_oracle(dev, monkeypatch):
    """coca_small at 96 px (576 image tokens, no CLS): the pooler attends over 576 keys."""
    import coca_cases as CC
    from multimodal_b200.models.coca import coca_for_pretraining
    from oracle import coca_oracle as CO

    monkeypatch.setitem(CC.CASES, "coca_576", _coca_case(96))
    kw = CC.CASES["coca_576"]["kwargs"]
    hd = kw["pooler_output_embed_dim"] // kw["pooler_n_head"]
    assert _streamed(kw["pooler_n_queries"], 576, hd) == 1
    m = CC.build(coca_for_pretraining, "coca_576")
    inp = CC.inputs("coca_576")
    ref = CO.coca_forward(m.state_dict(), kw, inp["images"], inp["texts"])
    m = m.to(dev)
    images, texts = inp["images"].to(dev), inp["texts"].to(dev)
    o = m.model(images, texts)
    assert (o.image_pooled_output.cpu() - ref["image_pooled_output"]).abs().max().item() < 5e-3
    assert (o.text_pooled_output.cpu() - ref["text_pooled_output"]).abs().max().item() < 5e-3
    mm = ref["multimodal_embeddings"]
    assert (o.multimodal_embeddings.cpu() - mm).abs().max().item() / mm.abs().max().item() < 2e-2
    with torch.no_grad():
        losses = m(images, texts)
    assert abs(losses["contrastive"].item() - ref["contrastive"].item()) < 1e-2
    assert abs(losses["captioning"].item() - ref["captioning"].item()) < 1e-2


def test_coca_576_image_tokens_training_gradients_against_oracle(dev, monkeypatch):
    import coca_cases as CC
    import test_gpu_coca_train as G

    monkeypatch.setitem(CC.CASES, "coca_576", _coca_case(96))
    G.coca_grad_parity(dev, "coca_576", "coca s576", with_contrastive=True, bar=4e-2)


# CoCa ViT-L/14 widths at 336 px and reduced depth: 576 image tokens, pooler 256 x 576 at head_dim 96
VIT_L_14_336 = dict(vision_patch_size=14, image_size=336, vision_n_layer=1, vision_n_head=16, vision_dim_feedforward=4096,
                    vision_include_cls_embed=False, vocab_size=49408, num_text_positions=77, text_hidden_dim=768,
                    text_n_layer=1, text_n_head=12, text_dim_feedforward=3072, text_output_dim=768, fusion_n_layer=1,
                    fusion_n_head=12, fusion_dim_feedforward=3072, multimodal_output_projection_dim=49408,
                    pooler_input_embed_dim=1024, pooler_output_embed_dim=768, pooler_n_head=8, pooler_n_queries=256,
                    cascaded_pooler=True)


def test_coca_vit_l_14_336_shapes_against_oracle(dev):
    """The real CoCa ViT-L/14 widths at 336 px (576 image tokens; 256 pooler queries over 576 keys at head_dim 96) at
    reduced depth, at the bars of test_gpu_coca.py::test_coca_vit_l_14_shapes_against_oracle."""
    from multimodal_b200.models.coca import coca_for_pretraining
    from oracle import coca_oracle as CO

    assert _streamed(256, 576, 96) == 1
    kw = dict(VIT_L_14_336)
    torch.manual_seed(0)
    m = coca_for_pretraining(**kw).eval()
    gen = torch.Generator().manual_seed(1)
    images = torch.randn(2, 3, 336, 336, generator=gen)
    texts = torch.randint(1, 49408, (2, 77), generator=gen)
    texts[1, 50:] = 0
    ref = CO.coca_forward(m.state_dict(), kw, images, texts)
    m = m.to(dev)
    o = m.model(images.to(dev), texts.to(dev))
    assert (o.image_pooled_output.cpu() - ref["image_pooled_output"]).abs().max().item() < 5e-3
    assert (o.text_pooled_output.cpu() - ref["text_pooled_output"]).abs().max().item() < 5e-3
    mm = ref["multimodal_embeddings"]
    assert (o.multimodal_embeddings.cpu() - mm).abs().max().item() / mm.abs().max().item() < 2e-2
    with torch.no_grad():
        losses = m(images.to(dev), texts.to(dev))
    assert abs(losses["captioning"].item() - ref["captioning"].item()) < 2e-2


def test_coca_vit_l_14_336_training_gradients_against_oracle(dev, monkeypatch):
    """The same widths under autograd: every parameter gradient, with the contrastive loss, against the fp32 oracle at
    the coca_small bar.  The pooler backward runs 256 queries over 576 keys at head_dim 96 on the streamed kernels."""
    import coca_cases as CC
    import test_gpu_coca_train as G

    monkeypatch.setitem(CC.CASES, "coca_l14_336", dict(kwargs=dict(VIT_L_14_336), batch=2))
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        G.coca_grad_parity(dev, "coca_l14_336", "coca l14@336", with_contrastive=True, bar=4e-2)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def test_transformer_encoder_600_masked_training_gradients(dev):
    """Pre-norm TransformerEncoder with a boolean [B, S, S] mask at S = 600 (head_dim 64), at the bars of
    test_gpu_coca_train.py::standalone_layers_grad_parity."""
    import copy

    import test_gpu_coca_train as G
    from multimodal_b200.modules.layers.transformer import TransformerEncoder

    assert _streamed(600, 600, 64) == 1
    torch.manual_seed(0)
    m = TransformerEncoder(n_layer=2, d_model=128, n_head=2, dim_feedforward=256, activation=torch.nn.GELU,
                           layer_norm_eps=1e-5, norm_first=True, final_layer_norm_eps=1e-5).to(dev)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.05 * torch.randn_like(p))
    ref_m = copy.deepcopy(m)
    B, S = 2, 600
    x = torch.randn(B, S, 128, device=dev)
    mask = torch.rand(B, S, S, device=dev) < 0.7
    mask[:, :, 0] = True
    w = torch.randn(B, S, 128, device=dev) / 11
    xr = x.clone().requires_grad_(True)
    (G._encoder_ref(ref_m, xr, mask) * w).sum().backward()
    xo = x.clone().requires_grad_(True)
    out = m(xo, mask, return_hidden_states=True)
    (out.last_hidden_state * w).sum().backward()
    assert _rel(xo.grad, xr.grad) < 5e-2
    for (k, p), (_, q) in zip(m.named_parameters(), ref_m.named_parameters()):
        assert p.grad is not None, k
        assert _rel(p.grad, q.grad) < 5e-2, (k, _rel(p.grad, q.grad))


def test_mhsa_head_dim_128_s300_masked_forward(dev):
    from multimodal_b200.modules.layers.multi_head_attention import MultiHeadSelfAttention

    assert _streamed(300, 300, 128) == 1
    torch.manual_seed(0)
    m = MultiHeadSelfAttention(256, 2).to(dev)
    B, S, d = 2, 300, 256
    x = torch.randn(B, S, d, device=dev)
    mask = torch.rand(B, S, S, device=dev) < 0.7
    mask[:, :, 0] = True
    with torch.no_grad():
        out = m(x, mask)
        qkv = torch.nn.functional.linear(x, m.input_proj.weight, m.input_proj.bias)
        q, k, v = (t.view(B, S, 2, 128).transpose(1, 2) for t in qkv.chunk(3, -1))
        s = (q @ k.transpose(-1, -2) / math.sqrt(128)).masked_fill(~mask[:, None], float("-inf"))
        a = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B, S, d)
        ref = torch.nn.functional.linear(a, m.output_proj.weight, m.output_proj.bias)
    assert _rel(out, ref) < 2e-2


def record(resident_only=False):
    dev = torch.device("cuda:0")
    print("PINNED_RESIDENT = {")
    for name in sorted(RESIDENT_PIN_CASES):
        print(f"    {name!r}: {_summaries(_run(_problem(*RESIDENT_PIN_CASES[name]), dev))!r},")
    print("}")
    if resident_only:
        return
    print("PINNED_STREAMED = {")
    for name in STREAMED_PIN_CASES:
        got = _summaries(_run(_problem(*dict(KERNEL_CASES)[name]), dev), streamed=True)
        print(f"    {name!r}: {got!r},")
    print("}")


if __name__ == "__main__":
    record(resident_only="--resident" in sys.argv)
