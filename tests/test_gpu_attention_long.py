"""Self-attention beyond S = 384: the streamed kernels behind ops.attention_fwd / attention_bwd (and their key-mask
variants), and the modules that now run at those lengths.

Kernel parity uses the bars of test_gpu_parity.py::test_attention_fwd_bwd against fp32 autograd of the reference
formula: out relative error < 8e-3, lse rtol 1e-4 / atol 2e-4, dqkv relative error < 1e-2.  Module tests compare every
parameter gradient with autograd over the fp32 oracles at the bars of the existing module parity tests.  The pinned
digests are recorded on an H100 by ``python tests/test_gpu_attention_long.py``, as in test_gpu_attention_pinned.py.
"""
import hashlib
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

SCALE = 0.125


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _rel(got, ref):
    got, ref = got.float(), ref.float()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-20)).item()


def _inputs(B, S, H, kmask, gen, dev):
    d = H * 64
    qkv = (torch.randn(B * S, 3 * d, generator=gen) * 0.7).bfloat16().to(dev)
    dout = (torch.randn(B * S, d, generator=gen) * 0.5).bfloat16().to(dev)
    m = None
    if kmask:
        # the construction of test_gpu_attention_pinned.py: random holes, a padded tail per sequence, and one sequence
        # with every key masked (its rows get no key)
        m = (torch.rand(B, S, generator=gen) > 0.2).to(torch.uint8)
        for b in range(B):
            m[b, S - 9 * b:] = 0
        m[B - 1] = 0
        m = m.to(dev)
    return qkv, dout, m


def _run(qkv, dout, m, B, S, H, causal, with_lse=True):
    from multimodal_b200 import ops

    d = H * 64
    dev = qkv.device
    out = torch.empty(B * S, d, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B * H * S, device=dev) if with_lse else None
    dqkv = torch.full_like(qkv, float("nan"))
    if m is not None:
        ops.attention_fwd_kmask(qkv, out, lse, m.view(-1), B, S, H, causal, SCALE)
        if with_lse:
            ops.attention_bwd_kmask(qkv, out, dout, lse, dqkv, m.view(-1), B, S, H, causal, SCALE)
    else:
        ops.attention_fwd(qkv, out, lse, B, S, H, causal, SCALE)
        if with_lse:
            ops.attention_bwd(qkv, out, dout, lse, dqkv, B, S, H, causal, SCALE)
    return out, lse, dqkv


def _scores(qf, m, B, S, H, causal):
    """fp32 scores with masked entries at -inf, plus the [B, 1, S, 1] flag of rows that see at least one key."""
    q, k, v = qf.view(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2) * SCALE
    vis = torch.ones(S, S, dtype=torch.bool, device=qf.device)
    if causal:
        vis = vis.tril()
    vis = vis.expand(B, 1, S, S)
    if m is not None:
        vis = vis & m.bool()[:, None, None, :]
    row_ok = vis.any(-1, keepdim=True)
    # rows with no visible key: any finite scores (their probabilities are zeroed below), so autograd stays finite
    s = s.masked_fill(~vis & row_ok, float("-inf"))
    return s, v, row_ok


def _ref(qf, m, B, S, H, causal):
    s, v, row_ok = _scores(qf, m, B, S, H, causal)
    p = torch.softmax(s, -1) * row_ok
    return (p @ v).transpose(1, 2).reshape(B * S, H * 64)


# (B, S, H, causal, key mask); B * H * ceil(S / 128) exceeds the 132 SMs of an H100 SXM in most cases
KERNEL_CASES = [
    (2, 385, 4, False, False), (3, 385, 2, True, True), (3, 448, 2, True, False), (2, 448, 12, False, True),
    (2, 513, 3, False, True), (4, 577, 16, False, False), (3, 577, 4, True, True), (2, 710, 12, True, True),
    (2, 710, 12, False, False), (1, 1024, 4, True, False), (2, 1024, 2, False, True), (2, 2048, 2, False, False),
    (1, 2048, 3, True, True), (1, 4097, 2, True, False), (1, 4097, 1, False, True),
]


@pytest.mark.parametrize("B,S,H,causal,kmask", KERNEL_CASES,
                         ids=[f"b{c[0]}_s{c[1]}_h{c[2]}{'_causal' if c[3] else ''}{'_kmask' if c[4] else ''}"
                              for c in KERNEL_CASES])
def test_streamed_attention_fwd_bwd(dev, B, S, H, causal, kmask):
    gen = torch.Generator().manual_seed(S * 31 + B * 7 + H + 1000 * causal + 3000 * kmask)
    qkv, dout, m = _inputs(B, S, H, kmask, gen, dev)
    out, lse, dqkv = _run(qkv, dout, m, B, S, H, causal)
    qf = qkv.float().requires_grad_(True)
    ref = _ref(qf, m, B, S, H, causal)
    assert _rel(out, ref) < 8e-3
    with torch.no_grad():
        s, _, row_ok = _scores(qkv.float(), m, B, S, H, causal)
        ref_lse = torch.where(row_ok[..., 0], torch.logsumexp(s, -1), torch.full_like(s[..., 0], float("-inf")))
    lse = lse.view(B, H, S)
    fin = torch.isfinite(ref_lse)
    assert torch.equal(torch.isfinite(lse), fin)
    assert (lse[~fin] == float("-inf")).all()
    torch.testing.assert_close(lse[fin], ref_lse[fin], rtol=1e-4, atol=2e-4)
    ref.backward(dout.float())
    assert torch.isfinite(dqkv.float()).all()
    assert _rel(dqkv, qf.grad) < 1e-2
    if m is not None:
        # rows with no visible key: O = 0; masked keys: exactly zero dK / dV rows
        o = out.float().view(B, S, H, 64)
        assert o[B - 1].abs().max().item() == 0.0
        g = dqkv.float().view(B, S, 3, H * 64)
        assert g[:, :, 1:][~m.bool()].abs().max().item() == 0.0


@pytest.mark.parametrize("S,causal,kmask", [(577, False, False), (1024, True, True)])
def test_streamed_forward_without_lse(dev, S, causal, kmask):
    """Forward-only callers pass lse = None: the same O, bit for bit."""
    B, H = 3, 4
    qkv, dout, m = _inputs(B, S, H, kmask, torch.Generator().manual_seed(5), dev)
    out, _, _ = _run(qkv, dout, m, B, S, H, causal)
    out2, _, _ = _run(qkv, dout, m, B, S, H, causal, with_lse=False)
    assert torch.equal(out, out2)


@pytest.mark.parametrize("S,causal,kmask", [(577, False, False), (710, True, True), (2048, False, True)])
def test_streamed_attention_is_run_to_run_deterministic(dev, S, causal, kmask):
    B, H = 4, 12
    qkv, dout, m = _inputs(B, S, H, kmask, torch.Generator().manual_seed(7), dev)
    a = _run(qkv, dout, m, B, S, H, causal)
    b = _run(qkv, dout, m, B, S, H, causal)
    torch.cuda.synchronize(dev)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8))


def test_bwd_launch_count():
    from multimodal_b200 import _lib

    lib = _lib.lib()
    assert lib.mmb_attention_bwd_launches(197) == 1 and lib.mmb_attention_bwd_launches(384) == 1
    assert lib.mmb_attention_bwd_launches(385) == 2 and lib.mmb_attention_bwd_launches(4097) == 2


# ---- pinned digests ---------------------------------------------------------------------------------------------
# (name, B, S, H, causal, key mask)
PIN_CASES = [
    ("s385", 3, 385, 4, False, False),
    ("s577", 2, 577, 16, False, False),
    ("s710_causal_kmask", 3, 710, 12, True, True),
    ("s1024_kmask", 2, 1024, 4, False, True),
    ("s4097_causal", 1, 4097, 2, True, False),
]

# sha256 of (out, lse, dqkv), recorded on an H100 80GB HBM3
PINNED = {
    's385': ('4b2bc3ef332a9b36705acda8c20244c8dda102ec490344d55f16f4bcd036e4bc', '6265ac96ea7b378366c3b7b7408a8e4fe39c8901b763be0abb202c854557a4e2', 'f4aba1a7fe3630f7684bb2f2e3bb0a0d3a38a19a204f994790987df8e0b15f58'),
    's577': ('a036cd389041047eeef97f2decf5dd8d0e23f923264ed3088e29aac382cb7641', 'c4b1b61c3d54a18cad5e76bf63413a1ccd54c817fcda6503c01eeb69ee7c073f', '3b811371cd20faa29e4d6e0a45d1a7dbf2c78d2fecd875047fe38cf40c581592'),
    's710_causal_kmask': ('eb9d8ef21fabcc70967193450734d983899d7a1e370efff5ac032f981811ab2a', '1eb4da2d597d009c4bc7cb754ba3044edc83069fb7cf546d93c2e9c40524d61f', '7bd0645821c924e2cd592a7f0257cf9f994a4c1b03af288d8a62bf9409028024'),
    's1024_kmask': ('78d4a08e05e54aa9281dfb90372c6c52d1eaf657fd8aa9290f5be3abf175a843', 'a173cafeb27f91ffbe14ffcc58a417f12f0410378b697b84cdf41a168c84e194', 'eb45e7f744d3bf659f7e9239953a0b1281b7bee92582a95d57bc1cc87ffe1054'),
    's4097_causal': ('f40bc48f3908b383337d7e619badc619d0a5ee635cf37bf7e566bd6a015ed53a', '9921cddf7ee837f490d7e7ac7d3472247a2c3c426d1ca1709a1c73aaadc795eb', 'cb02305a3d127b387ae04b33a8d28eb6c02669ab177574210411d39d3320270c'),
}


def _digest(t):
    return hashlib.sha256(t.detach().cpu().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()


def _pin_run(name, B, S, H, causal, kmask, dev):
    gen = torch.Generator().manual_seed(sum(map(ord, name)))
    qkv, dout, m = _inputs(B, S, H, kmask, gen, dev)
    res = _run(qkv, dout, m, B, S, H, causal)
    torch.cuda.synchronize(dev)
    return tuple(_digest(t) for t in res)


@pytest.mark.parametrize("case", PIN_CASES, ids=[c[0] for c in PIN_CASES])
def test_streamed_attention_bit_identical(dev, case):
    got = _pin_run(*case, dev)
    want = PINNED[case[0]]
    for what, a, b in zip(("out", "lse", "dqkv"), got, want):
        assert a == b, f"{case[0]}: {what} changed"


# ---- interop ----------------------------------------------------------------------------------------------------
def test_attention_probs_from_streamed_lse(dev):
    """FLAVA's output_attentions path: probabilities recomputed from QKV and the streamed forward's row LSE."""
    from multimodal_b200 import ops

    B, S, H = 3, 512, 2
    qkv, dout, m = _inputs(B, S, H, True, torch.Generator().manual_seed(11), dev)
    out, lse, _ = _run(qkv, dout, m, B, S, H, False)
    probs = torch.empty(B, H, S, S, device=dev)
    ops.attention_probs(qkv, lse, m.view(-1), probs, B, S, H, False, SCALE)
    s, _, row_ok = _scores(qkv.float(), m, B, S, H, False)
    ref = torch.softmax(s, -1) * row_ok
    torch.testing.assert_close(probs[:B - 1], ref[:B - 1], rtol=2e-3, atol=2e-5)
    assert probs[B - 1].abs().max().item() == 0.0        # the sequence with every key masked
    assert probs.masked_select(~m.bool()[:, None, None, :].expand_as(probs)).abs().max().item() == 0.0


# ---- modules ----------------------------------------------------------------------------------------------------
def _grad_report(mod, sd, bar, tag, skip=()):
    rows = []
    for k, p in mod.named_parameters():
        ref = sd[k].grad
        assert p.grad is not None and torch.isfinite(p.grad).all(), k
        if any(k.endswith(s) for s in skip):
            continue
        cos = torch.nn.functional.cosine_similarity(p.grad.flatten().float(), ref.flatten().float().to(p.device),
                                                    dim=0).item()
        rel = ((p.grad.float() - ref.float().to(p.device)).norm() / ref.float().norm().clamp_min(1e-30)).item()
        rows.append((k, rel, cos))
    print(f"{tag}: " + ", ".join(f"{k} {a:.2e}" for k, a, _ in sorted(rows, key=lambda r: -r[1])[:5]))
    assert len(rows) > 5
    for k, a, c in rows:
        assert a < bar and c > 0.995, (k, a, c)


def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def test_clip_vit_336_s577_gradients_against_fp32_oracle(dev):
    """CLIPViTEncoder in the ViT-L/14@336 layout (577 tokens) at reduced width and depth."""
    from multimodal_b200.models.clip.image_encoder import CLIPViTEncoder
    from oracle import clip_oracle as O

    _no_tf32()
    torch.manual_seed(0)
    m = CLIPViTEncoder(embedding_dim=128, patch_size=14, image_size=336, width=256, heads=4, layers=2).to(dev).train()
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    img = torch.randn(3, 3, 336, 336, generator=torch.Generator().manual_seed(1)).to(dev)
    ref = O.vit_encoder(img, sd, "", 4)
    w = torch.randn(ref.shape, generator=torch.Generator().manual_seed(2)).to(dev)
    (w * ref).sum().backward()
    out = m(img)
    assert _rel(out, ref.detach()) < 2e-2
    (w * out).sum().backward()
    _grad_report(m, sd, 3e-2, "clip vit s577", skip=("in_proj_bias",))


def test_clip_text_512_causal_gradients_against_fp32_oracle(dev):
    from multimodal_b200.models.clip.text_encoder import CLIPTextEncoder
    from oracle import clip_oracle as O

    _no_tf32()
    torch.manual_seed(0)
    m = CLIPTextEncoder(embedding_dim=128, context_length=512, vocab_size=1000, width=256, dim_feedforward=1024,
                        heads=4, layers=2).to(dev).train()
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    gen = torch.Generator().manual_seed(3)
    text = torch.randint(1, 998, (3, 512), generator=gen)
    text[0, 300] = 999      # EOT: the largest id
    text[1, 511] = 999
    text[2, 17] = 999
    text = text.to(dev)
    ref = O.text_encoder(text, sd, "", 4)
    w = torch.randn(ref.shape, generator=torch.Generator().manual_seed(4)).to(dev)
    (w * ref).sum().backward()
    out = m(text)
    assert _rel(out, ref.detach()) < 2e-2
    (w * out).sum().backward()
    _grad_report(m, sd, 3e-2, "clip text s512", skip=("in_proj_bias",))


# FLAVA with BERT-length text: text S = 512 with right padding, multimodal S = 1 + 17 + 512 = 530
FLAVA_LONG = dict(
    kwargs=dict(image_hidden_size=128, image_num_attention_heads=2, image_num_hidden_layers=1,
                image_intermediate_size=256, image_size=32, patch_size=8,
                text_hidden_size=128, text_num_attention_heads=2, text_num_hidden_layers=1,
                text_intermediate_size=256, vocab_size=100, max_position_embeddings=512,
                multimodal_hidden_size=128, multimodal_num_attention_heads=2, multimodal_num_hidden_layers=1,
                multimodal_intermediate_size=256, text_and_image_proj_size=64),
    batch=3, text_len=512)


def flava_long_model():
    from multimodal_b200.models.flava import flava_model

    torch.manual_seed(0)
    m = flava_model(**FLAVA_LONG["kwargs"])
    g = torch.Generator().manual_seed(11)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.05 * torch.randn(p.shape, generator=g))
    return m.eval()


def flava_long_inputs():
    kw, B, St = FLAVA_LONG["kwargs"], FLAVA_LONG["batch"], FLAVA_LONG["text_len"]
    g = torch.Generator().manual_seed(5)
    image = torch.randn(B, 3, kw["image_size"], kw["image_size"], generator=g)
    text = torch.randint(1, kw["vocab_size"], (B, St), generator=g)
    text[1, 300:] = 0       # right padding (pad_token_id = 0); row 0 keeps all 512 tokens
    text[2, 7:] = 0
    text_masked = text.clone()
    text_masked[:, 2] = kw["vocab_size"] - 1
    patches_mask = torch.rand(B, (kw["image_size"] // kw["patch_size"]) ** 2, generator=g) < 0.4
    return dict(image=image, text=text, text_masked=text_masked, image_patches_mask=patches_mask)


def test_flava_text_512_and_multimodal_530_gradients_against_fp32_oracle(dev):
    import test_gpu_flava_train as G

    _no_tf32()
    G._grad_parity(dev, flava_long_model(), G._cfg(FLAVA_LONG["kwargs"]), flava_long_inputs(), "flava s512/s530", 3e-2)


def test_flava_text_512_inference_matches_training_forward(dev):
    m = flava_long_model().to(dev)
    inp = {k: v.to(dev) for k, v in flava_long_inputs().items()}
    with torch.no_grad():
        o = m(image=inp["image"], text=inp["text"], skip_unmasked_mm_encoder=False)
    assert o.text.last_hidden_state.shape[1] == 512 and o.multimodal.last_hidden_state.shape[1] == 530
    m.train()
    o2 = m(image=inp["image"], text=inp["text"], skip_unmasked_mm_encoder=False)
    for a, b in ((o.text, o2.text), (o.multimodal, o2.multimodal)):
        assert torch.isfinite(a.last_hidden_state).all()
        assert _rel(a.last_hidden_state, b.last_hidden_state.detach()) < 1e-2


def _coca_case(image_size):
    import coca_cases as CC

    c = {k: (dict(v) if isinstance(v, dict) else v) for k, v in CC.CASES["coca_small"].items()}
    c["kwargs"].update(image_size=image_size, vision_include_cls_embed=False)
    return c


def test_coca_training_400_image_tokens_gradients_against_fp32_oracle(dev, monkeypatch):
    """CoCa vision tower at 400 tokens (80 px, patch 4, no CLS): the training runtime's TransformerStack."""
    import coca_cases as CC
    import test_gpu_coca_train as G

    monkeypatch.setitem(CC.CASES, "coca_long", _coca_case(80))
    _no_tf32()
    G.coca_grad_parity(dev, "coca_long", "coca s400", with_contrastive=False, bar=4e-2)


def test_coca_vision_encoder_inference_576_tokens_against_oracle(dev):
    """CoCa vision tower at 576 tokens (96 px, patch 4, no CLS; the 336-px ViT-L/14 count), inference runtime: past
    the generic forward's shared-memory bound, so the streamed kernel serves its self-attention.  (The attention
    pooler's cross-attention over 576 keys at head_dim 96 stays on the generic kernel, whose bound is unchanged.)"""
    import coca_cases as CC
    from multimodal_b200.models.coca import coca_for_pretraining
    from oracle import coca_oracle as CO

    case = _coca_case(96)
    torch.manual_seed(0)
    m = coca_for_pretraining(**case["kwargs"])
    g = torch.Generator().manual_seed(13)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.03 * torch.randn(p.shape, generator=g))
    m = m.eval()
    images = torch.randn(3, 3, 96, 96, generator=torch.Generator().manual_seed(6))
    sd = {k: v.detach().float() for k, v in m.state_dict().items()}
    ref = CO.vision_encoder(images, sd, dict(case["kwargs"]))
    m = m.to(dev)
    with torch.no_grad():
        o = m.model.vision_encoder(images.to(dev))
    assert o.last_hidden_state.shape == (3, 576, case["kwargs"]["pooler_input_embed_dim"])
    assert _rel(o.last_hidden_state.cpu(), ref) < 2e-2
    assert CC.CASES["coca_small"]["kwargs"]["image_size"] == 32   # the shared case is untouched


def record():
    dev = torch.device("cuda:0")
    print("PINNED = {")
    for case in PIN_CASES:
        print(f"    {case[0]!r}: {_pin_run(*case, dev)!r},")
    print("}")


if __name__ == "__main__":
    record()
