"""Pins the CLIP, FLAVA and CoCa module forwards and the standalone pre-norm encoder layers bit for bit, under
torch.no_grad() and with grad mode on.

Every tensor the inference forwards return is hashed: hidden states, pooler outputs, projected embeddings, attention
probabilities, multimodal logits, both CoCa losses and the CLIP towers' embeddings and text hidden state.  With grad
mode on, the forwards run the training path, which also returns the losses, last hidden states and CLIP embeddings
pinned here (gradients are not: some backward kernels use fp32 atomics).
The digests were recorded on an H100 80GB HBM3 by ``python tests/test_gpu_runtime_pinned.py``, which prints the table
below.  Every shape stays outside 385-512 tokens of unmasked head_dim-64 self-attention, the band where the inference
and training paths once chose different attention kernels.
"""
import hashlib
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import coca_cases as CC  # noqa: E402
import flava_cases as FC  # noqa: E402

pytestmark = pytest.mark.gpu


def _digest(t: torch.Tensor) -> str:
    t = t.detach().contiguous().reshape(-1)
    return hashlib.sha256(t.cpu().view(torch.uint8).numpy().tobytes()).hexdigest()


def _flava(name):
    from multimodal_b200.models.flava import flava_model

    return FC.build(flava_model, name), FC.inputs(name)


def _flava_512():
    from test_gpu_attention_long import flava_long_inputs, flava_long_model

    return flava_long_model(), flava_long_inputs()


def _flava_outputs(m, inp, dev, attentions=False):
    inp = {k: v.to(dev) for k, v in inp.items()}
    if attentions:
        m.set_output_attentions(True)
        o = m(image=inp["image"], text=inp["text"], skip_unmasked_mm_encoder=False)
    else:
        o = m(image=inp["image"], text=inp["text"], image_patches_mask=inp["image_patches_mask"],
              text_masked=inp["text_masked"], skip_unmasked_mm_encoder=False)
    res = FC.flatten_output(o)
    if attentions:
        for part in ("image", "text", "multimodal"):
            for i, a in enumerate(getattr(o, part).attentions):
                res[f"{part}.attentions.{i}"] = a
    return res


def _coca(name):
    from multimodal_b200.models.coca import coca_for_pretraining

    inp = CC.inputs(name)
    return CC.build(coca_for_pretraining, name), inp["images"], inp["texts"]


def _coca_l14():
    """The CoCa ViT-L/14 layer shapes of test_gpu_coca.test_coca_vit_l_14_shapes_against_oracle."""
    from multimodal_b200.models.coca import coca_for_pretraining

    kw = dict(vision_patch_size=14, vision_n_layer=2, vision_n_head=16, vision_dim_feedforward=4096,
              vision_include_cls_embed=False, vocab_size=49408, num_text_positions=77, text_hidden_dim=768,
              text_n_layer=1, text_n_head=12, text_dim_feedforward=3072, text_output_dim=768, fusion_n_layer=1,
              fusion_n_head=12, fusion_dim_feedforward=3072, multimodal_output_projection_dim=49408,
              pooler_input_embed_dim=1024, pooler_output_embed_dim=768, pooler_n_head=8, cascaded_pooler=True)
    torch.manual_seed(0)
    m = coca_for_pretraining(**kw).eval()
    gen = torch.Generator().manual_seed(1)
    images = torch.randn(2, 3, 224, 224, generator=gen)
    texts = torch.randint(1, 49408, (2, 77), generator=gen)
    texts[1, 50:] = 0
    return m, images, texts


def _coca_inference(m, images, texts, dev):
    images, texts = images.to(dev), texts.to(dev)
    with torch.no_grad():
        o = m.model(images, texts)
        losses = m(images, texts)
        v = m.model.vision_encoder(images)
    res = {f"model.{k}": t for k, t in o._asdict().items() if t is not None}
    res.update({f"loss.{k}": t for k, t in losses.items()})
    res["vision.last_hidden_state"] = v.last_hidden_state
    res.update({f"vision.hidden_states.{i}": h for i, h in enumerate(v.hidden_states)})
    return res


def _coca_grad(m, images, texts, dev):
    images, texts = images.to(dev), texts.to(dev)
    with torch.enable_grad():
        losses = m(images, texts)
        v = m.model.vision_encoder(images)
    assert losses["captioning"].requires_grad and v.last_hidden_state.requires_grad
    res = {f"loss.{k}": t for k, t in losses.items()}
    res["vision.last_hidden_state"] = v.last_hidden_state
    return res


def _text_decoder_no_cls():
    """CoCaTextDecoder(embed_cls=False) with a biased text_projection: inference-only configurations."""
    from multimodal_b200.models.coca.text_decoder import CoCaTextDecoder

    torch.manual_seed(0)
    m = CoCaTextDecoder(vocab_size=300, num_positions=20, embedding_dim=128, n_layer=2, n_head=2, dim_feedforward=256,
                        output_dim=96, embed_cls=False)
    m.text_projection = torch.nn.Linear(128, 96, bias=True)
    g = torch.Generator().manual_seed(17)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.03 * torch.randn(p.shape, generator=g))
    ids = torch.randint(1, 300, (3, 20), generator=g)
    ids[1, 12:] = 0
    return m.eval(), ids


def _head_dim_modules(hd):
    """A VisionTransformer and a CoCaTextDecoder with heads of head_dim `hd` (the general attention kernels) and a width
    that is a multiple of 128 (the LayerNorm kernels)."""
    from multimodal_b200.models.coca.text_decoder import CoCaTextDecoder
    from multimodal_b200.modules.encoders.vision_transformer import vision_transformer

    heads = 4 if hd == 96 else 2
    d = heads * hd
    torch.manual_seed(0)
    vit = vision_transformer(patch_size=8, hidden_dim=d, dim_feedforward=2 * d, n_layer=2, n_head=heads, image_size=32)
    txt = CoCaTextDecoder(vocab_size=300, num_positions=13, embedding_dim=d, n_layer=2, n_head=heads,
                          dim_feedforward=2 * d, output_dim=96)
    g = torch.Generator().manual_seed(19)
    with torch.no_grad():
        for p in list(vit.parameters()) + list(txt.parameters()):
            p.add_(0.03 * torch.randn(p.shape, generator=g))
    images = torch.randn(3, 3, 32, 32, generator=g)
    ids = torch.randint(1, 300, (3, 12), generator=g)
    ids[1, 7:] = 0
    return vit.eval(), txt.eval(), images, ids


def _vit_drop():
    """VisionTransformer with patch dropping and stochastic depth, left in train() mode."""
    from multimodal_b200.modules.encoders.vision_transformer import vision_transformer

    torch.manual_seed(0)
    vit = vision_transformer(patch_size=4, hidden_dim=128, dim_feedforward=256, n_layer=3, n_head=2, image_size=32,
                             patch_drop_rate=0.25, drop_path_rate=0.5)
    g = torch.Generator().manual_seed(23)
    with torch.no_grad():
        for p in vit.parameters():
            p.add_(0.03 * torch.randn(p.shape, generator=g))
    return vit.train(), torch.randn(4, 3, 32, 32, generator=g)


def _clip_small():
    """A width-128, 2-layer CLIP (head_dim 64) with perturbed weights, and a batch of 6 image / text pairs."""
    from multimodal_b200.models.clip.image_encoder import CLIPViTEncoder
    from multimodal_b200.models.clip.model import CLIP
    from multimodal_b200.models.clip.text_encoder import CLIPTextEncoder

    torch.manual_seed(0)
    m = CLIP(CLIPViTEncoder(64, 16, 64, 128, 2, 2),
             CLIPTextEncoder(embedding_dim=64, vocab_size=512, width=128, dim_feedforward=512, heads=2, layers=2))
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.03 * torch.randn(p.shape, generator=g))
    B = 6
    image = torch.randn(B, 3, 64, 64, generator=g)
    text = torch.randint(1, 500, (B, 77), generator=g)
    text[torch.arange(B), torch.randint(5, 77, (B,), generator=g)] = 511          # EOT = the largest id
    return m.train(), image, text


def _standalone(kind, drop=False):
    """A standalone pre-norm TransformerEncoder (3 layers, final LayerNorm) or TransformerEncoderLayer at width 128
    (head_dim 64) with perturbed weights, an input batch and a [B, S, S] bool mask; with `drop`, drop_path_rate 0.5."""
    from multimodal_b200.modules.layers.transformer import TransformerEncoder, TransformerEncoderLayer

    torch.manual_seed(0)
    rate = 0.5 if drop else None
    if kind == "layer":
        m = TransformerEncoderLayer(128, 2, 256, activation=torch.nn.GELU, layer_norm_eps=1e-5, norm_first=True,
                                    drop_path_rate=rate)
    else:
        m = TransformerEncoder(3, 128, 2, 256, activation=torch.nn.GELU, layer_norm_eps=1e-5, norm_first=True,
                               final_layer_norm_eps=1e-5, drop_path_rate=rate)
    g = torch.Generator().manual_seed(31)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.03 * torch.randn(p.shape, generator=g))
    x = torch.randn(4, 20, 128, generator=g)
    mask = torch.rand(4, 20, 20, generator=g) < 0.7
    mask[:, :, 0] = True
    return (m.train() if drop else m.eval()), x, mask


def _standalone_outputs(m, x, mask, dev):
    """Output and hidden states of one standalone call (the encoder with `return_hidden_states`)."""
    x, mask = x.to(dev), (mask.to(dev) if mask is not None else None)
    if not hasattr(m, "layer"):
        return {"output": m(x, mask)}
    o = m(x, mask, return_hidden_states=True)
    return {"last_hidden_state": o.last_hidden_state, **{f"hidden_states.{i}": h for i, h in enumerate(o.hidden_states)}}


def _clip_outputs(m, image, text, dev):
    """The embeddings of both CLIP towers."""
    return {"image.embeddings": m.encoder_a(image.to(dev)), "text.embeddings": m.encoder_b(text.to(dev))}


def _case(name, dev):
    """{output name: tensor} of one pinned forward."""
    if name.startswith("clip_small"):
        m, image, text = _clip_small()
        m = m.to(dev)
        if name.endswith("infer"):
            with torch.no_grad():
                res = _clip_outputs(m, image, text, dev)
                res["text.hidden_state"] = m.encoder_b(text.to(dev), return_hidden_state=True)
            return res
        with torch.enable_grad():
            res = _clip_outputs(m, image, text, dev)
        assert all(t.requires_grad for t in res.values())
        return res
    if name in ("coca_hd96.infer", "coca_hd128.infer"):
        vit, txt, images, ids = _head_dim_modules(96 if name == "coca_hd96.infer" else 128)
        with torch.no_grad():
            v = vit.to(dev)(images.to(dev))
            pooled, tokens = txt.to(dev)(ids.to(dev))
        res = {"vision.last_hidden_state": v.last_hidden_state, "text.pooled": pooled, "text.tokens": tokens}
        res.update({f"vision.hidden_states.{i}": h for i, h in enumerate(v.hidden_states)})
        return res
    if name == "vit_drop.infer":
        vit, images = _vit_drop()
        vit, images = vit.to(dev), images.to(dev)
        torch.manual_seed(29)
        with torch.no_grad():
            v = vit(images)
        return {"last_hidden_state": v.last_hidden_state,
                **{f"hidden_states.{i}": h for i, h in enumerate(v.hidden_states)}}
    if name.startswith("flava_small") or name.startswith("flava_long"):
        base, mode = name.rsplit(".", 1)
        m, inp = _flava(base)
        m = m.to(dev)
        if mode == "infer":
            with torch.no_grad():
                return _flava_outputs(m, inp, dev)
        with torch.enable_grad():
            out = _flava_outputs(m, inp, dev)
        return {k: v for k, v in out.items() if k.endswith("last_hidden_state")}
    if name == "flava_attentions.infer":
        m, inp = _flava("flava_small")
        with torch.no_grad():
            return _flava_outputs(m.to(dev), inp, dev, attentions=True)
    if name.startswith("flava_text512"):
        m, inp = _flava_512()
        m = m.to(dev)
        inp = {k: v.to(dev) for k, v in inp.items()}
        grad = name.endswith("grad")
        with torch.set_grad_enabled(grad):
            o = m(image=inp["image"], text=inp["text"], skip_unmasked_mm_encoder=False)
        res = FC.flatten_output(o)
        return {k: v for k, v in res.items() if k.endswith("last_hidden_state")} if grad else res
    if name.startswith("coca_"):
        base, mode = name.rsplit(".", 1)
        m, images, texts = _coca_l14() if base == "coca_l14" else _coca(base)
        m = m.to(dev)
        return (_coca_inference if mode == "infer" else _coca_grad)(m, images, texts, dev)
    if name.startswith("standalone_"):
        base, mode = name.rsplit(".", 1)
        m, x, mask = _standalone("layer" if base == "standalone_layer" else "encoder", drop=base == "standalone_drop")
        m = m.to(dev)
        if base != "standalone_encoder":
            mask = None     # the fused attention kernels
        torch.manual_seed(37)
        with torch.set_grad_enabled(mode == "grad"):
            res = _standalone_outputs(m, x, mask, dev)
        assert res.get("output", res.get("last_hidden_state")).requires_grad == (mode == "grad")
        return res
    if name == "text_decoder_no_cls.infer":
        m, ids = _text_decoder_no_cls()
        m = m.to(dev)
        with torch.no_grad():
            pooled, tokens = m(ids.to(dev))
        return {"pooled": pooled, "tokens": tokens}
    raise KeyError(name)


CASES = ["flava_small.infer", "flava_small.grad", "flava_long.infer", "flava_long.grad", "flava_attentions.infer",
         "flava_text512.infer", "flava_text512.grad", "coca_small.infer", "coca_small.grad", "coca_parallel.infer",
         "coca_parallel.grad", "coca_l14.infer", "coca_l14.grad", "text_decoder_no_cls.infer", "coca_hd96.infer",
         "coca_hd128.infer", "vit_drop.infer", "clip_small.infer", "clip_small.grad", "standalone_encoder.infer",
         "standalone_encoder.grad", "standalone_drop.infer", "standalone_layer.infer"]

# {case: {output: sha256 of its bytes}}, recorded on an H100 80GB HBM3
PINNED = {
    'flava_small.infer': {
        'image.hidden_states.0': '(3, 17, 128) torch.float32 9a8804e0a85df39dc8d23a76487e71b1ef8b00551b4c41b2adc7ea1f6ced64e5',
        'image.hidden_states.1': '(3, 17, 128) torch.float32 db2960578a25632938fb221fc9702322851eb83aa6002bc9eac5cc237c701dc3',
        'image.hidden_states.2': '(3, 17, 128) torch.float32 1a6250ee902fbc5fdb507771d73c36560297be6666e2f343d0080e0670daeb00',
        'image.last_hidden_state': '(3, 17, 128) torch.float32 a391b610fdba22fdc90bfd865a3b8a73e2dd90c3a9d642f1090b1e73bd580e4f',
        'image.pooler_output': '(3, 128) torch.float32 a56599156b548fdbbc0ff3cd85018a20b1ef2ed529a94e11b6af89e1baefe828',
        'image_masked.hidden_states.0': '(3, 17, 128) torch.float32 e8a2906f439663b4c236c1587ab239de2ce0e7acfb4d67d1c68388eb642b87eb',
        'image_masked.hidden_states.1': '(3, 17, 128) torch.float32 88e02ce45d4306c3aa57083f4676d0311c6dcd638eac26cb70d59b126ae8098e',
        'image_masked.hidden_states.2': '(3, 17, 128) torch.float32 da6a007f439f7087dd2f2311c6e4322a3c6d10dc1aa5624a8ac8422ab3662513',
        'image_masked.last_hidden_state': '(3, 17, 128) torch.float32 cb6016687260e4895ee9c5aadf48f4f90b3fd8116088e21270a8c63adfe403a5',
        'image_masked.pooler_output': '(3, 128) torch.float32 b26ab48da8fbd4b4ce7c7c65ff6d3036d228ab09e942255b9a2d8acfb23ffad4',
        'multimodal.hidden_states.0': '(3, 30, 256) torch.float32 3454bc63cae8255cf286b0e5c08b90090cf0ca70592036fb53233f3d793aa5b0',
        'multimodal.hidden_states.1': '(3, 30, 256) torch.float32 d398f2a4f616aec4da4a81f66b8d5c12ab22d751ab421cb0de8f83781bf8091b',
        'multimodal.last_hidden_state': '(3, 30, 256) torch.float32 4dfcbb2e2aa9dce5854523a06ae40eacc633cd4ae680ccb8771558e6a8c38e35',
        'multimodal.pooler_output': '(3, 256) torch.float32 12f1b33441b8a226ca1180590f58a37752268fb42e293ab2d05ff220477cedf3',
        'multimodal_masked.hidden_states.0': '(3, 30, 256) torch.float32 6dba701fc674a06bef323e58beeaed7b6dfbb2d6d98c315e314613c88de5c155',
        'multimodal_masked.hidden_states.1': '(3, 30, 256) torch.float32 d0801911a8264587e3db8625cdd8f8a0ac11e45dd099c0e5dbf25c80df2b4a2f',
        'multimodal_masked.last_hidden_state': '(3, 30, 256) torch.float32 d285b26ec5766bab226b3e40e8d5004a073af48cd943660cdd3709336f848372',
        'multimodal_masked.pooler_output': '(3, 256) torch.float32 9793415b0645237a820815186c7290c3db413dab753adb6f2f425b5aa332e5b5',
        'projected_image_embeddings': '(3, 64) torch.float32 3077ef64d7930996f491e1826dd9e5fb566ce704f61e29da7f6cab84bbe6e483',
        'projected_text_embeddings': '(3, 64) torch.float32 b934b9682c42092f7880071367d34e2c69c926ccc886996c56600dc9ccd6f265',
        'text.hidden_states.0': '(3, 12, 128) torch.float32 8106e4cf6822bf1ca1bdce8c08bac4a96570e7c3864a2fae265a0b37f65c19aa',
        'text.hidden_states.1': '(3, 12, 128) torch.float32 c7ab0466d7644e0f38f6d4adb9468fa4f4c7dcce42169093ee803b584a1f181f',
        'text.hidden_states.2': '(3, 12, 128) torch.float32 c97c2910a4fdc515fbe40adf48ce78098780c8823c7a38279f33296e23a6428b',
        'text.last_hidden_state': '(3, 12, 128) torch.float32 a21928553894012a27b4fca1fab28700b2e4337ad6298fb3d09b6bd517038512',
        'text.pooler_output': '(3, 128) torch.float32 d4aefd87972beaf44cd62684e71e52f89fe411f73304bcd249f02586902ebc01',
        'text_masked.hidden_states.0': '(3, 12, 128) torch.float32 3a5443c92c0ec5a3fc4553c57ae0eae87732e03b1578577c75117a2040537d47',
        'text_masked.hidden_states.1': '(3, 12, 128) torch.float32 3308aeaa9f89e19fd6934fc32cad5d126b006cbd4049eb76e6508ecb6506281a',
        'text_masked.hidden_states.2': '(3, 12, 128) torch.float32 2609ae89002b1d078176b817c55c09a589708fba7abbd7faf8392124419794de',
        'text_masked.last_hidden_state': '(3, 12, 128) torch.float32 d2d01cdb800a417ea975e12dd2e74ab31f27436d2a5aac81fb6b358f2ebdacf7',
        'text_masked.pooler_output': '(3, 128) torch.float32 817e3f8ed13f8e2e1d18c57a7c4175c80ca3a16f5af21913edd27103345faf02',
    },
    'flava_small.grad': {
        'image.last_hidden_state': '(3, 17, 128) torch.float32 a391b610fdba22fdc90bfd865a3b8a73e2dd90c3a9d642f1090b1e73bd580e4f',
        'image_masked.last_hidden_state': '(3, 17, 128) torch.float32 cb6016687260e4895ee9c5aadf48f4f90b3fd8116088e21270a8c63adfe403a5',
        'multimodal.last_hidden_state': '(3, 30, 256) torch.float32 4dfcbb2e2aa9dce5854523a06ae40eacc633cd4ae680ccb8771558e6a8c38e35',
        'multimodal_masked.last_hidden_state': '(3, 30, 256) torch.float32 d285b26ec5766bab226b3e40e8d5004a073af48cd943660cdd3709336f848372',
        'text.last_hidden_state': '(3, 12, 128) torch.float32 a21928553894012a27b4fca1fab28700b2e4337ad6298fb3d09b6bd517038512',
        'text_masked.last_hidden_state': '(3, 12, 128) torch.float32 d2d01cdb800a417ea975e12dd2e74ab31f27436d2a5aac81fb6b358f2ebdacf7',
    },
    'flava_long.infer': {
        'image.hidden_states.0': '(2, 257, 128) torch.float32 8c90077260d58aec29709f1b47bac28be8c54ff57325bcfc51b1b30f4ca6c922',
        'image.hidden_states.1': '(2, 257, 128) torch.float32 ab2afacd48db9f8ff9027089e9342b9969a5331cfc20b23fb293b2cefd80b0fd',
        'image.last_hidden_state': '(2, 257, 128) torch.float32 6896eb8bd56b889f6c050ac720635f9618da2cfc847c27166dd614ef1cc1aa3e',
        'image.pooler_output': '(2, 128) torch.float32 e9aa5d322d2c1991ca1ab04c86dd59918999dcaee8148e413ed5c8a3e6260127',
        'image_masked.hidden_states.0': '(2, 257, 128) torch.float32 7f9574d46a14570cff34d37176112bed160bf432967fcf69063cc5034611bdbf',
        'image_masked.hidden_states.1': '(2, 257, 128) torch.float32 ac24bbbb9b551bbfc579e0fa6ef2e96c1c05413dbf7c7bf3cedce20d7eb59212',
        'image_masked.last_hidden_state': '(2, 257, 128) torch.float32 a9c2d8269a332ed239413884bfe3cbde7c2c7b30685104aaf5c73a3089cf8783',
        'image_masked.pooler_output': '(2, 128) torch.float32 6d95b9ded56392bc7bc7c5b6218180701ec274d9bbcfcd0ab5af90747170839a',
        'multimodal.hidden_states.0': '(2, 274, 128) torch.float32 e28983a1a2495ab8fbd5b16ab7b7612cdbaadda04a0d801430b2c2f3d2b330ea',
        'multimodal.hidden_states.1': '(2, 274, 128) torch.float32 466c150ee317e88471ac5ff387de13e1840a547d69270a5dc7daa7014f554dd4',
        'multimodal.last_hidden_state': '(2, 274, 128) torch.float32 1b60ae21ae8878115405a1a079551e53bd927562ceaa3b6b9471361d727f9738',
        'multimodal.pooler_output': '(2, 128) torch.float32 b02adc613204bca9cbb71539bcc3e6a9df644849fcde5db30815b5f939aca267',
        'multimodal_masked.hidden_states.0': '(2, 274, 128) torch.float32 59df8dbcdf34e16fd3157b7aaedab7c4a8fa9afc6a6d1c86693ff55cdea1d1a7',
        'multimodal_masked.hidden_states.1': '(2, 274, 128) torch.float32 82ff738df686a35367748a124ee0b87cec143a72aae08299dd16544e2e303421',
        'multimodal_masked.last_hidden_state': '(2, 274, 128) torch.float32 ebb0f18262d8efbc7f38ffbaa3f12eef907544f6937d6f4e8acb53597a3431f7',
        'multimodal_masked.pooler_output': '(2, 128) torch.float32 acb4ef1a8ac89eb25cc2975df218044fa5713093af9ad521abdd64d37933c881',
        'projected_image_embeddings': '(2, 64) torch.float32 605098c5594494abba966b292b49d1147bb64161bd2bb5d7bcac65939a57a045',
        'projected_text_embeddings': '(2, 64) torch.float32 3b830952baa67eef93cfc560d591b2c5df9fd4ff801af7d0e9790b71ed6d9fcf',
        'text.hidden_states.0': '(2, 16, 128) torch.float32 221cd838344f1a962ecac5b85348cf62086275b5bd4211716486350f2d04c07c',
        'text.hidden_states.1': '(2, 16, 128) torch.float32 f958b2e1ce8cb998e809712f4b00a352083b27992b15a8c26d8fffd5d614bab5',
        'text.last_hidden_state': '(2, 16, 128) torch.float32 d01fbfc8c1fc375a2bbbe54c95c93ede10e9e232d982e0b5a59c9ae6a09d9c94',
        'text.pooler_output': '(2, 128) torch.float32 1bd6a2d1871bb7aad6966aeda9d41a8ed7377f81a4ed09b2a43b51452e5cd59f',
        'text_masked.hidden_states.0': '(2, 16, 128) torch.float32 fde0ca0aae2b9574bf320f03eaea3cd44f8ff2fd5ed18e9e3c3e083803874485',
        'text_masked.hidden_states.1': '(2, 16, 128) torch.float32 d354233e3f7c13ad2b635331fce02222ce4a696ee676c0b12ef8d1b1d5622427',
        'text_masked.last_hidden_state': '(2, 16, 128) torch.float32 437dcc40247425deb53c53e0ba724706d420c02b77c2a91c4b586e44721d729a',
        'text_masked.pooler_output': '(2, 128) torch.float32 43849ed73a2f0bb552ce284cea4064bb916f9f20e09444cdaeb65996b9bbc666',
    },
    'flava_long.grad': {
        'image.last_hidden_state': '(2, 257, 128) torch.float32 6896eb8bd56b889f6c050ac720635f9618da2cfc847c27166dd614ef1cc1aa3e',
        'image_masked.last_hidden_state': '(2, 257, 128) torch.float32 a9c2d8269a332ed239413884bfe3cbde7c2c7b30685104aaf5c73a3089cf8783',
        'multimodal.last_hidden_state': '(2, 274, 128) torch.float32 1b60ae21ae8878115405a1a079551e53bd927562ceaa3b6b9471361d727f9738',
        'multimodal_masked.last_hidden_state': '(2, 274, 128) torch.float32 ebb0f18262d8efbc7f38ffbaa3f12eef907544f6937d6f4e8acb53597a3431f7',
        'text.last_hidden_state': '(2, 16, 128) torch.float32 d01fbfc8c1fc375a2bbbe54c95c93ede10e9e232d982e0b5a59c9ae6a09d9c94',
        'text_masked.last_hidden_state': '(2, 16, 128) torch.float32 437dcc40247425deb53c53e0ba724706d420c02b77c2a91c4b586e44721d729a',
    },
    'flava_attentions.infer': {
        'image.attentions.0': '(3, 2, 17, 17) torch.float32 dc1c6455d47d1794c085882ae65ab8a3849857ac3519e15cf07555682ba4aeed',
        'image.attentions.1': '(3, 2, 17, 17) torch.float32 8651a3cff8215871b65ea546c32754d699fdbe300e0d19cb66e858d2026a6cd8',
        'image.hidden_states.0': '(3, 17, 128) torch.float32 9a8804e0a85df39dc8d23a76487e71b1ef8b00551b4c41b2adc7ea1f6ced64e5',
        'image.hidden_states.1': '(3, 17, 128) torch.float32 db2960578a25632938fb221fc9702322851eb83aa6002bc9eac5cc237c701dc3',
        'image.hidden_states.2': '(3, 17, 128) torch.float32 1a6250ee902fbc5fdb507771d73c36560297be6666e2f343d0080e0670daeb00',
        'image.last_hidden_state': '(3, 17, 128) torch.float32 a391b610fdba22fdc90bfd865a3b8a73e2dd90c3a9d642f1090b1e73bd580e4f',
        'image.pooler_output': '(3, 128) torch.float32 a56599156b548fdbbc0ff3cd85018a20b1ef2ed529a94e11b6af89e1baefe828',
        'image_masked.hidden_states.0': '(3, 17, 128) torch.float32 9a8804e0a85df39dc8d23a76487e71b1ef8b00551b4c41b2adc7ea1f6ced64e5',
        'image_masked.hidden_states.1': '(3, 17, 128) torch.float32 db2960578a25632938fb221fc9702322851eb83aa6002bc9eac5cc237c701dc3',
        'image_masked.hidden_states.2': '(3, 17, 128) torch.float32 1a6250ee902fbc5fdb507771d73c36560297be6666e2f343d0080e0670daeb00',
        'image_masked.last_hidden_state': '(3, 17, 128) torch.float32 a391b610fdba22fdc90bfd865a3b8a73e2dd90c3a9d642f1090b1e73bd580e4f',
        'image_masked.pooler_output': '(3, 128) torch.float32 a56599156b548fdbbc0ff3cd85018a20b1ef2ed529a94e11b6af89e1baefe828',
        'multimodal.attentions.0': '(3, 4, 30, 30) torch.float32 cb2d827f5815fe14602e4ad8208f56a4400aaf2f22ef8a93606e47d98260a305',
        'multimodal.hidden_states.0': '(3, 30, 256) torch.float32 3454bc63cae8255cf286b0e5c08b90090cf0ca70592036fb53233f3d793aa5b0',
        'multimodal.hidden_states.1': '(3, 30, 256) torch.float32 d398f2a4f616aec4da4a81f66b8d5c12ab22d751ab421cb0de8f83781bf8091b',
        'multimodal.last_hidden_state': '(3, 30, 256) torch.float32 4dfcbb2e2aa9dce5854523a06ae40eacc633cd4ae680ccb8771558e6a8c38e35',
        'multimodal.pooler_output': '(3, 256) torch.float32 12f1b33441b8a226ca1180590f58a37752268fb42e293ab2d05ff220477cedf3',
        'projected_image_embeddings': '(3, 64) torch.float32 3077ef64d7930996f491e1826dd9e5fb566ce704f61e29da7f6cab84bbe6e483',
        'projected_text_embeddings': '(3, 64) torch.float32 b934b9682c42092f7880071367d34e2c69c926ccc886996c56600dc9ccd6f265',
        'text.attentions.0': '(3, 2, 12, 12) torch.float32 560773b66d09d0fbd8200a70738311d7c8cf9fe9dde7edd94ce02e61a47115fa',
        'text.attentions.1': '(3, 2, 12, 12) torch.float32 ecd0c9ed4057ec6bf33c4d51f28851f0b4f91d1aa6946e3f53052fe72da138e0',
        'text.hidden_states.0': '(3, 12, 128) torch.float32 8106e4cf6822bf1ca1bdce8c08bac4a96570e7c3864a2fae265a0b37f65c19aa',
        'text.hidden_states.1': '(3, 12, 128) torch.float32 c7ab0466d7644e0f38f6d4adb9468fa4f4c7dcce42169093ee803b584a1f181f',
        'text.hidden_states.2': '(3, 12, 128) torch.float32 c97c2910a4fdc515fbe40adf48ce78098780c8823c7a38279f33296e23a6428b',
        'text.last_hidden_state': '(3, 12, 128) torch.float32 a21928553894012a27b4fca1fab28700b2e4337ad6298fb3d09b6bd517038512',
        'text.pooler_output': '(3, 128) torch.float32 d4aefd87972beaf44cd62684e71e52f89fe411f73304bcd249f02586902ebc01',
    },
    'flava_text512.infer': {
        'image.hidden_states.0': '(3, 17, 128) torch.float32 2c577a49d2b8db423aa90bd9c9a7b059195ed879d391bec20374423f3f802339',
        'image.hidden_states.1': '(3, 17, 128) torch.float32 6f61afa7b6a8d0c6fb585888ffe78b0e8c87b444ed94da0bf614ceaba6ede826',
        'image.last_hidden_state': '(3, 17, 128) torch.float32 e25c9767fb15ccb28991274812fa8a0f6911dd8578a7b189e8855774d0f847a8',
        'image.pooler_output': '(3, 128) torch.float32 be453bc1208922ae806685db9d65eda800ddeb343a8412108757f52b83858fb5',
        'image_masked.hidden_states.0': '(3, 17, 128) torch.float32 2c577a49d2b8db423aa90bd9c9a7b059195ed879d391bec20374423f3f802339',
        'image_masked.hidden_states.1': '(3, 17, 128) torch.float32 6f61afa7b6a8d0c6fb585888ffe78b0e8c87b444ed94da0bf614ceaba6ede826',
        'image_masked.last_hidden_state': '(3, 17, 128) torch.float32 e25c9767fb15ccb28991274812fa8a0f6911dd8578a7b189e8855774d0f847a8',
        'image_masked.pooler_output': '(3, 128) torch.float32 be453bc1208922ae806685db9d65eda800ddeb343a8412108757f52b83858fb5',
        'multimodal.hidden_states.0': '(3, 530, 128) torch.float32 b25da6ada4e435ad2f6740ba78536d31b41a9d775e545be75388ecaf67b1f91d',
        'multimodal.hidden_states.1': '(3, 530, 128) torch.float32 30ecfef8be381590cdbd3331121ee29a965c345ea2a13a5b1891e80afc11c0da',
        'multimodal.last_hidden_state': '(3, 530, 128) torch.float32 ed10d943fef2b3b865788134b47efb8083195b31b753b3d1a5fd9e32acffd724',
        'multimodal.pooler_output': '(3, 128) torch.float32 20fa93a0db1b24750e58f65a3d0d7254727d493c0d79a8632bb29be42ffefae2',
        'projected_image_embeddings': '(3, 64) torch.float32 10a7c1af383bb9eaf3a5efbb1152f17034d64200863e9ab5ce7b58306bb82799',
        'projected_text_embeddings': '(3, 64) torch.float32 a61b7d505888fedc98074e6ae4c81e7fc68a2f20297e956a397c17536c99fdf7',
        'text.hidden_states.0': '(3, 512, 128) torch.float32 7e6ac37abf87e5476980f15366c849837b1046e1a1c69308b889378efcb42594',
        'text.hidden_states.1': '(3, 512, 128) torch.float32 664782cc7b693a32d1c32373e015286a671e2ed780cc09debd0de93af50d868d',
        'text.last_hidden_state': '(3, 512, 128) torch.float32 ce5abc9c6524dcdc16ece2f53c0deec6934ac692340edd68ac172bbeb132fc07',
        'text.pooler_output': '(3, 128) torch.float32 5816b46096bcda1536daf57a2b50b87cef0b3d83abf6271ebf25b3dbff61d1a2',
    },
    'flava_text512.grad': {
        'image.last_hidden_state': '(3, 17, 128) torch.float32 e25c9767fb15ccb28991274812fa8a0f6911dd8578a7b189e8855774d0f847a8',
        'image_masked.last_hidden_state': '(3, 17, 128) torch.float32 e25c9767fb15ccb28991274812fa8a0f6911dd8578a7b189e8855774d0f847a8',
        'multimodal.last_hidden_state': '(3, 530, 128) torch.float32 ed10d943fef2b3b865788134b47efb8083195b31b753b3d1a5fd9e32acffd724',
        'text.last_hidden_state': '(3, 512, 128) torch.float32 ce5abc9c6524dcdc16ece2f53c0deec6934ac692340edd68ac172bbeb132fc07',
    },
    'coca_small.infer': {
        'loss.captioning': '() torch.float32 38a1140d1b1336f154249281295bab4cb81a8f410cd21677bfac6eeca777a2b9',
        'loss.contrastive': '() torch.float32 34d6ad6bda61d5040e83b6c78ff0195dded3c5f007784f212a99d439a08cafff',
        'model.image_pooled_output': '(4, 1, 384) torch.float32 87119eb65d87fe6baf2de2aee585f06c77a243c24e354922c9204162fdde8118',
        'model.multimodal_embeddings': '(4, 12, 512) torch.float32 b0c79ae61d07d82370875b24aea4ce5354abe8c285b6cd5042834293167765ce',
        'model.text_pooled_output': '(4, 384) torch.float32 e79c477178b708c01421d8af049b7620646ec4a11a74f6fa2bb82098ca929dbd',
        'vision.hidden_states.0': '(4, 64, 256) torch.float32 8d9bfc06bd3d5c06b39bc70f56bc9cc96c047f347d88e84e13b178bdb00ca03c',
        'vision.hidden_states.1': '(4, 64, 256) torch.float32 bc9d16e157ec9dd351d77b399e7f6652dc8ba9b99b1011c193435d75a3c13764',
        'vision.hidden_states.2': '(4, 64, 256) torch.float32 5974266c00372259a92fe22236934f7afbcf2feff7528c504e0993ec7fa0bada',
        'vision.last_hidden_state': '(4, 64, 256) torch.float32 5974266c00372259a92fe22236934f7afbcf2feff7528c504e0993ec7fa0bada',
    },
    'coca_small.grad': {
        'loss.captioning': '() torch.float32 38a1140d1b1336f154249281295bab4cb81a8f410cd21677bfac6eeca777a2b9',
        'loss.contrastive': '() torch.float32 34d6ad6bda61d5040e83b6c78ff0195dded3c5f007784f212a99d439a08cafff',
        'vision.last_hidden_state': '(4, 64, 256) torch.float32 5974266c00372259a92fe22236934f7afbcf2feff7528c504e0993ec7fa0bada',
    },
    'coca_parallel.infer': {
        'loss.captioning': '() torch.float32 17aa2b880e49fcf09ca2d32394a38364c9be18997276287df0be0df280093ca0',
        'loss.contrastive': '() torch.float32 29af79861a90d7ea58a604ba3da461b4c8f4c5ce357f463253e6cbd35a4cb563',
        'model.image_pooled_output': '(8, 128) torch.float32 d535f5016afaf2dff289ce5ad9584e4567d36e6cca3a7f210685da89dafbcb4a',
        'model.multimodal_embeddings': '(8, 8, 300) torch.float32 fab46019849c19fd5e973d116d9db40ac6f80d3bf5d2275a4d6f500e751627d4',
        'model.text_pooled_output': '(8, 128) torch.float32 1363704b77b8ad1a612e95ae4f1ac6e023efc75ea793f468db254e1fd8287ad8',
        'vision.hidden_states.0': '(8, 16, 128) torch.float32 788df8208eddbdc2d8dc2cfc58fb0ae94f85eee9272b1166a12a7523c78d0a55',
        'vision.hidden_states.1': '(8, 16, 128) torch.float32 4e8805e08b4d702636a3ec02adbeb9fe401dee4c0cc024ac03391bef0fe04b5c',
        'vision.last_hidden_state': '(8, 16, 128) torch.float32 4e8805e08b4d702636a3ec02adbeb9fe401dee4c0cc024ac03391bef0fe04b5c',
    },
    'coca_parallel.grad': {
        'loss.captioning': '() torch.float32 17aa2b880e49fcf09ca2d32394a38364c9be18997276287df0be0df280093ca0',
        'loss.contrastive': '() torch.float32 29af79861a90d7ea58a604ba3da461b4c8f4c5ce357f463253e6cbd35a4cb563',
        'vision.last_hidden_state': '(8, 16, 128) torch.float32 4e8805e08b4d702636a3ec02adbeb9fe401dee4c0cc024ac03391bef0fe04b5c',
    },
    'coca_l14.infer': {
        'loss.captioning': '() torch.float32 e4de99b67569fe8b5cad791573a92f9f703ab15faca254c8c586c1f7b6ac610f',
        'loss.contrastive': '() torch.float32 c747a8d06b05347c5cdd5b7d9f0362c61172f7aa3938f7ff082c1c86d9bad38e',
        'model.image_pooled_output': '(2, 1, 768) torch.float32 e89ed8e627433ea6c06ebc0cb92b26b891d68e1547d4a5afc1b0a1f0f0c7ab5f',
        'model.multimodal_embeddings': '(2, 76, 49408) torch.float32 45b89e2e9c92e518245d6aff56c54833b2c540a4f50ee2f74a44badf4463b4a7',
        'model.text_pooled_output': '(2, 768) torch.float32 7f89bef6764a9f26b5d0b9de07d736d75092389d668e6c6ad99389d975e9ce79',
        'vision.hidden_states.0': '(2, 256, 1024) torch.float32 286ecba3ee3eda534b5dd20e5053878faeccb69682255627a721fb8962904b52',
        'vision.hidden_states.1': '(2, 256, 1024) torch.float32 a9b093a6bf3f47ca7c7477d3e7cca4befe75fc8936a2fb472d4bee337490ec19',
        'vision.hidden_states.2': '(2, 256, 1024) torch.float32 49b840982c2d051ca5fe76210dc0505c72cb054ab942d70375e05f2914fcc307',
        'vision.last_hidden_state': '(2, 256, 1024) torch.float32 49b840982c2d051ca5fe76210dc0505c72cb054ab942d70375e05f2914fcc307',
    },
    'coca_l14.grad': {
        'loss.captioning': '() torch.float32 e4de99b67569fe8b5cad791573a92f9f703ab15faca254c8c586c1f7b6ac610f',
        'loss.contrastive': '() torch.float32 c747a8d06b05347c5cdd5b7d9f0362c61172f7aa3938f7ff082c1c86d9bad38e',
        'vision.last_hidden_state': '(2, 256, 1024) torch.float32 49b840982c2d051ca5fe76210dc0505c72cb054ab942d70375e05f2914fcc307',
    },
    'text_decoder_no_cls.infer': {
        'pooled': '(3, 96) torch.float32 4ba4cb180ee243644111ef7330578468a1c9aa52c868956c17edb35f3417bef2',
        'tokens': '(3, 20, 128) torch.float32 6f83ad91f4941ecf1021bc206d61d1806e9c8deedc50ae0c88714baf442ff723',
    },
    'coca_hd96.infer': {
        'text.pooled': '(3, 96) torch.float32 df8a09f65011359bde2f795280659d297d2c7fe12c73f8a29a694a94ffd16d3d',
        'text.tokens': '(3, 12, 384) torch.float32 578e27886854eeca0375936bedf31fae2dc9cb723dd6a0b0851934053fd33e40',
        'vision.hidden_states.0': '(3, 17, 384) torch.float32 7ab812352e8631f0b79ddb4b0705fb109c9a7c02833a6117f60c2e76419ba894',
        'vision.hidden_states.1': '(3, 17, 384) torch.float32 8f9a0891867fae69a5ca24b22e8c144e465ce9216c95ac1f8316f460bbd38b60',
        'vision.hidden_states.2': '(3, 17, 384) torch.float32 a03195aeacf199b136094b98a680e68490ef1f6135a72bd3c9bf0253da2a797d',
        'vision.last_hidden_state': '(3, 17, 384) torch.float32 ddec42f7f075a220c0915d30253e96e9addc84696991015ba35907d02e479152',
    },
    'coca_hd128.infer': {
        'text.pooled': '(3, 96) torch.float32 475162f4edd175574f75a37e3663cead4e4d61e19fd37e9b6b01b8f2334faf74',
        'text.tokens': '(3, 12, 256) torch.float32 14b1ce34bba70acb0022e9110f040ce70344fb8584690ff1857dd448b7241a82',
        'vision.hidden_states.0': '(3, 17, 256) torch.float32 351b996edbe39c247153173c2c25a6f8fbd353942f87e81194912ed3ffaf5e33',
        'vision.hidden_states.1': '(3, 17, 256) torch.float32 8fa35243b1d33e05758ac66ad9fa0737facf047c88b9e806be93a2ae8489c446',
        'vision.hidden_states.2': '(3, 17, 256) torch.float32 2f5d7c34985f4e7422e2effb2e3847d66760bd1490740a91fe38a1409c2c7c41',
        'vision.last_hidden_state': '(3, 17, 256) torch.float32 1cccd9c0d6cb73707a0f8c4b2ae8e6d4d90d3b9b232f4daccbe90b400c7c3a09',
    },
    'vit_drop.infer': {
        'hidden_states.0': '(4, 49, 128) torch.float32 a72ce5802d3d2c6ff02e3a7ba80c36d535edfa4ab0d32067813bf94c382df4e3',
        'hidden_states.1': '(4, 49, 128) torch.float32 440ce22451cf3c4a6db98f49025a01d223ceffa90f88db64fcabb7b6a7102a75',
        'hidden_states.2': '(4, 49, 128) torch.float32 5202f2a331bb8808a3e879dd3d756a718057f0815799ff20ca43a4bc4487f704',
        'hidden_states.3': '(4, 49, 128) torch.float32 437ca8147ac89289541a23bbfbb3f044d382965d8854a1ca9b840259343effeb',
        'last_hidden_state': '(4, 49, 128) torch.float32 9a8695b5e151fd81289c90be6f254083b12d0c3e69e551b41920f0fe43f3d267',
    },
    'clip_small.infer': {
        'image.embeddings': '(6, 64) torch.float32 37cf4a55f7b872b5ac1e7d732d658d269390e051db61cb5693e2a7d23372f4c4',
        'text.embeddings': '(6, 64) torch.float32 f9b77915bf2430ad93236172cdc3d49aff5ca3a673eefda1c8df4c2da5f894e3',
        'text.hidden_state': '(6, 77, 128) torch.float32 7d7a81ab171634ae070490a8272ee3c60279d4e9c834556c5913e3f11d93019d',
    },
    'clip_small.grad': {
        'image.embeddings': '(6, 64) torch.float32 37cf4a55f7b872b5ac1e7d732d658d269390e051db61cb5693e2a7d23372f4c4',
        'text.embeddings': '(6, 64) torch.float32 f9b77915bf2430ad93236172cdc3d49aff5ca3a673eefda1c8df4c2da5f894e3',
    },
    'standalone_encoder.infer': {
        'hidden_states.0': '(4, 20, 128) torch.float32 9d2d3d9fc40a1929827fccec26876dd39d07c3a57c7dc3367a68bddba21b09a2',
        'hidden_states.1': '(4, 20, 128) torch.float32 44ecc096c17cf09b63301cddaeff103101db20a2146c81e966eda5574c73bf9f',
        'hidden_states.2': '(4, 20, 128) torch.float32 91e73578053ab421bc58731fc4d4dd5dff9d227d7553eb2a4d8d3af344f0ec83',
        'hidden_states.3': '(4, 20, 128) torch.float32 ce8e54f33464f33d98c4d6d2fa1a47086ee65972330266092856198d79179d56',
        'last_hidden_state': '(4, 20, 128) torch.float32 ef4ad8177bf3f469852fb8bfda2d335f634c60d76c3fe94c16ab764a0f8c109d',
    },
    'standalone_encoder.grad': {
        'hidden_states.0': '(4, 20, 128) torch.float32 9d2d3d9fc40a1929827fccec26876dd39d07c3a57c7dc3367a68bddba21b09a2',
        'hidden_states.1': '(4, 20, 128) torch.float32 44ecc096c17cf09b63301cddaeff103101db20a2146c81e966eda5574c73bf9f',
        'hidden_states.2': '(4, 20, 128) torch.float32 91e73578053ab421bc58731fc4d4dd5dff9d227d7553eb2a4d8d3af344f0ec83',
        'hidden_states.3': '(4, 20, 128) torch.float32 ce8e54f33464f33d98c4d6d2fa1a47086ee65972330266092856198d79179d56',
        'last_hidden_state': '(4, 20, 128) torch.float32 ef4ad8177bf3f469852fb8bfda2d335f634c60d76c3fe94c16ab764a0f8c109d',
    },
    'standalone_drop.infer': {
        'hidden_states.0': '(4, 20, 128) torch.float32 9d2d3d9fc40a1929827fccec26876dd39d07c3a57c7dc3367a68bddba21b09a2',
        'hidden_states.1': '(4, 20, 128) torch.float32 831be8cd17d14c2a10ec1fc0fb037335fa7edd667894cddaf44a2987f38474c3',
        'hidden_states.2': '(4, 20, 128) torch.float32 b22710c0b864a6a69bfd6a084477f604a431b22ceb83b350ba689d0402031f89',
        'hidden_states.3': '(4, 20, 128) torch.float32 580b39fd455652233940b0f84b80a462ca3b76e53687a7adbdf708b73b8104ce',
        'last_hidden_state': '(4, 20, 128) torch.float32 bc0a74b24f291f7f5fc16bda0108db7132132b82256d907203a0f33847d415b7',
    },
    'standalone_layer.infer': {
        'output': '(4, 20, 128) torch.float32 c4306e38ee00eb9866b496cc9a428796cb5822d58bade6a7f14f0abdfd768594',
    },
}


def digests(name, dev):
    return {k: f"{tuple(t.shape)} {t.dtype} {_digest(t)}" for k, t in sorted(_case(name, dev).items())}


@pytest.mark.parametrize("name", CASES)
def test_forward_digests(name):
    dev = torch.device("cuda:0")
    got = digests(name, dev)
    want = PINNED[name]
    assert sorted(got) == sorted(want), name
    changed = [k for k in want if got[k] != want[k]]
    assert not changed, f"{name}: {changed}"


def record():
    dev = torch.device("cuda:0")
    print("PINNED = {")
    for name in CASES:
        print(f"    {name!r}: {{")
        for k, v in digests(name, dev).items():
            print(f"        {k!r}: {v!r},")
        print("    },")
    print("}")


if __name__ == "__main__":
    record()
