"""The CLIP, FLAVA and CoCa modules and the standalone pre-norm encoder compute the same forward values under
torch.no_grad() and with grad mode on, bit for bit.

The inference and training runtimes launch the same kernels on the same operands (ops.self_attention picks the
attention kernel for both); only the buffers that keep activations for the backward differ.  The cases are those of
test_gpu_runtime_pinned.py (the standalone pre-norm TransformerEncoder with its [B, S, S] mask), plus a CoCa vision
tower at 400 tokens, inside the band (385-512 tokens, unmasked head_dim-64 self-attention) where the two modes once
chose different attention kernels.  On an H100 the fused and the general forward give the same bits in that band, so
this test would not notice that split coming back (it only cost speed); tests/test_attention_router_cpu.py is what
guards the routing rule.
"""
import pytest
import torch

import test_gpu_runtime_pinned as P

pytestmark = pytest.mark.gpu


def _coca_modules(m, images, texts, dev):
    """Every CoCa submodule output, called one module at a time."""
    c = m.model
    images, texts = images.to(dev), texts.to(dev)
    v = c.vision_encoder(images)
    pooled = c.vision_pooler(v.last_hidden_state)
    cap = pooled[0] if isinstance(pooled, list) else pooled[:, 1:]
    text_pooled, tokens = c.text_decoder(texts)
    res = {"vision.last_hidden_state": v.last_hidden_state, "text.pooled": text_pooled, "text.tokens": tokens,
           "multimodal": c.multimodal_decoder(tokens, cap)}
    res.update({f"vision.hidden_states.{i}": h for i, h in enumerate(v.hidden_states)})
    res.update({f"pooler.{i}": p for i, p in enumerate(pooled)} if isinstance(pooled, list) else {"pooler": pooled})
    return res


def _vision_400():
    from multimodal_b200.models.coca import coca_for_pretraining
    from test_gpu_attention_long import _coca_case

    torch.manual_seed(0)
    m = coca_for_pretraining(**_coca_case(80)["kwargs"])
    g = torch.Generator().manual_seed(13)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.03 * torch.randn(p.shape, generator=g))
    images = torch.randn(3, 3, 80, 80, generator=torch.Generator().manual_seed(6))
    return m.eval(), images


def _outputs(name, dev):
    if name.startswith("flava"):
        if name == "flava_text512":
            m, inp = P._flava_512()
        else:
            m, inp = P._flava(name)
        return P._flava_outputs(m.to(dev), inp, dev)
    if name == "coca_vision_400":
        m, images = _vision_400()
        v = m.to(dev).model.vision_encoder(images.to(dev))
        assert v.last_hidden_state.shape[1] == 400
        return {"last_hidden_state": v.last_hidden_state,
                **{f"hidden_states.{i}": h for i, h in enumerate(v.hidden_states)}}
    if name == "standalone_encoder":
        m, x, mask = P._standalone("encoder")
        return P._standalone_outputs(m.to(dev), x, mask, dev)
    if name == "clip_small":
        m, image, text = P._clip_small()
        return P._clip_outputs(m.to(dev), image, text, dev)
    m, images, texts = P._coca_l14() if name == "coca_l14" else P._coca(name)
    return _coca_modules(m.to(dev), images, texts, dev)


@pytest.mark.parametrize("name", ["flava_small", "flava_long", "flava_text512", "coca_small", "coca_parallel",
                                  "coca_l14", "coca_vision_400", "clip_small", "standalone_encoder"])
def test_no_grad_equals_grad_mode_forward(name):
    dev = torch.device("cuda:0")
    with torch.no_grad():
        ref = {k: v.detach().clone() for k, v in _outputs(name, dev).items()}
    with torch.enable_grad():
        got = _outputs(name, dev)
    assert sorted(got) == sorted(ref)
    differ = [k for k in ref if not torch.equal(got[k].detach(), ref[k])]
    assert not differ, f"{name}: {differ}"
