"""One runtime per CLIP / FLAVA / CoCa module and per standalone pre-norm encoder serves both grad modes; these tests
check, WITHOUT a GPU, that its torch.no_grad() entry point (no save Workspace, scratch shared by the layers) and its
training forward (activations saved per call) compute the same bits, with the kernels swapped for their torch emulation (tests/emu_ops.py, with the
stochastic-depth variants of tests/emu_drop_path_ops.py).  The same property on the kernels proper:
tests/test_gpu_grad_mode_invariance.py."""
import pytest
import torch

import coca_cases as CC
import drop_path_cases as DP
import emu_drop_path_ops
import flava_cases as FC
import test_gpu_grad_mode_invariance as GI
import test_gpu_runtime_pinned as P
from test_gpu_coca_train import _cfg, _rel

CPU = torch.device("cpu")


@pytest.fixture()
def emu(monkeypatch):
    emu_drop_path_ops.install(monkeypatch)


def _assert_grad_modes_agree(outputs):
    with torch.no_grad():
        ref = {k: v.detach().clone() for k, v in outputs().items()}
    with torch.enable_grad():
        got = outputs()
    assert sorted(got) == sorted(ref)
    differ = [k for k in ref if not torch.equal(got[k].detach(), ref[k])]
    assert not differ, differ


@pytest.mark.parametrize("name", list(FC.CASES) + list(CC.CASES) + ["clip_small"])
def test_no_grad_forward_equals_training_forward(emu, name):
    """FLAVA: the image (patch mask), text (key-padding mask) and multimodal encoders of FLAVAModel; CoCa, one module at
    a time: vision encoder, poolers, text decoder ([B, S, S] causal x padding mask), multimodal decoder
    (cross-attention); CLIP: both towers' embeddings."""
    _assert_grad_modes_agree(lambda: GI._outputs(name, CPU))


@pytest.mark.parametrize("name", ["vit_cls", "vit_nocls"])
def test_no_grad_forward_equals_training_forward_with_drop_path(emu, name):
    """VisionTransformer in train() mode with drop_path_rate: both grad modes draw the same stochastic-depth factors
    and apply them in the same residual adds."""
    from multimodal_b200.modules.encoders.vision_transformer import vision_transformer

    def outputs():
        vit = DP.build_vit(vision_transformer, name).train()
        images, _ = DP.vit_inputs(name)
        torch.manual_seed(DP.VIT[name]["seed"])
        out = vit(images)
        return {"last_hidden_state": out.last_hidden_state,
                **{f"hidden_states.{i}": h for i, h in enumerate(out.hidden_states)}}

    _assert_grad_modes_agree(outputs)


@pytest.mark.parametrize("kind,masked,drop", [("encoder", False, False), ("encoder", True, False),
                                               ("encoder", False, True), ("encoder", True, True),
                                               ("layer", False, False), ("layer", True, False)])
def test_standalone_no_grad_forward_equals_training_forward(emu, monkeypatch, kind, masked, drop):
    """A standalone pre-norm TransformerEncoder (final LayerNorm, return_hidden_states) or TransformerEncoderLayer, with
    and without a [B, S, S] bool mask; with drop_path_rate in train() mode both grad modes draw the same factors under
    the same seed.  The CUDA-input check of the no_grad call is lifted for the emulated kernels."""
    from multimodal_b200 import engine_layers

    monkeypatch.setattr(engine_layers, "_cuda", lambda t, what: None)
    m, x, mask = P._standalone(kind, drop=drop)

    def outputs():
        torch.manual_seed(37)
        return P._standalone_outputs(m, x, mask if masked else None, CPU)

    _assert_grad_modes_agree(outputs)


def test_no_grad_head_dim_96_stacks_against_oracle(emu):
    """coca_small with head_dim-96 vision and text stacks: the no_grad forward against the fp32 oracle.  Training
    refuses that head_dim."""
    from multimodal_b200._lib import MMBError
    from multimodal_b200.models.coca import coca_for_pretraining
    from oracle import coca_oracle as CO

    kw = dict(CC.CASES["coca_small"]["kwargs"], pooler_input_embed_dim=384, vision_n_head=4, text_n_head=4)
    torch.manual_seed(0)
    m = coca_for_pretraining(**kw).eval()
    g = torch.Generator().manual_seed(13)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.03 * torch.randn(p.shape, generator=g))
    inp = CC.inputs("coca_small")
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    cfg = _cfg(kw)
    with torch.no_grad():
        v = m.model.vision_encoder(inp["images"])
        pooled, tokens = m.model.text_decoder(inp["texts"])
    ref_pooled, ref_tokens = CO.text_decoder(inp["texts"], sd, cfg)
    assert _rel(v.last_hidden_state, CO.vision_encoder(inp["images"], sd, cfg)) < 2e-2
    assert _rel(tokens, ref_tokens) < 2e-2 and _rel(pooled, ref_pooled) < 2e-2
    with pytest.raises(MMBError, match="training needs head_dim 64"):
        m.model.vision_encoder(inp["images"])


def test_no_grad_forward_between_training_forward_and_backward(emu):
    """A no_grad call of the CoCa text decoder (another batch size) between a training forward and its backward leaves
    that backward's gradients unchanged: the backward reads only what its own forward saved."""
    def grads(interleave):
        m, _, texts = P._coca("coca_small")
        dec = m.model.text_decoder
        pooled, tokens = dec(texts)
        if interleave:
            with torch.no_grad():
                dec(texts[:2])
        (pooled.sum() + tokens.square().sum()).backward()
        return {k: p.grad for k, p in dec.named_parameters() if p.grad is not None}

    ref, got = grads(False), grads(True)
    assert sorted(got) == sorted(ref)
    assert not [k for k in ref if not torch.equal(got[k], ref[k])]
