"""Host logic of the CoCa training runtime (engine_coca_train.py + the cross-attention / general-mask extensions of
engine.TransformerStack) WITHOUT a GPU: kernel wrappers swapped for their torch emulation (tests/emu_ops.py), the result
compared with autograd over the fp32 oracle (oracle/coca_oracle.py).  Kernels proper: tests/test_gpu_coca_train.py."""
import pytest
import torch

import coca_cases as CC
import emu_ops
import test_gpu_coca_train as G


@pytest.fixture()
def emu(monkeypatch):
    emu_ops.install(monkeypatch)


@pytest.mark.parametrize("name", list(CC.CASES))
def test_coca_training_schedule_against_oracle_with_emulated_kernels(emu, name):
    G.coca_grad_parity(torch.device("cpu"), name, "cpu_emu_" + name)


@pytest.mark.parametrize("masked", [False, True])
def test_standalone_encoder_layers_train_with_emulated_kernels(emu, masked):
    G.standalone_layers_grad_parity(torch.device("cpu"), masked)


def test_coca_model_forward_logits_path_with_emulated_kernels(emu):
    """`CoCaModel.forward` under autograd returns the vocabulary logits with a graph (LinearF32Function head, width 300 is
    not a multiple of 8): gradient of <w, logits> w.r.t. the projection and the first vision layer against the oracle."""
    from oracle import coca_oracle as CO
    from multimodal_b200.models.coca.coca_model import coca_for_pretraining

    name = "coca_parallel"
    m = CC.build(lambda **kw: coca_for_pretraining(**kw), name).train()
    cfg = G._cfg(CC.CASES[name]["kwargs"])
    inp = CC.inputs(name)
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    x = CO.vision_encoder(inp["images"], sd, cfg)
    both = CO.attention_pooler(x, sd, "model.vision_pooler", cfg["pooler_n_head"])
    _, tokens = CO.text_decoder(inp["texts"], sd, cfg)
    ref = CO.multimodal_decoder(tokens, both[:, 1:], sd, cfg)
    w = torch.randn(ref.shape, generator=torch.Generator().manual_seed(2)) / 10
    (ref * w).sum().backward()
    out = m.model(inp["images"], inp["texts"])
    assert out.multimodal_embeddings.requires_grad and out.multimodal_embeddings.shape == ref.shape
    assert G._rel(out.multimodal_embeddings, ref) < 2e-2
    (out.multimodal_embeddings * w).sum().backward()
    named = dict(m.named_parameters())
    for k in ("model.multimodal_decoder.output_projection.weight", "model.vision_encoder.embeddings.conv_projection.weight",
              "model.vision_pooler.query", "model.text_decoder.embeddings.cls_embedding"):
        assert G._rel(named[k].grad, sd[k].grad) < 5e-2, (k, G._rel(named[k].grad, sd[k].grad))
