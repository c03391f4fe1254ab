"""Host logic of the FLAVA training runtime (engine_flava_train.py + engine.TransformerStack) WITHOUT a GPU: the
kernel wrappers are swapped for their torch emulation (tests/emu_ops.py), so what is checked here is the schedule —
buffer routing, packed q/k/v parameter views, per-call saved activations (the same encoder runs twice before the
backward), gradient slots — against autograd over the fp32 oracle.  The kernels themselves are checked on the GPU
(tests/test_gpu_flava_train.py)."""
import math

import pytest
import torch

import emu_ops
import flava_cases as FC
import test_gpu_flava_train as G   # shared helpers only (its tests carry the gpu marker)


@pytest.fixture()
def emu(monkeypatch):
    emu_ops.install(monkeypatch)


def test_flava_training_schedule_against_oracle_with_emulated_kernels(emu):
    from multimodal_b200.models.flava import flava_model

    name = "flava_small"
    m = FC.build(flava_model, name)
    cpu = torch.device("cpu")
    m = G._grad_parity(cpu, m, G._cfg(FC.CASES[name]["kwargs"]), FC.inputs(name), "cpu_emu", 6e-2)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.01 * torch.randn_like(p))
            p.grad = None
    G._grad_parity(cpu, m, G._cfg(FC.CASES[name]["kwargs"]), FC.inputs(name), "cpu_emu_step2", 6e-2)


def test_flava_mm_direct_call_and_frozen_encoder_with_emulated_kernels(emu):
    G.test_flava_mm_encoder_direct_call_and_frozen_parts.__wrapped__(torch.device("cpu")) \
        if hasattr(G.test_flava_mm_encoder_direct_call_and_frozen_parts, "__wrapped__") \
        else G.test_flava_mm_encoder_direct_call_and_frozen_parts(torch.device("cpu"))


@pytest.mark.parametrize("name", ["unimodal", "multimodal"])
def test_pretraining_loss_gradients_with_emulated_kernels(emu, name):
    """Head schedules (engine_flava_heads.py) and the global contrastive loss (engine_loss.py: the batch of 5 takes the
    exact-fp32 SIMT schedule) on the emulated kernels."""
    G._loss_grad_parity(torch.device("cpu"), name, 1.0, "cpu_emu_" + name)


def test_flava_for_pretraining_step_with_emulated_kernels(emu):
    """FLAVAForPreTraining under autograd, end to end (two passes per encoder, multimodal encoder, ITM / MMM heads): the
    total loss and every reached parameter gradient against autograd over the two oracles chained the same way."""
    import flava_pretraining_cases as PC
    from oracle import flava_loss_oracle as LO
    from oracle import flava_oracle as FO
    from multimodal_b200.models.flava import flava_model, FLAVAForPreTraining
    from multimodal_b200.modules.losses.flava import FLAVAPretrainingLoss

    m = PC.build_model(flava_model, FLAVAForPreTraining, FLAVAPretrainingLoss).train()
    inp, _ = PC.model_inputs()
    out = m(**inp)
    total = sum(v for v in out.losses.values() if v is not None)
    total.backward()

    # oracle: same composition (models/flava/model.py:334-377)
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    msd = {k[len("model."):]: v for k, v in sd.items() if k.startswith("model.")}
    lsd = {k[len("loss."):]: v for k, v in sd.items() if k.startswith("loss.")}
    cfg = G._cfg(PC.MODEL_KW)
    keep = inp["image_patches_mask"].flatten(1).bool()
    mim = m.image_codebook(inp["image_for_codebook"]).flatten(1).clone()
    mim[~keep] = -1
    img_m = FO.image_encoder(inp["image"], msd, cfg, keep)
    txt_m = FO.text_encoder(inp["text_masked"], msd, cfg)
    mm = FO.mm_encoder(img_m["hidden_states"][-1], txt_m["hidden_states"][-1], msd, cfg)["last_hidden_state"]
    img = FO.image_encoder(inp["image"], msd, cfg)["last_hidden_state"][:, 0]
    txt = FO.text_encoder(inp["text"], msd, cfg)["last_hidden_state"][:, 0]
    kw = dict(multimodal_masked_sequence=mm, mlm_labels=inp["mlm_labels"], mim_labels=mim, itm_labels=inp["itm_labels"],
              projected_image_embeddings=FO._lin(img, msd, "image_projection"),
              projected_text_embeddings=FO._lin(txt, msd, "text_projection"))
    ref_total, parts = G._oracle_loss_total(lsd, kw, dict(contrastive=m.loss.contrastive_loss_weight))
    ref_total.backward()
    assert abs(total.item() - ref_total.item()) < 2e-2 * max(1.0, abs(ref_total.item())), (total.item(), ref_total.item())
    n = 0
    for k, p in m.named_parameters():
        ref = sd[k].grad
        if ref is None or ref.norm().item() == 0.0:
            assert p.grad is None or p.grad.abs().max().item() < 1e-6, k
            continue
        if k.endswith(".key.bias"):
            continue
        if k == "model.text_encoder.embeddings.word_embeddings.weight":
            ref = ref.clone()
            ref[0] = 0
        assert p.grad is not None, k
        assert G._rel(p.grad, ref) < 6e-2, (k, G._rel(p.grad, ref))
        n += 1
    assert n > 60
