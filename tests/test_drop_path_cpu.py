"""CPU tests of stochastic depth (`drop_path_rate`, modules/layers/stochastic_depth.py): the noise the package draws and
the generator state after it, pinned to the reference's own draws (tests/golden/drop_path_golden.pt); the module
structure, per-layer rates and parameters; the fp32 oracle fed the golden noise against the reference's outputs and
gradients; and the training schedules (which buffer gets which factor, forward and backward) with the kernels swapped
for their CPU emulation (tests/emu_ops.py, with the stochastic-depth variants of tests/emu_drop_path_ops.py) against the
golden and the oracle."""
import os

import pytest
import torch
from torch import nn

import drop_path_cases as DP
import emu_drop_path_ops

GOLD = os.path.join(os.path.dirname(__file__), "golden", "drop_path_golden.pt")


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD)


@pytest.fixture()
def emu(monkeypatch):
    emu_drop_path_ops.install(monkeypatch)


def _vit(name):
    from multimodal_b200.modules.encoders.vision_transformer import vision_transformer
    return DP.build_vit(vision_transformer, name)


def _layers(name):
    from multimodal_b200.modules.layers.transformer import TransformerEncoder, TransformerEncoderLayer
    return DP.build_layers(TransformerEncoderLayer, TransformerEncoder, name)


def _stack(m):
    return list(m.layer) if hasattr(m, "layer") else [m]


def _draw_vit(vit, B, seed):
    from multimodal_b200.modules.layers.stochastic_depth import drop_path_scales
    from multimodal_b200.modules.masking.random_masking import patch_keep_indices

    torch.manual_seed(seed)
    drop = patch_keep_indices(vit.embeddings, B, "cpu")     # patch-dropping draws come first, as in the reference
    scales = drop_path_scales(vit.encoder.layer, B, "cpu")
    return (drop[0] if drop is not None else None), scales


def _same_draws(scales, want, rates):
    assert scales is not None
    assert len(scales) == len(rates)
    for (sa, sf), (wa, wf), p in zip(scales, want, rates):
        for got, ref in ((sa, wa), (sf, wf)):
            assert (got is None) == (ref is None), p
            if ref is not None:
                assert got.dtype == torch.float32 and got.shape == ref.shape and got.is_contiguous()
                assert torch.equal(got.view(torch.int32), ref.contiguous().view(torch.int32)), p


@pytest.mark.parametrize("name", list(DP.VIT))
def test_vit_draws_match_reference(gold, name):
    g, c = gold["vit"][name], DP.VIT[name]
    vit = _vit(name)
    assert DP.CC.param_checksum(vit) == pytest.approx(g["param_checksum"], rel=1e-12)
    assert DP.layer_rates(vit.encoder.layer) == g["rates"]
    _, scales = _draw_vit(vit, c["B"], c["seed"])
    assert torch.equal(torch.get_rng_state(), g["rng_after"])
    _same_draws(scales, DP.pair_draws(g["rates"], True, g["noise"]), g["rates"])
    assert scales[0] == (None, None)       # layer 0 has p = 0: no draw


@pytest.mark.parametrize("name", list(DP.LAYERS))
def test_standalone_layer_draws_match_reference(gold, name):
    from multimodal_b200.modules.layers.stochastic_depth import drop_path_scales

    g, c = gold["layers"][name], DP.LAYERS[name]
    m = _layers(name)
    assert DP.CC.param_checksum(m) == pytest.approx(g["param_checksum"], rel=1e-12)
    assert DP.layer_rates(_stack(m)) == g["rates"]
    torch.manual_seed(c["seed"])
    scales = drop_path_scales(_stack(m), c["B"], "cpu")
    assert torch.equal(torch.get_rng_state(), g["rng_after"])
    if not g["noise"]:                     # one-layer encoder: linspace(0, r, 1) = [0], nothing drawn
        assert scales is None
    else:
        _same_draws(scales, DP.pair_draws(g["rates"], True, g["noise"]), g["rates"])


def test_module_structure_rates_and_parameters():
    from multimodal_b200.modules.encoders.vision_transformer import vision_transformer
    from multimodal_b200.modules.layers.stochastic_depth import StochasticDepth
    from multimodal_b200.modules.layers.transformer import TransformerEncoder, TransformerEncoderLayer
    from multimodal_b200.models.coca.coca_model import coca_vit

    enc = TransformerEncoder(5, 128, 2, 256, drop_path_rate=0.3)
    for layer, p in zip(enc.layer, torch.linspace(0, 0.3, 5)):
        assert isinstance(layer.attention_dropout, StochasticDepth)
        assert layer.attention_dropout is layer.feedforward_dropout
        assert layer.attention_dropout.p == p.item() and layer.attention_dropout.mode == "row"
    assert repr(enc.layer[4].attention_dropout) == f"StochasticDepth(p={torch.tensor(0.3).item()}, mode=row)"
    assert TransformerEncoder(1, 128, 2, 256, drop_path_rate=0.3).layer[0].attention_dropout.p == 0.0
    assert TransformerEncoderLayer(128, 2, 256, drop_path_rate=0.3).attention_dropout.p == 0.3
    plain = TransformerEncoderLayer(128, 2, 256)
    assert isinstance(plain.attention_dropout, nn.Dropout) and plain.attention_dropout is not plain.feedforward_dropout
    with pytest.raises(NotImplementedError):
        TransformerEncoderLayer(128, 2, 256, dropout=0.1, drop_path_rate=0.1)
    # no parameters: the same state-dict keys and the same seeded values as a model built without a rate
    for build in (lambda r: vision_transformer(patch_size=4, hidden_dim=128, dim_feedforward=256, n_layer=3, n_head=2,
                                               image_size=16, drop_path_rate=r),
                  lambda r: coca_vit(vision_patch_size=8, vision_dim_feedforward=256, vision_n_layer=2,
                                     vision_n_head=2, image_size=32, vocab_size=300, num_text_positions=9,
                                     text_hidden_dim=128, text_n_layer=1, text_n_head=2, text_dim_feedforward=256,
                                     text_output_dim=128, fusion_n_layer=1, fusion_n_head=2, fusion_dim_feedforward=256,
                                     multimodal_output_projection_dim=300, pooler_input_embed_dim=128,
                                     pooler_output_embed_dim=128, pooler_n_head=2, pooler_n_queries=16,
                                     vision_drop_path_rate=r)):
        torch.manual_seed(0)
        a = build(None).state_dict()
        torch.manual_seed(0)
        b = build(0.2).state_dict()
        assert list(a) == list(b)
        assert all(torch.equal(a[k], b[k]) for k in a)


def test_no_draw_in_eval_or_at_rate_zero_and_range_checks():
    from multimodal_b200.modules.layers.stochastic_depth import StochasticDepth, drop_path_scales
    from multimodal_b200.modules.layers.transformer import TransformerEncoder, TransformerEncoderLayer

    encs = [TransformerEncoder(3, 128, 2, 256, drop_path_rate=0.5).eval(),
            TransformerEncoder(3, 128, 2, 256, drop_path_rate=0.0).train(), TransformerEncoder(3, 128, 2, 256).train()]
    torch.manual_seed(1)
    state = torch.get_rng_state()
    for enc in encs:
        assert drop_path_scales(enc.layer, 4, "cpu") is None
    assert torch.equal(torch.get_rng_state(), state)
    # p == 1 zeroes the branch for every sample, without a division
    torch.manual_seed(1)
    s = drop_path_scales([TransformerEncoderLayer(128, 2, 256, drop_path_rate=1.0).train()], 4, "cpu")
    assert torch.equal(s[0][0], torch.zeros(4)) and torch.equal(s[0][1], torch.zeros(4))
    # out-of-range p raises at call time, before the training check (so in eval() too), as torchvision does
    for p in (-0.1, 1.5):
        for mode in (True, False):
            layer = TransformerEncoderLayer(128, 2, 256, drop_path_rate=p).train(mode)
            with pytest.raises(ValueError):
                drop_path_scales([layer], 4, "cpu")
            with pytest.raises(ValueError):
                layer.attention_dropout(torch.ones(4, 3))
    # the standalone module multiplies by the same noise the helper draws
    sd = StochasticDepth(0.25, "row").train()
    x = torch.randn(6, 5, 3)
    layer = TransformerEncoderLayer(128, 2, 256, drop_path_rate=0.25).train()
    torch.manual_seed(2)
    y = sd(x)
    torch.manual_seed(2)
    n = drop_path_scales([layer], 6, "cpu")[0][0]
    assert torch.equal(y, x * n.view(6, 1, 1))
    assert sd.eval()(x) is x


# ---------------------------------------------------------------------------------------------------------------------
# the fp32 oracle fed the golden noise, and the training schedules on the emulated kernels
# ---------------------------------------------------------------------------------------------------------------------
def _check_grads(named, rec, bar):
    """named: {name: parameter with .grad}; every gradient the golden records, within `bar` (sampled relative L2 and
    norm); a parameter the golden has no gradient for must have none or a zero one."""
    assert set(rec["names"]) <= set(named)
    for k, (_, r, rn) in zip(rec["names"], DP.sample_errors([named[k].grad for k in rec["names"]], rec)):
        assert r < bar and rn < bar, (k, r, rn)
    for k, p in named.items():
        if k not in rec["names"]:
            assert p.grad is None or p.grad.abs().max().item() == 0.0, k


@pytest.mark.parametrize("name", list(DP.VIT))
def test_oracle_with_golden_noise_matches_reference_vit(gold, name):
    g, c = gold["vit"][name], DP.VIT[name]
    vit = _vit(name)
    keep, _ = _draw_vit(vit, c["B"], c["seed"])
    scales = DP.pair_draws(g["rates"], True, g["noise"])
    sd = {"v." + k: v.detach().clone().requires_grad_(True) for k, v in vit.state_dict().items()}
    images, _ = DP.vit_inputs(name)
    out = DP.vision_encoder(images, sd, DP.vit_cfg(name), p="v", keep=keep, scales=scales)
    (mx, _, rn), = DP.sample_errors([out], {k: v[:1] for k, v in g["outputs"].items()})
    assert mx <= 2e-5 and rn <= 1e-5, (mx, rn)
    (out * DP.upstream(out.shape)).sum().backward()
    assert set(g["grads"]["names"]) == {k[2:] for k, v in sd.items() if v.grad is not None}
    _check_grads({k[2:]: v for k, v in sd.items()}, g["grads"], 1e-4)


@pytest.mark.parametrize("name", ["vit_cls", "vit_nocls"])
def test_vit_training_schedule_with_emulated_kernels(gold, emu, name):
    """VisionTransformer forward + backward (engine_coca_train.VisionTrainRuntime) on the emulated kernels: outputs,
    hidden_states and every parameter gradient against the reference (golden), with the same seed.  (The gathered
    patch-dropping kernels have no CPU emulation: vit_patch_drop runs on the GPU.)"""
    g, c = gold["vit"][name], DP.VIT[name]
    vit = _vit(name)
    images, _ = DP.vit_inputs(name)
    torch.manual_seed(c["seed"])
    out = vit(images)
    assert torch.equal(torch.get_rng_state(), g["rng_after"])
    for _, r, rn in DP.sample_errors([out.last_hidden_state] + list(out.hidden_states), g["outputs"]):
        assert r < 2e-2 and rn < 2e-2, (r, rn)
    (out.last_hidden_state * DP.upstream(out.last_hidden_state.shape)).sum().backward()
    _check_grads(dict(vit.named_parameters()), g["grads"], 5e-2)


@pytest.mark.parametrize("name", [n for n, c in DP.LAYERS.items() if c["grad"]])
def test_standalone_layers_train_with_emulated_kernels(gold, emu, name):
    g, c = gold["layers"][name], DP.LAYERS[name]
    m = _layers(name)
    x = DP.layer_inputs(name).requires_grad_(True)
    torch.manual_seed(c["seed"])
    y = m(x) if c["kind"] == "layer" else m(x, return_hidden_states=True).last_hidden_state
    assert torch.equal(torch.get_rng_state(), g["rng_after"])
    (_, r, rn), = DP.sample_errors([y], {k: v[:1] for k, v in g["outputs"].items()})
    assert r < 2e-2 and rn < 2e-2, (r, rn)
    (y * DP.upstream(y.shape)).sum().backward()
    _check_grads(dict(m.named_parameters()), g["grads"], 5e-2)


@pytest.mark.parametrize("rate,seed", [(0.5, 71), (1.0, 72)])
def test_coca_training_schedule_with_drop_path_against_oracle(emu, rate, seed):
    """coca_small: 2 vision layers without a final LayerNorm, so layer 1 draws (p = rate) and its last MLP branch's
    gradient enters through the scaled cast; at rate 1 both branches of layer 1 are zero for every sample."""
    scales = DP.coca_grad_parity(torch.device("cpu"), "coca_small", rate, None, seed, bar=5e-2)
    assert scales is not None and scales[0] == (None, None) and scales[1][1] is not None
