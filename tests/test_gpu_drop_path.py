"""GPU tests of stochastic depth (`drop_path_rate` / `vision_drop_path_rate`): the scaled residual-add + LayerNorm, LayerNorm
backward and cast kernels against their unscaled entry points and float64 sums, the device draws against the
reference's calls, gradients of CoCa and of real-width ViTs against autograd over the fp32 oracle fed the same noise,
exact invariants (dropped samples, p = 1, rate 0, eval, grad-mode invariance), the standalone layers and a short
training run."""
import math

import pytest
import torch

import coca_cases as CC
import drop_path_cases as DP

pytestmark = pytest.mark.gpu

EPS32 = 2.0 ** -24
WIDTHS = [128, 384, 768, 1024]


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _exact_fp32_reference():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _noise(B, p, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    n = torch.empty(B, device=dev).bernoulli_(1 - p, generator=g)
    return n.div_(1 - p) if p < 1 else n


# ---------------------------------------------------------------------------------------------------------------------
# kernel contracts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", WIDTHS)
def test_scaled_add_layernorm_forward(dev, d):
    from multimodal_b200 import ops

    B, S = 7, 33
    M = B * S
    g = torch.Generator(device=dev).manual_seed(d)
    x = torch.randn(M, d, device=dev, generator=g)
    y = torch.randn(M, d, device=dev, generator=g).to(torch.bfloat16)
    gamma, beta = torch.randn(d, device=dev, generator=g), torch.randn(d, device=dev, generator=g)
    s = _noise(B, 0.4, dev, d)
    assert (s == 0).any() and (s != 0).any()

    def run(scale, x_in, yy):
        xo = torch.full((M, d), float("nan"), device=dev)
        ln = torch.empty(M, d, device=dev, dtype=torch.bfloat16)
        lf = torch.empty(M, d, device=dev)
        mean, rstd = torch.empty(M, device=dev), torch.empty(M, device=dev)
        ops.add_layernorm_fwd(x_in, yy, xo, ln, lf, gamma, beta, mean, rstd, M, d, 1e-5, branch_scale=scale,
                              rows_per_scale=S)
        return xo, ln, lf, mean, rstd

    xo, ln, lf, mean, rstd = run(s, x, y)
    rows = s.repeat_interleave(S).view(M, 1)
    assert torch.equal(_bits(xo), _bits(x + rows * y.float()))        # x + fl32(s * y): one product, one add
    dropped = (rows == 0).expand(M, d)
    assert torch.equal(_bits(xo[dropped]), _bits(x[dropped]))
    # the LayerNorm is the unscaled kernel's on the same stream
    for a, b in zip((ln, lf, mean, rstd), run(None, xo.clone(), None)[1:]):
        assert torch.equal(_bits(a), _bits(b))
    # all scales 1: bit-identical to the unscaled entry point
    for a, b in zip(run(torch.ones(B, device=dev), x, y), run(None, x, y)):
        assert torch.equal(_bits(a), _bits(b))
    # float64 LayerNorm of the stream
    xd = xo.double()
    ref = (xd - xd.mean(-1, keepdim=True)) / torch.sqrt(xd.var(-1, unbiased=False, keepdim=True) + 1e-5)
    ref = ref * gamma.double() + beta.double()
    assert ((lf.double() - ref).abs() <= 1e-4 * (1 + ref.abs())).all()


@pytest.mark.parametrize("d", WIDTHS)
def test_scaled_layernorm_backward(dev, d):
    from multimodal_b200 import ops

    B, S = 9, 29
    M = B * S
    g = torch.Generator(device=dev).manual_seed(100 + d)
    x = torch.randn(M, d, device=dev, generator=g)
    dy = torch.randn(M, d, device=dev, generator=g).to(torch.bfloat16)
    gamma = torch.randn(d, device=dev, generator=g)
    gin = torch.randn(M, d, device=dev, generator=g)
    mean, rstd = x.mean(-1), torch.rsqrt(x.var(-1, unbiased=False) + 1e-5)
    s = _noise(B, 0.5, dev, d)

    def run(scale):
        go = torch.empty(M, d, device=dev)
        gb = torch.empty(M, d, device=dev, dtype=torch.bfloat16)
        dg, db, gs = (torch.zeros(d, device=dev) for _ in range(3))
        ops.layernorm_bwd(x, dy, None, mean, rstd, gamma, gin, go, gb, dg, db, M, d, gsum=gs, branch_scale=scale,
                          rows_per_scale=S)
        return go, gb, dg, db, gs

    go, gb, dg, db, gs = run(s)
    go0, gb0, dg0, db0, gs0 = run(None)
    for a, b in ((go, go0), (dg, dg0), (db, db0)):
        assert torch.equal(_bits(a), _bits(b))
    rows = s.repeat_interleave(S).view(M, 1)
    assert torch.equal(_bits(gb), _bits((rows * go).to(torch.bfloat16)))     # bf16(fl32(s * g))
    v = gb.double()
    err = (gs.double() - v.sum(0)).abs()
    assert (err <= (M + 10) * EPS32 * v.abs().sum(0) + 1e-30).all()
    for a, b in zip(run(torch.ones(B, device=dev)), (go0, gb0, dg0, db0, gs0)):
        assert torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize("d", WIDTHS)
def test_scaled_cast(dev, d):
    from multimodal_b200 import ops

    B, S = 5, 17
    x = torch.randn(B * S, d, device=dev, generator=torch.Generator(device=dev).manual_seed(d))
    s = _noise(B, 0.3, dev, d)
    out = ops.cast_bf16(x, branch_scale=s, rows_per_scale=S)
    assert torch.equal(_bits(out), _bits((s.repeat_interleave(S).view(-1, 1) * x).to(torch.bfloat16)))
    assert torch.equal(_bits(ops.cast_bf16(x, branch_scale=torch.ones(B, device=dev), rows_per_scale=S)),
                       _bits(ops.cast_bf16(x)))


# ---------------------------------------------------------------------------------------------------------------------
# draws on the device
# ---------------------------------------------------------------------------------------------------------------------
def test_device_draws_equal_the_reference_calls(dev):
    from multimodal_b200.modules.layers.stochastic_depth import drop_path_scales
    from multimodal_b200.modules.layers.transformer import TransformerEncoder

    enc = TransformerEncoder(4, 128, 2, 256, drop_path_rate=0.6).to(dev).train()
    B = 16
    torch.manual_seed(3)
    got = drop_path_scales(enc.layer, B, dev)
    state = torch.cuda.get_rng_state()
    torch.manual_seed(3)
    for (sa, sf), p in zip(got, torch.linspace(0, 0.6, 4).tolist()):
        if p == 0.0:
            assert sa is None and sf is None
            continue
        for s in (sa, sf):    # torchvision stochastic_depth(input [B, S, d] fp32, p, "row"), restated
            noise = torch.empty([B, 1, 1], dtype=torch.float32, device=dev).bernoulli_(1 - p)
            noise.div_(1 - p)
            assert s.device == noise.device and torch.equal(_bits(s), _bits(noise.view(B)))
    assert torch.equal(torch.cuda.get_rng_state(), state)


# ---------------------------------------------------------------------------------------------------------------------
# gradients against autograd over the fp32 oracle fed the same noise
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rate,patch_rate,seed", [(0.5, None, 41), (0.5, 0.5, 42), (1.0, None, 43)])
def test_coca_gradients_with_drop_path(dev, rate, patch_rate, seed):
    DP.coca_grad_parity(dev, "coca_small", rate, patch_rate, seed)


@pytest.mark.parametrize("tag,image,ps,d,heads,ff,cls,patch_rate", [
    ("vit_l14_w", 224, 14, 1024, 16, 4096, False, None),
    ("vit_l14_w_patch", 224, 14, 1024, 16, 4096, False, 0.75),
    ("vit_b16_w_patch", 224, 16, 768, 12, 3072, True, 0.5),
])
def test_vit_gradients_with_drop_path_at_real_width(dev, tag, image, ps, d, heads, ff, cls, patch_rate):
    from multimodal_b200.modules.encoders.vision_transformer import vision_transformer
    from multimodal_b200.modules.layers.stochastic_depth import drop_path_scales
    from multimodal_b200.modules.masking.random_masking import patch_keep_indices

    torch.manual_seed(0)
    n_layer = 3
    vit = vision_transformer(patch_size=ps, hidden_dim=d, dim_feedforward=ff, n_layer=n_layer, n_head=heads,
                             image_size=image, include_cls_embed=cls, layer_norm_eps=1e-5,
                             final_layer_norm_eps=1e-5 if cls else None, drop_path_rate=0.5,
                             patch_drop_rate=patch_rate)
    g = torch.Generator().manual_seed(13)
    with torch.no_grad():
        for p in vit.parameters():
            p.add_(0.03 * torch.randn(p.shape, generator=g))
    vit = vit.to(dev).train()
    B = 6
    images = torch.randn(B, 3, image, image, generator=g)
    cfg = dict(vision_patch_size=ps, vision_n_layer=n_layer, vision_n_head=heads, vision_layer_norm_eps=1e-5,
               vision_final_layer_norm_eps=1e-5 if cls else None)
    torch.manual_seed(5)
    keep = patch_keep_indices(vit.embeddings, B, dev)
    keep = keep[0].cpu() if keep is not None else None
    scales = [tuple(s.cpu() if s is not None else None for s in pr) for pr in drop_path_scales(vit.encoder.layer, B, dev)]
    sd = {"v." + k: v.detach().cpu().clone().requires_grad_(True) for k, v in vit.state_dict().items()}
    ref = DP.vision_encoder(images, sd, cfg, p="v", keep=keep, scales=scales)
    w = torch.randn(ref.shape, generator=g)
    (ref * w).sum().backward()
    torch.manual_seed(5)
    out = vit(images.to(dev))
    assert DP.rel(out.last_hidden_state.detach().cpu(), ref.detach()) < 2e-2
    (out.last_hidden_state * w.to(dev)).sum().backward()
    DP.check_grads(vit, {k[2:]: v for k, v in sd.items()}, tag)


# ---------------------------------------------------------------------------------------------------------------------
# exact invariants
# ---------------------------------------------------------------------------------------------------------------------
def _coca(dev, **kw):
    from multimodal_b200.models.coca.coca_model import coca_for_pretraining
    return CC.build(lambda **k: coca_for_pretraining(**k, **kw), "coca_small").to(dev)


def _vit(dev, rate, n_layer=4, cls=True):
    from multimodal_b200.modules.encoders.vision_transformer import vision_transformer

    torch.manual_seed(0)
    vit = vision_transformer(patch_size=4, hidden_dim=128, dim_feedforward=256, n_layer=n_layer, n_head=2,
                             image_size=32, include_cls_embed=cls, layer_norm_eps=1e-5, drop_path_rate=rate)
    return DP._perturb(vit).to(dev)


def test_dropped_samples_pass_the_stream_through_unchanged(dev):
    from multimodal_b200.modules.layers.stochastic_depth import drop_path_scales

    vit = _vit(dev, 0.9, n_layer=4).train()
    images = torch.randn(32, 3, 32, 32, device=dev)
    torch.manual_seed(8)
    scales = drop_path_scales(vit.encoder.layer, 32, dev)
    for grad in (False, True):
        torch.manual_seed(8)
        with torch.set_grad_enabled(grad):
            out = vit(images)
        hs = out.hidden_states
        n = 0
        for l, (sa, sf) in enumerate(scales):
            if sa is None:
                continue
            for b in ((sa == 0) & (sf == 0)).nonzero().view(-1).tolist():
                assert torch.equal(hs[l + 1][b], hs[l][b]), (grad, l, b)
                n += 1
        assert n > 0


def test_layer_with_p_one_gets_exactly_zero_gradients(dev):
    vit = _vit(dev, 1.0, n_layer=2).train()        # linspace(0, 1, 2): layer 1 has p = 1
    torch.manual_seed(4)
    out = vit(torch.randn(4, 3, 32, 32, device=dev))
    out.last_hidden_state.square().sum().backward()
    layer1 = vit.encoder.layer[1]
    for k, p in layer1.named_parameters():
        assert p.grad is not None and torch.count_nonzero(p.grad) == 0, k
    assert any(torch.count_nonzero(p.grad) > 0 for p in vit.encoder.layer[0].parameters())


def test_rate_zero_and_eval_are_bit_identical_to_no_rate(dev):
    images = torch.randn(6, 3, 32, 32, device=dev)
    plain = _vit(dev, None).train()
    zero = _vit(dev, 0.0).train()
    drop = _vit(dev, 0.5).eval()
    for grad in (False, True):
        with torch.set_grad_enabled(grad):
            torch.manual_seed(1)
            state = torch.cuda.get_rng_state()
            a = plain(images)
            b = zero(images)
            assert torch.equal(torch.cuda.get_rng_state(), state)
            c = drop(images)
            plain.eval()
            e = plain(images)
            plain.train()
            assert torch.equal(torch.cuda.get_rng_state(), state)
        assert torch.equal(a.last_hidden_state, b.last_hidden_state)
        assert torch.equal(c.last_hidden_state, e.last_hidden_state)
    m0, m1 = _coca(dev).eval(), _coca(dev, vision_drop_path_rate=0.5).eval()
    inp = {k: v.to(dev) for k, v in CC.inputs("coca_small").items()}
    with torch.no_grad():
        state = torch.cuda.get_rng_state()
        x, y = m0.model(inp["images"], inp["texts"]), m1.model(inp["images"], inp["texts"])
        assert torch.equal(torch.cuda.get_rng_state(), state)
    for u, v in zip(x[:3], y[:3]):
        assert torch.equal(u, v)


@pytest.mark.parametrize("patch_rate", [None, 0.5])
def test_no_grad_equals_grad_mode_forward_with_drop_path(dev, patch_rate):
    m = _coca(dev, vision_drop_path_rate=0.5, vision_patch_drop_rate=patch_rate).train()
    inp = {k: v.to(dev) for k, v in CC.inputs("coca_small").items()}
    torch.manual_seed(3)
    with torch.no_grad():
        a = m.model(inp["images"], inp["texts"])
        va = m.model.vision_encoder(inp["images"])
    torch.manual_seed(3)
    b = m.model(inp["images"], inp["texts"])
    vb = m.model.vision_encoder(inp["images"])
    assert b.image_pooled_output.requires_grad
    for x, y in zip(a[:3], b[:3]):
        assert torch.equal(x, y.detach())
    for x, y in zip(va.hidden_states + [va.last_hidden_state], vb.hidden_states + [vb.last_hidden_state]):
        assert torch.equal(x, y.detach())


@pytest.mark.parametrize("name", list(DP.LAYERS))
def test_standalone_layers_against_oracle_with_device_noise(dev, name):
    from multimodal_b200.modules.layers.stochastic_depth import drop_path_scales
    from multimodal_b200.modules.layers.transformer import TransformerEncoder, TransformerEncoderLayer

    c = DP.LAYERS[name]
    m = DP.build_layers(TransformerEncoderLayer, TransformerEncoder, name).to(dev)
    layers = list(m.layer) if hasattr(m, "layer") else [m]
    x = DP.layer_inputs(name)
    torch.manual_seed(c["seed"])
    scales = drop_path_scales(layers, c["B"], dev)
    scales = [tuple(s.cpu() if s is not None else None for s in pr) for pr in scales] if scales else None
    sd = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    if c["kind"] == "layer":
        ref = DP.encoder_layers(x, {"L.0." + k: v for k, v in sd.items()}, "L", 1, DP.HEADS, DP.EPS, scales,
                                c["norm_first"])
    else:
        ref = DP.encoder_layers(x, sd, "layer", c["n_layer"], DP.HEADS, DP.EPS, scales, c["norm_first"])
        ref = DP.CO._ln(ref, sd, "final_layer_norm", DP.EPS)
    torch.manual_seed(c["seed"])
    with torch.set_grad_enabled(c["grad"]):
        y = m(x.to(dev)) if c["kind"] == "layer" else m(x.to(dev)).last_hidden_state
    assert DP.rel(y.detach().cpu(), ref.detach()) < 2e-2
    if c["grad"]:
        w = DP.upstream(ref.shape)
        (ref * w).sum().backward()
        (y * w.to(dev)).sum().backward()
        DP.check_grads(m, sd, name)


# ---------------------------------------------------------------------------------------------------------------------
# training
# ---------------------------------------------------------------------------------------------------------------------
def test_coca_for_pretraining_trains_with_drop_path_and_patch_drop(dev):
    from multimodal_b200.models.coca.coca_model import coca_for_pretraining

    m = CC.build(lambda **kw: coca_for_pretraining(**kw, vision_drop_path_rate=0.1, vision_patch_drop_rate=0.5),
                 "coca_small").to(dev).train()
    inp = {k: v.to(dev) for k, v in CC.inputs("coca_small").items()}
    opt = torch.optim.SGD(m.parameters(), lr=0.02)
    hist = []
    for _ in range(4):
        torch.manual_seed(9)   # the same draws every step: the loss change measures the update, not the draw
        opt.zero_grad(set_to_none=True)
        out = m(inp["images"], inp["texts"])
        total = out["contrastive"] + out["captioning"]
        assert total.requires_grad and math.isfinite(total.item())
        total.backward()
        hist.append(total.item())
        opt.step()
    print("CoCaForPretraining (drop path 0.1, patch drop 0.5) total loss over SGD steps:", hist)
    assert hist[-1] < hist[0], hist
