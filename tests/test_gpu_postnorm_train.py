"""Post-norm `TransformerEncoderLayer` / `TransformerEncoder` on their runtime, and the ReLU activation kind.

* ReLU kernel contracts, by value: the FC1 epilogue (PRE and ReLU(PRE)), the DACT epilogue with its fused bias
  column sum, and the standalone activation kernels.
* Gradients of the post-norm runtime (and of a pre-norm encoder with ReLU) against fp32 autograd and the reference
  golden, at width 128 and at BERT-base shapes; the training forward equal to `infer`.
* MLP and the post-norm decoder layer at their ReLU defaults under no grad.
* No-grad digests of post-norm layers and encoders, recorded on an H100 80GB HBM3 by
  ``python tests/test_gpu_postnorm_train.py`` before the runtime replaced the forward-only layer loop; the runtime's
  `infer` reproduces them bit for bit.
"""
import copy
import hashlib
import os
import sys

import pytest
import torch
import torch.nn.functional as F
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import drop_path_cases as DP  # noqa: E402
import postnorm_cases as PN  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
BF = torch.bfloat16
GOLDEN = torch.load(os.path.join(HERE, "golden", "postnorm_golden.pt"), weights_only=False)


# ---------------------------------------------------------------------------------------------------------------------
# ReLU kernel contracts, by value
# ---------------------------------------------------------------------------------------------------------------------
GEMM_SHAPES = [(128, 256, 64), (136, 264, 72), (1000, 520, 200), (4096, 3072, 768)]   # (M, N, K): tile boundaries


def _special(t):
    """Puts ±0 and ±large entries into the rows / columns of a bf16 operand."""
    t[0] = 0.0
    t[1] = -0.0
    t[2, : t.shape[1] // 2] = 3e4
    t[3, : t.shape[1] // 2] = -3e4
    return t


@pytest.fixture(params=[0, 1], ids=["cta1", "cta2"])
def gemm_mode(request):
    from multimodal_b200 import _lib

    assert _lib.lib().mmb_gemm_set_mode(request.param, 0) == 0
    yield request.param
    _lib.lib().mmb_gemm_set_mode(-1, 0)


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_relu_act_epilogue(gemm_mode, M, N, K):
    """EPI_BF16_ACT with ReLU: PRE is the EPI_BF16 output of the same GEMM with bias, the second output ReLU(PRE)."""
    from multimodal_b200 import ops

    g = torch.Generator().manual_seed(M + N + K)
    A = _special(torch.randn(M, K, generator=g)).to(BF).to(DEV)
    W = torch.randn(N, K, generator=g).to(BF).to(DEV)
    bias = torch.randn(N, generator=g)
    bias[:2] = torch.tensor([0.0, -0.0])
    bias = bias.to(DEV)
    plain = ops.gemm(A, W, bias=bias)
    pre, act = ops.gemm(A, W, bias=bias, epilogue=ops.EPI_BF16_ACT, act=ops.ACT_RELU)
    assert torch.equal(pre, plain)
    assert torch.equal(act, torch.relu(plain))


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_relu_dact_epilogue(gemm_mode, M, N, K):
    """EPI_BF16_DACT with ReLU: the plain EPI_BF16 output where PRE > 0 and +0 elsewhere (PRE = ±0 included), and its
    fused colsum is the column sum of that output."""
    from multimodal_b200 import ops

    g = torch.Generator().manual_seed(3 * M + N + K)
    dY = _special(torch.randn(M, K, generator=g)).to(BF).to(DEV)
    W = torch.randn(K, N, generator=g).to(BF).to(DEV)      # stored [K, N]: the FC2 weight in the backward
    pre = torch.randn(M, N, generator=g)
    pre[:, :4] = torch.tensor([0.0, -0.0, 3e38, -3e38])
    pre = pre.to(BF).to(DEV)
    plain = ops.gemm(dY, W, b_mn=True)
    cs = torch.zeros(N, device=DEV)
    out = ops.gemm(dY, W, b_mn=True, epilogue=ops.EPI_BF16_DACT, aux=pre, act=ops.ACT_RELU, colsum=cs)
    want = torch.where(pre > 0, plain, torch.zeros((), dtype=BF, device=DEV))
    assert torch.equal(out, want)
    assert not torch.signbit(out[pre <= 0].float()).any()
    # the fused sum adds per-128-row-block partials in a fixed order: fp32 rounding of sum|terms| at most
    ref = want.double().sum(0)
    assert ((cs.double() - ref).abs() <= 1e-5 * want.double().abs().sum(0)).all()


def test_relu_standalone_kernels():
    from multimodal_b200 import ops

    g = torch.Generator().manual_seed(9)
    x = torch.randn(100003, generator=g)
    x[:6] = torch.tensor([0.0, -0.0, 3e38, -3e38, 1e-40, -1e-40])
    x = x.to(DEV)
    assert torch.equal(ops.act_fwd(x, ops.ACT_RELU), torch.relu(x))
    dy = torch.randn(100003, generator=g).to(BF).to(DEV)
    pre = x.to(BF)
    dx = torch.empty_like(dy)
    ops.act_bwd(dy, pre, dx, ops.ACT_RELU)
    assert torch.equal(dx, torch.where(pre > 0, dy, torch.zeros((), dtype=BF, device=DEV)))


# ---------------------------------------------------------------------------------------------------------------------
# Gradients against fp32 autograd
# ---------------------------------------------------------------------------------------------------------------------
def _ours(name):
    from multimodal_b200.modules.layers.transformer import TransformerEncoder, TransformerEncoderLayer

    return PN.build(TransformerEncoderLayer, TransformerEncoder, name).to(DEV)


def _golden_scales(name, m):
    """The golden's stochastic-depth noise as drop_path_scales returns it, on the device."""
    pairs = DP.pair_draws(DP.layer_rates(PN.layers_of(m)), m.training, GOLDEN[name]["noise"])
    return [tuple(None if s is None else s.to(DEV).contiguous() for s in p) for p in pairs]


def _step(m, x, mask, up):
    x = x.clone().requires_grad_(True)
    if hasattr(m, "layer"):
        o = m(x, mask, return_hidden_states=True)
        y, hidden = o.last_hidden_state, list(o.hidden_states)
    else:
        y, hidden = m(x, mask), []
    (y * up).sum().backward()
    return y, hidden, x.grad, {k: p.grad.clone() for k, p in m.named_parameters()}


def _ref_step(m, x, mask, up, scales=None, ref_forward=PN.ref_forward):
    ref = copy.deepcopy(m)
    ref.zero_grad(set_to_none=True)
    x = x.clone().requires_grad_(True)
    y, hidden = ref_forward(ref, x, mask, scales)
    (y * up).sum().backward()
    return y, hidden, x.grad, {k: p.grad for k, p in ref.named_parameters()}


@pytest.mark.parametrize("name", list(PN.CASES))
def test_postnorm_grads_against_fp32_autograd_and_golden(monkeypatch, name):
    """Width 128, 2 heads, at the reference defaults: gradients against fp32 autograd over the same parameters (fed the
    golden's stochastic-depth noise), with the ReLU bars of postnorm_cases, and against the reference's sampled
    values."""
    from multimodal_b200 import engine_layers

    m = _ours(name)
    scales = _golden_scales(name, m)
    if m.training:
        monkeypatch.setattr(engine_layers, "drop_path_scales", lambda layers, B, dev: scales)
    x, mask = PN.inputs(name)
    x, mask = x.to(DEV), (None if mask is None else mask.to(DEV))
    up = PN.upstream(x.shape).to(DEV)
    y, hidden, dx, grads = _step(m, x, mask, up)
    ry, rhidden, rdx, rgrads = _ref_step(m, x, mask, up, scales if m.training else None)
    assert PN.rel_max(y, ry) < 2e-2
    assert all(PN.rel_max(h, rh) < 2e-2 for h, rh in zip(hidden, rhidden))
    bad = PN.grad_errors(grads, rgrads, bar=PN.RELU_MAX_BAR, l2_bar=PN.SMALL_RELU_L2_BAR)
    assert not bad, bad
    assert not PN.grad_errors({"x": dx}, {"x": rdx}, relu=True)
    g = GOLDEN[name]
    names = g["grads"]["names"]
    fc1 = [".feedforward.model.0." in "." + k for k in names]
    for t, rec, bar in (([y] + hidden, g["outputs"], 4e-2), ([dx], g["input_grad"], PN.SMALL_RELU_L2_BAR),
                        ([grads[k] for k in names], g["grads"], PN.SMALL_RELU_L2_BAR)):
        for i, (max_err, rel, norm_rel) in enumerate(PN.sample_errors([u.cpu() for u in t], rec)):
            assert norm_rel < 2e-2 and (rec is g["grads"] and fc1[i] or rel < bar), (name, i, max_err, rel, norm_rel)


@pytest.mark.parametrize("S,B", [(128, 16), (512, 4)])
def test_postnorm_bert_base_grads(S, B):
    """d 768, 12 heads, ff 3072, ReLU, eps 1e-12, two layers: every gradient within relative L2 4e-2 and cosine 0.995
    of fp32 autograd, the FC1 gradients within postnorm_cases.BERT_RELU_FC1_L2_BAR."""
    from multimodal_b200.modules.layers.transformer import TransformerEncoder

    torch.manual_seed(0)
    m = TransformerEncoder(2, 768, 12, 3072).to(DEV)
    g = torch.Generator().manual_seed(S)
    x = torch.randn(B, S, 768, generator=g).to(DEV)
    up = torch.randn(B, S, 768, generator=g).to(DEV)
    _, _, dx, grads = _step(m, x, None, up)
    _, _, rdx, rgrads = _ref_step(m, x, None, up)
    bad = PN.grad_errors({**grads, "x": dx}, {**rgrads, "x": rdx}, relu=True)
    bad = {k: e for k, e in bad.items() if ".feedforward.model.0." not in "." + k}
    assert not bad, bad
    fc1 = {k: g for k, g in grads.items() if ".feedforward.model.0." in "." + k}
    bad = PN.grad_errors(fc1, rgrads, l2_bar=PN.BERT_RELU_FC1_L2_BAR)
    assert not bad, bad


def _ref_prenorm(m, x, mask=None, scales=None):
    """A pre-norm TransformerEncoder (transformer.py:95-111) in fp32 on the module's parameters."""
    hidden = [x]
    for layer in m.layer:
        at, mlp = layer.attention, layer.feedforward.model
        B, S, d = x.shape
        ln1, ln2 = layer.attention_layernorm, layer.feedforward_layernorm
        h = F.layer_norm(x, (d,), ln1.weight, ln1.bias, ln1.eps)
        q, k, v = (t.reshape(B, S, at.num_heads, -1).transpose(1, 2)
                   for t in F.linear(h, at.input_proj.weight, at.input_proj.bias).chunk(3, dim=-1))
        o = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, S, d)
        x = x + F.linear(o, at.output_proj.weight, at.output_proj.bias)
        h = F.layer_norm(x, (d,), ln2.weight, ln2.bias, ln2.eps)
        x = x + F.linear(mlp[1](F.linear(h, mlp[0].weight, mlp[0].bias)), mlp[-1].weight, mlp[-1].bias)
        hidden.append(x)
    fln = m.final_layer_norm
    return F.layer_norm(x, (x.shape[-1],), fln.weight, fln.bias, fln.eps), hidden


def test_prenorm_encoder_with_relu_trains():
    """A pre-norm TransformerEncoder with nn.ReLU trains on the pre-norm runtime, through the ReLU epilogues."""
    from multimodal_b200.modules.layers.transformer import TransformerEncoder

    torch.manual_seed(0)
    m = TransformerEncoder(2, 128, 2, 256, activation=nn.ReLU, layer_norm_eps=1e-5, norm_first=True,
                           final_layer_norm_eps=1e-5).to(DEV)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(4, 24, 128, generator=g).to(DEV)
    up = torch.randn(4, 24, 128, generator=g).to(DEV)
    _, _, dx, grads = _step(m, x, None, up)
    _, _, rdx, rgrads = _ref_step(m, x, None, up, ref_forward=_ref_prenorm)
    bad = PN.grad_errors({**grads, "x": dx}, {**rgrads, "x": rdx}, l2_bar=PN.SMALL_RELU_L2_BAR, relu=True)
    assert not bad, bad


@pytest.mark.parametrize("name", list(PN.CASES))
def test_postnorm_training_forward_equals_infer(name):
    m = _ours(name)
    x, mask = PN.inputs(name)
    x, mask = x.to(DEV), (None if mask is None else mask.to(DEV))

    def outputs():
        torch.manual_seed(PN.CASES[name]["seed"])
        if hasattr(m, "layer"):
            o = m(x, mask, return_hidden_states=True)
            return [o.last_hidden_state] + list(o.hidden_states)
        return [m(x, mask)]

    with torch.no_grad():
        ref = [t.clone() for t in outputs()]
    got = outputs()
    assert got[0].requires_grad
    assert all(torch.equal(a.detach(), b) for a, b in zip(got, ref))


# ---------------------------------------------------------------------------------------------------------------------
# Forward-only modules at their ReLU defaults
# ---------------------------------------------------------------------------------------------------------------------
def test_mlp_relu_no_grad():
    from multimodal_b200.modules.layers.mlp import MLP

    torch.manual_seed(0)
    m = MLP(256, 128, 512).to(DEV).eval()
    assert isinstance(m.model[1], nn.ReLU)
    x = torch.randn(6, 40, 256, device=DEV)
    with torch.no_grad():
        got = m(x)
        ref = F.linear(F.relu(F.linear(x, m.model[0].weight, m.model[0].bias)), m.model[-1].weight, m.model[-1].bias)
    assert PN.rel_max(got, ref) < 2e-2


def _ref_mha(at, q_in, kv_in):
    B, Sq, d = q_in.shape
    H = at.num_heads
    q = at.q_proj(q_in).view(B, Sq, H, -1).transpose(1, 2)
    k = at.k_proj(kv_in).view(B, kv_in.shape[1], H, -1).transpose(1, 2)
    v = at.v_proj(kv_in).view(B, kv_in.shape[1], H, -1).transpose(1, 2)
    o = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, Sq, d)
    return at.output_proj(o)


def test_postnorm_decoder_layer_relu_no_grad():
    """A post-norm TransformerDecoderLayer at its defaults (ReLU, cross-attention, eps 1e-12) under no grad against an
    fp32 restatement of transformer.py:430-470."""
    from multimodal_b200.modules.layers.transformer import TransformerDecoderLayer

    torch.manual_seed(0)
    m = TransformerDecoderLayer(128, 2, 256).to(DEV).eval()
    g = torch.Generator().manual_seed(8)
    x = torch.randn(3, 17, 128, generator=g).to(DEV)
    enc = torch.randn(3, 29, 128, generator=g).to(DEV)
    with torch.no_grad():
        got, _ = m(x, enc)
        d = 128
        h = F.layer_norm(x + _ref_mha(m.attention, x, x), (d,), m.attention_layernorm.weight,
                         m.attention_layernorm.bias, m.attention_layernorm.eps)
        h = F.layer_norm(h + _ref_mha(m.cross_attention, h, enc), (d,), m.cross_attention_layernorm.weight,
                         m.cross_attention_layernorm.bias, m.cross_attention_layernorm.eps)
        ff = m.feedforward.model
        ref = F.layer_norm(h + F.linear(F.relu(F.linear(h, ff[0].weight, ff[0].bias)), ff[-1].weight, ff[-1].bias),
                           (d,), m.feedforward_layernorm.weight, m.feedforward_layernorm.bias,
                           m.feedforward_layernorm.eps)
    assert PN.rel_max(got, ref) < 2e-2


# ---------------------------------------------------------------------------------------------------------------------
# No-grad digests
# ---------------------------------------------------------------------------------------------------------------------
def _digest(t: torch.Tensor) -> str:
    t = t.detach().contiguous().reshape(-1)
    return hashlib.sha256(t.cpu().view(torch.uint8).numpy().tobytes()).hexdigest()


# name -> (module kind, input dtype, [B, S, S] mask, final LayerNorm, drop_path_rate in train mode, head_dim)
PIN_CASES = {
    "layer.f32": ("layer", torch.float32, False, False, False, 64),
    "layer.f32.mask": ("layer", torch.float32, True, False, False, 64),
    "layer.bf16.mask": ("layer", torch.bfloat16, True, False, False, 64),
    "layer.hd96.mask": ("layer", torch.float32, True, False, False, 96),
    "layer.drop": ("layer", torch.float32, False, False, True, 64),
    "encoder.f32": ("encoder", torch.float32, False, False, False, 64),
    "encoder.f32.mask": ("encoder", torch.float32, True, False, False, 64),
    "encoder.bf16": ("encoder", torch.bfloat16, False, False, False, 64),
    "encoder.f32.final_ln": ("encoder", torch.float32, True, True, False, 64),
    "encoder.bf16.final_ln": ("encoder", torch.bfloat16, True, True, False, 64),
    "encoder.drop": ("encoder", torch.float32, True, True, True, 64),
}


def _pin_module(name):
    """A post-norm layer or 3-layer encoder with 2 heads of 64 (4 of 96: the LayerNorm kernels take widths that are
    multiples of 128), erf-GELU (an activation the forward-only layer loop could run), eps 1e-12, with perturbed
    weights; an input batch [4, 20, d] and a bool [B, S, S] mask."""
    from multimodal_b200.modules.layers.transformer import TransformerEncoder, TransformerEncoderLayer

    kind, dt, masked, final_ln, drop, hd = PIN_CASES[name]
    heads = 2 if hd == 64 else 4
    d = heads * hd
    torch.manual_seed(0)
    rate = 0.4 if drop else None
    if kind == "layer":
        m = TransformerEncoderLayer(d, heads, 2 * d, activation=torch.nn.GELU, drop_path_rate=rate)
    else:
        m = TransformerEncoder(3, d, heads, 2 * d, activation=torch.nn.GELU,
                               final_layer_norm_eps=1e-5 if final_ln else None, drop_path_rate=rate)
    g = torch.Generator().manual_seed(47)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.03 * torch.randn(p.shape, generator=g))
    x = torch.randn(4, 20, d, generator=g).to(dt)
    mask = None
    if masked:
        mask = torch.rand(4, 20, 20, generator=g) < 0.7
        mask[:, :, 0] = True
    return (m.train() if drop else m.eval()), x, mask


def _pin_outputs(name, dev):
    m, x, mask = _pin_module(name)
    m = m.to(dev)
    x, mask = x.to(dev), (mask.to(dev) if mask is not None else None)
    torch.manual_seed(5)   # the stochastic-depth noise of the train-mode cases
    with torch.no_grad():
        if not hasattr(m, "layer"):
            return {"output": m(x, mask)}
        o = m(x, mask, return_hidden_states=True)
    return {"last_hidden_state": o.last_hidden_state, **{f"hidden_states.{i}": h for i, h in enumerate(o.hidden_states)}}


def pin_digests(name, dev):
    return {k: f"{tuple(t.shape)} {t.dtype} {_digest(t)}" for k, t in sorted(_pin_outputs(name, dev).items())}


PINNED = {
    'layer.f32': {
        'output': '(4, 20, 128) torch.float32 9a96e849d518360b6606e0995a953f983f74ba36866a62bedccd0229c870f342',
    },
    'layer.f32.mask': {
        'output': '(4, 20, 128) torch.float32 8ae45222c28596ae83424e34f492fef3fa0443512c93103c8654e84ca214af3a',
    },
    'layer.bf16.mask': {
        'output': '(4, 20, 128) torch.bfloat16 eb620894d72f7ebd105ccd9f016a4335f8ca05db6b573bb1187322189a67bd35',
    },
    'layer.hd96.mask': {
        'output': '(4, 20, 384) torch.float32 69efa0d9b1c2fbad9607dc30c2f628547c46a22274f1b5e42024fff8f2497dc4',
    },
    'layer.drop': {
        'output': '(4, 20, 128) torch.float32 3264d26ce71d384949ad02383c5b2b69baa79f67806fc2380d26526e4207a8a3',
    },
    'encoder.f32': {
        'hidden_states.0': '(4, 20, 128) torch.float32 ece8e615c1b2978a762e4eb483e10ff6afec5c59f351a124b016e1f31fefdb96',
        'hidden_states.1': '(4, 20, 128) torch.float32 356d8666ad44c347fd8584d1164d4252b0197d24305e4bfc5a699c7c022a7b28',
        'hidden_states.2': '(4, 20, 128) torch.float32 fccb82e2076a21e0cc0d02667a2578fe5266160014bfbac4f067f68f881e8d0a',
        'hidden_states.3': '(4, 20, 128) torch.float32 02617de6fe4dbc4804a18dfd6f134a39277d38b7d268d6811a20d4e2cbf7f424',
        'last_hidden_state': '(4, 20, 128) torch.float32 02617de6fe4dbc4804a18dfd6f134a39277d38b7d268d6811a20d4e2cbf7f424',
    },
    'encoder.f32.mask': {
        'hidden_states.0': '(4, 20, 128) torch.float32 ece8e615c1b2978a762e4eb483e10ff6afec5c59f351a124b016e1f31fefdb96',
        'hidden_states.1': '(4, 20, 128) torch.float32 d3493cd86567fd22548f835639b7049bace31a447e98f0097eddae46f3aa7074',
        'hidden_states.2': '(4, 20, 128) torch.float32 fd93092227a84ef1bb4b179aa2b7f650735490b1597b91606a79b5ae54b878aa',
        'hidden_states.3': '(4, 20, 128) torch.float32 4b0c18d22c62ddd386f68e8e857e49820f385e181630c34b1f52119df73998f4',
        'last_hidden_state': '(4, 20, 128) torch.float32 4b0c18d22c62ddd386f68e8e857e49820f385e181630c34b1f52119df73998f4',
    },
    'encoder.bf16': {
        'hidden_states.0': '(4, 20, 128) torch.bfloat16 dba51e9e9e9a82f89bcd1d9783774343dabd79ee74c8848371c0b4c20c109f40',
        'hidden_states.1': '(4, 20, 128) torch.bfloat16 ca47ccdc631df12e3fe8fc51297cb8ab85828683a3edfa6e1805242293f9455d',
        'hidden_states.2': '(4, 20, 128) torch.bfloat16 23c94819a353a995ce8968c058192d6fb3db3555c222dde48b9cf7fac17bf83b',
        'hidden_states.3': '(4, 20, 128) torch.bfloat16 0734246e9c581ca80c4e4d934a63b1737269ca21ee99f2ebef85815d5ab7b50f',
        'last_hidden_state': '(4, 20, 128) torch.bfloat16 0734246e9c581ca80c4e4d934a63b1737269ca21ee99f2ebef85815d5ab7b50f',
    },
    'encoder.f32.final_ln': {
        'hidden_states.0': '(4, 20, 128) torch.float32 e4ce2fc0b1c62da1eb850df2355df4c675c80ae7bdcb0c74a1faf9486d748bf2',
        'hidden_states.1': '(4, 20, 128) torch.float32 20ee088485c35778b9f0358c643cb7bac566c9248f2ad1e140cfcc8c77cfd3e1',
        'hidden_states.2': '(4, 20, 128) torch.float32 99d230cacdb6b4ff03e1b83287f51e5983759fb3c95faf5cf2f482f38d0e1f9f',
        'hidden_states.3': '(4, 20, 128) torch.float32 0e3d63571e49bb589ed9081b917238cc15b798b36b4c271e4bac9175199dfb5d',
        'last_hidden_state': '(4, 20, 128) torch.float32 5561d5dd4700e1d7fe1e3e97b2b8981d05f4bcc3eeaba815e471a1c437204716',
    },
    'encoder.bf16.final_ln': {
        'hidden_states.0': '(4, 20, 128) torch.bfloat16 6f27105a5abf322cae188802871c39cd8980943aeb2c3846eea94b9cd56f55d6',
        'hidden_states.1': '(4, 20, 128) torch.bfloat16 daa3eb9e63948a61943f675daccc54304db877ceafd3fbcb907de80118012205',
        'hidden_states.2': '(4, 20, 128) torch.bfloat16 c0a4b7a9b8c0d0d3c4e24af0bd3505f56c03a2233cead87dcc2753b8fbb05c70',
        'hidden_states.3': '(4, 20, 128) torch.bfloat16 45b63e39600bb7bbc8c197c6d649e62b9f42bcfead8f60f2dae8793c048515bf',
        'last_hidden_state': '(4, 20, 128) torch.bfloat16 2eeeb305001f977206f30a3d364adecb64bbd72916fbb11811ea278c5522be80',
    },
    'encoder.drop': {
        'hidden_states.0': '(4, 20, 128) torch.float32 e4ce2fc0b1c62da1eb850df2355df4c675c80ae7bdcb0c74a1faf9486d748bf2',
        'hidden_states.1': '(4, 20, 128) torch.float32 20ee088485c35778b9f0358c643cb7bac566c9248f2ad1e140cfcc8c77cfd3e1',
        'hidden_states.2': '(4, 20, 128) torch.float32 ac5a26f6e43edd1d31c28369b5586700f3990269d32934630ba04ddc8a196ce9',
        'hidden_states.3': '(4, 20, 128) torch.float32 85ac49280e8f4d2617d39477d979cd3a983eaa2a98b0cedd24f1fad2611f437e',
        'last_hidden_state': '(4, 20, 128) torch.float32 a358c210843a3c8c09c4309411fc7867335d978c367d652a8d19100c935fda3a',
    },
}


@pytest.mark.parametrize("name", list(PIN_CASES))
def test_postnorm_no_grad_digests(name):
    got = pin_digests(name, torch.device("cuda:0"))
    want = PINNED[name]
    assert sorted(got) == sorted(want), name
    changed = [k for k in want if got[k] != want[k]]
    assert not changed, f"{name}: {changed}"


def record():
    dev = torch.device("cuda:0")
    print("PINNED = {")
    for name in PIN_CASES:
        print(f"    {name!r}: {{")
        for k, v in pin_digests(name, dev).items():
            print(f"        {k!r}: {v!r},")
        print("    },")
    print("}")


if __name__ == "__main__":
    record()
