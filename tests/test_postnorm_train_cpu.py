"""Post-norm `TransformerEncoderLayer` / `TransformerEncoder` at the reference defaults (ReLU, norm_first=False,
eps 1e-12) on `PostNormLayersRuntime`, WITHOUT a GPU: the kernels are swapped for their torch emulation
(tests/emu_relu_ops.py over tests/emu_drop_path_ops.py and tests/emu_ops.py), and the schedule is checked in both grad
modes against fp32 autograd over the same parameters and against the reference golden (tests/golden/postnorm_golden.pt).
The same schedule on the kernels proper: tests/test_gpu_postnorm_train.py."""
import copy
import os

import pytest
import torch
from torch import nn

import drop_path_cases as DP
import emu_ops
import emu_relu_ops
import postnorm_cases as PN

BF = torch.bfloat16
GOLDEN = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "postnorm_golden.pt"),
                    weights_only=False)


@pytest.fixture()
def emu(monkeypatch):
    from multimodal_b200 import engine_layers

    emu_relu_ops.install(monkeypatch)
    monkeypatch.setattr(engine_layers, "_cuda", lambda t, what: None)


def _ours(name):
    from multimodal_b200.modules.layers.transformer import TransformerEncoder, TransformerEncoderLayer

    return PN.build(TransformerEncoderLayer, TransformerEncoder, name)


def _train_step(m, name, x, mask):
    """Training forward (seeded as the golden's) + backward of <upstream, output>: (output, hidden_states, dx, grads)."""
    x = x.clone().requires_grad_(True)
    torch.manual_seed(PN.CASES[name]["seed"])
    if hasattr(m, "layer"):
        o = m(x, mask, return_hidden_states=True)
        y, hidden = o.last_hidden_state, o.hidden_states
    else:
        y, hidden = m(x, mask), []
    (y * PN.upstream(y.shape)).sum().backward()
    return y, hidden, x.grad, {k: p.grad.clone() for k, p in m.named_parameters()}


def _reference(m, name, x, mask):
    """fp32 autograd over a copy of `m` fed the golden's stochastic-depth noise."""
    ref = copy.deepcopy(m)
    ref.zero_grad(set_to_none=True)
    x = x.clone().requires_grad_(True)
    layers = PN.layers_of(ref)
    scales = DP.pair_draws(DP.layer_rates(layers), ref.training, GOLDEN[name]["noise"])
    y, hidden = PN.ref_forward(ref, x, mask, scales)
    (y * PN.upstream(y.shape)).sum().backward()
    return y, hidden, x.grad, {k: p.grad for k, p in ref.named_parameters()}


_rel_max = PN.rel_max


@pytest.mark.parametrize("name", list(PN.CASES))
def test_postnorm_training_against_fp32_autograd_and_golden(emu, name):
    """Every parameter gradient and the input gradient against fp32 autograd (postnorm_cases.grad_errors, with the ReLU
    bars explained there), and the output, hidden_states and gradients against the reference's own (sampled)
    values."""
    m = _ours(name)
    g = GOLDEN[name]
    assert DP.CC.param_checksum(m) == pytest.approx(g["param_checksum"], rel=1e-6)
    x, mask = PN.inputs(name)
    y, hidden, dx, grads = _train_step(m, name, x, mask)
    assert y.dtype == torch.float32 and y.requires_grad
    ry, rhidden, rdx, rgrads = _reference(m, name, x, mask)
    assert _rel_max(y, ry) < 2e-2
    for h, rh in zip(hidden, rhidden):
        assert _rel_max(h, rh) < 2e-2
    assert sorted(grads) == sorted(rgrads)
    bad = PN.grad_errors(grads, rgrads, bar=PN.RELU_MAX_BAR, l2_bar=PN.SMALL_RELU_L2_BAR)
    assert not bad, bad
    assert not PN.grad_errors({"x": dx}, {"x": rdx}, relu=True)
    # against the reference's sampled values: the FC1 gradients by their norm (their entries are held above), the
    # other gradients, which inherit the FC1 straddles below them, at the width-128 ReLU bar
    names = g["grads"]["names"]
    fc1 = [".feedforward.model.0." in "." + k for k in names]
    for t, rec, bar in (([y] + list(hidden), g["outputs"], 4e-2), ([dx], g["input_grad"], PN.SMALL_RELU_L2_BAR),
                        ([grads[k] for k in names], g["grads"], PN.SMALL_RELU_L2_BAR)):
        for i, (max_err, rel, norm_rel) in enumerate(PN.sample_errors(t, rec)):
            assert norm_rel < 2e-2 and (rec is g["grads"] and fc1[i] or rel < bar), (name, i, max_err, rel, norm_rel)


@pytest.mark.parametrize("name", list(PN.CASES))
def test_postnorm_no_grad_forward_equals_training_forward(emu, name):
    """torch.no_grad() (`infer`: shared scratch, nothing saved) and the training forward compute the same bits, with the
    same stochastic-depth draws under the same seed."""
    m = _ours(name)
    x, mask = PN.inputs(name)

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


def test_postnorm_no_grad_call_between_training_forward_and_backward(emu):
    """A no_grad call (another batch size) between a training forward and its backward leaves that backward's gradients
    unchanged: the backward reads only what its own forward saved."""
    def grads(interleave):
        m = _ours("encoder_final_ln_mask")
        x, mask = PN.inputs("encoder_final_ln_mask")
        x.requires_grad_(True)
        y = m(x, mask).last_hidden_state
        if interleave:
            with torch.no_grad():
                m(torch.randn(2, 9, PN.D))
        (y * PN.upstream(y.shape)).sum().backward()
        return {"x": x.grad, **{k: p.grad for k, p in m.named_parameters()}}

    ref, got = grads(False), grads(True)
    assert sorted(got) == sorted(ref)
    assert not [k for k in ref if not torch.equal(got[k], ref[k])]


def test_postnorm_training_needs_head_dim_64(emu):
    from multimodal_b200._lib import MMBError
    from multimodal_b200.modules.layers.transformer import TransformerEncoderLayer

    m = TransformerEncoderLayer(192, 2, 256)
    with torch.no_grad():
        assert m(torch.randn(2, 5, 192)).shape == (2, 5, 192)
    with pytest.raises(MMBError, match="training needs head_dim 64"):
        m(torch.randn(2, 5, 192))


def test_act_code_relu():
    from multimodal_b200 import ops
    from multimodal_b200._lib import MMBError
    from multimodal_b200.engine import act_code

    assert act_code(nn.ReLU()) == ops.ACT_RELU == emu_relu_ops.ACT_RELU == 2
    assert act_code(nn.GELU()) == ops.ACT_GELU_ERF
    with pytest.raises(MMBError, match="unsupported MLP activation"):
        act_code(nn.GELU(approximate="tanh"))


def test_relu_emulation_contract():
    """The emulated ReLU epilogues: PRE is the plain bf16 GEMM (+ bias) and the second output ReLU(PRE); DACT is the
    plain bf16 GEMM where PRE > 0 and +0 elsewhere, its colsum the column sum of that output; act_bwd selects."""
    g = torch.Generator().manual_seed(3)
    A = torch.randn(70, 48, generator=g).to(BF)
    W = torch.randn(40, 48, generator=g).to(BF)
    bias = torch.randn(40, generator=g)
    plain = emu_ops.gemm(A, W, bias=bias)
    pre, act = emu_relu_ops.gemm(A, W, bias=bias, epilogue=emu_ops.EPI_BF16_ACT, act=2)
    assert torch.equal(pre, plain) and torch.equal(act, torch.relu(plain))
    dY = torch.randn(70, 40, generator=g).to(BF)
    W2 = torch.randn(40, 24, generator=g).to(BF)
    pre2 = torch.randn(70, 24, generator=g).to(BF)
    pre2[0, :4] = torch.tensor([0.0, -0.0, 1e30, -1e30]).to(BF)
    cs = torch.zeros(24)
    out = emu_relu_ops.gemm(dY, W2, b_mn=True, epilogue=emu_ops.EPI_BF16_DACT, aux=pre2, act=2, colsum=cs)
    want = torch.where(pre2.float() > 0, emu_ops.gemm(dY, W2, b_mn=True).float(), torch.zeros(()))
    assert torch.equal(out.float(), want) and torch.equal(cs, want.sum(0))
    assert not torch.signbit(out.float()[pre2.float() <= 0]).any()
    dx = torch.empty_like(pre2)
    emu_relu_ops.act_bwd(out, pre2, dx, 2)
    assert torch.equal(dx, torch.where(pre2.float() > 0, out.float(), torch.zeros(())).to(BF))
    x = torch.tensor([-2.0, -0.0, 0.0, 3.5, 1e30, -1e30])
    assert torch.equal(emu_relu_ops.act_fwd(x, 2), torch.relu(x))
