"""ops.self_attention picks one kernel per (mask, head_dim), the same for the forward and the backward and whatever the
sequence length, so that a module computes the same values under torch.no_grad() and with grad mode on.  The kernel
wrappers are replaced by recorders: no GPU needed."""
import pytest
import torch

from multimodal_b200 import ops

KERNELS = ["attention_fwd", "attention_bwd", "attention_fwd_kmask", "attention_bwd_kmask", "attention_fwd_generic",
           "attention_bwd_generic"]


@pytest.fixture()
def calls(monkeypatch):
    seen = []
    for n in KERNELS:
        monkeypatch.setattr(ops, n, lambda *a, _n=n, **k: seen.append((_n, k.get("head_dim"), k.get("mask"))))
    return seen


@pytest.mark.parametrize("S", [77, 384, 385, 400, 512, 513, 1024])
@pytest.mark.parametrize("hd,mask,want", [(64, None, "attention"), (64, "kmask", "attention_kmask"),
                                         (64, "mask", "attention_generic"), (96, None, "attention_generic"),
                                         (128, None, "attention_generic"), (96, "mask", "attention_generic")])
def test_self_attention_router(calls, S, hd, mask, want):
    B, H = 2, 3
    d = H * hd
    qkv = torch.zeros(B * S, 3 * d, dtype=torch.bfloat16)
    out = torch.zeros(B * S, d, dtype=torch.bfloat16)
    km = torch.ones(B * S, dtype=torch.uint8) if mask == "kmask" else None
    m3 = torch.ones(B, S, S, dtype=torch.uint8) if mask == "mask" else None
    ops.self_attention(qkv, out, None, B, S, H, hd, True, hd ** -0.5, kmask=km, mask=m3)
    ops.self_attention(qkv, out, None, B, S, H, hd, True, hd ** -0.5, kmask=km, mask=m3, dout=out,
                       dqkv=torch.zeros_like(qkv))
    fwd, bwd = want.replace("attention", "attention_fwd"), want.replace("attention", "attention_bwd")
    assert [c[0] for c in calls] == [fwd, bwd]
    if want == "attention_generic":
        assert all(c[1] == hd and c[2] is m3 for c in calls)


def test_self_attention_refuses_two_masks(calls):
    B, S, H = 1, 8, 1
    qkv = torch.zeros(B * S, 192, dtype=torch.bfloat16)
    with pytest.raises(ops.MMBError):
        ops.self_attention(qkv, qkv[:, :64], None, B, S, H, 64, False, 0.125, kmask=torch.ones(S, dtype=torch.uint8),
                           mask=torch.ones(B, S, S, dtype=torch.uint8))
    assert calls == []


@pytest.mark.parametrize("hd", [96, 128])
def test_self_attention_refuses_key_mask_beyond_head_dim_64(calls, hd):
    """The key-masked kernels are 64 wide: a wider head with a key-padding mask is refused, not run on them."""
    B, S, H = 2, 8, 2
    qkv = torch.zeros(B * S, 3 * H * hd, dtype=torch.bfloat16)
    out = torch.zeros(B * S, H * hd, dtype=torch.bfloat16)
    km = torch.ones(B * S, dtype=torch.uint8)
    with pytest.raises(ops.MMBError, match="head_dim 64"):
        ops.self_attention(qkv, out, None, B, S, H, hd, False, hd ** -0.5, kmask=km)
    with pytest.raises(ops.MMBError, match="head_dim 64"):
        ops.self_attention(qkv, out, None, B, S, H, hd, False, hd ** -0.5, kmask=km, dout=out, dqkv=torch.zeros_like(qkv))
    assert calls == []
