"""TEST INFRASTRUCTURE ONLY: torch (CPU) emulation of the contracts of the decoding entry points (include/mmb200.h:
mmb_attention_fwd_decode, mmb_kv_cache_append), next to the emulation of the other kernels in tests/emu_ops.py.
``install(monkeypatch)`` swaps the `multimodal_b200.ops` wrappers for these functions; it is never imported by the
package and is not a fallback.
"""
import torch

from emu_ops import BF, _gen_attn


def attention_fwd_decode(q, k, v, out, *, B, Sq, Skv, H, head_dim, bsq, bsk, bsv, bso, scale, mask=None, mask_bs=0,
                         mask_qs=0, causal=False):
    """Split-KV decode attention: attention_fwd_generic's contract for Sq <= 16, the mask addressed with its strides
    (mask_bs = 0 / mask_qs = 0 broadcast over the batch / the query rows)."""
    assert Sq <= 16
    full = None
    if mask is not None:
        full = torch.as_strided(mask, (B, Sq, Skv), (mask_bs, mask_qs, 1)).contiguous()
    out.copy_(_gen_attn(q.float(), k.float(), v.float(), B, Sq, Skv, H, head_dim, bsq, scale, full, causal).to(BF))


def kv_cache_append(past, new_rows, out, out_bf16, *, B, H, Sp, Sn, head_dim):
    d = H * head_dim
    new = new_rows[:, :d].float().reshape(B, Sn, d)
    cat = new if past is None else torch.cat([past.float().transpose(1, 2).reshape(B, Sp, d), new], 1)
    if out is not None:
        out.view(B, Sp + Sn, d).copy_(cat.to(out.dtype))
    if out_bf16 is not None:
        out_bf16.view(B, Sp + Sn, d).copy_(cat.to(BF))


def install(monkeypatch):
    from multimodal_b200 import ops

    monkeypatch.setattr(ops, "attention_fwd_decode", attention_fwd_decode)
    monkeypatch.setattr(ops, "kv_cache_append", kv_cache_append)
