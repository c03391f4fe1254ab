"""Host logic of the benchmarked hot path WITHOUT a GPU: the CLIP towers' fused forward / backward schedule
(engine.ViTTower / TextTower / TransformerStack behind engine.RuntimeFunction) on the emulated kernel contracts
(tests/emu_ops.py) against autograd over the fp32 oracle (oracle/clip_oracle.py) — every parameter gradient.  The kernels
themselves and the full-size step are checked on the GPU (tests/test_gpu_parity.py); this test protects the schedule
(buffer routing, gradient slots, fused bias-gradient sums, gather-mode LayerNorms) on the CPU-only CI leg."""
import pytest
import torch

import emu_ops
import test_gpu_runtime_pinned as P
from oracle import clip_oracle as O


@pytest.fixture()
def emu(monkeypatch):
    emu_ops.install(monkeypatch)


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30)).item()


def test_clip_towers_schedule_against_oracle_with_emulated_kernels(emu):
    from multimodal_b200.models.clip.image_encoder import CLIPViTEncoder
    from multimodal_b200.models.clip.model import CLIP
    from multimodal_b200.models.clip.text_encoder import CLIPTextEncoder

    torch.manual_seed(0)
    m = CLIP(CLIPViTEncoder(64, 16, 64, 128, 2, 2),
             CLIPTextEncoder(embedding_dim=64, vocab_size=512, width=128, dim_feedforward=512, heads=2, layers=2)).train()
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.03 * torch.randn(p.shape, generator=g))
    B = 5
    image = torch.randn(B, 3, 64, 64, generator=g)
    text = torch.randint(1, 500, (B, 77), generator=g)
    text[torch.arange(B), torch.randint(5, 77, (B,), generator=g)] = 511          # EOT = the largest id
    sd = {k: v.detach().clone().requires_grad_(v.is_floating_point()) for k, v in m.state_dict().items()}
    ra, rb = O.clip_forward(image, text, sd, 2, 2)
    wa, wb = torch.randn(ra.shape, generator=g), torch.randn(rb.shape, generator=g)
    ((wa * ra).sum() + (wb * rb).sum()).backward()
    out = m(image, text)
    assert _rel(out.embeddings_a, ra) < 2e-2 and _rel(out.embeddings_b, rb) < 2e-2
    ((wa * out.embeddings_a).sum() + (wb * out.embeddings_b).sum()).backward()
    rows = []
    for k, p in m.named_parameters():
        ref = sd[k].grad
        assert p.grad is not None and torch.isfinite(p.grad).all(), k
        if ref.norm().item() == 0.0:
            assert p.grad.abs().max().item() < 1e-6, k
            continue
        if k.endswith("in_proj_bias"):     # the key third is exactly zero in exact arithmetic: compare q / v thirds
            d = ref.numel() // 3
            rows.append((k + "[q]", _rel(p.grad[:d], ref[:d])))
            rows.append((k + "[v]", _rel(p.grad[2 * d:], ref[2 * d:])))
            continue
        rows.append((k, _rel(p.grad, ref)))
    worst = sorted(rows, key=lambda r: -r[1])[:5]
    print(worst)
    assert len(rows) > 60
    for k, e in rows:
        assert e < 5e-2, (k, e)


def _contrastive_grads(m, image, text):
    """Parameter gradients of the contrastive loss through the modules and autograd."""
    from multimodal_b200.modules.losses.contrastive_loss_with_temperature import ContrastiveLossWithTemperature

    out = m(image, text)
    ContrastiveLossWithTemperature()(out.embeddings_a, out.embeddings_b).backward()
    return {k: p.grad.clone() for k, p in m.named_parameters()}


def _assert_equal_grads(got, ref):
    assert sorted(got) == sorted(ref)
    assert not [k for k in ref if not torch.equal(got[k], ref[k])]


def test_interleaved_forwards_leave_backward_gradients_unchanged(emu):
    """A no_grad forward and a second training forward (other batch sizes) between a training forward and its
    backward: every training forward keeps its activations in its own Workspace, so that backward is unaffected."""
    def grads(interleave):
        m, image, text = P._clip_small()
        w = torch.randn(6, 64, generator=torch.Generator().manual_seed(5))
        out = m(image, text)
        if interleave:
            with torch.no_grad():
                m(image[:2], text[:2])
            m(image[:3], text[:3])
        ((w * out.embeddings_a).sum() + (w * out.embeddings_b).sum()).backward()
        return {k: p.grad for k, p in m.named_parameters()}

    _assert_equal_grads(grads(True), grads(False))


def test_flattened_stores_accumulate_into_grad_views(emu):
    """With the towers' parameters re-homed into flat buffers (as the fused optimizer does), loss.backward() writes the
    gradients in place into the p.grad views of the flat gradient buffer, and re-attaches views that
    zero_grad(set_to_none=True) severed."""
    m, image, text = P._clip_small()
    ref = _contrastive_grads(m, image, text)
    m, image, text = P._clip_small()
    stores = [enc._runtime().store for enc in (m.encoder_a, m.encoder_b)]
    for st in stores:
        st.flatten_()
    for _ in range(2):
        _assert_equal_grads(_contrastive_grads(m, image, text), ref)
        for st in stores:
            assert all(p.grad.data_ptr() == st.grad(p).data_ptr() for p in st.params)
            st.zero_grads()
        m.zero_grad(set_to_none=True)


@pytest.mark.parametrize("micro_batch", [None, 2])
def test_trainer_step_gradients_equal_autograd_path(emu, monkeypatch, micro_batch):
    """ContrastiveTrainer.step drives the same tower runtimes through forward / backward / infer as the modules do under
    autograd: its flat gradients (read where the optimizer would consume them) are the autograd path's, bit for bit
    for the full batch.  In micro-batches the weight gradients are summed slice by slice, a different fp32 summation
    order, and the recomputed embeddings come from GEMMs over fewer rows: equal to 1e-5 relative."""
    from multimodal_b200 import ops
    from multimodal_b200.modules.losses.contrastive_loss_with_temperature import ContrastiveLossWithTemperature
    from multimodal_b200.train import ContrastiveTrainer

    m, image, text = P._clip_small()
    ref = _contrastive_grads(m, image, text)
    m, image, text = P._clip_small()
    tr = ContrastiveTrainer(m, ContrastiveLossWithTemperature())
    seen = {}
    monkeypatch.setattr(ops, "adamw_step", lambda p, g, *a: seen.setdefault(g.data_ptr(), g.clone()))
    tr.step(image, text, micro_batch=micro_batch)
    for prefix, enc, rt in (("encoder_a.", m.encoder_a, tr.img), ("encoder_b.", m.encoder_b, tr.txt)):
        flat = seen[rt.store.g.data_ptr()]
        for k, p in enc.named_parameters():
            o = rt.store.off[id(p)]
            got, want = flat[o:o + p.numel()].view(p.shape), ref[prefix + k]
            if micro_batch is None:
                assert torch.equal(got, want), prefix + k
            else:
                assert _rel(got, want) < 1e-5, (prefix + k, _rel(got, want))
