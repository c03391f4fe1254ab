"""Runtime of the contrastive loss with temperature (forward + all gradients in one schedule).

Restates modules/losses/contrastive_loss_with_temperature.py:26-115 + utils/distributed.py:28-58:

  sims_a = A_loc @ B_all^T, sims_b = B_loc @ A_all^T            (wgmma GEMMs, fp32 out; alpha applied in the CE kernel)
  logits = exp(logit_scale) * sims ; CE against labels rank*B + i (+ label smoothing) ; loss = (loss_a + loss_b) / 2
  gradients w.r.t. A_loc, B_loc, logit_scale are produced in the same pass (dsims from the CE kernel, two GEMMs each).

Distributed (world_size > 1): peers' embeddings are read straight out of their CUDA-IPC symmetric buffers by the TMA
producer of the similarity GEMM (multimodal_b200.symm), there is no NCCL all_gather on this path; the GLOBAL
backprop mode needs no gradient reduce-scatter either: each rank rebuilds the gradient that flows into its own
embeddings from its own logits row-block plus the peers' row-LSE vectors (SURVEY.md §5, 'no gradient traffic').

Tiny / unaligned problems (E % 8, B % 8 != 0 — e.g. the reference's 3x5 known-answer test) run the same schedule on
an exact-fp32 SIMT matmul kernel instead of the bf16 tensor-core GEMM.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import ops
from ._lib import MMBError
from .utils.distributed import BackpropType


def _dist_state():
    if torch.distributed.is_available() and torch.distributed.is_initialized():
        return torch.distributed.get_world_size(), torch.distributed.get_rank()
    return 1, 0


class ContrastiveFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b, logit_scale, smoothing, backprop_type, want_logits, mask=None):
        if a.shape != b.shape or a.dim() != 2:
            raise MMBError(f"contrastive loss expects two [B, E] tensors, got {tuple(a.shape)} and {tuple(b.shape)}")
        from .engine import _require_cuda

        for t in (a, b, logit_scale):    # the one device guard of the runtimes (no CPU path)
            _require_cuda(t.device)
        world, rank = _dist_state()
        a32 = a.detach().contiguous().float()
        b32 = b.detach().contiguous().float()
        s32 = logit_scale.detach().reshape(1).float().contiguous()
        res = contrastive_schedule(a32, b32, s32, smoothing, backprop_type, want_logits, world, rank, mask)
        loss, logits_a, logits_b, loss_a, loss_b, dA, dB, dS = res
        ctx.save_for_backward(dA, dB, dS)
        ctx.in_dtypes = (a.dtype, b.dtype, logit_scale.dtype, logit_scale.shape)
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(logits_a, logits_b)
        return loss, logits_a, logits_b, loss_a, loss_b

    @staticmethod
    def backward(ctx, g_loss, g_la, g_lb, g_lossa, g_lossb):
        if g_lossa is not None or g_lossb is not None:
            raise MMBError("only ContrastiveLossOutput.loss is differentiable in the fused loss (loss_a / loss_b are "
                           "reported values)")
        dA, dB, dS = ctx.saved_tensors
        da_t, db_t, ds_t, s_shape = ctx.in_dtypes
        if g_loss is None:
            return None, None, None, None, None, None, None
        g = g_loss.float()
        return (dA * g).to(da_t), (dB * g).to(db_t), (dS * g).reshape(s_shape).to(ds_t), None, None, None, None


def _tensor_path_ok(B: int, N: int, E: int) -> bool:
    return E % 8 == 0 and B % 8 == 0 and N % 8 == 0 and B >= 64 and E >= 64


def contrastive_schedule(a, b, s, smoothing, backprop_type, want_logits, world, rank, mask=None):
    """Forward + all gradients of the contrastive loss for this rank's [B, E] embeddings (fp32, CUDA).

    world == 1 follows contrastive_loss_with_temperature.py:31-33 (labels = arange(B), no communication).
    world  > 1: every rank publishes bf16 embeddings + row-LSE vectors in its symmetric buffer (symm.py); peers read
    them in place — the similarity / gradient GEMMs take the peer tensors as their TMA operands.
    mask (optional bool [B]): the reference keeps only the masked rows of both logit matrices and of the labels before
    the mean cross-entropy (contrastive_loss_with_temperature.py:97-100).  Here it becomes per-row weights
    mask_i / count(mask) of the mean; in GLOBAL mode the peers' weights travel with their row-LSE vectors.
    Returns (loss, logits_a, logits_b, loss_a, loss_b, dA, dB, dlogit_scale)."""
    from .symm import get_comm

    dev = a.device
    B, E = a.shape
    N = B * world
    f32, bf = torch.float32, torch.bfloat16
    tensor_path = _tensor_path_ok(B, N, E)
    if world > 1 and not tensor_path:
        raise MMBError(f"distributed contrastive loss needs B % 8 == 0, E % 8 == 0, B >= 64 (got B={B}, E={E})")
    RLA, RLB = torch.empty(B, device=dev, dtype=f32), torch.empty(B, device=dev, dtype=f32)
    dS = ops.zero_(torch.empty(1, device=dev, dtype=f32))
    logits_a = torch.empty((B, N), device=dev, dtype=f32) if want_logits else None
    logits_b = torch.empty((B, N), device=dev, dtype=f32) if want_logits else None
    out = torch.empty(3, device=dev, dtype=f32)
    lab = rank * B
    dist_on = torch.distributed.is_available() and torch.distributed.is_initialized()
    if backprop_type == BackpropType.GLOBAL or not dist_on:
        # no process group: _gather_embeddings_and_labels returns the live tensors whatever backprop_type says
        # (contrastive_loss_with_temperature.py:31-33), so the full gradient flows; an INITIALISED world of one rank
        # does go through gather_tensor and honours LOCAL / NONE (utils/distributed.py:50-58)
        lo, hi = 0, N
    elif backprop_type == BackpropType.LOCAL:
        lo, hi = lab, lab + B
    else:
        lo, hi = 0, 0
    # Fused path (default whenever the caller does not ask for the logits): the similarity GEMMs consume their
    # accumulators in the epilogue (online-softmax statistics forward, d loss / d sims backward) and fp32 logits are
    # never written to HBM — 1 GiB at BASELINE config 4.  want_logits keeps the materialising schedule.
    fused = tensor_path and not want_logits
    SA = SB = None
    if not fused:
        SA = torch.empty((B, N), device=dev, dtype=f32)
        SB = torch.empty((B, N), device=dev, dtype=f32)
    RW = CW = None
    if mask is not None:
        if mask.shape != (B,):
            raise ValueError(f"mask must have shape [{B}], got {tuple(mask.shape)}")
        mb = mask.to(device=dev).bool()
        RW = mb.to(f32) / mb.sum().to(f32)   # [B] scalars: plumbing (0/0 -> nan, as the reference's empty mean)
    if tensor_path:
        comm = get_comm(B, E, dev, world)
        p = comm.step % 2
        comm.step += 1
        my = comm.my
        ops.cast_bf16(a, my.a[p])
        ops.cast_bf16(b, my.b[p])
        if RW is not None:
            my.w[p].copy_(RW)
        comm.barrier()                                    # peers' embeddings are readable
        if fused:
            npp = ops.gemm_ce_num_parts(B)                # float4 partials per row and per-peer launch
            PA = torch.empty((B, world * npp, 4), device=dev, dtype=f32)
            PB = torch.empty((B, world * npp, 4), device=dev, dtype=f32)
            XA, XB = torch.empty(B, device=dev, dtype=f32), torch.empty(B, device=dev, dtype=f32)
            for r in range(world):                        # one launch per peer: its B operand is the peer's buffer
                ops.gemm_ce_stats(my.a[p], comm.slots[r].b[p], s, lab - r * B, PA, r * npp, XA)
                ops.gemm_ce_stats(my.b[p], comm.slots[r].a[p], s, lab - r * B, PB, r * npp, XB)
            ops.ce_stats_reduce(PA, world * npp, XA, B, N, smoothing, 0.5, RW, RLA, my.lse_a[p], dS)
            ops.ce_stats_reduce(PB, world * npp, XB, B, N, smoothing, 0.5, RW, RLB, my.lse_b[p], dS)
        else:
            for r in range(world):                        # TMA loads of the B operand read peer r's buffer in place
                ops.gemm(my.a[p], comm.slots[r].b[p], epilogue=ops.EPI_F32, out=SA[:, r * B:(r + 1) * B])
                ops.gemm(my.b[p], comm.slots[r].a[p], epilogue=ops.EPI_F32, out=SB[:, r * B:(r + 1) * B])
            ops.contrastive_ce_stats(SA, s, B, N, lab, smoothing, 0.5, RLA, my.lse_a[p], dS, logits_a, RW)
            ops.contrastive_ce_stats(SB, s, B, N, lab, smoothing, 0.5, RLB, my.lse_b[p], dS, logits_b, RW)
        LA = LB = None
        if hi > lo:
            if world > 1:
                comm.barrier()                            # peers' row-LSE vectors are readable
                LA, LB = torch.empty(N, device=dev, dtype=f32), torch.empty(N, device=dev, dtype=f32)
                for r in range(world):                    # 2*world copies of B floats (peer reads)
                    LA[r * B:(r + 1) * B].copy_(comm.slots[r].lse_a[p])
                    LB[r * B:(r + 1) * B].copy_(comm.slots[r].lse_b[p])
                if RW is not None:                        # every rank passes a mask or none does (same call site)
                    CW = torch.empty(N, device=dev, dtype=f32)
                    for r in range(world):
                        CW[r * B:(r + 1) * B].copy_(comm.slots[r].w[p])
            else:
                LA, LB, CW = my.lse_a[p], my.lse_b[p], RW
        DSA = torch.empty((B, N), device=dev, dtype=bf)
        DSB = torch.empty((B, N), device=dev, dtype=bf)
        if fused:
            for r in range(world):                        # recompute the logits tile, emit d loss / d sims directly
                c0 = r * B
                clo, chi = min(max(lo - c0, 0), B), min(max(hi - c0, 0), B)
                sl = slice(c0, c0 + B)
                ops.gemm_ce_grad(my.a[p], comm.slots[r].b[p], s, lab - c0, N, B, smoothing, 0.5, my.lse_a[p], RW,
                                 LB[sl] if (LB is not None and chi > clo) else None, CW[sl] if CW is not None else None,
                                 clo, chi, DSA[:, sl])
                ops.gemm_ce_grad(my.b[p], comm.slots[r].a[p], s, lab - c0, N, B, smoothing, 0.5, my.lse_b[p], RW,
                                 LA[sl] if (LA is not None and chi > clo) else None, CW[sl] if CW is not None else None,
                                 clo, chi, DSB[:, sl])
        else:
            ops.contrastive_ce_grad(SA, s, B, N, lab, smoothing, 0.5, my.lse_a[p], LB, lo, hi, DSA, None, RW, CW)
            ops.contrastive_ce_grad(SB, s, B, N, lab, smoothing, 0.5, my.lse_b[p], LA, lo, hi, DSB, None, RW, CW)
        dA = torch.empty((B, E), device=dev, dtype=f32)
        dB = torch.empty((B, E), device=dev, dtype=f32)
        for r in range(world):
            ops.gemm(DSA[:, r * B:(r + 1) * B], comm.slots[r].b[p], b_mn=True, epilogue=ops.EPI_F32, out=dA,
                     accumulate=r > 0)
            ops.gemm(DSB[:, r * B:(r + 1) * B], comm.slots[r].a[p], b_mn=True, epilogue=ops.EPI_F32, out=dB,
                     accumulate=r > 0)
    else:  # exact-fp32 SIMT path (single process, tiny / unaligned shapes)
        ops.matmul_f32(a, b, tb=True, out=SA)
        ops.matmul_f32(b, a, tb=True, out=SB)
        La, Lb = torch.empty(B, device=dev, dtype=f32), torch.empty(B, device=dev, dtype=f32)
        ops.contrastive_ce_stats(SA, s, B, N, 0, smoothing, 0.5, RLA, La, dS, logits_a, RW)
        ops.contrastive_ce_stats(SB, s, B, N, 0, smoothing, 0.5, RLB, Lb, dS, logits_b, RW)
        DSA = torch.empty((B, N), device=dev, dtype=f32)
        DSB = torch.empty((B, N), device=dev, dtype=f32)
        ops.contrastive_ce_grad(SA, s, B, N, 0, smoothing, 0.5, La, Lb if hi > lo else None, lo, hi, None, DSA, RW, RW)
        ops.contrastive_ce_grad(SB, s, B, N, 0, smoothing, 0.5, Lb, La if hi > lo else None, lo, hi, None, DSB, RW, RW)
        dA = ops.matmul_f32(DSA, b)
        dB = ops.matmul_f32(DSB, a)
    ops.sum_scale(RLA, B, 1.0 / B, out[1:2])
    ops.sum_scale(RLB, B, 1.0 / B, out[2:3])
    ops.sum_scale(RLA, B, 0.5 / B, out[0:1])
    ops.sum_scale(RLB, B, 0.5 / B, out[0:1], accumulate=True)
    empty = torch.empty(0, device=dev, dtype=f32)
    if mask is not None and want_logits:   # the reference returns the row-selected logits (:98-99)
        logits_a, logits_b = logits_a[mb], logits_b[mb]
    return (out[0], logits_a if want_logits else empty, logits_b if want_logits else empty, out[1], out[2], dA, dB,
            dS.reshape(()))


def _single_process(a, b, s, smoothing, want_logits):
    return contrastive_schedule(a, b, s, smoothing, BackpropType.GLOBAL, want_logits, 1, 0)


def contrastive_loss_apply(embeddings_a, embeddings_b, logit_scale, smoothing: float,
                           backprop_type: BackpropType = BackpropType.GLOBAL, mask: Optional[torch.Tensor] = None,
                           want_logits: bool = False) -> Tuple[torch.Tensor, ...]:
    return ContrastiveFunction.apply(embeddings_a, embeddings_b, logit_scale, float(smoothing), backprop_type,
                                     bool(want_logits), mask)
