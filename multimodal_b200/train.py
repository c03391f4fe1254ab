"""Data-parallel contrastive pre-training step: CLIP forward -> fused loss -> backward -> gradient all-reduce (NCCL,
overlapped with the backward) -> fused AdamW, driven without autograd (the explicit schedules in engine.py).

Mirrors the caller pattern of the reference's only plain-PyTorch loop, examples/flava/native/train.py:263-357
(zero_grad -> autocast forward -> loss -> backward [DDP all-reduce overlaps] -> optimizer.step), with
torch.optim.AdamW's update rule.  One process per GPU; NCCL is used for the gradient all-reduce only.
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.distributed as dist

from . import ops
from ._lib import MMBError
from .engine import ParamStore
from .engine_loss import _dist_state, contrastive_schedule
from .utils.distributed import BackpropType


class _CastBack:
    """Pending bf16 all-reduce whose result is cast back into the fp32 gradient buffer when waited for."""

    def __init__(self, work, src_bf16, dst_f32):
        self.work, self.src, self.dst = work, src_bf16, dst_f32

    def wait(self):
        self.work.wait()
        ops.cast_f32(self.src, self.dst)


class _FlatAdamW:
    def __init__(self, store: ParamStore, lr, betas, eps, weight_decay):
        if store.wb.numel() != store.total:
            raise MMBError("the fused AdamW step writes a bf16 shadow of every parameter (no fp32_only parameters)")
        store.flatten_()
        self.store = store
        self.m = torch.zeros_like(store.master)
        self.v = torch.zeros_like(store.master)
        self.lr, self.betas, self.eps, self.wd = lr, betas, eps, weight_decay
        self.t = 0

    def step(self, grad_scale: float):
        st = self.store
        self.t += 1
        ops.adamw_step(st.master, st.g, self.m, self.v, st.wb, st.total, self.lr, self.betas[0], self.betas[1], self.eps,
                       self.wd, self.t, grad_scale, True)
        st._shadow_fresh = True  # the kernel wrote the bf16 shadow of the updated weights


class ContrastiveTrainer:
    """model: multimodal_b200 CLIP (ViT image tower + text tower); loss_module: ContrastiveLossWithTemperature."""

    def __init__(self, model, loss_module, lr: float = 5e-4, betas=(0.9, 0.98), eps: float = 1e-6,
                 weight_decay: float = 0.2, label_smoothing: float = 0.0,
                 backprop_type: BackpropType = BackpropType.GLOBAL, grad_chunks: int = 3,
                 overlap_allreduce: Optional[bool] = None):
        self.model, self.loss_module = model, loss_module
        self.img = model.encoder_a._runtime()
        self.txt = model.encoder_b._runtime()
        self.world, self.rank = _dist_state()
        self.opt_img = _FlatAdamW(self.img.store, lr, betas, eps, weight_decay)
        self.opt_txt = _FlatAdamW(self.txt.store, lr, betas, eps, weight_decay)
        dev = self.img.store.device
        # logit_scale: a single fp32 scalar with its own (tiny) flat store; no weight decay (CLIP convention)
        self.ls = loss_module.logit_scale
        self.ls_buf = torch.zeros(4, device=dev, dtype=torch.float32)   # [value, pad...] 16 B aligned for the kernels
        self.ls_g = torch.zeros(4, device=dev, dtype=torch.float32)
        self.ls_m = torch.zeros(4, device=dev, dtype=torch.float32)
        self.ls_v = torch.zeros(4, device=dev, dtype=torch.float32)
        self.ls_t = 0
        self.lr, self.betas, self.eps = lr, betas, eps
        self.smoothing = label_smoothing
        self.backprop_type = backprop_type
        self.grad_chunks = max(1, grad_chunks)
        # Gradient all-reduce scheduling.  Default: both flat gradient buffers are reduced right after the backward, so
        # nothing runs beside the GEMMs (NCCL's CTAs would take SMs from the persistent one-CTA-per-SM GEMMs and push
        # their displaced CTAs into a second wave).  MMB_OVERLAP_ALLREDUCE=1 overlaps chunked all-reduces with the image
        # tower's backward instead; which is faster on a given multi-GPU box is not measured here.
        if overlap_allreduce is None:
            import os
            overlap_allreduce = os.environ.get("MMB_OVERLAP_ALLREDUCE", "0") == "1"
        self.overlap_allreduce = bool(overlap_allreduce)
        # MMB_GRAD_ALLREDUCE=bf16: compress the flat gradients to bf16 for the all-reduce (half the NVLink payload; the
        # reduced sum is cast back into the fp32 buffer the optimizer reads).  Default fp32: bit-identical semantics to a
        # single process on the concatenated batch.  Only applies to the non-overlapped schedule.
        import os as _os
        self.allreduce_bf16 = _os.environ.get("MMB_GRAD_ALLREDUCE", "fp32").lower() == "bf16"
        self.tower_streams = _os.environ.get("MMB_TOWER_STREAMS", "0") == "1"   # text tower on a side stream (see step())
        self._side = None
        self._gb = {}
        self._works: List = []
        self.kernel_launches = 0

    # -- gradient all-reduce (NCCL) ------------------------------------------------------------------------
    def _allreduce(self, t: torch.Tensor):
        if self.world > 1:
            if self.allreduce_bf16 and not self.overlap_allreduce and t.numel() >= (1 << 20):
                gb = self._gb.get(t.data_ptr())
                if gb is None or gb.numel() != t.numel():
                    gb = self._gb[t.data_ptr()] = torch.empty(t.numel(), device=t.device, dtype=torch.bfloat16)
                ops.cast_bf16(t, gb)
                work = dist.all_reduce(gb, op=dist.ReduceOp.SUM, async_op=True)
                self._works.append(_CastBack(work, gb, t))
                return
            self._works.append(dist.all_reduce(t, op=dist.ReduceOp.SUM, async_op=True))

    def _layer_boundaries(self, tower) -> List[int]:
        """Flat-buffer offsets at which the layer groups used for chunked all-reduce start."""
        st, layers = tower.store, tower.stack.layers
        L = len(layers)
        idx = sorted({(L * i) // self.grad_chunks for i in range(1, self.grad_chunks)})
        return [st.off[id(next(layers[i].parameters()))] for i in idx if 0 < i < L]

    def step(self, image: torch.Tensor, text: torch.Tensor, micro_batch: Optional[int] = None) -> torch.Tensor:
        """One optimisation step on this rank's batch; returns the (device) loss of this rank.

        micro_batch (optional, must divide the batch): activation recompute for batches whose saved activations do not
        fit the 180 GB of HBM (BASELINE config 4: ViT-L/14 at 4096 pairs per GPU would need ~830 GB).  The contrastive
        loss couples every pair of the GLOBAL batch, so the towers cannot simply be run on slices: pass 1 runs both
        towers slice by slice WITHOUT saving activations and collects the embeddings; the loss and the embedding
        gradients are computed once on the full batch (exactly as in the un-sliced step); pass 2 re-runs each slice with
        saving and back-propagates its rows of the embedding gradient, parameter gradients accumulating in the flat
        buffer.  One extra forward (4/3 of the compute) — the trade the reference's activation checkpointing makes
        (examples/flava/native/train.py:148-165).  Results are identical to the un-sliced step up to fp32 summation
        order."""
        img, txt = self.img, self.txt
        dev = image.device
        f32 = torch.float32
        B = image.shape[0]
        mb = B if micro_batch is None else int(micro_batch)
        if mb <= 0 or B % mb:
            raise MMBError(f"micro_batch {micro_batch} must divide the per-rank batch {B}")
        # reference: logit_scale.data.clamp_ every forward (contrastive_loss_with_temperature.py:193)
        self.ls.data.clamp_(self.loss_module.logit_scale_min, self.loss_module.logit_scale_max)
        self.ls_buf[0:1].copy_(self.ls.data.reshape(1))
        # ---------------- forward ----------------
        # The two towers are independent until the loss.  With tower_streams the text tower runs on a side stream: its
        # LayerNorm / attention / elementwise kernels (HBM- or latency-bound, small smem footprint) then share the SMs
        # with the image tower's persistent GEMM CTAs (bound by the L2 <-> SM path) instead of queueing behind them, and
        # each tower's kernels fill the other's tails.  Only kernels without shared scratch run concurrently (the fused
        # attention backward keeps its statistics in smem; the two-pass kernels share one D buffer -> S <= 256 only).
        S_img = (image.shape[2] // img.ps) * (image.shape[3] // img.ps) + 1   # CLS + patches
        par = self.tower_streams and mb == B and S_img <= 256 and text.shape[1] <= 256
        if par:
            main = torch.cuda.current_stream(dev)
            if self._side is None:
                self._side = torch.cuda.Stream(device=dev)
            side = self._side
            ev = torch.cuda.Event()
            ev.record(main)                      # inputs (and the previous optimizer step) are ordered before the side stream
            with torch.cuda.stream(side):
                side.wait_event(ev)
                (eb,), sb = txt.forward((text,), (), save=txt.ws)
                ev_t = torch.cuda.Event()
                ev_t.record(side)
            (ea,), sa = img.forward((image,), (), save=img.ws)
            main.wait_event(ev_t)
        elif mb == B:
            (ea,), sa = img.forward((image,), (), save=img.ws)
            (eb,), sb = txt.forward((text,), (), save=txt.ws)
        else:
            ea = torch.empty((B, img.E), device=dev, dtype=f32)
            eb = torch.empty((B, txt.E), device=dev, dtype=f32)
            for i in range(0, B, mb):
                img.infer(image[i:i + mb], out=ea[i:i + mb])
                txt.infer(text[i:i + mb], out=eb[i:i + mb])
        E = ea.shape[1]
        na, nb = torch.empty_like(ea), torch.empty_like(eb)
        ia, ib = torch.empty(B, device=dev, dtype=f32), torch.empty(B, device=dev, dtype=f32)
        ops.l2norm_fwd(ea, na, None, ia, B, E)
        ops.l2norm_fwd(eb, nb, None, ib, B, E)
        res = contrastive_schedule(na, nb, self.ls_buf[0:1], self.smoothing, self.backprop_type, False, self.world,
                                   self.rank)
        loss, _, _, _, _, dA, dB, dS = res
        # ---------------- backward ----------------
        dea, deb = torch.empty_like(ea), torch.empty_like(eb)
        ops.l2norm_bwd(dA, na, ia, dea, None, B, E)
        ops.l2norm_bwd(dB, nb, ib, deb, None, B, E)
        self._works = []
        if mb != B:
            for i in range(0, B, mb):                     # pass 2: re-forward with saving, back-propagate the slice
                sb = txt.forward((text[i:i + mb],), (), save=txt.ws)[1]   # the slice's embeddings are not kept
                txt.backward(sb, deb[i:i + mb])
            for i in range(0, B, mb):
                sa = img.forward((image[i:i + mb],), (), save=img.ws)[1]
                img.backward(sa, dea[i:i + mb])
            self._allreduce(txt.store.g)
            self._allreduce(img.store.g)
            bounds = None
        elif par:
            ev = torch.cuda.Event()
            ev.record(main)                      # deb is ready
            with torch.cuda.stream(self._side):
                self._side.wait_event(ev)
                txt.backward(sb, deb)
                ev_t = torch.cuda.Event()
                ev_t.record(self._side)
            img.backward(sa, dea)
            main.wait_event(ev_t)
            self._allreduce(txt.store.g)
            self._allreduce(img.store.g)
            bounds = None
        else:
            txt.backward(sb, deb)
            if self.overlap_allreduce:
                self._allreduce(txt.store.g)              # overlaps with the image tower's backward
            bounds = self._layer_boundaries(img) if (self.world > 1 and self.overlap_allreduce) else []
        if bounds is None:
            pass
        elif bounds:
            st = img.store
            cuts = bounds + [st.total]
            state = {"hi": len(cuts) - 1}

            def on_layer_done(l, _st=st, _cuts=cuts, _state=state, _layers=img.stack.layers):
                # layer l finished: every parameter at or after layer l's first offset that belongs to finished
                # layers is final; flush the highest unfinished chunk when we cross its lower boundary.
                off = _st.off[id(next(_layers[l].parameters()))]
                while _state["hi"] >= 1 and off <= _cuts[_state["hi"] - 1]:
                    lo, hi = _cuts[_state["hi"] - 1], _cuts[_state["hi"]]
                    self._allreduce(_st.g[lo:hi])
                    _state["hi"] -= 1

            img.backward(sa, dea, on_layer_done=on_layer_done)
            self._allreduce(st.g[0:cuts[0]])
        else:
            img.backward(sa, dea)
            if not self.overlap_allreduce:
                self._allreduce(txt.store.g)
            self._allreduce(img.store.g)
        self.ls_g[0:1].copy_(dS.reshape(1))
        self._allreduce(self.ls_g)
        for w in self._works:
            w.wait()
        # ---------------- optimizer ----------------
        gs = 1.0 / self.world
        self.opt_img.step(gs)
        self.opt_txt.step(gs)
        self.ls_t += 1
        ops.adamw_step(self.ls_buf, self.ls_g, self.ls_m, self.ls_v, None, 4, self.lr, self.betas[0], self.betas[1],
                       self.eps, 0.0, self.ls_t, gs, True)
        self.ls.data.copy_(self.ls_buf[0])
        return loss


class HostPrefetcher:
    """Double-buffered host->device staging of (image, text) batches on a side stream, so the H2D copy of step i+1
    overlaps the compute of step i.  `batches` is an iterable of pinned host tensor pairs (all of one shape); two
    persistent device buffer pairs are reused, guarded by events (no allocator traffic in the loop)."""

    def __init__(self, batches, device):
        self.it = iter(batches)
        self.device = device
        self.stream = torch.cuda.Stream(device=device)
        self.bufs = [None, None]          # (img, txt) device buffers
        self.free_ev = [None, None]       # recorded on the compute stream when the buffer's consumer was enqueued
        self.k = 0
        self._next = self._stage()

    def _stage(self):
        try:
            img_h, txt_h = next(self.it)
        except StopIteration:
            return None
        i = self.k & 1
        self.k += 1
        if self.bufs[i] is None:
            self.bufs[i] = (torch.empty(img_h.shape, dtype=img_h.dtype, device=self.device),
                            torch.empty(txt_h.shape, dtype=txt_h.dtype, device=self.device))
        img, txt = self.bufs[i]
        with torch.cuda.stream(self.stream):
            if self.free_ev[i] is not None:
                self.stream.wait_event(self.free_ev[i])   # the step that read this buffer has been fully enqueued+run
            img.copy_(img_h, non_blocking=True)
            txt.copy_(txt_h, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        return img, txt, ev, i

    def __iter__(self):
        return self

    def __next__(self):
        cur = self._next
        if cur is None:
            raise StopIteration
        img, txt, ev, i = cur
        main = torch.cuda.current_stream(self.device)
        main.wait_event(ev)
        if self._prev is not None:                      # the previous batch's step is enqueued on `main` by now
            e = torch.cuda.Event()
            e.record(main)
            self.free_ev[self._prev] = e
        self._prev = i
        self._next = self._stage()                      # H2D of the following batch overlaps this step's kernels
        return img, txt

    _prev = None
