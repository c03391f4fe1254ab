"""Host logic of the FLAVA training runtime at BERT length WITHOUT a GPU: text S = 512 with a key-padding mask and a
multimodal encoder at S = 530, with the kernel wrappers swapped for their torch emulation (tests/emu_ops.py), against
autograd over the fp32 oracle.  The kernels that serve these lengths are checked on the GPU
(tests/test_gpu_attention_long.py)."""
import torch
import pytest

import emu_ops
import test_gpu_attention_long as L   # shared case definition only (its tests carry the gpu marker)
import test_gpu_flava_train as G      # shared helpers only


@pytest.fixture()
def emu(monkeypatch):
    emu_ops.install(monkeypatch)


def test_flava_text_512_padding_mask_training_schedule_with_emulated_kernels(emu):
    inp = L.flava_long_inputs()
    assert inp["text"].shape[1] == 512 and (inp["text"] == 0).any()
    G._grad_parity(torch.device("cpu"), L.flava_long_model(), G._cfg(L.FLAVA_LONG["kwargs"]), inp, "cpu_emu_s512",
                   6e-2)
