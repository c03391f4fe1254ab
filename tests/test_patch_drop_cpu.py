"""CPU tests of random patch dropping (PatchEmbeddings(patch_drop_rate=...), FLIP): the index derivation of
multimodal_b200/modules/masking/random_masking.py and the keep-index fp32 oracle pinned to outputs of the unmodified
reference (tests/golden/patch_drop_golden.pt), the builders' argument checks, and what ptxas made of the kernels."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest
import torch

import patch_drop_cases as PD
from oracle import coca_oracle as CO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(os.path.dirname(__file__), "golden", "patch_drop_golden.pt")


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD)


@pytest.mark.parametrize("name", list(PD.MASKING))
def test_random_masking_mirror_matches_reference(gold, name):
    from multimodal_b200.modules.masking.random_masking import random_masking, random_masking_2d

    g, c = gold["masking"][name], PD.MASKING[name]
    x = PD.masking_input(name)
    assert torch.equal(x, g["x"])
    torch.manual_seed(c[3])
    if c[0] == "1d":
        r = random_masking(x, c[2])
        for k in ("x_masked", "mask", "ids_restore", "ids_keep"):
            assert getattr(r, k).dtype == g[k].dtype and torch.equal(getattr(r, k), g[k]), k
    else:
        assert torch.equal(random_masking_2d(x, c[2][0], c[2][1], c[4], c[5]), g["x_masked"])
    assert torch.equal(torch.get_rng_state(), g["rng_after"])


@pytest.mark.parametrize("name", list(PD.PATCH_EMBED))
def test_keep_indices_and_oracle_match_reference_patch_embeddings(gold, name):
    """Same seed: patch_keep_indices draws what the reference's forward draws, and the oracle fed those indices
    reproduces the reference's embeddings."""
    from multimodal_b200.modules.layers.patch_embedding import PatchEmbeddings
    from multimodal_b200.modules.masking.random_masking import patch_keep_indices

    g, c = gold["patch_embed"][name], PD.PATCH_EMBED[name]
    pe = PD.build_patch_embed(PatchEmbeddings, name)
    assert PD.param_checksum(pe) == pytest.approx(g["param_checksum"], rel=1e-12)
    images, mask = PD.patch_embed_inputs(name)
    torch.manual_seed(c["seed"])
    keep, random_mask, ids_restore = patch_keep_indices(pe, images.shape[0], images.device)
    assert torch.equal(torch.get_rng_state(), g["rng_after"])
    assert keep.dtype == torch.int32 and keep.is_contiguous()
    for got, want in ((random_mask, g["random_mask"]), (ids_restore, g["ids_restore"])):
        assert (got is None) == (want is None)
        if want is not None:
            assert got.dtype == want.dtype and torch.equal(got, want)
    sd = {k: v.detach() for k, v in pe.state_dict().items()}
    out = PD.patch_embed(images, sd, "", c["kw"]["patch_size"], keep, mask)
    assert out.shape == g["embeddings"].shape
    assert (out - g["embeddings"]).abs().max().item() <= 2e-5


@pytest.mark.parametrize("name", list(PD.COCA))
def test_keep_oracle_matches_reference_coca_in_training(gold, name):
    from multimodal_b200.models.coca import coca_for_pretraining
    from multimodal_b200.modules.masking.random_masking import patch_keep_indices

    g = gold["coca"][name]
    base, _, seed = PD.COCA[name]
    m = PD.build_coca(coca_for_pretraining, name).train()
    assert PD.param_checksum(m) == pytest.approx(g["param_checksum"], rel=1e-12)
    inp = PD.CC.inputs(base)
    torch.manual_seed(seed)
    keep = patch_keep_indices(m.model.vision_encoder.embeddings, inp["images"].shape[0], "cpu")[0]
    with PD.oracle_keeps(keep):
        out = CO.coca_forward(m.state_dict(), PD.CC.CASES[base]["kwargs"], inp["images"], inp["texts"])
    for k in ("image_pooled_output", "text_pooled_output", "multimodal_embeddings"):
        assert out[k].shape == g[k].shape, k
        assert (out[k] - g[k]).abs().max().item() <= 2e-5, (k, (out[k] - g[k]).abs().max())


def test_builders_accept_rates_and_reject_what_is_not_supported():
    from multimodal_b200.models.coca import coca_for_pretraining
    from multimodal_b200.modules.encoders.vision_transformer import vision_transformer
    from multimodal_b200.modules.layers.patch_embedding import PatchEmbeddings
    from multimodal_b200.modules.masking.random_masking import patch_keep_indices

    for rate in (0.5, 0.75, (0.5, 0.5)):
        vit = vision_transformer(patch_size=4, hidden_dim=32, dim_feedforward=64, n_layer=1, n_head=2, image_size=16,
                                 patch_drop_rate=rate)
        assert vit.embeddings.patch_drop_rate == rate
        PD.build_coca(coca_for_pretraining, "coca_small_r50")
    with pytest.raises(NotImplementedError):
        PatchEmbeddings(image_size=16, patch_size=4, hidden_size=32, hidden_dropout_prob=0.1, patch_drop_rate=0.5)
    pe = PatchEmbeddings(image_size=16, patch_size=4, hidden_size=32, patch_drop_rate=0.95)   # int(16 * 0.05) = 0
    assert patch_keep_indices(pe.eval(), 2, "cpu") is None
    with pytest.raises(AssertionError):
        patch_keep_indices(pe.train(), 2, "cpu")
    pe2 = PatchEmbeddings(image_size=16, patch_size=4, hidden_size=32, patch_drop_rate=(0.8, 0.0))   # int(4 * 0.2) = 0
    with pytest.raises(ValueError):
        patch_keep_indices(pe2.train(), 2, "cpu")


def _nvcc():
    p = shutil.which("nvcc")
    if p is None and os.path.exists("/usr/local/cuda/bin/nvcc"):
        p = "/usr/local/cuda/bin/nvcc"
    return p


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not installed")
def test_patch_drop_kernels_do_not_spill():
    from multimodal_b200 import _lib

    src = os.path.join(ROOT, "multimodal_b200", "csrc", "patch_drop.cu")
    with tempfile.TemporaryDirectory() as td:
        cmd = [_nvcc(), *_lib.NVCC_FLAGS, "-Xptxas", "-v", "-I", os.path.join(ROOT, "multimodal_b200", "csrc"),
               "-I", os.path.join(ROOT, "include"), "-c", src, "-o", os.path.join(td, "patch_drop.o")]
        out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
    log = out.stdout + out.stderr
    props = re.findall(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    names = ("im2col_gather_kernel", "vit_assemble_gather_fwd_kernel", "keep_inverse_kernel",
             "vit_assemble_gather_bwd_rows_kernel", "patch_drop_pos_bwd_kernel")
    for n in names:
        assert any(n in f for f, *_ in props), (n, props)
    for f, frame, st, ld in props:
        assert int(st) == 0 and int(ld) == 0, (f, st, ld)
