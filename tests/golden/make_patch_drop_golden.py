"""Generates tests/golden/patch_drop_golden.pt by running the UNMODIFIED reference (imported from /root/reference,
build container only) on the cases of tests/patch_drop_cases.py, on the CPU.

    python tests/golden/make_patch_drop_golden.py

Stored: for `random_masking` / `random_masking_2d` called directly, every output under its seed; for `PatchEmbeddings`
in training mode with a patch_drop_rate (float and tuple, with / without CLS token, with an image_patches_mask), the
parameter checksum, the three output fields and the CPU generator state after the forward; for the tiny CoCa models of
tests/coca_cases.py in training mode with a vision_patch_drop_rate, the three `CoCaModel.forward` tensors.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle", "iopath_shim"))
sys.path.insert(0, "/root/reference")
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

from torchmultimodal.models.coca.coca_model import coca_for_pretraining  # noqa: E402
from torchmultimodal.modules.layers.patch_embedding import PatchEmbeddings  # noqa: E402
from torchmultimodal.modules.masking.random_masking import random_masking, random_masking_2d  # noqa: E402

import patch_drop_cases as PD  # noqa: E402


def main():
    torch.set_num_threads(8)
    out = {"masking": {}, "patch_embed": {}, "coca": {}}
    for name, c in PD.MASKING.items():
        x = PD.masking_input(name)
        torch.manual_seed(c[3])
        if c[0] == "1d":
            r = random_masking(x, c[2])
            rec = {"x": x, "x_masked": r.x_masked, "mask": r.mask, "ids_restore": r.ids_restore, "ids_keep": r.ids_keep}
        else:
            rec = {"x": x, "x_masked": random_masking_2d(x, c[2][0], c[2][1], c[4], c[5])}
        rec["rng_after"] = torch.get_rng_state()
        out["masking"][name] = rec
    for name, c in PD.PATCH_EMBED.items():
        pe = PD.build_patch_embed(PatchEmbeddings, name)
        images, mask = PD.patch_embed_inputs(name)
        torch.manual_seed(c["seed"])
        with torch.no_grad():
            o = pe(images, image_patches_mask=mask)
        out["patch_embed"][name] = {"param_checksum": PD.param_checksum(pe), "embeddings": o.embeddings,
                                    "random_mask": o.random_mask, "ids_restore": o.ids_restore,
                                    "rng_after": torch.get_rng_state()}
    for name, (base, rate, seed) in PD.COCA.items():
        m = PD.build_coca(coca_for_pretraining, name).train()
        inp = PD.CC.inputs(base)
        torch.manual_seed(seed)
        with torch.no_grad():
            mo = m.model(inp["images"], inp["texts"])
        out["coca"][name] = {"param_checksum": PD.param_checksum(m), "image_pooled_output": mo.image_pooled_output,
                             "text_pooled_output": mo.text_pooled_output,
                             "multimodal_embeddings": mo.multimodal_embeddings}
    for part, recs in out.items():
        for name, rec in recs.items():
            print(part, name, {k: tuple(v.shape) for k, v in rec.items() if torch.is_tensor(v)})
    path = os.path.join(HERE, "patch_drop_golden.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path) / 1e6, "MB")


if __name__ == "__main__":
    main()
