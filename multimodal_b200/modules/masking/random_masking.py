"""Random patch dropping — drop-in for torchmultimodal/modules/masking/random_masking.py (`random_masking`,
`random_masking_2d`, `RandomMaskingOutput`), and the one place the keep indices of `PatchEmbeddings(patch_drop_rate=...)`
are derived.

The indices come from `torch.rand` and `torch.argsort` with the reference's calls, shapes, device and order, so with the
same seed on the same device the same patches are kept (ties in the noise break as torch's own argsort breaks them) and
the generator advances by the same amount.  The accelerated patch front end consumes only the indices
(`patch_keep_indices`): the kept patches are gathered inside its im2col and token-assembly kernels.  `x_masked` of the
two drop-in functions is the row gather of a caller's tensor that these functions return by contract."""
from typing import Iterable, NamedTuple, Optional, Tuple

import torch
from torch import nn, Tensor


class RandomMaskingOutput(NamedTuple):
    x_masked: Tensor
    mask: Tensor
    ids_restore: Tensor
    ids_keep: Tensor


def _keep_1d(n: int, length: int, mask_ratio: float, device) -> Tuple[Tensor, Tensor, Tensor]:
    """(ids_keep int64 [n, len_keep] in shuffle order, mask float [n, length] with 1 = dropped, ids_restore)."""
    len_keep = int(length * (1 - mask_ratio))
    noise = torch.rand(n, length, device=device)
    assert len_keep >= 1, "must keep at least 1 patch"
    ids_shuffle = torch.argsort(noise, dim=1)
    ids_restore = torch.argsort(ids_shuffle, dim=1)
    mask = (ids_restore >= len_keep).to(torch.float32)
    return ids_shuffle[:, :len_keep], mask, ids_restore


def _keep_2d(n: int, num_patches_h: int, num_patches_w: int, mask_ratio_h: float, mask_ratio_w: float,
             device) -> Tensor:
    """Kept patch indices int64 [n, Lh*Lw]: token i*Lw + j is patch rows[i]*num_patches_w + cols[j], rows and cols
    each in argsort order of their own noise (rows drawn first)."""
    len_keep_h = int(num_patches_h * (1 - mask_ratio_h))
    rows = torch.argsort(torch.rand(n, num_patches_h, device=device), dim=1)[:, :len_keep_h]
    len_keep_w = int(num_patches_w * (1 - mask_ratio_w))
    cols = torch.argsort(torch.rand(n, num_patches_w, device=device), dim=1)[:, :len_keep_w]
    return (rows.unsqueeze(2) * num_patches_w + cols.unsqueeze(1)).reshape(n, len_keep_h * len_keep_w)


def _gather_tokens(x: Tensor, ids_keep: Tensor) -> Tensor:
    return torch.gather(x, dim=1, index=ids_keep.unsqueeze(-1).expand(-1, -1, x.shape[-1]))


def random_masking(x: Tensor, mask_ratio: float) -> RandomMaskingOutput:
    """Per-sample random masking by argsort of uniform noise (MAE, arXiv 2111.06377).  x: [N, L, D]."""
    n, length, _ = x.shape
    ids_keep, mask, ids_restore = _keep_1d(n, length, mask_ratio, x.device)
    return RandomMaskingOutput(x_masked=_gather_tokens(x, ids_keep), mask=mask, ids_restore=ids_restore,
                               ids_keep=ids_keep)


def random_masking_2d(x: Tensor, mask_ratio_h: float, mask_ratio_w: float, num_patches_h: int,
                      num_patches_w: int) -> Tensor:
    """Row / column masking of a [N, num_patches_h * num_patches_w, D] patch grid (Audio-MAE, arXiv 2207.06405)."""
    ids_keep = _keep_2d(x.shape[0], num_patches_h, num_patches_w, mask_ratio_h, mask_ratio_w, x.device)
    return _gather_tokens(x, ids_keep)


def patch_keep_indices(embeddings: nn.Module, batch_size: int,
                       device) -> Optional[Tuple[Tensor, Optional[Tensor], Optional[Tensor]]]:
    """Patch dropping of `PatchEmbeddings` for one batch: None unless the module is training with a patch_drop_rate;
    otherwise (keep int32 [B, L], random_mask or None, ids_restore or None) — the mask and the restore order exist for a
    float rate only, as in the reference.  Draws the same random numbers as the reference's forward."""
    rate = embeddings.patch_drop_rate
    if not embeddings.training or rate is None:
        return None
    if isinstance(rate, Iterable):
        keep = _keep_2d(batch_size, embeddings.num_patches_h, embeddings.num_patches_w, rate[0], rate[1], device)
        if keep.shape[1] == 0:
            raise ValueError(f"patch_drop_rate {tuple(rate)} keeps no patch of the "
                             f"{embeddings.num_patches_h} x {embeddings.num_patches_w} grid")
        mask = ids_restore = None
    else:
        keep, mask, ids_restore = _keep_1d(batch_size, embeddings.num_patches_h * embeddings.num_patches_w, rate,
                                           device)
    return keep.to(torch.int32).contiguous(), mask, ids_restore
