"""CPU: the C-ABI shared library loads without a GPU and exports every symbol include/mmb200.h declares."""
import ctypes
import os
import re

from multimodal_b200 import _abi, _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "mmb200.h")).read()
    return sorted(set(re.findall(r"^int (mmb_\w+)\(", src, flags=re.M)))


def test_library_loads_and_exports_header_symbols():
    lib = ctypes.CDLL(str(_lib.LIB_PATH))
    names = _declared()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/mmb200.h but not exported"
    assert lib.mmb_version() >= 100


def test_ctypes_prototypes_cover_header():
    assert sorted(_abi.PROTOTYPES) == _declared()


def test_wgrad_split_heuristic():
    from multimodal_b200.ops import wgrad_splits

    for rows, cols, k in [(768, 3072, 201728), (3072, 768, 201728), (2304, 768, 201728), (768, 768, 201728), (512, 2048, 78848)]:
        s = wgrad_splits(rows, cols, k, n_units=66)     # H100 SXM: 132 SMs = 66 clusters
        tiles = -(-rows // 128) * -(-cols // 128) * s   # 128 x 128 CTA tiles on 132 SMs
        assert tiles >= 88 and s >= 1


def test_host_helpers_wgrad_splits_and_symm_layout():
    """Pure host logic: split-K choice fills >= 90 % of the last wave with the smallest split; the symmetric-buffer
    layout is 256-byte aligned and identical on every rank (peers index it without any exchange of offsets)."""
    import torch

    from multimodal_b200 import ops
    from multimodal_b200.symm import _Slots

    assert ops.wgrad_splits(768, 768, 201728, n_units=66) >= 2                 # 18 tiles cannot fill 66 clusters without split-K
    assert ops.wgrad_splits(8192, 8192, 4096, n_units=66) == 1                 # already >= 2 waves of tiles
    for rows, cols, k in ((768, 3072, 201728), (2304, 768, 201728), (512, 2048, 78848)):
        s = ops.wgrad_splits(rows, cols, k, n_units=66)
        tiles = -(-rows // 256) * -(-cols // 128)
        assert 1 <= s <= 64 and ((k + 63) // 64) // s >= 8
        waves = -(-tiles * s // 66)
        assert tiles * s / (waves * 66) >= 0.9 or s == 1
    B, E = 128, 256
    raw = torch.zeros(_Slots.size(B, E), dtype=torch.uint8)
    sl = _Slots(raw, B, E)
    assert sl.nbytes == _Slots.size(B, E)
    for lst in (sl.a, sl.b, sl.lse_a, sl.lse_b, sl.w):
        assert len(lst) == 2
        for t in lst:
            assert (t.data_ptr() - raw.data_ptr()) % 256 == 0
    assert sl.a[0].shape == (B, E) and sl.w[1].shape == (B,) and sl.flags.numel() == 32
