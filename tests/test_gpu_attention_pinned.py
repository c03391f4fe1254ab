"""Pins the fused self-attention kernels (ops.attention_fwd / attention_bwd and their key-mask variants) bit for bit.

Inputs come from a seeded CPU generator, so they are the same on every machine.  The test hashes the bytes of out, lse
and dqkv and compares them with digests recorded on an H100 by ``python tests/test_gpu_attention_pinned.py``, which
prints the table below.  A kernel change that reorders any floating-point operation shows up here as a changed digest;
the parity tests elsewhere only check a tolerance.
"""
import hashlib
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# (name, B, S, H, causal, key mask)
CASES = [
    ("s197", 4, 197, 12, False, False),
    ("s77_causal", 6, 77, 12, True, False),
    ("s224", 3, 224, 12, False, False),
    ("s225", 3, 225, 12, False, False),
    ("s257", 2, 257, 16, False, False),
    ("s1", 3, 1, 2, False, False),
    ("s16_causal", 5, 16, 4, True, False),
    ("s77_kmask", 4, 77, 12, False, True),
]

# sha256 of (out, lse, dqkv), recorded on an H100 80GB HBM3
PINNED = {
    's197': ('0aa36d31559ad2ef5be83831fbe2b55c725a6733b58824c49fec0ec3d65d724b', 'd8bcb896b67bb29caa926f57b2e9beca1a183730dfab2d6310017cc45269c177', 'b4d22f826e0bd667345c283e68fc955ac2e09049e69cc3966039e77608e428bb'),
    's77_causal': ('90ccd73e4183ae489a24c234b1615efd3b83c801d45559181524fb38d1e397bf', '958e1dd95a9a7bc36d04c0262bebe7e09123ea7372e6e02370c67e77568bef8f', '5dbbb30a9c24cac6dcce05bc6517317f1b00439524b9b3fff9093586a3acfd3d'),
    's224': ('6cf2a267c0989dd276dc9ef69bcaa03b0302067627bf462c686e51f19951b315', 'e8140dc5696d976f70c31de5f911abd8124e3b11e3e68a7839aea29ec8096242', '594ee0d2e2646a95f1df1e54b729800749303193448f826ee2f92ff63cc112d9'),
    's225': ('1c8788bd20da7b3454cf5c704dcc84bd0d545e8b9c5ba0ce9f0ae0fcb6c95831', '207eede358578e237fa828c22151888030bf65f832ec34d6785a980e37e03a5b', '5b379bda58a23630b633df9b4ac0cb22c3d34d96da8979605ab2c90bf7017480'),
    's257': ('ca059dc3eee77473eb6f74d47f617059d227522c3d49dd51301dfb5ef40289ae', '3fc8a8ab00f7479297ff6c7e03fb418b409cea382e24b1ff3d62cea19466c28c', 'a05adfc6eff8ebce7a29917c203687e7675fcd66a39a70c3d77b866f5f434c8e'),
    's1': ('050f037834feeed9a02c29d41cc38fc13f8eac472d2af3e87fd5083c50cc44fa', '0e67d47a9892a555022833200b8adfbc74a8ea3d96d3cf3bf42e7e82ea6cb1b8', '750ec76c6b784c0e3bd416c36fa5bc10673bd36c7fedc2513255aa163c0101ca'),
    's16_causal': ('1ebded1758585bc40379d7bda36cc73e1414b023eb0cdc1a77fe0d3e6a103fc4', '74eec291b82280e3ee1971221fb7cc0c0f5c5a3e8e21949b3da49dac0ce64753', '66404fcf7a63d47b97c0d77232478304456a30df903337abecde1510b645b4d9'),
    's77_kmask': ('40c01e60ba842c7a66fb2eb47b8aa4d78d3abae40acdd8a4e08d6eb0412746e5', '5cd340ddec46be40f2074c188fc3b8f58e83b5391962e8a57965ebf3e871db97', 'e8ee266e56e38d0de9fbcda886b3d109e5fea353a786b9ba09806af1a359e598'),
}


def _digest(t):
    return hashlib.sha256(t.detach().cpu().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()


def _run(name, B, S, H, causal, kmask, dev):
    from multimodal_b200 import ops

    d = H * 64
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    qkv = (torch.randn(B * S, 3 * d, generator=g) * 0.7).bfloat16().to(dev)
    dout = (torch.randn(B * S, d, generator=g) * 0.5).bfloat16().to(dev)
    out = torch.empty(B * S, d, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B * H * S, device=dev)
    dqkv = torch.empty_like(qkv)
    if kmask:
        # random holes, a padded tail per sequence, and one sequence with every key masked (its rows get no key)
        m = (torch.rand(B, S, generator=g) > 0.2).to(torch.uint8)
        for b in range(B):
            m[b, S - 9 * b:] = 0
        m[B - 1] = 0
        m = m.to(dev)
        ops.attention_fwd_kmask(qkv, out, lse, m, B, S, H, causal, 0.125)
        ops.attention_bwd_kmask(qkv, out, dout, lse, dqkv, m, B, S, H, causal, 0.125)
    else:
        ops.attention_fwd(qkv, out, lse, B, S, H, causal, 0.125)
        ops.attention_bwd(qkv, out, dout, lse, dqkv, B, S, H, causal, 0.125)
    torch.cuda.synchronize(dev)
    return _digest(out), _digest(lse), _digest(dqkv)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_attention_bit_identical(case):
    dev = torch.device("cuda:0")
    got = _run(*case, dev)
    want = PINNED[case[0]]
    for what, a, b in zip(("out", "lse", "dqkv"), got, want):
        assert a == b, f"{case[0]}: {what} changed"


def record():
    dev = torch.device("cuda:0")
    print("PINNED = {")
    for case in CASES:
        print(f"    {case[0]!r}: {_run(*case, dev)!r},")
    print("}")


if __name__ == "__main__":
    record()
