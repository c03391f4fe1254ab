"""Generates tests/golden/decoder_cache_golden.pt by running the UNMODIFIED reference MultiHeadAttentionWithCache,
TransformerDecoderLayer and TransformerDecoder (imported from /root/reference, build container only) in fp32 on the CPU,
on the cases of tests/decoder_cache_cases.py.

    python tests/golden/make_decoder_cache_golden.py

Stored per case: the inputs, the state-dict keys (the weights are re-created from seeds by the tests) and the result
tensors (output, key / value caches, hidden states).
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle", "iopath_shim"))
sys.path.insert(0, "/root/reference")
sys.path.insert(0, os.path.join(ROOT, "tests"))

from torchmultimodal.modules.layers import multi_head_attention, transformer  # noqa: E402

import decoder_cache_cases as DC  # noqa: E402


def main():
    torch.set_num_threads(8)
    ns = DC.namespace(multi_head_attention, transformer)
    out = {}
    for name in DC.CASES:
        m = DC.build(ns, name)
        inp = DC.inputs(name)
        with torch.no_grad():
            res = {k: v.detach().clone().contiguous() for k, v in DC.run(m, name, inp).items()}
        out[name] = {"inputs": inp, "keys": sorted(m.state_dict()), "results": res}
        print(name, {k: tuple(v.shape) for k, v in res.items()})
    path = os.path.join(HERE, "decoder_cache_golden.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path) / 1e6, "MB")


if __name__ == "__main__":
    main()
