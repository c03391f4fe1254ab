"""Generates tests/golden/postnorm_golden.pt by running the UNMODIFIED reference `TransformerEncoderLayer` /
`TransformerEncoder` (imported from /root/reference, build container only) at their defaults — ReLU, post-norm,
layer_norm_eps 1e-12 — on the cases of tests/postnorm_cases.py, on the CPU.

    python tests/golden/make_postnorm_golden.py

Stored per case: the parameter checksum, the noise every `StochasticDepth` call drew (in call order, recorded from the
reference's own forward), the output and hidden_states, and for the fixed upstream gradient `postnorm_cases.upstream`
the input gradient and every parameter gradient.  Tensors are stored as their norms and seeded samples of their entries
(`drop_path_cases.sample`), which keeps the file small.
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

from torchmultimodal.modules.layers.transformer import TransformerEncoder, TransformerEncoderLayer  # noqa: E402

import drop_path_cases as DP  # noqa: E402
import postnorm_cases as PN  # noqa: E402


def main():
    torch.set_num_threads(8)
    out = {}
    for name, c in PN.CASES.items():
        m = PN.build(TransformerEncoderLayer, TransformerEncoder, name)
        x, mask = PN.inputs(name)
        x.requires_grad_(True)
        torch.manual_seed(c["seed"])
        with DP.NoiseRecorder() as rec:
            if c["kind"] == "layer":
                y, hidden = m(x, attention_mask=mask), []
            else:
                r = m(x, attention_mask=mask, return_hidden_states=True)
                y, hidden = r.last_hidden_state, [h.detach() for h in r.hidden_states]
        (y * PN.upstream(y.shape)).sum().backward()
        named = [(k, p.grad) for k, p in m.named_parameters()]
        assert all(g is not None for _, g in named)
        out[name] = {"param_checksum": DP.CC.param_checksum(m), "noise": [n.detach().clone() for n in rec.noise],
                     "outputs": PN.sample([y] + hidden, PN.N_OUT),
                     "input_grad": PN.sample([x.grad], PN.N_GRAD),
                     "grads": {"names": [k for k, _ in named], **PN.sample([g for _, g in named], PN.N_GRAD)}}
        print(name, "draws", [tuple(n.shape) for n in rec.noise], "|y|", out[name]["outputs"]["norms"][0])
    path = os.path.join(HERE, "postnorm_golden.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path) / 1e6, "MB")


if __name__ == "__main__":
    main()
