"""Generates tests/golden/drop_path_golden.pt by running the UNMODIFIED reference (imported from /root/reference,
build container only) on the cases of tests/drop_path_cases.py, on the CPU.

    python tests/golden/make_drop_path_golden.py

Stored per case (training mode, drop_path_rate 0.5; `vision_transformer` with / without CLS token and with patch
dropping, a standalone pre-norm `TransformerEncoderLayer`, a post-norm `TransformerEncoder` under no grad, a one-layer
encoder): the parameter checksum, the per-layer p, the noise every `StochasticDepth` call drew (in call order, recorded
from the reference's own forward), the CPU generator state after the forward, the outputs and hidden_states, and — in
grad mode — every parameter gradient for the fixed upstream gradient `drop_path_cases.upstream`.  Outputs and gradients
are stored as their norms and seeded samples of their entries (`drop_path_cases.sample`), which keeps the file small.
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

from torchmultimodal.modules.encoders.vision_transformer import vision_transformer  # noqa: E402
from torchmultimodal.modules.layers.transformer import TransformerEncoder, TransformerEncoderLayer  # noqa: E402

import drop_path_cases as DP  # noqa: E402


def _grads(m):
    named = [(k, p.grad) for k, p in m.named_parameters() if p.grad is not None]
    return {"names": [k for k, _ in named], **DP.sample([g for _, g in named], DP.N_GRAD)}


def main():
    torch.set_num_threads(8)
    out = {"vit": {}, "layers": {}}
    for name, c in DP.VIT.items():
        vit = DP.build_vit(vision_transformer, name)
        images, _ = DP.vit_inputs(name)
        torch.manual_seed(c["seed"])
        with DP.NoiseRecorder() as rec:
            o = vit(images)
        rng_after = torch.get_rng_state()
        (o.last_hidden_state * DP.upstream(o.last_hidden_state.shape)).sum().backward()
        out["vit"][name] = {"param_checksum": DP.CC.param_checksum(vit), "rates": DP.layer_rates(vit.encoder.layer),
                            "noise": [n.detach().clone() for n in rec.noise], "rng_after": rng_after,
                            "outputs": DP.sample([o.last_hidden_state] + list(o.hidden_states), DP.N_OUT),
                            "grads": _grads(vit)}
    for name, c in DP.LAYERS.items():
        m = DP.build_layers(TransformerEncoderLayer, TransformerEncoder, name)
        x = DP.layer_inputs(name)
        torch.manual_seed(c["seed"])
        with torch.set_grad_enabled(c["grad"]), DP.NoiseRecorder() as rec:
            if c["kind"] == "layer":
                y, hidden = m(x), None
            else:
                r = m(x, return_hidden_states=True)
                y, hidden = r.last_hidden_state, [h.detach() for h in r.hidden_states]
        rng_after = torch.get_rng_state()
        if c["grad"]:
            (y * DP.upstream(y.shape)).sum().backward()
        layers = [m] if c["kind"] == "layer" else list(m.layer)
        out["layers"][name] = {"param_checksum": DP.CC.param_checksum(m), "rates": DP.layer_rates(layers),
                               "noise": [n.detach().clone() for n in rec.noise], "rng_after": rng_after,
                               "outputs": DP.sample([y] + (hidden or []), DP.N_OUT),
                               "grads": _grads(m) if c["grad"] else None}
    for part, recs in out.items():
        for name, rec in recs.items():
            print(part, name, "rates", rec["rates"], "draws", [tuple(n.shape) for n in rec["noise"]],
                  "kept", [int((n != 0).sum()) for n in rec["noise"]])
    path = os.path.join(HERE, "drop_path_golden.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path) / 1e6, "MB")


if __name__ == "__main__":
    main()
