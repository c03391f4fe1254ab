"""multimodal_b200 — H100-native dual-encoder forward + contrastive-loss hot path of TorchMultimodal."""
__version__ = "0.1.0"


def invalidate_weight_caches() -> None:
    """Force every runtime to re-cast its bf16 operand copies of the fp32 parameters on the next forward.

    Needed only after in-place writes through ``.data`` (``w.data.copy_()``, EMA updates, ``w.data.normal_()``): those do
    not bump the autograd version counter the runtimes watch.  ``load_state_dict``, optimizer steps and ordinary in-place
    ops under ``torch.no_grad()`` are detected automatically."""
    from .engine import invalidate_weight_caches as _inv

    _inv()
