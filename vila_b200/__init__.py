"""vila_b200 — H100-native (sm_90a) implementation of the VILA multimodal forward hot path.

`vila_b200.model.LlavaLlamaModel` keeps the reference's `llava.model` API; every GPU op goes through
the C-ABI in include/vila_b200.h (libvila_b200.so, built in-tree by `python -m vila_b200.build`).
"""
__version__ = "0.1.0"


def load(model_path=None, config=None, device="cuda", seed=0):
    """`llava.load` analogue (llava/entry.py:13-38).  Without a checkpoint directory the named
    architecture is random-initialised (there is no network / checkpoint in this environment)."""
    from .model import LlavaLlamaModel, nvila_8b
    from .model.loading import load_pretrained

    if model_path is not None:
        return load_pretrained(model_path, device=device)
    return LlavaLlamaModel(config or nvila_8b(), device=device).init_random(seed)
