"""llava/entry.py:29-55 — `llava.load(model_path, model_base=None, devices=None, **kwargs)`."""
import os
from typing import List, Optional

__all__ = ["load"]


def load(model_path: str, model_base: Optional[str] = None, devices: Optional[List[int]] = None, **kwargs):
    from llava.mm_utils import get_model_name_from_path
    from llava.model.builder import load_pretrained_model
    model_name = get_model_name_from_path(model_path)
    model_path = os.path.expanduser(model_path)
    if os.path.exists(os.path.join(model_path, "model")):
        model_path = os.path.join(model_path, "model")
    if devices is not None:
        assert "max_memory" not in kwargs, "`max_memory` should not be set when `devices` is set"
        kwargs["device"] = f"cuda:{devices[0]}"  # one model replica per GPU: the 8B weights fit one H100
    return load_pretrained_model(model_path, model_name, model_base, **kwargs)[1]
