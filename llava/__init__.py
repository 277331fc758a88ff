"""`llava` namespace shim: lets callers written against NVlabs/VILA (`import llava; llava.load(...)`,
`llava.Image`, `llava.model.LlavaLlamaModel`, `python -m llava.cli.infer`) run on the sm_90a hot path of
`vila_b200` unchanged.  Only the names on the hot path's boundary are provided (SURVEY.md §8b); the
reference's training stack, datasets and eval harnesses are out of scope.
Reference: llava/__init__.py, llava/entry.py:29, llava/media.py."""
from .entry import load
from .media import Image, Media, Video

__all__ = ["load", "Image", "Video", "Media"]
