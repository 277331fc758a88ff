"""vila_b200.model — mirrors the names callers import from `llava.model`."""
from .configuration import (LlavaConfig, Qwen2Config, SiglipVisionConfig, nvila_8b,
                            nvila_8b_dynamic_s2, nvila_lite_3b, nvila_video_8b, tiny_test_config)
from .llava_llama import (BasicImageEncoder, BasicVideoEncoder, LlavaLlamaModel, SyntheticTokenizer,
                          TSPVideoEncoder)
from .modeling_vila import VILAForCausalLM
from .projector import MultimodalProjector
from .qwen2 import GraphDecoder, PagedKVCache, Qwen2ForCausalLM
from .vision import SiglipVisionModel, SiglipVisionTower

__all__ = [n for n in dir() if not n.startswith("_")]
