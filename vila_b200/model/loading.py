"""Checkpoint IO in the reference's three-directory layout (llava_arch.py:158-204; resolved at load
by llava/model/utils/utils.py:25-55):

    <model_dir>/config.json                (top-level LlavaConfig fields)
    <model_dir>/llm/{config.json,*.safetensors}
    <model_dir>/vision_tower/{config.json,*.safetensors}
    <model_dir>/mm_projector/{config.json,*.safetensors}

State-dict prefixes inside the sub-directories follow HF: `model.*` / `lm_head.*` for the LLM,
`vision_model.*` for SigLIP, `layers.*` for the projector.
"""
from __future__ import annotations

import json
from pathlib import Path
from typing import Dict

import torch

from .configuration import LlavaConfig, Qwen2Config, SiglipVisionConfig
from .llava_llama import LlavaLlamaModel


SENTINEL_TOKEN = "<vila/sentinel>"     # llava/constants.py
MEDIA_TOKENS = {"image": "<image>", "video": "<vila/video>"}


def infer_stop_tokens(tok) -> list:
    """llava/utils/tokenizer.py:174-183: the stop tokens are the EOS token plus whatever the chat
    template puts right after an assistant turn — found by rendering a dummy conversation whose
    answers are a sentinel token and reading the token that follows each sentinel."""
    if not hasattr(tok, "sentinel_token"):
        tok.add_tokens([SENTINEL_TOKEN], special_tokens=True)
        tok.sentinel_token = SENTINEL_TOKEN
        tok.sentinel_token_id = tok.convert_tokens_to_ids(SENTINEL_TOKEN)
    turns = []
    for _ in range(10):
        turns += [{"role": "user", "content": "question"}, {"role": "assistant", "content": SENTINEL_TOKEN}]
    ids = tok(tok.apply_chat_template(turns, add_generation_prompt=False, tokenize=False)).input_ids
    stops = {tok.eos_token}
    for here, nxt in zip(ids[:-1], ids[1:]):
        if here == tok.sentinel_token_id:
            stops.add(tok.decode(nxt))
    return list(stops)


def prepare_tokenizer(tok, model_max_length=None, chat_template: str = None):
    """What build_llm_and_tokenizer does to the HF tokenizer after loading it
    (llava/model/language_model/builder.py:187-211): right padding, the model's context length, an
    optional chat template, `stop_tokens` / `stop_token_ids`, and the media tokens registered as
    special tokens with their ids in `media_token_ids` (sentinel first, then <image>, <vila/video> —
    the order fixes the ids of tokens a tokenizer does not have yet)."""
    tok.padding_side = "right"
    if model_max_length is not None:
        tok.model_max_length = model_max_length
    if chat_template is not None:
        tok.chat_template = chat_template.replace("    ", "").replace("\n", "")
    tok.stop_tokens = infer_stop_tokens(tok)
    tok.stop_token_ids = tok.convert_tokens_to_ids(tok.stop_tokens)
    tok.media_tokens = dict(MEDIA_TOKENS)
    tok.media_token_ids = {}
    for name, token in MEDIA_TOKENS.items():
        tok.add_tokens([token], special_tokens=True)
        tok.media_token_ids[name] = tok.convert_tokens_to_ids(token)
    return tok


def _load_dir_tensors(d: Path) -> Dict[str, torch.Tensor]:
    from safetensors.torch import load_file

    out: Dict[str, torch.Tensor] = {}
    files = sorted(d.glob("*.safetensors"))
    if not files:
        bins = sorted(d.glob("*.bin"))
        for b in bins:
            out.update(torch.load(b, map_location="cpu", weights_only=True))
        return out
    for f in files:
        out.update(load_file(str(f)))
    return out


def _pick(cfg: dict, cls):
    fields = {f for f in cls.__dataclass_fields__}
    return cls(**{k: v for k, v in cfg.items() if k in fields})


def config_from_dir(model_dir: Path) -> LlavaConfig:
    top = json.loads((model_dir / "config.json").read_text())
    llm = _pick(json.loads((model_dir / "llm" / "config.json").read_text()), Qwen2Config)
    vis_raw = json.loads((model_dir / "vision_tower" / "config.json").read_text())
    vis = _pick(vis_raw.get("vision_config", vis_raw), SiglipVisionConfig)
    proj = json.loads((model_dir / "mm_projector" / "config.json").read_text())
    kw = {}
    for k in ("mm_vision_select_layer", "mm_vision_select_feature", "image_aspect_ratio", "dynamic_s2",
              "s2_max_split_size", "s2_resize_output_to_scale_idx", "num_video_frames", "video_encoder",
              "min_tiles", "max_tiles", "video_max_tiles",
              "model_max_length", "image_token_id", "video_token_id", "pad_token_id"):
        if k in top and top[k] is not None:
            kw[k] = top[k]
    for k in ("newline_token_ids", "eos_token_ids"):
        if top.get(k) is not None:
            kw[k] = tuple(top[k])
    if top.get("tsp_pool_sizes") is not None:
        kw["tsp_pool_sizes"] = tuple(tuple(p) for p in top["tsp_pool_sizes"])
    if top.get("s2_scales"):
        s = top["s2_scales"]
        kw["s2_scales"] = tuple(int(x) for x in (s.split(",") if isinstance(s, str) else s))
    return LlavaConfig(llm_cfg=llm, vision_tower_cfg=vis,
                       mm_projector_type=proj.get("mm_projector_type", "mlp_downsample"), **kw)


def load_pretrained(model_path: str, device="cuda", model_cls=None, decode_weights: str = "bf16") -> LlavaLlamaModel:
    """decode_weights: "bf16", "fp8" or "w4a16", the weights the single-stream greedy decoder streams
    (Qwen2ForCausalLM.set_decode_weights); the checkpoint and every other path stay bf16."""
    if decode_weights not in ("bf16", "fp8", "w4a16"):
        raise ValueError(f"decode_weights must be 'bf16', 'fp8' or 'w4a16', got {decode_weights!r}")
    d = Path(model_path)
    cfg = config_from_dir(d)
    tok = None
    has_tok_files = any((d / "llm" / f).exists() for f in ("tokenizer.json", "vocab.json",
                                                            "tokenizer_config.json"))
    if has_tok_files:  # a real checkpoint ships the tokenizer next to the LLM
        from transformers import AutoTokenizer
        tok = AutoTokenizer.from_pretrained(str(d / "llm"), padding_side="right", use_fast=True)
        prepare_tokenizer(tok, cfg.model_max_length)
        if max(tok.media_token_ids.values()) >= cfg.llm_cfg.vocab_size:
            raise ValueError(f"media token ids {tok.media_token_ids} do not fit the LLM's {cfg.llm_cfg.vocab_size} "
                             "embedding rows")
        cfg.image_token_id, cfg.video_token_id = tok.media_token_ids["image"], tok.media_token_ids["video"]
        cfg.eos_token_ids = tuple(tok.stop_token_ids)
        if tok.pad_token_id is not None:
            cfg.pad_token_id = tok.pad_token_id
    model = (model_cls or LlavaLlamaModel)(cfg, device=device, tokenizer=tok)
    gc_file = d / "llm" / "generation_config.json"
    if gc_file.exists():  # HF from_pretrained populates model.generation_config from this file
        from types import SimpleNamespace
        gc = {"max_length": 20, "max_new_tokens": None, "do_sample": False, "pad_token_id": None,
              "bos_token_id": None, "eos_token_id": None, "temperature": 1.0, "top_p": 1.0, "top_k": 0}
        gc.update({k: v for k, v in json.loads(gc_file.read_text()).items() if k in gc})
        model.generation_config = SimpleNamespace(**gc)
        model.llm.generation_config = model.generation_config
    sd = {}
    sd.update({"llm." + k: v for k, v in _load_dir_tensors(d / "llm").items()})
    sd.update({"vision_tower.vision_tower." + k: v for k, v in _load_dir_tensors(d / "vision_tower").items()})
    sd.update({"mm_projector." + k: v for k, v in _load_dir_tensors(d / "mm_projector").items()})
    own = model.state_dict()
    if cfg.llm_cfg.tie_word_embeddings and "llm.lm_head.weight" not in sd:
        sd["llm.lm_head.weight"] = sd["llm.model.embed_tokens.weight"]  # tied checkpoints ship one copy
    missing = [k for k in own if k not in sd]
    if missing:
        raise RuntimeError(f"checkpoint {model_path} lacks {len(missing)} tensors, e.g. {missing[:4]}")
    with torch.no_grad():
        for k, p in own.items():
            p.copy_(sd[k].to(p.dtype))
    model.llm.set_decode_weights(decode_weights)
    return model


def save_pretrained(model: LlavaLlamaModel, model_path: str) -> None:
    from dataclasses import asdict

    from safetensors.torch import save_file

    d = Path(model_path)
    parts = {"llm": "llm.", "vision_tower": "vision_tower.vision_tower.", "mm_projector": "mm_projector."}
    sd = model.state_dict()
    for sub, prefix in parts.items():
        (d / sub).mkdir(parents=True, exist_ok=True)
        tensors = {k[len(prefix):]: v.detach().cpu().contiguous() for k, v in sd.items()
                   if k.startswith(prefix)}
        save_file(tensors, str(d / sub / "model.safetensors"))
    (d / "llm" / "config.json").write_text(json.dumps(asdict(model.config.llm_cfg)))
    (d / "vision_tower" / "config.json").write_text(json.dumps(asdict(model.config.vision_tower_cfg)))
    (d / "mm_projector" / "config.json").write_text(
        json.dumps({"mm_projector_type": model.config.mm_projector_type}))
    top = {k: v for k, v in model.config.to_dict().items() if k not in ("llm_cfg", "vision_tower_cfg")}
    (d / "config.json").write_text(json.dumps(top))
