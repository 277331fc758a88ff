"""LlavaLlamaModel — drop-in mirror of the reference VLM wrapper on the sm_90a kernels.

Reference surface kept (SURVEY.md §8b):
  class LlavaLlamaModel                       llava/model/language_model/llava_llama.py:41-163
  LlavaMetaModel.encode_images / merge_*      llava/model/llava_arch.py:255-394
  LlavaMetaForCausalLM._embed / generate / generate_content / default_generation_config   :412-555,823-963
  BasicImageEncoder / BasicVideoEncoder / TSPVideoEncoder    llava/model/encoders/**
Attributes: .llm .vision_tower .mm_projector .tokenizer .encoders .config, get_llm() /
get_vision_tower() / get_mm_projector() / get_lm_head().
What changes underneath: every tensor op is a call into libvila_b200.so; the text/media splice is one
gather kernel driven by a host-built index table (the reference syncs the device once per token,
llava_arch.py:463,470); dynamic-S2 stitching is one kernel per image.
"""
from __future__ import annotations

import copy
import gc
from collections import defaultdict, deque
from types import SimpleNamespace
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

import torch
from torch import nn

from .. import ops
from .configuration import LlavaConfig
from .projector import MultimodalProjector
from .qwen2 import Qwen2ForCausalLM, sampling_for_generate
from .vision import SiglipVisionTower

IGNORE_INDEX = -100
DEFAULT_IMAGE_TOKEN = "<image>"


# =================================================================================================
# tokenizer stand-in (no tokenizer files / network in this environment)
# =================================================================================================
class SyntheticTokenizer:
    """Minimal tokenizer exposing the attributes the hot path touches (`media_token_ids`,
    `stop_token_ids`, `padding_side`, `model_max_length`, `__call__(...).input_ids`, `decode`).
    Real checkpoints ship a HF tokenizer directory; `load_tokenizer` prefers it when present."""

    def __init__(self, config: LlavaConfig):
        self.media_token_ids = {"image": config.image_token_id, "video": config.video_token_id}
        self.media_tokens = {"image": "<image>", "video": "<vila/video>"}
        self.stop_token_ids = list(config.eos_token_ids)
        self.eos_token_id = config.eos_token_ids[0]
        self.pad_token_id = config.pad_token_id
        self.bos_token_id = None
        self.padding_side = "right"
        self.model_max_length = config.model_max_length
        self._newline = list(config.newline_token_ids)
        self._vocab = config.llm_cfg.vocab_size

    def __call__(self, text: str, **kw):
        ids: List[int] = []
        i = 0
        while i < len(text):
            for name, tok in self.media_tokens.items():
                if text.startswith(tok, i):
                    ids.append(self.media_token_ids[name])
                    i += len(tok)
                    break
            else:
                ch = text[i]
                ids.extend(self._newline if ch == "\n" else [3 + (ord(ch) % max(1, min(self._vocab, 256) - 3))])
                i += 1
        return SimpleNamespace(input_ids=ids)

    def decode(self, ids, skip_special_tokens: bool = True) -> str:
        ids = ids.tolist() if hasattr(ids, "tolist") else list(ids)
        return " ".join(str(int(i)) for i in ids if not (skip_special_tokens and int(i) in self.stop_token_ids))


# =================================================================================================
# media encoders
# =================================================================================================
class BaseEncoder(nn.Module):
    """llava/model/encoders/base.py"""

    def __init__(self, parent: nn.Module) -> None:
        super().__init__()
        self._parent = [parent]

    @property
    def parent(self) -> nn.Module:
        return self._parent[0]

    def embed_tokens(self, tokens: Optional[str]) -> Optional[torch.Tensor]:
        if tokens is None:
            return None
        token_ids = self.parent.tokenizer(tokens).input_ids
        token_ids = torch.tensor(token_ids, device=self.parent.device)
        return self.parent.llm.model.embed_tokens(token_ids)


class BasicImageEncoder(BaseEncoder):
    """llava/model/encoders/image/basic.py:11-79"""

    def __init__(self, parent, start_tokens: Optional[str] = None, end_tokens: Optional[str] = "\n"):
        super().__init__(parent)
        self.start_tokens = start_tokens
        self.end_tokens = end_tokens

    def _process_features(self, features, start_token_embeds, end_token_embeds):
        parts = [p for p in (start_token_embeds, features, end_token_embeds) if p is not None]
        return torch.cat(parts, dim=0) if len(parts) > 1 else features

    def forward(self, images: List[torch.Tensor], config: Dict[str, Any], **kw) -> List[torch.Tensor]:
        # host tensors (pinned by the caller) are copied H2D asynchronously BEFORE stacking so the
        # copy stays a pinned-memory DMA; the reference stacks on the host then moves the batch.
        dev = self.parent.device
        images = torch.stack([im.to(dev, non_blocking=True) for im in images], dim=0)
        features = self.parent.encode_images(images, block_sizes=config.get("block_sizes"))
        s, e = self.embed_tokens(self.start_tokens), self.embed_tokens(self.end_tokens)
        return [self._process_features(f, s, e) for f in features]


class BasicVideoEncoder(BaseEncoder):
    """llava/model/encoders/video/basic.py:11-53"""

    def __init__(self, parent, start_tokens: Optional[str] = None, end_tokens: Optional[str] = "\n"):
        super().__init__(parent)
        self.start_tokens = start_tokens
        self.end_tokens = end_tokens

    def _process_features(self, features, start_token_embeds, end_token_embeds):
        T = features.shape[0]
        if start_token_embeds is not None:
            features = torch.cat([start_token_embeds[None].expand(T, -1, -1), features], dim=1)
        if end_token_embeds is not None:
            features = torch.cat([features, end_token_embeds[None].expand(T, -1, -1)], dim=1)
        return features.flatten(0, 1)

    def forward(self, videos: List[torch.Tensor], config: Dict[str, Any]) -> List[torch.Tensor]:
        num_frames = [v.shape[0] for v in videos]
        features = self.parent._encode_frames(torch.cat(videos, dim=0))
        features = torch.split(features, num_frames)
        s, e = self.embed_tokens(self.start_tokens), self.embed_tokens(self.end_tokens)
        return [self._process_features(f, s, e) for f in features]


class TSPVideoEncoder(BasicVideoEncoder):
    """llava/model/encoders/video/tsp.py:15-66 — temporal/spatial mean pooling (tsp_pool kernel)."""

    def __init__(self, parent, pool_sizes: Sequence[Tuple[int, int, int]],
                 start_tokens: Optional[str] = None, end_tokens: Optional[str] = "\n",
                 sep_tokens: Optional[str] = None):
        super().__init__(parent, start_tokens=start_tokens, end_tokens=end_tokens)
        self.pool_sizes = [tuple(p) for p in pool_sizes]
        self.sep_tokens = sep_tokens

    def _process_features(self, inputs: torch.Tensor, start_token_embeds: Optional[torch.Tensor],
                          end_token_embeds: Optional[torch.Tensor],
                          sep_token_embeds: Optional[torch.Tensor]) -> torch.Tensor:
        """tsp.py:28-51: for every (t, h, w) pool size, mean-pool the frame features (one tsp_pool
        kernel instead of three chained view+mean ops), add the per-frame start / end tokens, then
        the separator."""
        nt, ns = inputs.shape[:2]
        nl = int(ns ** 0.5)
        parts = []
        for pt, ph, pw in self.pool_sizes:
            f = ops.tsp_pool(inputs.reshape(nt, nl, nl, -1).contiguous(), pt, ph, pw)
            f = f.flatten(1, 2)
            f = BasicVideoEncoder._process_features(self, f, start_token_embeds, end_token_embeds)
            if sep_token_embeds is not None:
                f = torch.cat([f, sep_token_embeds], dim=0)
            parts.append(f)
        return torch.cat(parts, dim=0)

    def forward(self, videos: List[torch.Tensor], config: Dict[str, Any]) -> List[torch.Tensor]:
        num_frames = [v.shape[0] for v in videos]
        features = self.parent._encode_frames(torch.cat(videos, dim=0))
        features = torch.split(features, num_frames)
        s, e = self.embed_tokens(self.start_tokens), self.embed_tokens(self.end_tokens)
        sep = self.embed_tokens(self.sep_tokens)
        return [self._process_features(f, s, e, sep) for f in features]


# =================================================================================================
# the VLM
# =================================================================================================
class LlavaLlamaModel(nn.Module):
    def __init__(self, config: LlavaConfig, device: Union[str, torch.device] = "cuda",
                 tokenizer=None):
        super().__init__()
        if not torch.cuda.is_available():
            raise RuntimeError("vila_b200.LlavaLlamaModel needs a CUDA (sm_90a) device: the hot path "
                               "has no CPU / eager fallback")
        from .. import _lib
        _lib.load()  # fail loudly if the extension is not built
        ops.ensure_workspace(device)  # stream-K scratch for the under-filled long-K GEMMs
        self.config = config
        dtype = torch.bfloat16
        self.llm = Qwen2ForCausalLM(config.llm_cfg, device, dtype)
        self.vision_tower = SiglipVisionTower(config, device, dtype)
        self.mm_projector = MultimodalProjector(config, device, dtype)
        self.tokenizer = tokenizer or SyntheticTokenizer(config)
        self.vocab_size = config.llm_cfg.vocab_size
        self.encoders = {"image": BasicImageEncoder(self)}
        if config.video_encoder == "tsp":
            self.encoders["video"] = TSPVideoEncoder(self, config.tsp_pool_sizes)
        else:
            self.encoders["video"] = BasicVideoEncoder(self)
        self.generation_config = None
        self.training = False
        self._vision_graphs = {}
        self._sp_runner_obj = None

    # ---- reference accessors (llava_arch.py:206-226) ----
    def get_llm(self):
        return self.llm

    def get_lm_head(self):
        return self.llm.lm_head

    def get_vision_tower(self):
        return self.vision_tower

    def get_mm_projector(self):
        return self.mm_projector

    @property
    def device(self):
        return self.llm.device

    @property
    def dtype(self):
        return self.llm.dtype

    # ---- weights ----
    @torch.no_grad()
    def init_random(self, seed: int = 0, device_rng: bool = False) -> "LlavaLlamaModel":
        """Random init of the named architecture (no checkpoints / network here): HF Qwen2 init
        (normal 0.02, norms 1), SigLIP _init_weights (modeling_siglip.py:786-825: xavier-uniform
        attention/MLP weights, position embedding std 1/sqrt(width)), default nn.Linear init for the
        projector.  Biases / LN params get small non-zero noise so that parity tests exercise them."""
        g = torch.Generator(device="cpu").manual_seed(seed)
        gd = torch.Generator(device=self.device).manual_seed(seed) if device_rng else None

        def fill(p: torch.Tensor, std: float, mean: float = 0.0):
            if gd is not None:  # fast path for the 8B-scale benchmark model (device RNG)
                rows = p.shape[0]
                step = max(1, (1 << 28) // max(1, p.numel() // rows))
                for r in range(0, rows, step):
                    blk = p[r:r + step]
                    blk.copy_((torch.randn(blk.shape, generator=gd, device=p.device) * std + mean).to(p.dtype))
                return
            # generate on the CPU for device-independent reproducibility, in chunks to bound memory
            flat_n = p.numel()
            if flat_n <= 1 << 26:
                p.copy_((torch.randn(p.shape, generator=g) * std + mean).to(p.dtype))
            else:
                rows = p.shape[0]
                step = max(1, (1 << 26) // max(1, flat_n // rows))
                for r in range(0, rows, step):
                    blk = p[r:r + step]
                    blk.copy_((torch.randn(blk.shape, generator=g) * std + mean).to(p.dtype))

        for name, p in self.named_parameters():
            if name.startswith("llm."):
                if "norm" in name:
                    fill(p, 0.02, 1.0)
                elif name.endswith("bias"):
                    fill(p, 0.02)
                else:
                    fill(p, 0.02)
            elif name.startswith("vision_tower."):
                if "layer_norm" in name or "post_layernorm" in name:
                    fill(p, 0.02, 1.0 if name.endswith("weight") else 0.0)
                elif "position_embedding" in name:
                    fill(p, 1.0 / (self.config.vision_tower_cfg.hidden_size ** 0.5))
                elif name.endswith("bias"):
                    fill(p, 0.02)
                else:
                    fan_out, fan_in = p.shape[0], p[0].numel()
                    fill(p, (2.0 / (fan_in + fan_out)) ** 0.5)
            else:  # projector
                if p.dim() == 1:
                    is_ln_w = False
                    fill(p, 0.02, 0.0)
                else:
                    fill(p, 1.0 / (p.shape[1] ** 0.5))
        # LayerNorm weights of the projector: centre at 1
        for op, mod in self.mm_projector._program:
            if op == "ln":
                mod.weight.add_(1.0)
        return self

    def reference_state_dict(self) -> Dict[str, torch.Tensor]:
        """State dict under the reference's names (llava_arch.py:170,178,194): `llm.*`,
        `vision_tower.vision_tower.*`, `mm_projector.layers.*`."""
        return {k: v for k, v in self.state_dict().items()}

    # ---- vision path ----
    @torch.inference_mode()
    def encode_images(self, images: torch.Tensor, block_sizes: Optional[List[Optional[Tuple[int, int]]]] = None):
        """llava_arch.py:366-394.  images [B,3,H,W] -> [B, N, hidden] or (dynamic-S2) list of [N_i, hidden]."""
        if block_sizes is None:
            block_sizes = [None] * len(images)
        tower, proj = self.get_vision_tower(), self.get_mm_projector()
        # pixels arrive as fp32 (media._to_tensor), fp16 (the reference calls .half(),
        # llava_arch.py:864) or bf16; every kernel below computes in the model dtype, and the
        # features stay in it (the reference casts them back only to feed them to a same-dtype LLM)
        images = images.to(device=self.device, dtype=self.dtype, non_blocking=True)
        if not getattr(self.config, "dynamic_s2", False):
            # tower + projector replayed from a CUDA graph cached per input shape (~190 launches per
            # call otherwise issued one by one from Python)
            key = tuple(images.shape)
            ent = self._vision_graphs.get(key)
            if ent is None:
                if len(self._vision_graphs) >= 4:
                    self._vision_graphs.pop(next(iter(self._vision_graphs)))
                static_in = torch.empty(key, dtype=self.dtype, device=self.device)
                static_in.copy_(images)
                proj(tower(static_in))  # warm-up
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    static_out = proj(tower(static_in))
                ent = (g, static_in, static_out)
                self._vision_graphs[key] = ent
            g, static_in, static_out = ent
            static_in.copy_(images, non_blocking=True)
            g.replay()
            return static_out
        feats = tower(images)  # [n_tiles, N, C]
        merged, new_bs = self._s2_merge_split(feats, block_sizes)
        x = proj(torch.cat(merged, dim=0))
        outs = []
        off = 0
        for ob in new_bs:
            n = ob[0] * ob[1]
            outs.append(ops.chessboard_merge(x[off:off + n].contiguous(), ob[0], ob[1]))
            off += n
        if all(o.shape[0] == outs[0].shape[0] for o in outs):
            return torch.stack(outs, dim=0)
        return outs

    def _s2_merge_split(self, feats: torch.Tensor, block_sizes):
        """merge_features_for_dynamic_s2 (:298-364) + split_chessboard (:375-378) per image as ONE
        kernel: -> (list of [bh*bw, N, n_scales*C] re-split tiles, new block sizes)."""
        tower = self.get_vision_tower()
        scales = tower.scales
        idx = tower.resize_output_to_scale_idx
        ratios = [s // scales[0] for s in scales]
        merged, new_bs = [], []
        cnt = 0
        for bs in block_sizes:
            if bs is None:
                merged.append(ops.s2_merge(feats[cnt:cnt + 1].contiguous(), [1] * len(scales),
                                           [1] * len(scales), 1, 1, share_tile=True))
                new_bs.append((1, 1))
                cnt += 1
                continue
            sh = ratios[:-1] + [bs[0]]
            sw = ratios[:-1] + [bs[1]]
            n = sum(a * b for a, b in zip(sh, sw))
            if idx == len(scales) - 1 or idx == -1:
                ob = tuple(bs)
            else:
                ob = (ratios[idx], ratios[idx])
            merged.append(ops.s2_merge(feats[cnt:cnt + n].contiguous(), sh, sw, ob[0], ob[1]))
            new_bs.append(ob)
            cnt += n
        assert cnt == len(feats), f"The number of blocks ({cnt}) does not match length of image_features ({len(feats)})!"
        return merged, new_bs

    def merge_features_for_dynamic_s2(self, image_features, block_sizes):
        """llava_arch.py:298-364, same return value: ([1, n_scales*C, H, W] feature map per image,
        new block sizes).  Built from the fused kernel's re-split tiles with one chessboard merge."""
        merged, new_bs = self._s2_merge_split(image_features, block_sizes)
        maps = []
        for tiles, ob in zip(merged, new_bs):
            side = int(round(tiles.shape[1] ** 0.5))
            flat = ops.chessboard_merge(tiles.contiguous(), ob[0], ob[1])
            maps.append(flat.view(ob[0] * side, ob[1] * side, -1).permute(2, 0, 1)[None])
        return maps, new_bs

    def repack_multimodal_data(self, inputs_embeds, attention_mask, position_ids, labels):
        """llava_arch.py:557-800.  Without a sequence-parallel group: sequence packing
        (model/packing.py).  With one, the reference re-shards the batch over ranks (:561-742); here
        the sharding happens inside the SP prefill (vila_b200/sp.py: zigzag chunks), so the inputs
        are returned unchanged."""
        if self._sp_runner() is not None:
            return inputs_embeds, attention_mask, position_ids, labels
        from .packing import repack_multimodal_data
        return repack_multimodal_data(inputs_embeds, attention_mask, position_ids, labels,
                                      getattr(self, "pad_to_multiple_of", None), self.config.pad_token_id)

    # ---- sequence parallelism (LongVILA; reference: llava/train/sequence_parallel/*, the SP branch of
    # repack_multimodal_data llava_arch.py:561-742, eval_vision_niah.py:83-140) ----
    def _sp_runner(self):
        """The SequenceParallelPrefill of the registered group, or None when SP is off
        (vila_b200.sp.set_sequence_parallel_group)."""
        from .. import sp
        if not sp.sequence_parallel_enabled():
            return None
        grp = sp.sequence_parallel_group()
        if self._sp_runner_obj is None or self._sp_runner_obj.group is not grp:
            self._sp_runner_obj = sp.SequenceParallelPrefill(self.llm, grp)
        return self._sp_runner_obj

    @torch.inference_mode()
    def _encode_frames(self, frames: torch.Tensor, batch: int = 32) -> torch.Tensor:
        """encode_images over video frames.  Under sequence parallelism the frames are sharded in
        contiguous ranges over the ranks (the reference's collator does the same split,
        sequence_parallel/input_utils.py:26-30): each rank copies / encodes only its own frames and
        one all-gather assembles [F, N, hidden] everywhere (no collective inside the tower)."""
        runner = self._sp_runner()
        if runner is None:
            return self.encode_images(frames)
        from .. import sp
        F_all = frames.shape[0]
        f0, f1 = sp.shard_frames(F_all, runner.world, runner.rank)
        feats = [self.encode_images(frames[i:min(i + batch, f1)]).clone() for i in range(f0, f1, batch)]
        if feats:
            local = torch.cat(feats, dim=0)
        else:
            r = self.mm_projector.downsample_rate
            g = (self.config.vision_tower_cfg.grid + r - 1) // r
            local = torch.empty(0, g * g, self.config.hidden_size, dtype=self.dtype, device=self.device)
        return runner.gather_frame_features(local, F_all)

    # ---- _embed (llava_arch.py:412-490) ----
    def __embed_media_tokens(self, media, media_config):
        embeds = defaultdict(deque)
        for name in media:
            embeds[name] = deque(self.encoders[name](media[name], media_config[name]))
        return embeds

    @torch.inference_mode()
    def _embed(self, input_ids: torch.Tensor, media: Optional[Dict[str, List[torch.Tensor]]],
               media_config: Optional[Dict[str, Dict[str, Any]]], labels: Optional[torch.Tensor],
               attention_mask: Optional[torch.Tensor]):
        media = media or {}
        media_config = media_config if media_config is not None else defaultdict(dict)
        ids_host = input_ids.detach().to("cpu")  # ONE D2H copy (the reference does one per token)
        labels_host = labels.detach().to("cpu") if labels is not None else torch.full_like(ids_host, IGNORE_INDEX)
        mask_host = (attention_mask.detach().to("cpu").to(torch.bool) if attention_mask is not None
                     else torch.ones_like(ids_host, dtype=torch.bool))
        media_embeds = self.__embed_media_tokens(media, {k: media_config.get(k, {}) for k in media})
        tok2name = {tid: name for name, tid in self.tokenizer.media_token_ids.items()}

        bsz = ids_host.shape[0]
        media_rows: List[torch.Tensor] = []
        media_off = 0
        srcs, labs = [], []
        media_id_list = torch.tensor(sorted(tok2name), dtype=ids_host.dtype)
        for k in range(bsz):
            # NOTE (reference quirk kept): positions index the UNMASKED input_ids (llava_arch.py:463)
            # while the text embeddings / labels come from the masked rows (:447)
            text_ids = ids_host[k][mask_host[k]]
            lab_k = labels_host[k][mask_host[k]]
            n_valid = lab_k.shape[0]
            ids_k = ids_host[k][:n_valid]
            # the index table is assembled from tensor segments (text runs / one arange per media
            # item): a 256-frame video is ONE segment of 65.8K rows, not 65.8K Python ints
            src_parts: List[torch.Tensor] = []
            lab_parts: List[torch.Tensor] = []
            prev = 0
            for pos in torch.nonzero(torch.isin(ids_k, media_id_list)).flatten().tolist():
                if pos > prev:
                    src_parts.append(text_ids[prev:pos].to(torch.int32))
                    lab_parts.append(lab_k[prev:pos])
                emb = media_embeds[tok2name[int(ids_k[pos])]].popleft()
                n = emb.shape[0]
                media_rows.append(emb)
                src_parts.append(-torch.arange(media_off + 1, media_off + n + 1, dtype=torch.int32))
                lab_parts.append(torch.full((n,), IGNORE_INDEX, dtype=lab_k.dtype))
                media_off += n
                prev = pos + 1
            if n_valid > prev:
                src_parts.append(text_ids[prev:n_valid].to(torch.int32))
                lab_parts.append(lab_k[prev:n_valid])
            srcs.append(torch.cat(src_parts) if src_parts else torch.zeros(0, dtype=torch.int32))
            labs.append(torch.cat(lab_parts) if lab_parts else torch.zeros(0, dtype=lab_k.dtype))
        for name in media_embeds:
            if media_embeds[name]:
                raise ValueError(f"Not all {name} embeddings are consumed!")

        # __truncate_sequence applies only in training (llava_arch.py:519-526); __batchify_sequence :528-555
        max_len = max(int(s.shape[0]) for s in srcs)
        hidden = self.config.hidden_size
        right = self.tokenizer.padding_side == "right"
        src_all = torch.zeros((bsz, max_len), dtype=torch.int32)
        lab_all = torch.full((bsz, max_len), IGNORE_INDEX, dtype=labels_host.dtype)
        mask_all = torch.zeros((bsz, max_len), dtype=torch.bool)
        for k in range(bsz):
            n = int(srcs[k].shape[0])
            sl = slice(0, n) if right else slice(max_len - n, max_len)
            src_all[k, sl] = srcs[k]
            lab_all[k, sl] = labs[k]
            mask_all[k, sl] = True
        dev = self.device
        media_buf = None
        if media_rows:  # one media item (a long video): no 0.5 GB copy
            media_buf = media_rows[0].contiguous() if len(media_rows) == 1 else torch.cat(media_rows, dim=0)
        embeds = ops.embed_splice(self.llm.model.embed_tokens.weight, media_buf,
                                  src_all.view(-1).to(dev, non_blocking=True))
        embeds = embeds.view(bsz, max_len, hidden)
        mask_dev = mask_all.to(dev)
        if not bool(mask_all.all()):
            embeds = embeds * mask_dev[..., None].to(embeds.dtype)  # padded rows are zeros (:538)
        return embeds, lab_all.to(dev), mask_dev

    # ---- forward (llava_llama.py:94-159) ----
    def forward(self, input_ids=None, media=None, images=None, media_config=None, attention_mask=None,
                position_ids=None, past_key_values=None, inputs_embeds=None, labels=None,
                packing: bool = True, force_packing: bool = False, seqlens_in_batch=None,
                dpo_forward: bool = False, **kwargs):
        if images is not None:
            if media is not None:
                raise ValueError("Both 'media' and 'images' are provided. Please provide only one.")
            media = {"image": images}
        if media_config is None:
            media_config = defaultdict(dict)
        if inputs_embeds is None:
            inputs_embeds, labels, attention_mask = self._embed(input_ids, media, media_config, labels,
                                                                attention_mask)
        runner = self._sp_runner()
        if runner is not None and past_key_values is None:
            return self._forward_sequence_parallel(runner, inputs_embeds, attention_mask, labels, dpo_forward)
        extra = {}
        if force_packing or (packing and self.training and not dpo_forward):
            # llava_llama.py:117-132: pack the padded batch into one row; the LLM then runs varlen
            # (block-diagonal causal) attention from `seqlens_in_batch`
            from .packing import repack_multimodal_data
            if seqlens_in_batch is None:
                seqlens_in_batch = torch.sum(attention_mask, dim=1)
            inputs_embeds, attention_mask, position_ids, labels = repack_multimodal_data(
                inputs_embeds, attention_mask, position_ids, labels,
                getattr(self, "pad_to_multiple_of", None), self.config.pad_token_id)
            extra["seqlens_in_batch"] = seqlens_in_batch
        outputs = self.llm(inputs_embeds=inputs_embeds, attention_mask=attention_mask,
                           position_ids=position_ids, past_key_values=past_key_values, labels=labels,
                           **extra)
        if dpo_forward:
            return outputs.logits, labels
        return outputs

    @torch.inference_mode()
    def _forward_sequence_parallel(self, runner, inputs_embeds, attention_mask, labels, dpo_forward):
        """forward under sequence parallelism: like the reference's SP branch every rank returns the
        logits (and labels) of ITS shard of the sequence — here the two zigzag chunks of
        sp.ZigzagPlan — plus `sp_plan` so callers can `undo_extract_local` / find the last token
        (eval_vision_niah.py:121-133)."""
        from .. import sp
        assert inputs_embeds.shape[0] == 1, "sequence parallelism shards ONE long sequence"
        emb = inputs_embeds[0]
        if attention_mask is not None:
            emb = emb[attention_mask[0].to(torch.bool)]
        S = emb.shape[0]
        plan = sp.make_plan(S, runner.world, runner.rank)
        padded = emb.new_zeros((plan.padded_len, emb.shape[1]))
        padded[:S] = emb
        hid_local, _ = runner.prefill_hidden(plan.extract_local(padded), plan)
        logits = self.llm.logits_from_hidden(hid_local)[None]
        local_labels = None
        if labels is not None:
            lab = labels[0][attention_mask[0].to(torch.bool)] if attention_mask is not None else labels[0]
            lab_p = torch.full((plan.padded_len,), IGNORE_INDEX, dtype=lab.dtype, device=lab.device)
            lab_p[:S] = lab
            local_labels = plan.extract_local(lab_p)[None]
        if dpo_forward:
            return logits, local_labels
        return SimpleNamespace(logits=logits, loss=None, past_key_values=None, labels=local_labels,
                               sp_plan=plan)

    __call__ = forward

    # ---- generate (llava_arch.py:823-833) ----
    @torch.inference_mode()
    def generate(self, input_ids=None, media=None, media_config=None, attention_mask=None,
                 **generation_kwargs):
        inputs_embeds, _, attention_mask = self._embed(input_ids, media, media_config, None,
                                                       attention_mask)
        # HF merges the model's generation_config under explicit kwargs; ours comes from the tokenizer
        # (default_generation_config, llava_arch.py:950-963) so eos / pad are known even when the
        # caller only passes max_new_tokens (explicit kwargs, e.g. eos_token_id=None, still win)
        if "generation_config" not in generation_kwargs:
            generation_kwargs["generation_config"] = self.default_generation_config
        return self.llm.generate(inputs_embeds=inputs_embeds, attention_mask=attention_mask,
                                 sp_runner=self._sp_runner(), **generation_kwargs)

    @torch.inference_mode()
    def generate_batch(self, requests: List[Dict[str, Any]], max_new_tokens: int = 128, slots: int = 8,
                       max_tokens_per_slot: Optional[int] = None, eos_token_id=None,
                       kv_cache: str = "bf16", sampling=None, prefix_cache: bool = False,
                       logprobs: Optional[int] = None, penalties=None):
        """Serve several independent requests with continuous batching over one shared paged KV pool
        (vila_b200/serving.py; the reference's servers run them one at a time, serving/server.py:65-73).
        requests: dicts with the `generate` arguments (`input_ids` [1, T], `media`, `media_config`).
        max_tokens_per_slot None: sized from the requests (serving.slot_geometry: 2048 tokens unless a
        request needs more, e.g. video or dynamic-S2 prompts).
        kv_cache: "bf16" (default) or "fp8" (e4m3 K/V with one fp32 scale per token and KV head, serving.py).
        sampling: None (default) decodes greedily; a serving.SamplingParams, or a list with one per request,
        samples on the device (serving.generate_batch).
        prefix_cache: True shares the K/V pages of the full 128-token prompt blocks that requests start with (the
        same video or image, one system prompt), and needs max_tokens_per_slot.  The model keeps the engine it
        builds (max_new = max_tokens_per_slot), and with it the cached blocks, for later calls with the same slots,
        max_tokens_per_slot, decode-weight mode, kv_cache, sampling (greedy or not), logprobs and penalties (asked
        for or not); any other call rebuilds it.
        logprobs: None (default) returns the new ids of every request in order; an int n in 0..20 returns (ids,
        logprobs) with one vila_b200.logprobs.TokenLogprob per id (serving.generate_batch).
        penalties: None (default) applies none; a vila_b200.penalties.PenaltyParams, or a list with one PenaltyParams or
        None per request, applies OpenAI's presence / frequency penalties on the device (serving.generate_batch)."""
        from ..serving import BatchedDecoder, generate_batch
        if prefix_cache and max_tokens_per_slot is None:
            raise ValueError("generate_batch(prefix_cache=True) needs max_tokens_per_slot: the engine and its cached "
                             "blocks are kept between calls, so its slot size cannot follow the requests")
        prompts = []
        for r in requests:
            emb, _, mask = self._embed(r["input_ids"], r.get("media"), r.get("media_config"), None,
                                       r.get("attention_mask"))
            prompts.append(emb[0][mask[0]] if mask is not None else emb[0])
        eos = self.tokenizer.stop_token_ids if eos_token_id is None else (
            [eos_token_id] if isinstance(eos_token_id, int) else list(eos_token_id))
        decoder = None
        if prefix_cache:
            key = (slots, max_tokens_per_slot, getattr(self.llm, "decode_weights", "bf16"), kv_cache,
                   sampling is not None, logprobs)
            key += (penalties is not None,)
            kept = getattr(self, "_prefix_engine", None)
            if kept is None or kept[0] != key:
                if kept is not None:  # free the old pool and its graphs before the new ones are allocated
                    kept = self._prefix_engine = None
                    gc.collect()
                kept = (key, BatchedDecoder(self.llm, slots, max_tokens_per_slot, max_new=max_tokens_per_slot,
                                            kv_cache=kv_cache, sampling=sampling is not None, prefix_cache=True,
                                            logprobs=logprobs, penalties=penalties is not None))
                self._prefix_engine = kept
            decoder = kept[1]
        return generate_batch(self.llm, prompts, max_new_tokens, eos, slots=slots,
                              max_tokens_per_slot=max_tokens_per_slot, decoder=decoder, kv_cache=kv_cache,
                              sampling=sampling, prefix_cache=prefix_cache, logprobs=logprobs, penalties=penalties)

    @property
    def default_generation_config(self):
        """llava_arch.py:950-963 (GenerationConfig fields as a plain namespace)."""
        gc = copy.deepcopy(self.generation_config) if self.generation_config is not None else \
            SimpleNamespace(max_length=20, max_new_tokens=None, do_sample=False, pad_token_id=None,
                            bos_token_id=None, eos_token_id=None, temperature=1.0, top_p=1.0, top_k=0)
        if self.tokenizer.eos_token_id is None:
            raise ValueError("Tokenizer must have an EOS token")
        if getattr(gc, "max_length", 20) == 20:
            gc.max_length = self.tokenizer.model_max_length
        if getattr(gc, "pad_token_id", None) is None:
            gc.pad_token_id = self.tokenizer.pad_token_id or self.tokenizer.eos_token_id
        if getattr(gc, "bos_token_id", None) is None:
            gc.bos_token_id = self.tokenizer.bos_token_id or self.tokenizer.eos_token_id
        if getattr(gc, "eos_token_id", None) is None:
            gc.eos_token_id = self.tokenizer.stop_token_ids
        return gc

    def compile_response_format(self, response_format):
        """llava_arch.py:802-821: compile `response_format` with xgrammar: type json_schema -> its schema (indent 2),
        any other type -> the builtin JSON grammar.  self.grammar_compiler is built from the HF tokenizer on first use
        (a caller may install one built from an explicit vocabulary first) and caches what it compiles.  A schema
        xgrammar cannot compile raises."""
        import xgrammar as xgr
        if getattr(self, "grammar_compiler", None) is None:
            self.grammar_compiler = xgr.GrammarCompiler(
                xgr.TokenizerInfo.from_huggingface(self.tokenizer, vocab_size=self.vocab_size))
        if response_format.type == "json_schema":
            return self.grammar_compiler.compile_json_schema(response_format.json_schema.schema_, indent=2)
        return self.grammar_compiler.compile_builtin_json_grammar()

    def get_xgr_logits_processor(self, response_format) -> List[Any]:
        """llava_arch.py:802-821: `response_format` as an HF-style logits processor, for the eager decode loop
        (Qwen2ForCausalLM.generate(logits_processor=...)), which calls it once per token on the host."""
        import xgrammar as xgr
        return [xgr.contrib.hf.LogitsProcessor(self.compile_response_format(response_format))]

    def grammar_matcher(self, response_format, stop_token_ids):
        """`response_format` as a fresh xgrammar GrammarMatcher for the graph decoder (GraphDecoder.start(grammar=)),
        whose stop tokens are the decode's EOS ids: the grammar allows them once the document is complete, and
        accepting one terminates the matcher."""
        import xgrammar as xgr
        return xgr.GrammarMatcher(self.compile_response_format(response_format),
                                  override_stop_tokens=list(stop_token_ids))

    def _prepare_content(self, prompt: Union[str, List]):
        """prompt -> (input_ids [1,T], media, media_config): the host half of generate_content
        (llava_arch.py:843-897)."""
        from . import media as media_utils
        text, images = media_utils.extract_media(prompt, self.config)
        media: Dict[str, List[torch.Tensor]] = {}
        media_config: Dict[str, Dict[str, Any]] = defaultdict(dict)
        if images:
            if getattr(self, "preprocess_on_device", True) and not any(isinstance(im, torch.Tensor) for im in images) \
                    and next(self.llm.parameters()).is_cuda:
                # resize + rescale + normalise + tiling as kernels (vila_resize_bicubic_tiles),
                # bit-identical to the PIL + SiglipImageProcessor path below
                tensors, block_sizes = media_utils.process_images_gpu(images, self.config, self.device)
            else:
                tensors, block_sizes = media_utils.process_images(images, self.config)
            if (self.config.image_aspect_ratio == "dynamic" and len(images) == 1
                    and not isinstance(images[0], torch.Tensor)):
                text = media_utils.dynamic_prompt(text, len(tensors))
            media["image"] = tensors
            if block_sizes is not None:
                media_config["image"]["block_sizes"] = block_sizes
        ids = media_utils.tokenize_conversation(text, self.tokenizer)
        return torch.tensor([ids], dtype=torch.long), media, media_config

    def generate_content(self, prompt: Union[str, List], generation_config=None,
                         response_format=None, stream: bool = False):
        """llava_arch.py:835-948: prompt = str or list of (str | image tensor [3,H,W] | PIL image).
        Image tensors must already be normalised; PIL images go through `media.process_image`.
        response_format: xgrammar-constrained decoding (llava_arch.py:846-849), streamed or not: the graph decoder
        masks every row with the grammar's token bitmask on the device (stream_content).
        stream=True (serving/server.py:259-264 calls it that way): returns an iterator of text
        chunks; the decode stays on the device and is drained every few tokens.  Both forms sample on the
        device when the generation config sets do_sample (its temperature, top_k, top_p and `seed`), with the
        same ids for the same seed."""
        if stream:
            return self._generate_content_stream(prompt, generation_config, response_format)
        if response_format:
            gc = generation_config or self.default_generation_config

            def constrained():
                return [t for ids, _ in self.stream_content(prompt, gc, response_format=response_format,
                                                             chunk_tokens=16) for t in ids]
            try:
                output_ids = constrained()
            except ValueError:
                if not getattr(gc, "do_sample", False):
                    raise
                gc.do_sample = False  # the reference's fallback: retry greedily (llava_arch.py:932-944)
                output_ids = constrained()
            return self.tokenizer.decode(output_ids, skip_special_tokens=True).strip()
        with torch.inference_mode():
            input_ids, media, media_config = self._prepare_content(prompt)
            gc = generation_config or self.default_generation_config
            try:
                output_ids = self.generate(input_ids=input_ids, media=media, media_config=media_config,
                                           generation_config=gc)
            except ValueError:
                if not getattr(gc, "do_sample", False):
                    raise
                gc.do_sample = False  # the reference's fallback: retry greedily (llava_arch.py:932-944)
                output_ids = self.generate(input_ids=input_ids, media=media, media_config=media_config,
                                           generation_config=gc)
            return self.tokenizer.decode(output_ids[0], skip_special_tokens=True).strip()

    def _generate_content_stream(self, prompt, generation_config, response_format, chunk_tokens: int = 8):
        kw = {} if response_format is None else {"response_format": response_format}
        for ids, _ in self.stream_content(prompt, generation_config, chunk_tokens=chunk_tokens, **kw):
            text = self.tokenizer.decode(ids, skip_special_tokens=True)
            if text:
                yield text

    def stream_content(self, prompt: Union[str, List], generation_config=None, *, logprobs: Optional[int] = None,
                       penalties=None, chunk_tokens: int = 8, response_format=None):
        """generate_content(stream=True) with per-token logprobs and OpenAI presence / frequency penalties, as a
        generator of (ids, entries) per chunk of up to chunk_tokens new ids (sampled on the device when the generation
        config sets do_sample, as generate_content).  entries: one vila_b200.logprobs.TokenLogprob per id with
        `logprobs` = n in 0..20 alternatives, else None.  penalties: a vila_b200.penalties.PenaltyParams, or None.  The
        last chunk ends with the EOS id when one was generated; its entry is there too.  Both options run on the
        device in the single-stream graph decoder (Qwen2ForCausalLM.stream_tokens).  response_format: a ResponseFormat
        (generate_content's mapping of its types, compile_response_format); every id is then one the grammar allows,
        and the stream ends when the grammar terminates (its stop tokens are the config's EOS ids).  Not with
        sequence-parallel decoding (NotImplementedError)."""
        from ..logprobs import check_top
        if logprobs is not None:
            check_top(logprobs)
        if ((logprobs is not None or (penalties is not None and not penalties.off) or response_format is not None)
                and self._sp_runner() is not None):
            raise NotImplementedError("stream_content: logprobs, penalties and response_format are not implemented "
                                      "with sequence-parallel decoding")
        with torch.inference_mode():
            input_ids, media, media_config = self._prepare_content(prompt)
            gc = generation_config or self.default_generation_config
            inputs_embeds, _, _ = self._embed(input_ids, media, media_config, None, None)
        sampling = sampling_for_generate(gc, 1)[0] if getattr(gc, "do_sample", False) else None
        kw = {}
        if response_format is not None:
            eos = getattr(gc, "eos_token_id", None)
            kw["grammar"] = self.grammar_matcher(response_format, [] if eos is None else
                                                 [eos] if isinstance(eos, int) else list(eos))
        for out in self.llm.stream_tokens(inputs_embeds[0], gc, chunk_tokens=chunk_tokens, sampling=sampling,
                                          logprobs=logprobs, penalties=penalties, **kw):
            yield out if logprobs is not None else (out, None)
