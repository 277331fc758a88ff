"""SigLIP vision tower on the sm_90a kernels.

API mirror of the reference wrappers:
  SiglipVisionTower(VisionTower)          llava/model/multimodal_encoder/siglip_encoder.py:25-36
  VisionTower.forward / feature_select    llava/model/multimodal_encoder/vision_encoder.py:44-52,133-177
  VisionTowerDynamicS2 (.scales, .resize_output_to_scale_idx, forward_feature)   :251-271
State-dict names equal the reference's (`vision_tower.vision_model.encoder.layers.N.self_attn.q_proj.weight`
...), but q/k/v live in ONE fused [3C, C] buffer (the named parameters are views into it) so the
three projections are a single wgmma GEMM (SURVEY §2.3 K3).
"""
from __future__ import annotations

from typing import List, Optional

import torch
from torch import nn

from .. import ops
from .configuration import LlavaConfig, SiglipVisionConfig


class _Holder(nn.Module):
    """Empty module used to build the reference's attribute tree."""


def _param(t: torch.Tensor) -> nn.Parameter:
    return nn.Parameter(t, requires_grad=False)


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class SiglipEncoderLayer(nn.Module):
    """modeling_siglip.py:718-764 (pre-LN MHA + GELU-tanh MLP with residuals)."""

    def __init__(self, cfg: SiglipVisionConfig, device, dtype):
        super().__init__()
        C, I = cfg.hidden_size, cfg.intermediate_size
        self.cfg = cfg
        kw = dict(device=device, dtype=dtype)
        self._qkv_w = torch.empty(3 * C, C, **kw)
        self._qkv_b = torch.empty(3 * C, **kw)
        att = _Holder()
        for i, name in enumerate(("q_proj", "k_proj", "v_proj")):
            lin = _Holder()
            lin.weight = _param(self._qkv_w[i * C:(i + 1) * C])
            lin.bias = _param(self._qkv_b[i * C:(i + 1) * C])
            setattr(att, name, lin)
        att.out_proj = _Holder()
        att.out_proj.weight = _param(torch.empty(C, C, **kw))
        att.out_proj.bias = _param(torch.empty(C, **kw))
        self.self_attn = att
        for name in ("layer_norm1", "layer_norm2"):
            ln = _Holder()
            ln.weight = _param(torch.empty(C, **kw))
            ln.bias = _param(torch.empty(C, **kw))
            setattr(self, name, ln)
        mlp = _Holder()
        mlp.fc1 = _Holder()
        mlp.fc1.weight = _param(torch.empty(I, C, **kw))
        mlp.fc1.bias = _param(torch.empty(I, **kw))
        mlp.fc2 = _Holder()
        mlp.fc2.weight = _param(torch.empty(C, I, **kw))
        mlp.fc2.bias = _param(torch.empty(C, **kw))
        self.mlp = mlp

    def forward(self, x: torch.Tensor, B: int, S: int) -> torch.Tensor:
        """x: [B*S, C] residual stream, updated in place and returned."""
        cfg = self.cfg
        C, H = cfg.hidden_size, cfg.num_attention_heads
        D = C // H
        h = ops.layernorm(x, self.layer_norm1.weight, self.layer_norm1.bias, cfg.layer_norm_eps)
        qkv = ops.linear(h, self._qkv_w, self._qkv_b, static_w=True).view(B * S, 3, H, D)
        attn = ops.fmha(qkv[:, 0], qkv[:, 1], qkv[:, 2], B=B, Sq=S, Sk=S, causal=False,
                        scale=D ** -0.5)
        ops.linear(attn.view(B * S, C), self.self_attn.out_proj.weight, self.self_attn.out_proj.bias,
                   residual=x, out=x, static_w=True)
        h = ops.layernorm(x, self.layer_norm2.weight, self.layer_norm2.bias, cfg.layer_norm_eps)
        f = ops.linear(h, self.mlp.fc1.weight, self.mlp.fc1.bias, act=ops.ACT_GELU_TANH, static_w=True)
        ops.linear(f, self.mlp.fc2.weight, self.mlp.fc2.bias, residual=x, out=x, static_w=True)
        return x


class SiglipVisionModel(nn.Module):
    """Parameter tree of the reference SiglipVisionModel (modeling_siglip.py:1242) restricted to what
    VILA evaluates: embeddings + encoder layers (+ post_layernorm kept only for checkpoint loading;
    the pooling head is dead compute for VILA and is not instantiated)."""

    def __init__(self, cfg: SiglipVisionConfig, device, dtype):
        super().__init__()
        self.config = cfg
        C = cfg.hidden_size
        kw = dict(device=device, dtype=dtype)
        self.k_real = cfg.num_channels * cfg.patch_size * cfg.patch_size
        self.k_pad = _round_up(self.k_real, 8)
        vm = _Holder()
        emb = _Holder()
        # Conv2d weight [C, 3, 14, 14] is a view of the K-padded GEMM operand [C, k_pad]
        self._patch_w = torch.zeros(C, self.k_pad, **kw)
        pe = _Holder()
        pe.weight = _param(self._patch_w[:, :self.k_real].view(C, cfg.num_channels, cfg.patch_size,
                                                                cfg.patch_size)
                           if self.k_pad == self.k_real else
                           self._patch_w.as_strided((C, cfg.num_channels, cfg.patch_size, cfg.patch_size),
                                                    (self.k_pad, cfg.patch_size * cfg.patch_size,
                                                     cfg.patch_size, 1)))
        pe.bias = _param(torch.empty(C, **kw))
        emb.patch_embedding = pe
        pos = _Holder()
        pos.weight = _param(torch.empty(cfg.num_patches, C, **kw))
        emb.position_embedding = pos
        vm.embeddings = emb
        enc = _Holder()
        enc.layers = nn.ModuleList([SiglipEncoderLayer(cfg, device, dtype)
                                    for _ in range(cfg.num_hidden_layers)])
        vm.encoder = enc
        pln = _Holder()
        pln.weight = _param(torch.ones(C, **kw))
        pln.bias = _param(torch.zeros(C, **kw))
        vm.post_layernorm = pln
        self.vision_model = vm

    def hidden_state(self, pixels: torch.Tensor, select_layer: int) -> torch.Tensor:
        """== model(pixels, output_hidden_states=True).hidden_states[select_layer]
        (modeling_siglip.py:320-329 embeddings, :994-1017 encoder loop)."""
        cfg = self.config
        B = pixels.shape[0]
        assert pixels.shape[1:] == (cfg.num_channels, cfg.image_size, cfg.image_size), pixels.shape
        emb = self.vision_model.embeddings
        a = ops.patch_im2col(pixels.contiguous(), cfg.patch_size, self.k_pad)
        x = ops.linear(a, self._patch_w, emb.patch_embedding.bias,
                       residual=emb.position_embedding.weight, res_row_mod=cfg.num_patches, static_w=True)
        n_states = cfg.num_hidden_layers + 1
        idx = select_layer if select_layer >= 0 else n_states + select_layer
        for i in range(idx):
            x = self.vision_model.encoder.layers[i](x, B, cfg.num_patches)
        return x.view(B, cfg.num_patches, cfg.hidden_size)


class SiglipVisionTower(nn.Module):
    """VisionTower / VisionTowerDynamicS2 (vision_encoder.py:32-52,133-177,251-271)."""

    def __init__(self, config: LlavaConfig, device="cuda", dtype=torch.bfloat16):
        super().__init__()
        self.select_layer = config.mm_vision_select_layer
        self.select_feature = config.mm_vision_select_feature
        self.vision_tower = SiglipVisionModel(config.vision_tower_cfg, device, dtype)
        self.is_loaded = True
        self.image_processor = None  # set by the loader when a preprocessor config is available
        if config.dynamic_s2:
            self.scales = sorted(config.s2_scales)
            self.max_split_size = config.s2_max_split_size
            self.resize_output_to_scale_idx = config.s2_resize_output_to_scale_idx

    @property
    def config(self):
        return self.vision_tower.config

    @property
    def dtype(self):
        return self.vision_tower.vision_model.embeddings.position_embedding.weight.dtype

    @property
    def device(self):
        return self.vision_tower.vision_model.embeddings.position_embedding.weight.device

    @property
    def hidden_size(self):
        n = len(self.scales) if hasattr(self, "scales") else 1
        return self.config.hidden_size * n

    def forward(self, images):
        """images [B,3,H,W] (any float dtype/device) -> [B, N, C] in images.dtype."""
        if isinstance(images, list):
            return [self.forward(im.unsqueeze(0))[0] for im in images]
        x = images.to(device=self.device, dtype=self.dtype)
        feats = self.vision_tower.hidden_state(x, self.select_layer)
        if self.select_feature == "patch":
            feats = feats[:, 1:]
        elif self.select_feature != "cls_patch":
            raise ValueError(f"Unexpected select feature: {self.select_feature}")
        return feats.to(images.dtype) if images.dtype != feats.dtype else feats

    forward_feature = forward
