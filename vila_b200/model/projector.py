"""mm_projector on the sm_90a kernels — API mirror of MultimodalProjector
(llava/model/multimodal_projector/base_projector.py:134-252): `forward(x)` with
`config.mm_projector_type` in {mlp_downsample, mlp_downsample_2x2_fix, mlp_downsample_3x3_fix,
mlpNx_gelu, linear, identity}; state-dict names `layers.{1,2,4,...}.{weight,bias}`.
"""
from __future__ import annotations

import re
from types import SimpleNamespace

import torch
from torch import nn

from .. import ops
from .configuration import LlavaConfig


class _P(nn.Module):
    def __init__(self, *shape_w, bias_shape=None, device=None, dtype=None):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(*shape_w, device=device, dtype=dtype),
                                   requires_grad=False)
        if bias_shape is not None:
            self.bias = nn.Parameter(torch.empty(bias_shape, device=device, dtype=dtype),
                                     requires_grad=False)


class MultimodalProjector(nn.Module):
    LN_EPS = 1e-5  # nn.LayerNorm default, base_projector.py:147

    def __init__(self, config: LlavaConfig, device="cuda", dtype=torch.bfloat16):
        super().__init__()
        kind = config.mm_projector_type
        self.config = SimpleNamespace(mm_projector_type=kind)
        C, H = config.mm_hidden_size, config.hidden_size
        kw = dict(device=device, dtype=dtype)
        layers = nn.Module()
        self.downsample_rate = 1
        # program: list of (op, layer_index) executed in order, mirroring the nn.Sequential indices
        if kind in ("mlp_downsample", "mlp_downsample_2x2_fix"):
            self.downsample_rate = 2
            specs = {1: ("ln", 4 * C), 2: ("lin_gelu", 4 * C, H), 4: ("lin", H, H)}
        elif kind == "mlp_downsample_3x3_fix":
            self.downsample_rate = 3
            specs = {1: ("ln", 9 * C), 2: ("lin_gelu", 9 * C, 3 * C), 4: ("ln", 3 * C),
                     5: ("lin_gelu", 3 * C, H), 7: ("lin", H, H)}
        elif kind == "linear":
            specs = {None: ("lin", C, H)}
        elif kind == "identity":
            specs = {}
        else:
            m = re.match(r"^mlp(\d+)x_gelu$", kind)
            if not m:
                raise ValueError(f"Unknown projector type: {kind}")
            depth = int(m.group(1))
            specs = {0: ("lin_gelu" if depth > 1 else "lin", C, H)}
            for i in range(1, depth):
                specs[2 * i] = ("lin_gelu" if i < depth - 1 else "lin", H, H)
        self._program = []
        for idx, spec in specs.items():
            if spec[0] == "ln":
                mod = _P(spec[1], bias_shape=spec[1], **kw)
            else:
                mod = _P(spec[2], spec[1], bias_shape=spec[2], **kw)
            if idx is None:
                layers = mod  # `self.layers = nn.Linear(...)` in the reference
            else:
                layers.add_module(str(idx), mod)
            self._program.append((spec[0], mod))
        self.layers = layers

    def forward(self, x: torch.Tensor, forward_top_down_prompt_head: bool = False, *a, **k):
        if forward_top_down_prompt_head:
            raise NotImplementedError("PS3 top-down prompt head is out of scope (SURVEY §2 row 19)")
        B, N, C = x.shape
        if self.downsample_rate > 1:
            s = int(N ** 0.5)
            x = ops.space_to_depth(x.contiguous(), s, s, self.downsample_rate)
            B, N, C = x.shape
        h = x.reshape(B * N, C)
        for op, mod in self._program:
            if op == "ln":
                h = ops.layernorm(h, mod.weight, mod.bias, self.LN_EPS)
            elif op == "lin_gelu":
                h = ops.linear(h, mod.weight, mod.bias, act=ops.ACT_GELU_ERF, static_w=True)
            else:
                h = ops.linear(h, mod.weight, mod.bias, static_w=True)
        return h.view(B, N, -1)
