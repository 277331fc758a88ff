"""Qwen2 / Llama-style causal LM on the sm_90a kernels (prefill + CUDA-graph decode).

The reference obtains this model from third-party `transformers` (AutoModelForCausalLM,
llava/model/language_model/builder.py:173-180) and calls `self.llm(inputs_embeds=...)`
(llava_llama.py:134-141) and `self.llm.generate(inputs_embeds=..., attention_mask=...)`
(llava_arch.py:833).  This module keeps that surface (`.model.embed_tokens`, `.model.layers`,
`.model.norm`, `.lm_head`, `.config`, `.vocab_size`, `forward`, `generate`) and the HF state-dict
names, while q/k/v and gate/up are stored fused (named parameters are views) so each decoder layer is
  prefill: RMSNorm -> QKV GEMM -> RoPE+KV-append -> wgmma FMHA (paged) -> O GEMM(+res)
           -> RMSNorm -> gate/up GEMM (SwiGLU epilogue) -> down GEMM(+res)
  decode : [RMSNorm+QKV GEMV] -> [RoPE+append+split-KV attention] -> [O GEMV+res]
           -> [RMSNorm+gate/up GEMV+SwiGLU] -> [down GEMV+res]      (5 launches, CUDA-graphed)
Arithmetic spec: in-tree copy llava/eval/vision_niah_vila/zigzag_ring_attn/modeling_qwen2.py
(RMSNorm :81-95, RoPE :99-160, MLP :164-176, attention :191-310, layer :633-706).
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import List, Optional, Sequence

import torch
from torch import nn

from .. import ops
from .configuration import Qwen2Config

PAGE = 128
_UNSET = object()


def _param(t):
    return nn.Parameter(t, requires_grad=False)


class _Holder(nn.Module):
    pass


class Embedding(nn.Module):
    """nn.Embedding stand-in whose lookup is the embed_splice gather kernel."""

    def __init__(self, vocab: int, hidden: int, device, dtype):
        super().__init__()
        self.weight = _param(torch.empty(vocab, hidden, device=device, dtype=dtype))

    def forward(self, ids: torch.Tensor) -> torch.Tensor:
        shape = ids.shape
        src = ids.reshape(-1).to(device=self.weight.device, dtype=torch.int32)
        return ops.embed_splice(self.weight, None, src).view(*shape, self.weight.shape[1])


class Qwen2DecoderLayer(nn.Module):
    def __init__(self, cfg: Qwen2Config, device, dtype):
        super().__init__()
        self.cfg = cfg
        Hd, I = cfg.hidden_size, cfg.intermediate_size
        Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        kw = dict(device=device, dtype=dtype)
        self._qkv_w = torch.empty((Hq + 2 * Hkv) * D, Hd, **kw)
        self._qkv_b = torch.empty((Hq + 2 * Hkv) * D, **kw)
        self._gu_w = torch.empty(2 * I, Hd, **kw)  # interleaved rows: gate_0, up_0, gate_1, ...
        att = _Holder()
        bounds = {"q_proj": (0, Hq * D), "k_proj": (Hq * D, (Hq + Hkv) * D),
                  "v_proj": ((Hq + Hkv) * D, (Hq + 2 * Hkv) * D)}
        for name, (a, b) in bounds.items():
            lin = _Holder()
            lin.weight = _param(self._qkv_w[a:b])
            lin.bias = _param(self._qkv_b[a:b])
            setattr(att, name, lin)
        att.o_proj = _Holder()
        att.o_proj.weight = _param(torch.empty(Hd, Hq * D, **kw))
        self.self_attn = att
        mlp = _Holder()
        mlp.gate_proj = _Holder()
        mlp.gate_proj.weight = _param(self._gu_w[0::2])
        mlp.up_proj = _Holder()
        mlp.up_proj.weight = _param(self._gu_w[1::2])
        mlp.down_proj = _Holder()
        mlp.down_proj.weight = _param(torch.empty(Hd, I, **kw))
        self.mlp = mlp
        self.input_layernorm = _Holder()
        self.input_layernorm.weight = _param(torch.empty(Hd, **kw))
        self.post_attention_layernorm = _Holder()
        self.post_attention_layernorm.weight = _param(torch.empty(Hd, **kw))


class PagedKVCache:
    """Paged KV pool [L, 2, P, 128, Hkv, D] + page table (DynamicCache replacement, SURVEY K17)."""

    def __init__(self, cfg: Qwen2Config, max_tokens: int, device, dtype=torch.bfloat16,
                 page_order: Optional[Sequence[int]] = None):
        self.n_pages = (max_tokens + PAGE - 1) // PAGE
        self.pool = torch.zeros(cfg.num_hidden_layers, 2, self.n_pages, PAGE,
                                cfg.num_key_value_heads, cfg.head_dim, device=device, dtype=dtype)
        order = list(range(self.n_pages)) if page_order is None else list(page_order)
        self.page_table = torch.tensor(order, dtype=torch.int32, device=device)
        self.length = 0
        self.max_tokens = self.n_pages * PAGE

    def k(self, layer: int) -> torch.Tensor:
        return self.pool[layer, 0]

    def v(self, layer: int) -> torch.Tensor:
        return self.pool[layer, 1]


# HF generate options that would change the output and that this decode loop does not implement: they
# are refused instead of being swallowed by **kw (value = the settings that mean "off").
_NEUTRAL_GENERATION_OPTIONS = {
    "num_beams": (None, 1), "num_beam_groups": (None, 1), "num_return_sequences": (None, 1),
    "repetition_penalty": (None, 1.0), "no_repeat_ngram_size": (None, 0), "min_new_tokens": (None, 0),
    "min_length": (None, 0), "penalty_alpha": (None, 0.0), "typical_p": (None, 1.0), "min_p": (None,),
    "bad_words_ids": (None,), "force_words_ids": (None,), "prefix_allowed_tokens_fn": (None,),
    "assistant_model": (None,), "streamer": (None,), "stopping_criteria": (None,),
}


def unsupported_generation_options(generation_config, kwargs) -> List[str]:
    """Names (with values) of result-changing HF generation options set to something other than off,
    looked up in the explicit kwargs first and in the generation config otherwise."""
    bad = []
    for name, neutral in _NEUTRAL_GENERATION_OPTIONS.items():
        v = kwargs[name] if name in kwargs else (getattr(generation_config, name, None) if generation_config is not None else None)
        if name == "stopping_criteria" and v is not None and len(v) == 0:
            continue
        if not any(v is n or (n is not None and v == n) for n in neutral):
            bad.append(f"{name}={v!r}")
    return bad


E4M3_MAX = 448.0


def quantize_e4m3_rows(w: torch.Tensor, rows_per_chunk: int = 16384):
    """Weight-only FP8 with one scale per output row, no calibration data:
        amax_n = max_k |W[n,k]| (fp32);  s_n = amax_n / 448, or 1 for an all-zero row;
        q = (W.float() / s_n).to(float8_e4m3fn)   (round to nearest even; |W / s| <= 448, no saturation)
    -> (q [N, K] float8_e4m3fn, s [N] fp32).  Rows are converted in chunks to bound the fp32 temporary."""
    N, K = w.shape
    q = torch.empty(N, K, dtype=torch.float8_e4m3fn, device=w.device)
    s = torch.empty(N, dtype=torch.float32, device=w.device)
    for a in range(0, N, rows_per_chunk):
        wf = w[a:a + rows_per_chunk].float()
        amax = wf.abs().amax(dim=1)
        sc = torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax))
        q[a:a + rows_per_chunk] = (wf / sc[:, None]).to(torch.float8_e4m3fn)
        s[a:a + rows_per_chunk] = sc
    return q, s


def quantize_kv_e4m3(x: torch.Tensor):
    """The FP8 KV cache's rule (kv_cache="fp8" of serving.BatchedDecoder; the kernels of csrc/kv_fp8.cu apply the
    same one), one fp32 scale per row of the last dim:
        amax = max|x|;  inv = 448 / amax (fp32);  code = (x.float() * inv).clamp(-448, 448) -> e4m3 (round to
        nearest even);  scale = amax / 448;  a row with amax == 0 gets all-zero codes and scale 0.
    The dequantised value is float(code) * scale.  -> (codes float8_e4m3fn, like x; scales fp32 x.shape[:-1])"""
    xf = x.float()
    amax = xf.abs().amax(dim=-1)
    nz = amax > 0
    lim = torch.full_like(amax, E4M3_MAX)  # tensor / tensor: IEEE division (a Python scalar would go through
    inv = torch.where(nz, lim / amax, torch.zeros_like(amax))  # a rounded reciprocal)
    codes = (xf * inv[..., None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    codes.view(torch.uint8).masked_fill_(~nz[..., None], 0)  # no negative zeros in an all-zero row
    return codes, amax / lim


W4_GROUP = 128  # consecutive k of one row sharing a scale and a zero point
W4_TILE = 16    # rows per packed tile (the m of the kernel's mma.sync m16n8k16)


def _w4_pack(q: torch.Tensor) -> torch.Tensor:
    """codes q uint8 [R, K] (0..15, R % 16 == 0) -> packed bytes [R / 16, 8 K] in the order
    vila_gemv_w4a16 reads (gemv_tma.cu): per 16-row tile [K/64][lane = 4g + c][mma step j][4 bytes], where
    the 8 nibbles of (tile, 64-k block b, g, c, j) are rows (g, g + 8) x k0 + (0..3), k0 = b + 16c + 4j,
    nibble p = 4 * (k % 2) + 2 * (k // 2 % 2) + (row is g + 8)."""
    R, K = q.shape
    t = q.view(R // W4_TILE, 2, 8, K // 64, 4, 4, 2, 2)      # [tile, h, g, b, c, j, kh, kl]
    t = t.permute(0, 3, 2, 4, 5, 7, 6, 1).reshape(-1, 2)    # [tile, b, g, c, j, kl, kh, h] -> nibble pairs
    return (t[:, 0] | (t[:, 1] << 4)).view(R // W4_TILE, 8 * K)


def _w4_unpack(packed: torch.Tensor, K: int) -> torch.Tensor:
    """inverse of _w4_pack -> codes uint8 [R, K]"""
    T = packed.shape[0]
    nib = torch.stack([packed & 15, packed >> 4], dim=-1)   # [T, 8K, 2]
    t = nib.view(T, K // 64, 8, 4, 4, 2, 2, 2)              # [tile, b, g, c, j, kl, kh, h]
    return t.permute(0, 7, 2, 1, 3, 4, 6, 5).reshape(T * W4_TILE, K)


def quantize_w4_groups(w: torch.Tensor, rows_per_chunk: int = 16384):
    """Weight-only 4-bit with a scale and a zero point per group of 128 consecutive k of a row (the
    reference's TinyChat W4A16 / AWQ format, round to nearest, no calibration data).  Per row n and group g,
    in fp32 on the bf16 values:
        lo = min(0, min w), hi = max(0, max w);  s = bf16((hi - lo) / 15), or 1 if that is 0
        z = clamp(round(-lo / s), 0, 15);  q = clamp(round(w / s) + z, 0, 15)   (round half to even)
    dequantized (q - z) * s; zero is exact.  -> (packed uint8 [ceil(N/16), 8 K], s bf16 [N, K/128],
    z uint8 [N, K/128]).  The packed byte order is vila_gemv_w4a16's and known only to this module:
    dequantize_w4_groups reads it back.  Rows are converted in chunks to bound the fp32 temporary."""
    N, K = w.shape
    if K % W4_GROUP:
        raise ValueError(f"quantize_w4_groups: K = {K} is not a multiple of {W4_GROUP}")
    G = K // W4_GROUP
    rows_per_chunk = max(W4_TILE, rows_per_chunk // W4_TILE * W4_TILE)
    T = (N + W4_TILE - 1) // W4_TILE
    packed = torch.empty(T, 8 * K, dtype=torch.uint8, device=w.device)
    s = torch.empty(N, G, dtype=torch.bfloat16, device=w.device)
    z = torch.empty(N, G, dtype=torch.uint8, device=w.device)
    for a in range(0, N, rows_per_chunk):
        wf = w[a:a + rows_per_chunk].float().view(-1, G, W4_GROUP)
        lo = wf.amin(dim=2).clamp(max=0)
        hi = wf.amax(dim=2).clamp(min=0)
        sc = ((hi - lo) / 15).to(torch.bfloat16).float()
        sc = torch.where(sc == 0, torch.ones_like(sc), sc)
        zp = torch.round(-lo / sc).clamp(0, 15)
        q = (torch.round(wf / sc[..., None]) + zp[..., None]).clamp(0, 15).to(torch.uint8).view(-1, K)
        n = q.shape[0]
        if n % W4_TILE:  # the last tile: rows past N are zero codes
            q = torch.cat([q, q.new_zeros(W4_TILE - n % W4_TILE, K)])
        packed[a // W4_TILE:a // W4_TILE + q.shape[0] // W4_TILE] = _w4_pack(q)
        s[a:a + n] = sc.to(torch.bfloat16)
        z[a:a + n] = zp.to(torch.uint8)
    return packed, s, z


def dequantize_w4_groups(packed: torch.Tensor, s: torch.Tensor, z: torch.Tensor) -> torch.Tensor:
    """(packed, s, z) of quantize_w4_groups -> the weights it stands for, (q - z) * s in fp32 [N, K]"""
    N, G = s.shape
    K = G * W4_GROUP
    q = _w4_unpack(packed, K)[:N].float().view(N, G, W4_GROUP)
    return ((q - z.float()[..., None]) * s.float()[..., None]).view(N, K)


class Qwen2ForCausalLM(nn.Module):
    def __init__(self, cfg: Qwen2Config, device="cuda", dtype=torch.bfloat16):
        super().__init__()
        self.config = cfg
        self.vocab_size = cfg.vocab_size
        m = _Holder()
        m.embed_tokens = Embedding(cfg.vocab_size, cfg.hidden_size, device, dtype)
        m.layers = nn.ModuleList([Qwen2DecoderLayer(cfg, device, dtype)
                                  for _ in range(cfg.num_hidden_layers)])
        m.norm = _Holder()
        m.norm.weight = _param(torch.empty(cfg.hidden_size, device=device, dtype=dtype))
        self.model = m
        self.lm_head = _Holder()
        if getattr(cfg, "tie_word_embeddings", False):
            # Qwen2.5-0.5B/1.5B/3B tie lm_head to the input embedding: ONE tensor, like HF tie_weights
            self.lm_head.weight = m.embed_tokens.weight
        else:
            self.lm_head.weight = _param(torch.empty(cfg.vocab_size, cfg.hidden_size, device=device,
                                                     dtype=dtype))
        # HF Qwen2RotaryEmbedding: inv_freq = 1 / theta^(arange(0, D, 2) / D), fp32
        D = cfg.head_dim
        self.inv_freq = (1.0 / (cfg.rope_theta ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))
                         ).to(device)
        self.generation_config = None
        self._decoder = None
        self._prefill_graphs = {}
        self.decode_weights = "bf16"
        self._fp8_weights = None
        self._w4_weights = None

    # ---- HF-style accessors ----
    @property
    def device(self):
        return self.lm_head.weight.device

    @property
    def dtype(self):
        return self.lm_head.weight.dtype

    def get_input_embeddings(self):
        return self.model.embed_tokens

    def get_output_embeddings(self):
        return self.lm_head

    # ---- prefill ----
    def new_cache(self, max_tokens: int, page_order=None) -> PagedKVCache:
        return PagedKVCache(self.config, max_tokens, self.device, self.dtype, page_order)

    def prefill_hidden_graphed(self, inputs_embeds: torch.Tensor, cache: PagedKVCache) -> torch.Tensor:
        """Same as prefill_hidden for the first chunk of a sequence (cache.length == 0), replayed
        from a CUDA graph cached per (S, cache): the ~230 launches of a prefill are submitted with no
        per-kernel host work, so PDL overlap is not throttled by Python.  The returned tensor is a
        static graph output: consume it before the next call with the same key."""
        S = inputs_embeds.shape[0]
        if cache.length != 0 or S == 0 or S > 4096:
            # long prompts (video) are not launch-bound, and a captured graph would pin GBs of
            # intermediates in its private pool
            return self.prefill_hidden(inputs_embeds, cache)
        # the captured graph bakes in per-layer K/V pointers (pool[li, 0/1]: they depend on n_pages)
        # and the page table: key on the pool geometry too and keep the cache alive in the entry so
        # the allocator cannot hand the same address to a differently-shaped pool
        key = (S, cache.pool.data_ptr(), tuple(cache.pool.shape), cache.page_table.data_ptr())
        ent = self._prefill_graphs.get(key)
        if ent is not None and ent[3] is not cache:
            ent = None  # a different cache object at a recycled address: re-capture
        if ent is None:
            if len(self._prefill_graphs) >= 8:  # bound the private pools held by cached graphs
                self._prefill_graphs.pop(next(iter(self._prefill_graphs)))
            static_in = torch.empty(S, self.config.hidden_size, dtype=self.dtype, device=self.device)
            static_in.copy_(inputs_embeds)
            self.prefill_hidden(static_in, cache)  # warm-up (allocator, function attributes)
            cache.length = 0
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                static_out = self.prefill_hidden(static_in, cache)
            cache.length = 0
            ent = (g, static_in, static_out, cache)
            self._prefill_graphs[key] = ent
        g, static_in, static_out, _ = ent
        static_in.copy_(inputs_embeds)
        g.replay()
        cache.length = S
        return static_out

    def prefill_hidden(self, inputs_embeds: torch.Tensor, cache: PagedKVCache,
                       position_ids: Optional[torch.Tensor] = None) -> torch.Tensor:
        """inputs_embeds [S, hidden] appended to `cache`; returns the final hidden states [S, hidden]
        BEFORE the last RMSNorm (the caller norms only the rows it needs)."""
        cfg = self.config
        S = inputs_embeds.shape[0]
        Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        p0 = cache.length
        assert p0 + S <= cache.max_tokens, "KV cache too small"
        if position_ids is None:
            position_ids = torch.arange(p0, p0 + S, dtype=torch.int32, device=self.device)
        else:
            position_ids = position_ids.to(device=self.device, dtype=torch.int32).contiguous()
        x = inputs_embeds.to(self.dtype).contiguous().clone()
        fused_rope = D == 128 and 0 < S <= 384
        # cos / sin once per request (shared by all layers and heads)
        table = ops.rope_table(position_ids, D, self.inv_freq) if S > 0 and D % 16 == 0 else None
        for li, layer in enumerate(self.model.layers):
            h = ops.rmsnorm(x, layer.input_layernorm.weight, cfg.rms_norm_eps)
            # short chunks: projection + RoPE + cache append in one kernel; else two kernels
            qkv = ops.linear_qkv_rope(h, layer._qkv_w, layer._qkv_b, table, Hq, Hkv, D, cache.k(li),
                                      cache.v(li), cache.page_table, p0, static_w=True) if fused_rope else None
            if qkv is None:
                qkv = ops.linear(h, layer._qkv_w, layer._qkv_b, static_w=True)
                if table is not None:
                    ops.rope_kv_append_table(qkv, table, Hq, Hkv, D, cache.k(li), cache.v(li),
                                             cache.page_table, p0)
                else:
                    ops.rope_kv_append(qkv, position_ids, Hq, Hkv, D, self.inv_freq, cache.k(li),
                                       cache.v(li), cache.page_table, p0)
            q = qkv.view(S, Hq + 2 * Hkv, D)[:, :Hq]
            attn = ops.fmha(q, cache.k(li), cache.v(li), B=1, Sq=S, Sk=p0 + S, causal=True,
                            scale=D ** -0.5, page_table=cache.page_table)
            ops.linear(attn.view(S, Hq * D), layer.self_attn.o_proj.weight, residual=x, out=x, static_w=True)
            h = ops.rmsnorm(x, layer.post_attention_layernorm.weight, cfg.rms_norm_eps)
            a = ops.linear(h, layer._gu_w, swiglu=True, static_w=True)
            ops.linear(a, layer.mlp.down_proj.weight, residual=x, out=x, static_w=True)
        cache.length = p0 + S
        return x

    def logits_from_hidden(self, hidden: torch.Tensor) -> torch.Tensor:
        """final RMSNorm + lm_head for the given rows [R, hidden] -> [R, V] (bf16 like HF)."""
        h = ops.rmsnorm(hidden.contiguous().clone(), self.model.norm.weight, self.config.rms_norm_eps)
        if h.shape[0] == 1:
            return ops.gemv(h[0], self.lm_head.weight, static_w=True).view(1, -1)
        return ops.linear(h, self.lm_head.weight, static_w=True)

    def forward_packed(self, inputs_embeds: torch.Tensor, attention_mask: torch.Tensor,
                       position_ids: torch.Tensor, seqlens_in_batch: torch.Tensor) -> torch.Tensor:
        """Packed (varlen) forward: inputs_embeds [1, T, H] holds the sequences back to back
        (model/packing.py), `seqlens_in_batch` their lengths; rows past sum(seqlens) (the reference's
        dummy token / pad_to_multiple_of rows, mask 0) take no part in attention.  Equivalent of HF
        Qwen2 + flash_attn_varlen_func(cu_seqlens) under the reference's `_get_unpad_data` patch
        (llava/model/utils/packing.py:12-36): GEMMs / norms / RoPE once over all T rows, block-diagonal
        causal attention as one wgmma FMHA launch per segment.  Returns logits [1, T, V]."""
        cfg = self.config
        Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        x = inputs_embeds[0].to(self.dtype).contiguous().clone()
        T = x.shape[0]
        lens = [int(n) for n in seqlens_in_batch.tolist()]
        assert sum(lens) <= T, "seqlens_in_batch exceed the packed length"
        pos = position_ids[0].to(device=self.device, dtype=torch.int32).clamp(min=0).contiguous()
        for layer in self.model.layers:
            h = ops.rmsnorm(x, layer.input_layernorm.weight, cfg.rms_norm_eps)
            qkv = ops.linear(h, layer._qkv_w, layer._qkv_b, static_w=True)
            ops.rope_kv_append(qkv, pos, Hq, Hkv, D, self.inv_freq)  # RoPE in place, no cache
            q3 = qkv.view(T, Hq + 2 * Hkv, D)
            attn = torch.zeros(T, Hq, D, dtype=self.dtype, device=self.device)
            o = 0
            for n in lens:
                if n > 0:
                    ops.fmha(q3[o:o + n, :Hq], q3[o:o + n, Hq:Hq + Hkv], q3[o:o + n, Hq + Hkv:], B=1,
                             Sq=n, Sk=n, causal=True, scale=D ** -0.5, out=attn[o:o + n])
                o += n
            ops.linear(attn.view(T, Hq * D), layer.self_attn.o_proj.weight, residual=x, out=x, static_w=True)
            h = ops.rmsnorm(x, layer.post_attention_layernorm.weight, cfg.rms_norm_eps)
            a = ops.linear(h, layer._gu_w, swiglu=True, static_w=True)
            ops.linear(a, layer.mlp.down_proj.weight, residual=x, out=x, static_w=True)
        return self.logits_from_hidden(x)[None]

    def forward(self, inputs_embeds: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                position_ids: Optional[torch.Tensor] = None, past_key_values=None, labels=None,
                use_cache: bool = False, seqlens_in_batch: Optional[torch.Tensor] = None, **kw):
        """Qwen2ForCausalLM.forward(inputs_embeds=[B,S,H]) -> namespace(logits=[B,S,V], loss=None).
        Padded positions (attention_mask False) are removed before the kernels and returned as 0.
        seqlens_in_batch: the row is a PACKED batch (forward_packed)."""
        if inputs_embeds.dim() == 2:
            inputs_embeds = inputs_embeds[None]
        if seqlens_in_batch is not None:
            out = self.forward_packed(inputs_embeds, attention_mask, position_ids, seqlens_in_batch)
            loss = None
            if labels is not None:
                shift_logits = out[:, :-1].float().reshape(-1, self.vocab_size)
                shift_labels = labels[:, 1:].reshape(-1).to(out.device).long()
                loss = torch.nn.functional.cross_entropy(shift_logits, shift_labels, ignore_index=-100)
            return SimpleNamespace(logits=out, loss=loss, past_key_values=None)
        B, S, _ = inputs_embeds.shape
        out = torch.zeros(B, S, self.vocab_size, dtype=self.dtype, device=self.device)
        for b in range(B):
            emb = inputs_embeds[b]
            keep = None
            if attention_mask is not None:
                keep = attention_mask[b].to(torch.bool)
                emb = emb[keep]
            if emb.shape[0] == 0:
                continue
            cache = self.new_cache(emb.shape[0])
            pos = None if position_ids is None else (position_ids[b][keep] if keep is not None
                                                     else position_ids[b])
            hid = self.prefill_hidden(emb, cache, pos)
            lg = self.logits_from_hidden(hid)
            if keep is None:
                out[b] = lg
            else:
                out[b][keep] = lg
        loss = None
        if labels is not None:
            # training loss is out of scope (SURVEY §2 row 14); provided for API completeness
            shift_logits = out[:, :-1].float().reshape(-1, self.vocab_size)
            shift_labels = labels[:, 1:].reshape(-1).to(out.device)
            loss = torch.nn.functional.cross_entropy(shift_logits, shift_labels, ignore_index=-100)
        return SimpleNamespace(logits=out, loss=loss, past_key_values=None)

    __call__ = forward

    # ---- decode ----
    def set_decode_weights(self, fmt: str) -> None:
        """Weights the single-stream greedy decoder (GraphDecoder: generate's greedy path, stream_greedy,
        sequence-parallel greedy generate) streams per token.
          "bf16"  the parameters themselves (default); frees any FP8 copies.
          "fp8"   e4m3 copies with one fp32 scale per output row (quantize_e4m3_rows) of every layer's
                  fused qkv, o_proj, interleaved gate/up and down_proj weights and of lm_head (a tied
                  lm_head is quantized as its own copy).  Half the bytes per token; for NVILA-8B the
                  copies take ~7.1 GB next to the bf16 weights, which stay.
          "w4a16" 4-bit copies with a bf16 scale and a uint8 zero point per group of 128 k
                  (quantize_w4_groups, run by vila_gemv_w4a16) of the same layer weights; lm_head gets an
                  e4m3 copy as in "fp8" mode (TinyChat / AWQ keep the output layer out of 4-bit).  For
                  NVILA-8B 3.96 GB per token.  Every linear K must be a multiple of 128 (ValueError
                  before anything is quantized).
        The copies are plain attributes: state_dict() and save_pretrained do not change, and switching
        modes frees the previous ones.  The continuous-batching engine (serving.BatchedDecoder /
        generate_batch, built after this call) runs the same copies with vila_gemv_batch_fp8 /
        vila_gemv_batch_w4a16.  What stays bf16 in every mode: the prefill (prompt K/V and last hidden
        state), the vision tower and projector, the eager sampling / logits-processor path and the embedding
        gather.  Every call drops the cached decoder (its graphs bake in weight pointers)."""
        if fmt not in ("bf16", "fp8", "w4a16"):
            raise ValueError(f"decode weights must be 'bf16', 'fp8' or 'w4a16', got {fmt!r}")
        if fmt == "w4a16":
            cfg = self.config
            ks = {"hidden_size": cfg.hidden_size, "num_attention_heads * head_dim":
                  cfg.num_attention_heads * cfg.head_dim, "intermediate_size": cfg.intermediate_size}
            bad = [f"{k} = {v}" for k, v in ks.items() if v % W4_GROUP]
            if bad:
                raise ValueError(f"w4a16 decode weights need every linear K to be a multiple of {W4_GROUP}: "
                                 + ", ".join(bad))
        self._decoder = None
        self._fp8_weights = None
        self._w4_weights = None
        if fmt == "w4a16":
            with torch.no_grad():
                layers = [SimpleNamespace(qkv=quantize_w4_groups(layer._qkv_w),
                                          o=quantize_w4_groups(layer.self_attn.o_proj.weight),
                                          gu=quantize_w4_groups(layer._gu_w),
                                          down=quantize_w4_groups(layer.mlp.down_proj.weight))
                          for layer in self.model.layers]
                self._w4_weights = SimpleNamespace(layers=layers, lm_head=quantize_e4m3_rows(self.lm_head.weight))
        if fmt == "fp8":
            with torch.no_grad():
                layers = [SimpleNamespace(qkv=quantize_e4m3_rows(layer._qkv_w),
                                          o=quantize_e4m3_rows(layer.self_attn.o_proj.weight),
                                          gu=quantize_e4m3_rows(layer._gu_w),
                                          down=quantize_e4m3_rows(layer.mlp.down_proj.weight))
                          for layer in self.model.layers]
                self._fp8_weights = SimpleNamespace(layers=layers, lm_head=quantize_e4m3_rows(self.lm_head.weight))
        self.decode_weights = fmt

    def decoder(self, max_new_tokens: int):
        """Greedy decode engine: the CUDA graph of per-layer kernels, reused while it holds enough tokens."""
        if self._decoder is None or self._decoder.max_new < max_new_tokens:
            self._decoder = GraphDecoder(self, max(max_new_tokens, 128))
        return self._decoder

    @torch.inference_mode()
    def generate(self, inputs_embeds: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                 generation_config=None, max_new_tokens: Optional[int] = None, do_sample=None,
                 eos_token_id=_UNSET, pad_token_id=None, logits_processor=None, temperature=None,
                 top_p=None, top_k=None, sp_runner=None, **kw) -> torch.Tensor:
        """HF GenerationMixin.generate(inputs_embeds=...) contract: returns ONLY the new ids
        [B, <=max_new_tokens] (pad-filled after EOS).  sp_runner: a sp.SequenceParallelPrefill ->
        the prompt is prefilled sequence-parallel across its group (greedy, batch size 1)."""
        gc = generation_config or self.generation_config
        refused = unsupported_generation_options(gc, kw)
        if refused:
            raise NotImplementedError("generate: greedy / temperature-top-k-top-p sampling / logits processors are "
                                      "implemented; not " + ", ".join(refused))

        def pick(name, given, default):
            if given is not None:
                return given
            v = getattr(gc, name, None) if gc is not None else None
            return default if v is None else v

        max_new = pick("max_new_tokens", max_new_tokens, None)
        if max_new is None:
            max_len = pick("max_length", None, 20)
            max_new = max(1, max_len - inputs_embeds.shape[-2])
        sample = bool(pick("do_sample", do_sample, False))
        # eos_token_id=None passed explicitly means "never stop" (benchmarks, parity tests)
        eos = None if eos_token_id is None else pick(
            "eos_token_id", None if eos_token_id is _UNSET else eos_token_id, None)
        eos_ids = [] if eos is None else ([eos] if isinstance(eos, int) else list(eos))
        pad = pick("pad_token_id", pad_token_id, eos_ids[0] if eos_ids else 0)
        if inputs_embeds.dim() == 2:
            inputs_embeds = inputs_embeds[None]
        outs = []
        for b in range(inputs_embeds.shape[0]):
            emb = inputs_embeds[b]
            if attention_mask is not None:
                emb = emb[attention_mask[b].to(torch.bool)]
            if sp_runner is not None and (sample or logits_processor or inputs_embeds.shape[0] != 1):
                raise NotImplementedError("sequence-parallel generate: greedy decoding, batch size 1")
            if sample or logits_processor:
                ids = self._generate_eager(emb, max_new, eos_ids, sample, logits_processor,
                                           pick("temperature", temperature, 1.0),
                                           pick("top_p", top_p, 1.0), pick("top_k", top_k, 0))
            else:
                ids = self._generate_greedy(emb, max_new, eos_ids, sp_runner=sp_runner)
            outs.append(ids)
        n = max(len(o) for o in outs)
        res = torch.full((len(outs), n), pad, dtype=torch.long, device=self.device)
        for b, o in enumerate(outs):
            res[b, :len(o)] = torch.tensor(o, dtype=torch.long, device=self.device)
        return res

    def _generate_greedy(self, emb: torch.Tensor, max_new: int, eos_ids: List[int],
                         check_every: int = 16, sp_runner=None) -> List[int]:
        S = emb.shape[0]
        dec = self.decoder(max_new)
        if sp_runner is not None:
            # sequence-parallel prefill (vila_b200/sp.py): every rank ends with the COMPLETE K/V in
            # its paged pool (in-place all-gather), so the greedy decode then runs replicated on
            # every rank from the same last hidden state -> identical ids everywhere
            from .. import sp
            plan = sp.make_plan(S, sp_runner.world, sp_runner.rank)
            cache = dec.cache_for(plan.padded_len + max_new,
                                  page_order_fn=lambda n: sp.sp_cache_page_order(plan, n),
                                  order_key=("sp", plan.world, plan.rank, plan.padded_len))
            padded = emb.new_zeros((plan.padded_len, emb.shape[1]))
            padded[:S] = emb
            hid_local, _ = sp_runner.prefill_hidden(plan.extract_local(padded), plan, pool=cache.pool)
            cache.length = S
            last = sp_runner.last_token_hidden(hid_local, plan)
            self.last_prefill_hidden = last.clone()
            dec.start(last, cache)
        else:
            cache = dec.cache_for(S + max_new)
            hid = self.prefill_hidden_graphed(emb, cache)
            dec.start(hid[-1], cache)
        done = 0
        ids: List[int] = []
        while done < max_new:
            n = min(check_every, max_new - done)
            dec.run(n)
            done += n
            if eos_ids:
                ids = dec.tokens(done)
                hit = [i for i, t in enumerate(ids) if t in eos_ids]
                if hit:
                    return ids[:hit[0] + 1]
        return dec.tokens(done)

    def stream_greedy(self, emb: torch.Tensor, generation_config=None, chunk_tokens: int = 8,
                      max_new_tokens: Optional[int] = None):
        """Greedy decode as a generator of id chunks (serving: `generate_content(stream=True)`): the
        loop stays on the device (CUDA graph); the host drains the token history every `chunk_tokens`
        tokens, which is also where EOS is noticed."""
        gc = generation_config or self.generation_config
        max_new = max_new_tokens or getattr(gc, "max_new_tokens", None)
        if max_new is None:
            max_new = max(1, (getattr(gc, "max_length", None) or 20) - emb.shape[0])
        eos = getattr(gc, "eos_token_id", None)
        eos_ids = [] if eos is None else ([eos] if isinstance(eos, int) else list(eos))
        with torch.inference_mode():
            S = emb.shape[0]
            dec = self.decoder(max_new)
            cache = dec.cache_for(S + max_new)
            hid = self.prefill_hidden_graphed(emb, cache)
            dec.start(hid[-1], cache)
            done = 0
            while done < max_new:
                n = min(chunk_tokens, max_new - done)
                dec.run(n)
                ids = dec.tokens(done + n)[done:]
                done += n
                hit = [i for i, t in enumerate(ids) if t in eos_ids]
                if hit:
                    yield ids[:hit[0] + 1]
                    return
                yield ids

    def _generate_eager(self, emb, max_new, eos_ids, sample, processors, temperature, top_p, top_k):
        """Non-graph path: logits come from the same kernels; the token choice (sampling /
        logits processors such as xgrammar, llava_arch.py:802-821) is host-side plumbing."""
        S = emb.shape[0]
        cache = self.new_cache(S + max_new)
        hid = self.prefill_hidden(emb, cache)
        logits = self.logits_from_hidden(hid[-1:])[0]
        ids: List[int] = []
        for _ in range(max_new):
            lg = logits.float()
            if processors:
                hist = torch.tensor([ids], dtype=torch.long, device=self.device)
                for proc in processors:
                    lg = proc(hist, lg[None])[0]
            if sample:
                lg = lg / max(temperature, 1e-5)
                if top_k and top_k > 0:
                    kth = torch.topk(lg, top_k).values[-1]
                    lg = lg.masked_fill(lg < kth, float("-inf"))
                probs = torch.softmax(lg, -1)
                if top_p < 1.0:
                    sp, si = torch.sort(probs, descending=True)
                    cut = torch.cumsum(sp, 0) - sp > top_p
                    sp = sp.masked_fill(cut, 0)
                    probs = torch.zeros_like(probs).scatter(0, si, sp)
                    probs = probs / probs.sum()
                tok = int(torch.multinomial(probs, 1))
            else:
                tok = int(torch.argmax(lg))
            ids.append(tok)
            if tok in eos_ids:
                break
            e = self.model.embed_tokens(torch.tensor([tok], device=self.device))
            hid = self.prefill_hidden(e, cache)
            logits = self.logits_from_hidden(hid)[0]
        return ids


class GraphDecoder:
    """Greedy decode loop living entirely on the device: per token 5 launches per layer + lm_head
    GEMV(argmax) + finalize (token history, position++, next embedding gather), captured in a CUDA
    graph and replayed without host synchronisation (the reference runs ~400 launches and one D2H
    stopping-criteria sync per token, SURVEY §3.1 HOT LOOP C).

    The decoder streams the weights of the LLM's decode-weight mode at construction
    (Qwen2ForCausalLM.set_decode_weights): in "fp8" mode every GEMV of start() and of each step, lm_head
    included, runs vila_gemv_fp8 on the e4m3 copies, so the first token is an fp8 lm_head result too.  In
    "w4a16" mode the layer GEMVs run vila_gemv_w4a16 on the 4-bit copies and lm_head vila_gemv_fp8 on its
    e4m3 copy.  The prompt's K/V and last hidden state come from the bf16 prefill in every mode."""

    MAX_SPLITS = 64

    def __init__(self, llm: Qwen2ForCausalLM, max_new: int):
        self.llm = llm
        cfg = llm.config
        dev, dt = llm.device, llm.dtype
        self.max_new = max_new
        # None unless in that mode.  Held here: the graphs bake in their pointers
        self.fp8 = llm._fp8_weights
        self.w4 = llm._w4_weights
        Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        self.num_splits = 8
        self.x = torch.zeros(cfg.hidden_size, device=dev, dtype=dt)
        self.qkv = torch.zeros((Hq + 2 * Hkv) * D, device=dev, dtype=dt)
        self.attn = torch.zeros(Hq * D, device=dev, dtype=dt)
        self.act = torch.zeros(cfg.intermediate_size, device=dev, dtype=dt)
        self.key = torch.zeros(1, device=dev, dtype=torch.int64)
        self.token = torch.zeros(1, device=dev, dtype=torch.int32)
        self.hist = torch.zeros(max_new + 8, device=dev, dtype=torch.int32)
        self.step = torch.zeros(1, device=dev, dtype=torch.int32)
        self.position = torch.zeros(1, device=dev, dtype=torch.int32)
        self.ws = torch.zeros(Hkv * self.MAX_SPLITS * (Hq // Hkv) * (D + 2), device=dev,
                              dtype=torch.float32)
        self.counters = torch.zeros(Hkv, device=dev, dtype=torch.int32)
        # long-context path (vila_decode_attention_split): fp32 split partials + their log-sum-exp
        self.o_partial = torch.zeros(self.MAX_SPLITS * Hq * D, device=dev, dtype=torch.float32)
        self.lse = torch.zeros(self.MAX_SPLITS * Hq, device=dev, dtype=torch.float32)
        self.split_tokens = 0  # > 0: the long-context path is active for the current cache
        self.cache: Optional[PagedKVCache] = None
        self.graphs = {}  # (num_splits, split_tokens) -> captured CUDA graph of one decode step (for self.cache)

    @property
    def graph(self):
        return self.graphs.get((self.num_splits, self.split_tokens))

    @property
    def launches_per_step(self) -> int:
        """kernels of one decode step: 5 per layer (7 on the long-context path: RoPE/append, split-KV
        attention, combine) + lm_head GEMV + finalize"""
        return (7 if self.split_tokens else 5) * self.llm.config.num_hidden_layers + 2

    LONG_CTX = 1024  # above: the wgmma split-KV path

    def pick_splits(self, ctx: int):
        """-> (num_splits, split_tokens).  Up to 512 tokens: 0 = one CTA per query head, nothing to
        combine (a pure latency chain at these sizes).  Up to 2048: 8 splits = one thread-block cluster
        per KV head of the SIMT kernel (DSMEM combine), split_tokens = 0.  Long contexts
        (video: 16K-66K tokens = 34-135 MB of K/V per layer) are a bandwidth problem: the wgmma FMHA
        kernel in split-KV mode, one CTA per SM (Hkv * splits <= #SMs), every split a whole number of
        128-token pages and all splits of (nearly) equal length."""
        if ctx <= 512:
            return 0, 0   # one CTA per query head, no split / combine (decode_attn_head_kernel)
        if ctx <= self.LONG_CTX:
            return 8, 0   # SIMT split-KV kernel, one 8-CTA cluster per KV head
        Hkv = self.llm.config.num_key_value_heads
        sms = torch.cuda.get_device_properties(self.llm.device).multi_processor_count
        pages = (ctx + PAGE - 1) // PAGE
        per_head = max(1, min(self.MAX_SPLITS, sms // Hkv))
        pps = (pages + per_head - 1) // per_head          # pages per split
        return (pages + pps - 1) // pps, pps * PAGE

    def cache_for(self, tokens: int, page_order_fn=None, order_key=None) -> PagedKVCache:
        """(Re)use a cache big enough; the graphs bake in the pool / page-table pointers.
        page_order_fn(n_pages) -> physical page of each logical 128-token block (sequence-parallel
        prefill: the zigzag all-gather layout, sp.sp_cache_page_order); order_key identifies it."""
        if (self.cache is None or self.cache.max_tokens < tokens
                or getattr(self, "_order_key", None) != order_key):
            n_tok = max(tokens, 1024)
            order = page_order_fn((n_tok + PAGE - 1) // PAGE) if page_order_fn is not None else None
            self.cache = self.llm.new_cache(n_tok, order)
            self._order_key = order_key
            self.graphs = {}
        self.cache.length = 0
        self.num_splits, self.split_tokens = self.pick_splits(self.cache.max_tokens if tokens > self.LONG_CTX
                                                              else tokens)
        return self.cache

    def _weights(self, li: Optional[int]):
        """-> (qkv, o, gate/up, down) of layer li, or lm_head for li None: each a dict of ops.gemv's
        weight arguments (w, and w_scale in fp8 mode, w_scale and w_zero for w4a16 layers)"""
        llm = self.llm
        if self.w4 is not None:
            if li is None:
                return dict(w=self.w4.lm_head[0], w_scale=self.w4.lm_head[1])
            f = self.w4.layers[li]
            return tuple(dict(w=p, w_scale=s, w_zero=z) for p, s, z in (f.qkv, f.o, f.gu, f.down))
        if self.fp8 is not None:
            if li is None:
                return dict(w=self.fp8.lm_head[0], w_scale=self.fp8.lm_head[1])
            f = self.fp8.layers[li]
            return tuple(dict(w=q, w_scale=s) for q, s in (f.qkv, f.o, f.gu, f.down))
        if li is None:
            return dict(w=llm.lm_head.weight)
        layer = llm.model.layers[li]
        return tuple(dict(w=w) for w in (layer._qkv_w, layer.self_attn.o_proj.weight, layer._gu_w,
                                         layer.mlp.down_proj.weight))

    def _lm_head(self):
        cfg = self.llm.config
        ops.gemv(self.x, norm_w=self.llm.model.norm.weight, norm_eps=cfg.rms_norm_eps, argmax_key=self.key,
                 write_out=False, static_w=True, **self._weights(None))

    def _step(self):
        llm, cfg, cache = self.llm, self.llm.config, self.cache
        Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        for li, layer in enumerate(llm.model.layers):
            w_qkv, w_o, w_gu, w_down = self._weights(li)
            ops.gemv(self.x, bias=layer._qkv_b, norm_w=layer.input_layernorm.weight,
                     norm_eps=cfg.rms_norm_eps, out=self.qkv, static_w=True, **w_qkv)
            if self.split_tokens:
                ops.decode_attention_split(self.qkv, self.position, cache.k(li), cache.v(li),
                                           cache.page_table, self.attn, self.o_partial, self.lse,
                                           llm.inv_freq, Hq, Hkv, D, self.num_splits, self.split_tokens,
                                           D ** -0.5)  # separate combine launch (no fused last-CTA combine:
                #                              one CTA per KV head would walk all partial rows serially)
            else:
                ops.decode_attention(self.qkv, self.position, cache.k(li), cache.v(li), cache.page_table,
                                     self.attn, self.ws, self.counters, llm.inv_freq, Hq, Hkv, D,
                                     self.num_splits, D ** -0.5)
            ops.gemv(self.attn, residual=self.x, out=self.x, static_w=True, **w_o)
            ops.gemv(self.x, norm_w=layer.post_attention_layernorm.weight,
                     norm_eps=cfg.rms_norm_eps, swiglu=True, out=self.act, static_w=True, **w_gu)
            ops.gemv(self.act, residual=self.x, out=self.x, static_w=True, **w_down)
        self._lm_head()
        ops.argmax_finalize(self.key, self.token, self.hist, self.step, self.position,
                            llm.model.embed_tokens.weight, self.x)

    def start(self, last_hidden: torch.Tensor, cache: PagedKVCache) -> None:
        """Seed the loop from the prefill: first new token = argmax(lm_head(norm(last_hidden)))."""
        assert cache is self.cache
        llm = self.llm
        self.step.zero_()
        self.key.zero_()
        self.position.fill_(cache.length - 1)  # finalize increments -> position of the new token
        self.x.copy_(last_hidden)
        self._lm_head()
        ops.argmax_finalize(self.key, self.token, self.hist, self.step, self.position,
                            llm.model.embed_tokens.weight, self.x)
        self._started = 1

    def run(self, n_tokens: int) -> None:
        """Produce n_tokens more tokens (the first call's first token already exists from start())."""
        n = n_tokens
        if self._started == 1:
            n -= 1
            self._started = 2
        if n <= 0:
            return
        g = self.graphs.get((self.num_splits, self.split_tokens))
        if g is None:
            # warm-up launch outside capture is not allowed to change state: capture directly
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._step()
            self.graphs[(self.num_splits, self.split_tokens)] = g
        for _ in range(n):
            g.replay()
        self.cache.length += n

    def tokens(self, n: int) -> List[int]:
        return self.hist[:n].tolist()

