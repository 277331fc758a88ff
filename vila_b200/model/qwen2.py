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

from collections import deque
from types import SimpleNamespace
from typing import List, Optional, Sequence

import torch
from torch import nn

from .. import grammar as grammar_rule
from .. import ops
from ..logprobs import MAX_TOP_LOGPROBS, TokenLogprob, check_top
from ..penalties import PenaltyParams
from ..sampling import SamplingParams, signed64
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


def sampling_for_generate(generation_config, rows: int, temperature=None, top_k=None,
                          top_p=None) -> List[SamplingParams]:
    """The SamplingParams of a do_sample generate, one per batch row: temperature / top_k / top_p from the
    explicit values first, then the generation config (1.0 / 0 / 1.0 when neither sets them; HF's default
    GenerationConfig has top_k 50).  Every row gets the config's `seed` attribute when it carries one, else a draw
    from the host torch default generator in row order (serving.sampling_for_requests), so torch.manual_seed
    reproduces a run.  Out-of-range values are ValueErrors."""
    from ..serving import sampling_for_requests
    gc = generation_config

    def pick(name, given, default):
        if given is not None:
            return given
        v = getattr(gc, name, None) if gc is not None else None
        return default if v is None else v

    params = SamplingParams(temperature=float(pick("temperature", temperature, 1.0)),
                            top_k=int(pick("top_k", top_k, 0)), top_p=float(pick("top_p", top_p, 1.0)),
                            seed=getattr(gc, "seed", None) if gc is not None else None)
    return sampling_for_requests(params, rows)


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
        # tensor / tensor: IEEE division on every device (CUDA runs a Python scalar divisor as a multiplication by
        # its rounded reciprocal, which misses amax / 448 by an ulp for some rows)
        sc = torch.where(amax > 0, amax / torch.full_like(amax, E4M3_MAX), torch.ones_like(amax))
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
        sc = ((hi - lo) / torch.full_like(hi, 15.0)).to(torch.bfloat16).float()  # IEEE division, as above
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


def _decode_chunks(dec, max_new: int, chunk_tokens: int, eos_ids, ahead: bool):
    """Run a started GraphDecoder for up to max_new tokens in chunks of chunk_tokens and yield (ids, entries or None)
    per chunk, cut after the first EOS id.  Each chunk's rows alone are read back, in one copy (GraphDecoder.read).
    ahead: chunk k + 1 is enqueued before the host waits for chunk k, so the device decodes while the host builds the
    logprob entries; a chunk decoded past EOS is then dropped.  Without it each chunk is read before the next runs, so
    nothing is decoded past the chunk that holds EOS.  A chunk shorter than asked for ends the stream: the decoder
    stopped because its grammar terminated."""
    reads = deque()
    done = 0
    while done < max_new or reads:
        if done < max_new:
            n = min(chunk_tokens, max_new - done)
            dec.run(n)
            reads.append((n, dec.read(done + n, start=done)))
            done += n
            if ahead and len(reads) == 1 and done < max_new:
                continue
        want, read = reads.popleft()
        ids, entries = read()
        hit = next((i + 1 for i, t in enumerate(ids) if t in eos_ids), None)
        if hit is not None:
            yield ids[:hit], None if entries is None else entries[:hit]
            return
        if ids:
            yield ids, entries
        if len(ids) < want:
            return


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
        """Weights the single-stream decoder (GraphDecoder: generate's greedy and sampled paths, stream_tokens /
        stream_greedy, sequence-parallel greedy generate) streams per token.
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
        state), the vision tower and projector, the eager logits-processor path and the embedding gather.
        Every call drops the cached decoder (its graphs bake in weight pointers)."""
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
        """Single-stream decode engine (greedy or sampled): the CUDA graphs of per-layer kernels, reused while it
        holds enough tokens."""
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
        the prompt is prefilled sequence-parallel across its group (greedy, batch size 1).
        do_sample without logits_processor samples on the device in the graph decoder (temperature, top_k, top_p
        from the kwargs, else the generation config; the rule of vila_b200/sampling.py).  Each row's seed is the
        config's `seed` attribute when it has one, else a draw from the host torch default generator in row order
        (torch.manual_seed reproduces a run).  With logits_processor the eager path chooses on the host."""
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
        per_row = None
        if sample and not logits_processor and sp_runner is None:
            per_row = sampling_for_generate(gc, inputs_embeds.shape[0], temperature, top_k, top_p)
        outs = []
        for b in range(inputs_embeds.shape[0]):
            emb = inputs_embeds[b]
            if attention_mask is not None:
                emb = emb[attention_mask[b].to(torch.bool)]
            if sp_runner is not None and (sample or logits_processor or inputs_embeds.shape[0] != 1):
                raise NotImplementedError("sequence-parallel generate: greedy decoding, batch size 1")
            if per_row is not None:
                ids = self._generate_greedy(emb, max_new, eos_ids, sampling=per_row[b])
            elif sample or logits_processor:
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
                         check_every: int = 16, sp_runner=None,
                         sampling: Optional[SamplingParams] = None, grammar=None) -> List[int]:
        """The graph decoder's loop: greedy, or sampled on the device with `sampling` (its seed set); constrained by
        `grammar` (a matcher with xgrammar's GrammarMatcher interface, GraphDecoder.start) when given."""
        S = emb.shape[0]
        if sp_runner is not None and grammar is not None:
            raise NotImplementedError("sequence-parallel decode: grammar-constrained decoding is not implemented")
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
            dec.start(hid[-1], cache, sampling, **({} if grammar is None else {"grammar": grammar}))
        # without EOS ids nothing is read until the end: one chunk of max_new
        chunks = _decode_chunks(dec, max_new, check_every if eos_ids else max_new, eos_ids, ahead=False)
        return [t for ids, _ in chunks for t in ids]

    def stream_greedy(self, emb: torch.Tensor, generation_config=None, chunk_tokens: int = 8,
                      max_new_tokens: Optional[int] = None):
        """Greedy decode as a generator of id chunks (serving: `generate_content(stream=True)`): the
        loop stays on the device (CUDA graph); the host drains the token history every `chunk_tokens`
        tokens, which is also where EOS is noticed."""
        return self.stream_tokens(emb, generation_config, chunk_tokens, max_new_tokens)

    def stream_tokens(self, emb: torch.Tensor, generation_config=None, chunk_tokens: int = 8,
                      max_new_tokens: Optional[int] = None, sampling: Optional[SamplingParams] = None,
                      logprobs: Optional[int] = None, penalties: Optional[PenaltyParams] = None, grammar=None):
        """stream_greedy, or with `sampling` (a SamplingParams with its seed set) the same loop sampled on the
        device: the ids are those of generate(do_sample=True) with the same parameters and seed.
        logprobs: None yields id lists; n in 0..20 yields (ids, [TokenLogprob ...]) per chunk, one entry per id (the
        token's log-probability under the raw row and its n most likely alternatives, vila_b200/logprobs.py),
        truncated at EOS as the ids are.  penalties: a PenaltyParams applies OpenAI's presence / frequency penalties
        over the ids generated so far before each choice (vila_b200/penalties.py).  grammar: a matcher with xgrammar's
        GrammarMatcher interface, whose token bitmask constrains every choice (vila_b200/grammar.py); the stream ends
        when it terminates.  All run on the device in the graph decoder (GraphDecoder.start)."""
        if sampling is not None and not sampling.greedy and sampling.seed is None:
            raise ValueError("stream_tokens: sampling needs a seed")
        if logprobs is not None:
            check_top(logprobs)
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
            dec.start(hid[-1], cache, sampling, logprobs=logprobs, penalties=penalties,
                      **({} if grammar is None else {"grammar": grammar}))
            # read-ahead only with logprobs: it overlaps building their entries with decoding, and would otherwise
            # only add a chunk of decoding past EOS
            for ids, entries in _decode_chunks(dec, max_new, chunk_tokens, eos_ids, ahead=logprobs is not None):
                yield ids if logprobs is None else (ids, entries)

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
    """Decode loop living entirely on the device: per token 5 launches per layer + lm_head
    GEMV(argmax) + finalize (token history, position++, next embedding gather), captured in a CUDA
    graph and replayed without host synchronisation (the reference runs ~400 launches and one D2H
    stopping-criteria sync per token, SURVEY §3.1 HOT LOOP C).

    `graphs` holds one step graph per mode and attention plan, captured on first use and keyed by (sampled,
    penalised, logprobs on, num_splits, split_tokens) (_graph_key).  A request's parameters are device scalars that
    start() writes, so every request of one mode and plan replays the same graph.

    Sampled decoding (start(..., params) with non-greedy SamplingParams) has the same number of launches as greedy:
    lm_head writes the bf16 logits row and vila_sample_finalize draws the token from it (the rule of
    vila_b200/sampling.py, t = the step counter) in place of argmax_finalize.

    Logprobs and presence / frequency penalties (start(..., logprobs=n, penalties=PenaltyParams)) add a launch each.
    The number of alternatives n is a device scalar (the history rows hold 20), so one graph serves every n:
      greedy + logprobs   lm_head writes the bf16 row and keeps its fused argmax key; argmax_finalize; then
                          vila_token_logprobs_row on the row (the ids are the greedy graph's)
      sampled + logprobs  the sampled step, then vila_token_logprobs_row on the row
      penalties           lm_head writes the row, vila_apply_penalties_row writes pen_logits over the decoder's own
                          int32 history, vila_sample_finalize chooses from pen_logits (at inv_T = 0 the first index of
                          the max: the greedy rule), then vila_token_logprobs_row on the raw row when logprobs are on
    The rules are those of vila_b200/logprobs.py and vila_b200/penalties.py; token_logprobs() reads the entries back.
    Their buffers are allocated on first use; a request with neither option runs the greedy or sampled graph.

    Grammar-constrained decoding (start(..., grammar=matcher), the rule of vila_b200/grammar.py) needs the matcher's
    token bitmask on the device before each choice, and the matcher needs each id on the host before it can fill the
    next mask.  So a constrained step is two graphs, keyed by _graph_key() + ("body",) / ("choose",):
      body    the layers and lm_head writing the bf16 row
      choose  [vila_apply_penalties_row] + vila_apply_token_bitmask_row + vila_sample_finalize (at inv_T = 0 the greedy
              rule over the allowed ids) + [vila_token_logprobs_row on the raw row]
    and the host loop for token t is: replay body(t); accept_token(t - 1); fill_next_token_bitmask into a pinned buffer
    and copy it to the device; replay choose(t); copy the token back; replay body(t + 1); wait for the token.  The
    matcher's host work overlaps the body, and the host's wait overlaps the next body (_run_constrained).  The loop
    stops when the matcher terminates (the body replayed for the step after the stop token is not used).  A request without a grammar runs exactly its unconstrained graph.

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
        # sampled steps: the lm_head logits row and the request's parameters (device scalars read by the graph)
        self.logits = torch.zeros(llm.lm_head.weight.shape[0], device=dev, dtype=dt)
        self.inv_temperature = torch.zeros(1, device=dev, dtype=torch.float32)
        self.top_k = torch.zeros(1, device=dev, dtype=torch.int32)
        self.top_p = torch.ones(1, device=dev, dtype=torch.float32)
        self.seed = torch.zeros(1, device=dev, dtype=torch.int64)
        self.sampled = False  # mode of the current request (start())
        self.penalised = False
        self.top_n: Optional[int] = None  # logprobs: alternatives per token, None = off
        self.ws = torch.zeros(Hkv * self.MAX_SPLITS * (Hq // Hkv) * (D + 2), device=dev,
                              dtype=torch.float32)
        self.counters = torch.zeros(Hkv, device=dev, dtype=torch.int32)
        # long-context path (vila_decode_attention_split): fp32 split partials + their log-sum-exp
        self.o_partial = torch.zeros(self.MAX_SPLITS * Hq * D, device=dev, dtype=torch.float32)
        self.lse = torch.zeros(self.MAX_SPLITS * Hq, device=dev, dtype=torch.float32)
        self.split_tokens = 0  # > 0: the long-context path is active for the current cache
        self.cache: Optional[PagedKVCache] = None
        self.graphs = {}  # _graph_key() -> captured CUDA graph of one decode step (for self.cache)
        # logprobs / penalties buffers, allocated on first use (_ensure_logprobs / _ensure_penalties)
        self.lp_hist = self.top_ids = self.top_lp = self.lp_n = self.lp_ws = self.lp_counter = None
        self.pen_logits = self.presence = self.frequency = None
        # grammar-constrained requests: the matcher, its mask buffers (allocated on first use, _ensure_grammar), the
        # ids chosen so far (on the host) and whether the matcher has terminated
        self.grammar = None
        self.mask = self.mask_host = self.mask_np = self.masked = self.token_host = self.token_ready = None
        self.grammar_ids: List[int] = []
        self.finished = False

    def _graph_key(self):
        """what a step graph depends on besides the cache: the current request's mode and the attention plan"""
        return self.sampled, self.penalised, self.top_n is not None, self.num_splits, self.split_tokens

    @property
    def launches_per_step(self) -> int:
        """kernels of one decode step: 5 per layer (7 on the long-context path: RoPE/append, split-KV
        attention, combine) + lm_head GEMV + finalize (argmax or sample), in either mode; + 1 with penalties
        (vila_apply_penalties_row), + 1 with logprobs (vila_token_logprobs_row) and + 1 with a grammar
        (vila_apply_token_bitmask_row)"""
        return ((7 if self.split_tokens else 5) * self.llm.config.num_hidden_layers + 2 + int(self.penalised)
                + int(self.top_n is not None) + int(self.grammar is not None))

    def _ensure_logprobs(self) -> None:
        if self.lp_hist is None:
            dev, cols = self.llm.device, self.max_new + 8
            self.lp_hist = torch.zeros(cols, device=dev, dtype=torch.float32)
            self.top_ids = torch.zeros(cols, MAX_TOP_LOGPROBS, device=dev, dtype=torch.int32)
            self.top_lp = torch.zeros(cols, MAX_TOP_LOGPROBS, device=dev, dtype=torch.float32)
            self.lp_n = torch.zeros(1, device=dev, dtype=torch.int32)
            self.lp_ws, self.lp_counter = ops.logprobs_row_workspace(self.logits.numel(), dev)

    def _ensure_penalties(self) -> None:
        if self.pen_logits is None:
            dev = self.llm.device
            self.pen_logits = torch.zeros_like(self.logits)
            self.presence = torch.zeros(1, device=dev, dtype=torch.float32)
            self.frequency = torch.zeros(1, device=dev, dtype=torch.float32)

    def _ensure_grammar(self) -> None:
        if self.mask is None:
            dev, W = self.llm.device, grammar_rule.bitmask_words(self.logits.numel())
            self.mask = torch.zeros(W, device=dev, dtype=torch.int32)
            self.mask_host = torch.zeros(1, W, dtype=torch.int32, pin_memory=True)
            self.mask_np = self.mask_host.numpy()
            self.masked = torch.zeros_like(self.logits)
            self.token_host = torch.zeros(1, dtype=torch.int32, pin_memory=True)
            self.token_ready = torch.cuda.Event()

    def _fill_mask(self) -> None:
        """the matcher's bitmask for the next token -> the device (asynchronous copy from pinned memory; the pinned
        buffer is refilled only after _wait_token has waited for the step that follows this copy)"""
        self.grammar.fill_next_token_bitmask(self.mask_host)
        if not grammar_rule.any_allowed(self.mask_np, self.logits.numel()):
            raise ValueError(f"GraphDecoder: the grammar allows no token after {len(self.grammar_ids)} tokens "
                             "(an all-zero bitmask)")
        self.mask.copy_(self.mask_host[0], non_blocking=True)

    def _copy_token(self) -> None:
        """enqueue the copy of the token just chosen to pinned memory, and an event after it"""
        self.token_host.copy_(self.token, non_blocking=True)
        self.token_ready.record()

    def _wait_token(self) -> None:
        """wait for _copy_token's event -> grammar_ids"""
        self.token_ready.synchronize()
        self.grammar_ids.append(int(self.token_host[0]))

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
        """the bf16 row when a kernel after lm_head reads it, the fused argmax key when argmax_finalize chooses (greedy
        + logprobs: both, from the same values)"""
        chooses_from_row = self.sampled or self.penalised or self.grammar is not None
        row = chooses_from_row or self.top_n is not None
        ops.gemv(self.x, norm_w=self.llm.model.norm.weight, norm_eps=self.llm.config.rms_norm_eps,
                 out=self.logits if row else None, write_out=row,
                 argmax_key=None if chooses_from_row else self.key, static_w=True, **self._weights(None))

    def _finalize(self):
        """the token (arg-max, or the draw in sampled mode; from the penalised and / or grammar-masked row when those
        are on) -> history, step++, position++, next x; then the token's logprobs on the raw row when they are on"""
        emb = self.llm.model.embed_tokens.weight
        row = self.logits
        if self.penalised:
            row = ops.apply_penalties_row(row, self.hist, self.step, self.presence, self.frequency, out=self.pen_logits)
        if self.grammar is not None:
            row = ops.apply_token_bitmask_row(row, self.mask, out=self.masked)
        if self.sampled or self.penalised or self.grammar is not None:
            ops.sample_finalize(row, self.inv_temperature, self.top_k, self.top_p, self.seed, self.step, self.token,
                                self.hist, self.position, emb, self.x)
        else:
            ops.argmax_finalize(self.key, self.token, self.hist, self.step, self.position, emb, self.x)
        if self.top_n is not None:  # n = self.lp_n, a device scalar: one graph for every n
            ops.token_logprobs_row(self.logits, self.token, self.step, lp_hist=self.lp_hist, workspace=self.lp_ws,
                                   counter=self.lp_counter, top_ids=self.top_ids, top_lp=self.top_lp,
                                   n_used=self.lp_n)

    def _step(self):
        self._body()
        self._finalize()

    def _body(self):
        """the step up to the logits: the layers and lm_head"""
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

    def start(self, last_hidden: torch.Tensor, cache: PagedKVCache, params: Optional[SamplingParams] = None, *,
              logprobs: Optional[int] = None, penalties: Optional[PenaltyParams] = None, grammar=None) -> None:
        """Seed the loop from the prefill: first new token = argmax(lm_head(norm(last_hidden))), or with
        non-greedy `params` (seed set) the draw of token index 0 from those logits; the following steps
        run the matching graph.  params None or greedy: exactly the greedy path.
        logprobs: None, or n in 0..20: every token's log-probability and its n most likely alternatives under the raw
        row (vila_b200/logprobs.py), entry 0 from this first row (token_logprobs()).  penalties: a PenaltyParams,
        applied to every row before the choice (vila_b200/penalties.py; the first token's history is empty, so its row
        is unchanged); None or both values 0 is the path without them.  grammar: a matcher with xgrammar's
        GrammarMatcher interface (fill_next_token_bitmask, accept_token, is_terminated) whose token bitmask masks every
        row before the choice (vila_b200/grammar.py); its bitmask width must be ceil(V / 32) for this model's V.  The
        first token's mask is filled here, before the first row is computed; an all-zero mask is a ValueError and an id
        the matcher does not accept a RuntimeError.  None of these works with a sequence-parallel cache
        (NotImplementedError)."""
        assert cache is self.cache
        top_n = None if logprobs is None else check_top(logprobs)
        penalised = penalties is not None and not penalties.off
        if (top_n is not None or penalised) and getattr(self, "_order_key", None) is not None:
            raise NotImplementedError("sequence-parallel decode: logprobs and penalties are not implemented")
        if grammar is not None and getattr(self, "_order_key", None) is not None:
            raise NotImplementedError("sequence-parallel decode: grammar-constrained decoding is not implemented")
        self.top_n, self.penalised = top_n, penalised
        self.grammar, self.grammar_ids, self.finished = grammar, [], False
        if top_n is not None:
            self._ensure_logprobs()
            self.lp_n.fill_(top_n)
        if penalised:
            self._ensure_penalties()
            self.presence.fill_(penalties.presence)
            self.frequency.fill_(penalties.frequency)
        self.sampled = params is not None and not params.greedy
        if (penalised or grammar is not None) and not self.sampled:
            self.inv_temperature.fill_(0.0)  # vila_sample_finalize's greedy rule on the penalised / masked row
        if self.sampled:
            if params.seed is None:
                raise ValueError("GraphDecoder.start: sampling needs a seed (serving.sampling_for_requests draws one)")
            self.inv_temperature.fill_(params.inv_temperature)
            self.top_k.fill_(min(params.top_k, 2 ** 31 - 1))
            self.top_p.fill_(params.top_p)
            self.seed.fill_(signed64(params.seed))
        self.step.zero_()
        self.key.zero_()
        self.position.fill_(cache.length - 1)  # finalize increments -> position of the new token
        self.x.copy_(last_hidden)
        if grammar is not None:
            self._ensure_grammar()
            self._fill_mask()
        self._lm_head()
        self._finalize()
        if grammar is not None:
            self._copy_token()
            self._wait_token()
        self._started = 1

    def run(self, n_tokens: int) -> None:
        """Produce n_tokens more tokens (the first call's first token already exists from start())."""
        n = n_tokens
        if self._started == 1:
            n -= 1
            self._started = 2
        if n <= 0:
            return
        if self.grammar is not None:
            self._run_constrained(n)
            return
        g = self._graph(self._graph_key(), self._step)
        for _ in range(n):
            g.replay()
        self.cache.length += n

    def _graph(self, key, body):
        g = self.graphs.get(key)
        if g is None:
            # warm-up launch outside capture is not allowed to change state: capture directly
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                body()
            self.graphs[key] = g
        return g

    def _run_constrained(self, n: int) -> None:
        """up to n more tokens of a grammar-constrained request, one host round trip each (see the class docstring);
        fewer when the matcher terminates, which sets `finished`.  Within the call, body(t + 1) is enqueued right after
        choose(t) and before the host waits for token t: it reads only device state (the token's embedding that
        choose(t) writes), so the device does not idle while the host wakes up, accepts the token and fills the next
        mask.  The first body of each call is enqueued by the call itself."""
        if self.finished:
            return
        key = self._graph_key()
        body, choose = self._graph(key + ("body",), self._body), self._graph(key + ("choose",), self._finalize)
        m = self.grammar
        body.replay()
        for i in range(n):
            if not m.accept_token(self.grammar_ids[-1]):
                raise RuntimeError(f"GraphDecoder: the grammar matcher rejected token {self.grammar_ids[-1]}, which "
                                   "its own bitmask allowed")
            if m.is_terminated():
                self.finished = True
                return
            self._fill_mask()
            choose.replay()
            self._copy_token()
            if i + 1 < n:
                body.replay()
            self._wait_token()
            self.cache.length += 1

    def tokens(self, n: int) -> List[int]:
        return self.hist[:n].tolist()

    def token_logprobs(self, n_tokens: int, start: int = 0) -> List[TokenLogprob]:
        """tokens start .. n_tokens - 1 of the current request with their logprobs and top alternatives (start() with
        logprobs): only those rows are copied to the host, so a stream that reads each chunk's new tokens does work
        in proportion to them.  ValueError without logprobs."""
        if self.top_n is None:
            raise ValueError("GraphDecoder.token_logprobs: the current request was started without logprobs")
        return self.read(n_tokens, start)()[1]

    def read(self, n_tokens: int, start: int = 0):
        """Tokens start .. n_tokens - 1 of the current request as a function returning (ids, entries): entries are their
        TokenLogprobs with logprobs, else None.  Only their rows are copied to the host, in one copy.  With logprobs
        that copy is enqueued now and the function waits for it alone, so steps enqueued in between decode while the
        host builds the entries (_decode_chunks reads chunk k while chunk k + 1 runs).  Ids alone, which no caller
        reads ahead, are copied by the function with a plain blocking copy."""
        n = self.top_n
        a, b = max(0, start), min(n_tokens, self.hist.numel())
        if self.grammar is not None:  # the ids are on the host already, and there may be fewer than asked for
            b = min(b, len(self.grammar_ids))
            a = min(a, b)
            if n is None:
                ids = self.grammar_ids[a:b]
                return lambda: (ids, None)
        if n is None:
            return lambda: (self.hist[a:b].tolist(), None)
        if a >= b:
            return lambda: ([], [])
        # one device-to-host copy: [id, logprob bits, top ids..., top logprob bits...] per token
        rows = torch.cat([self.hist[a:b, None], self.lp_hist[a:b, None].view(torch.int32), self.top_ids[a:b, :n],
                          self.top_lp[a:b, :n].view(torch.int32)], dim=1)
        done = None
        if rows.is_cuda:
            host = torch.empty(rows.shape, dtype=torch.int32, pin_memory=True)
            host.copy_(rows, non_blocking=True)
            done = torch.cuda.Event()
            done.record()
            rows = host

        def wait():
            if done is not None:
                done.synchronize()
            ids = rows[:, 0].tolist()
            lps = rows[:, 1].view(torch.float32).tolist()
            top_i = rows[:, 2:2 + n].tolist()
            top_v = rows[:, 2 + n:].contiguous().view(torch.float32).tolist()
            return ids, [TokenLogprob(t, lp, list(zip(ti, tv))) for t, lp, ti, tv in zip(ids, lps, top_i, top_v)]

        return wait

