"""Continuous batching over ONE shared paged KV pool (SURVEY §8 f3).

The reference serialises requests (`serving/server.py:65-73` semaphore / global lock around
`model.generate_content`, one HF `generate` loop per request).  Decode at batch 1 is a pure weight
stream (14.14 GB per token for NVILA-8B): serving B requests from the same stream multiplies the
tokens per byte by B.  Here:

  * one paged pool `[L, 2, P, 128, Hkv, D]` holds the K/V of every slot; slot s owns the page-table row
    `page_tables[s]` (vLLM-style indirection: the kernels only ever see (pool, page-table row));
  * a request is admitted by prefilling it into a free slot (the ordinary wgmma prefill path writes
    straight into that slot's pages), its first token comes from the prefill;
  * ONE CUDA graph advances all slots by one token: per layer RMSNorm → q/k/v GEMM (wgmma
    kernel, M = slots: every weight byte is read once for the whole batch) → batched decode
    attention (`vila_decode_attention_batch`: one CTA per (query head, slot), RoPE + KV append fused,
    per-slot position and page-table row, idle slots skipped) → o-proj GEMM(+res) → RMSNorm → gate/up
    GEMM (SwiGLU epilogue) → down GEMM(+res); then lm_head GEMM, greedy arg-max, embedding gather and
    position++ — all on the device, no host sync per token;
  * slots longer than HEAD_KERNEL_TOKENS (video, dynamic-S2) are attended by the batched split-KV
    kernel (`vila_decode_attention_split_batch`) in the same step; which kernel serves a slot follows
    only from that slot's own length, so a request's ids never depend on its neighbours;
  * finished slots (EOS / budget) are harvested and refilled between graph replays;
  * in the LLM's "fp8" / "w4a16" decode-weight modes (Qwen2ForCausalLM.set_decode_weights) the step's
    GEMMs run `vila_gemv_batch_*` on the quantized copies (up to 16 slots per launch, every weight byte
    read once per launch) and each slot's first token comes from the e4m3 lm_head; the prefill stays bf16;
  * with kv_cache="fp8" the pool holds e4m3 codes plus one fp32 scale per (token, KV head) row
    (quantize_kv_e4m3): a prompt is prefilled into a bf16 staging cache of one slot and converted into the
    slot's pages by vila_kv_quantize_fp8, and every slot, whatever its length, is attended by
    vila_decode_attention_fp8_batch (RoPE, e4m3 append and split-KV attention in one launch per layer);
  * with sampling=True each slot has its own temperature / top-k / top-p / seed (SamplingParams, the rule in
    vila_b200/sampling.py) in device arrays, and vila_sample_batch replaces the greedy arg-max, in the step graphs
    and for the first token at admission; a slot's draw depends only on its own logits, seed and token index;
  * with prefix_cache=True (vila_b200/prefix_cache.py) the full 128-token blocks of every admitted prompt are digested
    on the device (vila_prefix_block_hash) and kept in a trie of cached pages: a later prompt that starts with the same
    blocks at the same positions takes those pages into its page-table row and prefills only its suffix.  Full prompt
    pages are never written after the prefill (decode appends at positions >= S), so sharing needs no copy.  A hit
    request's ids equal those of a chunked prefill of its suffix over the donor's prefix pages; they may differ from
    its uncached ids, since the donor's prefill may have run its GEMMs at another M;
  * with logprobs=n (vila_b200/logprobs.py) vila_token_logprobs reads each step's logits row once the token is chosen
    and writes the token's log-probability and its n best alternatives into per-slot history buffers beside `hist`;
    the tokens are the same as without it;
  * with penalties=True (vila_b200/penalties.py) each slot has its own presence / frequency penalty in device arrays,
    and vila_apply_penalties writes the lm_head row with OpenAI's penalties over the slot's generated ids (`hist`) into
    a second buffer that the greedy arg-max or vila_sample_batch reads; logprobs keep reading the raw row.
"""
from __future__ import annotations

from collections import deque
from typing import Deque, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import ops
from .logprobs import TokenLogprob, check_top
from .penalties import PenaltyParams
from .prefix_cache import PrefixPages, random_keys
from .sampling import SamplingParams, signed64

PAGE = 128

# A slot of at most this many tokens (the new one included) is attended by decode_attn_head_kernel,
# longer slots by the batched split-KV kernel.  The head kernel could serve up to 4096 tokens (32-entry
# page table), but above ~1K tokens the split-KV kernel is faster (DESIGN.md §4); 2048 is the lowest
# threshold that leaves every slot of today's default 2048-token geometry on the head kernel.
HEAD_KERNEL_TOKENS = 16 * PAGE
# Split-KV configuration of the long slots: split j covers tokens [j*SPLIT_TOKENS, (j+1)*SPLIT_TOKENS).
# SPLIT_TOKENS is the same for every ladder entry, so a slot's result does not depend on the entry in
# use (the combine reads only the splits that hold tokens).  The ladder gives the number of splits
# launched per (slot, KV head), sized from the longest active slot, so that a batch of short slots does
# not launch thousands of CTAs that exit at once.  DESIGN.md §4 has the measurements behind both.
SPLIT_TOKENS = 1024
SPLIT_LADDER = (8, 16, 32, 68)
MAX_SLOT_TOKENS = SPLIT_LADDER[-1] * SPLIT_TOKENS  # 69,632: a 256-frame LongVILA request + 1K new tokens

KV_CACHE_FORMATS = ("bf16", "fp8")
# FP8 KV: split j covers tokens [j*FP8_SPLIT_TOKENS, (j+1)*FP8_SPLIT_TOKENS) for every slot length, so a slot's
# result does not depend on the ladder entry; the ladder (tokens covered) sizes the splits launched from the
# longest active slot.  DESIGN.md §4 has the measurements behind the split size.
FP8_SPLIT_TOKENS = 512
FP8_LADDER_TOKENS = (2048, 8192, 16384, 32768, MAX_SLOT_TOKENS)


def fp8_attention_config(longest: int) -> int:
    """splits launched by an fp8-KV decode step whose longest active slot holds `longest` tokens: those of the
    smallest ladder entry covering it"""
    for n in FP8_LADDER_TOKENS:
        if n >= longest:
            return (n + FP8_SPLIT_TOKENS - 1) // FP8_SPLIT_TOKENS
    raise ValueError(f"a slot of {longest} tokens exceeds the engine's limit ({MAX_SLOT_TOKENS})")


def attention_config(longest: int) -> Optional[int]:
    """Attention of a decode step whose longest active slot holds `longest` tokens (the run's appends
    included): None = decode_attn_head_kernel only, else the number of splits of the split-KV kernel
    (the smallest ladder entry covering `longest`)."""
    if longest <= HEAD_KERNEL_TOKENS:
        return None
    for n in SPLIT_LADDER:
        if n * SPLIT_TOKENS >= longest:
            return n
    raise ValueError(f"a slot of {longest} tokens exceeds the engine's limit ({MAX_SLOT_TOKENS})")


def slot_geometry(prompt_lens: Sequence[int], max_new_tokens: int, check_every: int, slots: int,
                  max_tokens_per_slot: Optional[int] = None) -> Tuple[int, Optional[int]]:
    """-> (max_tokens_per_slot, total_pages or None for slots * pages_per_slot).

    An explicit max_tokens_per_slot is kept as it is.  None sizes the slot from the requests: the
    smallest page multiple >= 2048 that holds the longest prompt + max_new_tokens + check_every (at most
    MAX_SLOT_TOKENS; a longer request is refused by generate_batch).  A batch that fits 2048 gets the
    2048-token geometry and its full pool; a larger slot gets a pool of the page budgets of the `slots`
    largest requests, so that one long request does not reserve `slots` long slots."""
    if max_tokens_per_slot is not None:
        return max_tokens_per_slot, None
    budgets = sorted(((n + max_new_tokens + check_every + PAGE - 1) // PAGE for n in prompt_lens), reverse=True)
    pages = min(max([2048 // PAGE] + budgets), MAX_SLOT_TOKENS // PAGE)
    if pages == 2048 // PAGE:
        return 2048, None
    return pages * PAGE, min(sum(min(b, pages) for b in budgets[:slots]), slots * pages)


class _SlotCache:
    """The view of one slot that Qwen2ForCausalLM.prefill_hidden needs (PagedKVCache duck type)."""

    def __init__(self, pool: torch.Tensor, page_table: torch.Tensor):
        self.pool, self.page_table = pool, page_table
        self.length = 0
        self.max_tokens = page_table.numel() * PAGE
        self.n_pages = pool.shape[2]

    def k(self, layer: int) -> torch.Tensor:
        return self.pool[layer, 0]

    def v(self, layer: int) -> torch.Tensor:
        return self.pool[layer, 1]


class PageAllocator:
    """Free list over the physical pages of the shared pool (host-side bookkeeping only)."""

    def __init__(self, n_pages: int):
        self.free: List[int] = list(range(n_pages - 1, -1, -1))  # pop() hands out page 0 first
        self.n_pages = n_pages

    def alloc(self, n: int) -> List[int]:
        if n > len(self.free):
            raise MemoryError(f"KV pool exhausted: {n} pages wanted, {len(self.free)} free of {self.n_pages}")
        return [self.free.pop() for _ in range(n)]

    def release(self, pages: Sequence[int]) -> None:
        self.free.extend(reversed(list(pages)))

    @property
    def available(self) -> int:
        return len(self.free)


class BatchedDecoder:
    """`slots` concurrent greedy decodes of one Qwen2ForCausalLM over a shared paged pool.

    Pages are handed out on demand (PageAllocator): a slot holds ceil(tokens / 128) pages, grows page by
    page while it decodes and returns them when it is released, so `total_pages` can be smaller than
    slots * pages_per_slot (long and short requests share the pool).  The page-table rows live on the
    device and are read by the kernels at every launch: changing them needs no graph re-capture.

    The decoder streams the weights of the LLM's decode-weight mode at construction (`decode_weights`):
    "bf16" runs the wgmma GEMMs on the parameters; "fp8" and "w4a16" run ops.gemv_batch on the copies
    set_decode_weights made, which the decoder holds (the captured graphs bake in their pointers).

    kv_cache "bf16" (default) keeps bf16 K/V in `pool`; "fp8" keeps e4m3 codes in `pool` and one fp32 scale per
    (layer, K|V, token, KV head) row in `pool_scale` (0.516x the bytes for head_dim 128), plus a bf16 staging
    cache of one slot (`staging`) that admit() prefills into.

    sampling False (default) picks every token greedily with torch.argmax.  True keeps per-slot device arrays of
    the sampling parameters (admit() writes them) and draws every token with vila_sample_batch, at token index
    `step_idx` of the slot; a slot admitted without parameters decodes greedily (temperature 0).

    prefix_cache False (default) prefills every prompt in full.  True shares the pages of full 128-token prompt blocks
    between requests whose prompts start alike (vila_b200/prefix_cache.py): `allocator` is then a PrefixPages,
    admit() prefills only the part of the prompt past the cached blocks, released blocks stay findable until their
    pages are needed, `prefix_stats` counts the work saved and clear_prefix_cache() drops the unused blocks.  The
    fp8 KV cache is not supported with it (its admission prefills into a bf16 staging cache, which would need the
    prefix in bf16).

    logprobs None (default) records no log-probabilities.  An int n in 0..20 keeps, beside `hist`, each token's
    log-probability under the raw model distribution (`lp_hist`) and its n most likely alternatives (`top_ids`,
    `top_lp`), written by vila_token_logprobs in every step graph and at admission; generated_logprobs(slot) reads
    them.

    penalties False (default) applies none.  True keeps per-slot fp32 `presence` / `frequency` arrays (admit() writes
    them; a slot admitted without PenaltyParams gets 0 and 0) and a bf16 [slots, V] buffer `pen_logits`: every step
    graph runs vila_apply_penalties on the lm_head output over the slot's generated ids, and the token is chosen from
    `pen_logits`.  The first token, chosen from the prefill logits, has no history and is never penalised."""

    def __init__(self, llm, slots: int = 8, max_tokens_per_slot: int = 2048, max_new: int = 1024,
                 total_pages: Optional[int] = None, kv_cache: str = "bf16", sampling: bool = False,
                 prefix_cache: bool = False, logprobs: Optional[int] = None, penalties: bool = False):
        if kv_cache not in KV_CACHE_FORMATS:
            raise ValueError(f"kv_cache must be one of {KV_CACHE_FORMATS}, got {kv_cache!r}")
        if prefix_cache and kv_cache == "fp8":
            raise ValueError("prefix_cache=True is not supported with kv_cache='fp8': the fp8 admission prefills into "
                             "a bf16 staging cache, which would need the cached prefix in bf16")
        self.kv_cache = kv_cache
        self.prefix_cache = bool(prefix_cache)
        self.logprobs = None if logprobs is None else check_top(logprobs)
        cfg = llm.config
        self.llm, self.slots = llm, slots
        self.decode_weights = getattr(llm, "decode_weights", "bf16")
        # None unless in that mode.  Held here: the graphs bake in their pointers
        self.fp8 = llm._fp8_weights if self.decode_weights == "fp8" else None
        self.w4 = llm._w4_weights if self.decode_weights == "w4a16" else None
        dev, dt = llm.device, llm.dtype
        Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        assert D == 128, "batched decode attention is specialised for head_dim 128"
        self.pages_per_slot = (max_tokens_per_slot + PAGE - 1) // PAGE
        assert self.pages_per_slot * PAGE <= MAX_SLOT_TOKENS, \
            f"slots of up to {MAX_SLOT_TOKENS} tokens (asked for {max_tokens_per_slot})"
        P = total_pages if total_pages is not None else slots * self.pages_per_slot
        L = cfg.num_hidden_layers
        fp8 = kv_cache == "fp8"
        self.pool = torch.zeros(L, 2, P, PAGE, Hkv, D, device=dev, dtype=torch.float8_e4m3fn if fp8 else dt)
        self.pool_scale = torch.zeros(L, 2, P, PAGE, Hkv, device=dev, dtype=torch.float32) if fp8 else None
        self.allocator = PrefixPages(P) if self.prefix_cache else PageAllocator(P)
        if self.prefix_cache:
            self.prefix_keys = random_keys()
        self.slot_pages: List[List[int]] = [[] for _ in range(slots)]
        # unassigned entries point at page 0; they are never dereferenced (tokens beyond a slot's length)
        self.page_tables = torch.zeros(slots, self.pages_per_slot, dtype=torch.int32, device=dev)
        self._pos_host = [-1] * slots  # host mirror of `positions` (advanced by run())
        self.positions = torch.full((slots,), -1, dtype=torch.int32, device=dev)  # < 0: idle slot
        self.x = torch.zeros(slots, cfg.hidden_size, device=dev, dtype=dt)
        self.attn = torch.zeros(slots, Hq * D, device=dev, dtype=dt)
        self.tokens = torch.zeros(slots, dtype=torch.int64, device=dev)
        self.max_new = max_new
        self.hist = torch.zeros(slots, max_new + 8, dtype=torch.int64, device=dev)
        self.step_idx = torch.zeros(slots, 1, dtype=torch.int64, device=dev)  # per-slot write column
        self.sampling = bool(sampling)
        if self.sampling:  # per-slot parameters of vila_sample_batch (admit() writes them)
            self.inv_temperature = torch.zeros(slots, dtype=torch.float32, device=dev)
            self.top_k = torch.zeros(slots, dtype=torch.int32, device=dev)
            self.top_p = torch.ones(slots, dtype=torch.float32, device=dev)
            self.seed = torch.zeros(slots, dtype=torch.int64, device=dev)
        if self.sampling or self.logprobs is not None:
            self._zero_pos = torch.zeros(1, dtype=torch.int32, device=dev)    # admission: row active, t = 0
            self._zero_step = torch.zeros(1, dtype=torch.int64, device=dev)
        if self.logprobs is not None:  # vila_token_logprobs writes column step_idx of each active slot
            self.lp_hist = torch.zeros(slots, max_new + 8, dtype=torch.float32, device=dev)
            self.top_ids = torch.zeros(slots, max_new + 8, self.logprobs, dtype=torch.int32, device=dev)
            self.top_lp = torch.zeros(slots, max_new + 8, self.logprobs, dtype=torch.float32, device=dev)
        self.penalties = bool(penalties)
        if self.penalties:  # per-slot parameters of vila_apply_penalties (admit() writes them) and its output rows
            self.presence = torch.zeros(slots, dtype=torch.float32, device=dev)
            self.frequency = torch.zeros(slots, dtype=torch.float32, device=dev)
            self.pen_logits = torch.zeros(slots, cfg.vocab_size, dtype=dt, device=dev)
        # attention configurations this slot size can need (attention_config): None, then ladder entries
        self.configs: List[Optional[int]] = [None] + [
            n for i, n in enumerate(SPLIT_LADDER)
            if self.pages_per_slot * PAGE > (SPLIT_LADDER[i - 1] * SPLIT_TOKENS if i else HEAD_KERNEL_TOKENS)]
        self.graphs: Dict[Optional[int], torch.cuda.CUDAGraph] = {}  # configuration -> step graph
        self.config: Optional[int] = None  # configuration of the last run()
        if fp8:
            # one slot of bf16 K/V with an identity page table: the prefill (and its FMHA over earlier chunks)
            # runs unchanged on it; configurations are split counts of the fp8 attention kernel
            self.staging = torch.zeros(L, 2, self.pages_per_slot, PAGE, Hkv, D, device=dev, dtype=dt)
            self.staging_pages = torch.arange(self.pages_per_slot, dtype=torch.int32, device=dev)
            tokens = self.pages_per_slot * PAGE
            self.configs = [fp8_attention_config(n) for i, n in enumerate(FP8_LADDER_TOKENS)
                            if i == 0 or tokens > FP8_LADDER_TOKENS[i - 1]]
            self.ws = torch.zeros(slots * Hq * self.configs[-1] * (D + 2), device=dev, dtype=torch.float32)
            self.counters = torch.zeros(slots * Hkv, device=dev, dtype=torch.int32)
        elif len(self.configs) > 1:
            n_max = self.configs[-1]
            # per-step copies of `positions` that hide the long slots from the head kernel and the short
            # ones from the split-KV kernel, and the split-KV work buffers (shared by all layers)
            self.pos_head = torch.full((slots,), -1, dtype=torch.int32, device=dev)
            self.pos_split = torch.full((slots,), -1, dtype=torch.int32, device=dev)
            self.o_partial = torch.zeros(slots * n_max * Hq * D, device=dev, dtype=torch.float32)
            self.lse = torch.zeros(slots * n_max * Hq, device=dev, dtype=torch.float32)
            self.counters = torch.zeros(slots * Hkv, device=dev, dtype=torch.int32)

    @property
    def launches_per_step(self) -> int:
        """library kernels of one step in the configuration of the last run(): 7 per layer (9 with the bf16
        split-KV kernel: RoPE/append and attention added; always 7 with the fp8 KV cache) + final RMSNorm and
        lm_head (+ vila_sample_batch with sampling, + vila_token_logprobs with logprobs, + vila_apply_penalties with
        penalties)"""
        per_layer = 7 if self.config is None or self.kv_cache == "fp8" else 9
        return (per_layer * self.llm.config.num_hidden_layers + 2 + (1 if self.sampling else 0)
                + (0 if self.logprobs is None else 1) + (1 if self.penalties else 0))

    # ---- prefix cache ---------------------------------------------------------------------------
    def prefix_digests(self, inputs_embeds: torch.Tensor) -> np.ndarray:
        """uint64 [S // 128, 2]: the digests of the prompt's full blocks under this decoder's keys (one
        vila_prefix_block_hash launch and one copy to the host)"""
        return ops.prefix_block_hash(inputs_embeds, *self.prefix_keys).cpu().numpy().view(np.uint64)

    def prefix_hits(self, digests: np.ndarray, S: int) -> List[int]:
        """cached pages an S-token prompt with these digests would take: at most (S - 1) // 128 blocks, so that at
        least one token is prefilled (it gives the first token) and the slot never writes into a shared page"""
        return self.allocator.match(digests, (S - 1) // PAGE)

    def _need_prefix_cache(self, what: str) -> None:
        if not self.prefix_cache:
            raise ValueError(f"{what} needs a decoder built with prefix_cache=True")

    @property
    def prefix_stats(self) -> Dict[str, int]:
        """lookups (admissions), hit_blocks / hit_tokens served from the cache, prefilled_tokens, cached_blocks (now)
        and evictions"""
        self._need_prefix_cache("prefix_stats")
        return dict(self.allocator.stats, cached_blocks=self.allocator.cached_blocks)

    def clear_prefix_cache(self) -> int:
        """drop every cached block that no live slot holds -> blocks dropped"""
        self._need_prefix_cache("clear_prefix_cache()")
        return self.allocator.clear()

    # ---- admission ------------------------------------------------------------------------------
    @torch.inference_mode()
    def admit(self, slot: int, inputs_embeds: torch.Tensor, params: Optional[SamplingParams] = None, *,
              digests: Optional[np.ndarray] = None, penalties: Optional[PenaltyParams] = None) -> None:
        """Prefill `inputs_embeds` [S, hidden] into the slot's pages and seed its decode state.  params: the slot's
        SamplingParams (sampling decoders only; None is greedy); its seed must be set.  digests: prefix_digests of
        the prompt, if the caller has them already (prefix-caching decoders).  penalties: the slot's PenaltyParams
        (decoders built with penalties=True only; None is 0 and 0).

        A prefix-caching decoder admits into an idle slot only (released, or never used), and if the admission raises
        it releases the slot again: the hit blocks are unpinned and the pages it took are returned, so a failed request
        leaves no page half-owned and no block registered over K/V that was not written."""
        if params is not None and not self.sampling:
            raise ValueError("admit(params=...) needs a decoder built with sampling=True")
        if penalties is not None and not self.penalties:
            raise ValueError("admit(penalties=...) needs a decoder built with penalties=True")
        if penalties is not None and not isinstance(penalties, PenaltyParams):
            raise ValueError(f"admit: penalties must be a PenaltyParams or None, got {type(penalties).__name__}")
        if self.sampling:
            params = params if params is not None else SamplingParams()
            if params.seed is None and not params.greedy:
                raise ValueError("admit: a sampled slot needs a seed (generate_batch draws one)")
        S = inputs_embeds.shape[0]
        assert S + 1 <= self.pages_per_slot * PAGE, "prompt longer than a slot"
        if not self.prefix_cache:
            self._fill(slot, inputs_embeds, params, 0, None, penalties)
            return
        if self.slot_pages[slot] or self._pos_host[slot] >= 0:
            raise ValueError(f"admit: slot {slot} is still in use: release() it first")
        if digests is None:
            digests = self.prefix_digests(inputs_embeds)
        hits = self.prefix_hits(digests, S)
        self.allocator.pin(hits)  # before any allocation: the hit pages cannot be evicted under this request
        self.slot_pages[slot] = list(hits)
        try:
            if hits:
                self.page_tables[slot, :len(hits)] = torch.tensor(hits, dtype=torch.int32,
                                                                  device=self.page_tables.device)
            self._fill(slot, inputs_embeds, params, PAGE * len(hits), digests, penalties)
        except BaseException:
            self.release(slot)
            raise
        self.allocator.stats["prefilled_tokens"] += S - PAGE * len(hits)

    def _fill(self, slot: int, inputs_embeds: torch.Tensor, params: Optional[SamplingParams], p0: int,
              digests: Optional[np.ndarray], penalties: Optional[PenaltyParams]) -> None:
        """admit()'s work once the slot's first p0 // 128 pages hold the cached prefix: pages for the rest, the prefill
        of inputs_embeds[p0:], registration of the new full blocks (prefix caching) and the first token"""
        llm = self.llm
        S = inputs_embeds.shape[0]
        self._ensure_pages(slot, S + 1)
        if self.kv_cache == "fp8":  # prefill in bf16, then one conversion into the slot's e4m3 pages
            hid = llm.prefill_hidden(inputs_embeds, _SlotCache(self.staging, self.staging_pages))
            ops.kv_quantize_fp8(self.staging, self.pool, self.pool_scale, self.page_tables[slot], S)
        elif p0:
            cache = _SlotCache(self.pool, self.page_tables[slot])
            cache.length = p0
            hid = llm.prefill_hidden(inputs_embeds[p0:], cache)
        else:
            hid = llm.prefill_hidden(inputs_embeds, _SlotCache(self.pool, self.page_tables[slot]))
        if self.prefix_cache:
            self.allocator.register(digests, self.slot_pages[slot], p0 // PAGE)
        if self.decode_weights == "bf16":
            logits = llm.logits_from_hidden(hid[-1:])
        else:  # the mode's lm_head, as GraphDecoder.start
            h = ops.rmsnorm(hid[-1:].contiguous(), llm.model.norm.weight, llm.config.rms_norm_eps)
            logits = ops.gemv_batch(h, **self._weights(None))
        if self.penalties:  # read by the step graphs only: token 0 has no history and is never penalised
            pen = penalties if penalties is not None else PenaltyParams()
            self.presence[slot] = pen.presence
            self.frequency[slot] = pen.frequency
        if self.sampling:  # token 0 by the same kernel: M = 1, t = 0
            self.inv_temperature[slot] = params.inv_temperature
            self.top_k[slot] = params.top_k
            self.top_p[slot] = params.top_p
            self.seed[slot] = signed64(params.seed or 0)
            i = slice(slot, slot + 1)
            ops.sample_batch(logits[:1], self.inv_temperature[i], self.top_k[i], self.top_p[i], self.seed[i],
                             self._zero_step, self._zero_pos, out=self.tokens[i])
            self.hist[slot, 0] = self.tokens[slot]
            self.step_idx[slot, 0] = 1
            self.x[i] = llm.model.embed_tokens.weight.index_select(0, self.tokens[i])
        else:
            tok = torch.argmax(logits[0].float())
            self.tokens[slot] = tok
            self.hist[slot, 0] = tok
            self.step_idx[slot, 0] = 1
            self.x[slot] = llm.model.embed_tokens.weight[tok]
        if self.logprobs is not None:  # entry 0 from the admission logits: M = 1, column 0
            self._logprobs(logits[:1], slice(slot, slot + 1), self._zero_step, self._zero_pos)
        self.positions[slot] = S  # position of the token just chosen == tokens cached so far
        self._pos_host[slot] = S

    def release(self, slot: int) -> None:
        self.positions[slot] = -1
        self._pos_host[slot] = -1
        self.allocator.release(self.slot_pages[slot])
        self.slot_pages[slot] = []

    def _ensure_pages(self, slot: int, n_tokens: int) -> None:
        """make sure the slot owns pages for its first n_tokens tokens"""
        need = min(self.pages_per_slot, (n_tokens + PAGE - 1) // PAGE) - len(self.slot_pages[slot])
        if need > 0:
            new = self.allocator.alloc(need)
            first = len(self.slot_pages[slot])
            self.slot_pages[slot].extend(new)
            self.page_tables[slot, first:first + need] = torch.tensor(new, dtype=torch.int32,
                                                                      device=self.page_tables.device)

    def _logprobs(self, logits: torch.Tensor, rows: slice, step: torch.Tensor, positions: torch.Tensor) -> None:
        top = dict(top_ids=self.top_ids[rows], top_lp=self.top_lp[rows]) if self.logprobs else {}
        ops.token_logprobs(logits, self.tokens[rows], step, positions, lp_hist=self.lp_hist[rows], **top)

    def _weights(self, li: Optional[int]):
        """quantized modes: (qkv, o, gate/up, down) of layer li, or lm_head for li None, each a dict of
        ops.gemv_batch's weight arguments"""
        q = self.w4 if self.w4 is not None else self.fp8
        if li is None:
            return dict(w=q.lm_head[0], w_scale=q.lm_head[1])
        f = q.layers[li]
        if self.w4 is not None:
            return tuple(dict(w=p, w_scale=s, w_zero=z) for p, s, z in (f.qkv, f.o, f.gu, f.down))
        return tuple(dict(w=w, w_scale=s) for w, s in (f.qkv, f.o, f.gu, f.down))

    # ---- one decode step for every active slot ----------------------------------------------------
    def _step(self, num_splits: Optional[int]) -> None:
        llm, cfg = self.llm, self.llm.config
        Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        x = self.x
        pos_head = self.positions
        fp8_kv = self.kv_cache == "fp8"
        if num_splits is not None and not fp8_kv:  # slot length pos + 1 picks the kernel (idle slots stay -1 in both)
            pos_head = self.pos_head
            long = self.positions >= HEAD_KERNEL_TOKENS
            pos_head.copy_(self.positions).masked_fill_(long, -1)
            self.pos_split.copy_(self.positions).masked_fill_(~long, -1)
        quant = self.decode_weights != "bf16"
        for li, layer in enumerate(llm.model.layers):
            h = ops.rmsnorm(x, layer.input_layernorm.weight, cfg.rms_norm_eps)
            if quant:
                w_qkv, w_o, w_gu, w_down = self._weights(li)
                qkv = ops.gemv_batch(h, bias=layer._qkv_b, static_w=True, **w_qkv)
            else:
                qkv = ops.linear(h, layer._qkv_w, layer._qkv_b, static_w=True)
            if fp8_kv:
                ops.decode_attention_fp8_batch(qkv, self.positions, self.pool[li, 0], self.pool[li, 1],
                                               self.pool_scale[li, 0], self.pool_scale[li, 1], self.page_tables,
                                               self.attn, self.ws, self.counters, llm.inv_freq, Hq, Hkv,
                                               num_splits, FP8_SPLIT_TOKENS, D ** -0.5)
            else:
                ops.decode_attention_batch(qkv, pos_head, self.pool[li, 0], self.pool[li, 1],
                                           self.page_tables, self.attn, llm.inv_freq, Hq, Hkv, D, D ** -0.5)
            if num_splits is not None and not fp8_kv:
                ops.decode_attention_split_batch(qkv, self.pos_split, self.pool[li, 0], self.pool[li, 1],
                                                 self.page_tables, self.attn, self.o_partial, self.lse,
                                                 self.counters, llm.inv_freq, Hq, Hkv, D, num_splits,
                                                 SPLIT_TOKENS, D ** -0.5)
            if quant:
                ops.gemv_batch(self.attn, residual=x, out=x, static_w=True, **w_o)
                h = ops.rmsnorm(x, layer.post_attention_layernorm.weight, cfg.rms_norm_eps)
                a = ops.gemv_batch(h, swiglu=True, static_w=True, **w_gu)
                ops.gemv_batch(a, residual=x, out=x, static_w=True, **w_down)
            else:
                ops.linear(self.attn, layer.self_attn.o_proj.weight, residual=x, out=x, static_w=True)
                h = ops.rmsnorm(x, layer.post_attention_layernorm.weight, cfg.rms_norm_eps)
                a = ops.linear(h, layer._gu_w, swiglu=True, static_w=True)
                ops.linear(a, layer.mlp.down_proj.weight, residual=x, out=x, static_w=True)
        h = ops.rmsnorm(x.clone(), llm.model.norm.weight, cfg.rms_norm_eps)
        if quant:
            logits = ops.gemv_batch(h, static_w=True, **self._weights(None))
        else:
            logits = ops.linear(h, llm.lm_head.weight, static_w=True)
        active = self.positions >= 0
        chosen_from = logits
        if self.penalties:  # idle rows (position < 0) are not written
            chosen_from = ops.apply_penalties(logits, self.hist, self.step_idx.view(-1), self.positions, self.presence,
                                              self.frequency, out=self.pen_logits)
        if self.sampling:  # idle slots (position < 0) keep their token
            ops.sample_batch(chosen_from, self.inv_temperature, self.top_k, self.top_p, self.seed, self.step_idx.view(-1),
                             self.positions, out=self.tokens)
        else:
            tok = torch.argmax(chosen_from.float(), dim=-1)
            self.tokens.copy_(torch.where(active, tok, self.tokens))
        if self.logprobs is not None:  # idle slots (position < 0) are not written
            self._logprobs(logits, slice(None), self.step_idx.view(-1), self.positions)
        col = self.step_idx.clamp(max=self.hist.shape[1] - 1)
        self.hist.scatter_(1, col, self.tokens[:, None])
        self.step_idx.add_(active[:, None].to(torch.int64))
        x.copy_(ops.embed_splice(llm.model.embed_tokens.weight, None, self.tokens.to(torch.int32)))
        self.positions.add_(active.to(torch.int32))

    @torch.inference_mode()
    def run(self, n_tokens: int) -> None:
        if not self.graphs:
            raise RuntimeError("call capture() (with every slot idle) before run()")
        longest = 0
        for s_ in range(self.slots):  # pages for the tokens this call will append
            if self._pos_host[s_] >= 0:
                self._ensure_pages(s_, self._pos_host[s_] + n_tokens + 1)
                self._pos_host[s_] += n_tokens
                longest = max(longest, self._pos_host[s_])  # tokens attended by the slot's last step
        longest = min(longest, self.pages_per_slot * PAGE)
        self.config = fp8_attention_config(longest) if self.kv_cache == "fp8" else attention_config(longest)
        g = self.graphs[self.config]
        for _ in range(n_tokens):
            g.replay()

    @torch.inference_mode()
    def capture(self) -> None:
        """Capture the step graph of every attention configuration this slot size can need.  Must be
        called with every slot idle (positions < 0): the capture launches the kernels once, idle slots
        are skipped by the attention kernels and leave no trace."""
        if self.graphs:
            return
        assert bool((self.positions < 0).all()), "capture() with idle slots only"
        saved = (self.tokens.clone(), self.hist.clone(), self.step_idx.clone(), self.x.clone())
        for c in self.configs:
            self._step(c)  # eager warm-up (allocator, function attributes); state restored below
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._step(c)
            self.graphs[c] = g
        for dst, src in zip((self.tokens, self.hist, self.step_idx, self.x), saved):
            dst.copy_(src)

    def generated(self, slot: int) -> List[int]:
        n = int(self.step_idx[slot, 0])
        return self.hist[slot, :n].tolist()

    def generated_logprobs(self, slot: int) -> List[TokenLogprob]:
        """one TokenLogprob per id of generated(slot) (decoders built with logprobs only)"""
        if self.logprobs is None:
            raise ValueError("generated_logprobs() needs a decoder built with logprobs=n")
        n = int(self.step_idx[slot, 0])
        ids, lps = self.hist[slot, :n].tolist(), self.lp_hist[slot, :n].tolist()
        top_ids, top_lp = self.top_ids[slot, :n].tolist(), self.top_lp[slot, :n].tolist()
        return [TokenLogprob(t, lp, list(zip(ti, tl))) for t, lp, ti, tl in zip(ids, lps, top_ids, top_lp)]


def sampling_for_requests(sampling: Union[None, SamplingParams, Sequence[SamplingParams]],
                          n: int) -> Optional[List[SamplingParams]]:
    """generate_batch's `sampling` -> one SamplingParams per request with every seed set (None stays None).  Missing
    seeds are drawn from the host torch default generator in request order."""
    if sampling is None:
        return None
    per = [sampling] * n if isinstance(sampling, SamplingParams) else list(sampling)
    if len(per) != n or not all(isinstance(p, SamplingParams) for p in per):
        raise ValueError(f"sampling must be a SamplingParams or a list of {n} of them (one per request)")
    out = []
    for p in per:
        if p.seed is None:
            seed = int(torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64))
            p = SamplingParams(p.temperature, p.top_k, p.top_p, seed)
        out.append(p)
    return out


def penalties_for_requests(penalties: Union[None, PenaltyParams, Sequence[Optional[PenaltyParams]]],
                           n: int) -> Optional[List[Optional[PenaltyParams]]]:
    """generate_batch's `penalties` -> one PenaltyParams or None per request (None stays None)"""
    if penalties is None:
        return None
    per = [penalties] * n if isinstance(penalties, PenaltyParams) else penalties
    if (not isinstance(per, (list, tuple)) or len(per) != n
            or not all(p is None or isinstance(p, PenaltyParams) for p in per)):
        raise ValueError(f"penalties must be a PenaltyParams or a list of {n} PenaltyParams or None (one per request)")
    return list(per)


@torch.inference_mode()
def generate_batch(llm, prompts: Sequence[torch.Tensor], max_new_tokens: int, eos_token_ids: Sequence[int] = (),
                   slots: int = 8, max_tokens_per_slot: Optional[int] = None, check_every: int = 8,
                   decoder: Optional[BatchedDecoder] = None, total_pages: Optional[int] = None,
                   kv_cache: str = "bf16",
                   sampling: Union[None, SamplingParams, Sequence[SamplingParams]] = None,
                   prefix_cache: bool = False, logprobs: Optional[int] = None,
                   penalties: Union[None, PenaltyParams, Sequence[Optional[PenaltyParams]]] = None
                   ) -> Union[List[List[int]], Tuple[List[List[int]], List[List[TokenLogprob]]]]:
    """Decode `prompts` (list of inputs_embeds [S_i, hidden]) with continuous batching: at most
    `slots` requests in flight; a finished request (EOS or max_new_tokens) frees its slot for the next
    one in the queue.  Returns the new ids per request (EOS included), in request order.
    max_tokens_per_slot None: the slot and the pool are sized from the requests (slot_geometry).
    The decoder runs the LLM's current decode-weight mode; a passed-in `decoder` of another mode is a
    ValueError.  kv_cache: "bf16" or "fp8" (BatchedDecoder); a passed-in `decoder` of the other KV format is a
    ValueError.
    sampling None: greedy (the decoder's torch arg-max).  Otherwise one SamplingParams for every request or a list
    with one per request, drawn on the device (BatchedDecoder(sampling=True)); a seed of None is drawn from the host
    torch default generator in request order, so torch.manual_seed reproduces a run.  A passed-in greedy decoder
    with sampling requested is a ValueError; a sampling decoder serves greedy requests as temperature-0 rows.
    prefix_cache True: requests share the pages of the full prompt blocks they start with (BatchedDecoder); a request
    is admitted when the pool can hold the pages it must newly take, ceil((S + max_new_tokens + check_every) / 128)
    minus its cached blocks, out of the free and evictable pages other than its own cached blocks.  A passed-in
    `decoder` with the other setting, or whose max_new is below max_new_tokens, is a ValueError.
    logprobs None: returns the ids.  An int n in 0..20: returns (ids, logprobs), logprobs[r] holding one TokenLogprob
    (the id, its log-probability under the raw model distribution and its n best alternatives) per id of ids[r]
    (vila_b200/logprobs.py).  A passed-in `decoder` built without logprobs or with fewer than n is a ValueError.
    penalties None: no repetition penalties.  Otherwise one PenaltyParams for every request or a list with one
    PenaltyParams or None (0 and 0) per request, applied on the device to every token after the first
    (BatchedDecoder(penalties=True), vila_b200/penalties.py); logprobs stay those of the raw model distribution.  A
    passed-in decoder built without penalties is a ValueError."""
    params = sampling_for_requests(sampling, len(prompts))
    pens = penalties_for_requests(penalties, len(prompts))
    if pens is not None and decoder is not None and not getattr(decoder, "penalties", False):
        raise ValueError("penalties were requested but the decoder was built with penalties=False")
    if logprobs is not None:
        logprobs = check_top(logprobs)
        have = getattr(decoder, "logprobs", None) if decoder is not None else logprobs
        if have is None or have < logprobs:
            raise ValueError(f"logprobs={logprobs} was requested but the decoder was built with logprobs={have}")
    if decoder is not None and getattr(decoder, "prefix_cache", False) != bool(prefix_cache):
        raise ValueError(f"decoder was built with prefix_cache={getattr(decoder, 'prefix_cache', False)}, "
                         f"prefix_cache={bool(prefix_cache)} was asked for")
    if decoder is not None and max_new_tokens > getattr(decoder, "max_new", max_new_tokens):
        raise ValueError(f"max_new_tokens={max_new_tokens} exceeds the decoder's max_new={decoder.max_new}: its "
                         f"history would stop short of the budget")
    if params is not None and decoder is not None and not getattr(decoder, "sampling", False):
        raise ValueError("sampling was requested but the decoder was built with sampling=False")
    mode = getattr(llm, "decode_weights", "bf16")
    if decoder is not None and getattr(decoder, "decode_weights", "bf16") != mode:
        raise ValueError(f"decoder streams {getattr(decoder, 'decode_weights', 'bf16')!r} weights, the LLM is in "
                         f"{mode!r} mode: build the decoder after set_decode_weights")
    if kv_cache not in KV_CACHE_FORMATS:
        raise ValueError(f"kv_cache must be one of {KV_CACHE_FORMATS}, got {kv_cache!r}")
    if decoder is not None and getattr(decoder, "kv_cache", "bf16") != kv_cache:
        raise ValueError(f"decoder keeps a {getattr(decoder, 'kv_cache', 'bf16')!r} KV cache, {kv_cache!r} was asked for")
    if decoder is None:
        max_tokens_per_slot, pool_pages = slot_geometry([p.shape[0] for p in prompts], max_new_tokens,
                                                        check_every, slots, max_tokens_per_slot)
        decoder = BatchedDecoder(llm, slots, max_tokens_per_slot, max_new=max_new_tokens,
                                 total_pages=total_pages if total_pages is not None else pool_pages,
                                 kv_cache=kv_cache, sampling=params is not None, prefix_cache=prefix_cache,
                                 logprobs=logprobs, penalties=pens is not None)
    dec = decoder
    dec.capture()
    cap = dec.pages_per_slot * PAGE
    for p in prompts:
        if p.shape[0] + max_new_tokens + check_every > cap:
            raise ValueError(f"prompt of {p.shape[0]} tokens + {max_new_tokens} new tokens exceeds the slot ({cap})")
    queue: Deque[int] = deque(range(len(prompts)))
    owner: Dict[int, int] = {}           # slot -> request
    out: List[Optional[List[int]]] = [None] * len(prompts)
    out_lp: List[List[TokenLogprob]] = [[] for _ in prompts]
    eos = set(int(e) for e in eos_token_ids)

    def harvest(slot: int, ids: List[int]) -> Optional[List[int]]:
        for i, t in enumerate(ids):
            if t in eos:
                return ids[:i + 1]
        return ids[:max_new_tokens] if len(ids) >= max_new_tokens else None

    try:
        digests: Dict[int, np.ndarray] = {}  # request -> prefix_digests, computed once while it heads the queue
        while queue or owner:
            for s in range(dec.slots):
                if s not in owner and queue:
                    # admit only when the pool can hold the prompt and the request's whole budget
                    head = prompts[queue[0]]
                    need = (head.shape[0] + max_new_tokens + check_every + PAGE - 1) // PAGE
                    available = dec.allocator.available
                    if prefix_cache:  # cached blocks are not taken again; pinning makes them unavailable
                        if queue[0] not in digests:
                            digests[queue[0]] = dec.prefix_digests(head)
                        hits = dec.prefix_hits(digests[queue[0]], head.shape[0])
                        need -= len(hits)
                        available -= dec.allocator.evictable_among(hits)
                    if need > available and owner:
                        break  # wait for a running request to finish and return its pages
                    r = queue.popleft()
                    kw = {"digests": digests.pop(r)} if prefix_cache else {}
                    if pens is not None:
                        kw["penalties"] = pens[r]
                    if params is None:
                        dec.admit(s, prompts[r], **kw)
                    else:
                        dec.admit(s, prompts[r], params[r], **kw)
                    owner[s] = r
            dec.run(check_every)
            for s in list(owner):
                done = harvest(s, dec.generated(s))
                if done is not None:
                    r = owner.pop(s)
                    out[r] = done
                    if logprobs is not None:  # truncated as the ids are; a larger decoder's top lists cut to n
                        out_lp[r] = [TokenLogprob(e.token, e.logprob, e.top[:logprobs])
                                     for e in dec.generated_logprobs(s)[:len(done)]]
                    dec.release(s)
    except BaseException:
        # a failed request fails the call, but a decoder that outlives it (a kept prefix-caching engine) must not keep
        # this call's slots: every slot that was admitted, or was being admitted, is released
        for s in range(dec.slots):
            if s in owner or getattr(dec, "slot_pages", [[]] * dec.slots)[s]:
                dec.release(s)
        raise
    ids = [o or [] for o in out]
    return ids if logprobs is None else (ids, out_lp)
