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
  * finished slots (EOS / budget) are harvested and refilled between graph replays.
"""
from __future__ import annotations

from collections import deque
from typing import Deque, Dict, List, Optional, Sequence, Tuple

import torch

from . import ops

PAGE = 128


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
    device and are read by the kernels at every launch: changing them needs no graph re-capture."""

    def __init__(self, llm, slots: int = 8, max_tokens_per_slot: int = 2048, max_new: int = 1024,
                 total_pages: Optional[int] = None):
        cfg = llm.config
        self.llm, self.slots = llm, slots
        dev, dt = llm.device, llm.dtype
        Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        assert D == 128, "batched decode attention is specialised for head_dim 128"
        self.pages_per_slot = (max_tokens_per_slot + PAGE - 1) // PAGE
        assert self.pages_per_slot <= 32, "vila_decode_attention_batch serves contexts up to 4096 tokens"
        P = total_pages if total_pages is not None else slots * self.pages_per_slot
        self.pool = torch.zeros(cfg.num_hidden_layers, 2, P, PAGE, Hkv, D, device=dev, dtype=dt)
        self.allocator = PageAllocator(P)
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
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.launches_per_step = 7 * cfg.num_hidden_layers + 2

    # ---- admission ------------------------------------------------------------------------------
    @torch.inference_mode()
    def admit(self, slot: int, inputs_embeds: torch.Tensor) -> None:
        """Prefill `inputs_embeds` [S, hidden] into the slot's pages and seed its decode state."""
        llm = self.llm
        S = inputs_embeds.shape[0]
        assert S + 1 <= self.pages_per_slot * PAGE, "prompt longer than a slot"
        self._ensure_pages(slot, S + 1)
        cache = _SlotCache(self.pool, self.page_tables[slot])
        hid = llm.prefill_hidden(inputs_embeds, cache)
        logits = llm.logits_from_hidden(hid[-1:])
        tok = torch.argmax(logits[0].float())
        self.tokens[slot] = tok
        self.hist[slot, 0] = tok
        self.step_idx[slot, 0] = 1
        self.x[slot] = llm.model.embed_tokens.weight[tok]
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

    # ---- one decode step for every active slot ----------------------------------------------------
    def _step(self) -> None:
        llm, cfg = self.llm, self.llm.config
        Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        x = self.x
        for li, layer in enumerate(llm.model.layers):
            h = ops.rmsnorm(x, layer.input_layernorm.weight, cfg.rms_norm_eps)
            qkv = ops.linear(h, layer._qkv_w, layer._qkv_b, static_w=True)
            ops.decode_attention_batch(qkv, self.positions, self.pool[li, 0], self.pool[li, 1],
                                       self.page_tables, self.attn, llm.inv_freq, Hq, Hkv, D, D ** -0.5)
            ops.linear(self.attn, layer.self_attn.o_proj.weight, residual=x, out=x, static_w=True)
            h = ops.rmsnorm(x, layer.post_attention_layernorm.weight, cfg.rms_norm_eps)
            a = ops.linear(h, layer._gu_w, swiglu=True, static_w=True)
            ops.linear(a, layer.mlp.down_proj.weight, residual=x, out=x, static_w=True)
        h = ops.rmsnorm(x.clone(), llm.model.norm.weight, cfg.rms_norm_eps)
        logits = ops.linear(h, llm.lm_head.weight, static_w=True)
        active = self.positions >= 0
        tok = torch.argmax(logits.float(), dim=-1)
        self.tokens.copy_(torch.where(active, tok, self.tokens))
        col = self.step_idx.clamp(max=self.hist.shape[1] - 1)
        self.hist.scatter_(1, col, self.tokens[:, None])
        self.step_idx.add_(active[:, None].to(torch.int64))
        x.copy_(ops.embed_splice(llm.model.embed_tokens.weight, None, self.tokens.to(torch.int32)))
        self.positions.add_(active.to(torch.int32))

    @torch.inference_mode()
    def run(self, n_tokens: int) -> None:
        if self.graph is None:
            raise RuntimeError("call capture() (with every slot idle) before run()")
        for s_ in range(self.slots):  # pages for the tokens this call will append
            if self._pos_host[s_] >= 0:
                self._ensure_pages(s_, self._pos_host[s_] + n_tokens + 1)
                self._pos_host[s_] += n_tokens
        for _ in range(n_tokens):
            self.graph.replay()

    @torch.inference_mode()
    def capture(self) -> None:
        """Capture the step graph.  Must be called with every slot idle (positions < 0): the capture
        launches the kernels once, idle slots are skipped by the attention kernel and leave no trace."""
        if self.graph is not None:
            return
        assert bool((self.positions < 0).all()), "capture() with idle slots only"
        saved = (self.tokens.clone(), self.hist.clone(), self.step_idx.clone(), self.x.clone())
        self._step()  # eager warm-up (allocator, function attributes); state restored below
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._step()
        self.graph = g
        for dst, src in zip((self.tokens, self.hist, self.step_idx, self.x), saved):
            dst.copy_(src)

    def generated(self, slot: int) -> List[int]:
        n = int(self.step_idx[slot, 0])
        return self.hist[slot, :n].tolist()


@torch.inference_mode()
def generate_batch(llm, prompts: Sequence[torch.Tensor], max_new_tokens: int, eos_token_ids: Sequence[int] = (),
                   slots: int = 8, max_tokens_per_slot: int = 2048, check_every: int = 8,
                   decoder: Optional[BatchedDecoder] = None, total_pages: Optional[int] = None) -> List[List[int]]:
    """Greedy-decode `prompts` (list of inputs_embeds [S_i, hidden]) with continuous batching: at most
    `slots` requests in flight; a finished request (EOS or max_new_tokens) frees its slot for the next
    one in the queue.  Returns the new ids per request (EOS included), in request order."""
    dec = decoder or BatchedDecoder(llm, slots, max_tokens_per_slot, max_new=max_new_tokens,
                                    total_pages=total_pages)
    dec.capture()
    cap = dec.pages_per_slot * PAGE
    for p in prompts:
        if p.shape[0] + max_new_tokens + check_every > cap:
            raise ValueError(f"prompt of {p.shape[0]} tokens + {max_new_tokens} new tokens exceeds the slot ({cap})")
    queue: Deque[int] = deque(range(len(prompts)))
    owner: Dict[int, int] = {}           # slot -> request
    out: List[Optional[List[int]]] = [None] * len(prompts)
    eos = set(int(e) for e in eos_token_ids)

    def harvest(slot: int, ids: List[int]) -> Optional[List[int]]:
        for i, t in enumerate(ids):
            if t in eos:
                return ids[:i + 1]
        return ids[:max_new_tokens] if len(ids) >= max_new_tokens else None

    while queue or owner:
        for s in range(dec.slots):
            if s not in owner and queue:
                # admit only when the pool can hold the prompt and the request's whole budget
                need = (prompts[queue[0]].shape[0] + max_new_tokens + check_every + PAGE - 1) // PAGE
                if need > dec.allocator.available and owner:
                    break  # wait for a running request to finish and return its pages
                r = queue.popleft()
                dec.admit(s, prompts[r])
                owner[s] = r
        dec.run(check_every)
        for s in list(owner):
            done = harvest(s, dec.generated(s))
            if done is not None:
                out[owner.pop(s)] = done
                dec.release(s)
    return [o or [] for o in out]
