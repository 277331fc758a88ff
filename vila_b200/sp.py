"""Sequence-parallel prefill (LongVILA, BASELINE config #5) — NVSwitch design.

Reference (what this replaces):
  inference: zigzag ring attention, llava/eval/vision_niah_vila/eval_vision_niah.py:83-140,
             zigzag_ring_attn/prepare_inputs.py:20-23 (rank r owns chunks r and 2P-1-r of 2P),
             monkey_patch.py:28-57 (P rounds of isend/irecv K,V + flash-attn + LSE merge per layer)
  training : llava/train/sequence_parallel/* (Ulysses all-to-all / ring / hybrid)
On NVSwitch every GPU reaches every peer at full bandwidth, and with GQA the KV stream is tiny
(2 KiB per token per layer), so the ring's P-1 serialized P2P rounds become ONE all-gather of K,V per
layer that lands DIRECTLY in the paged KV pool: the page table encodes the zigzag permutation, so
there is no reorder copy and no cross-rank softmax merge — each rank then runs the ordinary causal
wgmma FMHA for its two query chunks against the (paged) full-length KV.

Host logic (partitioning, page tables, padding) is pure Python/torch-CPU and is covered by
world_size-2 gloo tests; the kernels are the same C-ABI calls as the single-GPU path.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch

PAGE = 128


@dataclass
class ZigzagPlan:
    world: int
    rank: int
    seq_len: int         # real tokens
    padded_len: int      # multiple of 2 * world * PAGE
    chunk: int           # tokens per chunk (= padded_len / (2*world)), multiple of PAGE

    @property
    def chunk_pages(self) -> int:
        return self.chunk // PAGE

    def local_chunks(self, rank: Optional[int] = None) -> List[Tuple[int, int]]:
        """Global [start, end) of the two chunks owned by `rank` (prepare_inputs.py:20-23)."""
        r = self.rank if rank is None else rank
        a, b = r, 2 * self.world - 1 - r
        return [(a * self.chunk, (a + 1) * self.chunk), (b * self.chunk, (b + 1) * self.chunk)]

    def local_positions(self, rank: Optional[int] = None) -> torch.Tensor:
        return torch.cat([torch.arange(s, e, dtype=torch.int32) for s, e in self.local_chunks(rank)])

    def extract_local(self, x: torch.Tensor, rank: Optional[int] = None) -> torch.Tensor:
        """rows of a [padded_len, ...] tensor owned by `rank` (zigzag `extract_local`)."""
        return torch.cat([x[s:e] for s, e in self.local_chunks(rank)], dim=0)

    def page_table(self) -> torch.Tensor:
        """global KV block j (128 tokens) -> physical page of the gathered pool, whose layout is
        [rank][slot 0 | slot 1][chunk_pages]: rank o's region is exactly what o contributes to the
        all-gather, so the collective writes K/V in place."""
        cp = self.chunk_pages
        out = []
        for j in range(self.padded_len // PAGE):
            ch = j // cp
            owner, slot = (ch, 0) if ch < self.world else (2 * self.world - 1 - ch, 1)
            out.append(owner * 2 * cp + slot * cp + j % cp)
        return torch.tensor(out, dtype=torch.int32)

    def owner_of(self, pos: int) -> int:
        ch = pos // self.chunk
        return ch if ch < self.world else 2 * self.world - 1 - ch

    def undo_extract_local(self, gathered: torch.Tensor) -> torch.Tensor:
        """[world, 2*chunk, ...] rank-major local rows -> global order [padded_len, ...]."""
        out = gathered.new_empty((self.padded_len,) + tuple(gathered.shape[2:]))
        for r in range(self.world):
            (a0, a1), (b0, b1) = self.local_chunks(r)
            out[a0:a1] = gathered[r, :self.chunk]
            out[b0:b1] = gathered[r, self.chunk:]
        return out


def make_plan(seq_len: int, world: int, rank: int) -> ZigzagPlan:
    """Pad to a multiple of 2*world*128 (the reference pads to a multiple of 2*world,
    eval_vision_niah.py:88-98; we additionally align chunks to KV pages)."""
    unit = 2 * world * PAGE
    padded = (seq_len + unit - 1) // unit * unit
    return ZigzagPlan(world, rank, seq_len, padded, padded // (2 * world))


# ---- process-group registry (the reference's PROCESS_GROUP_MANAGER, llava/train/sequence_parallel/
# globals.py:84-149, reduced to the one group the inference path needs) ---------------------------
_SP_GROUP = None
_SP_ENABLED = False


def set_sequence_parallel_group(group=None, enabled: bool = True) -> None:
    """Enable sequence parallelism for LlavaLlamaModel.forward / generate over `group` (None = the
    default torch.distributed group).  Mirrors `set_pg_manager(sp_degree, ...)` of the reference."""
    global _SP_GROUP, _SP_ENABLED
    _SP_GROUP, _SP_ENABLED = group, enabled


def sequence_parallel_group():
    return _SP_GROUP


def sequence_parallel_enabled() -> bool:
    if not _SP_ENABLED:
        return False
    import torch.distributed as dist
    return dist.is_available() and dist.is_initialized()


def sp_cache_page_order(plan: "ZigzagPlan", n_pages: int) -> List[int]:
    """Page order of a decode-capable KV cache whose first padded_len/128 pages are the zigzag
    all-gather layout and whose remaining pages (tokens generated past the padded prompt) are
    identity-mapped."""
    base = plan.page_table().tolist()
    assert n_pages >= len(base)
    return base + list(range(len(base), n_pages))


def shard_frames(n_frames: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous frame range per rank for the vision tower (extract_local_from_list,
    llava/train/sequence_parallel/input_utils.py:26-30)."""
    per = (n_frames + world - 1) // world
    return min(rank * per, n_frames), min((rank + 1) * per, n_frames)


class SequenceParallelPrefill:
    """Prefill of one long sequence across `group` (one process per GPU, NCCL)."""

    def __init__(self, llm, group=None):
        import torch.distributed as dist
        self.llm = llm
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self._comm_stream = None  # created on first use (the host logic is testable without a GPU)
        self._plan_cache = {}

    @property
    def comm_stream(self):
        if self._comm_stream is None:
            self._comm_stream = torch.cuda.Stream(device=self.llm.device)
        return self._comm_stream

    def new_pool(self, plan: ZigzagPlan, extra_tokens: int = 0):
        cfg = self.llm.config
        n_pages = plan.padded_len // PAGE + (extra_tokens + PAGE - 1) // PAGE
        return torch.zeros(cfg.num_hidden_layers, 2, n_pages, PAGE, cfg.num_key_value_heads,
                           cfg.head_dim, device=self.llm.device, dtype=self.llm.dtype)

    def _device_plan(self, plan: ZigzagPlan):
        key = (plan.world, plan.rank, plan.padded_len)
        ent = self._plan_cache.get(key)
        if ent is None:
            ent = (plan.page_table().to(self.llm.device), plan.local_positions().to(self.llm.device))
            self._plan_cache = {key: ent}
        return ent

    @torch.inference_mode()
    def prefill_hidden(self, local_embeds: torch.Tensor, plan: ZigzagPlan, pool=None):
        """local_embeds [2*chunk, hidden] (rows of this rank's two zigzag chunks, padded rows zero).
        Returns this rank's final hidden states [2*chunk, hidden] (pre final-norm) and the pool
        [L, 2, >= padded_len/128 pages, 128, Hkv, D]; its first padded_len/128 pages are the gathered
        zigzag layout (extra pages, if any, are left for tokens decoded later).

        Per layer: q/k/v GEMM -> RoPE(global positions) + K/V rows into this rank's pool region ->
        the K/V all-gather is issued on `comm_stream`; rank 0's first chunk attends only to its own
        pages and runs under the exchange, every other chunk waits for the gathered K/V.  The
        exchange moves 118 MB per GPU per layer at S = 65.8K over NVSwitch (~0.2 ms of a ~9 ms layer)."""
        import torch.distributed as dist
        from . import ops
        llm, cfg = self.llm, self.llm.config
        Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        c, cp = plan.chunk, plan.chunk_pages
        assert local_embeds.shape[0] == 2 * c
        pool = pool if pool is not None else self.new_pool(plan)
        zz_pages = plan.padded_len // PAGE
        page_table, positions = self._device_plan(plan)
        (a0, a1), (b0, b1) = plan.local_chunks()
        x = local_embeds.to(llm.dtype).contiguous().clone()
        n_local_pages = 2 * cp
        compute = torch.cuda.current_stream()
        table = ops.rope_table(positions, D, llm.inv_freq)  # cos | sin of the GLOBAL positions, once
        for li, layer in enumerate(llm.model.layers):
            h = ops.rmsnorm(x, layer.input_layernorm.weight, cfg.rms_norm_eps)
            qkv = ops.linear(h, layer._qkv_w, layer._qkv_b, static_w=True)
            kpool, vpool = pool[li, 0], pool[li, 1]
            # RoPE with GLOBAL positions; K/V rows land in this rank's region of the pool
            ops.rope_kv_append_table(qkv[:c], table[:c], Hq, Hkv, D, kpool, vpool, page_table, a0)
            ops.rope_kv_append_table(qkv[c:], table[c:], Hq, Hkv, D, kpool, vpool, page_table, b0)
            q = qkv.view(2 * c, Hq + 2 * Hkv, D)[:, :Hq]
            attn = torch.empty(2 * c, Hq, D, dtype=llm.dtype, device=llm.device)
            if self.world > 1:
                # ONE in-place all-gather per tensor replaces the ring's P-1 P2P rounds; it runs on
                # the communication stream, ordered after this layer's K/V writes
                self.comm_stream.wait_stream(compute)
                lo = self.rank * n_local_pages
                with torch.cuda.stream(self.comm_stream):
                    for t in (kpool, vpool):
                        dist.all_gather_into_tensor(t[:zz_pages].view(-1),
                                                    t[lo:lo + n_local_pages].view(-1), group=self.group)
                if self.rank == 0:
                    # chunk 0 attends to global tokens [0, chunk) only = rank 0's own slot-0 pages:
                    # no remote K/V needed, so it overlaps the exchange
                    ops.fmha(q[:c], kpool, vpool, B=1, Sq=c, Sk=a1, causal=True, scale=D ** -0.5,
                             page_table=page_table, out=attn[:c])
                compute.wait_stream(self.comm_stream)
                if self.rank != 0:
                    ops.fmha(q[:c], kpool, vpool, B=1, Sq=c, Sk=a1, causal=True, scale=D ** -0.5,
                             page_table=page_table, out=attn[:c])
            else:
                ops.fmha(q[:c], kpool, vpool, B=1, Sq=c, Sk=a1, causal=True, scale=D ** -0.5,
                         page_table=page_table, out=attn[:c])
            ops.fmha(q[c:], kpool, vpool, B=1, Sq=c, Sk=b1, causal=True, scale=D ** -0.5,
                     page_table=page_table, out=attn[c:])
            ops.linear(attn.view(2 * c, Hq * D), layer.self_attn.o_proj.weight, residual=x, out=x, static_w=True)
            h = ops.rmsnorm(x, layer.post_attention_layernorm.weight, cfg.rms_norm_eps)
            a = ops.linear(h, layer._gu_w, swiglu=True, static_w=True)
            ops.linear(a, layer.mlp.down_proj.weight, residual=x, out=x, static_w=True)
        return x, pool

    def local_row_of(self, plan: ZigzagPlan, pos: int) -> Optional[int]:
        """row index of global position `pos` inside this rank's local rows (None: not owned)."""
        (a0, a1), (b0, b1) = plan.local_chunks()
        if a0 <= pos < a1:
            return pos - a0
        if b0 <= pos < b1:
            return plan.chunk + (pos - b0)
        return None

    @torch.inference_mode()
    def last_token_hidden(self, hidden_local: torch.Tensor, plan: ZigzagPlan) -> torch.Tensor:
        """final-layer hidden state [hidden] of the last REAL token on every rank (broadcast from its
        owner): what seeds the replicated greedy decode (gather of eval_vision_niah.py:121-133)."""
        import torch.distributed as dist
        last = plan.seq_len - 1
        owner = plan.owner_of(last)
        row = torch.empty(hidden_local.shape[1], dtype=hidden_local.dtype, device=hidden_local.device)
        if self.rank == owner:
            row.copy_(hidden_local[self.local_row_of(plan, last)])
        if self.world > 1:
            dist.broadcast(row, src=dist.get_global_rank(self.group, owner) if self.group else owner,
                           group=self.group)
        return row

    @torch.inference_mode()
    def last_token_logits(self, hidden_local: torch.Tensor, plan: ZigzagPlan) -> Optional[torch.Tensor]:
        """lm_head on the last REAL token, computed only by the rank that owns it; broadcast."""
        import torch.distributed as dist
        last = plan.seq_len - 1
        owner = plan.owner_of(last)
        V = self.llm.vocab_size
        logits = torch.empty(1, V, dtype=self.llm.dtype, device=self.llm.device)
        if self.rank == owner:
            row = self.local_row_of(plan, last)
            logits = self.llm.logits_from_hidden(hidden_local[row:row + 1])
        if self.world > 1:
            dist.broadcast(logits, src=dist.get_global_rank(self.group, owner) if self.group else owner,
                           group=self.group)
        return logits

    @torch.inference_mode()
    def gather_frame_features(self, local_feats: torch.Tensor, n_frames: int) -> torch.Tensor:
        """[f_local, N, C] per-rank frame features (contiguous ranges of shard_frames) -> [n_frames, N, C]
        on every rank; the ragged tail (n_frames % world != 0) is zero-padded for the collective and
        cut off afterwards (the reference all-reduces zero-padded embeddings, llava_arch.py:591-593)."""
        import torch.distributed as dist
        if self.world == 1:
            return local_feats
        per = (n_frames + self.world - 1) // self.world
        padded = local_feats.new_zeros((per,) + tuple(local_feats.shape[1:]))
        padded[:local_feats.shape[0]] = local_feats
        allf = local_feats.new_empty((self.world * per,) + tuple(local_feats.shape[1:]))
        dist.all_gather_into_tensor(allf, padded, group=self.group)
        return allf[:n_frames]
