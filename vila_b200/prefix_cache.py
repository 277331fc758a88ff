"""Prefix caching for the continuous-batching engine (vila_b200/serving.py, BatchedDecoder(prefix_cache=True)).

Requests whose prompts start alike (several questions about one video, a chat that resends its image every turn,
one long system prompt) share the K/V pages of that start instead of prefilling it again.

Block identity.  A prompt block is rows [128 i, 128 i + 128) of the request's inputs_embeds (bf16): the engine sees
embeddings, not ids plus media, and the same image or frames through LlavaLlamaModel._embed give the same bits.
vila_prefix_block_hash digests every full block on the device; `block_digests` below states its rule in numpy:
  w_j      the j-th 8-byte little-endian word of the block's 128 rows, read row-major over the logical columns
           (the row-stride padding is not read)
  fmix64   the murmur3 64-bit finalizer
  d_L      sum over j of fmix64(fmix64(w_j ^ key_L) + j * 0x9E3779B97F4A7C15) mod 2^64, for L = 0, 1
The digest is not cryptographic.  Each engine draws its two keys at random (`random_keys`), so that blocks that
collide under it cannot be prepared in advance; two different blocks still collide with probability about 2^-128.

Cached blocks form a trie: a node is (parent node, digest), and depth i covers positions [128 i, 128 i + 128), so
a block matches only if every earlier block matched at the same positions.  `PrefixPages` keeps the trie and the
state of every physical page of the pool:
  free       on the free list;
  owned      held by one live slot and not cached (a partial prompt page, decoded tokens, a block not registered);
  cached     a trie node, with a refcount equal to the number of live slots whose page-table row holds it; at
             refcount 0 it is evictable and can still be found.
Allocation takes from the free list first, then evicts evictable blocks: oldest last use first and, among blocks
last used by the same admission, the deepest first, so that no cached block is ever left without its parent (a
block's parent is used whenever the block is, and held by every slot that holds the block).
"""
from __future__ import annotations

import secrets
from typing import Dict, List, Sequence, Tuple

import numpy as np

PAGE = 128
GOLDEN = np.uint64(0x9E3779B97F4A7C15)
_M1, _M2 = np.uint64(0xff51afd7ed558ccd), np.uint64(0xc4ceb9fe1a85ec53)
_S33 = np.uint64(33)


def fmix64(k: np.ndarray) -> np.ndarray:
    """murmur3's 64-bit finalizer, element-wise on uint64 (wrapping)"""
    k = k ^ (k >> _S33)
    k = k * _M1
    k = k ^ (k >> _S33)
    k = k * _M2
    return k ^ (k >> _S33)


def block_digests(x, key0: int, key1: int) -> np.ndarray:
    """The digest rule of vila_prefix_block_hash: x [rows, cols] bf16 (a torch tensor on any device, any row stride)
    or its uint16 bit pattern as a numpy array; cols a multiple of 4.  -> uint64 [rows // 128, 2]."""
    if not isinstance(x, np.ndarray):
        import torch
        x = x.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)
    rows, cols = x.shape
    if cols % 4:
        raise ValueError(f"block_digests: cols must be a multiple of 4, got {cols}")
    n = rows // PAGE
    out = np.zeros((n, 2), dtype=np.uint64)
    if n == 0:
        return out
    words = np.ascontiguousarray(x[:n * PAGE]).view("<u8").reshape(n, PAGE * cols // 4)
    salt = np.arange(words.shape[1], dtype=np.uint64) * GOLDEN
    for b in range(n):
        for lane, key in enumerate((key0, key1)):
            out[b, lane] = fmix64(fmix64(words[b] ^ np.uint64(key)) + salt).sum(dtype=np.uint64)
    return out


def random_keys() -> Tuple[int, int]:
    """two 64-bit keys from the OS's entropy (not from torch's generator: drawing them must not move the sampling
    seeds that generate_batch draws from it)"""
    return secrets.randbits(64), secrets.randbits(64)


class PrefixPages:
    """Free list, trie of cached blocks and refcounts over the physical pages of one pool (host-side bookkeeping).

    It replaces serving.PageAllocator in a prefix-caching engine: alloc / release / available / n_pages keep their
    meaning (release decrements cached pages instead of freeing them; available counts free plus evictable pages),
    and match / pin / register / clear add the cache.  Page order from the free list is PageAllocator's."""

    def __init__(self, n_pages: int):
        self.free: List[int] = list(range(n_pages - 1, -1, -1))  # pop() hands out page 0 first
        self.n_pages = n_pages
        self.children: Dict[Tuple[int, int, int], int] = {}  # (parent page or -1, d_0, d_1) -> page
        self.node: Dict[int, Tuple[Tuple[int, int, int], int]] = {}  # cached page -> (trie key, depth)
        self.ref: Dict[int, int] = {}  # cached page -> live slots holding it
        self.last_use: Dict[int, int] = {}  # cached page -> admission tick of its last use
        self.evictable: Dict[int, None] = {}  # cached pages at refcount 0 (insertion-ordered set)
        self.tick = 0
        self.stats = dict(lookups=0, hit_blocks=0, hit_tokens=0, prefilled_tokens=0, evictions=0)

    # ---- PageAllocator surface ----------------------------------------------------------------------------
    @property
    def available(self) -> int:
        return len(self.free) + len(self.evictable)

    def alloc(self, n: int) -> List[int]:
        if n > self.available:
            raise MemoryError(f"KV pool exhausted: {n} pages wanted, {len(self.free)} free and "
                              f"{len(self.evictable)} evictable of {self.n_pages}")
        take = min(n, len(self.free))
        out = [self.free.pop() for _ in range(take)]
        if n > take:
            out += self._evict(n - take)
        return out

    def release(self, pages: Sequence[int]) -> None:
        """a slot's page-table row [0, len(pages)) is dropped: cached pages lose one holder, owned ones are freed"""
        owned = []
        for p in pages:
            if p in self.ref:
                self.ref[p] -= 1
                if self.ref[p] == 0:
                    self.evictable[p] = None
            else:
                owned.append(p)
        self.free.extend(reversed(owned))

    # ---- cache ----------------------------------------------------------------------------------------------
    def match(self, digests: np.ndarray, limit: int) -> List[int]:
        """pages of the longest cached chain of digests[0], digests[1], ... (at most `limit` blocks); no state
        changes"""
        hits: List[int] = []
        parent = -1
        for i in range(min(limit, len(digests))):
            page = self.children.get((parent, int(digests[i, 0]), int(digests[i, 1])))
            if page is None:
                break
            hits.append(page)
            parent = page
        return hits

    def evictable_among(self, pages: Sequence[int]) -> int:
        return sum(1 for p in pages if p in self.evictable)

    def pin(self, hits: Sequence[int]) -> None:
        """a new admission holds `hits` (a chain from match): one more holder each, used at a new tick"""
        self.tick += 1
        self.stats["lookups"] += 1
        self.stats["hit_blocks"] += len(hits)
        self.stats["hit_tokens"] += PAGE * len(hits)
        for p in hits:
            self.ref[p] += 1
            self.last_use[p] = self.tick
            self.evictable.pop(p, None)

    def register(self, digests: np.ndarray, pages: Sequence[int], first: int) -> int:
        """blocks first, first + 1, ... of the admission just pinned, held in the slot's own `pages` (page i holds
        block i), become trie nodes under pages[first - 1].  Stops at the first block that is already cached
        (another slot registered the same content): a node's parent must be a node the slot holds.
        -> blocks registered"""
        parent = pages[first - 1] if first else -1
        n = 0
        for i in range(first, len(digests)):
            key = (parent, int(digests[i, 0]), int(digests[i, 1]))
            if key in self.children:
                break
            page = pages[i]
            self.children[key] = page
            self.node[page] = (key, i)
            self.ref[page] = 1
            self.last_use[page] = self.tick
            parent = page
            n += 1
        return n

    def _evict(self, n: int) -> List[int]:
        order = sorted(self.evictable, key=lambda p: (self.last_use[p], -self.node[p][1]))[:n]
        for p in order:
            self._drop(p)
        self.stats["evictions"] += len(order)
        return order

    def _drop(self, p: int) -> None:
        key, _ = self.node.pop(p)
        del self.children[key], self.ref[p], self.last_use[p], self.evictable[p]

    def clear(self) -> int:
        """drop every evictable block (deepest first) onto the free list -> blocks dropped"""
        order = sorted(self.evictable, key=lambda p: -self.node[p][1])
        for p in order:
            self._drop(p)
        self.free.extend(reversed(order))
        return len(order)

    @property
    def cached_blocks(self) -> int:
        return len(self.node)
