"""CPU: prefix caching in the continuous-batching engine (vila_b200/prefix_cache.py, serving.BatchedDecoder(
prefix_cache=True)): the numpy digest rule of vila_prefix_block_hash, the page bookkeeping (trie, refcounts, LRU
eviction) on a CPU decoder whose prefill and hashing are stubbed, generate_batch's admission accounting, the argument
errors and the server's --prefix-cache routing."""
import asyncio
import inspect
import random
from collections import Counter
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from vila_b200 import serving
from vila_b200.prefix_cache import PAGE, block_digests, fmix64
from vila_b200.sampling import SamplingParams

HIDDEN = 64
K0, K1 = 0x0123456789ABCDEF, 0xFEDCBA9876543210


# ------------------------------------------------------------------------------------------------
# the digest rule
# ------------------------------------------------------------------------------------------------
def _rows(n, seed, cols=HIDDEN):
    return torch.randn(n, cols, generator=torch.Generator().manual_seed(seed)).to(torch.bfloat16)


def test_fmix64_known_values():
    # murmur3's fmix64: 0 is a fixed point; the constants make 1 -> 0xB456BCFC34C2CB2C
    assert int(fmix64(np.array([0], dtype=np.uint64))[0]) == 0
    assert int(fmix64(np.array([1], dtype=np.uint64))[0]) == 0xB456BCFC34C2CB2C


def test_digest_deterministic_and_sensitive():
    x = _rows(300, 1)
    d = block_digests(x, K0, K1)
    assert d.shape == (2, 2) and d.dtype == np.uint64
    assert np.array_equal(d, block_digests(x.clone(), K0, K1))
    bits = x.view(torch.int16)
    for r, c, b in ((0, 0, 0), (127, 63, 15), (64, 17, 7), (128, 0, 3), (255, 63, 0)):
        y = bits.clone()
        y[r, c] ^= (1 << b) if b < 15 else -(1 << 15)
        dy = block_digests(y.view(torch.bfloat16), K0, K1)
        blk = r // PAGE
        assert not np.array_equal(dy[blk], d[blk]) and np.array_equal(dy[1 - blk], d[1 - blk]), (r, c, b)
        assert (dy[blk] != d[blk]).all()  # both lanes change
    # two rows of a block swapped, and another key
    y = x.clone()
    y[[3, 90]] = x[[90, 3]]
    assert not np.array_equal(block_digests(y, K0, K1)[0], d[0])
    assert not np.array_equal(block_digests(x, K0 ^ 1, K1)[:, 0], d[:, 0])
    assert np.array_equal(block_digests(x, K0 ^ 1, K1)[:, 1], d[:, 1])  # the lanes are independent
    # the rows past the last full block do not count
    z = x.clone()
    z[256:] = 0
    assert np.array_equal(block_digests(z, K0, K1), d)


def test_digest_ignores_row_padding_and_short_inputs():
    x = _rows(260, 2)
    padded = torch.full((260, HIDDEN + 12), float("nan"), dtype=torch.bfloat16)
    padded[:, :HIDDEN] = x
    assert np.array_equal(block_digests(padded[:, :HIDDEN], K0, K1), block_digests(x, K0, K1))
    assert block_digests(x[:127], K0, K1).shape == (0, 2)
    with pytest.raises(ValueError):
        block_digests(_rows(128, 3, cols=6), K0, K1)


def test_digest_pinned_value():
    # one block of 128 x 4 bf16 whose 8-byte words are j (word j = row j): d_L = sum_j fmix64(fmix64(j ^ k) + j * G)
    words = np.arange(PAGE, dtype="<u8")
    x = words.view(np.uint16).reshape(PAGE, 4)
    got = block_digests(x, 0, 2 ** 64 - 1)
    g = 0x9E3779B97F4A7C15
    mask = 2 ** 64 - 1

    def fm(k):
        k ^= k >> 33
        k = (k * 0xff51afd7ed558ccd) & mask
        k ^= k >> 33
        k = (k * 0xc4ceb9fe1a85ec53) & mask
        return k ^ (k >> 33)

    want = [sum(fm((fm(j ^ key) + j * g) & mask) for j in range(PAGE)) & mask for key in (0, mask)]
    assert [int(v) for v in got[0]] == want == [0x1049C4062BCDAB7E, 0xFFDE19B69C99FAB3]


def test_hash_entry_point_argument_errors():
    """reported before any device call, so they hold without a GPU"""
    from vila_b200 import _lib, ops
    lib = _lib.load()
    buf = np.zeros(256 * 64 + 8, dtype=np.uint16)
    x = buf.ctypes.data + (-buf.ctypes.data) % 8
    out = np.zeros(8, dtype=np.uint64).ctypes.data
    for ld, rows, cols in ((64, 256, 62), (62, 256, 60), (60, 256, 64), (64, -1, 64)):
        assert lib.vila_prefix_block_hash(x, ld, rows, cols, 1, 2, out, None) != 0
        assert b"vila_prefix_block_hash" in lib.vila_last_error()
    assert lib.vila_prefix_block_hash(x + 2, 64, 256, 64, 1, 2, out, None) != 0
    assert lib.vila_prefix_block_hash(None, 64, 100, 64, 1, 2, None, None) == 0  # no full block: nothing to do
    assert "vila_prefix_block_hash" in _lib.SIGNATURES
    with pytest.raises(ValueError):
        ops.prefix_block_hash(torch.zeros(256, 64, dtype=torch.bfloat16), 2 ** 64, 0)


# ------------------------------------------------------------------------------------------------
# a CPU BatchedDecoder: prefill and hashing stubbed, step graphs that only advance the counters
# ------------------------------------------------------------------------------------------------
class _StepGraph:
    """what a replay does to the host-visible state: every active slot appends its position as the token"""

    def __init__(self, dec, log):
        self.dec, self.log = dec, log

    def replay(self):
        d = self.dec
        active = d.positions >= 0
        self.log.append(int(active.sum()))
        col = d.step_idx.clamp(max=d.hist.shape[1] - 1)
        d.hist.scatter_(1, col, torch.where(active, d.positions.to(torch.int64), d.tokens)[:, None])
        d.step_idx.add_(active[:, None].to(torch.int64))
        d.positions.add_(active.to(torch.int32))


def _hash_stub(x, key0, key1):
    return torch.from_numpy(block_digests(x, key0, key1).view(np.int64).copy())


@pytest.fixture
def cpu_hash(monkeypatch):
    monkeypatch.setattr(serving.ops, "prefix_block_hash", _hash_stub)


def _cpu_decoder(slots=4, max_tokens_per_slot=1024, total_pages=64, prefix_cache=True, max_new=64, kv_cache="bf16"):
    cfg = SimpleNamespace(num_attention_heads=2, num_key_value_heads=1, head_dim=128, num_hidden_layers=1,
                          hidden_size=HIDDEN, vocab_size=32)
    prefills = []

    def prefill_hidden(emb, cache):
        prefills.append((cache.length, emb.shape[0]))
        cache.length += emb.shape[0]
        return torch.zeros(emb.shape[0], HIDDEN, dtype=torch.bfloat16)

    llm = SimpleNamespace(config=cfg, device=torch.device("cpu"), dtype=torch.bfloat16, prefill_hidden=prefill_hidden,
                          logits_from_hidden=lambda h: torch.zeros(1, cfg.vocab_size, dtype=torch.bfloat16),
                          model=SimpleNamespace(embed_tokens=SimpleNamespace(
                              weight=torch.zeros(cfg.vocab_size, HIDDEN, dtype=torch.bfloat16))))
    dec = serving.BatchedDecoder(llm, slots=slots, max_tokens_per_slot=max_tokens_per_slot, max_new=max_new,
                                 total_pages=total_pages, kv_cache=kv_cache, prefix_cache=prefix_cache)
    log = []
    dec.graphs = {c: _StepGraph(dec, log) for c in dec.configs}
    return dec, prefills, log


def _blocks(seeds, tail=0, tail_seed=99):
    """a prompt made of 128-row blocks (one per seed) and `tail` more rows"""
    parts = [_rows(PAGE, s) for s in seeds] + ([_rows(tail, tail_seed)] if tail else [])
    return torch.cat(parts)


def check_invariants(dec):
    """every page in exactly one state, refcounts = live rows holding the page, parents cached, states add up"""
    a = dec.allocator
    free = a.free
    assert len(set(free)) == len(free)
    held = Counter(p for row in dec.slot_pages for p in row)
    cached = set(a.node)
    owned = {p for p in held if p not in cached}
    assert not (set(free) & cached) and not (set(free) & set(held))
    assert all(held[p] == 1 for p in owned)
    for p in cached:
        key, depth = a.node[p]
        assert a.children[key] == p
        assert a.ref[p] == held.get(p, 0)
        assert (p in a.evictable) == (a.ref[p] == 0)
        parent = key[0]
        assert (parent == -1 and depth == 0) or (parent in cached and a.node[parent][1] == depth - 1)
    assert len(a.children) == len(cached) == len(a.ref) == len(a.last_use)
    assert set(a.evictable) <= cached
    assert len(free) + len(cached) + len(owned) == a.n_pages
    assert a.available == len(free) + len(a.evictable)
    for s, row in enumerate(dec.slot_pages):
        assert dec.page_tables[s, :len(row)].tolist() == row
        # a live slot's row holds its cached blocks first, as one chain from the root
        n_c = 0
        while n_c < len(row) and row[n_c] in cached:
            n_c += 1
        assert all(p not in cached for p in row[n_c:])
        for i in range(n_c):
            assert a.node[row[i]][1] == i and a.node[row[i]][0][0] == (row[i - 1] if i else -1)


def test_cap_keeps_one_token_to_prefill(cpu_hash):
    dec, prefills, _ = _cpu_decoder()
    a = _blocks([1, 2])                     # S = 256, a multiple of 128
    dec.admit(0, a)
    assert prefills[-1] == (0, 256) and dec.prefix_stats["cached_blocks"] == 2
    dec.admit(1, a.clone())                 # identical prompt: (S - 1) // 128 = 1 block, 128 tokens prefilled
    assert prefills[-1] == (128, 128)
    assert dec.slot_pages[1][0] == dec.slot_pages[0][0] and dec.slot_pages[1][1] != dec.slot_pages[0][1]
    assert dec.prefix_stats["cached_blocks"] == 2  # block 1 is already cached: the slot keeps its copy uncached
    b = _blocks([1, 2], tail=44)            # S = 300: both full blocks hit, 44 tokens prefilled
    dec.admit(2, b)
    assert prefills[-1] == (256, 44) and dec.slot_pages[2][:2] == dec.slot_pages[0][:2]
    dec.admit(3, _blocks([1], tail=1))      # S = 129: one block
    assert prefills[-1] == (128, 1)
    check_invariants(dec)
    st = dec.prefix_stats
    assert (st["lookups"], st["hit_blocks"], st["hit_tokens"]) == (4, 4, 512)
    assert st["prefilled_tokens"] == 256 + 128 + 44 + 1
    dec.release(3)
    dec.admit(3, _rows(100, 5))
    assert prefills[-1] == (0, 100)
    check_invariants(dec)


def test_chain_breaks_at_first_difference(cpu_hash):
    dec, prefills, _ = _cpu_decoder()
    dec.admit(0, _blocks([1, 2, 3, 4], tail=5))
    dec.admit(1, _blocks([1, 7, 3, 4], tail=5))  # blocks 2 and 3 equal A's, but after a different block 1
    assert prefills[-1] == (128, 389)
    assert dec.slot_pages[1][0] == dec.slot_pages[0][0] and not set(dec.slot_pages[1][1:]) & set(dec.slot_pages[0])
    dec.admit(2, _blocks([9, 2, 3, 4], tail=5))  # a different first block: nothing matches
    assert prefills[-1] == (0, 517)
    # B's own blocks are registered under the shared block 0, so a third prompt can follow B's chain
    dec.admit(3, _blocks([1, 7, 3], tail=7))
    assert prefills[-1] == (384, 7) and dec.slot_pages[3][:3] == dec.slot_pages[1][:3]
    check_invariants(dec)


def test_refcounts_with_overlapping_slots(cpu_hash):
    dec, _, _ = _cpu_decoder()
    p = _blocks([1, 2, 3], tail=10)
    dec.admit(0, p)
    shared = dec.slot_pages[0][:3]
    dec.admit(1, p.clone())
    dec.admit(2, _blocks([1, 2], tail=3))
    a = dec.allocator
    assert [a.ref[q] for q in shared] == [3, 3, 2]
    dec.release(0)  # the donor leaves first: its blocks stay, held by the others
    assert [a.ref[q] for q in shared] == [2, 2, 1] and not a.evictable
    check_invariants(dec)
    dec.release(1)
    assert [a.ref[q] for q in shared] == [1, 1, 0] and list(a.evictable) == [shared[2]]
    dec.release(2)
    assert set(a.evictable) == set(shared) and a.available == a.n_pages
    check_invariants(dec)
    # a released prefix is still found
    dec.admit(0, p.clone())
    assert dec.slot_pages[0][:3] == shared and not a.evictable
    check_invariants(dec)


def test_eviction_lru_deepest_first(cpu_hash):
    dec, prefills, _ = _cpu_decoder(slots=2, max_tokens_per_slot=2048, total_pages=12)
    a = dec.allocator
    dec.admit(0, _blocks([1, 2, 3], tail=1))   # 4 pages: A0 A1 A2 + tail
    A = [a.node[p][0] for p in dec.slot_pages[0][:3]]  # trie keys: an evicted page is reused under another key
    dec.release(0)
    dec.admit(0, _blocks([5, 6], tail=1))      # 3 pages: B0 B1 + tail (A is older)
    B = [a.node[p][0] for p in dec.slot_pages[0][:2]]
    dec.release(0)
    assert a.available == 12 and len(a.free) == 7 and a.cached_blocks == 5
    # 9 pages: 7 free, then 2 evicted: A's two deepest blocks (oldest use, deepest first)
    dec.admit(1, _blocks([11, 12, 13, 14, 15, 16, 17, 18], tail=1))
    assert a.stats["evictions"] == 2 and A[2] not in a.children and A[1] not in a.children and A[0] in a.children
    assert all(k in a.children for k in B)
    check_invariants(dec)
    dec.release(1)
    # A's root block is found again (a hit touches it), so B is now the oldest: its deepest block goes first
    assert len(a.free) == 1
    dec.admit(0, _blocks([1, 22], tail=1))
    assert prefills[-1] == (128, 129) and dec.slot_pages[0][0] == a.children[A[0]]
    assert a.stats["evictions"] == 3 and B[0] in a.children and B[1] not in a.children
    dec.release(0)
    before = a.stats["evictions"]
    n_free = len(a.free)
    dec.admit(1, _rows(PAGE * (n_free + 1) - 1, 77))   # needs every free page + 1
    assert a.stats["evictions"] == before + 1 and B[0] not in a.children and A[0] in a.children
    check_invariants(dec)
    # clear drops every evictable block; live ones stay
    held, n_evictable = set(a.node) - set(a.evictable), len(a.evictable)
    assert held and n_evictable and dec.clear_prefix_cache() == n_evictable
    assert set(a.node) == held and not a.evictable
    check_invariants(dec)


def test_random_admissions_and_releases_keep_the_invariants(cpu_hash):
    rng = random.Random(1234)
    dec, prefills, _ = _cpu_decoder(slots=4, max_tokens_per_slot=1024, total_pages=30)
    a = dec.allocator
    live = {}
    families = [[rng.randrange(1000) for _ in range(7)] for _ in range(3)]
    for it in range(300):
        idle = [s for s in range(dec.slots) if s not in live]
        op = rng.random()
        if idle and op < 0.55:
            fam = rng.choice(families)
            n_shared = rng.randrange(0, 7)
            seeds = fam[:n_shared] + [rng.randrange(1000, 2000) for _ in range(rng.randrange(0, 7 - n_shared))]
            tail = rng.choice([0, 1, 60, 127]) if seeds else rng.randrange(1, 127)
            p = _blocks(seeds, tail=tail, tail_seed=rng.randrange(10 ** 6))
            S = p.shape[0]
            if S + 1 > dec.pages_per_slot * PAGE:
                continue
            d = dec.prefix_digests(p)
            hits = dec.prefix_hits(d, S)
            need = -(-(S + 1) // PAGE) - len(hits)
            if need > a.available - a.evictable_among(hits):
                continue
            s = rng.choice(idle)
            n_before = len(prefills)
            dec.admit(s, p, digests=d)
            assert len(prefills) == n_before + 1 and prefills[-1] == (PAGE * len(hits), S - PAGE * len(hits))
            assert dec.slot_pages[s][:len(hits)] == hits
            live[s] = S
        elif live and op < 0.8:
            s = rng.choice(sorted(live))
            dec.release(s)
            del live[s]
        elif live:
            n = rng.choice([1, 8, 64])
            grow = sum(max(0, min(dec.pages_per_slot, -(-(dec._pos_host[s] + n + 1) // PAGE)) - len(dec.slot_pages[s]))
                       for s in live)
            if grow > a.available:
                continue
            dec.run(n)
        elif rng.random() < 0.3:
            dec.clear_prefix_cache()
        check_invariants(dec)
    st = dec.prefix_stats
    assert st["hit_blocks"] > 20 and st["evictions"] > 0
    for s in sorted(live):
        dec.release(s)
    check_invariants(dec)
    dec.clear_prefix_cache()
    assert len(a.free) == a.n_pages


# ------------------------------------------------------------------------------------------------
# generate_batch accounting
# ------------------------------------------------------------------------------------------------
def test_generate_batch_shares_one_video_prompt(cpu_hash):
    """The pool holds one 16,470-token prompt plus 8 budgets: with prefix caching 8 requests that share the prompt
    run at once; without it they run one at a time."""
    S, max_new, check_every = 16470, 16, 8
    shared = S // PAGE
    own = -(-(S + max_new + check_every) // PAGE) - shared
    pool = shared + 8 * own
    video = _rows(S, 5)
    prompts = [video.clone() for _ in range(8)]
    results = {}
    for on in (True, False):
        dec, prefills, log = _cpu_decoder(slots=8, max_tokens_per_slot=(shared + own) * PAGE, total_pages=pool,
                                          prefix_cache=on, max_new=max_new)
        out = serving.generate_batch(None, prompts, max_new_tokens=max_new, check_every=check_every, decoder=dec,
                                     prefix_cache=on)
        assert [len(o) for o in out] == [max_new] * 8
        results[on] = (max(log), prefills, dec)
    busiest, prefills, dec = results[True]
    assert busiest == 8 and prefills[0] == (0, S) and prefills[1:] == [(shared * PAGE, S - shared * PAGE)] * 7
    assert dec.prefix_stats["hit_tokens"] == 7 * shared * PAGE
    assert dec.allocator.available == pool and len(dec.allocator.free) == pool - shared
    busiest, prefills, _ = results[False]
    assert busiest == 1 and prefills == [(0, S)] * 8


def test_generate_batch_argument_errors(cpu_hash):
    prompts = [_rows(10, 1)]
    with pytest.raises(ValueError, match="fp8"):
        _cpu_decoder(kv_cache="fp8")
    with pytest.raises(ValueError, match="prefix_cache"):
        serving.generate_batch(None, prompts, max_new_tokens=4, decoder=_cpu_decoder(prefix_cache=True)[0])
    with pytest.raises(ValueError, match="prefix_cache"):
        serving.generate_batch(None, prompts, max_new_tokens=4, decoder=_cpu_decoder(prefix_cache=False)[0],
                               prefix_cache=True)
    with pytest.raises(ValueError, match="max_new"):
        serving.generate_batch(None, prompts, max_new_tokens=65, decoder=_cpu_decoder(prefix_cache=False)[0])
    # the decoder's whole history is served (token 0 from the stubbed prefill, then one per step)
    assert serving.generate_batch(None, prompts, max_new_tokens=64, decoder=_cpu_decoder(prefix_cache=False)[0]) \
        == [[0] + list(range(10, 10 + 63))]
    from vila_b200.model.llava_llama import LlavaLlamaModel
    with pytest.raises(ValueError, match="max_tokens_per_slot"):
        LlavaLlamaModel.generate_batch(SimpleNamespace(), [], prefix_cache=True)
    sig = inspect.signature(LlavaLlamaModel.generate_batch)
    assert sig.parameters["prefix_cache"].default is False
    assert "prefix_cache=prefix_cache" in inspect.getsource(LlavaLlamaModel.generate_batch)


def test_prefix_cache_off_keeps_the_allocator():
    dec, _, _ = _cpu_decoder(prefix_cache=False)
    assert type(dec.allocator) is serving.PageAllocator and not dec.prefix_cache


# ------------------------------------------------------------------------------------------------
# a failed call leaves a kept engine consistent
# ------------------------------------------------------------------------------------------------
def _fail_once(obj, name, when):
    """obj.name raises RuntimeError on its when-th call (1-based), then behaves as before"""
    inner, calls = getattr(obj, name), [0]

    def wrapped(*a, **kw):
        calls[0] += 1
        if calls[0] == when:
            raise RuntimeError(f"injected failure in {name}")
        return inner(*a, **kw)

    setattr(obj, name, wrapped)


def _idle(dec):
    return all(not row for row in dec.slot_pages) and bool((dec.positions < 0).all()) and \
        all(p < 0 for p in dec._pos_host)


def _expected(prompts, n):
    return [[0] + list(range(p.shape[0], p.shape[0] + n - 1)) for p in prompts]


@pytest.mark.parametrize("where,when", [("prefill_hidden", 1), ("prefill_hidden", 2), ("prefill_hidden", 3),
                                        ("replay", 2)])
def test_failed_call_releases_everything_and_the_next_call_is_right(cpu_hash, where, when):
    """A prefill raising at the first admission (no hit), at the second one (after its hit blocks were pinned) or at
    the third (with two slots live), or a step raising with slots live: the call raises, every slot is released, the
    hit blocks are unpinned and nothing is registered over unwritten K/V; the same engine then serves the next call
    with the right ids, hitting only blocks whose K/V were written."""
    dec, prefills, _ = _cpu_decoder(slots=3, max_tokens_per_slot=1024, total_pages=24, max_new=16)
    shared = _blocks([1, 2, 3])
    first = [torch.cat([shared, _rows(20 + k, 200 + k)]) for k in range(3)]
    if where == "replay":
        for g in set(dec.graphs.values()):
            _fail_once(g, "replay", when)
    else:
        _fail_once(dec.llm, "prefill_hidden", when)
    with pytest.raises(RuntimeError, match="injected"):
        serving.generate_batch(None, first, max_new_tokens=16, check_every=4, decoder=dec, prefix_cache=True)
    check_invariants(dec)
    assert _idle(dec) and dec.allocator.available == dec.allocator.n_pages and not dec.allocator.ref.keys() - set(
        dec.allocator.evictable)
    registered = dec.prefix_stats["cached_blocks"]
    assert registered == (0 if (where, when) == ("prefill_hidden", 1) else 3)
    # the next call: a prompt of the same start (hits whatever was registered) and a new one
    second = [torch.cat([shared, _rows(50, 300)]), _rows(400, 301)]
    n_before = len(prefills)
    out = serving.generate_batch(None, second, max_new_tokens=16, check_every=4, decoder=dec, prefix_cache=True)
    assert out == _expected(second, 16)
    assert prefills[n_before:] == [(PAGE * registered, second[0].shape[0] - PAGE * registered), (0, 400)]
    check_invariants(dec)
    assert _idle(dec) and dec.allocator.available == dec.allocator.n_pages


def test_admit_refuses_a_busy_slot_and_stats_need_the_option(cpu_hash):
    dec, _, _ = _cpu_decoder()
    dec.admit(0, _blocks([1], tail=3))
    before = (list(dec.slot_pages[0]), dict(dec.allocator.ref))
    with pytest.raises(ValueError, match="release"):
        dec.admit(0, _blocks([1], tail=3))
    assert (dec.slot_pages[0], dec.allocator.ref) == before
    check_invariants(dec)
    off, _, _ = _cpu_decoder(prefix_cache=False)
    with pytest.raises(ValueError, match="prefix_cache=True"):
        off.prefix_stats
    with pytest.raises(ValueError, match="prefix_cache=True"):
        off.clear_prefix_cache()


# ------------------------------------------------------------------------------------------------
# server
# ------------------------------------------------------------------------------------------------
def _server_stub(calls):
    from tests.test_sampling_cpu import _server_stub as stub
    return stub(calls)


def test_server_prefix_cache_routing():
    from vila_b200 import server as S

    def req(**kw):
        return S.ChatCompletionRequest(model="m", max_tokens=2, messages=[S.ChatMessage(role="user", content="hi")],
                                       **kw)

    calls = {"batch": [], "single": 0}
    eng = S.Engine(_server_stub(calls), "m", slots=4, prefix_cache=True, max_tokens_per_slot=4096)

    async def scenario():
        lone = await eng.complete(req())
        many = await asyncio.gather(*[eng.complete(req()) for _ in range(3)])
        chunks = [c async for c in eng.stream(req(stream=True))]
        return lone, many, chunks

    lone, many, chunks = asyncio.run(scenario())
    assert lone["choices"][0]["message"]["content"] == "7 8"
    assert calls["single"] == 1 and len(chunks) == 3  # only the streaming request took the single-stream path
    assert calls["batch"][0] == (1, {"prefix_cache": True, "max_tokens_per_slot": 4096})  # a lone request too
    assert all(kw == {"prefix_cache": True, "max_tokens_per_slot": 4096} for _, kw in calls["batch"])
    # with --sample as well
    calls = {"batch": [], "single": 0}
    eng = S.Engine(_server_stub(calls), "m", sample=True, prefix_cache=True)
    asyncio.run(eng.complete(req(seed=3)))
    kw = calls["batch"][0][1]
    assert kw["prefix_cache"] and kw["max_tokens_per_slot"] == 20480 and kw["sampling"][0].seed == 3
    # fp8 K/V and prefix caching are refused at startup
    with pytest.raises(ValueError, match="fp8"):
        S.Engine(_server_stub(calls), "m", kv_cache="fp8", prefix_cache=True)
    src = inspect.getsource(S.main)
    assert "--prefix-cache" in src and "--max-tokens-per-slot" in src and "9.4 GB" in src
    assert 'ap.error("--prefix-cache is not supported with --kv-cache fp8")' in src
