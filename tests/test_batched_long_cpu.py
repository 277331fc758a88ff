"""CPU: host-side policy of the continuous-batching engine at video-length contexts (vila_b200/serving.py):
slot / pool sizing from the requests, the attention kernel chosen from the host's slot lengths, and
the scheduler over slots longer than 4096 tokens."""
from types import SimpleNamespace

import pytest
import torch

from vila_b200 import serving
from vila_b200.serving import (HEAD_KERNEL_TOKENS, MAX_SLOT_TOKENS, PAGE, SPLIT_LADDER, SPLIT_TOKENS,
                               BatchedDecoder, attention_config, generate_batch, slot_geometry)


def test_slot_geometry_short_batch_keeps_todays_geometry():
    # everything fits 2048: today's 16-page slots and the full slots * 16 pool
    assert slot_geometry([300, 1500, 40], 128, 8, slots=8) == (2048, None)
    assert slot_geometry([2048 - 128 - 8], 128, 8, slots=8) == (2048, None)
    # an explicit size is kept as it is, even a small one
    assert slot_geometry([16470], 128, 8, slots=4, max_tokens_per_slot=256) == (256, None)


def test_slot_geometry_video_next_to_short_requests():
    lens, max_new, check_every = [16470, 300, 300, 2100, 5000], 128, 8
    tokens, pool = slot_geometry(lens, max_new, check_every, slots=3)
    assert tokens % PAGE == 0 and tokens >= 16470 + max_new + check_every and tokens - PAGE < 16470 + max_new + check_every
    budgets = sorted(((n + max_new + check_every + PAGE - 1) // PAGE for n in lens), reverse=True)
    assert pool == sum(budgets[:3]) and pool < 3 * tokens // PAGE
    # the pool never exceeds slots x pages_per_slot
    tokens, pool = slot_geometry([16470] * 10, 128, 8, slots=4)
    assert pool == 4 * tokens // PAGE
    # a 2056-token 8-frame video prompt no longer fits 2048: the slot grows by whole pages
    tokens, pool = slot_geometry([2056, 2056], 512, 8, slots=8)
    assert tokens == 2688 and pool == 2 * 21


def test_too_long_requests_still_raise():
    from vila_b200.serving import generate_batch as gb
    # an explicit slot too small for a request
    with pytest.raises(ValueError):
        gb(None, [torch.zeros(1020, 4)], max_new_tokens=20, slots=1, check_every=4, decoder=_FakeDecoder(1, 8, 8))
    # the sized slot is capped at the engine's limit, so a longer request is refused, not truncated
    tokens, _ = slot_geometry([MAX_SLOT_TOKENS], 128, 8, slots=2)
    assert tokens == MAX_SLOT_TOKENS
    with pytest.raises(ValueError):
        gb(None, [torch.zeros(MAX_SLOT_TOKENS, 4)], max_new_tokens=20, slots=1, check_every=4,
           decoder=_FakeDecoder(1, MAX_SLOT_TOKENS // PAGE, MAX_SLOT_TOKENS // PAGE))


def test_attention_config_from_host_lengths():
    assert attention_config(0) is None and attention_config(1) is None
    assert attention_config(HEAD_KERNEL_TOKENS) is None              # 4096 tokens: head kernel
    assert attention_config(HEAD_KERNEL_TOKENS + 1) == SPLIT_LADDER[0]
    for i, n in enumerate(SPLIT_LADDER):
        lo = SPLIT_LADDER[i - 1] * SPLIT_TOKENS + 1 if i else HEAD_KERNEL_TOKENS + 1
        for length in (lo, (lo + n * SPLIT_TOKENS) // 2, n * SPLIT_TOKENS):
            got = attention_config(length)
            assert got == n and got * SPLIT_TOKENS >= length, (length, got)
    assert attention_config(16470 + 1024) * SPLIT_TOKENS >= 16470 + 1024
    assert attention_config(65814 + 1024) * SPLIT_TOKENS >= 65814 + 1024
    with pytest.raises(ValueError):
        attention_config(MAX_SLOT_TOKENS + 1)


class _Graph:
    def __init__(self, log, key):
        self.log, self.key = log, key

    def replay(self):
        self.log.append(self.key)


def _cpu_decoder(slots, max_tokens_per_slot, total_pages=200):
    """A BatchedDecoder over CPU tensors whose step graphs only record which configuration replays."""
    cfg = SimpleNamespace(num_attention_heads=2, num_key_value_heads=1, head_dim=128, num_hidden_layers=3,
                          hidden_size=64)
    llm = SimpleNamespace(config=cfg, device=torch.device("cpu"), dtype=torch.bfloat16)
    dec = BatchedDecoder(llm, slots=slots, max_tokens_per_slot=max_tokens_per_slot, max_new=64,
                         total_pages=total_pages)
    log = []
    dec.graphs = {c: _Graph(log, c) for c in dec.configs}
    return dec, log


def _seed(dec, slot, n_cached):
    dec._ensure_pages(slot, n_cached + 1)
    dec._pos_host[slot] = n_cached


def test_engine_picks_kernel_from_longest_slot_including_appends():
    dec, log = _cpu_decoder(slots=3, max_tokens_per_slot=17 * 1024)
    assert dec.configs == [None, 8, 16, 32]
    assert dec.o_partial.numel() == 3 * 32 * 2 * 128 and dec.counters.numel() == 3 * 1
    _seed(dec, 0, 300)
    _seed(dec, 2, HEAD_KERNEL_TOKENS - 8)
    dec.run(8)                                   # longest slot attends exactly 4096 tokens at its last step
    assert log == [None] * 8 and dec.config is None and dec.launches_per_step == 7 * 3 + 2
    dec.run(1)                                   # ... and 4097 now
    assert log[-1] == 8 and dec.launches_per_step == 9 * 3 + 2
    _seed(dec, 1, 16470)
    dec.run(4)
    assert log[-4:] == [32] * 4                  # 16,474 tokens > 16 * 1024
    dec.release(1)
    dec.run(2)
    assert log[-1] == 8
    assert dec.allocator.available == dec.allocator.n_pages - len(dec.slot_pages[0]) - len(dec.slot_pages[2])


def test_small_slots_capture_only_the_head_kernel():
    for tokens in (256, 1024, 2048, HEAD_KERNEL_TOKENS):
        dec, log = _cpu_decoder(slots=2, max_tokens_per_slot=tokens)
        assert dec.configs == [None] and not hasattr(dec, "o_partial")
    dec, _ = _cpu_decoder(slots=2, max_tokens_per_slot=HEAD_KERNEL_TOKENS + PAGE)
    assert dec.configs == [None, 8]
    dec, _ = _cpu_decoder(slots=1, max_tokens_per_slot=MAX_SLOT_TOKENS, total_pages=8)
    assert dec.configs == [None] + list(SPLIT_LADDER)
    with pytest.raises(AssertionError):
        _cpu_decoder(slots=1, max_tokens_per_slot=MAX_SLOT_TOKENS + PAGE, total_pages=8)


class _FakeDecoder:
    """serving.BatchedDecoder's host-visible surface with a deterministic token rule (request with prompt
    length S emits S, S+1, ...) and a record of the attention configuration of every run."""

    def __init__(self, slots, pages_per_slot, total_pages):
        self.slots, self.pages_per_slot = slots, pages_per_slot
        self.allocator = serving.PageAllocator(total_pages)
        self.slot_pages = [[] for _ in range(slots)]
        self.state = [None] * slots
        self.configs_run = []
        self.admitted = []

    def capture(self):
        pass

    def _ensure(self, s, n_tokens):
        need = min(self.pages_per_slot, -(-n_tokens // PAGE)) - len(self.slot_pages[s])
        if need > 0:
            self.slot_pages[s].extend(self.allocator.alloc(need))

    def admit(self, s, emb):
        assert self.state[s] is None
        S = emb.shape[0]
        assert S + 1 <= self.pages_per_slot * PAGE
        self._ensure(s, S + 1)
        self.state[s] = [S, [S]]
        self.admitted.append((s, S))

    def run(self, n):
        longest = 0
        for s, st in enumerate(self.state):
            if st is not None:
                self._ensure(s, st[0] + n + 1)
                last = st[1][-1]
                st[1].extend(last + 1 + i for i in range(n))
                st[0] += n
                longest = max(longest, st[0])
        self.configs_run.append(attention_config(min(longest, self.pages_per_slot * PAGE)))

    def generated(self, s):
        return list(self.state[s][1])

    def release(self, s):
        self.allocator.release(self.slot_pages[s])
        self.slot_pages[s], self.state[s] = [], None


def test_scheduler_over_long_slots():
    """Video-length prompts next to short ones through the sized geometry: FIFO admission, EOS frees the
    long slot for the next request, the pool holds the top-`slots` budgets and is returned in full, and
    the split-KV configuration is used exactly while a long slot is active."""
    lens = [16470, 300, 9000, 120, 5000, 260]
    max_new, check_every, slots = 24, 4, 3
    tokens, pool = slot_geometry(lens, max_new, check_every, slots)
    dec = _FakeDecoder(slots, tokens // PAGE, pool)
    prompts = [torch.zeros(n, 4) for n in lens]
    # EOS: request 0 stops at its 3rd token, request 2 at its 1st
    out = generate_batch(None, prompts, max_new_tokens=max_new, eos_token_ids=(16472, 9000), slots=slots,
                         check_every=check_every, decoder=dec)
    assert out[0] == [16470, 16471, 16472] and out[2] == [9000]
    for r in (1, 3, 4, 5):
        assert out[r] == list(range(lens[r], lens[r] + max_new))
    assert [s for _, s in dec.admitted] == lens
    assert dec.allocator.available == pool and all(x is None for x in dec.state)
    assert dec.configs_run[0] == attention_config(16470 + check_every) == 32
    assert None in dec.configs_run and dec.configs_run[-1] is None  # the short tail runs the head kernel
