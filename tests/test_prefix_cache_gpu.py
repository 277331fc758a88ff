"""GPU: prefix caching in the continuous-batching engine.

  * vila_prefix_block_hash is bit-identical to the numpy rule (vila_b200/prefix_cache.block_digests) over row counts,
    widths, row padding, crafted bit patterns and keys, and writes nothing past the last full block;
  * exact hit: a request admitted over a donor's cached blocks writes the K/V rows, and picks the first token, of a
    chunked prefill of its suffix over the donor's prefix, and the shared pages never change;
  * no hit: prompts that share no full block decode exactly as with prefix_cache=False, greedy and sampled;
  * image prompts through LlavaLlamaModel.generate_batch(prefix_cache=True) hit (the embeddings are bit-reproducible)
    and stay greedy choices of the fp32 oracle;
  * a pool small enough to evict keeps every rule above and never changes a page a live slot holds;
  * NVILA-8B at full size: 4 requests sharing a 16,384-token prefix.
"""
import dataclasses
import gc

import numpy as np
import pytest
import torch

from tests.helpers import greedy_ids_match, oracle_from_state_dict
from vila_b200.prefix_cache import PAGE, block_digests

pytestmark = pytest.mark.gpu

KEYS = [(0, 0), (0x0123456789ABCDEF, 0xFEDCBA9876543210), (2 ** 64 - 1, 0x9E3779B97F4A7C15)]


# ------------------------------------------------------------------------------------------------
# kernel
# ------------------------------------------------------------------------------------------------
def _hash_raw(x, key0, key1, extra_blocks=2):
    """vila_prefix_block_hash into an out buffer with `extra_blocks` sentinel entries past the last full block"""
    from vila_b200 import _lib
    from vila_b200.ops import _stream
    rows, cols = x.shape
    out = torch.full((rows // PAGE + extra_blocks, 2), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device="cuda")
    rc = _lib.load().vila_prefix_block_hash(x.data_ptr(), x.stride(0), rows, cols, key0, key1, out.data_ptr(),
                                            _stream())
    assert rc == 0, _lib.load().vila_last_error()
    torch.cuda.synchronize()
    got = out.cpu().numpy().view(np.uint64)
    assert (out[rows // PAGE:] == 0x5A5A5A5A5A5A5A5A).all(), "written past the last full block"
    return got[:rows // PAGE]


def _crafted(rows, cols, kind, g):
    if kind == "random":
        return torch.randn(rows, cols, device="cuda", generator=g).to(torch.bfloat16)
    if kind == "zeros":
        return torch.zeros(rows, cols, dtype=torch.bfloat16, device="cuda")
    bits = torch.randint(-2 ** 15, 2 ** 15, (rows, cols), device="cuda", generator=g, dtype=torch.int32)
    if kind == "signed_zeros":  # +0 and -0 only: equal as numbers, different as bits
        bits = torch.where(bits > 0, 0, -2 ** 15)
    elif kind == "nan_payloads":  # exponent all ones, random payloads and signs
        bits = (bits & -32641) | 0x7F80 | 1  # keep sign and mantissa, set the exponent, mantissa != 0
    return bits.to(torch.int16).view(torch.bfloat16)


@pytest.mark.parametrize("cols", [512, 3584])
def test_hash_kernel_matches_numpy_rule(cuda, cols):
    from vila_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(cols)
    for rows in (127, 128, 129, 300, 16470):
        kinds = ("random", "zeros", "signed_zeros", "nan_payloads") if rows <= 300 else ("random",)
        for kind in kinds:
            x = _crafted(rows, cols, kind, g)
            keys = KEYS if rows <= 300 else KEYS[1:2]
            for k0, k1 in keys:
                want = block_digests(x, k0, k1)
                got = _hash_raw(x, k0, k1)
                assert np.array_equal(got, want), (rows, cols, kind, hex(k0))
            # the wrapper: same bits, int64 view
            if kind == "random":
                w = ops.prefix_block_hash(x, *KEYS[1]).cpu().numpy().view(np.uint64)
                assert np.array_equal(w, block_digests(x, *KEYS[1]))
    # row padding full of NaN garbage is not read
    x = _crafted(300, cols, "random", g)
    buf = torch.full((300, cols + 68), float("nan"), dtype=torch.bfloat16, device="cuda")
    buf[:, :cols] = x
    assert np.array_equal(_hash_raw(buf[:, :cols], *KEYS[2]), block_digests(x, *KEYS[2]))
    assert np.array_equal(ops.prefix_block_hash(buf[:, :cols], *KEYS[2]).cpu().numpy().view(np.uint64),
                          block_digests(x, *KEYS[2]))
    # +0 / -0 and one NaN payload bit change the digest (bits, not values)
    z = torch.zeros(128, cols, dtype=torch.bfloat16, device="cuda")
    mz = z.clone()
    mz[77, 5] = -0.0
    assert not np.array_equal(_hash_raw(z, *KEYS[1]), _hash_raw(mz, *KEYS[1]))


# ------------------------------------------------------------------------------------------------
# models
# ------------------------------------------------------------------------------------------------
_MODELS = {}


def _release():
    _MODELS.clear()
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _free_models():
    yield
    _release()


def _model(kind):
    if kind not in _MODELS:
        _release()
        from vila_b200.model import LlavaLlamaModel, Qwen2Config, tiny_test_config
        cfg = tiny_test_config(llm_layers=3)
        if kind == "8b-shallow":
            cfg = dataclasses.replace(cfg, llm_cfg=Qwen2Config(num_hidden_layers=2))
        _MODELS[kind] = LlavaLlamaModel(cfg, device="cuda").init_random(23, device_rng=kind != "tiny")
    return _MODELS[kind]


def _emb(llm, S, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ids = torch.randint(0, llm.config.vocab_size, (S,), device="cuda", generator=g)
    return llm.model.embed_tokens.weight[ids].clone()


def _rows_of(dec, slot, t0, t1):
    """K/V rows [t0, t1) of a slot: [L, 2, t1 - t0, Hkv, D]"""
    t = torch.arange(t0, t1, device="cuda")
    pages = torch.tensor(dec.slot_pages[slot], device="cuda")[t // PAGE]
    return dec.pool[:, :, pages, t % PAGE]


def _chunked_reference(llm, donor, prompt, p0):
    """the donor prefilled into a private cache, its length set to p0, then prompt[p0:] prefilled
    -> (K/V rows [p0, S) as _rows_of lays them out, first token)"""
    S = prompt.shape[0]
    cache = llm.new_cache(max(S, donor.shape[0]) + PAGE)
    llm.prefill_hidden(donor, cache)
    cache.length = p0
    hid = llm.prefill_hidden(prompt[p0:], cache)
    tok = int(torch.argmax(llm.logits_from_hidden(hid[-1:])[0].float()))
    t = torch.arange(p0, S, device="cuda")
    return cache.pool[:, :, cache.page_table[t // PAGE].long(), t % PAGE], tok


def _exact_hit(llm, donor, prompt, total_pages=None, max_tokens=None):
    from vila_b200 import serving
    S_B = prompt.shape[0]
    max_tokens = max_tokens or (max(donor.shape[0], S_B) + 64 + PAGE) // PAGE * PAGE
    dec = serving.BatchedDecoder(llm, slots=2, max_tokens_per_slot=max_tokens, max_new=32, total_pages=total_pages,
                                 prefix_cache=True)
    dec.capture()
    dec.admit(0, donor)
    shared = list(dec.slot_pages[0][:donor.shape[0] // PAGE])
    snap = dec.pool[:, :, shared].clone()
    dec.admit(1, prompt)
    n_hit = dec.prefix_stats["hit_blocks"]
    p0 = PAGE * n_hit
    assert dec.slot_pages[1][:n_hit] == shared[:n_hit]
    want_kv, want_tok = _chunked_reference(llm, donor, prompt, p0)
    assert torch.equal(_rows_of(dec, 1, p0, S_B), want_kv), "K/V rows of the suffix differ from a chunked prefill"
    assert dec.generated(1)[0] == want_tok
    dec.run(16)
    torch.cuda.synchronize()
    assert len(dec.generated(0)) == len(dec.generated(1)) == 17
    assert torch.equal(dec.pool[:, :, shared], snap), "a shared page changed"
    return dec, n_hit


@pytest.mark.parametrize("kind", ["tiny", "8b-shallow"])
def test_exact_hit(cuda, kind):
    llm = _model(kind).llm
    A = _emb(llm, 700, 1)
    for n_shared, S_B, want_hit in ((640, 650, 5), (300, 900, 2), (512, 512, 3), (700, 700, 5), (100, 400, 0)):
        B = torch.cat([A[:n_shared], _emb(llm, S_B - n_shared, 2 + n_shared)]) if S_B > n_shared else A[:S_B].clone()
        _, n_hit = _exact_hit(llm, A, B)
        assert n_hit == want_hit, (n_shared, S_B)


def test_no_hit_changes_nothing(cuda):
    from vila_b200 import serving
    from vila_b200.sampling import SamplingParams
    llm = _model("tiny").llm
    prompts = [_emb(llm, n, 10 + i) for i, n in enumerate((300, 129, 40, 700, 256))]
    for sampling in (None, [SamplingParams(0.8, 20, 0.9, seed=s) for s in range(5)]):
        outs = [serving.generate_batch(llm, prompts, 12, slots=3, max_tokens_per_slot=1024, sampling=sampling,
                                       prefix_cache=on) for on in (False, True)]
        assert outs[0] == outs[1]


def test_image_prompts_hit_and_match_oracle(cuda):
    model = _model("tiny")
    cfg = model.config
    g = torch.Generator().manual_seed(5)
    S = cfg.vision_tower_cfg.image_size
    images = [torch.randn(3, S, S, generator=g).to(torch.bfloat16).cuda() for _ in range(9)]
    head = torch.randint(3, 900, (6,), generator=g).tolist() + [cfg.image_token_id] * len(images)
    questions = [torch.randint(3, 900, (5 + 3 * k,), generator=g).tolist() for k in range(4)]
    reqs = [(torch.tensor([head + q]), images) for q in questions]
    as_req = [{"input_ids": i, "media": {"image": list(ims)}, "media_config": {"image": {}}} for i, ims in reqs]
    max_new = 10
    first = model.generate_batch(as_req[:1], max_new_tokens=max_new, slots=2, max_tokens_per_slot=1024,
                                 eos_token_id=[], prefix_cache=True)
    cached = first + model.generate_batch(as_req[1:], max_new_tokens=max_new, slots=2, max_tokens_per_slot=1024,
                                          eos_token_id=[], prefix_cache=True)
    dec = model._prefix_engine[1]
    st = dec.prefix_stats
    assert st["lookups"] == 4 and st["hit_blocks"] >= 3, st  # the kept engine served the later calls' prefixes
    fresh = model.generate_batch(as_req, max_new_tokens=max_new, slots=2, max_tokens_per_slot=1024, eos_token_id=[])
    oracle = oracle_from_state_dict(model.state_dict(), cfg, torch.float32, device="cuda")
    for (ids, ims), c_ids, f_ids in zip(reqs, cached, fresh):
        want, logits = oracle.generate(ids, [im.float() for im in ims], max_new)
        margin = 3 * 2 ** -8 * logits.abs().max().item()
        greedy_ids_match(c_ids, want, logits, margin)
        greedy_ids_match(f_ids, want, logits, margin)
    # another setting rebuilds the engine and drops its cache
    model.generate_batch(as_req[:1], max_new_tokens=4, slots=3, max_tokens_per_slot=1024, prefix_cache=True)
    assert model._prefix_engine[1] is not dec and model._prefix_engine[1].prefix_stats["hit_blocks"] == 0


def test_pool_pressure_evicts_and_keeps_live_pages(cuda):
    """Requests on one shared 600-token start alternate with unrelated 850-token ones in a pool of 14 pages, one slot
    held throughout by a live request: cached blocks are evicted and the shared start is prefilled again.  A hit is
    checked against a chunked prefill over its donor when every hit block was registered by one admission that
    itself hit nothing (the donor's K/V then came from that prompt's full prefill)."""
    from vila_b200 import serving
    llm = _model("tiny").llm
    live = _emb(llm, 520, 40)
    family = _emb(llm, 600, 41)
    dec = serving.BatchedDecoder(llm, slots=2, max_tokens_per_slot=1024, max_new=16, total_pages=14,
                                 prefix_cache=True)
    dec.capture()
    dec.admit(0, live)
    held = list(dec.slot_pages[0])
    snap = dec.pool[:, :, held].clone()
    registered = {}  # page -> (admission, prompt, its p0) of the admission that registered it
    checked = refilled = 0
    for k in range(8):
        prompt = torch.cat([family, _emb(llm, 100 + 20 * k, 50 + k)]) if k % 2 == 0 else _emb(llm, 850, 60 + k)
        before = dec.prefix_stats["hit_blocks"]
        dec.admit(1, prompt)
        n_hit = dec.prefix_stats["hit_blocks"] - before
        p0 = PAGE * n_hit
        hits = dec.slot_pages[1][:n_hit]
        if k % 2 == 0 and k > 0 and n_hit < 4:
            refilled += 1
        sources = {registered[p][0] for p in hits}
        if n_hit and len(sources) == 1 and registered[hits[0]][2] == 0:
            want_kv, want_tok = _chunked_reference(llm, registered[hits[0]][1], prompt, p0)
            assert torch.equal(_rows_of(dec, 1, p0, prompt.shape[0]), want_kv), k
            assert dec.generated(1)[0] == want_tok
            checked += 1
        for p in dec.slot_pages[1][n_hit:]:
            if p in dec.allocator.node:
                registered[p] = (k, prompt, p0)
        dec.run(8)
        dec.release(1)
        assert torch.equal(dec.pool[:, :, held[:4]], snap[:, :, :4]), f"a page held by the live slot changed ({k})"
    st = dec.prefix_stats
    assert st["evictions"] > 0 and checked >= 1 and refilled >= 1, (st, checked, refilled)


# ------------------------------------------------------------------------------------------------
# full size: NVILA-8B, random init
# ------------------------------------------------------------------------------------------------
def test_fullsize_shared_video_prefix(cuda):
    from tests import test_fullsize_gpu as F
    from vila_b200 import serving

    _release()
    F._MODELS.clear()
    gc.collect()
    torch.cuda.empty_cache()
    try:
        llm = F.get_model("image").llm
        prefix = _emb(llm, 16384, 3)
        prompts = [torch.cat([prefix, _emb(llm, 86 + 4 * k, 70 + k)]) for k in range(4)]
        dec = serving.BatchedDecoder(llm, slots=4, max_tokens_per_slot=16384 + 256, max_new=16, prefix_cache=True)
        dec.capture()
        dec.admit(0, prompts[0])
        shared = list(dec.slot_pages[0][:128])
        snap = dec.pool[:, :, shared].clone()
        for k in range(1, 4):
            dec.admit(k, prompts[k])
            assert dec.slot_pages[k][:128] == shared
        assert dec.prefix_stats["hit_tokens"] == 3 * 16384
        want_kv, want_tok = _chunked_reference(llm, prompts[0], prompts[2], 16384)
        assert torch.equal(_rows_of(dec, 2, 16384, prompts[2].shape[0]), want_kv)
        assert dec.generated(2)[0] == want_tok
        del want_kv
        dec.run(8)
        torch.cuda.synchronize()
        assert all(len(dec.generated(k)) == 9 for k in range(4))
        assert torch.equal(dec.pool[:, :, shared], snap)
    finally:
        F._MODELS.clear()
        gc.collect()
        torch.cuda.empty_cache()
