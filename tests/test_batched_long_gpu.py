"""GPU: batched split-KV decode attention (vila_decode_attention_split_batch) and the continuous-batching
engine with slots longer than 4096 tokens (vila_b200/serving.py)."""
import pytest
import torch

from oracle import vila_oracle as O
from tests.helpers import check_decode_attention, greedy_ids_match, oracle_from_state_dict
from tests.test_kernels_gpu import _ops, bf

pytestmark = pytest.mark.gpu

CTXS = [0, 5, 127, 128, 4095, 4096, 16448, 65814]   # cached tokens (= position of the new token)
SPLIT_TOKENS, NUM_SPLITS = 1024, 68                 # the engine's largest ladder entry


def _pool_problem(Hq, Hkv, seed):
    """One shared pool with randomly permuted pages and garbage everywhere; slots of CTXS plus idle
    slots (position -1) at the front, in the middle and at the end."""
    D = 128
    g = torch.Generator(device="cuda").manual_seed(seed)
    positions = [-1, CTXS[0], CTXS[1], CTXS[2], -1, *CTXS[3:], -1]
    need = [(p + 1 + 127) // 128 if p >= 0 else 0 for p in positions]
    n_pages = sum(need) + 16                          # 16 pages nobody owns
    pt_stride = max(need) + 5
    perm = torch.randperm(n_pages, device="cuda", generator=g).to(torch.int32)
    # rows hold random page indices beyond the slot's pages (never dereferenced)
    pt = torch.randint(0, n_pages, (len(positions), pt_stride), device="cuda", generator=g, dtype=torch.int32)
    o = 0
    for b, n in enumerate(need):
        pt[b, :n] = perm[o:o + n]
        o += n
    k_pool = bf(torch.randn(n_pages, 128, Hkv, D, device="cuda", generator=g))
    v_pool = bf(torch.randn(n_pages, 128, Hkv, D, device="cuda", generator=g))
    N = (Hq + 2 * Hkv) * D
    qkv_buf = bf(torch.randn(len(positions), N + 64, device="cuda", generator=g))  # row stride > row
    pos = torch.tensor(positions, dtype=torch.int32, device="cuda")
    return positions, pos, pt.contiguous(), k_pool, v_pool, qkv_buf


_WORK = {}


def _batch_launch(ops, Hq, Hkv, positions, pos, pt, k_pool, v_pool, qkv_buf, out_buf, counters, num_splits):
    """work buffers and inv_freq are allocated once per shape, outside any graph capture"""
    D, B = 128, len(positions)
    N = (Hq + 2 * Hkv) * D
    key = (Hq, B, num_splits)
    if key not in _WORK:
        _WORK[key] = (torch.zeros(B * num_splits * Hq * D, dtype=torch.float32, device="cuda"),
                      torch.zeros(B * num_splits * Hq, dtype=torch.float32, device="cuda"),
                      O.rope_inv_freq(D, 1e6).cuda())
    o_partial, lse, inv = _WORK[key]
    ops.decode_attention_split_batch(qkv_buf[:, :N], pos, k_pool, v_pool, pt, out_buf[:, :Hq * D], o_partial, lse,
                                     counters, inv, Hq, Hkv, D, num_splits, SPLIT_TOKENS, D ** -0.5)


@pytest.mark.parametrize("Hq,Hkv", [(28, 4), (16, 2)])
def test_decode_attention_split_batch(cuda, Hq, Hkv):
    ops = _ops()
    D = 128
    positions, pos, pt, k_pool0, v_pool0, qkv0 = _pool_problem(Hq, Hkv, seed=Hq)
    B = len(positions)
    inv = O.rope_inv_freq(D, 1e6).cuda()
    sentinel = bf(torch.full((B, Hq * D + 32), 7.0, device=cuda))
    counters = torch.zeros(B * Hkv, dtype=torch.int32, device=cuda)
    results = []
    for _ in range(2):  # twice: identical results, counters re-armed
        k_pool, v_pool, qkv_buf, out_buf = k_pool0.clone(), v_pool0.clone(), qkv0.clone(), sentinel.clone()
        _batch_launch(ops, Hq, Hkv, positions, pos, pt, k_pool, v_pool, qkv_buf, out_buf, counters, NUM_SPLITS)
        torch.cuda.synchronize()
        assert int(counters.abs().sum()) == 0
        results.append((k_pool, v_pool, qkv_buf, out_buf))
    k_pool, v_pool, qkv_buf, out_buf = results[0]
    assert all(torch.equal(a, b) for a, b in zip(results[0], results[1]))
    assert torch.equal(out_buf[:, Hq * D:], sentinel[:, Hq * D:])      # nothing written past a row
    # every pool byte other than the appended rows is unchanged
    touched_k, touched_v = k_pool0.clone(), v_pool0.clone()
    N = (Hq + 2 * Hkv) * D
    for b, p in enumerate(positions):
        if p < 0:
            assert torch.equal(out_buf[b], sentinel[b]) and torch.equal(qkv_buf[b], qkv0[b])
            continue
        q = qkv0[b, :Hq * D].view(1, Hq, D).transpose(0, 1)
        kn = qkv0[b, Hq * D:(Hq + Hkv) * D].view(1, Hkv, D).transpose(0, 1)
        vn = qkv0[b, (Hq + Hkv) * D:N].view(1, Hkv, D)
        cos, sin = O.rope_cos_sin(torch.tensor([p]), D, 1e6, torch.bfloat16)
        qr, kr = O.apply_rope(q, kn, cos.cuda(), sin.cuda())
        page, row = int(pt[b, p // 128]), p % 128
        assert torch.equal(k_pool[page, row], kr.transpose(0, 1)[0])  # appended K/V exact
        assert torch.equal(v_pool[page, row], vn[0])
        touched_k[page, row], touched_v[page, row] = k_pool[page, row], v_pool[page, row]
        # fp32 attention over the slot's pages
        t = torch.arange(p, device=cuda)
        k_hist = k_pool0[pt[b, t // 128].long(), t % 128]
        v_hist = v_pool0[pt[b, t // 128].long(), t % 128]
        k_all = torch.cat([k_hist, kr.transpose(0, 1)], 0).float()
        v_all = torch.cat([v_hist, vn], 0).float()
        check_decode_attention(f"decode_attention_split_batch Hq={Hq} ctx={p}", out_buf[b, :Hq * D].view(Hq, D),
                               qr.transpose(0, 1), k_all, v_all, D ** -0.5)
        # bit-identical to the single-sequence kernel with counters and the same split configuration
        kp1, vp1 = k_pool0.clone(), v_pool0.clone()
        out1 = torch.zeros(Hq * D, dtype=torch.bfloat16, device=cuda)
        op1 = torch.zeros(NUM_SPLITS * Hq * D, dtype=torch.float32, device=cuda)
        lse1 = torch.zeros(NUM_SPLITS * Hq, dtype=torch.float32, device=cuda)
        cnt1 = torch.zeros(Hkv, dtype=torch.int32, device=cuda)
        ops.decode_attention_split(qkv0[b, :N].clone(), pos[b:b + 1], kp1, vp1, pt[b], out1, op1, lse1, inv,
                                   Hq, Hkv, D, NUM_SPLITS, SPLIT_TOKENS, D ** -0.5, counters=cnt1)
        assert torch.equal(out_buf[b, :Hq * D], out1), f"slot {b} (ctx {p}) differs from the single-sequence kernel"
        assert torch.equal(kp1[page, row], k_pool[page, row]) and torch.equal(vp1[page, row], v_pool[page, row])
    assert torch.equal(k_pool, touched_k) and torch.equal(v_pool, touched_v)

    # a smaller ladder entry that still covers every slot gives the same bits (the engine relies on it)
    short = [p if 0 <= p < 8 * SPLIT_TOKENS else -1 for p in positions]
    pos_s = torch.tensor(short, dtype=torch.int32, device=cuda)
    outs = []
    for n in (8, NUM_SPLITS):
        out_s = sentinel.clone()
        _batch_launch(ops, Hq, Hkv, short, pos_s, pt, k_pool0.clone(), v_pool0.clone(), qkv0.clone(), out_s,
                      counters, n)
        outs.append(out_s)
    assert torch.equal(outs[0], outs[1])

    # a captured graph replayed after the positions change equals eager launches
    pos_g = pos.clone()
    kpg, vpg, qkvg, outg = k_pool0.clone(), v_pool0.clone(), qkv0.clone(), sentinel.clone()
    src_k, src_v, src_q = k_pool0.clone(), v_pool0.clone(), qkv0.clone()
    _batch_launch(ops, Hq, Hkv, positions, pos_g, pt, kpg, vpg, qkvg, outg, counters, NUM_SPLITS)  # warm-up
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _batch_launch(ops, Hq, Hkv, positions, pos_g, pt, kpg, vpg, qkvg, outg, counters, NUM_SPLITS)
    moved = [p - 3 if p >= 3 else p for p in positions]
    pos_g.copy_(torch.tensor(moved, dtype=torch.int32, device=cuda))
    kpg.copy_(src_k); vpg.copy_(src_v); qkvg.copy_(src_q); outg.copy_(sentinel)
    graph.replay()
    torch.cuda.synchronize()
    ke, ve, qe, oe = src_k.clone(), src_v.clone(), src_q.clone(), sentinel.clone()
    _batch_launch(ops, Hq, Hkv, moved, pos_g, pt, ke, ve, qe, oe, counters, NUM_SPLITS)
    torch.cuda.synchronize()
    assert torch.equal(outg, oe) and torch.equal(kpg, ke) and torch.equal(vpg, ve) and torch.equal(qkvg, qe)
    assert int(counters.abs().sum()) == 0


# ------------------------------------------------------------------------------------------------
# engine, tiny model
# ------------------------------------------------------------------------------------------------
def _tiny():
    from vila_b200.model import LlavaLlamaModel, tiny_test_config
    cfg = tiny_test_config(llm_layers=3)
    return cfg, LlavaLlamaModel(cfg, device="cuda").init_random(21)


def _requests(cfg, text_lens, n_images, seed):
    g = torch.Generator().manual_seed(seed)
    S = cfg.vision_tower_cfg.image_size
    out = []
    for n_text, n_img in zip(text_lens, n_images):
        ids = torch.randint(3, 900, (n_text,), generator=g).tolist()
        images = [torch.randn(3, S, S, generator=g).to(torch.bfloat16) for _ in range(n_img)]
        for k in range(n_img):
            ids.insert(2 + 3 * k, cfg.image_token_id)
        out.append((torch.tensor([ids]), images))
    return out


def _prompt(model, ids, images):
    media = {"image": [im.cuda() for im in images]} if images else None
    emb, _, _ = model._embed(ids, media, {"image": {}} if images else None, None, None)
    return emb[0].clone()


def test_engine_long_slots_match_oracle(cuda):
    from vila_b200 import serving
    cfg, model = _tiny()
    reqs = _requests(cfg, [5000, 9000, 7, 12, 9], [0, 0, 1, 1, 1], seed=31)
    max_new = 10
    got = model.generate_batch([{"input_ids": i, "media": {"image": [im.cuda() for im in ims]} if ims else None}
                                for i, ims in reqs], max_new_tokens=max_new, slots=3, eos_token_id=[])
    assert [len(x) for x in got] == [max_new] * 5
    oracle = oracle_from_state_dict(model.state_dict(), cfg, torch.float32, device="cuda")
    for (ids, ims), g_ids in zip(reqs, got):
        want, logits = oracle.generate(ids, [im.cuda().float() for im in ims], max_new)
        greedy_ids_match(g_ids, want, logits, 3 * 2 ** -8 * logits.abs().max().item())

    prompts = [_prompt(model, i, ims) for i, ims in reqs]
    llm = model.llm
    # EOS in the long slot frees it early for the next request in the queue; every request is cut at
    # its first EOS and is otherwise unchanged
    eos_tok = got[1][2]
    again = serving.generate_batch(llm, prompts, max_new, eos_token_ids=[eos_tok], slots=3)
    for g_ids, a_ids in zip(got, again):
        assert a_ids == (g_ids[:g_ids.index(eos_tok) + 1] if eos_tok in g_ids else g_ids)

    # short requests in a 16K-token slot decoder: the same kernels as in a 2048-token one -> same ids
    short = prompts[2:]
    a = serving.generate_batch(llm, short, max_new, slots=3, max_tokens_per_slot=16384)
    b = serving.generate_batch(llm, short, max_new, slots=3, max_tokens_per_slot=2048)
    assert a == b

    # a request's ids do not depend on its neighbours, on the split path (9000) and the head path (short)
    both = serving.generate_batch(llm, [prompts[1], prompts[3], prompts[0]], max_new, slots=3)
    alone_long = serving.generate_batch(llm, [prompts[1]], max_new, slots=3,
                                        max_tokens_per_slot=9000 + max_new + 8 + 127)
    alone_short = serving.generate_batch(llm, [prompts[3]], max_new, slots=3)
    assert both[0] == alone_long[0] and both[1] == alone_short[0]
    assert both[2] == got[0]


# ------------------------------------------------------------------------------------------------
# full size: NVILA-Video-8B, random init
# ------------------------------------------------------------------------------------------------
def test_fullsize_video_next_to_image_requests(cuda):
    """Runs on the shared full-size model cache and leaves the device as empty as it found it: the model
    holds reference cycles, so dropping it from the cache frees its 15 GB only after a collection."""
    import gc

    from tests import test_fullsize_gpu as F

    def release():
        F._MODELS.clear()
        gc.collect()
        torch.cuda.empty_cache()

    release()
    try:
        _fullsize_video_next_to_image_requests(F.get_model("video"))
    finally:
        release()


def _fullsize_video_next_to_image_requests(model):
    from vila_b200 import serving
    cfg, llm = model.config, model.llm
    g = torch.Generator(device="cuda").manual_seed(7)
    frames = torch.randn(64, 3, 448, 448, device="cuda", generator=g).to(torch.bfloat16)
    enc = model.encoders["video"]([frames], {})[0]
    text = llm.model.embed_tokens(torch.arange(100, 122, device="cuda"))
    video = torch.cat([text[:10], enc, text[10:]], 0).clone()
    assert video.shape[0] == 16470
    del enc
    prompts = [video]
    for k in range(3):
        gk = torch.Generator().manual_seed(40 + k)
        ids = torch.randint(0, 151643, (20,), generator=gk).tolist()
        ids.insert(5, cfg.image_token_id)
        px = torch.randn(3, 448, 448, generator=gk).to(torch.bfloat16).cuda()
        prompts.append(_prompt(model, torch.tensor([ids]), [px]))
    max_new = 16
    got = serving.generate_batch(llm, prompts, max_new, slots=4)
    assert [len(x) for x in got] == [max_new] * 4
    tokens, _ = serving.slot_geometry([p.shape[0] for p in prompts], max_new, 8, 4)
    for i, p in enumerate(prompts):  # the same request with the other slots idle
        alone = serving.generate_batch(llm, [p], max_new, slots=4, max_tokens_per_slot=tokens)
        assert alone[0] == got[i], f"request {i}"
    # the video request's first 8 ids against a re-prefill of prompt + ids
    ext = torch.cat([video, llm.model.embed_tokens(torch.tensor(got[0][:8], device="cuda"))], 0)
    cache = llm.new_cache(ext.shape[0] + 8)
    hid = llm.prefill_hidden(ext, cache)
    S = video.shape[0]
    lg = llm.logits_from_hidden(hid[S - 1:S + 7]).float()
    checked = 0
    for i in range(8):
        top2 = torch.topk(lg[i], 2).values
        if (top2[0] - top2[1]) > 3 * 2 ** -8 * lg[i].abs().max():
            assert int(torch.argmax(lg[i])) == got[0][i], f"token {i}"
            checked += 1
    assert checked >= 1
    del cache, hid
    # two 8-frame video requests through the public API: sized from the requests, no ValueError
    reqs = []
    for k in range(2):
        fr = torch.randn(8, 3, 448, 448, device="cuda", generator=g).to(torch.bfloat16)
        ids = torch.tensor([[100 + k, 101, cfg.video_token_id, 102, 103]])
        reqs.append({"input_ids": ids, "media": {"video": [fr]}, "media_config": {"video": {}}})
    out = model.generate_batch(reqs, max_new_tokens=8, eos_token_id=[])
    assert [len(x) for x in out] == [8, 8]
