"""GPU: the two decode engines step by step against the fp32 oracle, at NVILA's head shapes and on every
decode attention path; and the batched decode attention entry point against fp32 attention.

Engines (GraphDecoder, serving.BatchedDecoder) are checked by teacher forcing: the engine
decodes greedily, then the oracle is fed the engine's OWN ids, so every step stays comparable whatever
the near-ties.  At every decoded position:
  * the id is a greedy choice of the fp32 oracle, up to 3 bf16 ulps at the logit scale;
  * the K and V the engine wrote, in every layer, are within check_close of the fp32 oracle's (bound from
    the oracle's own bf16 run).  K/V at position p of layer l depend on the hidden state of every earlier
    layer and on attention over the whole history, so this checks each step's RoPE, attention, o-proj and
    MLP, not only the final arg-max;
  * every other pool row is bit-identical to the pool right after the prefill.
Models are random-init, each with the tiny vision tower (the oracle gets only the `llm.*` weights):
  tiny          tiny_test_config(llm_layers=3): 4/2 heads (G=2), hidden 512, vocab 1024
  8b-shallow    NVILA-8B's LLM at full width with 2 layers: 28/4 heads (G=7), inter 18944, vocab 152,064
  lite-shallow  NVILA-Lite-3B's LLM with 2 layers: 16/2 heads (G=8), inter 11008, tied lm_head
"""
import dataclasses
import gc

import pytest
import torch

from oracle import vila_oracle as O
from tests.helpers import check_close, oracle_from_state_dict, report_rel
from tests.test_kernels_gpu import _ops, bf, ref_attention

pytestmark = pytest.mark.gpu

PAGE = 128


@pytest.fixture(autouse=True)
def _fp32_truth():
    """the fp32 oracle must really be fp32 on the device"""
    saved = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32,
             torch.get_float32_matmul_precision())
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved[:2]
    torch.set_float32_matmul_precision(saved[2])


# ------------------------------------------------------------------------------------------------
# models: one alive at a time (8b-shallow is ~3 GB of bf16 weights plus its two oracles)
# ------------------------------------------------------------------------------------------------
_MODELS = {}


def _release():
    """the model holds reference cycles: its memory returns only after a collection"""
    _MODELS.clear()
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _free_models():
    yield
    _release()


def _config(kind):
    from vila_b200.model import Qwen2Config, nvila_lite_3b, tiny_test_config
    cfg = tiny_test_config(llm_layers=3)
    if kind == "8b-shallow":
        cfg = dataclasses.replace(cfg, llm_cfg=Qwen2Config(num_hidden_layers=2))
    elif kind == "lite-shallow":
        cfg = dataclasses.replace(cfg, llm_cfg=dataclasses.replace(nvila_lite_3b().llm_cfg, num_hidden_layers=2))
    return cfg


def _model(kind):
    """-> (model, fp32 oracle, bf16 oracle), both oracles evaluated on the device"""
    if kind not in _MODELS:
        _release()
        from vila_b200.model import LlavaLlamaModel
        cfg = _config(kind)
        model = LlavaLlamaModel(cfg, device="cuda").init_random(23, device_rng=kind != "tiny")
        sd = {k: v for k, v in model.state_dict().items() if k.startswith("llm.")}
        _MODELS[kind] = (model, oracle_from_state_dict(sd, cfg, torch.float32, device="cuda"),
                         oracle_from_state_dict(sd, cfg, torch.bfloat16, device="cuda"))
    return _MODELS[kind]


def _prompt(llm, S, seed):
    """embeddings of S random token ids"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    ids = torch.randint(0, llm.config.vocab_size, (S,), device="cuda", generator=g)
    return llm.model.embed_tokens.weight[ids].clone()


# ------------------------------------------------------------------------------------------------
# teacher-forced comparison
# ------------------------------------------------------------------------------------------------
def _teacher_forced(o, emb, ids):
    """The oracle on the prompt, then on the embeddings of ids[:-1] with the prompt's K/V.
    -> (logits [len(ids), V] fp32: row i scores ids[i], per layer (k, v) [Hkv, S + len(ids) - 1, D])"""
    table = o.llm["model.embed_tokens.weight"]
    lg0, past = O.qwen2_forward(emb.to(table.dtype), o.llm, o.lcfg, last_only=True)
    lg, past = O.qwen2_forward(table[torch.tensor(ids[:-1], device=table.device)], o.llm, o.lcfg, past=past)
    return torch.cat([lg0, lg]).float(), past


def _decoded_rows(page_row, S, n_ids):
    """(pages, rows) of the positions a decode of n_ids ids wrote: S .. S + n_ids - 2 (the last id is
    never fed back)"""
    pos = torch.arange(S, S + n_ids - 1, device=page_row.device)
    return page_row[pos // PAGE].long(), pos % PAGE


def _check_sequence(name, pool, page_row, emb, ids, o32, o16):
    """ids and the K/V of every decoded position of one sequence against the teacher-forced oracle"""
    S, L = emb.shape[0], o32.lcfg.num_hidden_layers
    with torch.no_grad():
        truth, kv32 = _teacher_forced(o32, emb, ids)
        _, kv16 = _teacher_forced(o16, emb, ids)
    margin = 3 * 2 ** -8 * truth.abs().max().item()
    for i, t in enumerate(ids):
        best = truth[i].max().item()
        assert truth[i, t].item() >= best - margin, \
            f"{name}: step {i}: id {t} scores {truth[i, t].item():.4f}, the oracle's best {best:.4f} (margin {margin:.4f})"
    pages, rows = _decoded_rows(page_row, S, len(ids))
    for li in range(L):
        for j, kv in enumerate("KV"):
            got = pool[li, j][pages, rows]                      # [n - 1, Hkv, D]
            check_close(f"{name} layer {li} {kv}", got, kv32[li][j][:, S:].transpose(0, 1),
                        kv16[li][j][:, S:].transpose(0, 1))


def _check_untouched(before, after, decoded):
    """every pool row other than the decoded positions [(pages, rows)] is bit-identical to `before`"""
    expect = before.clone()
    for pages, rows in decoded:
        expect[:, :, pages, rows] = after[:, :, pages, rows]
    assert torch.equal(after, expect), "decode changed pool rows other than the decoded positions"


# ------------------------------------------------------------------------------------------------
# engine x context cases; every decode run crosses a page boundary
# ------------------------------------------------------------------------------------------------
# (model, engine, attention path, prompt tokens S, new tokens n)
#   head   decode_attn_head_kernel, one sequence             (GraphDecoder, S + n <= 512)
#   simt   SIMT split-KV kernel, one 8-CTA cluster / KV head  (GraphDecoder, S + n <= 1024)
#   split  wgmma split-KV + separate combine, pick_splits     (GraphDecoder, longer)
#   batch  BatchedDecoder, see _run_batched
_CONTEXTS = [(250, 24), (760, 24), (3060, 24), (16370, 16)]
_PATHS = ["head", "simt", "split", "split"]


def _cases():
    out = []
    for kind in ("tiny", "8b-shallow", "lite-shallow"):
        n_ctx = 4 if kind == "tiny" else 3  # video length on the tiny model only
        out += [(kind, "graph", path, S, n) for (S, n), path in zip(_CONTEXTS[:n_ctx], _PATHS)]
        if kind != "lite-shallow":
            out.append((kind, "batched", "batch", None, 16))
    return out


CASES = _cases()  # grouped by model: each model is built once


@pytest.mark.parametrize("kind,engine,path,S,n", CASES,
                         ids=[f"{k}-{e}" + (f"-{p}" if e == "graph" else "") + (f"-S{S}" if S else "")
                              for k, e, p, S, _ in CASES])
def test_engine_teacher_forced(cuda, kind, engine, path, S, n):
    with torch.inference_mode():
        if engine == "batched":
            _run_batched(kind, n)
        else:
            _run_single(kind, engine, path, S, n)


def _run_single(kind, engine, path, S, n):
    """GraphDecoder: cache_for -> prefill_hidden -> snapshot -> start -> run"""
    from vila_b200.model import GraphDecoder
    model, o32, o16 = _model(kind)
    llm = model.llm
    emb = _prompt(llm, S, seed=S)
    dec = GraphDecoder(llm, 128)
    cache = dec.cache_for(S + n)
    got_path = "split" if dec.split_tokens else "simt" if dec.num_splits else "head"
    assert got_path == path, f"{engine} at {S + n} tokens runs {got_path}, the case is for {path}"
    hid = llm.prefill_hidden(emb, cache)
    before = cache.pool.clone()
    dec.start(hid[-1], cache)
    dec.run(n)
    ids = dec.tokens(n)
    _check_untouched(before, cache.pool, [_decoded_rows(cache.page_table, S, n)])
    _check_sequence(f"{kind} {engine}/{path} S={S}", cache.pool, cache.page_table, emb, ids, o32, o16)


def _run_batched(kind, n):
    """BatchedDecoder with 4096-token slots: slot 0 S=1015 (head kernel past page 8), slot 1 S=2040
    (switches from the head to the split kernel mid-run), slot 2 idle, slot 3 S=3065 (split kernel).
    Then slot 0 is released, a 500-token prompt reuses its pages and all slots run again."""
    from vila_b200 import serving
    model, o32, o16 = _model(kind)
    llm = model.llm
    dec = serving.BatchedDecoder(llm, slots=4, max_tokens_per_slot=4096, max_new=64)
    assert dec.configs == [None, 8]
    dec.capture()
    lens = {0: 1015, 1: 2040, 3: 3065}
    prompts = {s: _prompt(llm, S, seed=S) for s, S in lens.items()}
    for s in lens:
        dec.admit(s, prompts[s])
    before = dec.pool.clone()
    dec.run(n - 1)
    assert dec.config == 8  # the head and the split kernel run in the same step
    assert dec.generated(2) == [] and int(dec.positions[2]) == -1
    _check_untouched(before, dec.pool, [_decoded_rows(dec.page_tables[s], S, n) for s, S in lens.items()])
    # slot 0 is checked before its pages return to the pool
    _check_sequence(f"{kind} batched slot 0 S=1015", dec.pool, dec.page_tables[0], prompts[0],
                    dec.generated(0), o32, o16)
    freed = list(dec.slot_pages[0])
    dec.release(0)
    lens[0], prompts[0] = 500, _prompt(llm, 500, seed=500)
    dec.admit(0, prompts[0])
    assert set(dec.slot_pages[0]) <= set(freed)
    before = dec.pool.clone()
    dec.run(n - 1)
    assert dec.generated(2) == [] and int(dec.positions[2]) == -1
    decoded = [_decoded_rows(dec.page_tables[0], 500, n)]
    for s in (1, 3):  # the second run's positions of the slots that kept running
        pages, rows = _decoded_rows(dec.page_tables[s], lens[s], 2 * n - 1)
        decoded.append((pages[n - 1:], rows[n - 1:]))
    _check_untouched(before, dec.pool, decoded)
    for s in (0, 1, 3):
        ids = dec.generated(s)
        assert len(ids) == (n if s == 0 else 2 * n - 1)
        _check_sequence(f"{kind} batched slot {s} S={lens[s]}", dec.pool, dec.page_tables[s], prompts[s],
                        ids, o32, o16)


# ------------------------------------------------------------------------------------------------
# kernel level: vila_decode_attention_batch (decode_attn_head_kernel over a batch of slots)
# ------------------------------------------------------------------------------------------------
# cached tokens of each slot (= position of the new token); -1: idle slot
BATCH_POSITIONS = [-1, 0, 1, 127, 128, 1023, 1024, 1500, 2047, -1, 4095]


def _batch_problem(Hq, Hkv, positions, pt_width, seed):
    """one shared pool with randomly permuted pages and random bf16 data everywhere; page-table rows of
    pt_width entries, those past a slot's pages hold other valid page indices (never read)"""
    D = 128
    g = torch.Generator(device="cuda").manual_seed(seed)
    need = [(p + 1 + PAGE - 1) // PAGE if p >= 0 else 0 for p in positions]
    n_pages = sum(need) + 16                          # 16 pages nobody owns
    perm = torch.randperm(n_pages, device="cuda", generator=g).to(torch.int32)
    pt = torch.randint(0, n_pages, (len(positions), pt_width), device="cuda", generator=g, dtype=torch.int32)
    o = 0
    for b, k in enumerate(need):
        pt[b, :k] = perm[o:o + k]
        o += k
    k_pool = bf(torch.randn(n_pages, PAGE, Hkv, D, device="cuda", generator=g))
    v_pool = bf(torch.randn(n_pages, PAGE, Hkv, D, device="cuda", generator=g))
    qkv_buf = bf(torch.randn(len(positions), (Hq + 2 * Hkv) * D + 64, device="cuda", generator=g))  # stride > row
    return pt, k_pool, v_pool, qkv_buf


def _batch_launch(ops, Hq, Hkv, qkv_buf, pos, k_pool, v_pool, pt, out_buf, inv):
    D = 128
    ops.decode_attention_batch(qkv_buf[:, :(Hq + 2 * Hkv) * D], pos, k_pool, v_pool, pt, out_buf[:, :Hq * D],
                               inv, Hq, Hkv, D, D ** -0.5)


@pytest.mark.parametrize("Hq,Hkv", [(28, 4), (16, 2), (4, 2)])
def test_decode_attention_batch(cuda, Hq, Hkv):
    ops = _ops()
    D = 128
    N = (Hq + 2 * Hkv) * D
    positions = BATCH_POSITIONS
    B = len(positions)
    pt, k0, v0, qkv0 = _batch_problem(Hq, Hkv, positions, 40, seed=100 * Hq + Hkv)  # 40 entries: clamped to 32
    pos = torch.tensor(positions, dtype=torch.int32, device=cuda)
    inv = O.rope_inv_freq(D, 1e6).to(cuda)
    sentinel = bf(torch.full((B, Hq * D + 32), 7.0, device=cuda))  # out row stride > row
    runs = []
    for _ in range(2):  # twice: the same bits
        kp, vp, qkv, out = k0.clone(), v0.clone(), qkv0.clone(), sentinel.clone()
        _batch_launch(ops, Hq, Hkv, qkv, pos, kp, vp, pt, out, inv)
        runs.append((kp, vp, qkv, out))
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(runs[0], runs[1]))
    kp, vp, qkv, out = runs[0]
    assert torch.equal(qkv, qkv0)                                       # q / k are rotated on chip
    assert torch.equal(out[:, Hq * D:], sentinel[:, Hq * D:])           # nothing written past a row
    touched_k, touched_v = k0.clone(), v0.clone()
    for b, p in enumerate(positions):
        if p < 0:
            assert torch.equal(out[b], sentinel[b])
            continue
        q = qkv0[b, :Hq * D].view(1, Hq, D).transpose(0, 1)
        kn = qkv0[b, Hq * D:(Hq + Hkv) * D].view(1, Hkv, D).transpose(0, 1)
        vn = qkv0[b, (Hq + Hkv) * D:N].view(1, Hkv, D)
        cos, sin = O.rope_cos_sin(torch.tensor([p]), D, 1e6, torch.bfloat16)
        qr, kr = O.apply_rope(q, kn, cos.to(cuda), sin.to(cuda))
        page, row = int(pt[b, p // PAGE]), p % PAGE
        assert torch.equal(kp[page, row], kr.transpose(0, 1)[0])     # appended K/V exact
        assert torch.equal(vp[page, row], vn[0])
        touched_k[page, row], touched_v[page, row] = kp[page, row], vp[page, row]
        t = torch.arange(p, device=cuda)
        k_all = torch.cat([k0[pt[b, t // PAGE].long(), t % PAGE], kr.transpose(0, 1)], 0).float()
        v_all = torch.cat([v0[pt[b, t // PAGE].long(), t % PAGE], vn], 0).float()
        ref = ref_attention(qr.transpose(0, 1)[None].float(), k_all[None], v_all[None], True, D ** -0.5)[0, 0]
        report_rel(f"decode_attention_batch Hq={Hq} Hkv={Hkv} ctx={p}", out[b, :Hq * D].view(Hq, D), ref, 1.5e-2)
        if p <= 1023:  # the single-sequence entry point runs the same kernel template (8-page rows)
            kp1, vp1 = k0.clone(), v0.clone()
            out1 = torch.zeros(Hq * D, dtype=torch.bfloat16, device=cuda)
            ws = torch.zeros(1, dtype=torch.float32, device=cuda)
            cnt = torch.zeros(Hkv, dtype=torch.int32, device=cuda)
            ops.decode_attention(qkv0[b, :N].clone(), pos[b:b + 1], kp1, vp1, pt[b], out1, ws, cnt, inv,
                                 Hq, Hkv, D, 0, D ** -0.5)
            assert torch.equal(out[b, :Hq * D], out1), f"slot {b} (ctx {p}) differs from decode_attention"
            assert torch.equal(kp1[page, row], kp[page, row]) and torch.equal(vp1[page, row], vp[page, row])
    assert torch.equal(kp, touched_k) and torch.equal(vp, touched_v)   # every other pool byte unchanged

    # page-table rows of 16 entries: the same bits for every slot that fits them (the kernel does not
    # check a position against the row width, so positions stay <= 2047 here)
    short = [p if p < 16 * PAGE else -1 for p in positions]
    out16 = sentinel.clone()
    _batch_launch(ops, Hq, Hkv, qkv0.clone(), torch.tensor(short, dtype=torch.int32, device=cuda), k0.clone(),
                  v0.clone(), pt[:, :16].contiguous(), out16, inv)
    torch.cuda.synchronize()
    for b, p in enumerate(short):
        assert torch.equal(out16[b], out[b] if p >= 0 else sentinel[b]), f"slot {b} with 16-entry rows"

    # a captured graph replayed after the positions move equals eager launches
    pos_g = pos.clone()
    kg, vg, qg, og = k0.clone(), v0.clone(), qkv0.clone(), sentinel.clone()
    _batch_launch(ops, Hq, Hkv, qg, pos_g, kg, vg, pt, og, inv)  # warm-up
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _batch_launch(ops, Hq, Hkv, qg, pos_g, kg, vg, pt, og, inv)
    moved = [p - 3 if p >= 3 else p for p in positions]
    pos_g.copy_(torch.tensor(moved, dtype=torch.int32, device=cuda))
    kg.copy_(k0); vg.copy_(v0); qg.copy_(qkv0); og.copy_(sentinel)
    graph.replay()
    ke, ve, qe, oe = k0.clone(), v0.clone(), qkv0.clone(), sentinel.clone()
    _batch_launch(ops, Hq, Hkv, qe, torch.tensor(moved, dtype=torch.int32, device=cuda), ke, ve, pt, oe, inv)
    torch.cuda.synchronize()
    assert torch.equal(og, oe) and torch.equal(kg, ke) and torch.equal(vg, ve) and torch.equal(qg, qe)
    assert not torch.equal(og, out)  # the replay used the moved positions
