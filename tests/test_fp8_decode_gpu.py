"""GPU: opt-in FP8 (e4m3, one fp32 scale per row) weights in the single-stream decoder.

  * vila_gemv_fp8 against the fp64 reference on the dequantized weights (tests.helpers.GemvErrors), at every GEMV
    shape of NVILA-8B and NVILA-Lite-3B and with every fusion; bit-repeatable, graph replay included;
  * GraphDecoder in fp8 mode, teacher-forced like tests/test_decode_engines_gpu.py: the prompt runs through
    the fp32 oracle with the bf16 weights; the first id and every decoded position use an oracle whose LLM
    linear weights and lm_head are the dequantized q * s (embedding and norms unchanged);
  * bf16 decoding, the bf16 weights and state_dict() are unchanged by a round trip through fp8 mode;
  * the public greedy paths follow the mode.
"""
import math

import pytest
import torch

from oracle import vila_oracle as O
from tests.helpers import check_close, check_gemv, e4m3_rows, gemv_plan, oracle_from_state_dict, ref_quantize_e4m3_rows
from tests.test_decode_engines_gpu import _fp32_truth  # noqa: F401  (autouse: the fp32 oracle is really fp32)
from tests.test_decode_engines_gpu import _CONTEXTS, _PATHS, _check_untouched, _config, _decoded_rows, _prompt
from tests.test_kernels_gpu import _ops, bf

pytestmark = pytest.mark.gpu


def rb(t):
    return t.to(torch.bfloat16).float()


def _quant(w):
    from vila_b200.model.qwen2 import quantize_e4m3_rows
    q, s = quantize_e4m3_rows(w)
    return q, s, q.float() * s[:, None]


# ------------------------------------------------------------------------------------------------
# kernel level
# ------------------------------------------------------------------------------------------------
# (name, N, K, fusion): the GEMVs of one decode step
#   8B:   hidden 3584, inter 18944, qkv (28 + 2*4) * 128, vocab 152,064
#   Lite: hidden 2048, inter 11008, qkv (16 + 2*2) * 128, vocab 151,936 (151,936 / 132 SMs leaves a short
#         last row block)
GEMV_CASES = [
    ("8b-qkv", 4608, 3584, "bias+norm"), ("8b-o", 3584, 3584, "residual"),
    ("8b-gate_up", 37888, 3584, "swiglu+norm"), ("8b-down", 3584, 18944, "residual"),
    ("8b-lm_head", 152064, 3584, "argmax+norm"),
    ("lite-qkv", 2560, 2048, "bias+norm"), ("lite-o", 2048, 2048, "residual"),
    ("lite-gate_up", 22016, 2048, "swiglu+norm"), ("lite-down", 2048, 11008, "residual"),
    ("lite-lm_head", 151936, 2048, "argmax+norm"),
    ("short-rows", 1003, 3584, "argmax+norm"),  # blocks of 8 rows on 132 SMs, the last one 3 rows
]


def _problem(N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = bf(torch.randn(K, device="cuda", generator=g))
    # rows of very different magnitude: the per-row scales matter
    w = bf(torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)
           * torch.exp(torch.randn(N, 1, device="cuda", generator=g)))
    b = bf(torch.randn(N, device="cuda", generator=g))
    r = bf(torch.randn(N, device="cuda", generator=g))
    nw = bf(1 + 0.1 * torch.randn(K, device="cuda", generator=g))
    return x, w, b, r, nw


def _launch(ops, fusion, x, q, s, b, r, nw, key=None):
    if fusion == "bias+norm":
        return ops.gemv(x, q, w_scale=s, bias=b, norm_w=nw, norm_eps=1e-6, static_w=True)
    if fusion == "residual":
        return ops.gemv(x, q, w_scale=s, residual=r, static_w=True)
    if fusion == "swiglu+norm":
        return ops.gemv(x, q, w_scale=s, norm_w=nw, norm_eps=1e-6, swiglu=True, static_w=True)
    return ops.gemv(x, q, w_scale=s, norm_w=nw, norm_eps=1e-6, argmax_key=key, static_w=True)


@pytest.mark.parametrize("name,N,K,fusion", GEMV_CASES, ids=[c[0] for c in GEMV_CASES])
def test_gemv_fp8(cuda, name, N, K, fusion):
    ops = _ops()
    x, w, b, r, nw = _problem(N, K, seed=N + K)
    q, s, deq = _quant(w)
    key = torch.zeros(1, dtype=torch.int64, device=cuda) if fusion == "argmax+norm" else None
    out = _launch(ops, fusion, x, q, s, b, r, nw, key)
    xn = O.rms_norm(x[None], nw, 1e-6)[0].float() if "norm" in fusion else x.float()
    acc = deq @ xn
    rq, rs = ref_quantize_e4m3_rows(w)
    assert torch.equal(q.view(torch.uint8), rq) and torch.equal(s, rs)
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    _, depth, regime = gemv_plan("fp8", N, K, fusion, sms)
    e = check_gemv(f"gemv_fp8 {name} {fusion}", out[None], x[None], e4m3_rows(rq, rs), N, depth=depth,
                   norm_w=nw if "norm" in fusion else None, bias=b if fusion == "bias+norm" else None,
                   residual=r[None] if fusion == "residual" else None, swiglu=fusion == "swiglu+norm",
                   record=dict(regime=regime))
    assert not e.failures(), f"gemv_fp8 {name} {fusion}: " + "; ".join(e.failures())
    if key is not None:  # the fused greedy arg-max: a best id of the fp32 reference, up to 3 bf16 ulps
        tok = int(key.item() & 0xFFFFFFFF)
        tok = 0xFFFFFFFF - tok
        margin = 3 * 2 ** -8 * acc.abs().max().item()
        assert 0 <= tok < N and acc[tok].item() >= acc.max().item() - margin, (tok, acc[tok].item(), acc.max().item())
        assert tok == int(torch.argmax(out.float()))  # the kernel's own logits decide
    # repeatable, and a captured graph replays the same bits
    key2 = torch.zeros_like(key) if key is not None else None
    again = _launch(ops, fusion, x, q, s, b, r, nw, key2)
    assert torch.equal(out, again) and (key is None or torch.equal(key, key2))
    key3 = torch.zeros_like(key) if key is not None else None
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_out = _launch(ops, fusion, x, q, s, b, r, nw, key3)
    if key3 is not None:
        key3.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, g_out) and (key is None or torch.equal(key, key3))


def test_gemv_fp8_rejects(cuda):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(5)
    K = 3576  # a multiple of 8 (the bf16 kernels take it), not of 16
    x = bf(torch.randn(K, device=cuda, generator=g))
    q, s, _ = _quant(bf(torch.randn(64, K, device=cuda, generator=g)))
    y = torch.full((64,), 7.0, dtype=torch.bfloat16, device=cuda)
    with pytest.raises(RuntimeError, match="K % 16"):
        ops.gemv(x, q, w_scale=s, out=y)
    torch.cuda.synchronize()
    assert bool((y == 7.0).all())  # nothing was launched
    x = bf(torch.randn(3584, device=cuda, generator=g))
    q, s, _ = _quant(bf(torch.randn(64, 3584, device=cuda, generator=g)))
    with pytest.raises(ValueError):
        ops.gemv(x, q, w_scale=s, variant=1)  # no register-staged form
    with pytest.raises(ValueError):
        ops.gemv(x, q)  # scales are required
    with pytest.raises(ValueError):
        ops.gemv(x, q, w_scale=s[:32])


# ------------------------------------------------------------------------------------------------
# GraphDecoder in fp8 mode, teacher-forced
# ------------------------------------------------------------------------------------------------
_MODEL = {}


def _release():
    import gc
    _MODEL.clear()
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _free_models():
    yield
    _release()


def _model(kind):
    """-> (model, o32, o16, q32, q16): the oracles with the bf16 weights, and the same oracles whose LLM
    linear weights and lm_head are the dequantized fp8 weights of the model's own copies"""
    if kind not in _MODEL:
        _release()
        from vila_b200.model import LlavaLlamaModel
        cfg = _config(kind)
        model = LlavaLlamaModel(cfg, device="cuda").init_random(23, device_rng=kind != "tiny")
        sd = {k: v for k, v in model.state_dict().items() if k.startswith("llm.")}
        llm = model.llm
        llm.set_decode_weights("fp8")
        lc = cfg.llm_cfg
        Hq, Hkv, D = lc.num_attention_heads, lc.num_key_value_heads, lc.head_dim

        def deq(qs):
            return qs[0].float() * qs[1][:, None]

        dq = {"llm.lm_head.weight": deq(llm._fp8_weights.lm_head)}
        for i, f in enumerate(llm._fp8_weights.layers):
            pre = f"llm.model.layers.{i}."
            qkv = deq(f.qkv)
            dq[pre + "self_attn.q_proj.weight"] = qkv[:Hq * D]
            dq[pre + "self_attn.k_proj.weight"] = qkv[Hq * D:(Hq + Hkv) * D]
            dq[pre + "self_attn.v_proj.weight"] = qkv[(Hq + Hkv) * D:]
            dq[pre + "self_attn.o_proj.weight"] = deq(f.o)
            gu = deq(f.gu)
            dq[pre + "mlp.gate_proj.weight"], dq[pre + "mlp.up_proj.weight"] = gu[0::2], gu[1::2]
            dq[pre + "mlp.down_proj.weight"] = deq(f.down)
        llm.set_decode_weights("bf16")
        oracles = []
        for dt in (torch.float32, torch.bfloat16):
            base = oracle_from_state_dict(sd, cfg, dt, device="cuda")
            quant = oracle_from_state_dict(sd, cfg, dt, device="cuda")
            quant.llm.update({k[len("llm."):]: v.to(dt) for k, v in dq.items()})
            oracles += [base, quant]
        del dq
        _MODEL[kind] = (model, oracles[0], oracles[2], oracles[1], oracles[3])
    return _MODEL[kind]


def _teacher_forced(base, quant, emb, ids):
    """The prompt on the bf16 weights (its K/V), its last position scored by the dequantized lm_head; then
    the embeddings of ids[:-1] on the dequantized weights.  -> (logits [len(ids), V] fp32, per layer (k, v))"""
    table = quant.llm["model.embed_tokens.weight"]
    prompt_w = dict(base.llm)
    prompt_w["lm_head.weight"] = quant.llm["lm_head.weight"]
    lg0, past = O.qwen2_forward(emb.to(table.dtype), prompt_w, quant.lcfg, last_only=True)
    lg, past = O.qwen2_forward(table[torch.tensor(ids[:-1], device=table.device)], quant.llm, quant.lcfg,
                               past=past)
    return torch.cat([lg0, lg]).float(), past


def _check_fp8_sequence(name, pool, page_row, emb, ids, o32, q32, o16, q16):
    """as test_decode_engines_gpu._check_sequence, against the fp8 teacher-forced oracle"""
    S, L = emb.shape[0], q32.lcfg.num_hidden_layers
    with torch.no_grad():
        truth, kv32 = _teacher_forced(o32, q32, emb, ids)
        _, kv16 = _teacher_forced(o16, q16, emb, ids)
    margin = 3 * 2 ** -8 * truth.abs().max().item()
    for i, t in enumerate(ids):
        best = truth[i].max().item()
        assert truth[i, t].item() >= best - margin, \
            f"{name}: step {i}: id {t} scores {truth[i, t].item():.4f}, the oracle's best {best:.4f} (margin {margin:.4f})"
    pages, rows = _decoded_rows(page_row, S, len(ids))
    for li in range(L):
        for j, kv in enumerate("KV"):
            got = pool[li, j][pages, rows]
            check_close(f"{name} layer {li} {kv}", got, kv32[li][j][:, S:].transpose(0, 1),
                        kv16[li][j][:, S:].transpose(0, 1))


def _fp8_cases():
    out = []
    for kind in ("tiny", "8b-shallow", "lite-shallow"):
        n_ctx = 4 if kind == "tiny" else 3
        out += [(kind, path, S, n) for (S, n), path in zip(_CONTEXTS[:n_ctx], _PATHS)]
    return out


FP8_CASES = _fp8_cases()


@pytest.mark.parametrize("kind,path,S,n", FP8_CASES, ids=[f"{k}-{p}-S{S}" for k, p, S, _ in FP8_CASES])
def test_graph_decoder_fp8_teacher_forced(cuda, kind, path, S, n):
    from vila_b200.model import GraphDecoder
    model, o32, o16, q32, q16 = _model(kind)
    llm = model.llm
    with torch.inference_mode():
        emb = _prompt(llm, S, seed=S)
        llm.set_decode_weights("fp8")
        try:
            dec = GraphDecoder(llm, 128)
            assert dec.fp8 is not None
            cache = dec.cache_for(S + n)
            got_path = "split" if dec.split_tokens else "simt" if dec.num_splits else "head"
            assert got_path == path, f"fp8 graph decoder at {S + n} tokens runs {got_path}, the case is for {path}"
            hid = llm.prefill_hidden(emb, cache)
            before = cache.pool.clone()
            dec.start(hid[-1], cache)
            dec.run(n)
            ids = dec.tokens(n)
        finally:
            llm.set_decode_weights("bf16")
        _check_untouched(before, cache.pool, [_decoded_rows(cache.page_table, S, n)])
        _check_fp8_sequence(f"{kind} fp8 graph/{path} S={S}", cache.pool, cache.page_table, emb, ids,
                            o32, q32, o16, q16)


# ------------------------------------------------------------------------------------------------
# bf16 unchanged by fp8 mode; public paths
# ------------------------------------------------------------------------------------------------
def _decode(llm, emb, n):
    from vila_b200.model import GraphDecoder
    dec = GraphDecoder(llm, 128)
    cache = dec.cache_for(emb.shape[0] + n)
    hid = llm.prefill_hidden(emb, cache)
    dec.start(hid[-1], cache)
    dec.run(n)
    return dec.tokens(n), cache.pool.clone()


@pytest.mark.parametrize("kind", ["lite-shallow", "tiny"])  # lite-shallow: tied lm_head
def test_bf16_unchanged_by_fp8_mode(cuda, kind):
    model = _model(kind)[0]
    llm = model.llm
    with torch.inference_mode():
        sd_before = {k: v.clone() for k, v in model.state_dict().items()}
        emb = _prompt(llm, 300, seed=7)
        ids_a, pool_a = _decode(llm, emb, 24)
        llm.set_decode_weights("fp8")
        assert llm.decode_weights == "fp8" and llm._decoder is None
        ids_q, _ = _decode(llm, emb, 24)
        sd_fp8 = model.state_dict()
        assert list(sd_fp8) == list(sd_before)  # the fp8 copies are not state
        assert all(torch.equal(sd_fp8[k], v) for k, v in sd_before.items())
        llm.set_decode_weights("bf16")
        assert llm.decode_weights == "bf16" and llm._fp8_weights is None
        ids_b, pool_b = _decode(llm, emb, 24)
        sd_after = model.state_dict()
        assert list(sd_after) == list(sd_before)
        assert all(torch.equal(sd_after[k], v) for k, v in sd_before.items())
    assert ids_a == ids_b and torch.equal(pool_a, pool_b)
    assert len(ids_q) == 24


def test_public_paths_fp8(cuda):
    model = _model("tiny")[0]
    llm = model.llm
    emb = _prompt(llm, 200, seed=11)
    llm.set_decode_weights("fp8")
    try:
        with torch.inference_mode():
            via_generate = llm.generate(inputs_embeds=emb[None], max_new_tokens=20, eos_token_id=None)[0].tolist()
            assert llm.decoder(20).fp8 is llm._fp8_weights
            via_stream = [t for chunk in llm.stream_greedy(emb, max_new_tokens=20, chunk_tokens=8) for t in chunk]
            direct, _ = _decode(llm, emb, 20)
        assert via_generate == via_stream == direct
    finally:
        llm.set_decode_weights("bf16")
