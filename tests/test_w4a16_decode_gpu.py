"""GPU: opt-in W4A16 (4-bit, group-128 scale and zero point) weights in the single-stream decoder.

  * vila_gemv_w4a16 against fp32 math on dequantize_w4_groups' output, at every layer GEMV shape of
    NVILA-8B, NVILA-Lite-3B and the tiny test model with their fusions, a short last row block with the
    argmax, and outlier activations; bit-repeatable, graph replay included; every rejection;
  * GraphDecoder in w4a16 mode, teacher-forced as tests/test_fp8_decode_gpu.py does: the oracle's layer
    weights are the dequantized 4-bit copies and its lm_head the dequantized e4m3 copy;
  * a bf16 -> w4a16 -> fp8 -> bf16 round trip leaves bf16 decoding, the pool and state_dict() unchanged;
  * the public greedy paths follow the mode.
"""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import vila_oracle as O
from tests.helpers import oracle_from_state_dict, report_rel
from tests.test_decode_engines_gpu import _fp32_truth  # noqa: F401  (autouse: the fp32 oracle is really fp32)
from tests.test_decode_engines_gpu import _CONTEXTS, _PATHS, _check_untouched, _config, _decoded_rows, _prompt
from tests.test_fp8_decode_gpu import _check_fp8_sequence, _decode, rb
from tests.test_kernels_gpu import _ops, bf

pytestmark = pytest.mark.gpu


def _quant(w):
    from vila_b200.model.qwen2 import dequantize_w4_groups, quantize_w4_groups
    packed, s, z = quantize_w4_groups(w)
    return packed, s, z, dequantize_w4_groups(packed, s, z)


# ------------------------------------------------------------------------------------------------
# kernel level
# ------------------------------------------------------------------------------------------------
# (name, N, K, fusion): the layer GEMVs of one decode step (lm_head stays e4m3 in this mode)
#   8B:   hidden 3584, inter 18944, qkv (28 + 2*4) * 128
#   Lite: hidden 2048, inter 11008, qkv (16 + 2*2) * 128
#   tiny: hidden 512, inter 1024, qkv (4 + 2*2) * 128: K = 512 is 256 bytes per row
GEMV_CASES = [
    ("8b-qkv", 4608, 3584, "bias+norm"), ("8b-o", 3584, 3584, "residual"),
    ("8b-gate_up", 37888, 3584, "swiglu+norm"), ("8b-down", 3584, 18944, "residual"),
    ("lite-qkv", 2560, 2048, "bias+norm"), ("lite-o", 2048, 2048, "residual"),
    ("lite-gate_up", 22016, 2048, "swiglu+norm"), ("lite-down", 2048, 11008, "residual"),
    ("tiny-qkv", 1024, 512, "bias+norm"), ("tiny-o", 512, 512, "residual"),
    ("tiny-gate_up", 2048, 512, "swiglu+norm"), ("tiny-down", 512, 1024, "residual"),
    ("short-rows", 1003, 3584, "argmax+norm"),  # 63 tiles on 132 SMs, the last one 11 rows
    ("outliers-down", 3584, 18944, "residual+outliers"),
]


def _problem(N, K, seed, outliers=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(K, device="cuda", generator=g)
    if outliers:  # a few activations at +-1e4 (no overflow may follow from any bf16 input)
        idx = torch.randperm(K, device="cuda", generator=g)[:6]
        x[idx] = torch.tensor([1e4, -1e4, 1e4, -1e4, 1e4, -1e4], device="cuda")
    x = bf(x)
    # rows of very different magnitude, and groups within a row of different spread
    w = bf(torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)
           * torch.exp(torch.randn(N, 1, device="cuda", generator=g))
           * torch.exp(0.5 * torch.randn(N, K // 128, device="cuda", generator=g)).repeat_interleave(128, 1))
    b = bf(torch.randn(N, device="cuda", generator=g))
    r = bf(torch.randn(N, device="cuda", generator=g))
    nw = bf(1 + 0.1 * torch.randn(K, device="cuda", generator=g))
    return x, w, b, r, nw


def _launch(ops, fusion, x, q, s, z, b, r, nw, key=None):
    kw = dict(w_scale=s, w_zero=z, static_w=True)
    if fusion == "bias+norm":
        return ops.gemv(x, q, bias=b, norm_w=nw, norm_eps=1e-6, **kw)
    if fusion.startswith("residual"):
        return ops.gemv(x, q, residual=r, **kw)
    if fusion == "swiglu+norm":
        return ops.gemv(x, q, norm_w=nw, norm_eps=1e-6, swiglu=True, **kw)
    return ops.gemv(x, q, norm_w=nw, norm_eps=1e-6, argmax_key=key, **kw)


@pytest.mark.parametrize("name,N,K,fusion", GEMV_CASES, ids=[c[0] for c in GEMV_CASES])
def test_gemv_w4a16(cuda, name, N, K, fusion):
    ops = _ops()
    x, w, b, r, nw = _problem(N, K, seed=N + K, outliers="outliers" in fusion)
    q, s, z, deq = _quant(w)
    key = torch.zeros(1, dtype=torch.int64, device=cuda) if fusion == "argmax+norm" else None
    out = _launch(ops, fusion, x, q, s, z, b, r, nw, key)
    xn = O.rms_norm(x[None], nw, 1e-6)[0].float() if "norm" in fusion else x.float()
    acc = deq @ xn
    if fusion == "bias+norm":
        ref, tol = rb(acc + b.float()), 2 ** -7
    elif fusion.startswith("residual"):
        ref, tol = rb(rb(acc) + r.float()), 2 ** -7
    elif fusion == "swiglu+norm":
        ref, tol = rb(rb(F.silu(rb(acc[0::2]))) * rb(acc[1::2])), 2 ** -6
    else:
        ref, tol = acc, 2 ** -7
    assert bool(torch.isfinite(out.float()).all())
    report_rel(f"gemv_w4a16 {name} {fusion}", out, ref, tol)
    if key is not None:  # the fused greedy arg-max: a best id of the fp32 reference, up to 3 bf16 ulps
        tok = 0xFFFFFFFF - int(key.item() & 0xFFFFFFFF)
        margin = 3 * 2 ** -8 * acc.abs().max().item()
        assert 0 <= tok < N and acc[tok].item() >= acc.max().item() - margin, (tok, acc[tok].item(), acc.max().item())
        assert tok == int(torch.argmax(out.float()))  # the kernel's own logits decide
    # repeatable, and a captured graph replays the same bits
    key2 = torch.zeros_like(key) if key is not None else None
    again = _launch(ops, fusion, x, q, s, z, b, r, nw, key2)
    assert torch.equal(out, again) and (key is None or torch.equal(key, key2))
    key3 = torch.zeros_like(key) if key is not None else None
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_out = _launch(ops, fusion, x, q, s, z, b, r, nw, key3)
    if key3 is not None:
        key3.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, g_out) and (key is None or torch.equal(key, key3))


def test_gemv_w4a16_rejects(cuda):
    from vila_b200 import _lib
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(5)
    x = bf(torch.randn(3584, device=cuda, generator=g))
    q, s, z, _ = _quant(bf(torch.randn(64, 3584, device=cuda, generator=g)))
    y = torch.full((64,), 7.0, dtype=torch.bfloat16, device=cuda)
    with pytest.raises(ValueError):
        ops.gemv(x, q, w_scale=s, w_zero=z, variant=1, out=y)  # no register-staged form
    with pytest.raises(ValueError):
        ops.gemv(x, q, w_scale=s, out=y)  # zero points are required
    with pytest.raises(ValueError):
        ops.gemv(x, q, w_zero=z, out=y)  # scales are required
    with pytest.raises(ValueError):
        ops.gemv(x, q, w_scale=s[:32], w_zero=z[:32], out=y)  # packed rows do not match
    with pytest.raises(ValueError):
        ops.gemv(x, q, w_scale=s[:, :14], w_zero=z, out=y)  # mis-shaped scales
    with pytest.raises(RuntimeError):
        ops.gemv(x, q, w_scale=s.float(), w_zero=z, out=y)  # scales are bf16
    bf16_w = bf(torch.randn(64, 3584, device=cuda, generator=g))
    with pytest.raises(ValueError):
        ops.gemv(x, bf16_w, w_zero=z, out=y)  # zero points only go with packed weights

    def raw(K, flags=0, scales=True):  # the C entry point, past ops.gemv's checks
        p = _lib.GemvParams()
        p.x, p.w, p.y = x.data_ptr(), q.data_ptr(), y.data_ptr()
        p.bias = p.norm_w = p.residual = p.argmax_key = None
        p.norm_eps, p.N, p.K, p.flags = 1e-6, 64, K, flags
        lib = _lib.load()
        rc = lib.vila_gemv_w4a16(C.byref(p), s.data_ptr() if scales else None, z.data_ptr() if scales else None,
                                 torch.cuda.current_stream().cuda_stream)
        return rc, lib.vila_last_error()

    rc, err = raw(3584 - 64)  # a multiple of 16, not of 128
    assert rc != 0 and b"K % 128" in err
    rc, err = raw(3584, flags=4)
    assert rc != 0 and b"register-staged" in err
    rc, err = raw(3584, scales=False)
    assert rc != 0 and b"zero points" in err
    torch.cuda.synchronize()
    assert bool((y == 7.0).all())  # nothing was launched


# ------------------------------------------------------------------------------------------------
# GraphDecoder in w4a16 mode, teacher-forced
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
    linear weights are dequantize_w4_groups of the model's own 4-bit copies and whose lm_head is its
    dequantized e4m3 copy"""
    if kind not in _MODEL:
        _release()
        from vila_b200.model import LlavaLlamaModel
        from vila_b200.model.qwen2 import dequantize_w4_groups
        cfg = _config(kind)
        model = LlavaLlamaModel(cfg, device="cuda").init_random(23, device_rng=kind != "tiny")
        sd = {k: v for k, v in model.state_dict().items() if k.startswith("llm.")}
        llm = model.llm
        llm.set_decode_weights("w4a16")
        lc = cfg.llm_cfg
        Hq, Hkv, D = lc.num_attention_heads, lc.num_key_value_heads, lc.head_dim
        f = llm._w4_weights
        dq = {"llm.lm_head.weight": f.lm_head[0].float() * f.lm_head[1][:, None]}
        for i, fl in enumerate(f.layers):
            pre = f"llm.model.layers.{i}."
            qkv = dequantize_w4_groups(*fl.qkv)
            dq[pre + "self_attn.q_proj.weight"] = qkv[:Hq * D]
            dq[pre + "self_attn.k_proj.weight"] = qkv[Hq * D:(Hq + Hkv) * D]
            dq[pre + "self_attn.v_proj.weight"] = qkv[(Hq + Hkv) * D:]
            dq[pre + "self_attn.o_proj.weight"] = dequantize_w4_groups(*fl.o)
            gu = dequantize_w4_groups(*fl.gu)
            dq[pre + "mlp.gate_proj.weight"], dq[pre + "mlp.up_proj.weight"] = gu[0::2], gu[1::2]
            dq[pre + "mlp.down_proj.weight"] = dequantize_w4_groups(*fl.down)
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


def _w4_cases():
    out = []
    for kind in ("tiny", "8b-shallow", "lite-shallow"):
        n_ctx = 4 if kind == "tiny" else 3
        out += [(kind, path, S, n) for (S, n), path in zip(_CONTEXTS[:n_ctx], _PATHS)]
    return out


W4_CASES = _w4_cases()


@pytest.mark.parametrize("kind,path,S,n", W4_CASES, ids=[f"{k}-{p}-S{S}" for k, p, S, _ in W4_CASES])
def test_graph_decoder_w4a16_teacher_forced(cuda, kind, path, S, n):
    from vila_b200.model import GraphDecoder
    model, o32, o16, q32, q16 = _model(kind)
    llm = model.llm
    with torch.inference_mode():
        emb = _prompt(llm, S, seed=S)
        llm.set_decode_weights("w4a16")
        try:
            dec = GraphDecoder(llm, 128)
            assert dec.w4 is not None and dec.fp8 is None
            cache = dec.cache_for(S + n)
            got_path = "split" if dec.split_tokens else "simt" if dec.num_splits else "head"
            assert got_path == path, f"w4a16 graph decoder at {S + n} tokens runs {got_path}, the case is for {path}"
            hid = llm.prefill_hidden(emb, cache)
            before = cache.pool.clone()
            dec.start(hid[-1], cache)
            dec.run(n)
            ids = dec.tokens(n)
        finally:
            llm.set_decode_weights("bf16")
        _check_untouched(before, cache.pool, [_decoded_rows(cache.page_table, S, n)])
        _check_fp8_sequence(f"{kind} w4a16 graph/{path} S={S}", cache.pool, cache.page_table, emb, ids,
                            o32, q32, o16, q16)


# ------------------------------------------------------------------------------------------------
# bf16 unchanged by the quantized modes; public paths
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["lite-shallow", "tiny"])  # lite-shallow: tied lm_head
def test_bf16_unchanged_by_w4a16_and_fp8_modes(cuda, kind):
    model = _model(kind)[0]
    llm = model.llm
    with torch.inference_mode():
        sd_before = {k: v.clone() for k, v in model.state_dict().items()}
        emb = _prompt(llm, 300, seed=7)
        ids_a, pool_a = _decode(llm, emb, 24)
        llm.set_decode_weights("w4a16")
        assert llm.decode_weights == "w4a16" and llm._decoder is None
        ids_w4, _ = _decode(llm, emb, 24)
        sd_w4 = model.state_dict()
        assert list(sd_w4) == list(sd_before)  # the 4-bit copies are not state
        assert all(torch.equal(sd_w4[k], v) for k, v in sd_before.items())
        llm.set_decode_weights("fp8")
        assert llm._w4_weights is None and llm._fp8_weights is not None
        ids_fp8, _ = _decode(llm, emb, 24)
        llm.set_decode_weights("bf16")
        assert llm.decode_weights == "bf16" and llm._fp8_weights is None and llm._w4_weights is None
        ids_b, pool_b = _decode(llm, emb, 24)
        sd_after = model.state_dict()
        assert list(sd_after) == list(sd_before)
        assert all(torch.equal(sd_after[k], v) for k, v in sd_before.items())
    assert ids_a == ids_b and torch.equal(pool_a, pool_b)
    assert len(ids_w4) == 24 and len(ids_fp8) == 24


def test_public_paths_w4a16(cuda):
    model = _model("tiny")[0]
    llm = model.llm
    emb = _prompt(llm, 200, seed=11)
    llm.set_decode_weights("w4a16")
    try:
        with torch.inference_mode():
            via_generate = llm.generate(inputs_embeds=emb[None], max_new_tokens=20, eos_token_id=None)[0].tolist()
            assert llm.decoder(20).w4 is llm._w4_weights
            via_stream = [t for chunk in llm.stream_greedy(emb, max_new_tokens=20, chunk_tokens=8) for t in chunk]
            direct, _ = _decode(llm, emb, 20)
        assert via_generate == via_stream == direct
    finally:
        llm.set_decode_weights("bf16")
