"""GPU: the opt-in FP8 (e4m3) KV cache of the continuous-batching engine.

  * vila_kv_quantize_fp8: codes and scales bit-identical to quantize_kv_e4m3 through randomly permuted pages;
    every other pool byte untouched;
  * vila_decode_attention_fp8_batch at (Hq, Hkv) = (28, 4), (16, 2), (4, 2), positions from 0 to 69,631 and
    idle slots: the appended row's codes and scale equal the rule applied to the rotated bf16 k / v of the bf16
    kernels on the same problem (so RoPE is checked bit for bit), the output is close to fp32 attention over the
    dequantised pool, and each slot's output and appended bytes are bit-identical alone, beside neighbours with
    random or +-1e4 outlier data, at every ladder entry and under graph replay;
  * serving.BatchedDecoder(kv_cache="fp8") on the scenario of test_decode_engines_gpu._run_batched, with bf16,
    w4a16 and (tiny model) fp8 weights, against an fp32 oracle teacher-forced on the engine's ids and on its
    dequantised K/V, the new token's own k / v rounded by the same rule; every prompt row the admission wrote is
    checked against the oracle's own prompt past, every decoded row against the oracle's k / v;
  * generate_batch(kv_cache="fp8") gives each request the same ids alone, with 3 slots and with 20; a decoder of
    the other KV format is refused; a bf16-KV decoder is unchanged by an fp8-KV decoder on the same LLM.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import vila_oracle as O
from tests import test_fp8_decode_gpu as T8
from tests import test_w4a16_decode_gpu as T4
from tests.helpers import _record, report_rel
from tests.test_decode_engines_gpu import _fp32_truth  # noqa: F401  (autouse: the fp32 oracle is really fp32)
from tests.test_decode_engines_gpu import _check_untouched, _decoded_rows, _prompt
from tests.test_kernels_gpu import _ops, bf, ref_attention

pytestmark = pytest.mark.gpu

PAGE, D = 128, 128


def _rule(x):
    from vila_b200.model.qwen2 import quantize_kv_e4m3
    return quantize_kv_e4m3(x)


def _deq(codes, scale):
    return codes.float() * scale[..., None]


def _u8(t):
    return t.view(torch.uint8)


# ------------------------------------------------------------------------------------------------
# vila_kv_quantize_fp8
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Hq,Hkv", [(28, 4), (16, 2), (4, 2)])
def test_kv_quantize_fp8(cuda, Hq, Hkv):
    ops = _ops()
    L, S, ps, P = 3, 300, 4, 9
    g = torch.Generator(device="cuda").manual_seed(Hq)
    src = bf(torch.randn(L, 2, ps, PAGE, Hkv, D, device=cuda, generator=g))
    src[0, 0, 0, 5] = 0                        # all-zero rows
    src[1, 1, 1, 7, 0, 3] = 1e4                # an outlier row
    src[2, 0, 0, 9, -1] *= 1e-6                # a row of subnormal codes
    row = torch.randperm(P, device=cuda, generator=g)[:ps].to(torch.int32)
    sentinel = torch.randint(0, 0x7E, (L, 2, P, PAGE, Hkv, D), device=cuda, dtype=torch.uint8, generator=g)
    dst = sentinel.clone().view(torch.float8_e4m3fn)
    sc0 = torch.full((L, 2, P, PAGE, Hkv), 7.0, device=cuda)
    sc = sc0.clone()
    ops.kv_quantize_fp8(src, dst, sc, row, S)
    torch.cuda.synchronize()
    t = torch.arange(S, device=cuda)
    x = src.view(L, 2, ps * PAGE, Hkv, D)[:, :, :S]
    codes, scales = _rule(x)
    pages, rows = row[t // PAGE].long(), t % PAGE
    assert torch.equal(_u8(dst[:, :, pages, rows]), _u8(codes))
    assert torch.equal(sc[:, :, pages, rows], scales)
    expect, expect_sc = sentinel.clone(), sc0.clone()
    expect[:, :, pages, rows] = _u8(codes)
    expect_sc[:, :, pages, rows] = scales
    assert torch.equal(_u8(dst), expect) and torch.equal(sc, expect_sc)  # rows >= S and other pages untouched


# ------------------------------------------------------------------------------------------------
# vila_decode_attention_fp8_batch
# ------------------------------------------------------------------------------------------------
POSITIONS = [-1, 0, 1, 127, 128, 1023, 1024, 2047, -1, 4095, 16469, 69631]


def _fp8_problem(Hq, Hkv, positions, pt_width, seed):
    """one shared e4m3 pool (codes from the rule on random bf16 rows) with randomly permuted pages"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    need = [(p + 1 + PAGE - 1) // PAGE if p >= 0 else 0 for p in positions]
    n_pages = sum(need) + 16
    perm = torch.randperm(n_pages, device="cuda", generator=g).to(torch.int32)
    pt = torch.randint(0, n_pages, (len(positions), pt_width), device="cuda", generator=g, dtype=torch.int32)
    o = 0
    for b, k in enumerate(need):
        pt[b, :k] = perm[o:o + k]
        o += k
    pools = []
    for _ in range(2):
        x = torch.randn(n_pages, PAGE, Hkv, D, device="cuda", generator=g)
        pools.append(_rule(bf(x)))
    qkv = bf(torch.randn(len(positions), (Hq + 2 * Hkv) * D + 64, device="cuda", generator=g))
    return pt, pools, qkv


def _rotated_new_row(ops, qkv_row, p, Hq, Hkv, inv):
    """the rotated bf16 k and the v of the new token, from the bf16 kernels on a bf16 copy of the problem"""
    pages = (p + 1 + PAGE - 1) // PAGE
    kp = torch.zeros(pages, PAGE, Hkv, D, dtype=torch.bfloat16, device="cuda")
    vp = torch.zeros_like(kp)
    pt = torch.arange(pages, dtype=torch.int32, device="cuda")[None]
    pos = torch.tensor([p], dtype=torch.int32, device="cuda")
    qkv = qkv_row[None].clone()
    out = torch.zeros(1, Hq * D, dtype=torch.bfloat16, device="cuda")
    if p <= 4095:
        ops.decode_attention_batch(qkv, pos, kp, vp, pt, out, inv, Hq, Hkv, D, D ** -0.5)
    else:
        n = (p + 1 + 1023) // 1024
        ops.decode_attention_split_batch(qkv, pos, kp, vp, pt, out,
                                         torch.zeros(n * Hq * D, device="cuda"), torch.zeros(n * Hq, device="cuda"),
                                         torch.zeros(Hkv, dtype=torch.int32, device="cuda"), inv, Hq, Hkv, D, n, 1024,
                                         D ** -0.5)
    return kp[p // PAGE, p % PAGE], vp[p // PAGE, p % PAGE]


# NVILA-8B, Lite-3B and the tiny model, and G = 13 / 16, which keep fewer V words in flight
@pytest.mark.parametrize("Hq,Hkv", [(28, 4), (16, 2), (4, 2), (13, 1), (32, 2)])
def test_decode_attention_fp8_batch(cuda, Hq, Hkv):
    from vila_b200 import serving
    ops = _ops()
    split = serving.FP8_SPLIT_TOKENS
    N = (Hq + 2 * Hkv) * D
    positions = POSITIONS
    B = len(positions)
    n_max = serving.fp8_attention_config(serving.MAX_SLOT_TOKENS)
    pt, ((k0, ks0), (v0, vs0)), qkv0 = _fp8_problem(Hq, Hkv, positions, serving.MAX_SLOT_TOKENS // PAGE,
                                                    seed=100 * Hq + Hkv)
    inv = O.rope_inv_freq(D, 1e6).to(cuda)
    ws = torch.zeros(B * Hq * n_max * (D + 2), device=cuda)
    counters = torch.zeros(B * Hkv, dtype=torch.int32, device=cuda)
    sentinel = bf(torch.full((B, Hq * D + 32), 7.0, device=cuda))

    def launch(qkv, pos, pools, pt_, out, n):
        (kp, ks), (vp, vs) = pools
        ops.decode_attention_fp8_batch(qkv[:, :N], pos, kp, vp, ks, vs, pt_, out[:, :Hq * D], ws, counters, inv,
                                       Hq, Hkv, n, split, D ** -0.5)

    def fresh(*ts):
        return [t.clone() for t in ts]

    def run(pos_list, n, pools=None, qkv=None, rows=None):
        """-> (out, pools after) for the slots `rows` (default all)"""
        rows = list(range(B)) if rows is None else rows
        pools = fresh(k0, ks0, v0, vs0) if pools is None else pools
        kp, ks, vp, vs = pools
        out = sentinel[rows].clone()
        q = (qkv0 if qkv is None else qkv)[rows].clone()
        pos = torch.tensor([pos_list[r] for r in rows], dtype=torch.int32, device=cuda)
        launch(q, pos, ((kp, ks), (vp, vs)), pt[rows].contiguous(), out, n)
        torch.cuda.synchronize()
        assert torch.equal(q, (qkv0 if qkv is None else qkv)[rows])  # q / k are rotated on chip only
        return out, (kp, ks, vp, vs)

    out, (kp, ks, vp, vs) = run(positions, n_max)
    assert torch.equal(out[:, Hq * D:], sentinel[:, Hq * D:])
    touched = [_u8(k0).clone(), ks0.clone(), _u8(v0).clone(), vs0.clone()]
    for b, p in enumerate(positions):
        if p < 0:
            assert torch.equal(out[b], sentinel[b])
            continue
        page, row = int(pt[b, p // PAGE]), p % PAGE
        kr, vn = _rotated_new_row(ops, qkv0[b, :N], p, Hq, Hkv, inv)
        (kc, kscale), (vc, vscale) = _rule(kr), _rule(vn)
        assert torch.equal(_u8(kp[page, row]), _u8(kc)) and torch.equal(ks[page, row], kscale)
        assert torch.equal(_u8(vp[page, row]), _u8(vc)) and torch.equal(vs[page, row], vscale)
        for i, a in enumerate((kp, ks, vp, vs)):
            touched[i][page, row] = _u8(a[page, row]) if a.dtype == torch.float8_e4m3fn else a[page, row]
        t = torch.arange(p, device=cuda)
        prow = pt[b, t // PAGE].long(), t % PAGE
        k_all = torch.cat([_deq(k0[prow], ks0[prow]), _deq(kc, kscale)[None]], 0)
        v_all = torch.cat([_deq(v0[prow], vs0[prow]), _deq(vc, vscale)[None]], 0)
        q = qkv0[b, :Hq * D].view(1, Hq, D).transpose(0, 1)
        cos, sin = O.rope_cos_sin(torch.tensor([p]), D, 1e6, torch.bfloat16)
        qr, _ = O.apply_rope(q, q[:Hkv], cos.to(cuda), sin.to(cuda))
        ref = ref_attention(qr.transpose(0, 1)[None].float(), k_all[None], v_all[None], True, D ** -0.5)[0, 0]
        report_rel(f"decode_attention_fp8_batch Hq={Hq} Hkv={Hkv} ctx={p}", out[b, :Hq * D].view(Hq, D), ref, 1.5e-2)
    assert torch.equal(_u8(kp), touched[0]) and torch.equal(ks, touched[1])    # every other pool byte unchanged
    assert torch.equal(_u8(vp), touched[2]) and torch.equal(vs, touched[3])

    def same_slot(b, got_out, got_pools, b_got=None):
        b_got = b if b_got is None else b_got
        p = positions[b]
        assert torch.equal(got_out[b_got], out[b]), f"slot {b} (ctx {p}): output differs"
        if p >= 0:
            page, row = int(pt[b, p // PAGE]), p % PAGE
            for a, ref_ in zip(got_pools, (kp, ks, vp, vs)):
                assert torch.equal(a[page, row].view(torch.uint8), ref_[page, row].view(torch.uint8)), \
                    f"slot {b} (ctx {p}): appended bytes differ"

    # alone, with the smallest ladder entry that covers it
    for b, p in enumerate(positions):
        n = serving.fp8_attention_config(p + 1) if p >= 0 else 1
        o1, pools1 = run(positions, n, rows=[b])
        same_slot(b, o1, pools1, 0)
    # every ladder entry, with the slots it cannot cover idle
    for n_tok in serving.FP8_LADDER_TOKENS:
        n = serving.fp8_attention_config(n_tok)
        short = [p if p < n * split else -1 for p in positions]
        o_n, pools_n = run(short, n)
        for b, p in enumerate(short):
            if p >= 0:
                same_slot(b, o_n, pools_n)
    # neighbours holding random or +-1e4 outlier data (pool rows and qkv rows of the other slots)
    g = torch.Generator(device="cuda").manual_seed(7)
    for parity in (0, 1):
        for scale in (1.0, 1e4):
            pools = fresh(k0, ks0, v0, vs0)
            qkv = qkv0.clone()
            for b, p in enumerate(positions):
                if b % 2 == parity or p < 0:
                    continue
                pages = pt[b, :(p + 1 + PAGE - 1) // PAGE].long()
                for c, s in ((0, 1), (2, 3)):
                    x = bf(torch.randn(len(pages), PAGE, Hkv, D, device=cuda, generator=g) * scale)
                    codes, sc = _rule(x)
                    pools[c][pages], pools[s][pages] = codes, sc
                qkv[b] = bf(torch.randn(qkv.shape[1], device=cuda, generator=g) * scale)
            o_nb, pools_nb = run(positions, n_max, pools=pools, qkv=qkv)
            for b in range(B):
                if b % 2 == parity:
                    same_slot(b, o_nb, pools_nb)

    # a captured graph replays the eager bits
    pools = fresh(k0, ks0, v0, vs0)
    pos_g = torch.tensor(positions, dtype=torch.int32, device=cuda)
    qg, og = qkv0.clone(), sentinel.clone()
    launch(qg, pos_g, ((pools[0], pools[1]), (pools[2], pools[3])), pt, og, n_max)  # warm-up
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        launch(qg, pos_g, ((pools[0], pools[1]), (pools[2], pools[3])), pt, og, n_max)
    for _ in range(2):
        for a, b0 in zip(pools, (k0, ks0, v0, vs0)):
            a.copy_(b0)
        og.copy_(sentinel)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(og, out)
        for a, ref_ in zip(pools, (kp, ks, vp, vs)):
            assert torch.equal(a.view(torch.uint8), ref_.view(torch.uint8))
    assert int(counters.abs().sum()) == 0  # the counters cleaned up after themselves


def test_decode_attention_fp8_batch_rejections(cuda):
    """bad arguments are errors through the raw entry point, and nothing is written"""
    import ctypes as C
    from vila_b200 import _lib
    from vila_b200._lib import DecodeAttnFp8Params
    lib = _lib.load()
    Hq, Hkv, B = 4, 2, 2
    pt, ((kp, ks), (vp, vs)), qkv = _fp8_problem(Hq, Hkv, [5, 9], 4, seed=3)
    pos = torch.tensor([5, 9], dtype=torch.int32, device=cuda)
    out = bf(torch.full((B, Hq * D), 7.0, device=cuda))
    ws = torch.zeros(B * Hq * 4 * 130, device=cuda)
    cnt = torch.zeros(B * Hkv, dtype=torch.int32, device=cuda)
    inv = O.rope_inv_freq(D, 1e6).to(cuda)
    before = [_u8(kp).clone(), _u8(vp).clone(), ks.clone(), vs.clone()]

    def raw(**kw):
        p = DecodeAttnFp8Params()
        p.qkv, p.position, p.k_pool, p.v_pool = qkv.data_ptr(), pos.data_ptr(), kp.data_ptr(), vp.data_ptr()
        p.k_scale, p.v_scale, p.page_table, p.out = ks.data_ptr(), vs.data_ptr(), pt.data_ptr(), out.data_ptr()
        p.ws, p.counters, p.inv_freq = ws.data_ptr(), cnt.data_ptr(), inv.data_ptr()
        p.Hq, p.Hkv, p.D, p.batch = Hq, Hkv, D, B
        p.qkv_stride, p.out_stride, p.pt_stride = qkv.stride(0), out.stride(0), pt.stride(0)
        p.num_splits, p.split_tokens, p.scale = 4, 512, D ** -0.5
        for k, v in kw.items():
            setattr(p, k, v)
        rc = lib.vila_decode_attention_fp8_batch(C.byref(p), torch.cuda.current_stream().cuda_stream)
        return rc, lib.vila_last_error()

    for kw, msg in (({"D": 64}, b"head_dim"), ({"Hq": 34}, b"16 query heads"), ({"k_pool": None}, b"pointer"),
                    ({"k_pool": kp.data_ptr() + 4}, b"misaligned"), ({"split_tokens": 200}, b"split"),
                    ({"Hq": 5}, b"multiple")):
        rc, err = raw(**kw)
        assert rc != 0 and msg in err, (kw, err)
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())
    after = [_u8(kp), _u8(vp), ks, vs]
    assert all(torch.equal(a, b) for a, b in zip(before, after))


# ------------------------------------------------------------------------------------------------
# engine level, teacher-forced against an oracle on e4m3-rounded K/V
# ------------------------------------------------------------------------------------------------
def _rq(x):
    """x rounded through the KV format (quantize_kv_e4m3, then dequantised), in x's dtype"""
    c, s = _rule(x)
    return _deq(c, s).to(x.dtype)


def _engine_kv(dec, slot, T):
    """per layer (k, v) [Hkv, T, D] fp32: the slot's dequantised rows [0, T) in the engine's pool"""
    pages, rows = _decoded_rows(dec.page_tables[slot], 0, T + 1)
    return [tuple(_deq(dec.pool[li, j][pages, rows], dec.pool_scale[li, j][pages, rows]).transpose(0, 1)
                  for j in range(2)) for li in range(dec.pool.shape[0])]


def _fp8_kv_teacher_forced(base, quant, emb, ids, engine_kv):
    """Teacher forcing on ids and on the engine's K/V: the prompt on the bf16 weights, its last position scored by
    the mode's lm_head; then each of ids[:-1] on the mode's weights, attending over the engine's dequantised rows
    before it and its own k / v rounded by the KV format's rule (the new row as later steps see it).
    -> (logits [len(ids), V] fp32, per layer (k, v) [Hkv, len(ids) - 1, D] of the decoded positions, unrounded,
    and the prompt's own per layer (k, v) [Hkv, S, D] from qwen2_forward's past, unrounded)"""
    p, cfg = quant.llm, quant.lcfg
    H, Hk = cfg.num_attention_heads, cfg.num_key_value_heads
    table = p["model.embed_tokens.weight"]
    prompt_w = dict(base.llm)
    prompt_w["lm_head.weight"] = p["lm_head.weight"]
    lg0, past = O.qwen2_forward(emb.to(table.dtype), prompt_w, cfg, last_only=True)
    S = emb.shape[0]
    logits, raw = [lg0], [([], []) for _ in range(cfg.num_hidden_layers)]
    for i, t in enumerate(ids[:-1]):
        x = table[t][None]
        cos, sin = O.rope_cos_sin(torch.tensor([S + i], device=x.device), D, cfg.rope_theta, x.dtype)
        for li in range(cfg.num_hidden_layers):
            pre = f"model.layers.{li}."
            a_ = pre + "self_attn."
            h = O.rms_norm(x, p[pre + "input_layernorm.weight"], cfg.rms_norm_eps)
            q = F.linear(h, p[a_ + "q_proj.weight"], p[a_ + "q_proj.bias"]).view(1, H, D).transpose(0, 1)
            k = F.linear(h, p[a_ + "k_proj.weight"], p[a_ + "k_proj.bias"]).view(1, Hk, D).transpose(0, 1)
            v = F.linear(h, p[a_ + "v_proj.weight"], p[a_ + "v_proj.bias"]).view(1, Hk, D).transpose(0, 1)
            q, k = O.apply_rope(q, k, cos, sin)
            raw[li][0].append(k)
            raw[li][1].append(v)
            kk = torch.cat([engine_kv[li][0][:, :S + i].to(x.dtype), _rq(k)], dim=1).repeat_interleave(H // Hk, 0)
            vv = torch.cat([engine_kv[li][1][:, :S + i].to(x.dtype), _rq(v)], dim=1).repeat_interleave(H // Hk, 0)
            att = F.softmax(torch.matmul(q, kk.transpose(1, 2)) / math.sqrt(D), dim=-1, dtype=torch.float32)
            a = torch.matmul(att.to(q.dtype), vv).transpose(0, 1).reshape(1, H * D)
            x = x + F.linear(a, p[a_ + "o_proj.weight"])
            h = O.rms_norm(x, p[pre + "post_attention_layernorm.weight"], cfg.rms_norm_eps)
            x = x + O.qwen2_mlp(h, p, pre + "mlp.")
        logits.append(F.linear(O.rms_norm(x, p["model.norm.weight"], cfg.rms_norm_eps), p["lm_head.weight"]))
    kv = [tuple(torch.cat(r, dim=1) for r in layer) for layer in raw]
    return torch.cat(logits).float(), kv, past


def _check_rows(name, codes, sc, t32, t16):
    """dequantised engine rows [n, Hkv, D] against the oracle's unrounded rows: |got - t32| <= half an e4m3 ulp at
    the row's scale (+ two fp32 roundings of the scale) + the bf16 engine's check_close bound (1.6 x the bf16
    oracle's error + 1e-3 of the largest value)"""
    got = _deq(codes, sc)
    a = codes.float().abs()
    half_ulp = torch.exp2(torch.floor(torch.log2(a.clamp(min=2.0 ** -6))) - 4)
    q_bound = half_ulp * sc[..., None] + 2.0 ** -21 * sc[..., None] * 448
    scale = t32.abs().max().item()
    ref_err = (t16 - t32).abs().max().item()
    bf_bound = 1.6 * ref_err + 1e-3 * scale
    excess = ((got - t32).abs() - q_bound).max().item()
    _record({"name": name, "scale": round(scale, 5), "err": (got - t32).abs().max().item(),
             "excess_over_quant": excess, "ref_err": ref_err, "bound": bf_bound, "ok": bool(excess <= bf_bound)})
    assert excess <= bf_bound, f"{name}: err beyond the quantisation bound {excess:.4e} > {bf_bound:.4e}"


def _check_fp8_kv_sequence(name, dec, slot, emb, ids, o32, q32, o16, q16):
    """ids: greedy choices of the fp32 oracle within 3 bf16 ulps; the dequantised K/V in every layer (_check_rows)
    of every prompt position, against the oracle's own prompt past (so admission's prefill and conversion are
    checked independently of the engine's pool), and of every decoded position"""
    S = emb.shape[0]
    engine_kv = _engine_kv(dec, slot, S + len(ids) - 1)
    with torch.no_grad():
        truth, kv32, past32 = _fp8_kv_teacher_forced(o32, q32, emb, ids, engine_kv)
        _, kv16, past16 = _fp8_kv_teacher_forced(o16, q16, emb, ids, engine_kv)
    margin = 3 * 2 ** -8 * truth.abs().max().item()
    for i, t in enumerate(ids):
        best = truth[i].max().item()
        assert truth[i, t].item() >= best - margin, \
            f"{name}: step {i}: id {t} scores {truth[i, t].item():.4f}, the oracle's best {best:.4f} (margin {margin:.4f})"
    prompt_rows = _decoded_rows(dec.page_tables[slot], 0, S + 1)
    decoded_rows = _decoded_rows(dec.page_tables[slot], S, len(ids))
    for li in range(o32.lcfg.num_hidden_layers):
        for j, kvn in enumerate("KV"):
            for what, (pages, rows), t32, t16 in (("prompt", prompt_rows, past32[li][j], past16[li][j]),
                                                 ("decoded", decoded_rows, kv32[li][j], kv16[li][j])):
                _check_rows(f"{name} layer {li} {kvn} {what}", dec.pool[li, j][pages, rows],
                            dec.pool_scale[li, j][pages, rows], t32.transpose(0, 1).float(),
                            t16.transpose(0, 1).float())


# fp8 decode weights with the fp8 KV cache on the tiny model: the sixth weight x KV combination
ENGINE_CASES = [(w, kind) for kind in ("tiny", "8b-shallow", "lite-shallow") for w in ("bf16", "w4a16")]
ENGINE_CASES.insert(2, ("fp8", "tiny"))


@pytest.mark.parametrize("weights,kind", ENGINE_CASES, ids=[f"{k}-{w}" for w, k in ENGINE_CASES])
def test_batched_decoder_fp8_kv_teacher_forced(cuda, weights, kind):
    """4096-token slots: slot 0 S=1015, slot 1 S=2040 (its ladder entry grows mid-run), slot 2 idle, slot 3
    S=3065; then slot 0 is released, a 500-token prompt reuses its pages and all slots run again"""
    from vila_b200 import serving
    # (prompt oracle, decode oracle) in fp32 and bf16: the prompt runs the bf16 weights in every mode
    model, o32, o16, q32, q16 = (T8 if weights == "fp8" else T4)._model(kind)
    oracles = (o32, o32, o16, o16) if weights == "bf16" else (o32, q32, o16, q16)
    llm = model.llm
    n = 16
    with torch.inference_mode():
        llm.set_decode_weights(weights)
        try:
            dec = serving.BatchedDecoder(llm, slots=4, max_tokens_per_slot=4096, max_new=64, kv_cache="fp8")
            assert dec.kv_cache == "fp8" and dec.decode_weights == weights
            assert dec.configs == [serving.fp8_attention_config(2048), serving.fp8_attention_config(8192)]
            dec.capture()
            lens = {0: 1015, 1: 2040, 3: 3065}
            prompts = {s: _prompt(llm, S, seed=S) for s, S in lens.items()}
            for s in lens:
                dec.admit(s, prompts[s])
            before, before_sc = _u8(dec.pool).clone(), dec.pool_scale.clone()
            dec.run(n - 1)
            assert dec.config == serving.fp8_attention_config(8192)
            assert dec.generated(2) == [] and int(dec.positions[2]) == -1
            decoded = [_decoded_rows(dec.page_tables[s], S, n) for s, S in lens.items()]
            _check_untouched(before, _u8(dec.pool), decoded)
            _check_untouched(before_sc, dec.pool_scale, decoded)
            _check_fp8_kv_sequence(f"{kind} {weights} fp8-KV slot 0 S=1015", dec, 0, prompts[0], dec.generated(0),
                                   *oracles)
            freed = list(dec.slot_pages[0])
            dec.release(0)
            lens[0], prompts[0] = 500, _prompt(llm, 500, seed=500)
            dec.admit(0, prompts[0])
            assert set(dec.slot_pages[0]) <= set(freed)
            before, before_sc = _u8(dec.pool).clone(), dec.pool_scale.clone()
            dec.run(n - 1)
            decoded = [_decoded_rows(dec.page_tables[0], 500, n)]
            for s in (1, 3):
                pages, rows = _decoded_rows(dec.page_tables[s], lens[s], 2 * n - 1)
                decoded.append((pages[n - 1:], rows[n - 1:]))
            _check_untouched(before, _u8(dec.pool), decoded)
            _check_untouched(before_sc, dec.pool_scale, decoded)
            for s in (0, 1, 3):
                ids = dec.generated(s)
                assert len(ids) == (n if s == 0 else 2 * n - 1)
                _check_fp8_kv_sequence(f"{kind} {weights} fp8-KV slot {s} S={lens[s]}", dec, s, prompts[s], ids,
                                       *oracles)
        finally:
            llm.set_decode_weights("bf16")
            if weights == "fp8":
                T8._release()


def test_generate_batch_fp8_kv(cuda):
    """same ids alone, with 3 slots and with 20; a decoder of the other KV format is refused; a bf16-KV decoder
    gives the same ids and pool bytes before and after an fp8-KV decoder ran on the same LLM"""
    from vila_b200 import serving
    model = T4._model("tiny")[0]
    llm = model.llm
    prompts = [_prompt(llm, S, seed=S) for S in (120, 333, 57, 410, 260)]

    def run_bf16():
        dec = serving.BatchedDecoder(llm, slots=3, max_tokens_per_slot=1024, max_new=32)
        dec.capture()
        for s, S in enumerate((300, 170)):
            dec.admit(s, _prompt(llm, S, seed=S))
        dec.run(16)
        return [dec.generated(s) for s in range(3)], dec.pool.clone(), dec

    with torch.inference_mode():
        ids_a, pool_a, bf_dec = run_bf16()
        got3 = serving.generate_batch(llm, prompts, max_new_tokens=24, slots=3, kv_cache="fp8")
        got20 = serving.generate_batch(llm, prompts * 4, max_new_tokens=24, slots=20, kv_cache="fp8")
        alone = [serving.generate_batch(llm, [p], max_new_tokens=24, slots=1, kv_cache="fp8")[0] for p in prompts]
        f8_dec = serving.BatchedDecoder(llm, slots=1, max_tokens_per_slot=1024, max_new=32, kv_cache="fp8")
        with pytest.raises(ValueError):
            serving.generate_batch(llm, prompts[:1], max_new_tokens=4, decoder=f8_dec)
        with pytest.raises(ValueError):
            serving.generate_batch(llm, prompts[:1], max_new_tokens=4, decoder=bf_dec, kv_cache="fp8")
        ids_b, pool_b, _ = run_bf16()
    assert all(len(a) == 24 for a in alone)
    assert got3 == alone and got20 == alone * 4
    assert ids_a == ids_b and torch.equal(pool_a, pool_b)
