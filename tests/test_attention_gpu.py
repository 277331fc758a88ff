"""GPU: every prefill attention call (fmha_fwd_kernel through ops.fmha) at its production shape, mask and KV
layout, in its call form, against the fp64 reference; and the RoPE inputs of that attention, bit for bit.

Table, from nvila_8b(), nvila_8b_dynamic_s2(), nvila_video_8b() and nvila_lite_3b(), one group per call site:
  siglip   vision.py SiglipEncoderLayer.forward: non-causal, H = 16, D = 72 (zero-padded to 96 by TMA), q/k/v
           the strided views qkv[:, 0 / 1 / 2] of the [B*S, 3, H, D] projection output.  S = num_patches,
           B = 1, 2, the tiles of a square dynamic-S2 image (media.tiling_plan) and the video frames; plus
           S = 729, B = 3, whose last KV block reads the next sequence's rows.  The output goes to a view with
           head stride 80 whose columns 72..79, and the rows after it, hold a sentinel.
  prefill  qwen2.py prefill_hidden: causal GQA (28/4 and 16/2 heads), q the [:, :Hq] view of the
           [S, Hq+2Hkv, D] qkv buffer, K/V in a PagedKVCache with a permuted page order, Sk = p0 + S.  Every
           page slot that holds no token (past Sk in the last page, the spare pages) holds garbage.
  packed   qwen2.py forward_packed: one causal launch per segment on views of q3[o:o+n], out=attn[o:o+n] of a
           shared buffer; the pad rows after the segments must keep their sentinel.
  sp       sp.py SequenceParallelPrefill: make_plan(S, world, rank) for world 2 and 4 and every rank, the pool
           in the plan's gathered zigzag layout, both chunk calls (Sk = a1, then b1) of a rank on one GPU.
Each case runs the three families of tests.helpers.attention_inputs (random, sink, probe) and checks:
  * tests.helpers.AttnErrors against tests.helpers.attention_reference (fp64): per element, per row, bias;
  * a second call gives the same bits, and variant=1 (the kernel pinned) the same bits as the default;
  * the K/V inputs (pools, qkv buffers) are unchanged, and nothing outside the output view is written.
The q / K / V values are written straight into the buffers the call site hands to the kernel (after RoPE
in the model); the RoPE kernels that produce them are checked bit for bit at the end of this file.
"""
import zlib

import pytest
import torch

from oracle import vila_oracle as O
from tests.helpers import (ATTN_FAMILIES, AttnErrors, _record, attention_errors, attention_inputs,
                           bf16_rounding_tie_distance)
from tests.test_kernels_gpu import _ops

pytestmark = pytest.mark.gpu

PAGE = 128
LLM_M_MAX = 16470          # 64-frame video prompt (the LLM projections' largest M)
OUT_SENTINEL = -4096.0     # exact in bf16, far outside any attention output here
PREFILL_SQ = [1, 7, 64, 65, 127, 128, 129, 279, 384, 385, 4096, LLM_M_MAX]
PREFILL_P0, PREFILL_P0_SQ = (77, 128, 16000), (1, 65, 129, 385)  # p0 > 0: eager decode, engine slots
PACKED_LENS = (129, 1, 300, 64)
PACKED_PAD = 21
SP_SEQ = LLM_M_MAX


def _cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------
# the production table
# ------------------------------------------------------------------------------------------------
def _table():
    from vila_b200.model.configuration import nvila_8b, nvila_8b_dynamic_s2, nvila_lite_3b, nvila_video_8b
    from vila_b200.model.media import tiling_plan

    cfgs = (("8b", nvila_8b()), ("8b-s2", nvila_8b_dynamic_s2()), ("video", nvila_video_8b()),
            ("lite", nvila_lite_3b()))
    vis, llms, frames, s2_tiles = set(), {}, 1, None
    for tag, cfg in cfgs:
        v = cfg.vision_tower_cfg
        vis.add((v.num_attention_heads, v.hidden_size // v.num_attention_heads, v.num_patches))
        l = cfg.llm_cfg
        llms.setdefault((l.num_attention_heads, l.num_key_value_heads, l.head_dim, l.hidden_size), []).append(tag)
        frames = max(frames, cfg.num_video_frames if tag == "video" else 1)
        if cfg.dynamic_s2:  # a square image: every scale's grid (1 + 4 + 9 tiles of 448)
            side = cfg.vision_tower_cfg.image_size * 3
            jobs, _ = tiling_plan(side, side, cfg)
            s2_tiles = sum((w // v.image_size) * (h // v.image_size) for w, h in jobs)
    rows = []
    for (H, D, S) in sorted(vis):
        for B in sorted({1, 2, s2_tiles, frames}):
            rows.append(dict(site="siglip", id=f"siglip.S{S}.B{B}", B=B, S=S, H=H, D=D))
        rows.append(dict(site="siglip", id="siglip.S729.B3", B=3, S=729, H=H, D=D))  # off production: KV tail
    for (Hq, Hkv, D, hidden), tags in llms.items():
        lt = f"llm{hidden}"
        for Sq in PREFILL_SQ:
            rows.append(dict(site="prefill", id=f"{lt}.prefill.S{Sq}.p0", Sq=Sq, p0=0, Hq=Hq, Hkv=Hkv, D=D))
        for p0 in PREFILL_P0:
            for Sq in PREFILL_P0_SQ:
                rows.append(dict(site="prefill", id=f"{lt}.prefill.S{Sq}.p{p0}", Sq=Sq, p0=p0, Hq=Hq, Hkv=Hkv, D=D))
        rows.append(dict(site="packed", id=f"{lt}.packed." + "-".join(map(str, PACKED_LENS)), lens=PACKED_LENS,
                         pad=PACKED_PAD, Hq=Hq, Hkv=Hkv, D=D))
        if "video" in tags:  # LongVILA: sequence-parallel prefill of the video model
            for world in (2, 4):
                for rank in range(world):
                    rows.append(dict(site="sp", id=f"{lt}.sp.S{SP_SEQ}.w{world}r{rank}", S=SP_SEQ, world=world,
                                     rank=rank, Hq=Hq, Hkv=Hkv, D=D))
    return rows, dict(s2_tiles=s2_tiles, frames=frames)


TABLE, DERIVED = _table()


def _seed(case, family):
    return zlib.crc32(case["id"].encode()) * 3 + ATTN_FAMILIES.index(family)


def _fresh_out(shape_rows, Hq, cols, dev):
    return torch.full((shape_rows, Hq, cols), OUT_SENTINEL, dtype=torch.bfloat16, device=dev)


# ------------------------------------------------------------------------------------------------
# the call sites
# ------------------------------------------------------------------------------------------------
def _siglip(ops, case, family, dev):
    """-> (checker, [output buffers of the default, repeated and variant=1 calls], inputs unchanged)"""
    B, S, H, D = case["B"], case["S"], case["H"], case["D"]
    scale = D ** -0.5
    pos = torch.arange(B * S, device=dev)
    q, k, v = attention_inputs(family, pos, pos, H, H, D, scale, sink=pos % S == 0, seed=_seed(case, family))
    qkv = torch.stack([q, k, v], dim=1)  # [B*S, 3, H, D]: the layout of ops.linear(...).view(B*S, 3, H, D)
    before = qkv.clone()
    bufs = []
    for variant in (0, 0, 1):
        buf = _fresh_out(B * S + 8, H, 80, dev)  # head stride 80: columns 72..79 and 8 rows past the end
        ops.fmha(qkv[:, 0], qkv[:, 1], qkv[:, 2], B=B, Sq=S, Sk=S, causal=False, scale=scale,
                 out=buf[:B * S, :, :D], variant=variant)
        bufs.append(buf)
    torch.cuda.synchronize()
    buf = bufs[0]
    outside = torch.cat([buf[:B * S, :, D:].reshape(-1), buf[B * S:].reshape(-1)])
    e = AttnErrors()
    for b in range(B):
        sl = slice(b * S, (b + 1) * S)
        attention_errors(buf[sl, :, :D], q[sl], k[sl], v[sl], causal=False, scale=scale, into=e, row0=b * S * H)
    return e, bufs, outside, torch.equal(qkv, before)


def _prefill(ops, case, family, dev):
    from vila_b200.model.configuration import Qwen2Config
    from vila_b200.model.qwen2 import PagedKVCache
    Sq, p0, Hq, Hkv, D = case["Sq"], case["p0"], case["Hq"], case["Hkv"], case["D"]
    scale = D ** -0.5
    Sk = p0 + Sq
    n_pages = _cdiv(Sk, PAGE) + 2  # two spare pages
    g = torch.Generator().manual_seed(_seed(case, family))
    cfg = Qwen2Config(hidden_size=Hq * D, num_hidden_layers=1, num_attention_heads=Hq, num_key_value_heads=Hkv)
    cache = PagedKVCache(cfg, n_pages * PAGE, dev, page_order=torch.randperm(n_pages, generator=g).tolist())
    slot = torch.arange(n_pages * PAGE, device=dev)  # token t lives in logical page t // 128
    q, k, v = attention_inputs(family, torch.arange(p0, Sk, device=dev), slot, Hq, Hkv, D, scale,
                               sink=slot == 0, garbage=slot >= Sk, seed=_seed(case, family))
    pt = cache.page_table.long()
    cache.k(0)[pt] = k.view(n_pages, PAGE, Hkv, D)
    cache.v(0)[pt] = v.view(n_pages, PAGE, Hkv, D)
    qkv = torch.zeros(Sq, (Hq + 2 * Hkv) * D, dtype=torch.bfloat16, device=dev)
    qkv.view(Sq, Hq + 2 * Hkv, D)[:, :Hq] = q
    qv = qkv.view(Sq, Hq + 2 * Hkv, D)[:, :Hq]
    pool0 = cache.pool.clone()
    outs = [ops.fmha(qv, cache.k(0), cache.v(0), B=1, Sq=Sq, Sk=Sk, causal=True, scale=scale,
                     page_table=cache.page_table, variant=variant) for variant in (0, 0, 1)]
    torch.cuda.synchronize()
    kseq = cache.k(0)[pt].reshape(-1, Hkv, D)[:Sk]  # K/V as stored, in token order
    vseq = cache.v(0)[pt].reshape(-1, Hkv, D)[:Sk]
    e = attention_errors(outs[0], q, kseq, vseq, causal=True, scale=scale)
    return e, outs, None, torch.equal(cache.pool, pool0)


def _packed(ops, case, family, dev):
    lens, Hq, Hkv, D = case["lens"], case["Hq"], case["Hkv"], case["D"]
    scale = D ** -0.5
    T = sum(lens) + case["pad"]
    starts = torch.tensor([sum(lens[:i]) for i in range(len(lens))], device=dev)
    pos = torch.arange(T, device=dev)
    q, k, v = attention_inputs(family, pos, pos, Hq, Hkv, D, scale, sink=torch.isin(pos, starts),
                               seed=_seed(case, family))
    q3 = torch.cat([q, k, v], dim=1)  # [T, Hq + 2 Hkv, D]: qkv.view(T, Hq + 2 * Hkv, D)
    before = q3.clone()
    bufs = []
    for variant in (0, 0, 1):
        attn = _fresh_out(T, Hq, D, dev)
        o = 0
        for n in lens:
            ops.fmha(q3[o:o + n, :Hq], q3[o:o + n, Hq:Hq + Hkv], q3[o:o + n, Hq + Hkv:], B=1, Sq=n, Sk=n,
                     causal=True, scale=scale, out=attn[o:o + n], variant=variant)
            o += n
        bufs.append(attn)
    torch.cuda.synchronize()
    e = AttnErrors()
    o = 0
    for n in lens:
        sl = slice(o, o + n)
        attention_errors(bufs[0][sl], q[sl], k[sl], v[sl], causal=True, scale=scale, into=e, row0=o * Hq)
        o += n
    return e, bufs, bufs[0][sum(lens):].reshape(-1), torch.equal(q3, before)


def _sp(ops, case, family, dev):
    from vila_b200.sp import make_plan
    Hq, Hkv, D = case["Hq"], case["Hkv"], case["D"]
    scale = D ** -0.5
    plan = make_plan(case["S"], case["world"], case["rank"])
    c = plan.chunk
    n_pages = plan.padded_len // PAGE
    pt = plan.page_table().to(dev)
    key_pos = torch.arange(plan.padded_len, device=dev)
    q, k, v = attention_inputs(family, plan.local_positions().to(dev).long(), key_pos, Hq, Hkv, D, scale,
                               sink=key_pos == 0, seed=_seed(case, family))
    kpool = torch.zeros(n_pages, PAGE, Hkv, D, dtype=torch.bfloat16, device=dev)
    vpool = torch.zeros_like(kpool)
    kpool[pt.long()] = k.view(n_pages, PAGE, Hkv, D)  # the gathered layout: global block j at page pt[j]
    vpool[pt.long()] = v.view(n_pages, PAGE, Hkv, D)
    qkv = torch.zeros(2 * c, Hq + 2 * Hkv, D, dtype=torch.bfloat16, device=dev)
    qkv[:, :Hq] = q
    qv = qkv[:, :Hq]
    k0, v0 = kpool.clone(), vpool.clone()
    (a0, a1), (b0, b1) = plan.local_chunks()
    bufs, first_only = [], None
    for variant in (0, 0, 1):
        attn = _fresh_out(2 * c, Hq, D, dev)
        ops.fmha(qv[:c], kpool, vpool, B=1, Sq=c, Sk=a1, causal=True, scale=scale, page_table=pt,
                 out=attn[:c], variant=variant)
        if first_only is None:
            first_only = attn[c:].clone().reshape(-1)  # the second chunk's rows before its own call
        ops.fmha(qv[c:], kpool, vpool, B=1, Sq=c, Sk=b1, causal=True, scale=scale, page_table=pt,
                 out=attn[c:], variant=variant)
        bufs.append(attn)
    torch.cuda.synchronize()
    kseq = kpool[pt.long()].reshape(-1, Hkv, D)
    vseq = vpool[pt.long()].reshape(-1, Hkv, D)
    e = attention_errors(bufs[0][:c], q[:c], kseq[:a1], vseq[:a1], causal=True, scale=scale)
    attention_errors(bufs[0][c:], q[c:], kseq[:b1], vseq[:b1], causal=True, scale=scale, into=e, row0=c * Hq)
    return e, bufs, first_only, torch.equal(kpool, k0) and torch.equal(vpool, v0)


SITES = {"siglip": _siglip, "prefill": _prefill, "packed": _packed, "sp": _sp}


def _shape(case):
    keys = ("B", "S", "Sq", "p0", "lens", "world", "rank", "H", "Hq", "Hkv", "D")
    return {k: (list(case[k]) if k == "lens" else case[k]) for k in keys if k in case}


@pytest.mark.parametrize("case", TABLE, ids=[c["id"] for c in TABLE])
def test_attention(cuda, case):
    ops = _ops()
    failures = []
    for family in ATTN_FAMILIES:
        e, outs, outside, inputs_kept = SITES[case["site"]](ops, case, family, cuda)
        what = f"{case['id']} {family}"
        assert torch.equal(outs[0], outs[1]), f"{what}: two calls differ"
        assert torch.equal(outs[0], outs[2]), f"{what}: variant=1 differs from the default dispatch"
        assert inputs_kept, f"{what}: the K/V inputs changed"
        if outside is not None:
            assert bool((outside == OUT_SENTINEL).all()), \
                f"{what}: {int((outside != OUT_SENTINEL).sum())} elements written outside the output view"
        _record({"name": "attention", "site": case["site"], "case": case["id"], **_shape(case), "family": family,
                 **e.summary()})
        failures += [f"{what}: {f}" for f in e.failures()]
        del outs, e
    torch.cuda.empty_cache()
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("site", list(SITES))
def test_attention_coverage(site):
    """one row per call site: the cases its group runs, and the production shapes they must include"""
    rows = [c for c in TABLE if c["site"] == site]
    if site == "siglip":
        got = {(c["S"], c["B"]) for c in rows}
        want = {(1024, 1), (1024, 2), (1024, DERIVED["s2_tiles"]), (1024, DERIVED["frames"]), (729, 3)}
        assert DERIVED["s2_tiles"] == 14 and DERIVED["frames"] == 64 and want <= got
    elif site == "prefill":
        got = {(c["Hq"], c["Hkv"], c["Sq"], c["p0"]) for c in rows}
        for heads in ((28, 4), (16, 2)):
            assert {heads + (s, 0) for s in PREFILL_SQ} <= got
            assert {heads + (s, p) for p in PREFILL_P0 for s in PREFILL_P0_SQ} <= got
    elif site == "packed":
        assert {(c["Hq"], c["Hkv"]) for c in rows} == {(28, 4), (16, 2)}
    else:
        assert sorted((c["world"], c["rank"]) for c in rows) == [(2, 0), (2, 1), (4, 0), (4, 1), (4, 2), (4, 3)]
    _record({"name": "attention coverage", "site": site, "cases": len(rows), "families": list(ATTN_FAMILIES),
             "ids": [c["id"] for c in rows]})


# ------------------------------------------------------------------------------------------------
# RoPE inputs, bit for bit
# ------------------------------------------------------------------------------------------------
SP_MAX_POS = 65824  # > 65,814, the LongVILA 256-frame prompt of the sequence-parallel prefill


def _inv_freq(D, dev):
    return O.rope_inv_freq(D, 1e6).to(dev)  # = Qwen2ForCausalLM.inv_freq (fp32)


def test_rope_table_exact(cuda):
    """rope_table == bf16(cos / sin in fp64 of the fp32 angle fp32(pos) * inv_freq), except entries within
    4 fp32 ulps of a bf16 rounding boundary (sincosf is accurate to ~1 fp32 ulp), which may be one bf16 ulp
    off; positions 0 .. 65,823 (sequence-parallel prompts)."""
    ops = _ops()
    for D in (128,):
        inv = _inv_freq(D, cuda)
        pos = torch.arange(SP_MAX_POS, dtype=torch.int32, device=cuda)
        tab = ops.rope_table(pos, D, inv)
        ang = pos.float()[:, None] * inv[None, :]  # fp32 product, as HF's fp32 freqs
        x64 = torch.cat([torch.cos(ang.double()), torch.sin(ang.double())], dim=1)
        want = x64.to(torch.bfloat16)
        diff = tab != want
        near = bf16_rounding_tie_distance(x64) < 4.0
        off_ulps = (tab.double() - want.double()).abs() / torch.ldexp(torch.ones_like(x64), torch.frexp(
            torch.maximum(tab.double().abs(), want.double().abs()))[1] - 8)
        _record({"name": "rope_table exact", "D": D, "positions": SP_MAX_POS, "entries": tab.numel(),
                 "near_tie": int(near.sum()), "differ": int(diff.sum()), "differ_near_tie": int((diff & near).sum())})
        assert not bool((diff & ~near).any()), \
            f"D={D}: {int((diff & ~near).sum())} entries differ away from a rounding boundary"
        assert bool((off_ulps[diff] <= 1.0).all()), f"D={D}: an entry near a boundary is more than one ulp off"


def _rope_emulated(x, table, Hq, Hkv, D):
    """HF apply_rotary_pos_emb on bf16 tensors: y0 = bf16(bf16(x0 c) + bf16(-x1 s)), y1 = bf16(bf16(x1 c) +
    bf16(x0 s)) on the q and k heads of qkv [S, (Hq+2Hkv) D]; v heads unchanged"""
    S = x.shape[0]
    h = x.view(S, Hq + 2 * Hkv, D).float()
    c, s = table[:, None, :D // 2].float(), table[:, None, D // 2:].float()
    x0, x1 = h[:, :Hq + Hkv, :D // 2], h[:, :Hq + Hkv, D // 2:]

    def rb(t):
        return t.to(torch.bfloat16).float()
    y = h.clone()
    y[:, :Hq + Hkv, :D // 2] = rb(rb(x0 * c) + rb(-x1 * s))
    y[:, :Hq + Hkv, D // 2:] = rb(rb(x1 * c) + rb(x0 * s))
    return y.to(torch.bfloat16).view(S, -1)


@pytest.mark.parametrize("Hq,Hkv", [(28, 4), (16, 2)])
def test_rope_rotation_exact(cuda, Hq, Hkv):
    """rope_kv_append_table and rope_kv_append (per-element sincosf) rotate q and k exactly as HF's bf16 ops
    do, given the table; positions spread up to 65.8K"""
    ops = _ops()
    D, S = 128, 1000
    g = torch.Generator(device=cuda).manual_seed(Hq)
    x = (torch.randn(S, (Hq + 2 * Hkv) * D, device=cuda, generator=g) * 3).to(torch.bfloat16)
    pos = torch.randint(0, SP_MAX_POS, (S,), device=cuda, generator=g).to(torch.int32)
    pos[:4] = torch.tensor([0, 1, 65535, SP_MAX_POS - 1], dtype=torch.int32, device=cuda)
    inv = _inv_freq(D, cuda)
    table = ops.rope_table(pos, D, inv)
    want = _rope_emulated(x, table, Hq, Hkv, D)
    a = x.clone()
    ops.rope_kv_append_table(a, table, Hq, Hkv, D)
    b = x.clone()
    ops.rope_kv_append(b, pos, Hq, Hkv, D, inv)
    assert torch.equal(a, want), f"table rotation: {int((a != want).sum())} elements differ"
    assert torch.equal(b, want), f"sincosf rotation: {int((b != want).sum())} elements differ"


@pytest.mark.parametrize("p0", [77, 200, 16000 + 77])
def test_rope_pool_scatter_exact(cuda, p0):
    """the K/V pool append of rope_kv_append_table and rope_kv_append: token p0 + s lands in page
    page_table[(p0 + s) // 128], row (p0 + s) % 128, bit for bit (rotated k, unrotated v), across page
    boundaries with p0 not a multiple of 128; every other slot keeps its contents"""
    ops = _ops()
    Hq, Hkv, D, S = 28, 4, 128, 300
    g = torch.Generator(device=cuda).manual_seed(p0)
    x = torch.randn(S, (Hq + 2 * Hkv) * D, device=cuda, generator=g).to(torch.bfloat16)
    pos = torch.arange(p0, p0 + S, dtype=torch.int32, device=cuda)
    inv = _inv_freq(D, cuda)
    table = ops.rope_table(pos, D, inv)
    n_pages = _cdiv(p0 + S, PAGE) + 1
    pt = torch.randperm(n_pages, device=cuda, generator=g).to(torch.int32)
    rot = _rope_emulated(x, table, Hq, Hkv, D).view(S, Hq + 2 * Hkv, D)
    t = pos.long()
    for name, run in (("table", lambda q, kp, vp: ops.rope_kv_append_table(q, table, Hq, Hkv, D, kp, vp, pt, p0)),
                      ("sincosf", lambda q, kp, vp: ops.rope_kv_append(q, pos, Hq, Hkv, D, inv, kp, vp, pt, p0))):
        kp = torch.full((n_pages, PAGE, Hkv, D), OUT_SENTINEL, dtype=torch.bfloat16, device=cuda)
        vp = kp.clone()
        run(x.clone(), kp, vp)
        pages, rows = pt.long()[t // PAGE], t % PAGE
        assert torch.equal(kp[pages, rows], rot[:, Hq:Hq + Hkv]), f"{name}: k rows differ"
        assert torch.equal(vp[pages, rows], rot[:, Hq + Hkv:]), f"{name}: v rows differ"
        kp[pages, rows] = OUT_SENTINEL
        vp[pages, rows] = OUT_SENTINEL
        assert bool((kp == OUT_SENTINEL).all() and (vp == OUT_SENTINEL).all()), f"{name}: wrote outside its slots"
