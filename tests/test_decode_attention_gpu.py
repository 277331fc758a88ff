"""GPU: every decode attention call at its production context, split plan and KV layout, in its call form,
against the fp64 reference (tests.helpers.attention_reference, Sq = 1, non-causal over the keys 0..pos).

Table, from nvila_8b(), nvila_8b_dynamic_s2(), nvila_video_8b() and nvila_lite_3b() (28/4 and 16/2 heads,
D = 128), one group per call site:
  single  GraphDecoder._step: ops.decode_attention (num_splits 0: decode_attn_head_kernel; 8: the cluster
          kernel) or ops.decode_attention_split (rope_kv_append + fmha split mode + decode_combine_kernel), the
          plan from GraphDecoder.pick_splits run on this device, under cache_for's rule (the plan of a long
          context comes from cache.max_tokens); a permuted page table over a pool with two spare pages.
  batched BatchedDecoder._step: positions split at HEAD_KERNEL_TOKENS into decode_attention_batch and
          decode_attention_split_batch writing one attn buffer, at serving.attention_config of the longest slot.
  fp8     BatchedDecoder._step with kv_cache="fp8": decode_attention_fp8_batch at every FP8_LADDER_TOKENS entry
          that covers the batch (serving.fp8_attention_config).
Each case runs the three families of tests.helpers.decode_attention_inputs (random, sink, leak) and checks:
  * AttnErrors: per element, per row and bias (the fp8 kernel's bias only over slots of >= FP8_BIAS_MIN_KEYS
    keys and not on the sink family: tests.helpers.FP8_BIAS_MIN_KEYS);
  * pos = 0: the output is the new V row exactly;
  * the appended K (rotated) and V rows are bit-equal to the reference (fp8: codes and scales to the rule), and
    every other pool byte is unchanged;
  * the split paths leave the rotated q / k in qkv; the head, cluster and fp8 kernels leave qkv untouched;
  * output rows of idle slots and the columns past Hq * D of a wider buffer keep their sentinel;
  * work buffers start NaN-filled, counters start and end at zero; a second call on fresh copies gives the same
    bits.
"""
import types
import zlib

import pytest
import torch

from tests.helpers import (DECODE_FAMILIES, FP8_BIAS_MIN_KEYS, SENTINEL_V, AttnErrors, _record, attention_errors,
                           decode_attention_inputs, scatter_tokens)
from tests.test_kernels_gpu import _ops

pytestmark = pytest.mark.gpu

PAGE = 128
D = 128
SCALE = D ** -0.5
OUT_SENTINEL = -4096.0
EXTRA_COLS = 64  # columns past Hq * D in the output buffer
SPARE_PAGES = 2


def _cdiv(a, b):
    return -(-a // b)


def _heads():
    from vila_b200.model.configuration import nvila_8b, nvila_8b_dynamic_s2, nvila_lite_3b, nvila_video_8b
    out = {}
    for cfg in (nvila_8b(), nvila_8b_dynamic_s2(), nvila_video_8b(), nvila_lite_3b()):
        l = cfg.llm_cfg
        out[(l.num_attention_heads, l.num_key_value_heads)] = l
    return out


HEADS = _heads()

# single: (cache tokens as GraphDecoder.cache_for gets them, positions)
SINGLE_HEAD = (512, (0, 1, 127, 128, 129, 511))
SINGLE_CLUSTER = ((600, (0, 7, 8, 9, 599)), (1024, (0, 7, 8, 9, 512, 1023)))
SINGLE_SPLIT_TOTALS = (1025, 4096, 16470 + 1024, 65814 + 1024)
# batched: one step per SPLIT_LADDER entry, each with short, idle and boundary slots
BATCH_STEPS = ((-1, 0, 1023, 1024, 1025, 2047, 2048, 8191),
               (8192, 2047, -1, 16383, 1025),
               (16384, 32767, -1, 5),
               (32768, 69631, -1, 2048, 1))
FP8_STEPS = ((-1, 0, 1, 511, 512, 513, 2047),
             (2048, 8191, -1, 1),
             (16469, -1, 512),
             (32768, 69631, -1, 1))


def _graph_decoder_stub(l, dev):
    """what GraphDecoder.pick_splits reads: the LLM's config and device, MAX_SPLITS and LONG_CTX"""
    from vila_b200.model.qwen2 import GraphDecoder
    return types.SimpleNamespace(llm=types.SimpleNamespace(config=l, device=dev), MAX_SPLITS=GraphDecoder.MAX_SPLITS,
                                 LONG_CTX=GraphDecoder.LONG_CTX)


def single_plan(l, tokens, dev):
    """GraphDecoder.cache_for(tokens): the cache's size and the plan of its steps -> (max_tokens, ns, st)"""
    from vila_b200.model.qwen2 import GraphDecoder
    max_tokens = _cdiv(max(tokens, 1024), PAGE) * PAGE
    stub = _graph_decoder_stub(l, dev)
    ns, st = GraphDecoder.pick_splits(stub, max_tokens if tokens > GraphDecoder.LONG_CTX else tokens)
    return max_tokens, ns, st


def _split_positions(max_tokens, st, ns):
    """near the start (most splits empty), every kind of split edge at the first, a middle and the last split
    boundary, a page edge, and the cache's last slot"""
    ps = {5, 255, 256, max_tokens - 1}
    for j in sorted({1, ns // 2, ns - 1}):
        ps |= {j * st - 1, j * st, j * st + 1}
    return sorted(p for p in ps if 0 <= p < max_tokens)


def _table():
    rows = []
    for (Hq, Hkv) in HEADS:
        h = f"{Hq}x{Hkv}"
        tokens, ps = SINGLE_HEAD
        rows += [dict(site="single", kind="head", id=f"single.{h}.head.t{tokens}.p{p}", Hq=Hq, Hkv=Hkv, tokens=tokens,
                      pos=p) for p in ps]
        for tokens, ps in SINGLE_CLUSTER:
            rows += [dict(site="single", kind="cluster", id=f"single.{h}.cluster.t{tokens}.p{p}", Hq=Hq, Hkv=Hkv,
                          tokens=tokens, pos=p) for p in ps]
        for tokens in SINGLE_SPLIT_TOTALS:
            rows.append(dict(site="single", kind="split", id=f"single.{h}.split.t{tokens}", Hq=Hq, Hkv=Hkv,
                             tokens=tokens, pos=None))  # positions from the device's plan
        for i, ps in enumerate(BATCH_STEPS):
            rows.append(dict(site="batched", id=f"batched.{h}.step{i}", Hq=Hq, Hkv=Hkv, positions=ps))
        for i, ps in enumerate(FP8_STEPS):
            rows.append(dict(site="fp8", id=f"fp8.{h}.step{i}", Hq=Hq, Hkv=Hkv, positions=ps))
    return rows


TABLE = _table()


def _seed(case, family, extra=0):
    return zlib.crc32(case["id"].encode()) * 7 + DECODE_FAMILIES.index(family) + 3 * extra


def _nan(n, dev):
    return torch.full((n,), float("nan"), dtype=torch.float32, device=dev)


def _rope_inputs(dev):
    from oracle import vila_oracle as O
    return O.rope_inv_freq(D, 1e6).to(dev)  # = Qwen2ForCausalLM.inv_freq (fp32)


def _summary(e):
    s = e.summary()
    return {"excess": s["excess"], "worst_row": s["worst_row"], "bias_ulp": s["bias_ulp"], "max_ulps": s["max_ulps"]}


# ------------------------------------------------------------------------------------------------
# single sequence (GraphDecoder)
# ------------------------------------------------------------------------------------------------
def _single_call(ops, case, family, pos, plan, dev):
    """-> (failures, record)"""
    Hq, Hkv = case["Hq"], case["Hkv"]
    G = Hq // Hkv
    max_tokens, ns, st = plan
    n_pages = max_tokens // PAGE
    g = torch.Generator().manual_seed(_seed(case, family, pos))
    perm = torch.randperm(n_pages + SPARE_PAGES, generator=g)
    pt = perm[:n_pages].to(torch.int32).to(dev)
    chunks = (PAGE, st) if st else (PAGE, _cdiv(pos + 1, ns)) if ns else (PAGE,)
    inp = decode_attention_inputs(family, pos, Hq, Hkv, D, SCALE, _seed(case, family, pos), chunks=chunks, device=dev)
    kp = inp.k_garbage[None, None].expand(n_pages + SPARE_PAGES, PAGE, Hkv, D).contiguous()
    vp = torch.full_like(kp, SENTINEL_V)
    scatter_tokens(kp, pt, inp.k_hist)
    scatter_tokens(vp, pt, inp.v_hist)
    inv = _rope_inputs(dev)
    position = torch.tensor([pos], dtype=torch.int32, device=dev)
    outs, state = [], None
    for _ in range(2):
        qkv, k, v = inp.qkv.clone(), kp.clone(), vp.clone()
        buf = torch.full((Hq * D + EXTRA_COLS,), OUT_SENTINEL, dtype=torch.bfloat16, device=dev)
        counters = torch.zeros(Hkv, dtype=torch.int32, device=dev)
        if st:
            o_partial, lse = _nan(64 * Hq * D, dev), _nan(64 * Hq, dev)
            ops.decode_attention_split(qkv, position, k, v, pt, buf[:Hq * D], o_partial, lse, inv, Hq, Hkv, D, ns, st,
                                       SCALE)
        else:
            ws = _nan(Hkv * 64 * G * (D + 2), dev)
            ops.decode_attention(qkv, position, k, v, pt, buf[:Hq * D], ws, counters, inv, Hq, Hkv, D, ns, SCALE)
        torch.cuda.synchronize()
        outs.append(buf)
        if state is None:
            state = (qkv, k, v, counters)
    qkv, k, v, counters = state
    bad = []
    if not torch.equal(outs[0], outs[1]):
        bad.append("two calls differ")
    out = outs[0][:Hq * D].view(1, Hq, D)
    if not bool((outs[0][Hq * D:] == OUT_SENTINEL).all()):
        bad.append("columns past Hq * D written")
    if int(counters.abs().sum()):
        bad.append("counters not re-armed")
    page, row = pt[pos // PAGE].long(), pos % PAGE
    if not torch.equal(k[page, row], inp.k_new) or not torch.equal(v[page, row], inp.v_new):
        bad.append("appended K/V row differs from the reference")
    kw, vw = kp.clone(), vp.clone()
    kw[page, row], vw[page, row] = inp.k_new, inp.v_new
    if not (torch.equal(k, kw) and torch.equal(v, vw)):
        bad.append("pool bytes other than the appended row changed")
    want_qkv = torch.cat([inp.q.reshape(-1), inp.k_new.reshape(-1), inp.v_new.reshape(-1)]) if st else inp.qkv
    if not torch.equal(qkv, want_qkv):
        bad.append("qkv is not " + ("the rotated q / k" if st else "untouched"))
    if pos == 0 and not torch.equal(out[0], inp.v_new.repeat_interleave(G, dim=0)):
        bad.append("pos 0: output is not v_new")
    K, V = inp.keys()
    e = attention_errors(out, inp.q[None], K, V, causal=False, scale=SCALE)
    bad += e.failures()
    return bad, e


def _single_positions(case, plan):
    if case["pos"] is not None:
        return [case["pos"]]
    max_tokens, ns, st = plan
    return _split_positions(max_tokens, st, ns)


def run_single(ops, case, family, dev):
    l = HEADS[(case["Hq"], case["Hkv"])]
    plan = single_plan(l, case["tokens"], dev)
    kind = "head" if plan[1] == 0 else "cluster" if plan[2] == 0 else "split"
    assert kind == case["kind"], f"{case['id']}: the device's plan {plan} is not the {case['kind']} path"
    res = []
    for pos in _single_positions(case, plan):
        bad, e = _single_call(ops, case, family, pos, plan, dev)
        res.append((dict(pos=pos, plan=dict(max_tokens=plan[0], num_splits=plan[1], split_tokens=plan[2])), bad, e))
    return res


# ------------------------------------------------------------------------------------------------
# batched (BatchedDecoder): bf16 pool and fp8 pool
# ------------------------------------------------------------------------------------------------
def _batch_layout(positions, gen):
    """every active slot owns ceil((pos + 1) / 128) pages, handed out interleaved over one pool (long and short
    slots are neighbours), plus spare pages; unused page-table entries point at spare pages"""
    need = [_cdiv(p + 1, PAGE) if p >= 0 else 0 for p in positions]
    width = max(max(need), 1)
    P = sum(need) + SPARE_PAGES
    perm = torch.randperm(P, generator=gen).tolist()
    pt = torch.empty(len(positions), width, dtype=torch.int32)
    o = 0
    for b, n in enumerate(need):
        pt[b, :n] = torch.tensor(perm[o:o + n], dtype=torch.int32)
        spare = perm[sum(need):]
        pt[b, n:] = torch.tensor([spare[i % len(spare)] for i in range(width - n)], dtype=torch.int32)
        o += n
    return pt, P


def _batch_inputs(case, family, positions, kind, dev):
    from vila_b200 import serving
    Hq, Hkv = case["Hq"], case["Hkv"]
    inps = []
    for b, p in enumerate(positions):
        if p < 0:
            inps.append(None)
            continue
        if kind == "fp8":
            chunks = (PAGE, serving.FP8_SPLIT_TOKENS)
        else:
            chunks = (PAGE, serving.SPLIT_TOKENS) if p >= serving.HEAD_KERNEL_TOKENS else (PAGE,)
        inps.append(decode_attention_inputs(family, p, Hq, Hkv, D, SCALE, _seed(case, family, b), chunks=chunks,
                                            device=dev))
    return inps


def _qkv_rows(inps, Hq, Hkv, dev, gen_seed):
    g = torch.Generator(device=dev).manual_seed(gen_seed)
    qkv = torch.randn(len(inps), (Hq + 2 * Hkv) * D, device=dev, generator=g).to(torch.bfloat16)  # idle rows: noise
    for b, inp in enumerate(inps):
        if inp is not None:
            qkv[b] = inp.qkv
    return qkv


def _common_batch_checks(outs, Hq, positions, counters_list, bad):
    if not torch.equal(outs[0], outs[1]):
        bad.append("two calls differ")
    buf = outs[0]
    if not bool((buf[:, Hq * D:] == OUT_SENTINEL).all()):
        bad.append("columns past Hq * D written")
    for b, p in enumerate(positions):
        if p < 0 and not bool((buf[b] == OUT_SENTINEL).all()):
            bad.append(f"idle slot {b}: output row written")
    if any(int(c.abs().sum()) for c in counters_list):
        bad.append("counters not re-armed")


def run_batched(ops, case, family, dev):
    from vila_b200 import serving
    Hq, Hkv = case["Hq"], case["Hkv"]
    G = Hq // Hkv
    positions = case["positions"]
    B = len(positions)
    gen = torch.Generator().manual_seed(_seed(case, family))
    pt_cpu, P = _batch_layout(positions, gen)
    pt = pt_cpu.to(dev)
    inps = _batch_inputs(case, family, positions, "bf16", dev)
    kg = next(i for i in inps if i is not None).k_garbage
    kp = kg[None, None].expand(P, PAGE, Hkv, D).contiguous()
    vp = torch.full_like(kp, SENTINEL_V)
    for b, inp in enumerate(inps):
        if inp is not None:
            scatter_tokens(kp, pt_cpu[b], inp.k_hist)
            scatter_tokens(vp, pt_cpu[b], inp.v_hist)
    qkv0 = _qkv_rows(inps, Hq, Hkv, dev, _seed(case, family, 99))
    num_splits = serving.attention_config(max(positions) + 1)
    assert num_splits is not None
    pos_t = torch.tensor(positions, dtype=torch.int32, device=dev)
    long = pos_t >= serving.HEAD_KERNEL_TOKENS
    pos_head = pos_t.clone().masked_fill_(long, -1)
    pos_split = pos_t.clone().masked_fill_(~long, -1)
    inv = _rope_inputs(dev)
    outs, cnts, state = [], [], None
    for _ in range(2):
        qkv, k, v = qkv0.clone(), kp.clone(), vp.clone()
        buf = torch.full((B, Hq * D + EXTRA_COLS), OUT_SENTINEL, dtype=torch.bfloat16, device=dev)
        attn = buf[:, :Hq * D]
        o_partial, lse = _nan(B * num_splits * Hq * D, dev), _nan(B * num_splits * Hq, dev)
        counters = torch.zeros(B * Hkv, dtype=torch.int32, device=dev)
        ops.decode_attention_batch(qkv, pos_head, k, v, pt, attn, inv, Hq, Hkv, D, SCALE)
        ops.decode_attention_split_batch(qkv, pos_split, k, v, pt, attn, o_partial, lse, counters, inv, Hq, Hkv, D,
                                         num_splits, serving.SPLIT_TOKENS, SCALE)
        torch.cuda.synchronize()
        outs.append(buf)
        cnts.append(counters)
        if state is None:
            state = (qkv, k, v)
    qkv, k, v = state
    bad = []
    _common_batch_checks(outs, Hq, positions, cnts, bad)
    kw, vw = kp.clone(), vp.clone()
    e = AttnErrors()
    for b, (p, inp) in enumerate(zip(positions, inps)):
        if inp is None:
            if not torch.equal(qkv[b], qkv0[b]):
                bad.append(f"idle slot {b}: qkv changed")
            continue
        page, row = pt_cpu[b, p // PAGE].item(), p % PAGE
        if not torch.equal(k[page, row], inp.k_new) or not torch.equal(v[page, row], inp.v_new):
            bad.append(f"slot {b} (pos {p}): appended K/V row differs from the reference")
        kw[page, row], vw[page, row] = inp.k_new, inp.v_new
        rotated = torch.cat([inp.q.reshape(-1), inp.k_new.reshape(-1), inp.v_new.reshape(-1)])
        want = rotated if p >= serving.HEAD_KERNEL_TOKENS else inp.qkv
        if not torch.equal(qkv[b], want):
            bad.append(f"slot {b} (pos {p}): qkv is not " + ("the rotated q / k" if p >= serving.HEAD_KERNEL_TOKENS
                                                              else "untouched"))
        out = outs[0][b, :Hq * D].view(1, Hq, D)
        if p == 0 and not torch.equal(out[0], inp.v_new.repeat_interleave(G, dim=0)):
            bad.append(f"slot {b}: pos 0 output is not v_new")
        K, V = inp.keys()
        attention_errors(out, inp.q[None], K, V, causal=False, scale=SCALE, into=e, row0=b * Hq)
    if not (torch.equal(k, kw) and torch.equal(v, vw)):
        bad.append("pool bytes other than the appended rows changed")
    bad += e.failures()
    return [(dict(positions=list(positions), plan=dict(num_splits=num_splits, split_tokens=serving.SPLIT_TOKENS,
                                                       head_kernel_tokens=serving.HEAD_KERNEL_TOKENS)), bad, e)]


def run_fp8(ops, case, family, dev):
    from vila_b200 import serving
    from vila_b200.model.qwen2 import quantize_kv_e4m3
    Hq, Hkv = case["Hq"], case["Hkv"]
    positions = case["positions"]
    B = len(positions)
    gen = torch.Generator().manual_seed(_seed(case, family))
    pt_cpu, P = _batch_layout(positions, gen)
    pt = pt_cpu.to(dev)
    inps = _batch_inputs(case, family, positions, "fp8", dev)
    kg = next(i for i in inps if i is not None).k_garbage
    gkc, gks = quantize_kv_e4m3(kg)
    gvc, gvs = quantize_kv_e4m3(torch.full_like(kg, SENTINEL_V))
    kc = gkc[None, None].expand(P, PAGE, Hkv, D).contiguous()
    vc = gvc[None, None].expand(P, PAGE, Hkv, D).contiguous()
    ks = gks[None, None].expand(P, PAGE, Hkv).contiguous()
    vs = gvs[None, None].expand(P, PAGE, Hkv).contiguous()
    refs = []
    for b, inp in enumerate(inps):
        if inp is None:
            refs.append(None)
            continue
        K, V = inp.keys()
        c_k, s_k = quantize_kv_e4m3(K)  # history as kv_quantize_fp8 leaves it, the new row by the rule
        c_v, s_v = quantize_kv_e4m3(V)
        p = inp.pos
        for pool, src in ((kc, c_k), (vc, c_v), (ks, s_k), (vs, s_v)):
            scatter_tokens(pool.view(torch.uint8) if pool.dtype == torch.float8_e4m3fn else pool, pt_cpu[b],
                           (src.view(torch.uint8) if src.dtype == torch.float8_e4m3fn else src)[:p])
        refs.append((c_k, s_k, c_v, s_v))
    qkv0 = _qkv_rows(inps, Hq, Hkv, dev, _seed(case, family, 99))
    pos_t = torch.tensor(positions, dtype=torch.int32, device=dev)
    inv = _rope_inputs(dev)
    longest = max(positions) + 1
    res = []
    for n in serving.FP8_LADDER_TOKENS:
        if n < longest:
            continue
        num_splits = serving.fp8_attention_config(n)
        outs, cnts, state = [], [], None
        for _ in range(2):
            qkv, k, v, sk, sv = qkv0.clone(), kc.clone(), vc.clone(), ks.clone(), vs.clone()
            buf = torch.full((B, Hq * D + EXTRA_COLS), OUT_SENTINEL, dtype=torch.bfloat16, device=dev)
            ws = _nan(B * Hq * num_splits * (D + 2), dev)
            counters = torch.zeros(B * Hkv, dtype=torch.int32, device=dev)
            ops.decode_attention_fp8_batch(qkv, pos_t, k, v, sk, sv, pt, buf[:, :Hq * D], ws, counters, inv, Hq, Hkv,
                                           num_splits, serving.FP8_SPLIT_TOKENS, SCALE)
            torch.cuda.synchronize()
            outs.append(buf)
            cnts.append(counters)
            if state is None:
                state = (qkv, k, v, sk, sv)
        qkv, k, v, sk, sv = state
        bad = []
        _common_batch_checks(outs, Hq, positions, cnts, bad)
        if not torch.equal(qkv, qkv0):
            bad.append("qkv changed")
        want = [t.clone() for t in (kc, vc, ks, vs)]
        e, eb = AttnErrors(), AttnErrors()  # eb: the slots whose rounding bias is checked (FP8_BIAS_MIN_KEYS)
        for b, (p, inp) in enumerate(zip(positions, inps)):
            if inp is None:
                continue
            c_k, s_k, c_v, s_v = refs[b]
            page, row = pt_cpu[b, p // PAGE].item(), p % PAGE
            got_rows = (k[page, row], v[page, row], sk[page, row], sv[page, row])
            for name, gr, wr in zip(("K codes", "V codes", "K scale", "V scale"), got_rows,
                                    (c_k[p], c_v[p], s_k[p], s_v[p])):
                a = gr.view(torch.uint8) if gr.dtype == torch.float8_e4m3fn else gr
                w = wr.view(torch.uint8) if wr.dtype == torch.float8_e4m3fn else wr
                if not torch.equal(a, w):
                    bad.append(f"slot {b} (pos {p}): appended {name} differ from the rule")
            for t, src in zip(want, (c_k[p], c_v[p], s_k[p], s_v[p])):
                t[page, row] = src
            out = outs[0][b, :Hq * D].view(1, Hq, D)
            Kd = c_k.double() * s_k[..., None].double()  # fp64 over the dequantised pool
            Vd = c_v.double() * s_v[..., None].double()
            if p == 0:  # one key, p = 1: the output is bf16(code * bf16(vscale)), the dequantised new row
                v0 = (c_v[0].float() * s_v[0][:, None].to(torch.bfloat16).float()).to(torch.bfloat16)
                if not torch.equal(out[0], v0.repeat_interleave(Hq // Hkv, dim=0)):
                    bad.append(f"slot {b}: pos 0 output is not the new V row")
            attention_errors(out, inp.q[None], Kd, Vd, causal=False, scale=SCALE, into=e, row0=b * Hq)
            if p + 1 >= FP8_BIAS_MIN_KEYS:
                attention_errors(out, inp.q[None], Kd, Vd, causal=False, scale=SCALE, into=eb, row0=b * Hq)
        for got_t, want_t in zip((k, v, sk, sv), want):
            a = got_t.view(torch.uint8) if got_t.dtype == torch.float8_e4m3fn else got_t
            w = want_t.view(torch.uint8) if want_t.dtype == torch.float8_e4m3fn else want_t
            if not torch.equal(a, w):
                bad.append("pool bytes other than the appended rows changed")
                break
        bad += [f for f in e.failures() if not f.startswith("rounding bias")]
        if family != "sink":
            bad += [f"bias over slots of >= {FP8_BIAS_MIN_KEYS} keys: {f}" for f in eb.failures()
                    if f.startswith("rounding bias")]
        res.append((dict(positions=list(positions), plan=dict(ladder_tokens=n, num_splits=num_splits,
                                                              split_tokens=serving.FP8_SPLIT_TOKENS)), bad, e))
    assert res, f"{case['id']}: no ladder entry covers {longest} tokens"
    return res


SITES = {"single": run_single, "batched": run_batched, "fp8": run_fp8}


@pytest.mark.parametrize("case", TABLE, ids=[c["id"] for c in TABLE])
def test_decode_attention(cuda, case):
    ops = _ops()
    failures = []
    for family in DECODE_FAMILIES:
        for where, bad, e in SITES[case["site"]](ops, case, family, cuda):
            _record({"name": "decode attention", "site": case["site"], "case": case["id"], "Hq": case["Hq"],
                     "Hkv": case["Hkv"], **where, "family": family, **_summary(e)})
            failures += [f"{case['id']} {family} {where}: {f}" for f in bad]
    torch.cuda.empty_cache()
    assert not failures, "\n".join(failures[:40])


def test_decode_attention_plans(cuda):
    """the plans the table reaches on this device: pick_splits for every single-sequence cache, the batched
    ladder, the fp8 ladder (recorded, so a change of SM count or ladder shows in the record)"""
    from vila_b200 import serving
    plans = {}
    for (Hq, Hkv), l in HEADS.items():
        for tokens in (SINGLE_HEAD[0],) + tuple(t for t, _ in SINGLE_CLUSTER) + SINGLE_SPLIT_TOTALS:
            max_tokens, ns, st = single_plan(l, tokens, cuda)
            assert ns * st >= max_tokens if st else ns in (0, 8)
            plans[f"{Hq}x{Hkv}.t{tokens}"] = dict(max_tokens=max_tokens, num_splits=ns, split_tokens=st)
    steps = {f"step{i}": serving.attention_config(max(ps) + 1) for i, ps in enumerate(BATCH_STEPS)}
    assert sorted(steps.values()) == sorted(serving.SPLIT_LADDER)  # every ladder entry is run
    fp8 = {f"step{i}": [n for n in serving.FP8_LADDER_TOKENS if n >= max(ps) + 1] for i, ps in enumerate(FP8_STEPS)}
    assert set(serving.FP8_LADDER_TOKENS) == {n for v in fp8.values() for n in v}
    _record({"name": "decode attention plans", "sms": torch.cuda.get_device_properties(cuda).multi_processor_count,
             "single": plans, "batched": steps, "fp8": fp8})
