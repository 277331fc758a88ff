"""CPU: the decode-attention checker of tests/test_decode_attention_gpu.py, checked without a GPU.

Three fp32 emulations restate the arithmetic of the decode attention kernels:
  emulate_simt   decode_attn_head_kernel (splits = 1) and decode_attn_kernel (splits > 1, the cluster path),
                 decode.cu: split s covers tokens [s per, (s + 1) per), per = ceil(n_tok / splits); token t of a
                 split goes to half-warp (t - t0) % 16, which keeps a running maximum m, l summed from the
                 unrounded p and o += bf16(p) v; the 16 half-warp partials, then the splits, are combined in a
                 fixed order in fp32.  The new token's K/V come from registers, never from the pool row at pos.
  emulate_split  fmha_fwd_kernel in split mode + decode_combine_kernel or the fused last-CTA combine
                 (fmha_wgmma.cu, decode.cu): the G query heads of a KV group are the rows of the tile, 128-token
                 blocks, a normalised fp32 partial and lse = m + log2 l per split (-inf for an empty one), the
                 combine over all splits (single sequence) or over the nsp that hold tokens (batched).  The new
                 row is read from the pool, where rope_kv_append wrote it.
  emulate_fp8    decode_attn_fp8_kernel (kv_fp8.cu): K/V as e4m3 codes with one fp32 scale per row (the rule of
                 quantize_kv_e4m3), score = (q . code_k * kscale) * scale log2(e), 128-token chunks,
                 pb = bf16(p * vscale), the combine of the splits that hold tokens.
tests.helpers.AttnErrors accepts each, with margin, on the three families of decode_attention_inputs at G = 7 and
G = 8, and rejects each fault planted below through the check named for it (FAULTS).
"""
import pytest
import torch

from tests.helpers import DECODE_FAMILIES, SENTINEL_V, attention_errors, decode_attention_inputs, decode_edges
from vila_b200.model.qwen2 import quantize_kv_e4m3

PAGE = 128
D = 128
SCALE = D ** -0.5
SL2 = (torch.tensor(SCALE, dtype=torch.float32) * torch.tensor(1.4426950408889634, dtype=torch.float32)).item()
HEADS = {7: (14, 2), 8: (16, 2)}  # G -> (Hq, Hkv): two KV groups, so "the last group" is not the only one


def _cdiv(a, b):
    return -(-a // b)


def _bf16(t):
    return t.to(torch.bfloat16).float()


def _bf16_rz(t):
    """bf16 by truncation (round toward zero)"""
    return (t.to(torch.float32).view(torch.int32) & -65536).view(torch.float32)


def _round_p(p, fault):
    return _bf16_rz(p) if fault == "p_truncated" else _bf16(p)


def _combine(ms, ls, os, fault=None):
    """fixed-order fp32 combine of partials (m [n, H], l [n, H], o [n, H, D]) with unnormalised o: the
    half-warp and cross-split combines of decode.cu.  -> (m, l, o)"""
    mm = ms.amax(dim=0)
    w = torch.where(ms == float("-inf"), torch.zeros_like(ms), torch.exp2(ms - mm))
    wo = w
    if fault == "stale_max":  # the numerator's weights against the first partial's maximum, not the current one
        m0 = ms[0]
        wo = torch.where(ms == float("-inf"), torch.zeros_like(ms), torch.exp2(ms - m0))
    ll = torch.zeros_like(mm)
    oo = torch.zeros_like(os[0])
    for s in range(ms.shape[0]):
        ll = ll + ls[s] * w[s]
        oo = oo + os[s] * wo[s][:, None]
    return mm, ll, oo


def _q_heads(q, Hkv, fault):
    """q [Hq, D] fp32 as the kernels index it; gqa_last: the last head of the last KV group reads its
    neighbour's row"""
    q = q.float().clone()
    if fault == "gqa_last":
        q[-1] = q[-2]
    return q


def emulate_simt(q, kseq, vseq, k_new, v_new, pos, splits, fault=None):
    """decode_attn_head_kernel (splits = 1) / decode_attn_kernel (cluster, splits <= 8) for one sequence.
    q [Hq, D] bf16 (rotated); kseq, vseq [slots, Hkv, D] bf16 in token order as the page table maps them,
    row pos holding what the pool held before the call; k_new, v_new [Hkv, D] the registers' row.
    -> bf16 output [Hq, D]"""
    Hq = q.shape[0]
    Hkv = kseq.shape[1]
    hk = torch.arange(Hq) // (Hq // Hkv)
    Q = _q_heads(q, Hkv, fault)
    n_tok = pos + 1
    per = _cdiv(n_tok, splits)
    pm, pl, po = [], [], []
    for s in range(splits):
        t0 = s * per
        t1 = min(n_tok, t0 + per)
        if fault == "split_edge_drop" and s < splits - 1:
            t1 = min(n_tok, t0 + per - 1)
        if fault == "split_edge_twice" and s < splits - 1:
            t1 = min(n_tok, t0 + per + 1)
        if fault == "tail_unmasked" and t1 == n_tok:
            t1 = _cdiv(n_tok, PAGE) * PAGE
        toks = [t for t in range(t0, t1) if not (fault == "drop_prev" and t == pos - 1)]
        if fault == "new_twice" and t0 <= pos < t1:
            toks.append(pos)  # once from the registers, once more from the freshly appended pool row
        # half-warp hw takes the split's tokens t0 + hw, t0 + hw + 16, ... in order
        lanes = [[t for t in toks if (t - t0) % 16 == hw] for hw in range(16)]
        m = torch.full((16, Hq), float("-inf"))
        l = torch.zeros(16, Hq)
        o = torch.zeros(16, Hq, D)
        for step in range(max(len(x) for x in lanes) if toks else 0):
            for hw in range(16):
                if step >= len(lanes[hw]):
                    continue
                t = lanes[hw][step]
                fresh = t == pos and fault != "stale_new"
                K = (k_new if fresh else kseq[t]).float()[hk]
                V = (v_new if fresh else vseq[t]).float()[hk]
                sc = (Q * K).sum(dim=1) * SL2
                m_new = torch.maximum(m[hw], sc)
                alpha = torch.exp2(m[hw] - m_new)
                pexp = torch.exp2(sc - m_new)
                l[hw] = l[hw] * alpha + pexp
                o[hw] = o[hw] * alpha[:, None] + _round_p(pexp, fault)[:, None] * V
                m[hw] = m_new
        mm, ll, oo = _combine(m, l, o, fault if splits == 1 else None)
        pm.append(mm)
        pl.append(ll)
        po.append(oo)
    if splits > 1:
        _, ll, oo = _combine(torch.stack(pm), torch.stack(pl), torch.stack(po), fault)
    return (oo / ll[:, None]).to(torch.bfloat16)


def emulate_split(q, kseq, vseq, pos, num_splits, split_tokens, batched=False, fault=None):
    """fmha_fwd_kernel in split mode + the combine, for one sequence.  kseq, vseq [>= num_splits *
    split_tokens, Hkv, D] bf16 in token order after rope_kv_append (row pos = the new row); every slot a
    128-token block loads, the ones past pos included.  batched: the fused combine of the batched launch,
    over the splits that hold tokens.  -> bf16 output [Hq, D]"""
    Hq = q.shape[0]
    Hkv = kseq.shape[1]
    G = Hq // Hkv
    Q = _q_heads(q, Hkv, fault)
    total = pos + 1
    lse = torch.empty(num_splits, Hq)
    opart = torch.empty(num_splits, Hq, D)
    for z in range(num_splits):
        start = z * split_tokens
        Sk = max(0, min(split_tokens, total - start))
        if fault == "split_edge_drop" and 0 < Sk < split_tokens:
            Sk -= 1  # Sk = total - start - 1: the last split loses its last key
        for hk in range(Hkv):
            rows = slice(hk * G, (hk + 1) * G)
            m = torch.full((G,), float("-inf"))
            l = torch.zeros(G)
            O = torch.zeros(G, D)
            for j in range(_cdiv(Sk, PAGE)):
                kv0 = start + j * PAGE
                K, V = kseq[kv0:kv0 + PAGE, hk].float(), vseq[kv0:kv0 + PAGE, hk].float()
                S = Q[rows] @ K.t()
                lim = Sk - 1 + (1 if fault == "split_edge_twice" and z < num_splits - 1 else 0)
                if fault != "tail_unmasked":
                    S = S.masked_fill(j * PAGE + torch.arange(PAGE)[None, :] > lim, float("-inf"))
                m_new = torch.maximum(m, S.amax(dim=1) * SL2)
                m_use = torch.where(m_new == float("-inf"), torch.zeros_like(m_new), m_new)
                alpha = torch.exp2(m - m_use)
                P = torch.exp2(S * SL2 - m_use[:, None])
                l = l * alpha + P.sum(dim=1)
                O = O * alpha[:, None] + _round_p(P, fault) @ V
                m = m_new
            inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
            opart[z, rows] = O * inv[:, None]
            empty = -torch.inf if fault != "empty_lse_zero" else 0.0
            lse[z, rows] = torch.where(l > 0, m + torch.log2(l), torch.full_like(l, empty))
    nsp = min(num_splits, _cdiv(total, split_tokens)) if batched else num_splits
    lse, opart = lse[:nsp], opart[:nsp]
    mx = lse.amax(dim=0)
    w = torch.where(lse == float("-inf"), torch.zeros_like(lse), torch.exp2(lse - mx))
    den = torch.zeros(Hq)
    acc = torch.zeros(Hq, D)
    for s in range(nsp):
        den = den + w[s]
        acc = acc + w[s][:, None] * opart[s]
    inv = torch.where(den > 0, 1.0 / den, torch.zeros_like(den))
    return (acc * inv[:, None]).to(torch.bfloat16)


def emulate_fp8(q, kc, ks, vc, vs, pos, num_splits, split_tokens, fault=None):
    """decode_attn_fp8_kernel for one slot.  kc, vc [slots, Hkv, D] e4m3 codes and ks, vs [slots, Hkv] fp32
    scales in token order after the append (row pos = the quantised new row).  -> bf16 output [Hq, D]"""
    Hq = q.shape[0]
    Hkv = kc.shape[1]
    G = Hq // Hkv
    Q = _q_heads(q, Hkv, fault)
    kf, vf = kc.float(), vc.float()
    if fault == "kscale_neighbour":
        ks = torch.roll(ks, -1, dims=0)  # token t scaled by token t + 1's scale
    n_used = min(pos // split_tokens + 1, num_splits)
    out = torch.empty(Hq, D)
    for hk in range(Hkv):
        rows = slice(hk * G, (hk + 1) * G)
        rec = []
        for sp in range(n_used):
            t0 = sp * split_tokens
            t1 = min(pos + 1, t0 + split_tokens)
            m = torch.full((G,), float("-inf"))
            l = torch.zeros(G)
            acc = torch.zeros(G, D)
            for c0 in range(t0, t1, PAGE):
                n = min(PAGE, t1 - c0)
                sc = (Q[rows] @ kf[c0:c0 + n, hk].t()) * ks[c0:c0 + n, hk][None, :] * SL2
                m_new = torch.maximum(m, sc.amax(dim=1))
                alpha = torch.exp2(m - m_new)
                pe = torch.exp2(sc - m_new[:, None])
                l = l * alpha + pe.sum(dim=1)
                vsc = vs[c0:c0 + n, hk][None, :]
                pb = _bf16(pe) * vsc if fault == "vscale_after_round" else _round_p(pe * vsc, fault)
                acc = acc * alpha[:, None] + pb @ vf[c0:c0 + n, hk]
                m = m_new
            rec.append((m, l, acc))
        if n_used == 1:
            m, l, acc = rec[0]
            out[rows] = acc / l[:, None]
        else:
            _, ll, oo = _combine(torch.stack([r[0] for r in rec]), torch.stack([r[1] for r in rec]),
                                 torch.stack([r[2] for r in rec]), "stale_max" if fault == "stale_max" else None)
            out[rows] = oo / ll[:, None]
    return out.to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------
# cases: one per kernel family, the pool as the kernel sees it through the page table (token order)
# ------------------------------------------------------------------------------------------------
# kernel -> (pos, plan): head kernel over 3 pages; the cluster at 8 splits (per = 76, not a page multiple);
# the wgmma split mode with 5 of 8 splits empty; the batched fused combine (3 of 8 splits hold tokens);
# fp8 at three of four 256-token splits
CASES = {
    "head": (300, dict(splits=1)),
    "cluster": (600, dict(splits=8)),
    "split": (300, dict(num_splits=8, split_tokens=128)),
    "split_batch": (300, dict(num_splits=8, split_tokens=128, batched=True)),
    "fp8": (700, dict(num_splits=4, split_tokens=256)),
}


def _chunks(kernel, pos, plan):
    if kernel in ("head", "cluster"):
        return (PAGE, _cdiv(pos + 1, plan["splits"]))
    return (PAGE, plan["split_tokens"])


def run_case(kernel, family, G, fault=None, seed=0):
    """-> (AttnErrors, emulated output)"""
    pos, plan = CASES[kernel]
    Hq, Hkv = HEADS[G]
    inp = decode_attention_inputs(family, pos, Hq, Hkv, D, SCALE, seed * 101 + G, chunks=_chunks(kernel, pos, plan))
    slots = max(_cdiv(pos + 1, PAGE) * PAGE, plan.get("num_splits", 1) * plan.get("split_tokens", 0))
    kseq = inp.k_garbage[None].expand(slots, Hkv, D).clone()
    vseq = torch.full((slots, Hkv, D), SENTINEL_V, dtype=torch.bfloat16)
    kseq[:pos], vseq[:pos] = inp.k_hist, inp.v_hist
    K, V = inp.keys()
    if kernel in ("head", "cluster"):
        got = emulate_simt(inp.q, kseq, vseq, inp.k_new, inp.v_new, pos, plan["splits"], fault)
    elif kernel.startswith("split"):
        kseq[pos], vseq[pos] = inp.k_new, inp.v_new  # rope_kv_append ran first
        got = emulate_split(inp.q, kseq, vseq, pos, plan["num_splits"], plan["split_tokens"],
                            plan.get("batched", False), fault)
    else:
        kc, ks = quantize_kv_e4m3(kseq)
        vc, vs = quantize_kv_e4m3(vseq)
        kn, kns = quantize_kv_e4m3(inp.k_new)
        vn, vns = quantize_kv_e4m3(inp.v_new)
        kc[pos], ks[pos], vc[pos], vs[pos] = kn, kns, vn, vns
        got = emulate_fp8(inp.q, kc, ks, vc, vs, pos, plan["num_splits"], plan["split_tokens"], fault)
        K = kc[:pos + 1].double() * ks[:pos + 1, :, None].double()  # the reference: fp64 over the dequantised pool
        V = vc[:pos + 1].double() * vs[:pos + 1, :, None].double()
    e = attention_errors(got[None], inp.q[None], K, V, causal=False, scale=SCALE)
    return e, got


def bias_exempt(kernel, family):
    """the fp8 kernel on the sink family: one key carries the row, and its bf16(p * vscale) is one rounding
    shared by G * 128 outputs (test_fp8_sink_bias_is_one_shared_rounding).  Every other check still applies."""
    return kernel.startswith("fp8") and family == "sink"


def _caught(e):
    """the checks of AttnErrors that fail"""
    out = set()
    if not e.excess <= 1.0:
        out.add("element")
    if not e.worst_row <= e.ROW_RMS:
        out.add("row")
    if not abs(e.bias) <= e.BIAS_ULP:
        out.add("bias")
    return out


def test_leak_family_promise():
    """decode_attention_inputs' leak family: every garbage key scores >= 16 above every visible key for every
    head (asserted inside), and the edge keys are where the plan puts them"""
    e = decode_edges(600, (128, 76))
    want = {0, 75, 76, 127, 128, 151, 152, 255, 256, 227, 228, 303, 304, 379, 380, 383, 384, 455, 456, 511,
            512, 531, 532, 599, 600, 607, 608}
    assert set(torch.nonzero(e).view(-1).tolist()) == {t for t in want if t <= 600}
    for G in HEADS:
        decode_attention_inputs("leak", 600, *HEADS[G], D, SCALE, 1, chunks=(128, 76))


@pytest.mark.parametrize("G", list(HEADS))
@pytest.mark.parametrize("family", DECODE_FAMILIES)
@pytest.mark.parametrize("kernel", list(CASES))
def test_checker_accepts_kernel_arithmetic(kernel, family, G):
    """Each emulated kernel passes every check with margin: no element uses more than 0.6 of its bound (a single
    flipped rounding costs at most 0.5 of it), no row exceeds 2 of the per-row bound's 3, and the rounding
    bias of the output stays within 0.05 ulp.  Decode has Hq rows only, so the bias is a mean over Hq * 128
    elements: +-0.29 / sqrt(1792) = +-0.007 at G = 7."""
    for seed in range(2):
        e, _ = run_case(kernel, family, G, seed=seed)
        bad = [f for f in e.failures() if not (f.startswith("rounding bias") and bias_exempt(kernel, family))]
        assert not bad, (kernel, family, G, seed, e.summary())
        assert e.excess <= 0.6 and e.worst_row <= 2.0, (kernel, family, G, seed, e.summary())
        assert bias_exempt(kernel, family) or abs(e.bias) <= 0.05, (kernel, family, G, seed, e.summary())


def test_fp8_sink_bias_is_one_shared_rounding():
    """Why the fp8 kernel is exempt from the bias check on the sink family (bias_exempt): the sink key has
    p = 1 for every head, so pb = bf16(vscale_0) is ONE rounding that all G * 128 outputs of its KV group
    share, and the group's outputs move together by its relative error (up to 2^-9).  With a few KV groups the
    mean signed error is then a mean of a few such shifts, not of independent roundings: 0.12 ulp here.  Taking
    the sink's V scale as bf16(vscale_0) in the reference removes the shift and the bias falls to the
    independent-rounding level."""
    kernel, family, G = "fp8", "sink", 7
    e, got = run_case(kernel, family, G)
    assert e.excess <= 0.6 and e.worst_row <= 2.0 and abs(e.bias) > 0.1, e.summary()
    pos, plan = CASES[kernel]
    Hq, Hkv = HEADS[G]
    inp = decode_attention_inputs(family, pos, Hq, Hkv, D, SCALE, G, chunks=_chunks(kernel, pos, plan))
    K, V = inp.keys()
    kc, ks = quantize_kv_e4m3(K)
    vc, vs = quantize_kv_e4m3(V)
    vs[0] = vs[0].to(torch.bfloat16).float()
    e2 = attention_errors(got[None], inp.q[None], kc.double() * ks[..., None].double(),
                          vc.double() * vs[..., None].double(), causal=False, scale=SCALE)
    assert not e2.failures() and abs(e2.bias) <= 0.05, e2.summary()


def test_pos0_is_v_new():
    """pos = 0: one key, p = 1, so every kernel's output is bf16(v_new) exactly"""
    for G in HEADS:
        Hq, Hkv = HEADS[G]
        inp = decode_attention_inputs("random", 0, Hq, Hkv, D, SCALE, 5)
        kseq = inp.k_garbage[None].expand(PAGE, Hkv, D).clone()
        vseq = torch.full((PAGE, Hkv, D), SENTINEL_V, dtype=torch.bfloat16)
        want = inp.v_new.repeat_interleave(G, dim=0)
        assert torch.equal(emulate_simt(inp.q, kseq, vseq, inp.k_new, inp.v_new, 0, 1), want)
        kseq[0], vseq[0] = inp.k_new, inp.v_new
        assert torch.equal(emulate_split(inp.q, kseq, vseq, 0, 1, 128), want)


# fault -> (kernel, family, G, the checks that must catch it: any one of them)
FAULTS = {
    "stale_new": ("head", "leak", 7, {"element"}),           # the new token read from the stale pool row
    "new_twice": ("head", "leak", 7, {"element", "row"}),    # the new token counted twice (registers and pool)
    "drop_prev": ("cluster", "leak", 7, {"element", "row"}),  # token pos - 1 dropped
    "split_edge_drop": ("cluster", "leak", 7, {"element", "row"}),   # the last key of a split dropped
    "split_edge_twice": ("cluster", "leak", 7, {"element", "row"}),  # the next split's first key counted twice
    "split_edge_drop_wgmma": ("split", "leak", 7, {"element", "row"}),   # Sk = total - start - 1
    "split_edge_twice_wgmma": ("split", "leak", 8, {"element", "row"}),  # a split reads one key past its end
    "empty_lse_zero": ("split", "leak", 7, {"bias"}),        # an empty split weighted as if it held tokens
    "tail_unmasked": ("head", "leak", 8, {"element"}),       # the last page read past pos
    "tail_unmasked_wgmma": ("split_batch", "leak", 8, {"element"}),
    "gqa_last": ("cluster", "random", 7, {"element"}),       # last group: a query head reads its neighbour's q
    "stale_max": ("cluster", "random", 8, {"element"}),      # combine weights against a stale maximum
    "stale_max_fp8": ("fp8", "random", 7, {"element"}),
    "kscale_neighbour": ("fp8", "random", 7, {"element"}),   # fp8: the next token's K scale
    # P truncated instead of rounded.  The SIMT kernels start every half-warp run with p = 1 and give p = 1 to
    # each new running maximum, exactly representable either way: with the few tokens per half-warp of the
    # cluster path (5 here) truncation moves the bias by -0.04 only, which no check sees; over the head
    # kernel's longer runs it reaches -0.11 (random, G = 7), just past BIAS_ULP.  The wgmma and fp8 kernels
    # round every p of a 128-token block: -0.27 and -0.37.
    "p_truncated": ("head", "random", 7, {"bias"}),
    "p_truncated_wgmma": ("split", "random", 8, {"bias"}),
    "p_truncated_fp8": ("fp8", "random", 8, {"bias"}),
}


def _base(fault):
    for suffix in ("_wgmma", "_fp8"):
        if fault.endswith(suffix):
            return fault[:-len(suffix)]
    return fault


@pytest.mark.parametrize("fault", list(FAULTS))
def test_checker_rejects_planted_fault(fault):
    kernel, family, G, checks = FAULTS[fault]
    e, bad = run_case(kernel, family, G, fault=_base(fault))
    _, clean = run_case(kernel, family, G)
    assert not torch.equal(clean, bad), f"{fault}: the planted fault does not change the output here"
    assert checks & _caught(e), (fault, e.summary())
    if _base(fault) == "p_truncated":  # every element stays within its bound: only the mean sees it
        assert _caught(e) == {"bias"} and e.bias < -0.1, e.summary()


@pytest.mark.parametrize("family", DECODE_FAMILIES)
def test_vscale_after_rounding_is_invisible(family):
    """fp8: applying the V scale after rounding P (bf16(p) vscale instead of bf16(p vscale)) changes the output
    bits but not its error statistics: both round P with a relative error below 2^-8, so no check can tell
    the two apart and the kernel's order is pinned by its own comment and review, not by this checker."""
    for G in HEADS:
        e, bad = run_case("fp8", family, G, fault="vscale_after_round")
        _, clean = run_case("fp8", family, G)
        assert not torch.equal(clean, bad)
        assert not e.failures(), e.summary()
