"""CPU: the exact-or-tie checker (tests.helpers.TieErrors) and the fp64 references of the norms (norm.cu) and the
media data-movement kernels (data_movement.cu), on fp32 emulations of the kernels' arithmetic.

* LayerNorm / RMSNorm: the CTA-per-row and warp-per-row kernels emulated in fp32 in their own summation order (per
  thread or lane chains over 16-byte vectors, the xor-shuffle tree, the block tree; fused multiply-adds where
  nvcc contracts them; rsqrtf as a correctly rounded reciprocal square root).  They pass the checker on every
  input family at every production width: every fp32 value lies within the derived eps of the fp64 value, and
  no flip needs more than half of it (the margins are recorded).
* Planted faults, each rejected by the check it names.
* The fp64 S2 and TSP references agree with oracle.vila_oracle's restatements of the reference.
* norm_plan by hand at its boundaries.
"""
import math

import pytest
import torch

from oracle import vila_oracle as O
from tests.helpers import (NORM_FAMILIES, TieErrors, _record, bf16_rne64, bf16_ulp, layernorm_reference,
                           norm_inputs, norm_plan, rmsnorm_reference, rmsnorm_then, s2_merge_reference,
                           tsp_pool_reference)

F32 = torch.float32
LN_WIDTHS = (1152, 4608, 13824, 10368, 3456, 144, 576, 1296, 432)  # SigLIP, projectors (8B, S2, Lite), tiny
RMS_WIDTHS = (3584, 2048, 512)  # Qwen2-7B, Qwen2.5-3B, tiny
# stated largest tie-window fraction per family
MAX_WINDOW = {"random": 0.01, "offset": 0.01, "outlier": 0.01, "small": 0.01}
# largest part of eps a flip may use.  Offset rows sum exactly in fp32 (integers of a few bits), so their
# mean's error is the one rounding of sum / cols, computed exactly by layernorm_reference and used in full by
# every element it dominates: there the check is that the bound holds, elsewhere that it holds with margin 2
NEEDED = {"random": 0.5, "offset": 1.0, "outlier": 0.5, "small": 0.5}


# ------------------------------------------------------------------------------------------------
# fp32 emulations of norm.cu
# ------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """fp32 fma: the product is exact in fp64, the sum rounds once more there (below fp32's resolution)"""
    return (a.double() * b.double() + c.double()).float()


def rsqrtf(x):
    return (1.0 / x.double().sqrt()).float()


def bf16_rz(t):
    """fp32 -> bf16 toward zero (truncation), as fp32"""
    u = t.contiguous().view(torch.int32) & ~0xFFFF
    return u.view(F32)


def _lanes(regime):
    return 256 if regime == "cta" else 32


def _vectors(x32, regime):
    """[R, cols] -> ([R, iters, lanes, 8] zero-padded, valid [iters, lanes]) in the order a thread / lane owns
    them: vector i goes to thread i % lanes, its iteration i // lanes"""
    R, cols = x32.shape
    nvec, L = cols // 8, _lanes(regime)
    it = -(-nvec // L)
    v = torch.zeros(R, it * L, 8, dtype=F32)
    v[:, :nvec] = x32.view(R, nvec, 8)
    valid = torch.arange(it * L) < nvec
    return v.view(R, it, L, 8), valid.view(it, L)


def _tree(part, regime):
    """partials [R, lanes] -> the row total as warp_sum (and block_sum) reduce them"""
    def warp_sum(v):  # [R, W, 32]
        idx = torch.arange(32)
        for o in (16, 8, 4, 2, 1):
            v = v + v[..., idx ^ o]
        return v
    R = part.shape[0]
    if regime == "warp":
        return warp_sum(part.view(R, 1, 32))[:, 0, 0]
    w = warp_sum(part.view(R, 8, 32))[:, :, 0]
    t = torch.cat([w, torch.zeros(R, 24, dtype=F32)], dim=1)
    return warp_sum(t.view(R, 1, 32))[:, 0, 0]


def _row_sum(v, valid, regime, drop_vector0=False):
    """sum of the elements: each vector's 8 values chained left to right, then added to the thread's sum"""
    R, it, L, _ = v.shape
    s = torch.zeros(R, L, dtype=F32)
    for i in range(it):
        p = v[:, i, :, 0]
        for k in range(1, 8):
            p = p + v[:, i, :, k]
        keep = valid[i].clone()
        if drop_vector0 and i == 0:
            keep[0] = False
        s = torch.where(keep, s + p, s)
    return _tree(s, regime)


def _row_sumsq(v, valid, regime, centre=None):
    """sum of (x - centre)^2 (or x^2): q = fma(d, d, q) element by element"""
    R, it, L, _ = v.shape
    q = torch.zeros(R, L, dtype=F32)
    for i in range(it):
        for k in range(8):
            d = v[:, i, :, k] if centre is None else v[:, i, :, k] - centre[:, None]
            q = torch.where(valid[i], fma32(d, d, q), q)
    return _tree(q, regime)


def emu_layernorm(x, w, b, eps, regime, fault=None):
    """layernorm_kernel / layernorm_warp_kernel in fp32 -> (fp32 value before the rounding, bf16 output as fp32)"""
    x32 = x.float()
    R, cols = x32.shape
    v, valid = _vectors(x32, regime)
    mean = _row_sum(v, valid, regime, drop_vector0=fault == "drop_vector") / cols
    if fault == "single_pass":
        var = _row_sumsq(v, valid, regime) / cols - mean * mean
    else:
        var = _row_sumsq(v, valid, regime, centre=mean) / cols
    e = {"eps_1e-5": 1e-5, "eps_1e-6": 1e-6}.get(fault, eps)
    rstd = rsqrtf(var + torch.tensor(e, dtype=F32))
    d = (x32 - mean[:, None]) * rstd[:, None]
    if fault == "bias_first":
        y = (d + b.float()) * w.float()
    else:
        y = fma32(d, w.float(), b.float())
    out = bf16_rz(y) if fault == "round_toward_zero" else y.to(torch.bfloat16).float()
    return y, out


def emu_rmsnorm(x, w, eps, regime, fault=None):
    """rmsnorm_kernel / rmsnorm_warp_kernel in fp32 -> (fp32 x * rstd before its rounding, bf16 output as fp32)"""
    x32 = x.float()
    R, cols = x32.shape
    v, valid = _vectors(x32, regime)
    e = {"eps_1e-5": 1e-5, "eps_1e-6": 1e-6}.get(fault, eps)
    rstd = rsqrtf(_row_sumsq(v, valid, regime) / cols + torch.tensor(e, dtype=F32))
    t = x32 * rstd[:, None]
    if fault == "no_intermediate_rounding":
        y = t * w.float()
    else:
        y = t.to(torch.bfloat16).float() * w.float()
    out = bf16_rz(y) if fault == "round_toward_zero" else y.to(torch.bfloat16).float()
    return t, out


def check_layernorm(x, w, b, eps, out, regime, max_window=0.01, pre=None):
    """-> (TieErrors, needed ratio max |pre - ref_final| / eps over the elements, when the fp32 value is known)"""
    depth = norm_plan(1 << 20 if regime == "warp" else 1, x.shape[1])["depth"]
    e = TieErrors(max_window)
    ratio = 0.0
    for r0, r1, ref, eps_e in layernorm_reference(x, w, b, eps, depth):
        e.add(out[r0:r1], ref, eps_e, where=f"rows {r0}..")
        if pre is not None:
            ratio = max(ratio, float(((pre[r0:r1].double() - ref).abs() / eps_e).max()))
    return e, ratio


def check_rmsnorm(x, w, eps, out, regime, max_window=0.01, pre=None):
    depth = norm_plan(1 << 20 if regime == "warp" else 1, x.shape[1])["depth"]
    e = TieErrors(max_window)
    ratio = 0.0
    for r0, r1, t, eps_e in rmsnorm_reference(x, eps, depth):
        e.add(out[r0:r1], t, eps_e, then=rmsnorm_then(w), where=f"rows {r0}..")
        if pre is not None:
            ratio = max(ratio, float(((pre[r0:r1].double() - t).abs() / eps_e).max()))
    return e, ratio


def _regimes(cols):
    return ("cta", "warp") if cols <= 2048 else ("cta",)


# ------------------------------------------------------------------------------------------------
# the emulations pass with margin
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cols", LN_WIDTHS)
def test_layernorm_emulation_passes(cols):
    for regime in _regimes(cols):
        for fam in NORM_FAMILIES:
            x, w, b = norm_inputs(fam, 24, cols, seed=cols + len(fam))
            eps = 1e-6 if cols in (1152, 144) else 1e-5
            pre, out = emu_layernorm(x, w, b, eps, regime)
            e, ratio = check_layernorm(x, w, b, eps, out, regime, MAX_WINDOW[fam], pre)
            _record({"name": f"layernorm emulation {regime} {cols} {fam}", "eps_used": float(f"{ratio:.3e}"),
                     **e.summary()})
            e.check(f"layernorm {regime} {cols} {fam}")
            assert e.needed <= NEEDED[fam], f"{regime} {cols} {fam}: a flip needs {e.needed:.2f} of eps"
            assert ratio <= 1.0, f"{regime} {cols} {fam}: the emulation errs by {ratio:.2f} x eps"


@pytest.mark.parametrize("cols", RMS_WIDTHS)
def test_rmsnorm_emulation_passes(cols):
    for regime in _regimes(cols):
        for fam in NORM_FAMILIES:
            x, w, _ = norm_inputs(fam, 24, cols, seed=cols + len(fam), rms=True)
            pre, out = emu_rmsnorm(x, w, 1e-6, regime)
            e, ratio = check_rmsnorm(x, w, 1e-6, out, regime, MAX_WINDOW[fam], pre)
            _record({"name": f"rmsnorm emulation {regime} {cols} {fam}", "eps_used": float(f"{ratio:.3e}"),
                     **e.summary()})
            e.check(f"rmsnorm {regime} {cols} {fam}")
            assert e.needed <= NEEDED[fam], f"{regime} {cols} {fam}: a flip needs {e.needed:.2f} of eps"
            assert ratio <= 1.0, f"{regime} {cols} {fam}: the emulation errs by {ratio:.2f} x eps"


def test_constant_rows_exact():
    """a constant row has x - mean = 0 exactly (its fp32 sum and mean are exact): LayerNorm gives bf16(b); an
    all-zero RMSNorm row gives rsqrt(eps) * 0 = 0"""
    x, w, b = norm_inputs("constant", 8, 1152, seed=1)
    for regime in ("cta", "warp"):
        _, out = emu_layernorm(x, w, b, 1e-6, regime)
        assert torch.equal(out, b.float().expand_as(out))
        z, w2, _ = norm_inputs("constant", 8, 2048, seed=2, rms=True)
        _, o2 = emu_rmsnorm(z, w2, 1e-6, regime)
        assert torch.equal(o2, torch.zeros_like(o2))


# ------------------------------------------------------------------------------------------------
# planted norm faults
# ------------------------------------------------------------------------------------------------
OUTSIDE = "outside their exact-or-tie set"


@pytest.mark.parametrize("fault,fam,eps,regime", [
    ("single_pass", "offset", 1e-6, "cta"),
    ("single_pass", "offset", 1e-6, "warp"),
    ("drop_vector", "random", 1e-6, "cta"),
    ("drop_vector", "random", 1e-6, "warp"),
    ("eps_1e-5", "small", 1e-6, "cta"),      # the projector's eps at a SigLIP call site
    ("eps_1e-6", "small", 1e-5, "cta"),      # and the other way round
    ("bias_first", "random", 1e-6, "cta"),
    ("round_toward_zero", "random", 1e-6, "cta"),
    ("round_toward_zero", "random", 1e-6, "warp"),
])
def test_layernorm_faults_rejected(fault, fam, eps, regime):
    x, w, b = norm_inputs(fam, 64, 1152, seed=7)
    _, out = emu_layernorm(x, w, b, eps, regime, fault=fault)
    e, _ = check_layernorm(x, w, b, eps, out, regime, MAX_WINDOW[fam])
    bad = e.failures()
    _record({"name": f"layernorm fault {fault} {fam} {regime}", "bad": e.bad, **e.summary()})
    assert bad and OUTSIDE in bad[0], (fault, bad)


@pytest.mark.parametrize("fault,fam,regime", [
    ("no_intermediate_rounding", "random", "cta"),
    ("no_intermediate_rounding", "random", "warp"),
    ("eps_1e-5", "small", "cta"),
    ("round_toward_zero", "random", "cta"),
    ("round_toward_zero", "random", "warp"),
])
def test_rmsnorm_faults_rejected(fault, fam, regime):
    x, w, _ = norm_inputs(fam, 64, 2048, seed=8, rms=True)
    _, out = emu_rmsnorm(x, w, 1e-6, regime, fault=fault)
    e, _ = check_rmsnorm(x, w, 1e-6, out, regime, MAX_WINDOW[fam])
    bad = e.failures()
    _record({"name": f"rmsnorm fault {fault} {fam} {regime}", "bad": e.bad, **e.summary()})
    assert bad and OUTSIDE in bad[0], (fault, bad)


def test_checker_rejects_a_generous_eps():
    """an eps four times too large shows as a too-wide window instead of passing quietly"""
    x, w, b = norm_inputs("random", 64, 1152, seed=9)
    _, out = emu_layernorm(x, w, b, 1e-6, "cta")
    e = TieErrors(0.01)
    for r0, r1, ref, eps_e in layernorm_reference(x, w, b, 1e-6, 18):
        e.add(out[r0:r1], ref, eps_e * 2.0 ** 14)
    bad = e.failures()
    assert bad and "tie window covers" in bad[-1], bad


def test_norm_plan_boundaries():
    assert norm_plan(8191, 1152) == dict(regime="cta", chain=8, warp=5, block=5, depth=18)
    assert norm_plan(8192, 1152) == dict(regime="warp", chain=40, warp=5, block=0, depth=45)
    assert norm_plan(8192, 2048) == dict(regime="warp", chain=64, warp=5, block=0, depth=69)
    assert norm_plan(8192, 2056) == dict(regime="cta", chain=16, warp=5, block=5, depth=26)
    assert norm_plan(16470, 3584)["regime"] == "cta"
    assert norm_plan(1, 13824) == dict(regime="cta", chain=56, warp=5, block=5, depth=66)


# ------------------------------------------------------------------------------------------------
# data movement: emulations of the index math, the fp64 references, planted faults
# ------------------------------------------------------------------------------------------------
def emu_s2_merge(tiles, sh, sw, out_bh, out_bw, share_tile=False, fault=None):
    """s2_merge_kernel in fp32: per scale, window [floor(o I / O), ceil((o + 1) I / O)) summed row by row, times
    fl(1 / n), rounded; written to output tile (oy / side) * out_bw + ox / side, channel slot s"""
    n, N, C = tiles.shape
    side = int(round(N ** 0.5))
    ns = len(sh)
    OH, OW = out_bh * side, out_bw * side
    t32 = tiles.float()
    out = torch.empty(out_bh * out_bw, N, ns * C, dtype=F32)
    tile0, t0 = [], 0
    for s in range(ns):
        tile0.append(t0)
        if not share_tile:
            t0 += sh[s] * sw[s]
    if fault == "last_tile0":
        tile0[-1] -= 1
    oy = torch.arange(OH)[:, None].expand(OH, OW)
    ox = torch.arange(OW)[None, :].expand(OH, OW)
    for s in range(ns):
        IH, IW = sh[s] * side, sw[s] * side
        y0, x0 = oy * IH // OH, ox * IW // OW
        if fault == "floor_end":
            y1, x1 = (oy + 1) * IH // OH, (ox + 1) * IW // OW
        else:
            y1, x1 = ((oy + 1) * IH + OH - 1) // OH, ((ox + 1) * IW + OW - 1) // OW
        acc = torch.zeros(OH, OW, C, dtype=F32)
        for dy in range(int((y1 - y0).max())):
            for dx in range(int((x1 - x0).max())):
                y, x = y0 + dy, x0 + dx
                m = (y < y1) & (x < x1)
                yc, xc = y.clamp(max=IH - 1), x.clamp(max=IW - 1)
                tile = (tile0[s] + (yc // side) * sw[s] + xc // side).clamp(min=0)
                tok = (yc % side) * side + xc % side
                acc = torch.where(m[..., None], acc + t32[tile, tok], acc)
        cnt = ((y1 - y0) * (x1 - x0)).to(F32).clamp_min(1)
        val = (acc * (1.0 / cnt)[..., None]).to(torch.bfloat16).float()
        slot = ns - 1 - s if fault == "scale_order" else s
        if fault == "split_transposed":
            otile = (ox // side) * out_bh + oy // side
        else:
            otile = (oy // side) * out_bw + ox // side
        otok = (oy % side) * side + ox % side
        out[otile.reshape(-1), otok.reshape(-1), slot * C:(slot + 1) * C] = val.reshape(-1, C)
    return out


def check_s2(tiles, sh, sw, ob, out, share_tile=False, max_window=0.01):
    ref, eps = s2_merge_reference(tiles, sh, sw, ob[0], ob[1], share_tile)
    assert out.shape == ref.shape, (out.shape, ref.shape)
    return TieErrors(max_window).add(out, ref, eps)


S2_SIDE, S2_C = 8, 16


def _s2_tiles(bs, seed):
    n = 1 + 4 + bs[0] * bs[1]
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, S2_SIDE * S2_SIDE, S2_C, generator=g).to(torch.bfloat16)


@pytest.mark.parametrize("bs,idx", [((3, 4), -1), ((2, 5), -1), ((1, 9), -1), ((5, 6), -1), ((3, 3), 0),
                                    ((4, 3), 1), ((2, 6), 1)])
def test_s2_merge_emulation_passes(bs, idx):
    tiles = _s2_tiles(bs, sum(bs))
    sh, sw = [1, 2, bs[0]], [1, 2, bs[1]]
    ob = tuple(bs) if idx in (-1, 2) else ((1, 1) if idx == 0 else (2, 2))
    out = emu_s2_merge(tiles, sh, sw, *ob)
    e = check_s2(tiles, sh, sw, ob, out)
    _record({"name": f"s2 emulation {bs} idx {idx}", **e.summary()})
    e.check(f"s2 {bs} idx {idx}")


def test_s2_share_tile_emulation_passes():
    tiles = _s2_tiles((1, 1), 3)[:1]
    out = emu_s2_merge(tiles, [1, 1, 1], [1, 1, 1], 1, 1, share_tile=True)
    check_s2(tiles, [1, 1, 1], [1, 1, 1], (1, 1), out, share_tile=True).check("s2 share tile")
    assert torch.equal(out, tiles.float().repeat(1, 1, 3))


@pytest.mark.parametrize("fault,bs,idx", [("floor_end", (3, 4), -1), ("floor_end", (3, 4), 1),
                                          ("scale_order", (3, 4), -1), ("last_tile0", (3, 4), -1),
                                          ("split_transposed", (3, 4), -1), ("split_transposed", (2, 5), -1)])
def test_s2_faults_rejected(fault, bs, idx):
    tiles = _s2_tiles(bs, 11)
    sh, sw = [1, 2, bs[0]], [1, 2, bs[1]]
    ob = tuple(bs) if idx == -1 else (2, 2)
    out = emu_s2_merge(tiles, sh, sw, *ob, fault=fault)
    bad = check_s2(tiles, sh, sw, ob, out).failures()
    assert bad and OUTSIDE in bad[0], (fault, bad)


@pytest.mark.parametrize("bs,idx", [((3, 4), -1), ((3, 3), 0), ((4, 3), 1)])
def test_s2_reference_matches_oracle(bs, idx):
    """the fp64 reference == the oracle's merge_features_for_dynamic_s2 + split_chessboard run in fp32"""
    tiles = _s2_tiles(bs, 5).float()
    feats, nbs = O.merge_features_for_dynamic_s2(tiles, [bs], [448, 896, 1344], idx)
    want = O.split_chessboard(feats[0], *nbs[0]).flatten(2).transpose(1, 2)
    ref, _ = s2_merge_reference(tiles, [1, 2, bs[0]], [1, 2, bs[1]], *nbs[0])
    assert ref.shape == want.shape
    assert float((ref - want.double()).abs().max()) <= 4 * 2.0 ** -24 * float(want.abs().max())


def emu_s2d(x, h, w, r, fault=None):
    """s2d_kernel: out[b, i, j, (q r + p) C + c] = x[b, r i + q, r j + p, c], zero outside; fault
    'border_first': the zero border at the top / left"""
    B, _, C = x.shape
    ho, wo = -(-h // r), -(-w // r)
    pad_y, pad_x = (ho * r - h, wo * r - w) if fault == "border_first" else (0, 0)
    xs = x.view(B, h, w, C)
    out = torch.zeros(B, ho, wo, r, r, C, dtype=x.dtype)
    for q in range(r):
        for p in range(r):
            yi = torch.arange(ho) * r + q - pad_y
            xj = torch.arange(wo) * r + p - pad_x
            my, mx = (yi >= 0) & (yi < h), (xj >= 0) & (xj < w)
            blk = xs[:, yi.clamp(0, h - 1)][:, :, xj.clamp(0, w - 1)]
            out[:, :, :, q, p] = blk * (my[:, None] & mx[None, :])[None, :, :, None]
    return out.reshape(B, ho * wo, r * r * C)


@pytest.mark.parametrize("r", [2, 3])
def test_s2d_emulation_and_border_fault(r):
    x = torch.randn(2, 32 * 32, 16).to(torch.bfloat16)
    want = O.flat_square(x.view(2, 32, 32, 16), r).reshape(2, -1, r * r * 16)
    assert torch.equal(emu_s2d(x, 32, 32, r), want)
    if r == 3:  # 32 -> 11: one zero row / column, at the bottom / right
        assert not torch.equal(emu_s2d(x, 32, 32, r, fault="border_first"), want)


def emu_tsp(x, pt, ph, pw, fault=None):
    """tsp_pool_v8_kernel in fp32: t-sum / pt -> bf16, summed over h, / ph -> bf16, summed over w, / pw -> bf16"""
    T, h, w, C = x.shape
    v = x.float().view(T // pt, pt, h // ph, ph, w // pw, pw, C)
    if fault == "one_rounding":
        acc = torch.zeros(T // pt, h // ph, w // pw, C, dtype=F32)
        for c3 in range(pw):
            for c2 in range(ph):
                for c1 in range(pt):
                    acc = acc + v[:, c1, :, c2, :, c3]
        return (acc / (pt * ph * pw)).to(torch.bfloat16).float()

    def rb(t):
        return t.to(torch.bfloat16).float()
    sw = torch.zeros(T // pt, h // ph, w // pw, C, dtype=F32)
    inner_n, outer_n = (ph, pw) if fault != "hw_swapped" else (pw, ph)
    for a in range(outer_n):
        sh = torch.zeros_like(sw)
        for bb in range(inner_n):
            st = torch.zeros_like(sw)
            for c1 in range(pt):
                c2, c3 = (bb, a) if fault != "hw_swapped" else (a, bb)
                st = st + v[:, c1, :, c2, :, c3]
            sh = sh + rb(st / pt)
        sw = sw + rb(sh / inner_n)
    return rb(sw / outer_n)


TSP_POOLS = [(8, 1, 1), (4, 1, 1), (2, 2, 2), (4, 2, 2), (3, 1, 1), (1, 2, 4)]


@pytest.mark.parametrize("pool", TSP_POOLS)
def test_tsp_emulation_passes_and_matches_oracle(pool):
    """the emulation passes the fp64 reference; so does the oracle's chain of bf16 .mean() calls (what the
    reference computes)"""
    T = 24 if pool[0] == 3 else 16
    x = (torch.randn(T, 8, 8, 64) * 3).to(torch.bfloat16)
    ref, eps = tsp_pool_reference(x, *pool)
    e = TieErrors(0.01).add(emu_tsp(x, *pool), ref, eps)
    _record({"name": f"tsp emulation {pool}", **e.summary()})
    e.check(f"tsp {pool}")
    o = x
    for dim, p in enumerate(pool):
        o = O.tsp_pool(o, p, dim)
    TieErrors(0.01).add(o.float(), ref, eps).check(f"tsp oracle {pool}")


@pytest.mark.parametrize("fault,pool", [("one_rounding", (4, 2, 2)), ("one_rounding", (2, 2, 2)),
                                        ("hw_swapped", (2, 2, 4)), ("hw_swapped", (1, 4, 2))])
def test_tsp_faults_rejected(fault, pool):
    x = (torch.randn(16, 8, 8, 64) * 3).to(torch.bfloat16)
    ref, eps = tsp_pool_reference(x, *pool)
    bad = TieErrors(0.01).add(emu_tsp(x, *pool, fault=fault), ref, eps).failures()
    assert bad and OUTSIDE in bad[0], (fault, bad)


def test_bf16_rne64_is_one_rounding():
    """next to a tie, fp64 -> fp32 -> bf16 rounds twice; bf16_rne64 rounds once"""
    x = torch.tensor([1.0 + 2.0 ** -8 + 2.0 ** -30, 1.0 + 2.0 ** -8 - 2.0 ** -30, -3.0 - 2.0 ** -7 + 2.0 ** -40,
                      0.75, 1.0 + 3 * 2.0 ** -8], dtype=torch.float64)
    want = torch.tensor([1.0 + 2.0 ** -7, 1.0, -3.0, 0.75, 1.0 + 2.0 ** -6], dtype=torch.float64)
    assert torch.equal(bf16_rne64(x), want)
    assert math.isclose(float(bf16_ulp(torch.tensor([1.5]))[0]), 2.0 ** -7)
