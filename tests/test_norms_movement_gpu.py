"""GPU: every LayerNorm, RMSNorm and media data-movement call at its production shape and dispatch regime
(norm.cu, data_movement.cu), against fp64, exact outside bf16 rounding ties (tests.helpers.TieErrors).

Table, from nvila_8b(), nvila_8b_dynamic_s2(), nvila_video_8b(), nvila_lite_3b() and tiny_test_config():
  * LayerNorm: SigLIP's layer_norm1 / layer_norm2 (width 1152, the vision eps) on 1024 B rows for B = 1, 2, 13
    (Lite: 12 tiles + thumbnail), 14 (a square dynamic-S2 image), 35 (a (5, 6) layout), 8, 16 and 64 video
    frames, and 8191 / 8192 rows (both regimes); the projector's ln (eps 1e-5) at 4608 with 256 B rows, 13824
    (dynamic S2) with 256 bh bw rows, Lite's 10368 / 3456 with 121 B rows; the tiny widths; the regime edges
    (8195, 144), (9000, 2048), (8192, 2056).
  * RMSNorm (eps = rms_norm_eps): prefill at 3584 with S in {1, 279, 384, 385, 8000, 16470} and at 2048 with S in
    {1, 144, 8191, 8192, 16470}; the batched engine's slot counts {1, 3, 8, 16}; (8200, 4096) and (8192, 512).
    The residual_add form runs once per regime.
  * data movement, bit for bit (exact-or-tie where the kernel averages): patch_im2col, space_to_depth, s2_merge
    for every block size the dynamic-S2 tiling can produce, chessboard_merge, tsp_pool (vector and scalar kernel),
    embed_splice.
Each case calls the C entry point with an output buffer one row or tile longer than needed, filled with a
sentinel that must survive, and repeats the call, which must give the same bits.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from oracle import vila_oracle as O
from tests.helpers import (NORM_FAMILIES, TieErrors, _record, layernorm_reference, norm_inputs, norm_plan,
                           rmsnorm_reference, rmsnorm_then, s2_merge_reference, tsp_pool_reference)

pytestmark = pytest.mark.gpu

SENT = -3.0e38  # finite bf16 sentinel
MAX_WINDOW = 0.01  # largest tie-window fraction a case may have (tests/test_norms_movement_cpu.py measures it)


def _cfgs():
    from vila_b200.model.configuration import (nvila_8b, nvila_8b_dynamic_s2, nvila_lite_3b, nvila_video_8b,
                                               tiny_test_config)
    return dict(b8=nvila_8b(), s2=nvila_8b_dynamic_s2(), video=nvila_video_8b(), lite=nvila_lite_3b(),
                tiny=tiny_test_config())


def _grids():
    """the dynamic-S2 block sizes: every (cols, rows) grid with 9 <= cols rows <= 12, and (5, 6)"""
    from vila_b200.model.media import target_ratios
    return [g for g in target_ratios(9, 12) if g[0] * g[1] >= 9] + [(5, 6)]


def _norm_table():
    c = _cfgs()
    vis = c["b8"].vision_tower_cfg
    tok = vis.num_patches  # 1024
    C1 = vis.hidden_size
    ln_p = 1e-5  # MultimodalProjector.LN_EPS
    rows = []

    def ln(name, r, cols, eps):
        rows.append(dict(op="layernorm", name=name, rows=r, cols=cols, eps=eps))

    def rms(name, r, cols, eps):
        rows.append(dict(op="rmsnorm", name=name, rows=r, cols=cols, eps=eps))
    for B in (1, 2, c["b8"].num_video_frames, 13, 14, 16, 35, c["video"].num_video_frames):
        ln(f"siglip-B{B}", tok * B, C1, vis.layer_norm_eps)
    for r in (8191, 8192):
        ln(f"siglip-rows{r}", r, C1, vis.layer_norm_eps)
    for B in (1, 2, 64):
        ln(f"proj8b-B{B}", 256 * B, 4 * C1, ln_p)
    C3 = c["s2"].mm_hidden_size  # 3456
    for bh, bw in ((3, 3), (3, 4), (5, 6)):
        ln(f"projs2-{bh}x{bw}", 256 * bh * bw, 4 * C3, ln_p)
    ln("projs2-rows7", 7, 4 * C3, ln_p)
    for B in (1, 13):
        ln(f"lite-ln1-B{B}", 121 * B, 9 * C1, ln_p)
        ln(f"lite-ln2-B{B}", 121 * B, 3 * C1, ln_p)
    tv = c["tiny"].vision_tower_cfg
    ln("tiny-siglip", tv.num_patches * 3, tv.hidden_size, tv.layer_norm_eps)
    for k, w in (("tiny-proj2", 4), ("tiny-proj3a", 9), ("tiny-proj3b", 3), ("tiny-projs2", 12)):
        ln(k, 16 * 3, w * tv.hidden_size, ln_p)
    ln("edge-8195x144", 8195, 144, 1e-6)
    ln("edge-9000x2048", 9000, 2048, 1e-6)
    ln("edge-8192x2056", 8192, 2056, 1e-6)
    l8, ll = c["b8"].llm_cfg, c["lite"].llm_cfg
    for S in (1, 279, 384, 385, 8000, 16470):
        rms(f"8b-S{S}", S, l8.hidden_size, l8.rms_norm_eps)
    for S in (1, 144, 8191, 8192, 16470):
        rms(f"lite-S{S}", S, ll.hidden_size, ll.rms_norm_eps)
    for M in (1, 3, 8, 16):
        rms(f"8b-slots{M}", M, l8.hidden_size, l8.rms_norm_eps)
        rms(f"lite-slots{M}", M, ll.hidden_size, ll.rms_norm_eps)
    rms("edge-8200x4096", 8200, 4096, 1e-6)
    rms("edge-8192x512", 8192, 512, 1e-6)
    rms("edge-33x2048", 33, 2048, 1e-6)
    rms("edge-280x3584", 280, 3584, 1e-6)
    rms("edge-8193x2048", 8193, 2048, 1e-6)
    lt = c["tiny"].llm_cfg
    rms("tiny-S40", 40, lt.hidden_size, lt.rms_norm_eps)
    for r in rows:
        r.update(norm_plan(r["rows"], r["cols"]))
        r["id"] = f"{r['op']}-{r['name']}-{r['rows']}x{r['cols']}"
    return rows


NORM_TABLE = _norm_table()
FAMILY_MAX_ROWS = 16470  # the offset / outlier / small families run on every case up to this many rows


def _lib():
    from vila_b200 import _lib as L, ops
    ops.ensure_workspace("cuda")
    return L


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def _sent(shape, extra_rows=1):
    return torch.full((shape[0] + extra_rows, *shape[1:]), SENT, dtype=torch.bfloat16, device="cuda")


def _untouched(buf, n, what):
    tail = buf[n:]
    assert bool((tail == SENT).all()), f"{what}: the kernel wrote past its output"


def _layernorm(x, w, b, eps):
    L = _lib()
    rows, cols = x.shape
    out = _sent((rows, cols))
    L.check(L.load().vila_layernorm(_p(x), _p(w), _p(b), _p(out), rows, cols, eps, _stream()), "vila_layernorm")
    return out


def _rmsnorm(x, w, eps, res=None):
    L = _lib()
    rows, cols = x.shape
    out = _sent((rows, cols))
    L.check(L.load().vila_rmsnorm(_p(x), _p(res), _p(w), _p(out), rows, cols, eps, _stream()), "vila_rmsnorm")
    return out


def _check_norm(case, fam, x, w, b, out):
    e = TieErrors(MAX_WINDOW)
    if case["op"] == "layernorm":
        for r0, r1, ref, eps in layernorm_reference(x, w, b, case["eps"], case["depth"]):
            e.add(out[r0:r1], ref, eps, where=f"rows {r0}..")
    else:
        for r0, r1, t, eps in rmsnorm_reference(x, case["eps"], case["depth"]):
            e.add(out[r0:r1], t, eps, then=rmsnorm_then(w), where=f"rows {r0}..")
    return e


@pytest.mark.parametrize("case", NORM_TABLE, ids=[c["id"] for c in NORM_TABLE])
def test_norm(cuda, case):
    rows, cols = case["rows"], case["cols"]
    fams = NORM_FAMILIES if rows <= FAMILY_MAX_ROWS else ("random",)
    for k, fam in enumerate(fams):
        x, w, b = norm_inputs(fam, rows, cols, seed=rows * 7 + cols + k, device="cuda",
                              rms=case["op"] == "rmsnorm")
        x0 = x.clone()
        if case["op"] == "layernorm":
            out = _layernorm(x, w, b, case["eps"])
            again = _layernorm(x, w, b, case["eps"])
        else:
            out = _rmsnorm(x, w, case["eps"])
            again = _rmsnorm(x, w, case["eps"])
        torch.cuda.synchronize()
        _untouched(out, rows, case["id"])
        assert torch.equal(out, again), f"{case['id']} {fam}: a repeat call gave different bits"
        assert torch.equal(x, x0), f"{case['id']} {fam}: the input was modified"
        e = _check_norm(case, fam, x, w, b, out[:rows])
        _record({"name": f"norm {case['id']} {fam}", "regime": case["regime"], "depth": case["depth"],
                 **e.summary()})
        e.check(f"{case['id']} {fam}")


@pytest.mark.parametrize("op,rows,cols", [("layernorm", 1024, 1152), ("layernorm", 16384, 1152),
                                          ("rmsnorm", 279, 3584), ("rmsnorm", 16470, 2048)])
def test_norm_constant_rows(cuda, op, rows, cols):
    """a constant LayerNorm row gives exactly bf16(b); an all-zero RMSNorm row gives exactly 0, no NaN"""
    x, w, b = norm_inputs("constant", rows, cols, seed=3, device="cuda", rms=op == "rmsnorm")
    if op == "layernorm":
        out = _layernorm(x, w, b, 1e-6)[:rows]
        assert torch.equal(out, b.expand_as(out))
    else:
        out = _rmsnorm(x, w, 1e-6)[:rows]
        assert torch.equal(out, torch.zeros_like(out))


@pytest.mark.parametrize("rows,cols", [(279, 3584), (16470, 2048)])  # CTA-per-row, warp-per-row
def test_rmsnorm_residual_add(cuda, rows, cols):
    """the residual_add form of the C ABI (no call site uses it): x_inout becomes bf16(x + r) bit for bit and the
    output normalises that"""
    x, w, _ = norm_inputs("random", rows, cols, seed=5, device="cuda", rms=True)
    r, _, _ = norm_inputs("outlier", rows, cols, seed=6, device="cuda", rms=True)
    xs = (x.float() + r.float()).to(torch.bfloat16)
    xi = x.clone()
    out = _rmsnorm(xi, w, 1e-6, res=r)
    torch.cuda.synchronize()
    _untouched(out, rows, "rmsnorm residual")
    assert torch.equal(xi, xs)
    case = dict(op="rmsnorm", eps=1e-6, **norm_plan(rows, cols))
    e = _check_norm(case, "random", xs, w, None, out[:rows])
    _record({"name": f"rmsnorm residual_add {rows}x{cols}", "regime": case["regime"], **e.summary()})
    e.check(f"rmsnorm residual_add {rows}x{cols}")


def test_norm_coverage():
    """the table holds the named production shapes and both regimes of each norm"""
    ids = {(c["op"], c["rows"], c["cols"]) for c in NORM_TABLE}
    for need in [("layernorm", 1024, 1152), ("layernorm", 65536, 1152), ("layernorm", 8191, 1152),
                 ("layernorm", 8192, 1152), ("layernorm", 16384, 4608), ("layernorm", 7, 13824),
                 ("layernorm", 121, 3456), ("layernorm", 8195, 144), ("layernorm", 9000, 2048),
                 ("layernorm", 8192, 2056), ("layernorm", 256, 4608), ("layernorm", 16384, 1152),
                 ("rmsnorm", 16470, 3584), ("rmsnorm", 8192, 2048), ("rmsnorm", 8191, 2048), ("rmsnorm", 1, 3584),
                 ("rmsnorm", 8200, 4096), ("rmsnorm", 8192, 512), ("rmsnorm", 33, 2048), ("rmsnorm", 16, 3584)]:
        assert need in ids, need
    for op in ("layernorm", "rmsnorm"):
        assert {c["regime"] for c in NORM_TABLE if c["op"] == op} == {"cta", "warp"}, op
    _record({"name": "norm coverage", "cases": len(NORM_TABLE),
             "regimes": {c["id"]: c["regime"] for c in NORM_TABLE}})


# ------------------------------------------------------------------------------------------------
# data movement
# ------------------------------------------------------------------------------------------------
def _bf(shape, seed, scale=1.0):
    """seeded N(0, scale^2) bf16 tensor, drawn in pieces of 2^26 elements (no fp32 copy of a large table)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty(shape, dtype=torch.bfloat16, device="cuda")
    flat = out.view(-1)
    step = 1 << 26
    for i in range(0, flat.numel(), step):
        n = min(step, flat.numel() - i)
        flat[i:i + n] = (torch.randn(n, device="cuda", generator=g) * scale).to(torch.bfloat16)
    return out


def test_patch_im2col(cuda):
    """B = 1, 14 and 64 images of 448 x 448: k_pad 592, columns 588..591 zero"""
    L = _lib()
    for B in (1, 14, 64):
        px = _bf((B, 3, 448, 448), B)
        rows = B * 32 * 32
        out = _sent((rows, 592))
        L.check(L.load().vila_patch_im2col(_p(px), _p(out), B, 3, 448, 448, 14, 592, _stream()), "im2col")
        again = out.clone()
        L.check(L.load().vila_patch_im2col(_p(px), _p(again), B, 3, 448, 448, 14, 592, _stream()), "im2col")
        torch.cuda.synchronize()
        _untouched(out, rows, f"im2col B={B}")
        assert torch.equal(out, again), f"B={B}: a repeat call gave different bits"
        ref = F.unfold(px.float(), kernel_size=14, stride=14).transpose(1, 2).reshape(-1, 588)
        assert torch.equal(out[:rows, :588].float(), ref), f"B={B}"
        assert bool((out[:rows, 588:] == 0).all()), f"B={B}: columns 588..591 must be zero"
        del px, out, again, ref


S2D_CASES = [(1, 32, 32, 1152, 2), (64, 32, 32, 1152, 2), (14, 32, 32, 1152, 3), (1, 32, 32, 1152, 3),
             (12, 32, 32, 3456, 2), (30, 32, 32, 3456, 2),
             (2, 27, 27, 64, 2), (2, 27, 27, 64, 3), (2, 5, 7, 64, 2)]  # odd borders, a non-square map


@pytest.mark.parametrize("B,h,w,C,r", S2D_CASES)
def test_space_to_depth(cuda, B, h, w, C, r):
    L = _lib()
    x = _bf((B, h * w, C), B + r + h)
    ho, wo = -(-h // r), -(-w // r)
    out = _sent((B, ho * wo, r * r * C))
    L.check(L.load().vila_space_to_depth(_p(x), _p(out), B, h, w, C, r, _stream()), "space_to_depth")
    torch.cuda.synchronize()
    _untouched(out, B, "space_to_depth")
    ref = O.flat_square(x.view(B, h, w, C), r).reshape(B, ho * wo, r * r * C)
    assert torch.equal(out[:B], ref)


def _s2_call(tiles, sh, sw, ob, share=False):
    L = _lib()
    n, N, Cc = tiles.shape
    out = _sent((ob[0] * ob[1], N, len(sh) * Cc))
    a = (C.c_int * len(sh))(*sh)
    b = (C.c_int * len(sw))(*sw)
    L.check(L.load().vila_s2_merge(_p(tiles), _p(out), 32, Cc, len(sh), a, b, ob[0], ob[1], 1 if share else 0,
                                   _stream()), "s2_merge")
    return out


S2_CASES = [(g, -1) for g in _grids()] + [((3, 4), 0), ((3, 4), 1), ((5, 6), 0), ((2, 6), 1), ((1, 9), 1)]


@pytest.mark.parametrize("bs,idx", S2_CASES, ids=[f"{b[0]}x{b[1]}-idx{i}" for b, i in S2_CASES])
def test_s2_merge(cuda, bs, idx):
    ratios = [1, 2, 3]  # s2_scales (448, 896, 1344) / 448
    sh, sw = ratios[:-1] + [bs[0]], ratios[:-1] + [bs[1]]
    ob = tuple(bs) if idx == -1 else (ratios[idx], ratios[idx])
    tiles = _bf((1 + 4 + bs[0] * bs[1], 1024, 1152), bs[0] * 16 + bs[1])
    out = _s2_call(tiles, sh, sw, ob)
    again = _s2_call(tiles, sh, sw, ob)
    torch.cuda.synchronize()
    n = ob[0] * ob[1]
    _untouched(out, n, "s2_merge")
    assert torch.equal(out, again)
    ref, eps = s2_merge_reference(tiles, sh, sw, ob[0], ob[1])
    e = TieErrors(MAX_WINDOW).add(out[:n], ref, eps)
    _record({"name": f"s2_merge {bs} idx {idx}", **e.summary()})
    e.check(f"s2_merge {bs} idx {idx}")


def test_s2_merge_share_tile(cuda):
    """block_size None: one tile, its features repeated over the scales"""
    tiles = _bf((1, 1024, 1152), 77)
    out = _s2_call(tiles, [1, 1, 1], [1, 1, 1], (1, 1), share=True)
    torch.cuda.synchronize()
    _untouched(out, 1, "s2_merge share")
    f1, _ = O.merge_features_for_dynamic_s2(tiles, [None], [448, 896, 1344], -1)
    assert torch.equal(out[:1], f1[0].flatten(2).transpose(1, 2))


@pytest.mark.parametrize("bs", _grids(), ids=[f"{b[0]}x{b[1]}" for b in _grids()])
def test_chessboard_merge(cuda, bs):
    L = _lib()
    bh, bw = bs
    proj = _bf((bh * bw, 256, 3584), bh * 7 + bw)
    out = _sent((bh * 16 * bw * 16, 3584))
    L.check(L.load().vila_chessboard_merge(_p(proj), _p(out), bh, bw, 16, 3584, _stream()), "chessboard_merge")
    torch.cuda.synchronize()
    n = bh * bw * 256
    _untouched(out, n, "chessboard_merge")
    assert torch.equal(out[:n], O.merge_chessboard(proj, bh, bw)[0].flatten(1).transpose(0, 1))


def _tsp_call(x, pool):
    L = _lib()
    T, h, w, Cc = x.shape
    pt, ph, pw = pool
    out = _sent((T // pt, h // ph, w // pw, Cc))
    L.check(L.load().vila_tsp_pool(_p(x), _p(out), T, h, w, Cc, pt, ph, pw, _stream()), "tsp_pool")
    return out


TSP_POOLS = [(8, 1, 1), (4, 1, 1), (2, 2, 2), (3, 1, 1), (4, 2, 2), (1, 1, 1)]


def test_tsp_pool(cuda):
    """64 frames of 16 x 16 x 3584 (63 for the pool of 3) through every pool of TSP_POOLS, on both kernels: the
    vector one on an aligned input, the scalar one through a view offset by one element; they must give the
    same bits"""
    flat = _bf((64 * 256 * 3584 + 8,), 21, scale=3.0)
    for pool in TSP_POOLS:
        T = 63 if pool[0] == 3 else 64
        x = flat[:T * 256 * 3584].view(T, 16, 16, 3584)
        x_odd = flat[1:T * 256 * 3584 + 1].view(T, 16, 16, 3584)  # 2-byte aligned: the scalar kernel
        x_odd_copy = x_odd.clone()  # the same values, aligned: the vector kernel
        n = T // pool[0]
        outs = []
        for inp in (x, x_odd, x_odd_copy):
            o = _tsp_call(inp, pool)
            torch.cuda.synchronize()
            _untouched(o, n, f"tsp_pool {pool}")
            outs.append(o[:n])
        assert torch.equal(outs[1], outs[2]), f"{pool}: the scalar kernel differs from the vector kernel"
        assert torch.equal(outs[0], _tsp_call(x, pool)[:n]), f"{pool}: a repeat call gave different bits"
        ref, eps = tsp_pool_reference(x, *pool)
        e = TieErrors(MAX_WINDOW).add(outs[0], ref, eps)
        _record({"name": f"tsp_pool {pool}", **e.summary()})
        e.check(f"tsp_pool {pool}")
        del x_odd_copy, outs, ref, eps


def test_embed_splice(cuda):
    """the 8B [152064, 3584] and Lite [151936, 2048] tables: 16,518 source rows with 16,448 media rows, indices 0,
    V - 1, -1 and -n_media; then the batched engine's text-only form (media None)"""
    L = _lib()
    for V, H in ((152064, 3584), (151936, 2048)):
        table = _bf((V, H), V)
        n_media = 16448
        media = _bf((n_media, H), H)
        g = torch.Generator(device="cuda").manual_seed(1)
        text = torch.randint(0, V, (70,), device="cuda", generator=g, dtype=torch.int32)
        text[:4] = torch.tensor([0, V - 1, 0, V - 1], dtype=torch.int32)
        src = torch.cat([text[:35], -1 - torch.arange(n_media, device="cuda", dtype=torch.int32), text[35:]])
        src[40], src[41] = -1, -n_media  # repeated media rows: first and last
        assert src.numel() == 16518
        for med, s in ((media, src), (None, text)):
            out = _sent((s.numel(), H))
            L.check(L.load().vila_embed_splice(_p(table), _p(med), _p(s), _p(out), s.numel(), H, _stream()),
                    "embed_splice")
            torch.cuda.synchronize()
            _untouched(out, s.numel(), f"embed_splice {V}x{H}")
            sl = s.long()
            ref = torch.where((sl >= 0)[:, None], table[sl.clamp(min=0)],
                              media[(-1 - sl).clamp(min=0)] if med is not None else table[0:1])
            assert torch.equal(out[:s.numel()], ref), f"{V}x{H} media={med is not None}"
        del table, media, out, ref


# ------------------------------------------------------------------------------------------------
# call census: the table is the set of calls the model makes
# ------------------------------------------------------------------------------------------------
MOVEMENT_OPS = ("patch_im2col", "space_to_depth", "s2_merge", "chessboard_merge", "tsp_pool", "embed_splice")


def test_call_census(cuda, monkeypatch):
    """every ops.layernorm / ops.rmsnorm call of the tiny model (one forward per projector type, a dynamic-S2 encode,
    a TSP video encode, a prefill with logits_from_hidden, a continuous-batching decode) has an (op, width, eps) of
    the table: the vision eps at vision width, 1e-5 at projector widths, rms_norm_eps for RMSNorm; and every
    data-movement op of the table runs.  A fresh model per run: encode_images caches a CUDA graph per shape."""
    from vila_b200 import ops
    from vila_b200.model import LlavaLlamaModel, tiny_test_config
    calls = []

    def wrap(name):
        fn = getattr(ops, name)

        def rec(*a, **k):
            if name == "layernorm":
                calls.append(("layernorm", a[0].shape[-1], float(a[3])))
            elif name == "rmsnorm":
                calls.append(("rmsnorm", a[0].shape[-1], float(a[2])))
            else:
                calls.append((name,))
            return fn(*a, **k)
        monkeypatch.setattr(ops, name, rec)
    for name in ("layernorm", "rmsnorm") + MOVEMENT_OPS:
        wrap(name)
    g = torch.Generator().manual_seed(0)

    def px(n, size):
        return torch.randn(n, 3, size, size, generator=g).to(torch.bfloat16).cuda()
    for proj in ("mlp_downsample", "mlp_downsample_2x2_fix", "mlp_downsample_3x3_fix"):
        cfg = tiny_test_config(projector=proj)
        LlavaLlamaModel(cfg, device="cuda").init_random(1).encode_images(px(2, 112))
    cfg = tiny_test_config(dynamic_s2=True, image_size=56)
    LlavaLlamaModel(cfg, device="cuda").init_random(2).encode_images(px(1 + 4 + 6 + 1, 56),
                                                                     block_sizes=[(2, 3), None])
    cfg = tiny_test_config(projector="mlp_downsample_2x2_fix", video_encoder="tsp",
                           tsp_pool_sizes=((4, 1, 1), (2, 2, 2)))
    model = LlavaLlamaModel(cfg, device="cuda").init_random(3)
    model.encoders["video"]([px(8, 112)], {})
    llm = model.llm
    emb = (torch.randn(40, cfg.hidden_size, generator=g) * 0.05).to(torch.bfloat16).cuda()
    hid = llm.prefill_hidden(emb, llm.new_cache(256))
    llm.logits_from_hidden(hid[-1:])
    ids = torch.tensor([[5, 6, cfg.image_token_id, 7, 8]])
    model.generate_batch([{"input_ids": ids, "media": {"image": [px(1, 112)[0]]}},
                          {"input_ids": ids[:, :2], "media": None}],
                         max_new_tokens=3, slots=2, max_tokens_per_slot=256, eos_token_id=[])
    torch.cuda.synchronize()
    table = {(c["op"], c["cols"], c["eps"]) for c in NORM_TABLE}
    norms = {c for c in calls if len(c) == 3}
    vis, llm_cfg = cfg.vision_tower_cfg, cfg.llm_cfg
    proj_widths = {k * m * vis.hidden_size for k in (3, 4, 9) for m in (1, len(cfg.s2_scales))}
    for op, cols, eps in sorted(norms):
        assert (op, cols, eps) in table, f"{op} at width {cols}, eps {eps} is not a row of the table"
        if op == "rmsnorm":
            assert cols == llm_cfg.hidden_size and eps == llm_cfg.rms_norm_eps
        elif cols == vis.hidden_size:
            assert eps == vis.layer_norm_eps
        else:
            assert cols in proj_widths and eps == 1e-5, (cols, eps)
    ran = {c[0] for c in calls}
    assert set(MOVEMENT_OPS) <= ran, set(MOVEMENT_OPS) - ran
    _record({"name": "norm call census", "calls": len(calls), "norm_calls": sorted(norms),
             "ops": sorted(ran)})
