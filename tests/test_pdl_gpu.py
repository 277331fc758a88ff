"""The programmatic-dependent-launch (PDL) contract of every C-ABI entry point, against a late-finishing producer (GPU).

Every vila_* kernel is launched with PDL and lets its successor become resident while it still runs, so a kernel may
start before its predecessor has finished.  It is correct only if it reads nothing the predecessor produces, and writes
nothing the predecessor still reads, before its griddepcontrol.wait.  A torch kernel never lets its successor in early,
so the per-kernel suites (which launch after torch ops or a synchronize) cannot see a breach; only the decoders' CUDA
graphs and the prefill / vision chains, where the predecessor is one of our kernels, can.

Each row of CASES is one consumer at one production shape and regime, with its contract: the arguments that are
STATIC (parameters, allowed to be read before the wait) and those that are PRODUCED (read only after it), plus the
buffers it writes.  Per case:
  1. reference: the consumer on fully prepared inputs after a synchronize;
  2. late run: every produced input holds poison (in range: another permutation, position, token, finite values) and
     every output a sentinel; vila_test_pdl_late (which triggers its dependents at once, spins DELAY_NS, snapshots the
     outputs and then writes the true inputs) is launched and then, with nothing in between, the consumer's recorded
     C call.  The outputs must equal the reference bit for bit (no early read) and the snapshot the sentinel (no early
     write);
  3. the same pair captured in a CUDA graph and replayed once gives the same bits;
  4. a torch.profiler trace of the eager pair shows nothing between producer and consumer; whether the consumer
     started before the producer ended is recorded.
test_probe_sees_the_window is the positive control: without a window the whole file would pass vacuously.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Tuple

import pytest
import torch

from tests.helpers import _record, dispatch_flavour

pytestmark = pytest.mark.gpu

DELAY_NS = 200_000  # the producer's spin: far longer than a launch, far shorter than a test
PAGE = 128


# ------------------------------------------------------------------------------------------------
# recording one C call of an ops wrapper, to replay it later with nothing in between
# ------------------------------------------------------------------------------------------------
class _Recorder:
    def __init__(self, lib):
        self.lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self.lib, name)
        if name in ("vila_last_error", "vila_set_workspace", "vila_device_info"):
            return fn

        def rec(*args):
            self.calls.append((name, fn, args))
            return 0
        return rec


def record(fn: Callable):
    """Run an ops wrapper with the library swapped for a recorder: -> (entry point, replay(), wrapper's result).  The
    wrapper marshals the arguments exactly as production does; replay() issues that one C call on the stream that was
    current while recording, and checks its return code."""
    from vila_b200 import _lib
    real = _lib.load()
    rec = _Recorder(real)
    orig = _lib.load
    _lib.load = lambda: rec
    try:
        ret = fn()
    finally:
        _lib.load = orig
    assert len(rec.calls) == 1, [c[0] for c in rec.calls]
    name, f, args = rec.calls[0]

    def replay():
        rc = f(*args)
        assert rc == 0, (name, rc, real.vila_last_error())
    return name, replay, ret


# ------------------------------------------------------------------------------------------------
# the case table
# ------------------------------------------------------------------------------------------------
@dataclass
class Case:
    id: str
    entry: str = ""
    regime: str = ""
    launch: Optional[Callable] = None
    static: Dict[str, torch.Tensor] = field(default_factory=dict)
    produced: Dict[str, Tuple[torch.Tensor, Optional[torch.Tensor]]] = field(default_factory=dict)  # (buffer, poison)
    outputs: Dict[str, Tuple[torch.Tensor, Optional[torch.Tensor]]] = field(default_factory=dict)  # (buffer, sentinel)
    inout: Dict[str, Tuple[torch.Tensor, Optional[torch.Tensor]]] = field(default_factory=dict)  # (buffer, poison)


_GEN = [0]


def _g():
    _GEN[0] += 1
    return torch.Generator(device="cuda").manual_seed(1000 + _GEN[0])


def bf(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=_g()) * scale).to(torch.bfloat16)


def f32(*shape, scale=1.0):
    return torch.randn(*shape, device="cuda", generator=_g()) * scale


def _poison_like(t: torch.Tensor) -> torch.Tensor:
    """finite values of t's type that differ from t's (integer buffers name their in-range poison explicitly)"""
    if t.dtype in (torch.bfloat16, torch.float16, torch.float32):
        s = max(float(t.float().abs().max()), 1.0)
        return (torch.randn(t.shape, device=t.device, generator=_g()) * s * 0.5).to(t.dtype)
    if t.dtype == torch.float8_e4m3fn:
        return (torch.randn(t.shape, device=t.device, generator=_g()) * 64).to(t.dtype)
    if t.dtype == torch.uint8:
        return torch.randint(0, 256, t.shape, device=t.device, generator=_g(), dtype=torch.int32).to(torch.uint8)
    raise AssertionError(f"an integer produced buffer of {t.dtype} needs an explicit in-range poison")


def _sentinel_like(t: torch.Tensor) -> torch.Tensor:
    if t.dtype in (torch.bfloat16, torch.float16, torch.float32):
        return torch.full_like(t, -77.0)
    if t.dtype == torch.float8_e4m3fn:
        return torch.full(t.shape, -3.0, device=t.device).to(t.dtype)
    if t.dtype == torch.uint8:
        return torch.full_like(t, 0xA5)
    return torch.full_like(t, -5)


def _bytes(t: torch.Tensor) -> torch.Tensor:
    assert t.is_contiguous()
    return t.view(-1).view(torch.uint8) if t.element_size() == 1 else t.reshape(-1).view(torch.uint8)


def _page_tables(n_pages: int, rows: int, per_row: int, seed: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """-> (page table, poison): two different valid assignments of distinct pages to `rows` rows of `per_row` pages"""
    g = torch.Generator().manual_seed(seed)
    a = torch.randperm(n_pages, generator=g)[:rows * per_row].view(rows, per_row)
    b = torch.randperm(n_pages, generator=g)[:rows * per_row].view(rows, per_row)
    if torch.equal(a, b):
        b = a.roll(1, dims=1)
    return a.to(torch.int32).cuda(), b.to(torch.int32).cuda()


def _roll_rows(t: torch.Tensor) -> torch.Tensor:
    """t with its rows rotated by one (any dtype: e4m3 has no torch.roll)"""
    return torch.roll(t.view(torch.uint8), 1, 0).view(t.dtype)


def _inv_freq(D=128, theta=1e6):
    return (1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.float32) / D))).cuda()


def _ops():
    from vila_b200 import ops
    ops.ensure_workspace("cuda")
    return ops


# ---- projections ------------------------------------------------------------------------------
# (vila_linear_cfg code, M, N, K): one production shape per gemm_bf16 regime; "auto" runs vila_linear itself on the
# shape dispatch_flavour maps to that regime
LINEAR_ROWS = [
    ("skinny", 3000, 279, 3584, 3584),      # Qwen2 o_proj at a one-image prompt (small-M path)
    ("skinny-pair", 3001, 279, 4608, 3584),  # q/k/v at a one-image prompt, W multicast to a CTA pair
    ("tile128", 128, 1024, 1152, 1152),     # SigLIP q/k/v/out_proj of one 448^2 tile
    ("tile256", 256, 4096, 4304, 1152),     # SigLIP fc1 over four tiles
    ("stream-k", 1128, 279, 3584, 18944),   # Qwen2 down_proj at a one-image prompt
    ("pair", 4128, 1024, 4304, 1152),       # CTA-pair tiles, W multicast
    ("split-k2", 5128, 256, 1152, 4304),    # SigLIP fc2, few tiles, long K
    ("auto", None, 1000, 3584, 3584),       # vila_linear's own dispatch at S = 1000
]


def case_linear(label, code, M, N, K, static_w):
    ops = _ops()
    x, w = bf(M, K), bf(N, K, scale=1 / math.sqrt(K))
    bias, res = bf(N), bf(M, N)
    out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    name, launch, _ = record(lambda: ops.linear(x, w, bias, residual=res, out=out, block_n=code, static_w=static_w))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    regime = f"{label}" + (f" (dispatch {dispatch_flavour(M, N, K, sms, 96 << 20)})" if code is None else "")
    c = Case(f"linear-{label}-{'static' if static_w else 'produced'}_w", name, regime, launch,
             produced={"x": (x, None), "bias": (bias, None), "residual": (res, None)}, outputs={"out": (out, None)})
    if static_w:
        c.static["w"] = w
    else:
        c.produced["w"] = (w, None)
    return c


def case_linear_inplace_residual():
    """the decoder-layer form: out aliases the residual stream (o_proj / down_proj of a prefill)"""
    ops = _ops()
    M, N, K = 279, 3584, 3584
    x, w, y = bf(M, K), bf(N, K, scale=1 / math.sqrt(K)), bf(M, N)
    name, launch, _ = record(lambda: ops.linear(x, w, residual=y, out=y, block_n=3000, static_w=True))
    return Case("linear-residual-in-place", name, "skinny, out == residual", launch, static={"w": w},
                produced={"x": (x, None)}, inout={"y": (y, None)})


def case_qkv_rope(static_w):
    ops = _ops()
    M, K, Hq, Hkv, D = 279, 3584, 28, 4, 128
    N = (Hq + 2 * Hkv) * D
    x, w, bias = bf(M, K), bf(N, K, scale=1 / math.sqrt(K)), bf(N)
    p0 = 77
    pos = torch.arange(p0, p0 + M, dtype=torch.int32, device="cuda")
    tab = ops.rope_table(pos, D, _inv_freq(D))
    n_pages = 8
    pt, pt_poison = _page_tables(n_pages, 1, (p0 + M + PAGE - 1) // PAGE, 3)
    pt, pt_poison = pt.view(-1), pt_poison.view(-1)
    kp = torch.zeros(n_pages, PAGE, Hkv, D, dtype=torch.bfloat16, device="cuda")
    vp = torch.zeros_like(kp)
    out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    torch.cuda.synchronize()
    name, launch, got = record(lambda: ops.linear_qkv_rope(x, w, bias, tab, Hq, Hkv, D, kp, vp, pt, p0,
                                                           static_w=static_w))
    c = Case(f"linear_qkv_rope-{'static' if static_w else 'produced'}_w", name, "small-M GEMM + table RoPE + append",
             launch, produced={"x": (x, None), "bias": (bias, None), "rope_table": (tab, None), "page_table": (pt, pt_poison)},
             outputs={"qkv": (got, None), "k_pool": (kp, None), "v_pool": (vp, None)})
    if static_w:
        c.static["w"] = w
    else:
        c.produced["w"] = (w, None)
    return c


# ---- attention ---------------------------------------------------------------------------------
def case_fmha_vit():
    ops = _ops()
    S, H, D = 1024, 16, 72  # SigLIP: one 448^2 tile, 16 heads of 72
    qkv = bf(S, 3, H, D)
    out = torch.empty(S, H, D, dtype=torch.bfloat16, device="cuda")
    name, launch, _ = record(lambda: ops.fmha(qkv[:, 0], qkv[:, 1], qkv[:, 2], B=1, Sq=S, Sk=S, causal=False,
                                              scale=D ** -0.5, out=out))
    return Case("fmha-vit-dense", name, "dense, D=72", launch, produced={"qkv": (qkv, None)}, outputs={"o": (out, None)})


def case_fmha_paged():
    ops = _ops()
    Sq, p0, Hq, Hkv, D = 279, 77, 28, 4, 128
    Sk = p0 + Sq
    n_pages = 6
    pt, pt_poison = _page_tables(n_pages, 1, (Sk + PAGE - 1) // PAGE, 5)
    q = bf(Sq, Hq, D)
    kp, vp = bf(n_pages, PAGE, Hkv, D), bf(n_pages, PAGE, Hkv, D)
    out = torch.empty(Sq, Hq, D, dtype=torch.bfloat16, device="cuda")
    name, launch, _ = record(lambda: ops.fmha(q, kp, vp, B=1, Sq=Sq, Sk=Sk, causal=True, scale=D ** -0.5, out=out,
                                              page_table=pt))
    return Case("fmha-causal-paged", name, "causal GQA, paged K/V", launch,
                produced={"q": (q, None), "k_pool": (kp, None), "v_pool": (vp, None), "page_table": (pt, pt_poison)},
                outputs={"o": (out, None)})


# ---- norms ---------------------------------------------------------------------------------------
def case_layernorm(rows, cols, regime):
    ops = _ops()
    x, w, b = bf(rows, cols), bf(cols), bf(cols)
    name, launch, out = record(lambda: ops.layernorm(x, w, b, 1e-6))
    return Case(f"layernorm-{rows}x{cols}", name, regime, launch,
                produced={"x": (x, None), "weight": (w, None), "bias": (b, None)}, outputs={"out": (out, None)})


def case_rmsnorm(rows, cols, residual, regime):
    ops = _ops()
    x, w = bf(rows, cols), bf(cols)
    r = bf(rows, cols) if residual else None
    name, launch, out = record(lambda: ops.rmsnorm(x, w, 1e-6, residual_add=r))
    c = Case(f"rmsnorm-{rows}x{cols}{'-residual_add' if residual else ''}", name, regime, launch,
             produced={"weight": (w, None)}, outputs={"out": (out, None)})
    if residual:
        c.produced["residual_add"] = (r, None)
        c.inout["x_inout"] = (x, None)
    else:
        c.produced["x"] = (x, None)
    return c


# ---- data movement -------------------------------------------------------------------------------
def case_im2col():
    ops = _ops()
    px = bf(1, 3, 448, 448)
    name, launch, out = record(lambda: ops.patch_im2col(px, 14, 592))
    return Case("patch_im2col-448", name, "one 448^2 tile", launch, produced={"pixels": (px, None)},
                outputs={"out": (out, None)})


def case_space_to_depth():
    ops = _ops()
    x = bf(1, 32 * 32, 1152)
    name, launch, out = record(lambda: ops.space_to_depth(x, 32, 32, 2))
    return Case("space_to_depth-2x2", name, "flat_square_2x2", launch, produced={"x": (x, None)},
                outputs={"out": (out, None)})


def case_s2_merge():
    ops = _ops()
    tiles = bf(1 + 4 + 6, 1024, 1152)  # dynamic S2, scales 448 / 896 and a 2x3 grid
    name, launch, out = record(lambda: ops.s2_merge(tiles, [1, 2, 2], [1, 2, 3], 2, 3))
    return Case("s2_merge-2x3", name, "dynamic S2 merge", launch, produced={"tiles": (tiles, None)},
                outputs={"out": (out, None)})


def case_chessboard():
    ops = _ops()
    tiles = bf(2 * 3, 256, 3584)
    name, launch, out = record(lambda: ops.chessboard_merge(tiles, 2, 3))
    return Case("chessboard_merge-2x3", name, "projected tiles", launch, produced={"tiles": (tiles, None)},
                outputs={"out": (out, None)})


def case_tsp(C_):
    ops = _ops()
    x = bf(8, 16, 16, C_)
    name, launch, out = record(lambda: ops.tsp_pool(x, 4, 2, 2))
    return Case(f"tsp_pool-C{C_}", name, "vector" if C_ % 8 == 0 else "scalar", launch, produced={"x": (x, None)},
                outputs={"out": (out, None)})


def case_resize():
    from vila_b200 import _lib
    from vila_b200.ops import _bicubic_tables
    H, W, ow, oh, tile = 375, 500, 896, 448, 448
    src = torch.randint(0, 256, (H, W, 3), dtype=torch.int32, device="cuda", generator=_g()).to(torch.uint8)
    kx, bx, cx = _bicubic_tables(W, ow, src.device)
    ky, by, cy = _bicubic_tables(H, oh, src.device)
    cx, bx, cy, by = cx.clone(), bx.clone(), cy.clone(), by.clone()
    tmp = torch.empty(H, ow, 3, dtype=torch.uint8, device="cuda")
    out = torch.empty(2, 3, tile, tile, dtype=torch.bfloat16, device="cuda")
    args = (src.data_ptr(), H, W, ow, oh, cx.data_ptr(), bx.data_ptr(), kx, cy.data_ptr(), by.data_ptr(), ky,
            tmp.data_ptr(), out.data_ptr(), tile, 0, 0.5, 0.5)
    lib = _lib.load()

    def launch():
        assert lib.vila_resize_bicubic_tiles(*args, torch.cuda.current_stream().cuda_stream) == 0

    # the filter tables are built on the host once per size and uploaded: read after the wait all the same
    return Case("resize_bicubic_tiles-2x1", "vila_resize_bicubic_tiles", "horizontal then vertical pass", launch,
                produced={"src": (src, None), "coef_x": (cx, torch.roll(cx, 1, 0)), "bounds_x": (bx, torch.roll(bx, 1, 0)),
                          "coef_y": (cy, torch.roll(cy, 1, 0)), "bounds_y": (by, torch.roll(by, 1, 0))},
                outputs={"tmp": (tmp, None), "out": (out, None)})


def case_embed_splice():
    ops = _ops()
    V, Hd = 4096, 3584
    table, media = bf(V, Hd), bf(256, Hd)
    src = torch.cat([torch.arange(0, 20), -1 - torch.arange(256), torch.arange(20, 40)]).to(torch.int32).cuda()
    poison = torch.cat([torch.arange(100, 120), -1 - torch.arange(255, -1, -1), torch.arange(300, 320)])
    name, launch, out = record(lambda: ops.embed_splice(table, media, src))
    return Case("embed_splice-media", name, "text + one image", launch,
                produced={"table": (table, None), "media": (media, None),
                          "src": (src, poison.to(torch.int32).cuda())}, outputs={"out": (out, None)})


def _rope_common(S, Hq=28, Hkv=4, D=128, p0=0, decode=False):
    qkv = bf(S, (Hq + 2 * Hkv) * D)
    pos = torch.arange(p0, p0 + S, dtype=torch.int32, device="cuda")
    n_pages = (p0 + S + PAGE - 1) // PAGE + 2
    pt, pt_poison = _page_tables(n_pages, 1, (p0 + S + PAGE - 1) // PAGE, 7)
    kp = torch.zeros(n_pages, PAGE, Hkv, D, dtype=torch.bfloat16, device="cuda")
    return qkv, pos, pt.view(-1), pt_poison.view(-1), kp, torch.zeros_like(kp)


def case_rope_kv_append():
    ops = _ops()
    qkv, pos, pt, ptp, kp, vp = _rope_common(279, p0=77)
    inv = _inv_freq()
    name, launch, _ = record(lambda: ops.rope_kv_append(qkv, pos, 28, 4, 128, inv, kp, vp, pt, 77))
    return Case("rope_kv_append-prefill", name, "positions table-free", launch,
                produced={"positions": (pos, pos + 5), "inv_freq": (inv, None), "page_table": (pt, ptp)},
                inout={"qkv": (qkv, None)}, outputs={"k_pool": (kp, None), "v_pool": (vp, None)})


def case_rope_kv_append_table():
    ops = _ops()
    qkv, pos, pt, ptp, kp, vp = _rope_common(1000)
    tab = ops.rope_table(pos, 128, _inv_freq())
    name, launch, _ = record(lambda: ops.rope_kv_append_table(qkv, tab, 28, 4, 128, kp, vp, pt, 0))
    return Case("rope_kv_append_table-1000", name, "long prefill", launch,
                produced={"rope_table": (tab, None), "page_table": (pt, ptp)}, inout={"qkv": (qkv, None)},
                outputs={"k_pool": (kp, None), "v_pool": (vp, None)})


def case_rope_table():
    ops = _ops()
    pos = torch.arange(0, 1000, dtype=torch.int32, device="cuda")
    inv = _inv_freq()
    name, launch, tab = record(lambda: ops.rope_table(pos, 128, inv))
    return Case("rope_table-1000", name, "one request", launch,
                produced={"positions": (pos, pos + 3), "inv_freq": (inv, None)}, outputs={"table": (tab, None)})


# ---- decode GEMVs -------------------------------------------------------------------------------
def _gemv_case(fmt, N, K, fusion, static_w, variant=0):
    """fmt bf16 / fp8 / w4; fusion: norm (RMSNorm prologue + bias, the q/k/v form), swiglu (norm + SwiGLU, gate/up),
    residual (o_proj / down_proj), argmax (norm + argmax, lm_head)"""
    from vila_b200.model.qwen2 import quantize_e4m3_rows, quantize_w4_groups
    ops = _ops()
    x = bf(K)
    w = bf(N, K, scale=1 / math.sqrt(K))
    static, produced = {}, {"x": (x, None)}
    kw = dict(static_w=static_w, variant=variant)
    params = {}
    if fmt == "fp8":
        q, s = quantize_e4m3_rows(w)
        params = {"w": q, "w_scale": s}
        kw.update(w_scale=s)
        w = q
    elif fmt == "w4":
        pk, s, z = quantize_w4_groups(w)
        params = {"w": pk, "w_scale": s, "w_zero": z}
        kw.update(w_scale=s, w_zero=z)
        w = pk
    else:
        params = {"w": w}
    outputs = {}
    inout = {}
    if fusion in ("norm", "swiglu", "argmax"):
        nw = bf(K)
        params["norm_w"] = nw
        kw["norm_w"] = nw
    if fusion == "norm":
        b = bf(N)
        produced["bias"] = (b, None)
        kw["bias"] = b
    if fusion == "swiglu":
        kw["swiglu"] = True
    if fusion == "residual":
        r = bf(N)
        produced["residual"] = (r, None)
        kw["residual"] = r
    out = torch.empty(N // 2 if fusion == "swiglu" else N, dtype=torch.bfloat16, device="cuda")
    kw["out"] = out
    outputs["y"] = (out, None)
    if fusion == "argmax":
        key = torch.zeros(1, dtype=torch.int64, device="cuda")
        kw["argmax_key"] = key
        outputs["argmax_key"] = (key, torch.zeros_like(key))  # zero before the launch: the running max starts there
    for k_, v_ in params.items():
        if static_w:
            static[k_] = v_
        elif v_.dtype in (torch.uint8,) and k_ != "w_zero":
            produced[k_] = (v_, torch.roll(v_, 1, 0))
        elif v_.dtype in (torch.uint8,):
            produced[k_] = (v_, (v_ + 1) % 16)
        elif v_.dtype == torch.float8_e4m3fn:
            produced[k_] = (v_, _roll_rows(v_))
        else:
            produced[k_] = (v_, None if k_ != "w_scale" else v_.flip(0) + (1e-3 if v_.dtype == torch.float32 else 0))
    name, launch, _ = record(lambda: ops.gemv(x, w, **kw))
    kind = {0: "tma", 1: "register-staged"}[variant] if fmt == "bf16" else "tma"
    return Case(f"gemv-{fmt}-{kind}-{fusion}-{N}x{K}-{'static' if static_w else 'produced'}_w", name,
                f"{fmt} {kind} {fusion}", launch, static=static, produced=produced, outputs=outputs, inout=inout)


def _gemv_batch_case(fmt, M, N, K, fusion, static_w):
    from vila_b200.model.qwen2 import quantize_e4m3_rows, quantize_w4_groups
    ops = _ops()
    x = bf(M, K)
    w = bf(N, K, scale=1 / math.sqrt(K))
    if fmt == "fp8":
        q, s = quantize_e4m3_rows(w)
        params, kw = {"w": q, "w_scale": s}, dict(w_scale=s)
    else:
        q, s, z = quantize_w4_groups(w)
        params, kw = {"w": q, "w_scale": s, "w_zero": z}, dict(w_scale=s, w_zero=z)
    n_out = N // 2 if fusion == "swiglu" else N
    base = torch.empty(M, (n_out + 7) // 8 * 8, dtype=torch.bfloat16, device="cuda")
    out = base[:, :n_out]
    produced, inout = {"x": (x, None)}, {}
    if fusion == "swiglu":
        kw["swiglu"] = True
        outputs = {"y": (base, None)}
    else:  # residual added in place: y is the residual stream
        b = bf(N)
        kw.update(bias=b, residual=out)
        produced["bias"] = (b, None)
        inout["y"] = (base, None)
        outputs = {}
    static = {}
    for k_, v_ in params.items():
        if static_w:
            static[k_] = v_
        else:
            produced[k_] = (v_, _roll_rows(v_) if v_.dtype != torch.float32 else v_.flip(0) + 1e-3)
    name, launch, _ = record(lambda: ops.gemv_batch(x, q, out=out, static_w=static_w, **kw))
    return Case(f"gemv_batch-{fmt}-{fusion}-M{M}-{N}x{K}-{'static' if static_w else 'produced'}_w", name,
                f"batched {fmt} {fusion}", launch, static=static, produced=produced, outputs=outputs, inout=inout)


def case_argmax_finalize():
    ops = _ops()
    V, Hd, cols = 4096, 3584, 64
    keys = []
    for _ in range(2):  # two valid keys of the lm_head GEMV (value, ~index), from two different rows
        k = torch.zeros(1, dtype=torch.int64, device="cuda")
        ops.gemv(bf(512), bf(V, 512), argmax_key=k, out=torch.empty(V, dtype=torch.bfloat16, device="cuda"))
        keys.append(k)
    key, key_poison = keys
    table = bf(V, Hd)
    tok = torch.zeros(1, dtype=torch.int32, device="cuda")
    hist = torch.zeros(cols, dtype=torch.int32, device="cuda")
    step = torch.tensor([9], dtype=torch.int32, device="cuda")
    pos = torch.tensor([400], dtype=torch.int32, device="cuda")
    x_next = torch.empty(Hd, dtype=torch.bfloat16, device="cuda")
    torch.cuda.synchronize()
    name, launch, _ = record(lambda: ops.argmax_finalize(key, tok, hist, step, pos, table, x_next))
    return Case("argmax_finalize", name, "greedy step end", launch, produced={"embed_table": (table, None)},
                inout={"key": (key, key_poison), "step": (step, step + 20), "position": (pos, pos - 100)},
                outputs={"token_out": (tok, None), "token_hist": (hist, None), "x_next": (x_next, None)})


# ---- decode attention ----------------------------------------------------------------------------
HQ, HKV, D = 28, 4, 128


def case_decode_attention(mode):
    """mode head (<= 512 tokens), cluster (<= 1024), split (9..64 splits through ws / counters): GraphDecoder's
    pick_splits ladder for one sequence"""
    ops = _ops()
    pos_v, splits = {"head": (300, 0), "cluster": (900, 8), "split": (1800, 16)}[mode]
    n_pages = 20
    per_row = 16
    pt, ptp = _page_tables(n_pages, 1, per_row, 11)
    pt = pt.view(-1)
    qkv = bf(1, (HQ + 2 * HKV) * D)
    kp, vp = bf(n_pages, PAGE, HKV, D), bf(n_pages, PAGE, HKV, D)
    pos = torch.tensor([pos_v], dtype=torch.int32, device="cuda")
    out = torch.empty(1, HQ * D, dtype=torch.bfloat16, device="cuda")
    ws = torch.empty(HKV * max(splits, 1) * (HQ // HKV) * (D + 2), dtype=torch.float32, device="cuda")
    cnt = torch.zeros(HKV, dtype=torch.int32, device="cuda")
    inv = _inv_freq()
    name, launch, _ = record(lambda: ops.decode_attention(qkv, pos, kp, vp, pt, out, ws, cnt, inv, HQ, HKV, D, splits,
                                                          D ** -0.5))
    return Case(f"decode_attention-{mode}", name, f"{mode}, position {pos_v}", launch, static={"page_table": pt},
                produced={"position": (pos, pos - 37), "inv_freq": (inv, None)},
                inout={"qkv": (qkv, None), "k_pool": (kp, None), "v_pool": (vp, None)},
                outputs={"out": (out, None), "ws": (ws, None), "counters": (cnt, torch.zeros_like(cnt))})


def case_decode_attention_split():
    """the wgmma split-KV path of GraphDecoder.pick_splits past LONG_CTX"""
    from vila_b200.model.qwen2 import GraphDecoder
    ops = _ops()
    ctx = 5000
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    pages = (ctx + PAGE - 1) // PAGE
    per_head = max(1, min(GraphDecoder.MAX_SPLITS, sms // HKV))
    pps = (pages + per_head - 1) // per_head
    splits, split_tokens = (pages + pps - 1) // pps, pps * PAGE
    n_pages = pages + 4
    pt, _ = _page_tables(n_pages, 1, pages, 13)
    pt = pt.view(-1)
    qkv = bf(1, (HQ + 2 * HKV) * D)
    kp, vp = bf(n_pages, PAGE, HKV, D), bf(n_pages, PAGE, HKV, D)
    pos = torch.tensor([ctx - 1], dtype=torch.int32, device="cuda")
    out = torch.empty(1, HQ * D, dtype=torch.bfloat16, device="cuda")
    op = torch.empty(splits * HQ * D, dtype=torch.float32, device="cuda")
    lse = torch.empty(splits * HQ, dtype=torch.float32, device="cuda")
    cnt = torch.zeros(HKV, dtype=torch.int32, device="cuda")
    inv = _inv_freq()
    name, launch, _ = record(lambda: ops.decode_attention_split(qkv, pos, kp, vp, pt, out, op, lse, inv, HQ, HKV, D,
                                                                splits, split_tokens, D ** -0.5, counters=cnt))
    return Case("decode_attention_split", name, f"{splits} x {split_tokens} tokens, position {ctx - 1}", launch,
                static={"page_table": pt}, produced={"position": (pos, pos - 300), "inv_freq": (inv, None)},
                inout={"qkv": (qkv, None), "k_pool": (kp, None), "v_pool": (vp, None)},
                outputs={"out": (out, None), "o_partial": (op, None), "lse": (lse, None),
                         "counters": (cnt, torch.zeros_like(cnt))})


def case_decode_attention_batch():
    ops = _ops()
    B, per_row = 4, 16
    n_pages = B * per_row + 4
    pt, _ = _page_tables(n_pages, B, per_row, 17)
    qkv = bf(B, (HQ + 2 * HKV) * D)
    kp, vp = bf(n_pages, PAGE, HKV, D), bf(n_pages, PAGE, HKV, D)
    pos = torch.tensor([300, -1, 1500, 2047], dtype=torch.int32, device="cuda")
    out = torch.empty(B, HQ * D, dtype=torch.bfloat16, device="cuda")
    inv = _inv_freq()
    name, launch, _ = record(lambda: ops.decode_attention_batch(qkv, pos, kp, vp, pt, out, inv, HQ, HKV, D, D ** -0.5))
    return Case("decode_attention_batch", name, "head kernel, 4 slots one idle", launch, static={"page_table": pt},
                produced={"positions": (pos, torch.tensor([299, 5, -1, 2000], dtype=torch.int32, device="cuda")),
                          "inv_freq": (inv, None)},
                inout={"qkv": (qkv, None), "k_pool": (kp, None), "v_pool": (vp, None)}, outputs={"out": (out, None)})


def case_decode_attention_split_batch():
    from vila_b200 import serving
    ops = _ops()
    B = 2
    longest = 5000
    splits = serving.attention_config(longest)
    per_row = splits * serving.SPLIT_TOKENS // PAGE
    n_pages = B * per_row + 2
    pt, _ = _page_tables(n_pages, B, per_row, 19)
    qkv = bf(B, (HQ + 2 * HKV) * D)
    kp, vp = bf(n_pages, PAGE, HKV, D), bf(n_pages, PAGE, HKV, D)
    pos = torch.tensor([longest - 1, 2100], dtype=torch.int32, device="cuda")
    out = torch.empty(B, HQ * D, dtype=torch.bfloat16, device="cuda")
    op = torch.empty(B * splits * HQ * D, dtype=torch.float32, device="cuda")
    lse = torch.empty(B * splits * HQ, dtype=torch.float32, device="cuda")
    cnt = torch.zeros(B * HKV, dtype=torch.int32, device="cuda")
    inv = _inv_freq()
    name, launch, _ = record(lambda: ops.decode_attention_split_batch(qkv, pos, kp, vp, pt, out, op, lse, cnt, inv, HQ,
                                                                      HKV, D, splits, serving.SPLIT_TOKENS, D ** -0.5))
    return Case("decode_attention_split_batch", name, f"{splits} splits, 2 slots", launch, static={"page_table": pt},
                produced={"positions": (pos, torch.tensor([3000, 2600], dtype=torch.int32, device="cuda")),
                          "inv_freq": (inv, None)},
                inout={"qkv": (qkv, None), "k_pool": (kp, None), "v_pool": (vp, None)},
                outputs={"out": (out, None), "o_partial": (op, None), "lse": (lse, None),
                         "counters": (cnt, torch.zeros_like(cnt))})


def case_kv_quantize_fp8():
    ops = _ops()
    L, S = 2, 300
    src = bf(L, 2, 3, PAGE, HKV, D)
    P = 8
    dst = torch.zeros(L, 2, P, PAGE, HKV, D, device="cuda").to(torch.float8_e4m3fn)
    dsc = torch.zeros(L, 2, P, PAGE, HKV, dtype=torch.float32, device="cuda")
    row, rowp = _page_tables(P, 1, 3, 23)
    row, rowp = row.view(-1), rowp.view(-1)
    name, launch, _ = record(lambda: ops.kv_quantize_fp8(src, dst, dsc, row, S))
    return Case("kv_quantize_fp8", name, "prefill staging -> e4m3 pool", launch,
                produced={"src": (src, None), "page_table": (row, rowp)},
                outputs={"dst": (dst, None), "dst_scale": (dsc, None)})


def case_decode_attention_fp8(longest):
    from vila_b200 import serving
    from vila_b200.model.qwen2 import quantize_kv_e4m3
    ops = _ops()
    B = 2
    splits = serving.fp8_attention_config(longest)
    st = serving.FP8_SPLIT_TOKENS
    per_row = splits * st // PAGE
    n_pages = B * per_row + 2
    pt, _ = _page_tables(n_pages, B, per_row, 29)
    qkv = bf(B, (HQ + 2 * HKV) * D)
    kq, ks = quantize_kv_e4m3(bf(n_pages, PAGE, HKV, D))
    vq, vs = quantize_kv_e4m3(bf(n_pages, PAGE, HKV, D))
    kq, ks, vq, vs = (t.contiguous() for t in (kq, ks, vq, vs))
    pos = torch.tensor([longest - 1, -1], dtype=torch.int32, device="cuda")
    out = torch.empty(B, HQ * D, dtype=torch.bfloat16, device="cuda")
    ws = torch.empty(B * HQ * splits * (D + 2), dtype=torch.float32, device="cuda")
    cnt = torch.zeros(B * HKV, dtype=torch.int32, device="cuda")
    inv = _inv_freq()
    name, launch, _ = record(lambda: ops.decode_attention_fp8_batch(qkv, pos, kq, vq, ks, vs, pt, out, ws, cnt, inv,
                                                                    HQ, HKV, splits, st, D ** -0.5))
    return Case(f"decode_attention_fp8_batch-{longest}", name, f"{splits} x {st} tokens, one idle slot", launch,
                static={"page_table": pt},
                produced={"positions": (pos, torch.tensor([longest // 2, 700], dtype=torch.int32, device="cuda")),
                          "qkv": (qkv, None), "inv_freq": (inv, None)},
                inout={"k_pool": (kq, None), "v_pool": (vq, None), "k_scale": (ks, None), "v_scale": (vs, None)},
                outputs={"out": (out, None), "ws": (ws, None), "counters": (cnt, torch.zeros_like(cnt))})


# ---- sampling, logprobs, penalties, grammar, prefix hash ------------------------------------------
VOCAB = 151_936  # Qwen2's lm_head rows


def case_sample_batch():
    ops = _ops()
    M = 4
    logits = bf(M, VOCAB, scale=3)
    it = torch.tensor([0.0, 1.0, 1.4, 0.7], device="cuda")
    tk = torch.tensor([0, 50, 0, 1], dtype=torch.int32, device="cuda")
    tp = torch.tensor([1.0, 0.9, 0.8, 1.0], device="cuda")
    seed = torch.tensor([1, 2, 3, 4], dtype=torch.int64, device="cuda")
    step = torch.tensor([0, 5, 9, 2], dtype=torch.int64, device="cuda")
    pos = torch.tensor([10, 20, -1, 40], dtype=torch.int32, device="cuda")
    out = torch.zeros(M, dtype=torch.int64, device="cuda")
    nk = torch.zeros(M, dtype=torch.int32, device="cuda")
    name, launch, _ = record(lambda: ops.sample_batch(logits, it, tk, tp, seed, step, pos, out=out, n_kept=nk))
    return Case("sample_batch", name, "4 rows, greedy / top-k / top-p / idle", launch,
                produced={"logits": (logits, None), "inv_temperature": (it, it.flip(0)),
                          "top_k": (tk, torch.tensor([7, 0, 3, 0], dtype=torch.int32, device="cuda")),
                          "top_p": (tp, tp.flip(0)), "seed": (seed, seed + 100), "step": (step, step + 3),
                          "positions": (pos, pos.flip(0))},
                outputs={"tokens": (out, None), "n_kept": (nk, None)})


def case_sample_finalize():
    ops = _ops()
    Hd, cols = 3584, 64
    logits = bf(VOCAB, scale=3)
    it = torch.tensor([1.2], device="cuda")
    tk = torch.tensor([40], dtype=torch.int32, device="cuda")
    tp = torch.tensor([0.9], device="cuda")
    seed = torch.tensor([77], dtype=torch.int64, device="cuda")
    step = torch.tensor([5], dtype=torch.int32, device="cuda")
    pos = torch.tensor([400], dtype=torch.int32, device="cuda")
    tok = torch.zeros(1, dtype=torch.int32, device="cuda")
    hist = torch.zeros(cols, dtype=torch.int32, device="cuda")
    table = bf(VOCAB, Hd)
    x_next = torch.empty(Hd, dtype=torch.bfloat16, device="cuda")
    name, launch, _ = record(lambda: ops.sample_finalize(logits, it, tk, tp, seed, step, tok, hist, pos, table, x_next))
    return Case("sample_finalize", name, "one row, sampled", launch,
                produced={"logits": (logits, None), "inv_temperature": (it, it * 0.5),
                          "top_k": (tk, tk * 0 + 3), "top_p": (tp, tp * 0 + 1.0), "seed": (seed, seed + 1),
                          "embed_table": (table, None)},
                inout={"step": (step, step + 11), "position": (pos, pos + 50)},
                outputs={"token_out": (tok, None), "token_hist": (hist, None), "x_next": (x_next, None)})


def case_token_logprobs():
    ops = _ops()
    M, cols, n = 4, 16, 5
    logits = bf(M, VOCAB, scale=3)
    tokens = torch.tensor([5, 100, 151_000, 7], dtype=torch.int64, device="cuda")
    step = torch.tensor([0, 3, 15, 40], dtype=torch.int64, device="cuda")
    pos = torch.tensor([10, -1, 30, 40], dtype=torch.int32, device="cuda")
    lp = torch.zeros(M, cols, dtype=torch.float32, device="cuda")
    ti = torch.zeros(M, cols, n, dtype=torch.int32, device="cuda")
    tl = torch.zeros(M, cols, n, dtype=torch.float32, device="cuda")
    name, launch, _ = record(lambda: ops.token_logprobs(logits, tokens, step, pos, lp_hist=lp, top_ids=ti, top_lp=tl))
    return Case("token_logprobs", name, "4 rows, one idle", launch,
                produced={"logits": (logits, None), "tokens": (tokens, tokens.flip(0)), "step": (step, step.flip(0)),
                          "positions": (pos, pos.flip(0))},
                outputs={"lp_hist": (lp, None), "top_ids": (ti, None), "top_lp": (tl, None)})


def case_token_logprobs_row():
    ops = _ops()
    cols, n = 16, 5
    logits = bf(VOCAB, scale=3)
    tok = torch.tensor([1234], dtype=torch.int32, device="cuda")
    step = torch.tensor([4], dtype=torch.int32, device="cuda")
    n_used = torch.tensor([3], dtype=torch.int32, device="cuda")
    lp = torch.zeros(cols, dtype=torch.float32, device="cuda")
    ti = torch.zeros(cols, n, dtype=torch.int32, device="cuda")
    tl = torch.zeros(cols, n, dtype=torch.float32, device="cuda")
    ws, cnt = ops.logprobs_row_workspace(VOCAB, "cuda")
    name, launch, _ = record(lambda: ops.token_logprobs_row(logits, tok, step, lp_hist=lp, top_ids=ti, top_lp=tl,
                                                            n_used=n_used, workspace=ws, counter=cnt))
    return Case("token_logprobs_row", name, "one row over the GPU", launch,
                produced={"logits": (logits, None), "token": (tok, tok + 99), "step": (step, step + 5),
                          "n_used": (n_used, n_used + 2)},
                outputs={"lp_hist": (lp, None), "top_ids": (ti, None), "top_lp": (tl, None), "workspace": (ws, None),
                         "counter": (cnt, torch.zeros_like(cnt))})


def case_apply_penalties():
    ops = _ops()
    M, cols = 3, 32
    logits = bf(M, VOCAB, scale=3)
    hist = torch.randint(0, 500, (M, cols), dtype=torch.int64, device="cuda", generator=_g())
    step = torch.tensor([10, 32, 5], dtype=torch.int64, device="cuda")
    pos = torch.tensor([10, 20, -1], dtype=torch.int32, device="cuda")
    pres = torch.tensor([0.5, 1.0, 0.2], device="cuda")
    freq = torch.tensor([0.3, 0.1, 0.7], device="cuda")
    out = torch.empty(M, VOCAB, dtype=torch.bfloat16, device="cuda")
    name, launch, _ = record(lambda: ops.apply_penalties(logits, hist, step, pos, pres, freq, out=out))
    return Case("apply_penalties", name, "3 rows, one idle", launch,
                produced={"logits": (logits, None), "history": (hist, (hist + 777) % VOCAB),
                          "step": (step, step.flip(0)), "positions": (pos, pos.flip(0)),
                          "presence": (pres, pres + 1), "frequency": (freq, freq + 1)},
                outputs={"out": (out, None)})


def case_apply_penalties_row():
    ops = _ops()
    cols = 64
    logits = bf(VOCAB, scale=3)
    hist = torch.randint(0, 500, (cols,), dtype=torch.int32, device="cuda", generator=_g())
    step = torch.tensor([20], dtype=torch.int32, device="cuda")
    pres, freq = torch.tensor([0.5], device="cuda"), torch.tensor([0.25], device="cuda")
    out = torch.empty(VOCAB, dtype=torch.bfloat16, device="cuda")
    name, launch, _ = record(lambda: ops.apply_penalties_row(logits, hist, step, pres, freq, out=out))
    return Case("apply_penalties_row", name, "one row", launch,
                produced={"logits": (logits, None), "history": (hist, (hist + 777) % VOCAB), "step": (step, step + 30),
                          "presence": (pres, pres + 1), "frequency": (freq, freq + 1)},
                outputs={"out": (out, None)})


def case_bitmask(in_place):
    ops = _ops()
    W = (VOCAB + 31) // 32
    logits = bf(VOCAB, scale=3)
    mask = torch.randint(-2 ** 31, 2 ** 31 - 1, (W,), dtype=torch.int32, device="cuda", generator=_g())
    c = Case(f"apply_token_bitmask_row{'-in_place' if in_place else ''}", regime="in place" if in_place else "to out")
    if in_place:
        c.entry, c.launch, _ = record(lambda: ops.apply_token_bitmask_row(logits, mask, out=logits))
        c.inout["logits"] = (logits, None)
    else:
        out = torch.empty(VOCAB, dtype=torch.bfloat16, device="cuda")
        c.entry, c.launch, _ = record(lambda: ops.apply_token_bitmask_row(logits, mask, out=out))
        c.produced["logits"] = (logits, None)
        c.outputs["out"] = (out, None)
    c.produced["bitmask"] = (mask, ~mask)
    return c


def case_prefix_hash():
    ops = _ops()
    x = bf(1000, 3584)
    name, launch, out = record(lambda: ops.prefix_block_hash(x, 0x1234, 0x5678))
    return Case("prefix_block_hash", name, "7 blocks", launch, produced={"x": (x, None)}, outputs={"out": (out, None)})


CASES = {}


def _add(entry, builder, *args):
    """one row: the C entry point the builder's case must call, the builder and its arguments"""
    CASES[(builder.__name__, args)] = (entry, builder, args)


for _row in LINEAR_ROWS:
    for _st in (False, True):
        _add("vila_linear" if _row[1] is None else "vila_linear_cfg", case_linear, *_row, _st)
_add("vila_linear_cfg", case_linear_inplace_residual)
for _st in (False, True):
    _add("vila_linear_qkv_rope", case_qkv_rope, _st)
_add("vila_fmha", case_fmha_vit)
_add("vila_fmha", case_fmha_paged)
_add("vila_layernorm", case_layernorm, 1024, 1152, "CTA per row")
_add("vila_layernorm", case_layernorm, 16384, 1152, "warp per row")
_add("vila_rmsnorm", case_rmsnorm, 279, 3584, False, "CTA per row")
_add("vila_rmsnorm", case_rmsnorm, 279, 3584, True, "CTA per row")
_add("vila_rmsnorm", case_rmsnorm, 8192, 1536, True, "warp per row")
_add("vila_patch_im2col", case_im2col)
_add("vila_space_to_depth", case_space_to_depth)
_add("vila_s2_merge", case_s2_merge)
_add("vila_chessboard_merge", case_chessboard)
_add("vila_tsp_pool", case_tsp, 1152)
_add("vila_tsp_pool", case_tsp, 1154)
_add("vila_resize_bicubic_tiles", case_resize)
_add("vila_embed_splice", case_embed_splice)
_add("vila_rope_kv_append", case_rope_kv_append)
_add("vila_rope_kv_append_table", case_rope_kv_append_table)
_add("vila_rope_table", case_rope_table)
for _st in (False, True):
    _add("vila_gemv", _gemv_case, "bf16", 4608, 3584, "norm", _st, 0)
    _add("vila_gemv", _gemv_case, "bf16", 4608, 3584, "norm", _st, 1)
    _add("vila_gemv", _gemv_case, "bf16", 3584, 18944, "residual", _st, 0)
    _add("vila_gemv", _gemv_case, "bf16", 37888, 3584, "swiglu", _st, 0)
    _add("vila_gemv", _gemv_case, "bf16", 32768, 3584, "argmax", _st, 0)
    _add("vila_gemv_fp8", _gemv_case, "fp8", 37888, 3584, "swiglu", _st)
    _add("vila_gemv_fp8", _gemv_case, "fp8", 3584, 18944, "residual", _st)
    _add("vila_gemv_w4a16", _gemv_case, "w4", 4608, 3584, "norm", _st)
    _add("vila_gemv_w4a16", _gemv_case, "w4", 3584, 18944, "residual", _st)
    _add("vila_gemv_batch_fp8", _gemv_batch_case, "fp8", 8, 37888, 3584, "swiglu", _st)
    _add("vila_gemv_batch_w4a16", _gemv_batch_case, "w4", 16, 3584, 18944, "residual", _st)
_add("vila_argmax_finalize", case_argmax_finalize)
for _m in ("head", "cluster", "split"):
    _add("vila_decode_attention", case_decode_attention, _m)
_add("vila_decode_attention_split", case_decode_attention_split)
_add("vila_decode_attention_batch", case_decode_attention_batch)
_add("vila_decode_attention_split_batch", case_decode_attention_split_batch)
_add("vila_kv_quantize_fp8", case_kv_quantize_fp8)
_add("vila_decode_attention_fp8_batch", case_decode_attention_fp8, 2048)
_add("vila_decode_attention_fp8_batch", case_decode_attention_fp8, 9000)
_add("vila_sample_batch", case_sample_batch)
_add("vila_sample_finalize", case_sample_finalize)
_add("vila_token_logprobs", case_token_logprobs)
_add("vila_token_logprobs_row", case_token_logprobs_row)
_add("vila_apply_penalties", case_apply_penalties)
_add("vila_apply_penalties_row", case_apply_penalties_row)
_add("vila_apply_token_bitmask_row", case_bitmask, False)
_add("vila_apply_token_bitmask_row", case_bitmask, True)
_add("vila_prefix_block_hash", case_prefix_hash)
# launching entry points without a row of their own: vila_fmha_cfg runs vila_fmha's kernels under a forced flavour
# (the rows above run the flavours production picks), and the two vila_test_pdl_* hooks are this file's producer and
# probe
NOT_CONSUMERS = {"vila_fmha_cfg", "vila_test_pdl_late", "vila_test_pdl_probe"}


def _case_id(key):
    name, args = key
    return "-".join([name.replace("case_", "").lstrip("_")] + [str(a) for a in args])


# ------------------------------------------------------------------------------------------------
# the harness
# ------------------------------------------------------------------------------------------------
def _copy_rows(pairs: List[Tuple[torch.Tensor, torch.Tensor]]) -> torch.Tensor:
    rows = [(src.data_ptr(), dst.data_ptr(), src.numel() * src.element_size()) for src, dst in pairs]
    return torch.tensor(rows if rows else [[0, 0, 0]], dtype=torch.int64, device="cuda")[:len(rows)].contiguous()


class _Pair:
    """the late producer + the consumer's recorded call, for one case"""

    def __init__(self, c: Case):
        from vila_b200 import ops
        self.c, self.ops = c, ops
        for name, t in list(c.static.items()) + [(n, b) for n, (b, _) in {**c.produced, **c.outputs, **c.inout}.items()]:
            assert t.is_cuda and t.is_contiguous(), (c.id, name)
        self.true = {n: b.clone() for n, (b, _) in {**c.produced, **c.inout}.items()}
        self.poison = {}
        for n, (b, p) in {**c.produced, **c.inout}.items():
            p = _poison_like(b) if p is None else p.to(b.dtype).reshape(b.shape).contiguous()
            assert not torch.equal(_bytes(p), _bytes(self.true[n])), (c.id, n, "poison equals the true value")
            self.poison[n] = p
        self.sentinel = {n: (_sentinel_like(b) if s is None else s.to(b.dtype).reshape(b.shape).contiguous())
                         for n, (b, s) in c.outputs.items()}
        self.side = {n: torch.empty_like(b) for n, (b, _) in {**c.outputs, **c.inout}.items()}
        self.snap = _copy_rows([(b, self.side[n]) for n, (b, _) in {**c.outputs, **c.inout}.items()])
        self.late = _copy_rows([(self.true[n], b) for n, (b, _) in {**c.produced, **c.inout}.items()])

    def set_state(self, late: bool):
        c = self.c
        for n, (b, _) in c.outputs.items():
            b.copy_(self.sentinel[n])
        for n, (b, _) in {**c.produced, **c.inout}.items():
            b.copy_(self.poison[n] if late else self.true[n])
        for s in self.side.values():
            _bytes(s).fill_(0x5A)

    def pair(self):
        self.ops.pdl_late(self.snap, self.late, DELAY_NS)
        self.c.launch()

    def results(self):
        return {n: b.clone() for n, (b, _) in {**self.c.outputs, **self.c.inout}.items()}

    def check(self, ref, how: str):
        c = self.c
        for n, (b, _) in {**c.outputs, **c.inout}.items():
            assert torch.equal(_bytes(b), _bytes(ref[n])), \
                f"{c.id} [{how}]: {n} differs from the synchronized run: an input read before the dependency wait"
            before = self.sentinel[n] if n in c.outputs else self.poison[n]
            assert torch.equal(_bytes(self.side[n]), _bytes(before)), \
                f"{c.id} [{how}]: {n} was written before the dependency wait"


def _trace_pair(p: _Pair):
    """-> (nothing between producer and consumer, consumer started before the producer ended), or None without GPU
    activity records"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        p.pair()
        torch.cuda.synchronize()
    acts = []
    for e in prof.events():
        if getattr(e, "device_type", None) is not None and str(e.device_type).endswith("CUDA"):
            acts.append((e.time_range.start, e.time_range.end, e.name))
    acts.sort()
    idx = [i for i, a in enumerate(acts) if "pdl_late_kernel" in a[2]]
    if not idx or idx[0] + 1 >= len(acts):
        return None
    prod, nxt = acts[idx[0]], acts[idx[0] + 1]
    clean = not any(k in nxt[2].lower() for k in ("memcpy", "memset"))
    return clean, nxt[0] < prod[1], nxt[2]


@pytest.fixture(scope="module")
def side_stream(cuda):
    from vila_b200 import ops
    ops.ensure_workspace("cuda")
    if not ops.pdl_enabled():
        pytest.fail("VILA_B200_NO_PDL is set: this file tests the launches with programmatic dependent launch on")
    s = torch.cuda.Stream()
    _warm_up(s)
    return s


def _warm_up(stream):
    """launch the producer and the probe once: the first launch of a kernel loads its module (lazy loading), which
    can hold the host until the stream drains and so close the window of that one launch"""
    from vila_b200 import ops
    with torch.cuda.stream(stream):
        e = _copy_rows([])
        flag = torch.zeros(1, dtype=torch.int32, device="cuda")
        seen = torch.zeros(2, dtype=torch.int32, device="cuda")
        ops.pdl_late(e, e, 0)
        ops.pdl_probe(flag, seen)
    torch.cuda.synchronize()


def test_probe_sees_the_window(side_stream):
    """positive control: the probe reads the flag before its wait (old value) and after it (new value); eager and in
    a CUDA graph.  Without this window every case below would pass vacuously.  (Before the warm-up in side_stream,
    the eager probe saw (new, new) on an H100: the first launch of a kernel loads its module and closes the window.)"""
    from vila_b200 import ops
    with torch.cuda.stream(side_stream):
        flag = torch.tensor([1], dtype=torch.int32, device="cuda")
        new = torch.tensor([2], dtype=torch.int32, device="cuda")
        seen = torch.zeros(2, dtype=torch.int32, device="cuda")
        late = _copy_rows([(new, flag)])
        snap = _copy_rows([])
        torch.cuda.synchronize()
        ops.pdl_late(snap, late, DELAY_NS)
        ops.pdl_probe(flag, seen)
        torch.cuda.synchronize()
        eager = seen.tolist()
        flag.fill_(1)
        seen.zero_()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side_stream):
            ops.pdl_late(snap, late, DELAY_NS)
            ops.pdl_probe(flag, seen)
        flag.fill_(1)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        graph = seen.tolist()
    _record({"name": "pdl probe", "eager": eager, "graph": graph, "delay_ns": DELAY_NS, "ok": True})
    assert eager == [1, 2], f"no PDL overlap window on this device / stream (probe saw {eager})"
    assert graph == [1, 2], f"no PDL overlap window inside a CUDA graph (probe saw {graph})"


def test_late_producer_refuses_bad_delay(cuda):
    from vila_b200 import ops
    e = torch.zeros(0, 3, dtype=torch.int64, device="cuda")
    with pytest.raises(RuntimeError, match="delay_ns"):
        ops.pdl_late(e, e, 2_000_001)


@pytest.mark.parametrize("key", list(CASES), ids=[_case_id(k) for k in CASES])
def test_pdl_contract(side_stream, key):
    entry, builder, args = CASES[key]
    with torch.cuda.stream(side_stream):
        c = builder(*args)
        assert c.entry == entry, (c.id, c.entry, entry)
        p = _Pair(c)
        # 1. reference: fully prepared inputs, a synchronize on each side
        p.set_state(late=False)
        torch.cuda.synchronize()
        c.launch()
        torch.cuda.synchronize()
        ref = p.results()
        # 2. late producer, then the consumer with nothing in between
        p.set_state(late=True)
        torch.cuda.synchronize()
        p.pair()
        torch.cuda.synchronize()
        p.check(ref, "eager")
        # 3. the same pair in a CUDA graph, replayed once
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side_stream):
            p.pair()
        p.set_state(late=True)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        p.check(ref, "graph")
        del g
        # 4. the same eager pair under torch.profiler: what runs between producer and consumer
        p.set_state(late=True)
        torch.cuda.synchronize()
        tr = _trace_pair(p)
        p.check(ref, "traced")
    row = {"name": "pdl contract", "case": c.id, "entry": c.entry, "regime": c.regime,
           "static": sorted(c.static), "produced": sorted(c.produced), "written": sorted({**c.outputs, **c.inout}),
           "trace": "unavailable" if tr is None else {"clean": tr[0], "overlap_seen": tr[1], "next": tr[2][:60]},
           "ok": True}
    _record(row)
    if tr is not None:
        assert tr[0], f"{c.id}: {tr[2]} runs between the producer and the consumer"
        assert "pdl_late_kernel" not in tr[2]


# ------------------------------------------------------------------------------------------------
# end to end: the same model run with PDL on and with PDL off (VILA_B200_NO_PDL=1) gives the same bits.  This also
# covers the junctions between the kernels of one entry point (decode_attention_split, resize_bicubic_tiles,
# linear_qkv_rope), which the late producer cannot reach.  The flag is read once per process: one child each.
# ------------------------------------------------------------------------------------------------
def _e2e_child(out_path: str) -> None:
    """the tiny model: image encoding, prefills on the linear_qkv_rope path (S = 279) and the table path (S = 1000),
    GraphDecoder greedy / sampled ids and a split-KV context, BatchedDecoder ids and logprobs for every decode-weight x
    KV-cache format (prefix caching on the bf16 K/V) -> saved to out_path"""
    from vila_b200 import serving
    from vila_b200.model import LlavaLlamaModel, tiny_test_config
    torch.cuda.set_device(0)
    cfg = tiny_test_config()
    model = LlavaLlamaModel(cfg, device="cuda").init_random(0)
    llm = model.llm
    res = {}
    g = torch.Generator().manual_seed(1)
    S = cfg.vision_tower_cfg.image_size
    image = torch.randn(3, S, S, generator=g).to(torch.bfloat16).cuda()
    res["encode_images"] = model.encode_images(image[None]).clone()
    ids = torch.randint(3, 900, (10,), generator=g).tolist()
    ids.insert(3, cfg.image_token_id)
    ids = torch.tensor([ids])
    res["image_prompt_logits"] = model(input_ids=ids, media={"image": [image]}).logits.clone()
    res["image_prompt_greedy"] = model.generate(input_ids=ids, media={"image": [image]}, max_new_tokens=16,
                                                eos_token_id=None).cpu()

    def prompt(n, seed):
        gg = torch.Generator(device="cuda").manual_seed(seed)
        t = torch.randint(0, llm.config.vocab_size, (n,), device="cuda", generator=gg)
        return llm.model.embed_tokens.weight[t].clone()

    for n in (279, 1000):
        res[f"prefill_{n}"] = llm(inputs_embeds=prompt(n, n)[None]).logits.clone()
    res["graph_greedy_split_kv"] = llm.generate(inputs_embeds=prompt(1500, 7)[None], max_new_tokens=24,
                                                eos_token_id=None).cpu()
    torch.manual_seed(0)  # the sampled rows draw their seeds from the host generator
    res["graph_sampled"] = llm.generate(inputs_embeds=prompt(200, 8)[None], max_new_tokens=24, do_sample=True,
                                        temperature=0.9, top_k=40, top_p=0.95, eos_token_id=None).cpu()
    shared = prompt(300, 9)
    for weights in ("bf16", "fp8", "w4a16"):
        llm.set_decode_weights(weights)
        for kv in ("bf16", "fp8"):
            dec = serving.BatchedDecoder(llm, slots=3, max_tokens_per_slot=2048, max_new=32, kv_cache=kv,
                                         prefix_cache=kv == "bf16", logprobs=2)  # fp8 K/V: no prefix caching
            dec.capture()
            dec.admit(0, torch.cat([shared, prompt(40, 10)]))
            dec.admit(1, torch.cat([shared, prompt(90, 11)]))
            dec.run(16)
            res[f"batched_{weights}_{kv}"] = [(dec.generated(s), [tuple(t) for t in dec.generated_logprobs(s)])
                                             for s in (0, 1)]
            del dec
    llm.set_decode_weights("bf16")
    torch.cuda.synchronize()
    torch.save({k: (v.cpu() if torch.is_tensor(v) else v) for k, v in res.items()}, out_path)


def _run_child(tmp_path, no_pdl: bool):
    import os
    import subprocess
    import sys
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    out = tmp_path / f"e2e_{'off' if no_pdl else 'on'}.pt"
    env = {k: v for k, v in os.environ.items() if k != "VILA_B200_NO_PDL"}
    if no_pdl:
        env["VILA_B200_NO_PDL"] = "1"
    code = ("import sys; from tests.test_pdl_gpu import _e2e_child; from vila_b200 import ops; "
            f"assert ops.pdl_enabled() is {not no_pdl}; _e2e_child(sys.argv[1])")
    r = subprocess.run([sys.executable, "-c", code, str(out)], cwd=root, env=env, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    return torch.load(out, weights_only=False)


def test_model_paths_pdl_on_equal_pdl_off(cuda, tmp_path):
    on = _run_child(tmp_path, no_pdl=False)
    off = _run_child(tmp_path, no_pdl=True)
    assert on.keys() == off.keys()
    for k in on:
        a, b = on[k], off[k]
        same = torch.equal(a, b) if torch.is_tensor(a) else a == b
        assert same, f"{k}: PDL on and PDL off differ"
    _record({"name": "pdl on == pdl off", "model": "tiny", "compared": sorted(on), "ok": True})
