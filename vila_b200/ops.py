"""Tensor-level wrappers over the C-ABI (include/vila_b200.h).

PyTorch is used only for device memory (torch.empty), the current CUDA stream and dtype bookkeeping;
every operation below is one call into libvila_b200.so.  No function here has an eager fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from . import _lib
from ._lib import (DecodeAttnFp8Params, DecodeAttnParams, DecodeAttnSplitParams, FmhaParams, GemvBatchParams,
                   GemvParams, LogprobsParams, LogprobsRowParams, PenaltyParams, PenaltyRowParams,
                   SampleFinalizeParams, SampleParams, check)

ACT_NONE, ACT_GELU_TANH, ACT_GELU_ERF, ACT_SILU = 0, 1, 2, 3


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _chk(t: torch.Tensor, name: str, dtype=torch.bfloat16) -> None:
    if not t.is_cuda:
        raise RuntimeError(f"vila_b200.ops: {name} must be a CUDA tensor (no CPU fallback exists)")
    if t.dtype != dtype:
        raise RuntimeError(f"vila_b200.ops: {name} must be {dtype}, got {t.dtype}")


_WORKSPACE = {}


def ensure_workspace(device, nbytes: int = 96 << 20) -> torch.Tensor:
    """Allocate (once per device) and register the zero-initialised stream-K scratch."""
    key = torch.device(device).index or 0
    ws = _WORKSPACE.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.zeros(nbytes, dtype=torch.uint8, device=device)
        _WORKSPACE[key] = ws
    check(_lib.load().vila_set_workspace(ws.data_ptr(), ws.numel()), "vila_set_workspace")
    return ws


def linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *,
           act: int = ACT_NONE, residual: Optional[torch.Tensor] = None, res_row_mod: int = 0,
           swiglu: bool = False, out: Optional[torch.Tensor] = None,
           block_n: Optional[int] = None, static_w: bool = False) -> torch.Tensor:
    """out = epilogue(x @ w.T).  x [M,K] (row stride arbitrary), w [N,K].
    static_w: w is a parameter (VILA_FLAG_STATIC_W): it may be fetched before the PDL wait."""
    _chk(x, "x"); _chk(w, "w")
    assert x.dim() == 2 and w.dim() == 2 and x.shape[1] == w.shape[1], (x.shape, w.shape)
    assert x.stride(1) == 1 and w.stride(1) == 1
    M, K = x.shape
    N = w.shape[0]
    n_out = N // 2 if swiglu else N
    if out is None:
        out = torch.empty((M, n_out), dtype=torch.bfloat16, device=x.device)
    else:
        assert out.shape == (M, n_out) and out.stride(1) == 1
    if M == 0:
        return out
    ld_res = 0
    if residual is not None:
        _chk(residual, "residual")
        assert residual.dim() == 2 and residual.stride(1) == 1 and residual.shape[1] == N
        ld_res = residual.stride(0)
    lib = _lib.load()
    args = (_p(x), x.stride(0), _p(w), w.stride(0), _p(bias), _p(residual), ld_res, res_row_mod,
            _p(out), out.stride(0), M, N, K, act, (1 if swiglu else 0) | (2 if static_w else 0), _stream())
    if block_n is None:
        check(lib.vila_linear(*args), "vila_linear")
    else:
        check(lib.vila_linear_cfg(block_n, *args), "vila_linear_cfg")
    return out


def layernorm(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float) -> torch.Tensor:
    _chk(x, "x")
    cols = x.shape[-1]
    x2 = x.reshape(-1, cols)
    assert x2.is_contiguous()
    out = torch.empty_like(x2)
    check(_lib.load().vila_layernorm(_p(x2), _p(w), _p(b), _p(out), x2.shape[0], cols, eps,
                                     _stream()), "vila_layernorm")
    return out.view(x.shape)


def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float,
            residual_add: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Qwen2RMSNorm.  With residual_add: x += residual_add (in place) before normalising."""
    _chk(x, "x")
    cols = x.shape[-1]
    x2 = x.view(-1, cols)
    assert x2.is_contiguous()
    out = torch.empty_like(x2)
    check(_lib.load().vila_rmsnorm(_p(x2), _p(residual_add), _p(w), _p(out), x2.shape[0], cols,
                                   eps, _stream()), "vila_rmsnorm")
    return out.view(x.shape)


def fmha(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, *, B: int, Sq: int, Sk: int,
         causal: bool, scale: float, out: Optional[torch.Tensor] = None,
         page_table: Optional[torch.Tensor] = None, variant: int = 0) -> torch.Tensor:
    """q [B*Sq, Hq, D] view; k/v either [B*Sk, Hkv, D] views or paged pools [P, 128, Hkv, D].
    variant (test hook, vila_fmha_cfg): 0 default, 1 / 2 the wgmma kernel, 3 / 4 with polynomial exp2."""
    _chk(q, "q"); _chk(k, "k"); _chk(v, "v")
    assert q.dim() == 3 and q.stride(2) == 1
    Hq, D = q.shape[1], q.shape[2]
    if out is None:
        out = torch.empty((B * Sq, Hq, D), dtype=torch.bfloat16, device=q.device)
    p = FmhaParams()
    p.q, p.q_tok_stride, p.q_head_stride = q.data_ptr(), q.stride(0), q.stride(1)
    p.k, p.v = k.data_ptr(), v.data_ptr()
    if k.dim() == 4:  # paged [P, 128, Hkv, D]
        assert k.shape[1] == 128 and k.stride() == v.stride() and k.stride(3) == 1
        Hkv = k.shape[2]
        p.kv_page_stride, p.kv_tok_stride, p.kv_head_stride = k.stride(0), k.stride(1), k.stride(2)
        p.kv_num_pages = k.shape[0]
        if page_table is not None:
            assert page_table.dtype == torch.int32 and page_table.is_cuda
            pt = page_table.view(B, -1)
            p.page_table, p.page_table_stride = pt.data_ptr(), pt.stride(0)
        else:
            assert B == 1
            p.page_table, p.page_table_stride = None, 0
    else:
        assert k.dim() == 3 and k.stride() == v.stride() and k.stride(2) == 1
        Hkv = k.shape[1]
        p.kv_page_stride, p.kv_tok_stride, p.kv_head_stride = 0, k.stride(0), k.stride(1)
        p.kv_num_pages = 0
        p.page_table, p.page_table_stride = None, 0
    p.o, p.o_tok_stride, p.o_head_stride = out.data_ptr(), out.stride(0), out.stride(1)
    p.B, p.Sq, p.Sk, p.Hq, p.Hkv, p.D = B, Sq, Sk, Hq, Hkv, D
    p.causal = 1 if causal else 0
    p.scale = scale
    if variant == 0:
        check(_lib.load().vila_fmha(C.byref(p), _stream()), "vila_fmha")
    else:
        check(_lib.load().vila_fmha_cfg(variant, C.byref(p), _stream()), "vila_fmha_cfg")
    return out


def patch_im2col(pixels: torch.Tensor, patch: int, k_pad: int) -> torch.Tensor:
    _chk(pixels, "pixels")
    assert pixels.is_contiguous() and pixels.dim() == 4
    B, Cc, H, W = pixels.shape
    out = torch.empty((B * (H // patch) * (W // patch), k_pad), dtype=torch.bfloat16,
                      device=pixels.device)
    check(_lib.load().vila_patch_im2col(_p(pixels), _p(out), B, Cc, H, W, patch, k_pad, _stream()),
          "vila_patch_im2col")
    return out


_COEFF_CACHE = {}


def _bicubic_tables(in_size: int, out_size: int, device):
    key = (in_size, out_size, str(device))
    ent = _COEFF_CACHE.get(key)
    if ent is None:
        from .model.media import bicubic_coeffs
        ksize, bounds, coeffs = bicubic_coeffs(in_size, out_size)
        if len(_COEFF_CACHE) > 64:
            _COEFF_CACHE.clear()
        ent = (ksize, bounds.to(device), coeffs.to(device))
        _COEFF_CACHE[key] = ent
    return ent


def resize_bicubic_tiles(src: torch.Tensor, out_w: int, out_h: int, out: torch.Tensor, tile: int,
                         tile_index0: int, mean: float, std: float) -> torch.Tensor:
    """src uint8 [H, W, 3] (device) -> PIL-exact bicubic resize to (out_w, out_h), rescale, normalise,
    cut into tile x tile blocks written to out[tile_index0 ...] (bf16 [n, 3, tile, tile])."""
    _chk(src, "src", torch.uint8); _chk(out, "out")
    assert src.dim() == 3 and src.shape[2] == 3 and src.is_contiguous() and out.is_contiguous()
    H, W = int(src.shape[0]), int(src.shape[1])
    n = (out_w // tile) * (out_h // tile)
    assert out.shape[1:] == (3, tile, tile) and tile_index0 + n <= out.shape[0]
    kx, bx, cx = _bicubic_tables(W, out_w, src.device)
    ky, by, cy = _bicubic_tables(H, out_h, src.device)
    tmp = torch.empty((H, out_w, 3), dtype=torch.uint8, device=src.device)
    check(_lib.load().vila_resize_bicubic_tiles(_p(src), H, W, out_w, out_h, _p(cx), _p(bx), kx, _p(cy),
                                                _p(by), ky, _p(tmp), _p(out), tile, tile_index0, mean,
                                                std, _stream()), "vila_resize_bicubic_tiles")
    return out


def space_to_depth(x: torch.Tensor, h: int, w: int, r: int) -> torch.Tensor:
    """x [B, h*w, C] -> [B, ceil(h/r)*ceil(w/r), r*r*C]"""
    _chk(x, "x")
    assert x.is_contiguous() and x.dim() == 3 and x.shape[1] == h * w
    B, _, Cc = x.shape
    ho, wo = (h + r - 1) // r, (w + r - 1) // r
    out = torch.empty((B, ho * wo, r * r * Cc), dtype=torch.bfloat16, device=x.device)
    check(_lib.load().vila_space_to_depth(_p(x), _p(out), B, h, w, Cc, r, _stream()),
          "vila_space_to_depth")
    return out


def s2_merge(tiles: torch.Tensor, splits_h: Sequence[int], splits_w: Sequence[int], out_bh: int,
             out_bw: int, share_tile: bool = False) -> torch.Tensor:
    """tiles [n_tiles, side*side, C] of ONE image -> [out_bh*out_bw, side*side, n_scales*C]"""
    _chk(tiles, "tiles")
    assert tiles.is_contiguous() and tiles.dim() == 3
    n, N, Cc = tiles.shape
    side = int(round(N ** 0.5))
    ns = len(splits_h)
    out = torch.empty((out_bh * out_bw, N, ns * Cc), dtype=torch.bfloat16, device=tiles.device)
    sh = (C.c_int * ns)(*splits_h)
    sw = (C.c_int * ns)(*splits_w)
    check(_lib.load().vila_s2_merge(_p(tiles), _p(out), side, Cc, ns, sh, sw, out_bh, out_bw,
                                    1 if share_tile else 0, _stream()), "vila_s2_merge")
    return out


def chessboard_merge(tiles: torch.Tensor, bh: int, bw: int) -> torch.Tensor:
    """[bh*bw, s*s, C] -> [(bh*s)*(bw*s), C]"""
    _chk(tiles, "tiles")
    assert tiles.is_contiguous() and tiles.shape[0] == bh * bw
    _, N, Cc = tiles.shape
    s = int(round(N ** 0.5))
    out = torch.empty((bh * s * bw * s, Cc), dtype=torch.bfloat16, device=tiles.device)
    check(_lib.load().vila_chessboard_merge(_p(tiles), _p(out), bh, bw, s, Cc, _stream()),
          "vila_chessboard_merge")
    return out


def tsp_pool(x: torch.Tensor, pt: int, ph: int, pw: int) -> torch.Tensor:
    """x [T, h, w, C] -> [T/pt, h/ph, w/pw, C]"""
    _chk(x, "x")
    assert x.is_contiguous() and x.dim() == 4
    T, h, w, Cc = x.shape
    out = torch.empty((T // pt, h // ph, w // pw, Cc), dtype=torch.bfloat16, device=x.device)
    check(_lib.load().vila_tsp_pool(_p(x), _p(out), T, h, w, Cc, pt, ph, pw, _stream()),
          "vila_tsp_pool")
    return out


def embed_splice(table: torch.Tensor, media: Optional[torch.Tensor], src: torch.Tensor) -> torch.Tensor:
    _chk(table, "table")
    assert src.dtype == torch.int32 and src.is_cuda and table.is_contiguous()
    if media is not None:
        assert media.is_contiguous() and media.shape[-1] == table.shape[1]
    rows, cols = src.numel(), table.shape[1]
    out = torch.empty((rows, cols), dtype=torch.bfloat16, device=table.device)
    check(_lib.load().vila_embed_splice(_p(table), _p(media), _p(src), _p(out), rows, cols,
                                        _stream()), "vila_embed_splice")
    return out


def rope_kv_append(qkv: torch.Tensor, positions: torch.Tensor, Hq: int, Hkv: int, D: int,
                   inv_freq: torch.Tensor, k_pool: Optional[torch.Tensor] = None,
                   v_pool: Optional[torch.Tensor] = None, page_table: Optional[torch.Tensor] = None,
                   cache_pos0: int = 0) -> None:
    _chk(qkv, "qkv")
    assert qkv.is_contiguous() and qkv.shape[-1] == (Hq + 2 * Hkv) * D
    assert positions.dtype == torch.int32 and inv_freq.dtype == torch.float32
    S = qkv.shape[0]
    check(_lib.load().vila_rope_kv_append(_p(qkv), _p(positions), S, Hq, Hkv, D, _p(inv_freq),
                                          _p(k_pool), _p(v_pool), _p(page_table), cache_pos0,
                                          _stream()), "vila_rope_kv_append")


def rope_kv_append_table(qkv: torch.Tensor, table: torch.Tensor, Hq: int, Hkv: int, D: int,
                         k_pool: Optional[torch.Tensor] = None, v_pool: Optional[torch.Tensor] = None,
                         page_table: Optional[torch.Tensor] = None, cache_pos0: int = 0) -> None:
    """rope_kv_append with the cos | sin table of rope_table(positions) (long prefills)."""
    _chk(qkv, "qkv"); _chk(table, "table")
    assert qkv.is_contiguous() and qkv.shape[-1] == (Hq + 2 * Hkv) * D
    S = qkv.shape[0]
    assert table.shape == (S, D) and table.is_contiguous()
    check(_lib.load().vila_rope_kv_append_table(_p(qkv), _p(table), S, Hq, Hkv, D, _p(k_pool), _p(v_pool),
                                                _p(page_table), cache_pos0, _stream()),
          "vila_rope_kv_append_table")


def rope_table(positions: torch.Tensor, D: int, inv_freq: torch.Tensor) -> torch.Tensor:
    """cos | sin table [S, D] bf16 of a request's positions (shared by all layers and heads)."""
    assert positions.dtype == torch.int32 and inv_freq.dtype == torch.float32 and positions.is_cuda
    S = positions.numel()
    table = torch.empty((S, D), dtype=torch.bfloat16, device=positions.device)
    check(_lib.load().vila_rope_table(_p(positions), S, D, _p(inv_freq), _p(table), _stream()),
          "vila_rope_table")
    return table


def linear_qkv_rope(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor],
                    table: torch.Tensor, Hq: int, Hkv: int, D: int,
                    k_pool: Optional[torch.Tensor] = None, v_pool: Optional[torch.Tensor] = None,
                    page_table: Optional[torch.Tensor] = None, cache_pos0: int = 0,
                    static_w: bool = False) -> Optional[torch.Tensor]:
    """q/k/v projection + RoPE + KV-cache append in one kernel (short prefill chunks: M <= 384,
    head_dim 128; table = rope_table(positions)).  Returns qkv [M, (Hq+2Hkv)*D] whose q heads are
    rotated (k / v heads live in the pools when given), or None when the shape is not covered
    (caller: linear + rope_kv_append)."""
    _chk(x, "x"); _chk(w, "w")
    M, K = x.shape
    N = (Hq + 2 * Hkv) * D
    if D != 128 or M > 384 or M == 0:
        return None
    assert w.shape == (N, K) and x.stride(1) == 1 and w.stride(1) == 1
    assert table.shape == (M, D) and table.dtype == torch.bfloat16 and table.is_contiguous()
    ensure_workspace(x.device)
    out = torch.empty((M, N), dtype=torch.bfloat16, device=x.device)
    rc = _lib.load().vila_linear_qkv_rope(_p(x), x.stride(0), _p(w), w.stride(0), _p(bias), _p(out),
                                          out.stride(0), M, K, Hq, Hkv, D, _p(table),
                                          _p(k_pool), _p(v_pool), _p(page_table), cache_pos0,
                                          2 if static_w else 0, _stream())
    if rc == 3:
        return None
    check(rc, "vila_linear_qkv_rope")
    return out


def gemv(x: torch.Tensor, w: torch.Tensor, *, bias=None, norm_w=None, norm_eps: float = 1e-6,
         residual=None, swiglu: bool = False, out: Optional[torch.Tensor] = None,
         argmax_key: Optional[torch.Tensor] = None, write_out: bool = True,
         static_w: bool = False, variant: int = 0, w_scale: Optional[torch.Tensor] = None,
         w_zero: Optional[torch.Tensor] = None) -> Optional[torch.Tensor]:
    """y = W x with the fused RMSNorm prologue and bias / residual / SwiGLU / argmax epilogues.
    w bf16 [N, K]; or w torch.float8_e4m3fn [N, K] with w_scale fp32 [N] (one scale per row), which
    runs vila_gemv_fp8; or w uint8, the packed 4-bit codes of quantize_w4_groups, with w_scale bf16
    [N, K/128] and w_zero uint8 [N, K/128] (one scale and zero point per group of 128 k), which runs
    vila_gemv_w4a16.  The quantized forms are TMA-ring kernels only: variant=1 is refused."""
    fp8 = w.dtype == torch.float8_e4m3fn
    w4 = w.dtype == torch.uint8
    _chk(x, "x"); _chk(w, "w", w.dtype if fp8 or w4 else torch.bfloat16)
    if w4:
        if w_scale is None or w_zero is None:
            raise ValueError("gemv: packed 4-bit weights need w_scale (bf16 [N, K/128]) and w_zero (uint8 [N, K/128])")
        _chk(w_scale, "w_scale"); _chk(w_zero, "w_zero", torch.uint8)
        if w_scale.dim() != 2 or w_zero.shape != w_scale.shape or not (w_scale.is_contiguous() and w_zero.is_contiguous()):
            raise ValueError(f"gemv: w_scale and w_zero must be contiguous [N, K/128] tensors of one shape, got "
                             f"{tuple(w_scale.shape)} and {tuple(w_zero.shape)}")
        N, K = w_scale.shape[0], w_scale.shape[1] * 128
        if w.shape != ((N + 15) // 16, 8 * K) or not w.is_contiguous():
            raise ValueError(f"gemv: packed 4-bit weights of [{N}, {K}] must be a contiguous uint8 "
                             f"[{(N + 15) // 16}, {8 * K}] tensor, got {tuple(w.shape)}")
        if variant == 1:
            raise ValueError("gemv: the register-staged variant has no 4-bit form")
    elif w_zero is not None:
        raise ValueError("gemv: w_zero is only meaningful with packed 4-bit (uint8) weights")
    else:
        N, K = w.shape
    assert x.numel() == K and w.is_contiguous()
    if fp8:
        if w_scale is None:
            raise ValueError("gemv: float8_e4m3fn weights need w_scale (fp32 [N])")
        _chk(w_scale, "w_scale", torch.float32)
        if w_scale.shape != (N,) or not w_scale.is_contiguous():
            raise ValueError(f"gemv: w_scale must be a contiguous fp32 [{N}] tensor, got {tuple(w_scale.shape)}")
        if variant == 1:
            raise ValueError("gemv: the register-staged variant has no float8_e4m3fn form")
    elif w_scale is not None and not w4:
        raise ValueError("gemv: w_scale is only meaningful with float8_e4m3fn or packed 4-bit weights")
    if out is None and write_out:
        out = torch.empty((N // 2 if swiglu else N,), dtype=torch.bfloat16, device=x.device)
    p = GemvParams()
    p.x, p.w, p.bias, p.norm_w = _p(x), _p(w), _p(bias), _p(norm_w)
    p.norm_eps = norm_eps
    p.residual, p.y = _p(residual), _p(out)
    p.N, p.K, p.flags = N, K, (1 if swiglu else 0) | (2 if static_w else 0) | (4 if variant == 1 else 0)
    p.argmax_key = _p(argmax_key)
    if fp8:
        check(_lib.load().vila_gemv_fp8(C.byref(p), _p(w_scale), _stream()), "vila_gemv_fp8")
    elif w4:
        check(_lib.load().vila_gemv_w4a16(C.byref(p), _p(w_scale), _p(w_zero), _stream()), "vila_gemv_w4a16")
    else:
        check(_lib.load().vila_gemv(C.byref(p), _stream()), "vila_gemv")
    return out


GEMV_BATCH_MAX_M = 16  # activation rows per vila_gemv_batch_* launch


def gemv_batch(x: torch.Tensor, w: torch.Tensor, *, w_scale: torch.Tensor, w_zero: Optional[torch.Tensor] = None,
               bias: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None, swiglu: bool = False,
               out: Optional[torch.Tensor] = None, static_w: bool = False) -> torch.Tensor:
    """y[m] = epilogue(W x[m]) for the rows of x [M, K] on quantized weights, every weight byte read once per
    group of 16 rows: w torch.float8_e4m3fn [N, K] with w_scale fp32 [N] (vila_gemv_batch_fp8), or the
    packed 4-bit codes of quantize_w4_groups with w_scale bf16 [N, K/128] and w_zero uint8 [N, K/128]
    (vila_gemv_batch_w4a16).  Epilogue: bias, residual [M, N] (may be `out`: added in place) or SwiGLU on
    interleaved rows (out [M, N/2]).  M > 16 runs one launch per 16 rows; a row's result depends on that
    row alone, so it is the same for any M.  bf16 weights are refused: their batches run ops.linear."""
    fp8 = w.dtype == torch.float8_e4m3fn
    w4 = w.dtype == torch.uint8
    if not (fp8 or w4):
        raise ValueError(f"gemv_batch: weights must be float8_e4m3fn or packed 4-bit (uint8), got {w.dtype}; "
                         "bf16 batches run ops.linear")
    if w_scale is None:
        raise ValueError("gemv_batch: w_scale is required")
    if w4:
        if w_zero is None:
            raise ValueError("gemv_batch: packed 4-bit weights need w_scale (bf16 [N, K/128]) and w_zero (uint8 [N, K/128])")
        if w_scale.dim() != 2 or w_zero.shape != w_scale.shape or not (w_scale.is_contiguous() and w_zero.is_contiguous()):
            raise ValueError(f"gemv_batch: w_scale and w_zero must be contiguous [N, K/128] tensors of one shape, got "
                             f"{tuple(w_scale.shape)} and {tuple(w_zero.shape)}")
        N, K = w_scale.shape[0], w_scale.shape[1] * 128
        if w.shape != ((N + 15) // 16, 8 * K) or not w.is_contiguous():
            raise ValueError(f"gemv_batch: packed 4-bit weights of [{N}, {K}] must be a contiguous uint8 "
                             f"[{(N + 15) // 16}, {8 * K}] tensor, got {tuple(w.shape)}")
    else:
        if w_zero is not None:
            raise ValueError("gemv_batch: w_zero is only meaningful with packed 4-bit (uint8) weights")
        N, K = w.shape
        if w_scale.shape != (N,) or not w_scale.is_contiguous() or not w.is_contiguous():
            raise ValueError(f"gemv_batch: e4m3 weights need a contiguous fp32 w_scale [{N}], got {tuple(w_scale.shape)}")
    if x.dim() != 2 or x.shape[1] != K or x.stride(1) != 1:
        raise ValueError(f"gemv_batch: x must be [M, {K}] with unit column stride, got {tuple(x.shape)}")
    if swiglu and residual is not None:
        raise ValueError("gemv_batch: residual and swiglu do not combine")
    M = x.shape[0]
    n_out = N // 2 if swiglu else N
    if out is None:  # rows padded to a 16-byte multiple: the kernel takes such row strides only
        out = torch.empty((M, (n_out + 7) // 8 * 8), dtype=torch.bfloat16, device=x.device)[:, :n_out]
    else:
        if out.shape != (M, n_out) or out.stride(1) != 1:
            raise ValueError(f"gemv_batch: out must be [{M}, {n_out}] with unit column stride, got {tuple(out.shape)}")
    if residual is not None:
        if residual.shape != (M, N) or residual.stride(1) != 1:
            raise ValueError(f"gemv_batch: residual must be [{M}, {N}] with unit column stride, got {tuple(residual.shape)}")
    if bias is not None:
        if bias.shape != (N,) or not bias.is_contiguous():
            raise ValueError(f"gemv_batch: bias must be a contiguous [{N}] tensor, got {tuple(bias.shape)}")
    for t, name, dt in ((x, "x", torch.bfloat16), (w, "w", w.dtype), (out, "out", torch.bfloat16),
                        (w_scale, "w_scale", torch.bfloat16 if w4 else torch.float32), (w_zero, "w_zero", torch.uint8),
                        (residual, "residual", torch.bfloat16), (bias, "bias", torch.bfloat16)):
        if t is not None:
            _chk(t, name, dt)
    lib = _lib.load()
    for m0 in range(0, M, GEMV_BATCH_MAX_M):
        m1 = min(M, m0 + GEMV_BATCH_MAX_M)
        p = GemvBatchParams()
        p.x, p.ldx, p.w, p.bias = x[m0].data_ptr(), x.stride(0), _p(w), _p(bias)
        p.residual = None if residual is None else residual[m0].data_ptr()
        p.ld_res = 0 if residual is None else residual.stride(0)
        p.y, p.ldy = out[m0].data_ptr(), out.stride(0)
        p.M, p.N, p.K, p.flags = m1 - m0, N, K, (1 if swiglu else 0) | (2 if static_w else 0)
        if fp8:
            check(lib.vila_gemv_batch_fp8(C.byref(p), _p(w_scale), _stream()), "vila_gemv_batch_fp8")
        else:
            check(lib.vila_gemv_batch_w4a16(C.byref(p), _p(w_scale), _p(w_zero), _stream()), "vila_gemv_batch_w4a16")
    return out


def gemv_batch_partition(N: int, K: int, fp8: bool) -> dict:
    """the partition vila_gemv_batch_* use for (N, K) on the current device (vila_gemv_batch_partition)"""
    out = (C.c_int32 * 6)()
    check(_lib.load().vila_gemv_batch_partition(N, K, 1 if fp8 else 0, out), "vila_gemv_batch_partition")
    return dict(zip(("cluster", "ctas", "tiles_per_cluster", "parts", "max_active_clusters", "smem_bytes"), out))


def argmax_finalize(key: torch.Tensor, token_out: torch.Tensor, token_hist=None, step_counter=None,
                    position=None, embed_table=None, x_next=None) -> None:
    hidden = embed_table.shape[1] if embed_table is not None else 0
    check(_lib.load().vila_argmax_finalize(_p(key), _p(token_out), _p(token_hist),
                                           _p(step_counter), _p(position), _p(embed_table),
                                           _p(x_next), hidden, _stream()), "vila_argmax_finalize")


def decode_attention(qkv: torch.Tensor, position: torch.Tensor, k_pool: torch.Tensor,
                     v_pool: torch.Tensor, page_table: torch.Tensor, out: torch.Tensor,
                     ws: torch.Tensor, counters: torch.Tensor, inv_freq: torch.Tensor, Hq: int,
                     Hkv: int, D: int, num_splits: int, scale: float) -> None:
    p = DecodeAttnParams()
    p.qkv, p.position, p.k_pool, p.v_pool = _p(qkv), _p(position), _p(k_pool), _p(v_pool)
    p.page_table, p.out, p.ws, p.counters = _p(page_table), _p(out), _p(ws), _p(counters)
    p.inv_freq = _p(inv_freq)
    p.Hq, p.Hkv, p.D, p.num_splits, p.scale = Hq, Hkv, D, num_splits, scale
    check(_lib.load().vila_decode_attention(C.byref(p), _stream()), "vila_decode_attention")


def decode_attention_split(qkv: torch.Tensor, position: torch.Tensor, k_pool: torch.Tensor,
                           v_pool: torch.Tensor, page_table: torch.Tensor, out: torch.Tensor,
                           o_partial: torch.Tensor, lse: torch.Tensor, inv_freq: torch.Tensor, Hq: int,
                           Hkv: int, D: int, num_splits: int, split_tokens: int, scale: float,
                           counters: Optional[torch.Tensor] = None) -> None:
    """Long-context decode attention: RoPE + KV append, wgmma FMHA in split-KV mode, combine
    (counters int32 [Hkv], zeroed once: the combine is fused into the split kernel)."""
    assert o_partial.dtype == torch.float32 and o_partial.numel() >= num_splits * Hq * D
    assert lse.dtype == torch.float32 and lse.numel() >= num_splits * Hq
    p = DecodeAttnSplitParams()
    p.qkv, p.position, p.k_pool, p.v_pool = _p(qkv), _p(position), _p(k_pool), _p(v_pool)
    p.page_table, p.kv_num_pages, p.out = _p(page_table), k_pool.shape[0], _p(out)
    p.o_partial, p.lse, p.inv_freq = _p(o_partial), _p(lse), _p(inv_freq)
    p.counters = _p(counters)
    p.Hq, p.Hkv, p.D, p.num_splits, p.split_tokens, p.scale = Hq, Hkv, D, num_splits, split_tokens, scale
    check(_lib.load().vila_decode_attention_split(C.byref(p), _stream()), "vila_decode_attention_split")


def decode_attention_batch(qkv: torch.Tensor, positions: torch.Tensor, k_pool: torch.Tensor,
                           v_pool: torch.Tensor, page_tables: torch.Tensor, out: torch.Tensor,
                           inv_freq: torch.Tensor, Hq: int, Hkv: int, D: int, scale: float) -> None:
    """qkv [B, (Hq+2Hkv)*D], positions int32 [B] (< 0: idle slot), page_tables int32 [B, max_pages],
    out [B, Hq*D]; one shared paged pool [P, 128, Hkv, D]."""
    _chk(qkv, "qkv"); _chk(out, "out")
    B = qkv.shape[0]
    assert qkv.dim() == 2 and out.shape == (B, Hq * D) and qkv.stride(1) == 1 and out.stride(1) == 1
    assert positions.dtype == torch.int32 and positions.numel() == B and positions.is_contiguous()
    assert page_tables.dtype == torch.int32 and page_tables.dim() == 2 and page_tables.shape[0] == B
    p = DecodeAttnParams()
    p.qkv, p.position, p.k_pool, p.v_pool = _p(qkv), _p(positions), _p(k_pool), _p(v_pool)
    p.page_table, p.out, p.ws, p.counters = _p(page_tables), _p(out), None, None
    p.inv_freq = _p(inv_freq)
    p.Hq, p.Hkv, p.D, p.num_splits, p.scale = Hq, Hkv, D, 0, scale
    check(_lib.load().vila_decode_attention_batch(C.byref(p), B, qkv.stride(0), out.stride(0),
                                                  page_tables.stride(0), min(32, page_tables.shape[1]),
                                                  _stream()), "vila_decode_attention_batch")


def decode_attention_split_batch(qkv: torch.Tensor, positions: torch.Tensor, k_pool: torch.Tensor,
                                 v_pool: torch.Tensor, page_tables: torch.Tensor, out: torch.Tensor,
                                 o_partial: torch.Tensor, lse: torch.Tensor, counters: torch.Tensor,
                                 inv_freq: torch.Tensor, Hq: int, Hkv: int, D: int, num_splits: int,
                                 split_tokens: int, scale: float) -> None:
    """Long-context decode attention of B sequences over one shared paged pool [P, 128, Hkv, D]:
    qkv [B, (Hq+2Hkv)*D] (q / k rotated in place), positions int32 [B] (< 0: idle slot), page_tables
    int32 [B, pages] (pages of the slot's tokens; num_splits * split_tokens must cover them), out
    [B, Hq*D]; work buffers o_partial fp32 >= B*num_splits*Hq*D, lse fp32 >= B*num_splits*Hq, counters
    int32 [B*Hkv] (zeroed once, self-cleaning)."""
    _chk(qkv, "qkv"); _chk(out, "out")
    B = qkv.shape[0]
    assert qkv.dim() == 2 and out.shape == (B, Hq * D) and qkv.stride(1) == 1 and out.stride(1) == 1
    assert positions.dtype == torch.int32 and positions.numel() == B and positions.is_contiguous()
    assert page_tables.dtype == torch.int32 and page_tables.dim() == 2 and page_tables.shape[0] == B
    assert page_tables.stride(1) == 1
    assert o_partial.dtype == torch.float32 and o_partial.numel() >= B * num_splits * Hq * D
    assert lse.dtype == torch.float32 and lse.numel() >= B * num_splits * Hq
    assert counters.dtype == torch.int32 and counters.numel() >= B * Hkv
    p = DecodeAttnSplitParams()
    p.qkv, p.position, p.k_pool, p.v_pool = _p(qkv), _p(positions), _p(k_pool), _p(v_pool)
    p.page_table, p.kv_num_pages, p.out = _p(page_tables), k_pool.shape[0], _p(out)
    p.o_partial, p.lse, p.inv_freq, p.counters = _p(o_partial), _p(lse), _p(inv_freq), _p(counters)
    p.Hq, p.Hkv, p.D, p.num_splits, p.split_tokens, p.scale = Hq, Hkv, D, num_splits, split_tokens, scale
    check(_lib.load().vila_decode_attention_split_batch(C.byref(p), B, qkv.stride(0), out.stride(0),
                                                        page_tables.stride(0), _stream()),
          "vila_decode_attention_split_batch")


def _need(cond: bool, msg: str) -> None:
    if not cond:
        raise ValueError(msg)


def kv_quantize_fp8(src: torch.Tensor, dst: torch.Tensor, dst_scale: torch.Tensor, page_row: torch.Tensor,
                    S: int) -> None:
    """Rows [0, S) of every layer's K and V of a bf16 cache src [L, 2, pages, 128, Hkv, 128] (identity pages: a
    prefill's staging cache) -> the e4m3 pool dst [L, 2, P, 128, Hkv, 128] and its fp32 scales dst_scale
    [L, 2, P, 128, Hkv], token t going to page page_row[t // 128] (vila_kv_quantize_fp8, one launch).  The rule is
    quantize_kv_e4m3's (vila_b200/model/qwen2.py)."""
    _need(src.dim() == 6 and src.shape[1] == 2 and src.shape[3] == 128 and src.shape[5] == 128 and src.is_contiguous(),
          f"kv_quantize_fp8: src must be a contiguous [L, 2, pages, 128, Hkv, 128] cache, got {tuple(src.shape)}")
    L, _, ps, _, Hkv, D = src.shape
    _need(dst.dim() == 6 and dst.shape[:2] == (L, 2) and dst.shape[3:] == (128, Hkv, D) and dst.is_contiguous(),
          f"kv_quantize_fp8: dst must be a contiguous [{L}, 2, P, 128, {Hkv}, {D}] pool, got {tuple(dst.shape)}")
    _need(dst_scale.shape == dst.shape[:5] and dst_scale.is_contiguous(),
          f"kv_quantize_fp8: dst_scale must be a contiguous {tuple(dst.shape[:5])} tensor, got {tuple(dst_scale.shape)}")
    _need(page_row.dim() == 1 and page_row.is_contiguous(), "kv_quantize_fp8: page_row must be a contiguous 1-D row")
    _need(0 <= S <= ps * 128 and (S + 127) // 128 <= page_row.numel(),
          f"kv_quantize_fp8: S={S} exceeds the source ({ps * 128} tokens) or the page row ({page_row.numel()} pages)")
    for t, name, dt in ((src, "src", torch.bfloat16), (dst, "dst", torch.float8_e4m3fn),
                        (dst_scale, "dst_scale", torch.float32), (page_row, "page_row", torch.int32)):
        _need(t.dtype == dt, f"kv_quantize_fp8: {name} must be {dt}, got {t.dtype}")
    for t, name in ((src, "src"), (dst, "dst"), (dst_scale, "dst_scale"), (page_row, "page_row")):
        _chk(t, name, t.dtype)
    check(_lib.load().vila_kv_quantize_fp8(_p(src), ps * 128, _p(dst), _p(dst_scale), dst.shape[2], _p(page_row),
                                           page_row.numel(), L, Hkv, D, S, _stream()), "vila_kv_quantize_fp8")


def decode_attention_fp8_batch(qkv: torch.Tensor, positions: torch.Tensor, k_pool: torch.Tensor,
                               v_pool: torch.Tensor, k_scale: torch.Tensor, v_scale: torch.Tensor,
                               page_tables: torch.Tensor, out: torch.Tensor, ws: torch.Tensor, counters: torch.Tensor,
                               inv_freq: torch.Tensor, Hq: int, Hkv: int, num_splits: int, split_tokens: int,
                               scale: float) -> None:
    """One decode step of B sequences over one shared e4m3 pool (vila_decode_attention_fp8_batch): qkv
    [B, (Hq+2Hkv)*128] bf16 pre-RoPE (not modified), positions int32 [B] (< 0: idle slot), k_pool / v_pool e4m3
    [P, 128, Hkv, 128] with k_scale / v_scale fp32 [P, 128, Hkv], page_tables int32 [B, pages], out [B, Hq*128].
    RoPE, e4m3 append of the new row at positions[b], attention over [0, positions[b]]; split j covers tokens
    [j*split_tokens, (j+1)*split_tokens) and num_splits * split_tokens must exceed every position.  Work buffers:
    ws fp32 >= B*Hq*num_splits*130, counters int32 [B*Hkv] (zeroed once, self-cleaning)."""
    D = 128
    _need(Hq >= 1 and Hkv >= 1 and Hq % Hkv == 0 and Hq // Hkv <= 16,
          f"decode_attention_fp8_batch: Hq / Hkv must be an integer <= 16 (Hq={Hq}, Hkv={Hkv})")
    _need(qkv.dim() == 2 and qkv.shape[1] == (Hq + 2 * Hkv) * D and qkv.stride(1) == 1,
          f"decode_attention_fp8_batch: qkv must be [B, {(Hq + 2 * Hkv) * D}] with unit column stride "
          f"(head_dim 128), got {tuple(qkv.shape)}")
    B = qkv.shape[0]
    _need(out.shape == (B, Hq * D) and out.stride(1) == 1,
          f"decode_attention_fp8_batch: out must be [{B}, {Hq * D}], got {tuple(out.shape)}")
    _need(positions.numel() == B and positions.is_contiguous(), f"decode_attention_fp8_batch: positions must be [{B}]")
    _need(page_tables.dim() == 2 and page_tables.shape[0] == B and page_tables.stride(1) == 1,
          f"decode_attention_fp8_batch: page_tables must be [{B}, pages], got {tuple(page_tables.shape)}")
    for pool, sc, name in ((k_pool, k_scale, "k"), (v_pool, v_scale, "v")):
        _need(pool.dim() == 4 and pool.shape[1:] == (128, Hkv, D) and pool.is_contiguous(),
              f"decode_attention_fp8_batch: {name}_pool must be a contiguous [P, 128, {Hkv}, 128] pool, "
              f"got {tuple(pool.shape)}")
        _need(sc.shape == pool.shape[:3] and sc.is_contiguous(),
              f"decode_attention_fp8_batch: {name}_scale must be a contiguous {tuple(pool.shape[:3])} tensor")
    _need(split_tokens >= 128 and split_tokens % 128 == 0 and split_tokens <= 2048 and num_splits >= 1,
          f"decode_attention_fp8_batch: bad split configuration ({num_splits} x {split_tokens})")
    _need(ws.numel() >= B * Hq * num_splits * (D + 2) and counters.numel() >= B * Hkv,
          "decode_attention_fp8_batch: ws needs B*Hq*num_splits*130 floats and counters B*Hkv ints")
    for t, name, dt in ((qkv, "qkv", torch.bfloat16), (out, "out", torch.bfloat16), (positions, "positions", torch.int32),
                        (page_tables, "page_tables", torch.int32), (k_pool, "k_pool", torch.float8_e4m3fn),
                        (v_pool, "v_pool", torch.float8_e4m3fn), (k_scale, "k_scale", torch.float32),
                        (v_scale, "v_scale", torch.float32), (ws, "ws", torch.float32),
                        (counters, "counters", torch.int32), (inv_freq, "inv_freq", torch.float32)):
        _need(t.dtype == dt, f"decode_attention_fp8_batch: {name} must be {dt}, got {t.dtype}")
    for t in (qkv, out, positions, page_tables, k_pool, v_pool, k_scale, v_scale, ws, counters, inv_freq):
        _chk(t, "every tensor", t.dtype)
    p = DecodeAttnFp8Params()
    p.qkv, p.position, p.k_pool, p.v_pool = _p(qkv), _p(positions), _p(k_pool), _p(v_pool)
    p.k_scale, p.v_scale, p.page_table, p.out = _p(k_scale), _p(v_scale), _p(page_tables), _p(out)
    p.ws, p.counters, p.inv_freq = _p(ws), _p(counters), _p(inv_freq)
    p.Hq, p.Hkv, p.D, p.batch = Hq, Hkv, D, B
    p.qkv_stride, p.out_stride, p.pt_stride = qkv.stride(0), out.stride(0), page_tables.stride(0)
    p.num_splits, p.split_tokens, p.scale = num_splits, split_tokens, scale
    check(_lib.load().vila_decode_attention_fp8_batch(C.byref(p), _stream()), "vila_decode_attention_fp8_batch")


SAMPLE_MAX_VOCAB = 8 * 40960  # one cluster of 8 CTAs per row, each holding at most 40,960 fp32 scores


def sample_batch(logits: torch.Tensor, inv_temperature: torch.Tensor, top_k: torch.Tensor, top_p: torch.Tensor,
                 seed: torch.Tensor, step: torch.Tensor, positions: torch.Tensor, *, out: torch.Tensor,
                 n_kept: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The next token of each row of logits [M, V] bf16 (unit column stride, any row stride), drawn on the device by
    the rule of vila_b200/sampling.py (vila_sample_batch, one launch).  Per row: inv_temperature fp32 (0: greedy),
    top_k int32 (0: off), top_p fp32 (1: off), seed int64, step int64 (index t of the token), positions int32 (< 0:
    idle row, out untouched); out int64 [M]; n_kept int32 [M] or None gets the size of each row's kept set.  The
    parameter values live on the device and are validated where they are set (SamplingParams); the kernel reads
    inv_temperature <= 0 as greedy and top_k < 0 or >= V as off."""
    _need(logits.dim() == 2 and logits.stride(1) == 1 and logits.stride(0) >= logits.shape[1],
          f"sample_batch: logits must be [M, V] with unit column stride, got {tuple(logits.shape)} strides "
          f"{tuple(logits.stride())}")
    M, V = logits.shape
    _need(1 <= M <= 65535 and 1 <= V <= SAMPLE_MAX_VOCAB,
          f"sample_batch: M={M} must be in 1..65535 and V={V} in 1..{SAMPLE_MAX_VOCAB}")
    arrays = [(logits, "logits", torch.bfloat16), (inv_temperature, "inv_temperature", torch.float32),
              (top_k, "top_k", torch.int32), (top_p, "top_p", torch.float32), (seed, "seed", torch.int64),
              (step, "step", torch.int64), (positions, "positions", torch.int32), (out, "out", torch.int64)]
    if n_kept is not None:
        arrays.append((n_kept, "n_kept", torch.int32))
    for t, name, dt in arrays:
        _need(t.dtype == dt, f"sample_batch: {name} must be {dt}, got {t.dtype}")
        if t is not logits:
            _need(t.dim() == 1 and t.numel() == M and t.is_contiguous(),
                  f"sample_batch: {name} must be a contiguous [{M}] vector, got {tuple(t.shape)}")
    for t, name, _ in arrays:
        _chk(t, name, t.dtype)
    p = SampleParams()
    p.logits, p.ld = _p(logits), logits.stride(0)
    p.inv_temperature, p.top_k, p.top_p = _p(inv_temperature), _p(top_k), _p(top_p)
    p.seed, p.step, p.position, p.tokens, p.n_kept = _p(seed), _p(step), _p(positions), _p(out), _p(n_kept)
    p.M, p.V = M, V
    check(_lib.load().vila_sample_batch(C.byref(p), _stream()), "vila_sample_batch")
    return out


def sample_finalize(logits: torch.Tensor, inv_temperature: torch.Tensor, top_k: torch.Tensor, top_p: torch.Tensor,
                    seed: torch.Tensor, step: torch.Tensor, token_out: torch.Tensor, token_hist=None, position=None,
                    embed_table=None, x_next=None) -> None:
    """The single-stream decoder's end of a sampled step (vila_sample_finalize, one launch): the token of the bf16
    logits row [V] drawn by the rule of vila_b200/sampling.py with the device scalars inv_temperature fp32,
    top_k int32, top_p fp32 and seed int64 at token index t = step (int32 [1]); bit-identical to sample_batch with
    M = 1.  Then token_out (int32 [1]) = token, token_hist[t] = token (int32, optional), step + 1, position + 1
    (int32 [1], optional) and x_next = embed_table[token] (bf16 [*, hidden] and [hidden], optional, together)."""
    _need(logits.dim() == 1 and logits.is_contiguous() and 1 <= logits.numel() <= SAMPLE_MAX_VOCAB,
          f"sample_finalize: logits must be a contiguous [V] row with V in 1..{SAMPLE_MAX_VOCAB}, got "
          f"{tuple(logits.shape)}")
    _need((embed_table is None) == (x_next is None), "sample_finalize: embed_table and x_next go together")
    arrays = [(logits, "logits", torch.bfloat16), (inv_temperature, "inv_temperature", torch.float32),
              (top_k, "top_k", torch.int32), (top_p, "top_p", torch.float32), (seed, "seed", torch.int64),
              (step, "step", torch.int32), (token_out, "token_out", torch.int32)]
    for t, name, dt in ((position, "position", torch.int32), (token_hist, "token_hist", torch.int32),
                        (embed_table, "embed_table", torch.bfloat16), (x_next, "x_next", torch.bfloat16)):
        if t is not None:
            arrays.append((t, name, dt))
    for t, name, dt in arrays:
        _need(t.dtype == dt, f"sample_finalize: {name} must be {dt}, got {t.dtype}")
        if name in ("inv_temperature", "top_k", "top_p", "seed", "step", "token_out", "position"):
            _need(t.numel() == 1, f"sample_finalize: {name} must be a single value, got {tuple(t.shape)}")
    hidden = 0
    if embed_table is not None:
        hidden = embed_table.shape[-1]
        _need(embed_table.dim() == 2 and embed_table.is_contiguous() and x_next.numel() == hidden
              and x_next.is_contiguous(),
              f"sample_finalize: embed_table must be a contiguous [*, hidden] table and x_next a contiguous [hidden] "
              f"vector, got {tuple(embed_table.shape)} and {tuple(x_next.shape)}")
    for t, name, _ in arrays:
        _chk(t, name, t.dtype)
    p = SampleFinalizeParams()
    p.logits, p.inv_temperature, p.top_k, p.top_p, p.seed = (_p(logits), _p(inv_temperature), _p(top_k), _p(top_p),
                                                             _p(seed))
    p.step, p.position, p.token_out, p.token_hist = _p(step), _p(position), _p(token_out), _p(token_hist)
    p.embed_table, p.x_next = _p(embed_table), _p(x_next)
    p.V, p.hidden = logits.numel(), hidden
    check(_lib.load().vila_sample_finalize(C.byref(p), _stream()), "vila_sample_finalize")


def token_logprobs(logits: torch.Tensor, tokens: torch.Tensor, step: torch.Tensor, positions: torch.Tensor, *,
                   lp_hist: torch.Tensor, top_ids: Optional[torch.Tensor] = None,
                   top_lp: Optional[torch.Tensor] = None) -> None:
    """The log-probability of each row's chosen token and its n most likely alternatives, by the rule of
    vila_b200/logprobs.py (vila_token_logprobs, one launch).  logits [M, V] bf16 (unit column stride, any row stride);
    per row: tokens int64 (the chosen token), step int64 (the history column, clamped to cols - 1), positions int32
    (< 0: idle row, nothing written).  Outputs at column min(step, cols - 1) of each row: lp_hist fp32 [M, cols],
    top_ids int32 [M, cols, n] and top_lp fp32 [M, cols, n], best first (both None: n = 0)."""
    _need(logits.dim() == 2 and logits.stride(1) == 1 and logits.stride(0) >= logits.shape[1],
          f"token_logprobs: logits must be [M, V] with unit column stride, got {tuple(logits.shape)} strides "
          f"{tuple(logits.stride())}")
    M, V = logits.shape
    _need(1 <= M <= 65535 and 1 <= V <= SAMPLE_MAX_VOCAB,
          f"token_logprobs: M={M} must be in 1..65535 and V={V} in 1..{SAMPLE_MAX_VOCAB}")
    _need((top_ids is None) == (top_lp is None), "token_logprobs: top_ids and top_lp go together")
    _need(lp_hist.dim() == 2 and lp_hist.shape[0] == M and lp_hist.shape[1] >= 1 and lp_hist.is_contiguous(),
          f"token_logprobs: lp_hist must be a contiguous [{M}, cols] buffer, got {tuple(lp_hist.shape)}")
    cols = lp_hist.shape[1]
    n = 0 if top_ids is None else top_ids.shape[-1]
    arrays = [(logits, "logits", torch.bfloat16), (tokens, "tokens", torch.int64), (step, "step", torch.int64),
              (positions, "positions", torch.int32), (lp_hist, "lp_hist", torch.float32)]
    if top_ids is not None:
        for t, name in ((top_ids, "top_ids"), (top_lp, "top_lp")):
            _need(t.dim() == 3 and t.shape == (M, cols, n) and t.is_contiguous(),
                  f"token_logprobs: {name} must be a contiguous [{M}, {cols}, n] buffer, got {tuple(t.shape)}")
        _need(0 <= n <= 20 and n <= V, f"token_logprobs: n={n} must be in 0..20 and <= V={V}")
        arrays += [(top_ids, "top_ids", torch.int32), (top_lp, "top_lp", torch.float32)]
    for t, name, dt in arrays:
        _need(t.dtype == dt, f"token_logprobs: {name} must be {dt}, got {t.dtype}")
        if name in ("tokens", "step", "positions"):
            _need(t.dim() == 1 and t.numel() == M and t.is_contiguous(),
                  f"token_logprobs: {name} must be a contiguous [{M}] vector, got {tuple(t.shape)}")
    for t, name, _ in arrays:
        _chk(t, name, t.dtype)
    p = LogprobsParams()
    p.logits, p.ld, p.tokens, p.step, p.position = _p(logits), logits.stride(0), _p(tokens), _p(step), _p(positions)
    p.lp_hist = _p(lp_hist)
    p.top_ids, p.top_lp = (_p(top_ids), _p(top_lp)) if n else (None, None)
    p.M, p.V, p.cols, p.n = M, V, cols, n
    check(_lib.load().vila_token_logprobs(C.byref(p), _stream()), "vila_token_logprobs")


def apply_penalties(logits: torch.Tensor, history: torch.Tensor, step: torch.Tensor, positions: torch.Tensor,
                    presence: torch.Tensor, frequency: torch.Tensor, *, out: torch.Tensor) -> torch.Tensor:
    """OpenAI presence / frequency penalties by the rule of vila_b200/penalties.py (vila_apply_penalties, one launch).
    logits [M, V] bf16 (unit column stride, any row stride); history int64 [M, cols] (contiguous) of generated ids;
    per row: step int64 (t: history columns 0..min(t, cols) - 1 count), positions int32 (< 0: idle row, its output
    row is not written), presence and frequency fp32.  out: a contiguous bf16 [M, V] buffer.  -> out"""
    _need(logits.dim() == 2 and logits.stride(1) == 1 and logits.stride(0) >= logits.shape[1],
          f"apply_penalties: logits must be [M, V] with unit column stride, got {tuple(logits.shape)} strides "
          f"{tuple(logits.stride())}")
    M, V = logits.shape
    _need(1 <= M <= 65535 and 1 <= V <= SAMPLE_MAX_VOCAB,
          f"apply_penalties: M={M} must be in 1..65535 and V={V} in 1..{SAMPLE_MAX_VOCAB}")
    _need(history.dim() == 2 and history.shape[0] == M and history.shape[1] >= 1 and history.is_contiguous(),
          f"apply_penalties: history must be a contiguous [{M}, cols] buffer, got {tuple(history.shape)}")
    _need(out.shape == (M, V) and out.is_contiguous(),
          f"apply_penalties: out must be a contiguous [{M}, {V}] buffer, got {tuple(out.shape)}")
    arrays = [(logits, "logits", torch.bfloat16), (history, "history", torch.int64), (step, "step", torch.int64),
              (positions, "positions", torch.int32), (presence, "presence", torch.float32),
              (frequency, "frequency", torch.float32), (out, "out", torch.bfloat16)]
    for t, name, dt in arrays:
        _need(t.dtype == dt, f"apply_penalties: {name} must be {dt}, got {t.dtype}")
        if name in ("step", "positions", "presence", "frequency"):
            _need(t.dim() == 1 and t.numel() == M and t.is_contiguous(),
                  f"apply_penalties: {name} must be a contiguous [{M}] vector, got {tuple(t.shape)}")
    for t, name, _ in arrays:
        _chk(t, name, t.dtype)
    p = PenaltyParams()
    p.logits, p.ld, p.history, p.step, p.position = _p(logits), logits.stride(0), _p(history), _p(step), _p(positions)
    p.presence, p.frequency, p.out = _p(presence), _p(frequency), _p(out)
    p.M, p.V, p.cols = M, V, history.shape[1]
    check(_lib.load().vila_apply_penalties(C.byref(p), _stream()), "vila_apply_penalties")
    return out


LOGPROBS_ROW_CHUNK = 1152  # entries per CTA of vila_token_logprobs_row


def logprobs_row_workspace(V: int, device) -> tuple:
    """-> (workspace, counter): the scratch of token_logprobs_row for rows of V entries (one chunk's max, exp-sum and
    20 candidate keys per 1152 entries) and its zeroed arrival counter, which every launch leaves at zero"""
    chunks = (V + LOGPROBS_ROW_CHUNK - 1) // LOGPROBS_ROW_CHUNK
    return (torch.zeros(chunks * 21, dtype=torch.int64, device=device),
            torch.zeros(1, dtype=torch.int32, device=device))


def token_logprobs_row(logits: torch.Tensor, token: torch.Tensor, step: torch.Tensor, *, lp_hist: torch.Tensor,
                       workspace: torch.Tensor, counter: torch.Tensor, top_ids: Optional[torch.Tensor] = None,
                       top_lp: Optional[torch.Tensor] = None, n_used: Optional[torch.Tensor] = None) -> None:
    """token_logprobs' rule on one row, spread over one CTA per 1152 entries (vila_token_logprobs_row, one launch),
    for the single-stream graph decoder.  logits: a contiguous bf16 row [V]; token int32 [1] (the chosen token); step
    int32 [1], the decoder's counter already advanced past the token: the outputs go to column min(step - 1, cols - 1)
    of lp_hist fp32 [cols], top_ids int32 [cols, n] and top_lp fp32 [cols, n], best first (both None: n = 0).
    n_used: optional int32 [1] on the device, the number k of alternatives this launch computes (clamped to 0..n; the
    entries past k are not written), so that one captured launch serves every k up to n.
    workspace / counter: logprobs_row_workspace(V)."""
    _need(logits.dim() == 1 and logits.is_contiguous() and 1 <= logits.numel() <= SAMPLE_MAX_VOCAB,
          f"token_logprobs_row: logits must be a contiguous [V] row with V in 1..{SAMPLE_MAX_VOCAB}, got "
          f"{tuple(logits.shape)}")
    V = logits.numel()
    _need((top_ids is None) == (top_lp is None), "token_logprobs_row: top_ids and top_lp go together")
    _need(lp_hist.dim() == 1 and lp_hist.numel() >= 1 and lp_hist.is_contiguous(),
          f"token_logprobs_row: lp_hist must be a contiguous [cols] buffer, got {tuple(lp_hist.shape)}")
    cols = lp_hist.numel()
    n = 0 if top_ids is None else top_ids.shape[-1]
    need_ws = (V + LOGPROBS_ROW_CHUNK - 1) // LOGPROBS_ROW_CHUNK * 168
    arrays = [(logits, "logits", torch.bfloat16), (token, "token", torch.int32), (step, "step", torch.int32),
              (lp_hist, "lp_hist", torch.float32), (workspace, "workspace", torch.int64),
              (counter, "counter", torch.int32)]
    if n_used is not None:
        arrays.append((n_used, "n_used", torch.int32))
    if top_ids is not None:
        for t, name in ((top_ids, "top_ids"), (top_lp, "top_lp")):
            _need(t.dim() == 2 and t.shape == (cols, n) and t.is_contiguous(),
                  f"token_logprobs_row: {name} must be a contiguous [{cols}, n] buffer, got {tuple(t.shape)}")
        _need(0 <= n <= 20 and n <= V, f"token_logprobs_row: n={n} must be in 0..20 and <= V={V}")
        arrays += [(top_ids, "top_ids", torch.int32), (top_lp, "top_lp", torch.float32)]
    for t, name, dt in arrays:
        _need(t.dtype == dt, f"token_logprobs_row: {name} must be {dt}, got {t.dtype}")
        if name in ("token", "step", "counter", "n_used"):
            _need(t.numel() == 1, f"token_logprobs_row: {name} must be a single value, got {tuple(t.shape)}")
    _need(workspace.is_contiguous() and workspace.numel() * 8 >= need_ws,
          f"token_logprobs_row: workspace must be a contiguous buffer of at least {need_ws} bytes for V={V} "
          f"(logprobs_row_workspace), got {workspace.numel() * workspace.element_size()}")
    for t, name, _ in arrays:
        _chk(t, name, t.dtype)
    p = LogprobsRowParams()
    p.logits, p.token, p.step, p.lp_hist = _p(logits), _p(token), _p(step), _p(lp_hist)
    p.top_ids, p.top_lp = (_p(top_ids), _p(top_lp)) if n else (None, None)
    p.n_used = _p(n_used)
    p.workspace, p.workspace_bytes, p.counter = _p(workspace), workspace.numel() * 8, _p(counter)
    p.V, p.cols, p.n = V, cols, n
    check(_lib.load().vila_token_logprobs_row(C.byref(p), _stream()), "vila_token_logprobs_row")


def apply_penalties_row(logits: torch.Tensor, history: torch.Tensor, step: torch.Tensor, presence: torch.Tensor,
                        frequency: torch.Tensor, *, out: torch.Tensor) -> torch.Tensor:
    """apply_penalties' rule, bit for bit, on the single-stream graph decoder's one row (vila_apply_penalties_row, one
    launch).  logits: a contiguous bf16 row [V]; history int32 [cols] (contiguous) of generated ids; step int32 [1]
    (t: history entries 0..min(t, cols) - 1 count); presence and frequency fp32 [1].  out: a contiguous bf16 [V]
    buffer.  -> out"""
    _need(logits.dim() == 1 and logits.is_contiguous() and 1 <= logits.numel() <= SAMPLE_MAX_VOCAB,
          f"apply_penalties_row: logits must be a contiguous [V] row with V in 1..{SAMPLE_MAX_VOCAB}, got "
          f"{tuple(logits.shape)}")
    V = logits.numel()
    _need(history.dim() == 1 and history.numel() >= 1 and history.is_contiguous(),
          f"apply_penalties_row: history must be a contiguous [cols] buffer, got {tuple(history.shape)}")
    _need(out.shape == (V,) and out.is_contiguous(),
          f"apply_penalties_row: out must be a contiguous [{V}] buffer, got {tuple(out.shape)}")
    arrays = [(logits, "logits", torch.bfloat16), (history, "history", torch.int32), (step, "step", torch.int32),
              (presence, "presence", torch.float32), (frequency, "frequency", torch.float32),
              (out, "out", torch.bfloat16)]
    for t, name, dt in arrays:
        _need(t.dtype == dt, f"apply_penalties_row: {name} must be {dt}, got {t.dtype}")
        if name in ("step", "presence", "frequency"):
            _need(t.numel() == 1, f"apply_penalties_row: {name} must be a single value, got {tuple(t.shape)}")
    for t, name, _ in arrays:
        _chk(t, name, t.dtype)
    p = PenaltyRowParams()
    p.logits, p.history, p.step, p.presence, p.frequency = (_p(logits), _p(history), _p(step), _p(presence),
                                                           _p(frequency))
    p.out, p.V, p.cols = _p(out), V, history.numel()
    check(_lib.load().vila_apply_penalties_row(C.byref(p), _stream()), "vila_apply_penalties_row")
    return out


def apply_token_bitmask_row(logits: torch.Tensor, bitmask: torch.Tensor, *, out: torch.Tensor) -> torch.Tensor:
    """The single-stream decoder's logits row masked by a grammar matcher's token bitmask (vila_apply_token_bitmask_row,
    one launch; the rule of vila_b200/grammar.py): out[j] = logits[j] where bit j % 32 of bitmask[j // 32] is set,
    -inf elsewhere.  logits: a contiguous bf16 row [V]; bitmask: contiguous int32 with at least ceil(V / 32) words
    (xgrammar's layout; bits at or above V are ignored); out: a contiguous bf16 [V] buffer, logits itself for in
    place.  -> out"""
    _need(logits.dim() == 1 and logits.is_contiguous() and logits.numel() >= 1,
          f"apply_token_bitmask_row: logits must be a contiguous [V] row, got {tuple(logits.shape)}")
    V = logits.numel()
    W = (V + 31) // 32
    _need(bitmask.is_contiguous() and bitmask.numel() >= W,
          f"apply_token_bitmask_row: bitmask must be contiguous with at least {W} words, got {tuple(bitmask.shape)}")
    _need(out.shape == (V,) and out.is_contiguous(),
          f"apply_token_bitmask_row: out must be a contiguous [{V}] buffer, got {tuple(out.shape)}")
    arrays = [(logits, "logits", torch.bfloat16), (bitmask, "bitmask", torch.int32), (out, "out", torch.bfloat16)]
    for t, name, dt in arrays:
        _need(t.dtype == dt, f"apply_token_bitmask_row: {name} must be {dt}, got {t.dtype}")
    for t, name, _ in arrays:
        _chk(t, name, t.dtype)
    check(_lib.load().vila_apply_token_bitmask_row(_p(logits), _p(bitmask), _p(out), V, _stream()),
          "vila_apply_token_bitmask_row")
    return out


def prefix_block_hash(x: torch.Tensor, key0: int, key1: int) -> torch.Tensor:
    """The 128-bit digest of every full 128-row block of x [rows, cols] bf16 (unit column stride, any row stride that
    is a multiple of 4; cols a multiple of 4) under the 64-bit keys key0 / key1, by the rule of
    vila_b200/prefix_cache.py (vila_prefix_block_hash, one launch).  -> int64 [rows // 128, 2] on x's device, the
    uint64 digests' bits (.view(torch.uint64) or numpy .view(np.uint64) to read them unsigned)."""
    _need(x.dim() == 2 and x.stride(1) == 1 and (x.shape[0] <= 1 or x.stride(0) >= x.shape[1]),
          f"prefix_block_hash: x must be [rows, cols] with unit column stride, got {tuple(x.shape)} strides "
          f"{tuple(x.stride())}")
    _need(0 <= key0 < 2 ** 64 and 0 <= key1 < 2 ** 64, "prefix_block_hash: the keys are unsigned 64-bit integers")
    _chk(x, "x")
    rows, cols = x.shape
    out = torch.empty(rows // 128, 2, dtype=torch.int64, device=x.device)
    ld = x.stride(0) if rows > 1 else cols
    check(_lib.load().vila_prefix_block_hash(_p(x), ld, rows, cols, key0, key1, _p(out), _stream()),
          "vila_prefix_block_hash")
    return out


def pdl_late(snap: torch.Tensor, late: torch.Tensor, delay_ns: int) -> None:
    """Test hook (vila_test_pdl_late): a producer that lets the next launch start at once, spins delay_ns on the device,
    then copies every snap row and then every late row.  snap / late: int64 [n, 3] device tensors of (src, dst, bytes)
    rows (vila_pdl_copy)."""
    for t, name in ((snap, "snap"), (late, "late")):
        _need(t.dtype == torch.int64 and t.dim() == 2 and t.shape[1] == 3 and t.is_contiguous(),
              f"pdl_late: {name} must be a contiguous int64 [n, 3] tensor of (src, dst, bytes), got {tuple(t.shape)}")
        _chk(t, name, torch.int64)
    check(_lib.load().vila_test_pdl_late(_p(snap), snap.shape[0], _p(late), late.shape[0], delay_ns, _stream()),
          "vila_test_pdl_late")


def pdl_probe(flag: torch.Tensor, seen: torch.Tensor) -> None:
    """Test hook (vila_test_pdl_probe): seen[0] = flag[0] before the kernel's dependency wait, seen[1] = flag[0] after."""
    for t, name in ((flag, "flag"), (seen, "seen")):
        _need(t.dtype == torch.int32, f"pdl_probe: {name} must be int32, got {t.dtype}")
        _chk(t, name, torch.int32)
    _need(seen.numel() >= 2, "pdl_probe: seen needs two entries")
    check(_lib.load().vila_test_pdl_probe(_p(flag), _p(seen), None, _stream()), "vila_test_pdl_probe")


def pdl_enabled() -> bool:
    """Whether this process launches its kernels with programmatic dependent launch (VILA_B200_NO_PDL unset or not
    starting with '1'); read once per process.  Needs no device."""
    on = C.c_int(-1)
    check(_lib.load().vila_test_pdl_probe(None, None, C.byref(on), None), "vila_test_pdl_probe")
    return on.value == 1
