"""Kernel-level parity (GPU): every C-ABI entry point against the oracle's restatement of the
reference op on the same seeded inputs.  Reference math runs in fp32 on bf16-rounded inputs; the
tolerance is bf16 output rounding (2^-8 relative) plus accumulation-order noise:
    max|cuda - ref| <= 1.5e-2 * max|ref|      (stated per test where tighter)
Integer / pure-permutation kernels must be bit-exact.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import vila_oracle as O

pytestmark = pytest.mark.gpu


def _ops():
    from vila_b200 import ops
    ops.ensure_workspace("cuda")
    return ops


def bf(x):
    return x.to(torch.bfloat16)


def rel_err(a, b):
    return (a.float() - b.float()).abs().max().item() / max(b.float().abs().max().item(), 1e-6)


def rb(x):  # round-trip through bf16 (emulate the reference's bf16 tensor between ops)
    return x.to(torch.bfloat16).float()


# ------------------------------------------------------------------------------------------------
# GEMM
# ------------------------------------------------------------------------------------------------
def _tiles128(M, N):
    return ((M + 127) // 128) * ((N + 127) // 128)


GEMM_SHAPES = [
    (128, 128, 64), (256, 256, 128), (1024, 1152, 1152), (280, 3584, 3584), (1000, 4304, 1152),
    (1024, 1152, 4304), (2048, 1152, 592), (24, 512, 1536), (257, 3584, 4608), (130, 136, 72),
    (256, 512, 1088),  # odd number of k-blocks (17): uneven halves for the split-K pairs
]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
@pytest.mark.parametrize("block_n", [None, 64, 128, 256, 1064, 1128, 1256, 3000, 3001, 4128, 4256, 5128])  # 1000+: stream-K, 3000/3001: skinny single / CTA pair, 4xxx: CTA-pair tiles, 5128: split-K pairs
def test_linear_plain(cuda, M, N, K, block_n):
    if block_n in (3000, 3001) and M > 512:
        pytest.skip("skinny kernel handles M <= 512")
    if block_n == 5128 and (_tiles128(M, N) > 74 or K <= 64):
        pytest.skip("split-K pairs: one tile per SM pair, >= 2 k-blocks")
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    x = bf(torch.randn(M, K, device=cuda, generator=g))
    w = bf(torch.randn(N, K, device=cuda, generator=g) / math.sqrt(K))
    out = ops.linear(x, w, block_n=block_n)
    ref = x.float() @ w.float().t()
    assert rel_err(out, ref) < 8e-3, rel_err(out, ref)


@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("with_res", [False, True])
def test_linear_epilogues(cuda, act, with_res):
    ops = _ops()
    M, N, K = 300, 1152, 1152
    g = torch.Generator(device="cuda").manual_seed(5)
    x = bf(torch.randn(M, K, device=cuda, generator=g))
    w = bf(torch.randn(N, K, device=cuda, generator=g) / math.sqrt(K))
    b = bf(torch.randn(N, device=cuda, generator=g))
    res = bf(torch.randn(M, N, device=cuda, generator=g)) if with_res else None
    out = ops.linear(x, w, b, act=act, residual=res)
    ref = rb(x.float() @ w.float().t() + b.float())
    if act == 1:
        ref = rb(O.gelu_tanh(ref))
    elif act == 2:
        ref = rb(F.gelu(ref))
    if with_res:
        ref = rb(ref + res.float())
    assert rel_err(out, ref) < 1e-2


def test_linear_streamk_epilogues_and_workspace_is_clean(cuda):
    """stream-K partial tiles go through the fp32 workspace; the epilogue (bias, GELU, residual,
    SwiGLU) must be applied exactly once, results must be bit-reproducible and the tile counters
    must be left zeroed."""
    ops = _ops()
    ws = ops.ensure_workspace("cuda")
    g = torch.Generator(device="cuda").manual_seed(77)
    for (M, N, K) in [(279, 3584, 18944), (1024, 1152, 4304), (279, 1024, 2048)]:
        x = bf(torch.randn(M, K, device=cuda, generator=g))
        w = bf(torch.randn(N, K, device=cuda, generator=g) / math.sqrt(K))
        b = bf(torch.randn(N, device=cuda, generator=g))
        res = bf(torch.randn(M, N, device=cuda, generator=g))
        for bn in (1064, 1128, 1256, 4128, 4256) + ((3000, 3001) if M <= 512 else ()) + ((5128,) if _tiles128(M, N) <= 74 else ()):
            out = ops.linear(x, w, b, act=1, residual=res, block_n=bn, static_w=True)
            assert torch.equal(out, ops.linear(x, w, b, act=1, residual=res, block_n=bn, static_w=True))
            ref = rb(rb(O.gelu_tanh(rb(x.float() @ w.float().t() + b.float()))) + res.float())
            assert rel_err(out, ref) < 1e-2, (M, N, K, bn)
            out2 = ops.linear(x, w, swiglu=True, block_n=bn)
            gate = rb(x.float() @ w.float()[0::2].t())
            up = rb(x.float() @ w.float()[1::2].t())
            assert rel_err(out2, rb(rb(F.silu(gate)) * up)) < 1e-2
            torch.cuda.synchronize()
            assert int(ws[:65536].view(torch.int32).abs().max()) == 0  # tile counters self-clean
    # regular (non skinny) path for the same epilogues, M <= 512
    out = ops.linear(x, w, b, act=1, residual=res, block_n=2128)
    assert rel_err(out, ref) < 1e-2


@pytest.mark.parametrize("M", [1, 33, 279, 384])
def test_linear_qkv_rope_fused_equals_two_kernels(cuda, M):
    """vila_linear_qkv_rope (q/k/v projection with RoPE + paged KV append) must be bit-identical
    to vila_linear followed by vila_rope_kv_append (same rounding points), including the pool scatter
    through a permuted page table and a non-zero cache offset."""
    ops = _ops()
    Hq, Hkv, D, K = 6, 2, 128, 512
    N = (Hq + 2 * Hkv) * D
    g = torch.Generator(device="cuda").manual_seed(100 + M)
    x = bf(torch.randn(M, K, device=cuda, generator=g))
    w = bf(torch.randn(N, K, device=cuda, generator=g) / math.sqrt(K))
    b = bf(torch.randn(N, device=cuda, generator=g))
    p0 = 77
    pos = torch.arange(p0, p0 + M, dtype=torch.int32, device=cuda) * 3 + 5
    inv_freq = (1.0 / (1e6 ** (torch.arange(0, D, 2, dtype=torch.float32) / D))).to(cuda)
    n_pages = (p0 + M + 127) // 128 + 2
    table = torch.randperm(n_pages, generator=torch.Generator().manual_seed(1)).to(torch.int32).to(cuda)
    pools = [torch.zeros(n_pages, 128, Hkv, D, dtype=torch.bfloat16, device=cuda) for _ in range(4)]
    ref = ops.linear(x, w, b, block_n=3000)  # the same small-M GEMM, plain epilogue
    ops.rope_kv_append(ref, pos, Hq, Hkv, D, inv_freq, pools[0], pools[1], table, p0)
    tab = ops.rope_table(pos, D, inv_freq)
    got = ops.linear_qkv_rope(x, w, b, tab, Hq, Hkv, D, pools[2], pools[3], table, p0)
    assert got is not None
    assert torch.equal(got[:, :Hq * D], ref[:, :Hq * D])
    assert torch.equal(pools[2], pools[0]) and torch.equal(pools[3], pools[1])
    # without pools the rotated k and the plain v stay in the output buffer
    ref2 = ops.linear(x, w, b, block_n=3000)
    ops.rope_kv_append(ref2, pos, Hq, Hkv, D, inv_freq)
    assert torch.equal(ops.linear_qkv_rope(x, w, b, tab, Hq, Hkv, D), ref2)
    # not covered -> None (the caller falls back to the two kernels)
    assert ops.linear_qkv_rope(torch.zeros(400, K, dtype=torch.bfloat16, device=cuda), w, b,
                               torch.zeros(400, D, dtype=torch.bfloat16, device=cuda), Hq, Hkv, D) is None


def test_linear_chain_under_pdl(cuda):
    """Back-to-back dependent kernels (programmatic dependent launch): every consumer must wait for
    its producer; weights flagged static may be fetched early.  The chained run must equal, bit for
    bit, the same calls separated by synchronizes (and both must match the fp32 oracle)."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(78)
    x = bf(torch.randn(300, 1024, device=cuda, generator=g))
    ws_ = [bf(torch.randn(1024, 1024, device=cuda, generator=g) / 32) for _ in range(6)]
    nw = bf(torch.ones(1024, device=cuda))

    def chain(sync):
        h = x
        for w in ws_:
            h = ops.linear(ops.rmsnorm(h.clone(), nw, 1e-6), w, static_w=True)
            if sync:
                torch.cuda.synchronize()
        y = x.clone()
        for w in ws_:
            ops.linear(y.clone(), w, residual=y, out=y, static_w=True)
            if sync:
                torch.cuda.synchronize()
        return h, y

    torch.cuda.synchronize()
    h_sync, y_sync = chain(True)
    h, y = chain(False)
    torch.cuda.synchronize()
    assert torch.equal(h, h_sync) and torch.equal(y, y_sync)
    ref = x.float()
    r = x.float()
    for w in ws_:
        ref = rb(O.rms_norm(ref.to(torch.bfloat16), nw, 1e-6).float() @ w.float().t())
        r = rb(rb(r @ w.float().t()) + r)
    assert rel_err(h, ref) < 3e-2
    # in-place residual chains (out aliases residual)
    assert rel_err(y, r) < 3e-2


def test_linear_posemb_residual_and_strides(cuda):
    """patch-embed form: residual row = m % 1024 (position embedding), padded K, strided output."""
    ops = _ops()
    M, N, K = 2048, 1152, 592
    g = torch.Generator(device="cuda").manual_seed(6)
    x = bf(torch.randn(M, K, device=cuda, generator=g))
    w = bf(torch.randn(N, K, device=cuda, generator=g) / math.sqrt(K))
    b = bf(torch.randn(N, device=cuda, generator=g))
    pos = bf(torch.randn(1024, N, device=cuda, generator=g))
    big = torch.zeros(M, N + 64, dtype=torch.bfloat16, device=cuda)
    ops.linear(x, w, b, residual=pos, res_row_mod=1024, out=big[:, 32:32 + N])
    ref = rb(rb(x.float() @ w.float().t() + b.float()) + pos.float().repeat(2, 1))
    assert rel_err(big[:, 32:32 + N], ref) < 1e-2
    assert big[:, :32].abs().max() == 0 and big[:, 32 + N:].abs().max() == 0


def test_linear_swiglu(cuda):
    ops = _ops()
    M, I, K = 280, 2048, 1024
    g = torch.Generator(device="cuda").manual_seed(7)
    x = bf(torch.randn(M, K, device=cuda, generator=g))
    wg = bf(torch.randn(I, K, device=cuda, generator=g) / math.sqrt(K))
    wu = bf(torch.randn(I, K, device=cuda, generator=g) / math.sqrt(K))
    w = torch.stack([wg, wu], dim=1).reshape(2 * I, K).contiguous()  # interleaved rows
    out = ops.linear(x, w, swiglu=True)
    gate = rb(x.float() @ wg.float().t())
    up = rb(x.float() @ wu.float().t())
    ref = rb(rb(F.silu(gate)) * up)
    assert out.shape == (M, I)
    assert rel_err(out, ref) < 1e-2


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def ref_attention(q, k, v, causal, scale):
    """q [B,Sq,Hq,D], k/v [B,Sk,Hkv,D] fp32 -> [B,Sq,Hq,D]; softmax fp32, P cast to bf16 (reference).
    Heads are processed in groups only to bound the score tensor at long sequence lengths."""
    B, Sq, Hq, D = q.shape
    Sk, Hkv = k.shape[1], k.shape[2]
    rep = Hq // Hkv
    mask = None
    if causal:
        mask = torch.ones(Sq, Sk, dtype=torch.bool, device=q.device).tril(Sk - Sq)
    step = max(1, min(Hq, (1 << 29) // max(1, B * Sq * Sk)))
    out = torch.empty(B, Sq, Hq, D, dtype=torch.float32, device=q.device)
    for h0 in range(0, Hq, step):
        hs = list(range(h0, min(Hq, h0 + step)))
        qq = q[:, :, hs].permute(0, 2, 1, 3).float()
        kk = k[:, :, [h // rep for h in hs]].permute(0, 2, 1, 3).float()
        vv = v[:, :, [h // rep for h in hs]].permute(0, 2, 1, 3).float()
        att = qq @ kk.transpose(-1, -2) * scale
        if mask is not None:
            att = att.masked_fill(~mask, float("-inf"))
        p = rb(torch.softmax(att, dim=-1))
        out[:, :, hs] = (p @ vv).permute(0, 2, 1, 3)
        del att, p
    return out


@pytest.mark.parametrize("B,S,H,D", [(2, 1024, 16, 72), (1, 256, 2, 72), (3, 128, 4, 72), (1, 729, 3, 72)])
def test_fmha_noncausal_siglip(cuda, B, S, H, D):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(B * S + H)
    qkv = bf(torch.randn(B * S, 3, H, D, device=cuda, generator=g))
    q, k, v = qkv[:, 0], qkv[:, 1], qkv[:, 2]
    out = ops.fmha(q, k, v, B=B, Sq=S, Sk=S, causal=False, scale=D ** -0.5)
    ref = ref_attention(q.view(B, S, H, D), k.view(B, S, H, D), v.view(B, S, H, D), False, D ** -0.5)
    assert rel_err(out.view(B, S, H, D), ref) < 1.5e-2


@pytest.mark.parametrize("Sq,Sk,Hq,Hkv", [(280, 280, 28, 4), (128, 128, 4, 4), (1000, 1000, 8, 2),
                                          (300, 812, 14, 2), (1, 130, 4, 1)])
def test_fmha_causal_gqa(cuda, Sq, Sk, Hq, Hkv):
    ops = _ops()
    D = 128
    g = torch.Generator(device="cuda").manual_seed(Sq + Sk)
    q = bf(torch.randn(Sq, Hq, D, device=cuda, generator=g))
    k = bf(torch.randn(Sk, Hkv, D, device=cuda, generator=g))
    v = bf(torch.randn(Sk, Hkv, D, device=cuda, generator=g))
    out = ops.fmha(q, k, v, B=1, Sq=Sq, Sk=Sk, causal=True, scale=D ** -0.5)
    ref = ref_attention(q[None], k[None], v[None], True, D ** -0.5)[0]
    assert rel_err(out, ref) < 1.5e-2


def test_fmha_paged(cuda):
    ops = _ops()
    D, Hq, Hkv, Sq, Sk = 128, 8, 2, 200, 700
    g = torch.Generator(device="cuda").manual_seed(11)
    q = bf(torch.randn(Sq, Hq, D, device=cuda, generator=g))
    k = bf(torch.randn(Sk, Hkv, D, device=cuda, generator=g))
    v = bf(torch.randn(Sk, Hkv, D, device=cuda, generator=g))
    n_pages = 16
    perm = torch.randperm(n_pages, device=cuda, generator=g).to(torch.int32)
    k_pool = torch.zeros(n_pages, 128, Hkv, D, dtype=torch.bfloat16, device=cuda)
    v_pool = torch.zeros_like(k_pool)
    for j in range((Sk + 127) // 128):
        n = min(128, Sk - j * 128)
        k_pool[perm[j], :n] = k[j * 128:j * 128 + n]
        v_pool[perm[j], :n] = v[j * 128:j * 128 + n]
    out = ops.fmha(q, k_pool, v_pool, B=1, Sq=Sq, Sk=Sk, causal=True, scale=D ** -0.5,
                   page_table=perm.contiguous())
    ref = ref_attention(q[None], k[None], v[None], True, D ** -0.5)[0]
    assert rel_err(out, ref) < 1.5e-2


# ---- the attention kernel pinned through vila_fmha_cfg(variant=1) and the default dispatch --
@pytest.mark.parametrize("B", [1, 8, 64])
def test_fmha2_noncausal_siglip(cuda, B):
    from tests.helpers import report_rel
    ops = _ops()
    S, H, D = 1024, 16, 72
    g = torch.Generator(device="cuda").manual_seed(100 + B)
    qkv = bf(torch.randn(B * S, 3, H, D, device=cuda, generator=g))
    q, k, v = qkv[:, 0], qkv[:, 1], qkv[:, 2]
    ref = ref_attention(q.view(B, S, H, D), k.view(B, S, H, D), v.view(B, S, H, D), False, D ** -0.5)
    out1 = ops.fmha(q, k, v, B=B, Sq=S, Sk=S, causal=False, scale=D ** -0.5, variant=1)
    report_rel(f"fmha1 noncausal d=72 B={B}", out1.view(B, S, H, D), ref, 1.5e-2)
    auto = ops.fmha(q, k, v, B=B, Sq=S, Sk=S, causal=False, scale=D ** -0.5)
    assert torch.equal(auto, out1)  # the default dispatch runs the same kernel, bit-exact


@pytest.mark.parametrize("Sq,Sk", [(4096, 4096), (16448, 16448), (2048, 6000), (129, 129), (300, 812)])
def test_fmha2_causal_gqa_paged(cuda, Sq, Sk):
    """causal GQA d=128 over a PAGED, permuted KV pool: full prefill at 4K / 16.4K (64 video frames)
    and chunked prefill (Sq < Sk)."""
    from tests.helpers import report_rel
    ops = _ops()
    D, Hq, Hkv = 128, 28, 4
    g = torch.Generator(device="cuda").manual_seed(Sq + Sk)
    q = bf(torch.randn(Sq, Hq, D, device=cuda, generator=g))
    k = bf(torch.randn(Sk, Hkv, D, device=cuda, generator=g))
    v = bf(torch.randn(Sk, Hkv, D, device=cuda, generator=g))
    n_blk = (Sk + 127) // 128
    n_pages = n_blk + 5
    perm = torch.randperm(n_pages, device=cuda, generator=g).to(torch.int32).contiguous()
    k_pool = bf(torch.randn(n_pages, 128, Hkv, D, device=cuda, generator=g))  # garbage elsewhere
    v_pool = bf(torch.randn(n_pages, 128, Hkv, D, device=cuda, generator=g))
    kp = torch.zeros(n_blk * 128, Hkv, D, dtype=torch.bfloat16, device=cuda)
    vp = torch.zeros_like(kp)
    kp[:Sk], vp[:Sk] = k, v
    k_pool[perm[:n_blk].long()] = kp.view(n_blk, 128, Hkv, D)
    v_pool[perm[:n_blk].long()] = vp.view(n_blk, 128, Hkv, D)
    ref = ref_attention(q[None], k[None], v[None], True, D ** -0.5)[0]
    out1 = ops.fmha(q, k_pool, v_pool, B=1, Sq=Sq, Sk=Sk, causal=True, scale=D ** -0.5,
                    page_table=perm, variant=1)
    report_rel(f"fmha1 causal GQA paged Sq={Sq} Sk={Sk}", out1, ref, 1.5e-2)


def test_fmha2_lazy_rescale_growing_maxima(cuda):
    """Scores that keep growing along the KV axis: every KV block raises the row maxima, some by a
    lot and some by little, so the O rescale runs with factors far from and close to 1; d=72 and d=128."""
    from tests.helpers import report_rel
    ops = _ops()
    for (D, H, Hkv, S, causal) in [(128, 8, 2, 2048, True), (72, 16, 16, 1024, False)]:
        g = torch.Generator(device="cuda").manual_seed(D)
        q = bf(torch.randn(S, H, D, device=cuda, generator=g))
        ramp = torch.linspace(0.2, 6.0, S, device=cuda)[:, None, None]       # |k| grows with position
        k = bf(torch.randn(S, Hkv, D, device=cuda, generator=g) * ramp)
        v = bf(torch.randn(S, Hkv, D, device=cuda, generator=g))
        ref = ref_attention(q[None], k[None], v[None], causal, D ** -0.5)[0]
        for variant in (1, 3, 4):  # 3 / 4: every 4th / 2nd exp2 as a polynomial
            out = ops.fmha(q, k, v, B=1, Sq=S, Sk=S, causal=causal, scale=D ** -0.5, variant=variant)
            assert torch.isfinite(out.float()).all()
            report_rel(f"fmha{variant} growing maxima d={D}", out, ref, 1.5e-2)


def test_rope_kv_append(cuda):
    ops = _ops()
    S, Hq, Hkv, D = 37, 4, 2, 128
    g = torch.Generator(device="cuda").manual_seed(16)
    qkv = bf(torch.randn(S, (Hq + 2 * Hkv) * D, device=cuda, generator=g))
    pos = torch.arange(60000, 60000 + S, dtype=torch.int32, device=cuda)
    inv = O.rope_inv_freq(D, 1e6).to(cuda)
    pt = torch.tensor([3, 1], dtype=torch.int32, device=cuda)
    k_pool = torch.zeros(4, 128, Hkv, D, dtype=torch.bfloat16, device=cuda)
    v_pool = torch.zeros_like(k_pool)
    work = qkv.clone()
    ops.rope_kv_append(work, pos, Hq, Hkv, D, inv, k_pool, v_pool, pt, cache_pos0=100)
    q = qkv[:, :Hq * D].view(S, Hq, D).transpose(0, 1)
    k = qkv[:, Hq * D:(Hq + Hkv) * D].view(S, Hkv, D).transpose(0, 1)
    cos, sin = O.rope_cos_sin(pos.cpu().long(), D, 1e6, torch.bfloat16)
    qr, kr = O.apply_rope(q, k, cos.to(cuda), sin.to(cuda))
    got_q = work[:, :Hq * D].view(S, Hq, D).transpose(0, 1)
    got_k = work[:, Hq * D:(Hq + Hkv) * D].view(S, Hkv, D).transpose(0, 1)
    assert rel_err(got_q, qr) < 2 ** -6 and rel_err(got_k, kr) < 2 ** -6
    assert (got_q.float() - qr.float()).abs().mean().item() < 2e-3
    # cache contents: positions 100..136 -> page pt[0] rows 100..127, page pt[1] rows 0..8
    v = qkv[:, (Hq + Hkv) * D:].view(S, Hkv, D)
    assert torch.equal(v_pool[3, 100:128], v[:28]) and torch.equal(v_pool[1, :9], v[28:])
    assert torch.equal(k_pool[3, 100:128], got_k.transpose(0, 1)[:28])
    # table-driven vectorised variant (long prefills): bit-identical, qkv and both pools
    k2, v2, work2 = torch.zeros_like(k_pool), torch.zeros_like(v_pool), qkv.clone()
    ops.rope_kv_append_table(work2, ops.rope_table(pos, D, inv), Hq, Hkv, D, k2, v2, pt, cache_pos0=100)
    assert torch.equal(work2, work) and torch.equal(k2, k_pool) and torch.equal(v2, v_pool)
    # decode form: cache slot = the position itself (cache_pos0 < 0), one row
    k3, v3 = torch.zeros_like(k_pool), torch.zeros_like(v_pool)
    one = qkv[:1].clone()
    ops.rope_kv_append(one, torch.tensor([130], dtype=torch.int32, device=cuda), Hq, Hkv, D, inv, k3, v3, pt, cache_pos0=-1)
    assert k3[1, 2].abs().sum() > 0 and v3[1, 2].abs().sum() > 0 and k3[3].abs().sum() == 0


# ------------------------------------------------------------------------------------------------
# decode kernels
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", [0, 1])  # 0: TMA-ring kernel, 1: register-staged kernel
@pytest.mark.parametrize("N,K", [(4608, 3584), (3584, 3584), (3584, 18944), (512, 2048), (1000, 1536),
                                 (152064, 3584), (37888, 3584), (64, 512)])
def test_gemv_bias_residual_norm(cuda, N, K, variant):
    from tests.helpers import check_gemv, gemv_plan
    ops = _ops()
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    g = torch.Generator(device="cuda").manual_seed(N + K)
    x = bf(torch.randn(K, device=cuda, generator=g))
    w = bf(torch.randn(N, K, device=cuda, generator=g) / math.sqrt(K))
    b = bf(torch.randn(N, device=cuda, generator=g))
    r = bf(torch.randn(N, device=cuda, generator=g))
    nw = bf(torch.randn(K, device=cuda, generator=g))
    out = ops.gemv(x, w, bias=b, residual=r, variant=variant, static_w=True)
    assert torch.equal(out, ops.gemv(x, w, bias=b, residual=r, variant=variant))  # deterministic
    _, depth, regime = gemv_plan("bf16", N, K, "bias+residual", sms, variant=variant)
    e = check_gemv(f"gemv bias+residual N={N} K={K} v{variant}", out[None], x[None], w, N, depth=depth, bias=b,
                   residual=r[None], record=dict(regime=regime))
    assert not e.failures(), e.failures()
    out = ops.gemv(x, w, norm_w=nw, norm_eps=1e-6, variant=variant)
    _, depth, regime = gemv_plan("bf16", N, K, "norm", sms, variant=variant)
    e = check_gemv(f"gemv norm N={N} K={K} v{variant}", out[None], x[None], w, N, depth=depth, norm_w=nw,
                   record=dict(regime=regime))
    assert not e.failures(), e.failures()


@pytest.mark.parametrize("variant", [0, 1])
def test_gemv_swiglu(cuda, variant):
    from tests.helpers import check_gemv, gemv_plan
    ops = _ops()
    I, K = 18944, 3584
    g = torch.Generator(device="cuda").manual_seed(21)
    x = bf(torch.randn(K, device=cuda, generator=g))
    wg = bf(torch.randn(I, K, device=cuda, generator=g) / math.sqrt(K))
    wu = bf(torch.randn(I, K, device=cuda, generator=g) / math.sqrt(K))
    w = torch.stack([wg, wu], dim=1).reshape(2 * I, K).contiguous()
    out = ops.gemv(x, w, swiglu=True, variant=variant, static_w=True)
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    _, depth, regime = gemv_plan("bf16", 2 * I, K, "swiglu", sms, variant=variant)
    e = check_gemv(f"gemv swiglu v{variant}", out[None], x[None], w, 2 * I, depth=depth, swiglu=True,
                   record=dict(regime=regime))
    assert not e.failures(), e.failures()


def test_gemv_argmax_and_finalize(cuda):
    from tests.helpers import check_gemv, gemv_plan
    ops = _ops()
    V, K = 152064, 3584
    g = torch.Generator(device="cuda").manual_seed(22)
    x = bf(torch.randn(K, device=cuda, generator=g))
    w = bf(torch.randn(V, K, device=cuda, generator=g) * 0.02)
    key = torch.zeros(1, dtype=torch.int64, device=cuda)
    logits = ops.gemv(x, w, argmax_key=key)
    tok = torch.zeros(1, dtype=torch.int32, device=cuda)
    hist = torch.zeros(8, dtype=torch.int32, device=cuda)
    step = torch.zeros(1, dtype=torch.int32, device=cuda)
    posn = torch.full((1,), 41, dtype=torch.int32, device=cuda)
    table = bf(torch.randn(V, 64, device=cuda, generator=g))
    xn = torch.zeros(64, dtype=torch.bfloat16, device=cuda)
    ops.argmax_finalize(key, tok, hist, step, posn, table, xn)
    # the kernel's own logits decide (ties -> lowest index, like torch.argmax)
    expect = int(torch.argmax(logits.float()))
    assert int(tok) == expect and int(hist[0]) == expect and int(step) == 1 and int(posn) == 42
    assert int(key) == 0 and torch.equal(xn, table[expect])
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    _, depth, regime = gemv_plan("bf16", V, K, "argmax", sms)
    e = check_gemv("gemv argmax lm_head", logits[None], x[None], w, V, depth=depth, record=dict(regime=regime))
    assert not e.failures(), e.failures()
    ref = w.float() @ x.float()
    top2 = torch.topk(ref, 2).values
    if (top2[0] - top2[1]) > 0.05:
        assert expect == int(torch.argmax(ref))


_DECODE_CASES = [(0, 1), (5, 1), (300, 4), (1000, 8), (130, 16),
                 (0, 0), (5, 0), (127, 0), (128, 0), (300, 0), (407, 0), (1023, 0),  # 0: one CTA per query head
                 (16448, 37), (16448, 64), (65814, 37), (65814, 64), (4000, 8)]
# GQA groups of the decoder's models: G=7 (NVILA-8B), G=8 (NVILA-Lite-3B), G=2 (the tiny test model);
# splits 0 (one CTA per query head), 8 (one cluster per KV head), 16 (global-memory combine)
_DECODE_GQA_CASES = [(ctx, s, hq, hkv) for hq, hkv in ((28, 4), (16, 2), (4, 2)) for s in (0, 8, 16)
                     for ctx in (5, 300, 1000) if not (hq == 28 and (ctx, s) in _DECODE_CASES)]


@pytest.mark.parametrize("ctx,splits,Hq,Hkv",
                         [pytest.param(c, s, 28, 4, id=f"{c}-{s}") for c, s in _DECODE_CASES] +
                         [pytest.param(*case, id="-".join(map(str, case))) for case in _DECODE_GQA_CASES])
def test_decode_attention(cuda, ctx, splits, Hq, Hkv):
    """(16448, *) / (65814, *): decode right after a 64-frame / 256-frame video prefill (README.md:69-70
    publishes decode throughput for exactly that), splits as GraphDecoder.pick_splits chooses them."""
    from tests.helpers import check_decode_attention
    ops = _ops()
    D = 128
    g = torch.Generator(device="cuda").manual_seed(ctx + splits)
    n_pages = max(16, (ctx + 1 + 127) // 128 + 3)
    perm = torch.randperm(n_pages, device=cuda, generator=g).to(torch.int32).contiguous()
    k_hist = bf(torch.randn(ctx, Hkv, D, device=cuda, generator=g))
    v_hist = bf(torch.randn(ctx, Hkv, D, device=cuda, generator=g))
    k_pool = torch.zeros(n_pages, 128, Hkv, D, dtype=torch.bfloat16, device=cuda)
    v_pool = torch.zeros_like(k_pool)
    n_blk = (ctx + 127) // 128
    if n_blk:
        kp = torch.zeros(n_blk * 128, Hkv, D, dtype=torch.bfloat16, device=cuda)
        vp = torch.zeros_like(kp)
        kp[:ctx], vp[:ctx] = k_hist, v_hist
        k_pool[perm[:n_blk].long()] = kp.view(n_blk, 128, Hkv, D)
        v_pool[perm[:n_blk].long()] = vp.view(n_blk, 128, Hkv, D)
    qkv = bf(torch.randn((Hq + 2 * Hkv) * D, device=cuda, generator=g))
    pos = torch.tensor([ctx], dtype=torch.int32, device=cuda)
    inv = O.rope_inv_freq(D, 1e6).to(cuda)
    out = torch.zeros(Hq * D, dtype=torch.bfloat16, device=cuda)
    ws = torch.zeros(Hkv * splits * (Hq // Hkv) * (D + 2), dtype=torch.float32, device=cuda)
    counters = torch.zeros(Hkv, dtype=torch.int32, device=cuda)
    for _ in range(2):  # twice: counters must re-arm themselves
        out.zero_()
        ops.decode_attention(qkv, pos, k_pool, v_pool, perm, out, ws, counters, inv, Hq, Hkv, D,
                             splits, D ** -0.5)
    q = qkv[:Hq * D].view(1, Hq, D).transpose(0, 1)
    kn = qkv[Hq * D:(Hq + Hkv) * D].view(1, Hkv, D).transpose(0, 1)
    vn = qkv[(Hq + Hkv) * D:].view(1, Hkv, D)
    cos, sin = O.rope_cos_sin(torch.tensor([ctx]), D, 1e6, torch.bfloat16)
    qr, kr = O.apply_rope(q, kn, cos.to(cuda), sin.to(cuda))
    k_all = torch.cat([k_hist, kr.transpose(0, 1)], 0)
    v_all = torch.cat([v_hist, vn], 0)
    check_decode_attention(f"decode_attention Hq={Hq} Hkv={Hkv} ctx={ctx} splits={splits}", out.view(Hq, D),
                           qr.transpose(0, 1), k_all, v_all, D ** -0.5)
    # KV append happened
    assert torch.equal(k_pool[perm[ctx // 128], ctx % 128], kr.transpose(0, 1)[0])
    assert torch.equal(v_pool[perm[ctx // 128], ctx % 128], vn[0])
    assert int(counters.abs().sum()) == 0


# ------------------------------------------------------------------------------------------------
# preprocessing kernel (f2): bit-exact vs PIL bicubic + SiglipImageProcessor arithmetic
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", [(640, 480), (1600, 800), (97, 131), (3000, 500), (448, 448), (333, 1000)])
@pytest.mark.parametrize("mode", ["resize", "dynamic", "dynamic_s2", "pad"])
def test_preprocess_tiles_bit_exact_vs_pil(cuda, w, h, mode):
    """vila_resize_bicubic_tiles through media.process_image_gpu == PIL resize + crop + x/255 +
    (x-0.5)/0.5 + .to(bf16) (media.process_image, validated against the reference's mm_utils and
    SiglipImageProcessor), and == the numpy oracle of Pillow's resampler."""
    import numpy as np
    from PIL import Image as PILImage
    from oracle import pil_resample as R
    from vila_b200.model import LlavaConfig, media
    _ops()
    cfg = LlavaConfig(image_aspect_ratio=mode, dynamic_s2=(mode == "dynamic_s2"))
    img = PILImage.fromarray(np.random.RandomState(w * 3 + h).randint(0, 256, (h, w, 3), dtype=np.uint8))
    if mode == "dynamic_s2":
        want, bs = media.process_image(img, cfg, enable_dynamic_s2=True)
        got, bs2 = media.process_image_gpu(img, cfg)
        assert tuple(bs) == tuple(bs2)
    elif mode == "dynamic":
        want = media.process_image(img, cfg, enable_dynamic_res=True)
        got = media.process_image_gpu(img, cfg)
    else:
        want = media.process_image(img, cfg)[None]
        got = media.process_image_gpu(img, cfg)
    assert got.shape == want.shape and got.dtype == torch.bfloat16
    assert torch.equal(got.cpu(), want.to(torch.bfloat16))
    if mode == "resize":  # and against the oracle of the resampler directly
        u8 = R.resize_bicubic_u8(np.asarray(img), 448, 448)
        assert torch.equal(got[0].cpu(), torch.from_numpy(R.siglip_normalise(u8)).to(torch.bfloat16))


@pytest.mark.parametrize("ctx,splits,split_tokens", [(130, 2, 128), (3000, 12, 256), (16448, 33, 512),
                                                     (65814, 37, 1792), (65814, 64, 1152), (1000, 37, 512)])
def test_decode_attention_split_long_context(cuda, ctx, splits, split_tokens):
    """vila_decode_attention_split (RoPE + append, wgmma FMHA in split-KV mode, combine) vs fp32
    attention over the whole context; (1000, 37, 512): most splits are empty."""
    from tests.helpers import check_decode_attention, report_rel
    ops = _ops()
    Hq, Hkv, D = 28, 4, 128
    assert splits * split_tokens >= ctx + 1
    g = torch.Generator(device="cuda").manual_seed(ctx + splits)
    n_blk = (ctx + 127) // 128
    n_pages = (ctx + 1 + 127) // 128 + 3
    perm = torch.randperm(n_pages, device=cuda, generator=g).to(torch.int32).contiguous()
    k_hist = bf(torch.randn(ctx, Hkv, D, device=cuda, generator=g))
    v_hist = bf(torch.randn(ctx, Hkv, D, device=cuda, generator=g))
    k_pool = bf(torch.randn(n_pages, 128, Hkv, D, device=cuda, generator=g))  # garbage beyond ctx
    v_pool = bf(torch.randn(n_pages, 128, Hkv, D, device=cuda, generator=g))
    kp = torch.zeros(n_blk * 128, Hkv, D, dtype=torch.bfloat16, device=cuda)
    vp = torch.zeros_like(kp)
    kp[:ctx], vp[:ctx] = k_hist, v_hist
    tail_k = k_pool[perm[n_blk - 1].long(), ctx % 128:].clone() if ctx % 128 else None
    k_pool[perm[:n_blk].long()] = kp.view(n_blk, 128, Hkv, D)
    v_pool[perm[:n_blk].long()] = vp.view(n_blk, 128, Hkv, D)
    if tail_k is not None:  # keep garbage (not zeros) after the last cached token of the last page
        k_pool[perm[n_blk - 1].long(), ctx % 128:] = tail_k
    qkv0 = bf(torch.randn((Hq + 2 * Hkv) * D, device=cuda, generator=g))
    pos = torch.tensor([ctx], dtype=torch.int32, device=cuda)
    inv = O.rope_inv_freq(D, 1e6).to(cuda)
    out = torch.zeros(Hq * D, dtype=torch.bfloat16, device=cuda)
    o_partial = torch.zeros(splits * Hq * D, dtype=torch.float32, device=cuda)
    lse = torch.zeros(splits * Hq, dtype=torch.float32, device=cuda)
    qkv = qkv0.clone()
    ops.decode_attention_split(qkv, pos, k_pool, v_pool, perm, out, o_partial, lse, inv, Hq, Hkv, D, splits,
                               split_tokens, D ** -0.5)
    # fused combine (last split CTA of a KV head merges): same result bit for bit, counters re-armed
    out_f = torch.zeros_like(out)
    cnt_f = torch.zeros(Hkv, dtype=torch.int32, device=cuda)
    for _ in range(2):
        kp2, vp2 = k_pool.clone(), v_pool.clone()
        ops.decode_attention_split(qkv0.clone(), pos, kp2, vp2, perm, out_f, o_partial, lse, inv, Hq, Hkv, D,
                                   splits, split_tokens, D ** -0.5, counters=cnt_f)
        assert torch.equal(out_f, out) and int(cnt_f.abs().sum()) == 0
    q = qkv0[:Hq * D].view(1, Hq, D).transpose(0, 1)
    kn = qkv0[Hq * D:(Hq + Hkv) * D].view(1, Hkv, D).transpose(0, 1)
    vn = qkv0[(Hq + Hkv) * D:].view(1, Hkv, D)
    cos, sin = O.rope_cos_sin(torch.tensor([ctx]), D, 1e6, torch.bfloat16)
    qr, kr = O.apply_rope(q, kn, cos.to(cuda), sin.to(cuda))
    k_all = torch.cat([k_hist, kr.transpose(0, 1)], 0)
    v_all = torch.cat([v_hist, vn], 0)
    ref = ref_attention(qr.transpose(0, 1)[None], k_all[None], v_all[None], True, D ** -0.5)[0, 0]
    check_decode_attention(f"decode_attention_split ctx={ctx} splits={splits}", out.view(Hq, D), qr.transpose(0, 1),
                           k_all, v_all, D ** -0.5)
    assert torch.equal(k_pool[perm[ctx // 128], ctx % 128], kr.transpose(0, 1)[0])
    assert torch.equal(v_pool[perm[ctx // 128], ctx % 128], vn[0])
    # the SIMT split kernel on the same problem agrees (both within bf16 noise of the fp32 reference)
    out2 = torch.zeros_like(out)
    ws = torch.zeros(Hkv * 16 * (Hq // Hkv) * (D + 2), dtype=torch.float32, device=cuda)
    counters = torch.zeros(Hkv, dtype=torch.int32, device=cuda)
    ops.decode_attention(qkv0.clone(), pos, k_pool, v_pool, perm, out2, ws, counters, inv, Hq, Hkv, D, 16, D ** -0.5)
    report_rel(f"decode_attention (SIMT) ctx={ctx}", out2.view(Hq, D), ref, 1.5e-2)
