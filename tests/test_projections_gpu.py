"""GPU: every bf16 projection the model issues, at its production shape, in its call form and in every
GEMM dispatch regime it can reach, against an fp64 reference; and the bf16 decode GEMV at NVILA-Lite-3B's
shapes (tests.helpers.GemvErrors; the other decode GEMVs run in tests/test_gemv_gpu.py).

Table.  One row per distinct (N, K, epilogue, aliasing), generated from nvila_8b(), nvila_8b_dynamic_s2(),
nvila_video_8b() and nvila_lite_3b():
  LLM (qwen2.py prefill_hidden, serving.py BatchedDecoder.step, sp.py):  q/k/v + bias; o_proj and
    down_proj adding the residual stream in place (residual=x, out=x); gate/up with interleaved SwiGLU
    (the _gu_w layout); lm_head plain.
  SigLIP (vision.py):  q/k/v + bias; out_proj and fc2 + bias + residual in place; fc1 + bias + GELU-tanh;
    patch embed, K padded to 592, + bias + position embedding (residual row m % 1024).
  Projectors (projector.py, built on the meta device):  every lin_gelu (+ bias + GELU-erf) and lin
    (+ bias) of mlp_downsample, mlp_downsample_2x2_fix (8B, video, dynamic S2: K = 4 * 3456) and
    mlp_downsample_3x3_fix (Lite).

M values.  tests.helpers.dispatch_flavour mirrors gemm_bf16's choice of kernel; for every M in
[1, M_max] it gives the regime, and each row runs the first and last M of every regime run, one interior
M that is not a multiple of 128, M = 1, 7, 8, 9, and (when M_max allows) one M with more than 8 m-blocks
and a partial last band of the tile rasteriser.  M_max is the largest M the model issues: 16,470 for the
LLM (a 64-frame video prompt), 1,024 for lm_head (engine slots; full-prompt logits of one image),
64 x 1,024 for SigLIP and 64 frames' tokens for the projectors.

Each case writes x with the norm kernel the model runs just before (RMSNorm for the LLM, LayerNorm for
the ViT and projectors), calls ops.linear as the call site does (static_w=True, same aliasing), and checks:
  * default dispatch == ops.linear(block_n=dispatch_flavour(...)), bit for bit (pins the mirror);
  * a second call gives the same bits;
  * the stream-K tile counters (first 64 KiB of the workspace) are zero afterwards;
  * tests.helpers.Bf16Errors against the fp64 reference (tests.helpers.linear_reference), computed in
    row blocks: per element, per row and rounding bias.
Every case is recorded (tests.helpers._record) with its regime and error in ulps.
"""
import math

import pytest
import torch

from oracle import vila_oracle as O
from tests.helpers import REGIME, Bf16Errors, _record, check_gemv, dispatch_flavour, gemv_plan, linear_reference
from tests.test_fp8_decode_gpu import GEMV_CASES
from tests.test_kernels_gpu import _ops, bf

pytestmark = pytest.mark.gpu

LLM_M_MAX = 16470      # 64-frame video prompt
LM_HEAD_M_MAX = 1024   # engine slots / full-prompt logits of one image
FRAMES = 64
COUNTER_BYTES = 64 * 1024


@pytest.fixture(autouse=True)
def _fp32_truth():
    """the fp32 parts of the reference (the GEMV's RMSNorm) must really be fp32 on the device"""
    saved = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32,
             torch.get_float32_matmul_precision())
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved[:2]
    torch.set_float32_matmul_precision(saved[2])


# ------------------------------------------------------------------------------------------------
# the production table
# ------------------------------------------------------------------------------------------------
def _table():
    from vila_b200.model.configuration import nvila_8b, nvila_8b_dynamic_s2, nvila_lite_3b, nvila_video_8b
    from vila_b200.model.projector import MultimodalProjector

    rows = {}

    def add(name, N, K, epi, m_max, norm):
        key = (N, K, epi)
        if key in rows:
            if name not in rows[key]["name"].split("="):
                rows[key]["name"] += "=" + name
            rows[key]["m_max"] = max(rows[key]["m_max"], m_max)
        else:
            rows[key] = dict(name=name, N=N, K=K, epi=epi, m_max=m_max, norm=norm)

    for tag, cfg in (("8b", nvila_8b()), ("8b-s2", nvila_8b_dynamic_s2()), ("video", nvila_video_8b()),
                     ("lite", nvila_lite_3b())):
        llm = cfg.llm_cfg
        H, I, D = llm.hidden_size, llm.intermediate_size, llm.head_dim
        Hq, Hkv = llm.num_attention_heads, llm.num_key_value_heads
        lt = f"llm{H}"
        add(f"{lt}.qkv", (Hq + 2 * Hkv) * D, H, "bias", LLM_M_MAX, "rms")
        add(f"{lt}.o_proj", H, Hq * D, "residual", LLM_M_MAX, "rms")
        add(f"{lt}.gate_up", 2 * I, H, "swiglu", LLM_M_MAX, "rms")
        add(f"{lt}.down_proj", H, I, "residual", LLM_M_MAX, "rms")
        add(f"{lt}.lm_head", llm.vocab_size, H, "plain", LM_HEAD_M_MAX, "rms")
        v = cfg.vision_tower_cfg
        C, VI, P = v.hidden_size, v.intermediate_size, v.num_patches
        vit_max = FRAMES * P
        add("siglip.qkv", 3 * C, C, "bias", vit_max, "ln")
        add("siglip.out_proj", C, C, "bias+residual", vit_max, "ln")
        add("siglip.fc1", VI, C, "bias+gelu_tanh", vit_max, "ln")
        add("siglip.fc2", C, VI, "bias+residual", vit_max, "ln")
        add("siglip.patch", C, -(-v.num_channels * v.patch_size ** 2 // 8) * 8, "bias+posemb", vit_max, "ln")
        proj = MultimodalProjector(cfg, device="meta")
        r = proj.downsample_rate
        m_max = FRAMES * (-(-v.grid // r)) ** 2  # space_to_depth pads the grid to a multiple of r
        lins = [(op, mod) for op, mod in proj._program if op != "ln"]
        for i, (op, mod) in enumerate(lins):
            N, K = mod.weight.shape
            add(f"proj-{tag}.{op}{i}", N, K, "bias+gelu_erf" if op == "lin_gelu" else "bias", m_max, "ln")
    return list(rows.values())


TABLE = _table()


def _case_ms(N, K, m_max, sms, ws_bytes):
    """{M: regime code}: both ends of every regime run, one interior M (not a multiple of 128) per run,
    M = 1, 7, 8, 9 and one M with a partial last band of 8 m-blocks; plus the runs themselves"""
    runs = []
    for M in range(1, m_max + 1):
        f = dispatch_flavour(M, N, K, sms, ws_bytes)
        if runs and runs[-1][2] == f:
            runs[-1][1] = M
        else:
            runs.append([M, M, f])
    ms = {M for M in (1, 7, 8, 9) if M <= m_max}
    for lo, hi, _ in runs:
        ms |= {lo, hi}
        mid = (lo + hi) // 2
        if mid % 128 == 0:
            mid -= 1
        if lo < mid < hi:
            ms.add(mid)
    if m_max > 8 * 128:
        mb = -(-m_max // 128)
        ms.add(m_max if mb % 8 else 9 * 128 - 52)  # 9 m-blocks: a band of one
    return {M: dispatch_flavour(M, N, K, sms, ws_bytes) for M in sorted(ms)}, runs


def _inputs(row, dev):
    N, K, m_max = row["N"], row["K"], row["m_max"]
    g = torch.Generator(device=dev).manual_seed(N * 31 + K)
    x_raw = torch.randn(m_max, K, device=dev, generator=g)
    for i, ch in enumerate((7, K // 3, K // 2 + 1, K - 9)):  # outlier channels
        x_raw[:, ch] = 50.0 if i % 2 == 0 else -50.0
    x_raw = bf(x_raw)
    nw = bf(1 + 0.1 * torch.randn(K, device=dev, generator=g))
    nb = bf(0.1 * torch.randn(K, device=dev, generator=g))
    w = bf(torch.randn(N, K, device=dev, generator=g) / math.sqrt(K))
    if row["epi"] == "bias+posemb":
        w[:, 3 * 14 * 14:] = 0  # the padded K columns of the patch-embedding weight
    b = bf(torch.randn(N, device=dev, generator=g)) if "bias" in row["epi"] else None
    res = None
    if row["epi"].endswith("residual"):
        res = bf(torch.randn(m_max, N, device=dev, generator=g))
    elif row["epi"] == "bias+posemb":
        res = bf(torch.randn(1024, N, device=dev, generator=g))
    return x_raw, nw, nb, w, b, res


def _call(ops, row, x_raw, nw, nb, w, b, res, M, block_n=None):
    """the model's call form: x written by the norm kernel just before, then ops.linear"""
    epi = row["epi"]
    buf = res[:M].clone() if epi.endswith("residual") else None  # the residual stream, updated in place
    xr = x_raw[:M]
    x = ops.rmsnorm(xr, nw, 1e-6) if row["norm"] == "rms" else ops.layernorm(xr, nw, nb, 1e-6)
    act = {"bias+gelu_tanh": ops.ACT_GELU_TANH, "bias+gelu_erf": ops.ACT_GELU_ERF}.get(epi, ops.ACT_NONE)
    if buf is not None:
        out = ops.linear(x, w, b, residual=buf, out=buf, block_n=block_n, static_w=True)
    elif epi == "bias+posemb":
        out = ops.linear(x, w, b, residual=res, res_row_mod=1024, block_n=block_n, static_w=True)
    else:
        out = ops.linear(x, w, b, act=act, swiglu=epi == "swiglu", block_n=block_n, static_w=True)
    return x, out


def _reference_errors(row, x, w, wd, b, res, got):
    epi, N = row["epi"], row["N"]
    M = x.shape[0]
    e = Bf16Errors()
    step = max(1, (1 << 25) // N)
    for r0 in range(0, M, step):
        r1 = min(M, r0 + step)
        P = x[r0:r1].double() @ wd.t()
        if epi.endswith("residual"):
            resid = res[r0:r1]
        elif epi == "bias+posemb":
            resid = res[torch.arange(r0, r1, device=x.device) % 1024]
        else:
            resid = None
        act = epi.split("+")[1] if "gelu" in epi else None
        ref_final = linear_reference(P, bias=b, act=act, residual=resid, swiglu=epi == "swiglu")
        e.add(got[r0:r1], ref_final, r0)
        del P, ref_final
    return e


@pytest.mark.parametrize("row", TABLE, ids=[r["name"] for r in TABLE])
def test_projection(cuda, row):
    ops = _ops()
    ws = ops.ensure_workspace(cuda)
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    N, K = row["N"], row["K"]
    cases, runs = _case_ms(N, K, row["m_max"], sms, ws.numel())
    x_raw, nw, nb, w, b, res = _inputs(row, cuda)
    wd = w.double()
    failures = []
    for M, flav in cases.items():
        x, got = _call(ops, row, x_raw, nw, nb, w, b, res, M)
        _, again = _call(ops, row, x_raw, nw, nb, w, b, res, M)
        _, forced = _call(ops, row, x_raw, nw, nb, w, b, res, M, block_n=flav)
        torch.cuda.synchronize()
        what = f"{row['name']} M={M} ({REGIME[flav]})"
        assert torch.equal(got, forced), f"{what}: default dispatch differs from vila_linear_cfg {flav}: " \
                                         "the mirror tests.helpers.dispatch_flavour is out of step with gemm_bf16"
        assert torch.equal(got, again), f"{what}: not repeatable"
        assert int(ws[:COUNTER_BYTES].view(torch.int32).abs().max()) == 0, f"{what}: stream-K counters left set"
        del again, forced
        e = _reference_errors(row, x, w, wd, b, res, got)
        _record({"name": "projection", "layer": row["name"], "N": N, "K": K, "epi": row["epi"], "M": M,
                 "regime": REGIME[flav], **e.summary()})
        failures += [f"{what}: {f}" for f in e.failures()]
        del x, got
    reachable = {REGIME[f] for _, _, f in runs}
    tested = {REGIME[f] for f in cases.values()}
    _record({"name": "projection coverage", "layer": row["name"], "M_max": row["m_max"],
             "regimes": [f"{REGIME[f]} {lo}-{hi}" for lo, hi, f in runs], "cases": len(cases)})
    assert tested == reachable, (row["name"], reachable - tested)
    del x_raw, w, wd, res
    torch.cuda.empty_cache()
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------
# bf16 decode GEMV at NVILA-Lite-3B's shapes
# ------------------------------------------------------------------------------------------------
LITE_GEMV = [c for c in GEMV_CASES if c[0].startswith("lite-")]


@pytest.mark.parametrize("variant", [0, 1])  # 0: TMA-ring kernel, 1: register-staged kernel
@pytest.mark.parametrize("name,N,K,fusion", LITE_GEMV, ids=[c[0] for c in LITE_GEMV])
def test_gemv_bf16_lite(cuda, name, N, K, fusion, variant):
    ops = _ops()
    g = torch.Generator(device=cuda).manual_seed(N + K + variant)
    x = torch.randn(K, device=cuda, generator=g)
    x[[7, K // 2]] = 50.0
    x = bf(x)
    w = bf(torch.randn(N, K, device=cuda, generator=g) / math.sqrt(K))  # lite-lm_head: the tied embedding
    b = bf(torch.randn(N, device=cuda, generator=g))
    r = bf(torch.randn(N, device=cuda, generator=g))
    nw = bf(1 + 0.1 * torch.randn(K, device=cuda, generator=g))
    key = torch.zeros(1, dtype=torch.int64, device=cuda) if fusion == "argmax+norm" else None

    def launch(k=None):
        if fusion == "bias+norm":
            return ops.gemv(x, w, bias=b, norm_w=nw, norm_eps=1e-6, static_w=True, variant=variant)
        if fusion == "residual":
            return ops.gemv(x, w, residual=r, static_w=True, variant=variant)
        if fusion == "swiglu+norm":
            return ops.gemv(x, w, norm_w=nw, norm_eps=1e-6, swiglu=True, static_w=True, variant=variant)
        return ops.gemv(x, w, norm_w=nw, norm_eps=1e-6, argmax_key=k, static_w=True, variant=variant)

    out = launch(key)
    again = launch(torch.zeros_like(key) if key is not None else None)
    torch.cuda.synchronize()
    assert torch.equal(out, again)
    xn = O.rms_norm(x[None], nw, 1e-6)[0] if "norm" in fusion else x
    P = (w.double() @ xn.double())[None]
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    _, depth, regime = gemv_plan("bf16", N, K, fusion, sms, variant=variant)
    e = check_gemv("gemv bf16", out[None], x[None], w, N, depth=depth, norm_w=nw if "norm" in fusion else None,
                   bias=b if fusion == "bias+norm" else None, residual=r[None] if fusion == "residual" else None,
                   swiglu=fusion == "swiglu+norm",
                   record=dict(layer=name, N=N, K=K, epi=fusion, variant=variant, regime=regime))
    e.check(f"gemv {name} variant {variant}")
    if key is not None:  # the fused arg-max: the kernel's own logits decide, and it is a best id of fp64
        tok = 0xFFFFFFFF - int(key.item() & 0xFFFFFFFF)
        assert tok == int(torch.argmax(out.float()))
        margin = 3 * 2 ** -8 * P.abs().max().item()
        assert P[0, tok].item() >= P.max().item() - margin
