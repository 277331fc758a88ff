"""GPU: every decode GEMV call site (bf16, FP8 and W4A16; single-stream and batched) at its production shape,
fusion and partition, against an fp64 reference with a per-element bound (tests.helpers.GemvErrors).

Table, from nvila_8b(), nvila_lite_3b() and tiny_test_config() (one row per (format, N, K, fusion) a decoder
issues):
  * single-stream bf16 (qwen2.GraphDecoder): NVILA-8B's qkv (bias + RMSNorm), o_proj (residual, in place),
    gate_up (SwiGLU + RMSNorm), down_proj (residual, in place) and lm_head (arg-max + RMSNorm), on the TMA-ring
    kernel (variant 0) and the register-staged one (variant 1).  Lite's shapes run in
    tests/test_projections_gpu.py::test_gemv_bf16_lite;
  * single-stream e4m3 / W4A16: every layer shape of the three models, the e4m3 lm_heads (W4A16 mode uses them
    too), N = 1003, outlier activations, and shapes the mirror (tests.helpers.gemv_tma_plan / gemv_w4_plan)
    picks to reach further k-split regimes, each with a short last row block;
  * batched e4m3 / W4A16 (serving.BatchedDecoder): every layer shape and the e4m3 lm_heads, M = 17 (two launches)
    and M in {1, 2, 7, 8, 9, 15, 16}: both column tiles (kNT = 1, 2), the residual added in place.

Inputs: weight rows spread in magnitude, W4 groups spread in magnitude plus an all-zero, an all-positive and an
all-negative group; batched x rows 2^-8, 1 and 2^8 in turn, some with activations at +-1e4.  The reference's
weights come from the re-derived quantizers (tests.helpers.ref_quantize_*), which must match the package's bit
for bit.  Each case checks GemvErrors, that only the output slice of a sentinel-filled buffer was written, that a
repeat call gives the same bits and (batched) that every row equals its M = 1 run and the device partition the
mirror tests.helpers.batch_partition.  The arg-max tests plant ties of the maximum logit in different CTAs.
"""
import math

import pytest
import torch

from tests.helpers import (_record, batch_partition, check_gemv, e4m3_rows, gemv_depth, gemv_plan, gemv_xn,
                           ref_quantize_e4m3_rows, ref_quantize_w4, ref_w4_pack, w4_rows)

pytestmark = pytest.mark.gpu

SMS_H100 = 132  # H100 SXM; the GPU cases take the device's own count
SENT = -3.0e38  # finite bf16 sentinel
CHUNK_ROWS = 8192  # weight rows generated at a time: a case holds ~2 bf16 copies of its weight, not fp32 ones


def _llms():
    from vila_b200.model.configuration import nvila_8b, nvila_lite_3b, tiny_test_config
    return (("8b", nvila_8b().llm_cfg), ("lite", nvila_lite_3b().llm_cfg), ("tiny", tiny_test_config().llm_cfg))


def _layers(llm):
    H, I, D = llm.hidden_size, llm.intermediate_size, llm.head_dim
    Hq, Hkv = llm.num_attention_heads, llm.num_key_value_heads
    return [("qkv", (Hq + 2 * Hkv) * D, H, "bias+norm"), ("o", H, Hq * D, "residual"),
            ("gate_up", 2 * I, H, "swiglu+norm"), ("down", H, I, "residual")]


def _single_table():
    rows = []
    llms = _llms()
    llm8 = llms[0][1]
    for name, N, K, fusion in _layers(llm8) + [("lm_head", llm8.vocab_size, llm8.hidden_size, "argmax+norm")]:
        for variant in (0, 1):
            rows.append(dict(fmt="bf16", name=f"8b-{name}", N=N, K=K, fusion=fusion, variant=variant))
    for fmt in ("fp8", "w4a16"):
        for tag, llm in llms:
            rows += [dict(fmt=fmt, name=f"{tag}-{n}", N=N, K=K, fusion=f) for n, N, K, f in _layers(llm)]
        if fmt == "fp8":
            rows += [dict(fmt=fmt, name=f"{tag}-lm_head", N=llm.vocab_size, K=llm.hidden_size, fusion="argmax+norm")
                     for tag, llm in llms]
        rows.append(dict(fmt=fmt, name="n1003", N=1003, K=3584, fusion="argmax+norm"))
        rows.append(dict(fmt=fmt, name="8b-down-outliers", N=3584, K=18944, fusion="residual", outliers=True))
        rows.append(dict(fmt=fmt, name="8b-qkv-outliers", N=4608, K=3584, fusion="bias+norm", outliers=True))
        # further k-split regimes, each with a short last row block
        seen = {gemv_plan(fmt, r["N"], r["K"], r["fusion"], SMS_H100)[0]["ksplit"] for r in rows if r["fmt"] == fmt}
        for K in (512, 2048, 3584, 11008, 18944):
            for N in (201, 1003, 2001):
                ks = gemv_plan(fmt, N, K, "residual", SMS_H100)[0]["ksplit"]
                if ks not in seen:
                    seen.add(ks)
                    rows.append(dict(fmt=fmt, name=f"ks{ks}-N{N}-K{K}", N=N, K=K, fusion="residual"))
    return rows


def _batch_table():
    rows = []
    llms = _llms()
    for fmt in ("w4a16", "fp8"):
        for tag, llm in llms:
            rows += [dict(fmt=fmt, name=f"{tag}-{n}", N=N, K=K, fusion=f.split("+")[0]) for n, N, K, f in _layers(llm)]
    rows += [dict(fmt="fp8", name=f"{tag}-lm_head", N=llm.vocab_size, K=llm.hidden_size, fusion="none")
             for tag, llm in llms[:2]]
    return rows


SINGLE_TABLE = _single_table()
BATCH_TABLE = _batch_table()
BATCH_M = (1, 2, 7, 8, 9, 15, 16)


def edge_groups(w):
    """in place on w [N >= 3, K >= 384]: row 0's first group all zero, row 1's second group all positive, row 2's
    third group all negative"""
    w[0, :128] = 0
    w[1, 128:256] = w[1, 128:256].abs()
    w[2, 256:384] = -w[2, 256:384].abs()
    return w


def _ops():
    from vila_b200 import ops
    ops.ensure_workspace("cuda")
    return ops


def _weights(fmt, N, K, seed):
    """-> (kernel weight kwargs, fp64 weight rows for gemv_reference); the quantizers checked bit for bit against
    their re-derivation"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = torch.empty(N, K, dtype=torch.bfloat16, device="cuda")
    for r0 in range(0, N, CHUNK_ROWS):  # an lm_head's fp32 temporaries in pieces
        n = min(N, r0 + CHUNK_ROWS) - r0
        w[r0:r0 + n] = (torch.randn(n, K, device="cuda", generator=g) / math.sqrt(K)
                        * torch.exp(torch.randn(n, 1, device="cuda", generator=g))
                        * torch.exp(0.5 * torch.randn(n, K // 128, device="cuda", generator=g)).repeat_interleave(128, 1))
    w = edge_groups(w)  # zero, abs and negation are exact in bf16
    if fmt == "bf16":
        return dict(w=w), w
    if fmt == "fp8":
        from vila_b200.model.qwen2 import quantize_e4m3_rows
        q, s = quantize_e4m3_rows(w)
        rq, rs = ref_quantize_e4m3_rows(w)
        assert torch.equal(q.view(torch.uint8), rq) and torch.equal(s, rs), "quantize_e4m3_rows != its rule"
        return dict(w=q, w_scale=s), e4m3_rows(rq, rs)
    from vila_b200.model.qwen2 import quantize_w4_groups
    packed, s, z = quantize_w4_groups(w)
    rq, rs, rz = ref_quantize_w4(w)
    assert torch.equal(s.float(), rs) and torch.equal(z, rz), "quantize_w4_groups' scales / zeros != its rule"
    assert torch.equal(packed, ref_w4_pack(rq)), "quantize_w4_groups' packed bytes != gemv_tma.cu's layout"
    return dict(w=packed, w_scale=s, w_zero=z), w4_rows(rq, rs, rz)


def _x(M, K, seed, outliers=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(M, K, device="cuda", generator=g)
    if M > 1:
        x *= torch.tensor([2.0 ** (8 * (m % 3 - 1)) for m in range(M)], device="cuda")[:, None]
    for m in range(M):
        if outliers or (M > 1 and m % 5 == 3):
            x[m, torch.randperm(K, device="cuda", generator=g)[:6]] = torch.tensor([1e4, -1e4] * 3, device="cuda")
    return x.to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------
# single stream
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("row", SINGLE_TABLE,
                         ids=[f"{r['fmt']}-{r['name']}" + (f"-v{r['variant']}" if "variant" in r else "")
                              for r in SINGLE_TABLE])
def test_gemv_single(cuda, row):
    ops = _ops()
    fmt, N, K, fusion = row["fmt"], row["N"], row["K"], row["fusion"]
    variant = row.get("variant", 0)
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    plan, depth, regime = gemv_plan(fmt, N, K, fusion, sms, variant=variant)
    wkw, wrows = _weights(fmt, N, K, seed=N + K)
    g = torch.Generator(device="cuda").manual_seed(N)
    x = _x(1, K, seed=K, outliers=row.get("outliers", False))[0]
    b = torch.randn(N, device=cuda, generator=g).to(torch.bfloat16)
    r = torch.randn(N, device=cuda, generator=g).to(torch.bfloat16)
    nw = (1 + 0.1 * torch.randn(K, device=cuda, generator=g)).to(torch.bfloat16)
    swiglu, norm = fusion.startswith("swiglu"), "norm" in fusion
    n_out = N // 2 if swiglu else N
    argmax = fusion.startswith("argmax")

    def launch(key=None, write_out=True):
        buf = torch.full((n_out + 64,), SENT, dtype=torch.bfloat16, device=cuda)
        out = buf[:n_out]
        kw = dict(static_w=True, variant=variant, **wkw)
        if norm:
            kw.update(norm_w=nw, norm_eps=1e-6)
        if fusion.startswith("bias"):
            kw["bias"] = b
        if fusion.startswith("residual"):  # GraphDecoder adds into the hidden state in place
            out.copy_(r)
            kw["residual"] = out
        ops.gemv(x, out=out if write_out else None, swiglu=swiglu, argmax_key=key, write_out=write_out, **kw)
        return buf

    key = torch.zeros(1, dtype=torch.int64, device=cuda) if argmax else None
    buf = launch(key)
    again = launch(torch.zeros_like(key) if argmax else None)
    torch.cuda.synchronize()
    got = buf[:n_out]
    assert bool((buf[n_out:] == SENT).all()), "wrote past the output"
    assert torch.equal(buf, again), "not repeatable"
    what = f"{fmt} {row['name']} {fusion} v{variant}"
    e = check_gemv("gemv single", got[None], x[None], wrows, N, depth=depth, norm_w=nw if norm else None,
                   bias=b if fusion.startswith("bias") else None,
                   residual=r[None] if fusion.startswith("residual") else None, swiglu=swiglu,
                   record=dict(fmt=fmt, layer=row["name"], N=N, K=K, fusion=fusion, variant=variant, regime=regime,
                               depth=depth))
    assert not e.failures(), f"{what} ({regime}): " + "; ".join(e.failures())
    if argmax:  # the key: the kernel's own logits decide, the lowest index among equal ones
        tok = 0xFFFFFFFF - int(key.item() & 0xFFFFFFFF)
        assert tok == int(torch.argmax(got.float())), what
        key2 = torch.zeros_like(key)
        launch(key2, write_out=False)
        assert torch.equal(key, key2), f"{what}: the key differs without the logits written"


# ------------------------------------------------------------------------------------------------
# batched
# ------------------------------------------------------------------------------------------------
def _batch_call(ops, x, wkw, fusion, b, r, N, n_out):
    """one gemv_batch call in BatchedDecoder's form (residual added in place) into a sentinel-filled buffer:
    -> the buffer [M + 1, padded]; the output is buf[:M, :n_out]"""
    M = x.shape[0]
    buf = torch.full((M + 1, (max(N, n_out) + 7) // 8 * 8 + 8), SENT, dtype=torch.bfloat16, device=x.device)
    out = buf[:M, :n_out]
    kw = dict(static_w=True, out=out, **wkw)
    if fusion == "bias":
        kw["bias"] = b
    elif fusion == "residual":
        out.copy_(r[:M])
        kw["residual"] = out
    elif fusion == "swiglu":
        kw["swiglu"] = True
    ops.gemv_batch(x, **kw)
    return buf


@pytest.mark.parametrize("row", BATCH_TABLE, ids=[f"{r['fmt']}-{r['name']}" for r in BATCH_TABLE])
def test_gemv_batch(cuda, row):
    ops = _ops()
    fmt, N, K, fusion = row["fmt"], row["N"], row["K"], row["fusion"]
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    dev = ops.gemv_batch_partition(N, K, fmt == "fp8")
    active = {dev["cluster"]: dev["max_active_clusters"]}
    mirror = batch_partition(N, K, fmt == "fp8", sms, lambda cl: active.get(cl, sms // cl))
    got_p = {k: dev[k] for k in ("cluster", "ctas", "tiles_per_cluster", "parts")}
    assert got_p == {k: mirror[k] for k in got_p}, f"device partition {dev} != the mirror's {mirror}"
    depth = gemv_depth("batch-fp8" if fmt == "fp8" else "batch-w4", K, mirror)
    wkw, wrows = _weights(fmt, N, K, seed=N + K + 1)
    g = torch.Generator(device="cuda").manual_seed(N + 1)
    Mmax = 17
    x = _x(Mmax, K, seed=K + 1)
    b = torch.randn(N, device=cuda, generator=g).to(torch.bfloat16)
    r = (torch.randn(Mmax, N, device=cuda, generator=g)
         * torch.tensor([2.0 ** (8 * (m % 3 - 1)) for m in range(Mmax)], device=cuda)[:, None]).to(torch.bfloat16)
    n_out = N // 2 if fusion == "swiglu" else N
    buf = _batch_call(ops, x, wkw, fusion, b, r, N, n_out)
    torch.cuda.synchronize()
    full = buf[:Mmax, :n_out]
    assert bool((buf[:Mmax, n_out:] == SENT).all()) and bool((buf[Mmax] == SENT).all()), "wrote past N or M"
    assert torch.equal(_batch_call(ops, x, wkw, fusion, b, r, N, n_out), buf), "not repeatable"
    what = f"batched {fmt} {row['name']} {fusion}"
    regime = f"cluster {mirror['cluster']} x {mirror['tiles_per_cluster']} tiles, {mirror['parts']} parts"
    e = check_gemv("gemv batch", full, x, wrows, N, depth=depth, bias=b if fusion == "bias" else None,
                   residual=r if fusion == "residual" else None, swiglu=fusion == "swiglu",
                   record=dict(fmt=fmt, layer=row["name"], N=N, K=K, fusion=fusion, M=Mmax, regime=regime,
                               partition=got_p, max_active_clusters=dev["max_active_clusters"], depth=depth))
    assert not e.failures(), f"{what} ({regime}): " + "; ".join(e.failures())
    for M in BATCH_M:  # both column tiles and every M give each row the bits of the M = 17 run
        b2 = _batch_call(ops, x[:M], wkw, fusion, b, r, N, n_out)
        assert torch.equal(b2[:M, :n_out], full[:M]), f"{what}: M={M} differs from M=17"
        assert bool((b2[:M, n_out:] == SENT).all()) and bool((b2[M] == SENT).all()), f"{what}: M={M} wrote past N or M"
    for m in range(Mmax):
        one = _batch_call(ops, x[m:m + 1], wkw, fusion, b, r[m:m + 1], N, n_out)
        assert torch.equal(one[0, :n_out], full[m]), f"{what}: row {m} alone differs"


def test_gemv_batch_partitions(cuda):
    """the partition the device returns for every batched shape of the table (recorded), against the mirror"""
    from vila_b200 import ops
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    seen = set()
    for row in BATCH_TABLE:
        key = (row["N"], row["K"], row["fmt"])
        if key in seen:
            continue
        seen.add(key)
        dev = ops.gemv_batch_partition(row["N"], row["K"], row["fmt"] == "fp8")
        mirror = batch_partition(row["N"], row["K"], row["fmt"] == "fp8", sms,
                                 lambda cl: dev["max_active_clusters"] if cl == dev["cluster"] else sms // cl)
        _record({"name": "gemv batch partition", "fmt": row["fmt"], "layer": row["name"], "N": row["N"],
                 "K": row["K"], **dev, "mirror_default_active": {k: batch_partition(
                     row["N"], row["K"], row["fmt"] == "fp8", sms)[k] for k in ("cluster", "tiles_per_cluster")}})
        assert {k: dev[k] for k in ("cluster", "ctas", "tiles_per_cluster", "parts")} == \
            {k: mirror[k] for k in ("cluster", "ctas", "tiles_per_cluster", "parts")}, (row, dev, mirror)


# ------------------------------------------------------------------------------------------------
# arg-max ties
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sign", ["positive", "negative"])
@pytest.mark.parametrize("fmt", ["bf16", "fp8"])
def test_argmax_ties_lowest_index(cuda, fmt, sign):
    """three identical lm_head rows in different CTAs carry the largest logit (in a row of all-negative logits for
    sign="negative"): the fused key resolves to the lowest of them, and argmax_finalize writes that token"""
    ops = _ops()
    V, K = 152064, 3584
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(K, device=cuda, generator=g).to(torch.bfloat16)
    nw = (1 + 0.1 * torch.randn(K, device=cuda, generator=g)).to(torch.bfloat16)
    xn = gemv_xn(x[None], nw)[0].float()
    w = torch.empty(V, K, dtype=torch.bfloat16, device=cuda)
    for r0 in range(0, V, CHUNK_ROWS):
        n = min(V, r0 + CHUNK_ROWS) - r0
        wc = torch.randn(n, K, device=cuda, generator=g) / math.sqrt(K)
        if sign == "negative":  # every logit -sum |w x|
            wc = -wc.abs() * torch.sign(xn)
        w[r0:r0 + n] = wc.to(torch.bfloat16)
        del wc
    tie = [5000, 70001, 150000]  # blocks of 1,152 rows on 132 SMs: three different CTAs
    if sign == "negative":  # the tied rows are the smallest in magnitude
        w[tie] = (w[tie[0]] * 0.25).to(torch.bfloat16)
    else:
        w[tie] = (w[tie[0]].abs() * torch.sign(xn) * 2.0).to(torch.bfloat16)
    wkw = dict(w=w)
    if fmt == "fp8":
        from vila_b200.model.qwen2 import quantize_e4m3_rows
        q, s = quantize_e4m3_rows(w)
        wkw = dict(w=q, w_scale=s)
    key = torch.zeros(1, dtype=torch.int64, device=cuda)
    logits = ops.gemv(x, norm_w=nw, norm_eps=1e-6, argmax_key=key, static_w=True, **wkw)
    torch.cuda.synchronize()
    lf = logits.float()
    assert bool((lf[tie] == lf.max()).all()), "the planted rows do not tie at the maximum"
    if sign == "negative":
        assert bool((lf < 0).all())
    tok = 0xFFFFFFFF - int(key.item() & 0xFFFFFFFF)
    assert tok == tie[0] == int(torch.argmax(lf)), (tok, tie)
    out = torch.zeros(1, dtype=torch.int32, device=cuda)
    hist = torch.zeros(4, dtype=torch.int32, device=cuda)
    step = torch.zeros(1, dtype=torch.int32, device=cuda)
    pos = torch.full((1,), 9, dtype=torch.int32, device=cuda)
    table = torch.randn(V, 64, device=cuda, generator=g).to(torch.bfloat16)
    nxt = torch.zeros(64, dtype=torch.bfloat16, device=cuda)
    ops.argmax_finalize(key, out, hist, step, pos, table, nxt)
    torch.cuda.synchronize()
    assert int(out) == tie[0] and int(hist[0]) == tie[0] and int(step) == 1 and int(pos) == 10
    assert int(key) == 0 and torch.equal(nxt, table[tie[0]])
