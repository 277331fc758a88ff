"""GPU: the continuous-batching engine on the opt-in FP8 and W4A16 decode weights.

  * vila_gemv_batch_fp8 / vila_gemv_batch_w4a16 against fp32 math on the dequantized copies, at every layer
    shape of NVILA-8B, NVILA-Lite-3B and the tiny test model in both formats, the e4m3 lm_heads and an
    N = 1003 case, for M in {1, 5, 8, 16, 20} with their fusions;
  * row independence: every output row is bit-identical to the same row run alone (M = 1) and to a run in
    which the other rows hold random data or +-1e4 outliers; repeatable, graph replay included;
  * every rejection, through ops and through the raw C entry points, leaves y untouched;
  * serving.BatchedDecoder in "fp8" and "w4a16" mode, teacher-forced on the scenario of
    test_decode_engines_gpu._run_batched against the oracle on the dequantized copies;
  * generate_batch gives every request the same ids alone, with 3 slots and with 20 (two launch groups);
  * bf16 BatchedDecoder ids and pool are unchanged by a bf16 -> w4a16 -> fp8 -> bf16 round trip.
"""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from tests import test_fp8_decode_gpu as T8
from tests import test_w4a16_decode_gpu as T4
from tests.helpers import report_rel
from tests.test_decode_engines_gpu import _fp32_truth  # noqa: F401  (autouse: the fp32 oracle is really fp32)
from tests.test_decode_engines_gpu import _check_untouched, _decoded_rows, _prompt
from tests.test_fp8_decode_gpu import _check_fp8_sequence, rb
from tests.test_kernels_gpu import _ops, bf

pytestmark = pytest.mark.gpu

# ------------------------------------------------------------------------------------------------
# kernel level
# ------------------------------------------------------------------------------------------------
#   8B:   hidden 3584, inter 18944, qkv (28 + 2*4) * 128, vocab 152,064
#   Lite: hidden 2048, inter 11008, qkv (16 + 2*2) * 128, vocab 151,936
#   tiny: hidden 512, inter 1024, qkv (4 + 2*2) * 128
_LAYERS = [
    ("8b-qkv", 4608, 3584, "bias"), ("8b-o", 3584, 3584, "residual"),
    ("8b-gate_up", 37888, 3584, "swiglu"), ("8b-down", 3584, 18944, "residual"),
    ("lite-qkv", 2560, 2048, "bias"), ("lite-o", 2048, 2048, "residual"),
    ("lite-gate_up", 22016, 2048, "swiglu"), ("lite-down", 2048, 11008, "residual"),
    ("tiny-qkv", 1024, 512, "bias"), ("tiny-o", 512, 512, "residual"),
    ("tiny-gate_up", 2048, 512, "swiglu"), ("tiny-down", 512, 1024, "residual"),
]
KERNEL_CASES = ([("w4a16",) + c for c in _LAYERS] + [("fp8",) + c for c in _LAYERS]
                + [("fp8", "8b-lm_head", 152064, 3584, "none"), ("fp8", "lite-lm_head", 151936, 2048, "none"),
                   ("w4a16", "n1003", 1003, 3584, "none"), ("fp8", "n1003", 1003, 3584, "none")])
M_VALUES = (1, 5, 8, 16, 20)


def _weights(fmt, N, K, seed):
    """-> (dict of gemv_batch weight arguments, dequantized fp32 [N, K])"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = bf(torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)
           * torch.exp(torch.randn(N, 1, device="cuda", generator=g))
           * torch.exp(0.5 * torch.randn(N, K // 128, device="cuda", generator=g)).repeat_interleave(128, 1))
    if fmt == "w4a16":
        q, s, z, deq = T4._quant(w)
        return dict(w=q, w_scale=s, w_zero=z), deq
    q, s, deq = T8._quant(w)
    return dict(w=q, w_scale=s), deq


def _acts(M, K, seed, outliers=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(M, K, device="cuda", generator=g)
    if outliers:
        x[:, torch.randperm(K, device="cuda", generator=g)[:6]] = torch.tensor([1e4, -1e4] * 3, device="cuda")
    return bf(x)


def _run(ops, fusion, x, wa, b, r, inplace=False):
    if fusion == "bias":
        return ops.gemv_batch(x, bias=b, static_w=True, **wa)
    if fusion == "residual":
        res = r.clone()
        return ops.gemv_batch(x, residual=res, out=res if inplace else None, static_w=True, **wa)
    if fusion == "swiglu":
        return ops.gemv_batch(x, swiglu=True, static_w=True, **wa)
    return ops.gemv_batch(x, static_w=True, **wa)


def _reference(fusion, acc, b, r):
    if fusion == "bias":
        return rb(acc + b.float()), 2 ** -7
    if fusion == "residual":
        return rb(rb(acc) + r.float()), 2 ** -7
    if fusion == "swiglu":
        return rb(rb(F.silu(rb(acc[:, 0::2]))) * rb(acc[:, 1::2])), 2 ** -6
    return acc, 2 ** -7


@pytest.mark.parametrize("fmt,name,N,K,fusion", KERNEL_CASES, ids=[f"{c[0]}-{c[1]}-{c[4]}" for c in KERNEL_CASES])
def test_gemv_batch(cuda, fmt, name, N, K, fusion):
    ops = _ops()
    wa, deq = _weights(fmt, N, K, seed=N + K)
    g = torch.Generator(device="cuda").manual_seed(N)
    b = bf(torch.randn(N, device="cuda", generator=g))
    Mmax = max(M_VALUES)
    x = _acts(Mmax, K, seed=K)
    r = bf(torch.randn(Mmax, N, device="cuda", generator=g))
    full = _run(ops, fusion, x, wa, b, r)  # M = 20: two launches
    acc = x.float() @ deq.T
    ref, tol = _reference(fusion, acc, b, r)
    assert bool(torch.isfinite(full.float()).all())
    for m in range(Mmax):  # per output row, against max|ref| of that row
        report_rel(f"gemv_batch {fmt} {name} {fusion} row {m}", full[m], ref[m], tol)
    # outputs past N and x rows past M are never written: out is a slice of a wider sentinel-filled tensor
    n_out = full.shape[1]
    sent = torch.full((Mmax + 1, (n_out + 7) // 8 * 8 + 8), 7.0, dtype=torch.bfloat16, device=cuda)
    fuse = {"bias": dict(bias=b), "residual": dict(residual=r.clone()), "swiglu": dict(swiglu=True), "none": {}}
    ops.gemv_batch(x, out=sent[:Mmax, :n_out], static_w=True, **wa, **fuse[fusion])
    assert torch.equal(sent[:Mmax, :n_out], full)
    assert bool((sent[:Mmax, n_out:] == 7.0).all()) and bool((sent[Mmax] == 7.0).all()), "wrote past N or M"
    # every M gives the same bits per row, and each row equals the same row alone
    for M in M_VALUES[:-1]:
        assert torch.equal(_run(ops, fusion, x[:M], wa, b, r[:M]), full[:M]), f"M={M} differs from M=20"
    for m in range(Mmax):
        assert torch.equal(_run(ops, fusion, x[m:m + 1], wa, b, r[m:m + 1])[0], full[m]), f"row {m} alone differs"
    # the other rows hold random data or outliers: the even rows keep their bits
    for outliers in (False, True):
        x2 = x.clone()
        x2[1::2] = _acts(Mmax // 2, K, seed=K + 1, outliers=outliers)
        y2 = _run(ops, fusion, x2, wa, b, r)
        assert torch.equal(y2[0::2], full[0::2]), f"outliers={outliers}: rows depend on their neighbours"
        if outliers:
            assert bool(torch.isfinite(y2.float()).all())
    if fusion == "residual":  # the engine adds in place
        assert torch.equal(_run(ops, fusion, x, wa, b, r, inplace=True), full)
    # repeatable, and a captured graph replays the same bits
    assert torch.equal(_run(ops, fusion, x[:16], wa, b, r[:16]), full[:16])
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    xs = x[:8].clone()
    with torch.cuda.graph(graph):
        g_out = _run(ops, fusion, xs, wa, b, r[:8])
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g_out, full[:8])


def test_gemv_batch_partition_is_fixed_by_shape():
    """the partition follows from (N, K) and the device: cluster sizes 1..8, one CTA per SM at most"""
    from vila_b200 import ops
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for N, K, fp8 in ((4608, 3584, False), (3584, 18944, False), (37888, 3584, True), (152064, 3584, True),
                      (2048, 11008, True), (1024, 512, False)):
        p = ops.gemv_batch_partition(N, K, fp8)
        assert p["cluster"] in (1, 2, 4, 8) and p["ctas"] % p["cluster"] == 0 and p["ctas"] <= sms, p
        assert p["max_active_clusters"] >= p["ctas"] // p["cluster"], p  # one wave
        assert p == ops.gemv_batch_partition(N, K, fp8)


def test_gemv_batch_rejects(cuda):
    from vila_b200 import _lib
    ops = _ops()
    K, N = 3584, 64
    w4, _ = _weights("w4a16", N, K, seed=1)
    w8, _ = _weights("fp8", N, K, seed=2)
    x = _acts(17, K, seed=3)
    y = torch.full((17, N), 7.0, dtype=torch.bfloat16, device=cuda)
    with pytest.raises(ValueError):
        ops.gemv_batch(x[:4], bf(torch.randn(N, K, device=cuda)), w_scale=w8["w_scale"], out=y[:4])  # bf16
    with pytest.raises(ValueError):
        ops.gemv_batch(x[:4], w4["w"], w_scale=w4["w_scale"], out=y[:4])                  # no zero points
    with pytest.raises(ValueError):
        ops.gemv_batch(x[:4], w8["w"], w_scale=w8["w_scale"][:32], out=y[:4])              # mis-shaped scales
    with pytest.raises(ValueError):
        ops.gemv_batch(x[:4, :K - 128], w8["w"], w_scale=w8["w_scale"], out=y[:4])         # K mismatch
    with pytest.raises(RuntimeError):
        ops.gemv_batch(x[:4], w8["w"], w_scale=w8["w_scale"].double(), out=y[:4])          # fp32 scales
    with pytest.raises(RuntimeError, match="aligned"):
        ops.gemv_batch(x.view(-1)[1:1 + 4 * K].view(4, K), w8["w"], w_scale=w8["w_scale"], out=y[:4])
    with pytest.raises(RuntimeError, match="16-byte multiples"):
        ops.gemv_batch(x.view(-1)[:4 * (K + 4)].view(4, K + 4)[:, :K], w8["w"], w_scale=w8["w_scale"], out=y[:4])

    def raw(fmt, M=4, K_=K, N_=N, flags=0, scales=True, x_off=0):  # past ops.gemv_batch's checks
        p = _lib.GemvBatchParams()
        p.x, p.ldx = x.data_ptr() + 2 * x_off, x.stride(0)
        p.w = (w4 if fmt == "w4a16" else w8)["w"].data_ptr()
        p.bias = p.residual = None
        p.ld_res = 0
        p.y, p.ldy = y.data_ptr(), y.stride(0)
        p.M, p.N, p.K, p.flags = M, N_, K_, flags
        lib, st = _lib.load(), torch.cuda.current_stream().cuda_stream
        if fmt == "w4a16":
            rc = lib.vila_gemv_batch_w4a16(C.byref(p), w4["w_scale"].data_ptr() if scales else None,
                                           w4["w_zero"].data_ptr() if scales else None, st)
        else:
            rc = lib.vila_gemv_batch_fp8(C.byref(p), w8["w_scale"].data_ptr() if scales else None, st)
        return rc, lib.vila_last_error()

    for fmt in ("w4a16", "fp8"):
        for kw, msg in ((dict(M=0), b"outside 1..16"), (dict(M=17), b"outside 1..16"),
                        (dict(K_=K - 8), b"K %"), (dict(scales=False), b"required"),
                        (dict(N_=63, flags=1), b"even N"), (dict(x_off=1), b"aligned"),
                        (dict(flags=4), b"flags")):
            rc, err = raw(fmt, **kw)
            assert rc != 0 and msg in err, (fmt, kw, err)
    rc, err = raw("w4a16", K_=K - 64)  # a multiple of 16, not of 128
    assert rc != 0 and b"K % 128" in err
    torch.cuda.synchronize()
    assert bool((y == 7.0).all())  # nothing was launched


# ------------------------------------------------------------------------------------------------
# engine level
# ------------------------------------------------------------------------------------------------
def _release_all():
    T8._release()
    T4._release()


@pytest.fixture(scope="module", autouse=True)
def _free_models():
    yield
    _release_all()


def _qmodel(mode, kind):
    """(model, o32, o16, q32, q16) of test_fp8_decode_gpu / test_w4a16_decode_gpu: one model alive at a time"""
    own, other = (T8, T4) if mode == "fp8" else (T4, T8)
    if kind not in own._MODEL:
        other._release()
    return own._model(kind)


ENGINE_CASES = [(mode, kind) for kind in ("tiny", "8b-shallow", "lite-shallow") for mode in ("fp8", "w4a16")]


@pytest.mark.parametrize("mode,kind", ENGINE_CASES, ids=[f"{k}-{m}" for m, k in ENGINE_CASES])
def test_batched_decoder_quantized_teacher_forced(cuda, mode, kind):
    """the scenario of test_decode_engines_gpu._run_batched: 4096-token slots on the head and the split
    kernel, an idle slot, a released slot whose pages are reused"""
    from vila_b200 import serving
    model, o32, o16, q32, q16 = _qmodel(mode, kind)
    llm = model.llm
    n = 16
    with torch.inference_mode():
        llm.set_decode_weights(mode)
        try:
            dec = serving.BatchedDecoder(llm, slots=4, max_tokens_per_slot=4096, max_new=64)
            assert dec.decode_weights == mode and dec.configs == [None, 8]
            assert (dec.fp8 if mode == "fp8" else dec.w4) is not None
            dec.capture()
            lens = {0: 1015, 1: 2040, 3: 3065}
            prompts = {s: _prompt(llm, S, seed=S) for s, S in lens.items()}
            for s in lens:
                dec.admit(s, prompts[s])
            before = dec.pool.clone()
            dec.run(n - 1)
            assert dec.config == 8
            assert dec.generated(2) == [] and int(dec.positions[2]) == -1
            _check_untouched(before, dec.pool, [_decoded_rows(dec.page_tables[s], S, n) for s, S in lens.items()])
            _check_fp8_sequence(f"{kind} {mode} batched slot 0 S=1015", dec.pool, dec.page_tables[0], prompts[0],
                                dec.generated(0), o32, q32, o16, q16)
            freed = list(dec.slot_pages[0])
            dec.release(0)
            lens[0], prompts[0] = 500, _prompt(llm, 500, seed=500)
            dec.admit(0, prompts[0])
            assert set(dec.slot_pages[0]) <= set(freed)
            before = dec.pool.clone()
            dec.run(n - 1)
            assert dec.generated(2) == [] and int(dec.positions[2]) == -1
            decoded = [_decoded_rows(dec.page_tables[0], 500, n)]
            for s in (1, 3):
                pages, rows = _decoded_rows(dec.page_tables[s], lens[s], 2 * n - 1)
                decoded.append((pages[n - 1:], rows[n - 1:]))
            _check_untouched(before, dec.pool, decoded)
            for s in (0, 1, 3):
                ids = dec.generated(s)
                assert len(ids) == (n if s == 0 else 2 * n - 1)
                _check_fp8_sequence(f"{kind} {mode} batched slot {s} S={lens[s]}", dec.pool, dec.page_tables[s],
                                    prompts[s], ids, o32, q32, o16, q16)
        finally:
            llm.set_decode_weights("bf16")


def test_generate_batch_w4a16_slot_independence(cuda):
    from vila_b200 import serving
    model = _qmodel("w4a16", "tiny")[0]
    llm = model.llm
    prompts = [_prompt(llm, S, seed=S) for S in (120, 333, 57, 410, 260)]
    with torch.inference_mode():
        llm.set_decode_weights("w4a16")
        try:
            got3 = serving.generate_batch(llm, prompts, max_new_tokens=24, slots=3)
            got20 = serving.generate_batch(llm, prompts * 4, max_new_tokens=24, slots=20)  # 20 slots: two groups
            alone = [serving.generate_batch(llm, [p], max_new_tokens=24, slots=1)[0] for p in prompts]
        finally:
            llm.set_decode_weights("bf16")
    assert all(len(a) == 24 for a in alone)
    assert got3 == alone and got20 == alone * 4


def test_bf16_batched_unchanged_by_quantized_modes(cuda):
    from vila_b200 import serving
    model = _qmodel("w4a16", "lite-shallow")[0]  # tied lm_head
    llm = model.llm

    def run():
        dec = serving.BatchedDecoder(llm, slots=3, max_tokens_per_slot=1024, max_new=32)
        assert dec.decode_weights == "bf16"
        dec.capture()
        for s, S in enumerate((300, 170)):
            dec.admit(s, _prompt(llm, S, seed=S))
        dec.run(16)
        return [dec.generated(s) for s in range(3)], dec.pool.clone()

    with torch.inference_mode():
        ids_a, pool_a = run()
        llm.set_decode_weights("w4a16")
        dec_w4 = serving.BatchedDecoder(llm, slots=3, max_tokens_per_slot=1024, max_new=32)
        assert dec_w4.decode_weights == "w4a16"
        llm.set_decode_weights("fp8")
        with pytest.raises(ValueError):  # a decoder of another mode
            serving.generate_batch(llm, [_prompt(llm, 50, seed=1)], max_new_tokens=4, decoder=dec_w4)
        del dec_w4
        llm.set_decode_weights("bf16")
        ids_b, pool_b = run()
    assert ids_a == ids_b and torch.equal(pool_a, pool_b)
