"""CPU: the FP8 (e4m3) decode-weight quantizer rule, the decode-weight mode's arguments, and the fp8 GEMV
entry point failing loudly without a device."""
import pytest
import torch


def _quant(w):
    from vila_b200.model.qwen2 import quantize_e4m3_rows
    return quantize_e4m3_rows(w)


def test_scales_are_row_amax_over_448():
    g = torch.Generator().manual_seed(0)
    w = (torch.randn(64, 256, generator=g) * torch.exp(torch.randn(64, 1, generator=g))).to(torch.bfloat16)
    q, s = _quant(w)
    assert q.dtype == torch.float8_e4m3fn and q.shape == w.shape and s.dtype == torch.float32 and s.shape == (64,)
    assert torch.equal(s, w.float().abs().amax(dim=1) / 448)
    assert torch.equal(q, (w.float() / s[:, None]).to(torch.float8_e4m3fn))
    qf = q.float()
    assert bool(torch.isfinite(qf).all()) and qf.abs().max().item() <= 448
    assert torch.equal(qf.abs().amax(dim=1), torch.full((64,), 448.0))  # each row's largest reaches the top
    # dequantized error: within half an e4m3 step (3 mantissa bits) of each value, or of the subnormal step
    err = (qf * s[:, None] - w.float()).abs()
    assert bool((err <= torch.maximum(w.float().abs() * 2 ** -4, s[:, None] * 2 ** -10) * 1.0001).all())


def test_grid_values_round_trip_exactly():
    # every finite e4m3 code times a power-of-two scale (exact in fp32 and bf16)
    codes = torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn).float()
    codes = codes[torch.isfinite(codes)]
    assert codes.abs().max().item() == 448
    for scale in (2.0 ** -12, 2.0 ** -3, 1.0):
        w = (codes * scale)[None].to(torch.bfloat16)
        assert torch.equal(w.float(), codes[None] * scale)
        q, s = _quant(w)
        assert s.item() == scale
        assert torch.equal(q.float(), codes[None])  # the same codes, bit for bit
        assert torch.equal(q.float() * s[:, None], w.float())


def test_zero_row_gets_scale_one():
    w = torch.zeros(3, 64, dtype=torch.bfloat16)
    w[1] = torch.linspace(-2, 2, 64)
    q, s = _quant(w)
    assert s[0].item() == 1.0 and s[2].item() == 1.0 and s[1].item() == (torch.tensor(2.0) / 448).item()
    assert torch.equal(q[0].float(), torch.zeros(64)) and torch.equal(q[2].float(), torch.zeros(64))


def test_interleaved_gate_up_rows_are_quantized_per_row():
    g = torch.Generator().manual_seed(1)
    gate = torch.randn(8, 128, generator=g).to(torch.bfloat16)
    up = (torch.randn(8, 128, generator=g) * 50).to(torch.bfloat16)
    gu = torch.stack([gate, up], dim=1).reshape(16, 128)  # rows: gate_0, up_0, gate_1, ...
    q, s = _quant(gu)
    qg, sg = _quant(gate)
    qu, su = _quant(up)
    assert torch.equal(s[0::2], sg) and torch.equal(s[1::2], su)
    assert torch.equal(q[0::2].float(), qg.float()) and torch.equal(q[1::2].float(), qu.float())


def test_chunked_rows_match_one_pass():
    from vila_b200.model.qwen2 import quantize_e4m3_rows
    w = torch.randn(100, 64, generator=torch.Generator().manual_seed(2)).to(torch.bfloat16)
    q1, s1 = quantize_e4m3_rows(w)
    q2, s2 = quantize_e4m3_rows(w, rows_per_chunk=7)
    assert torch.equal(s1, s2) and torch.equal(q1.float(), q2.float())


def _cpu_llm():
    from vila_b200.model import tiny_test_config
    from vila_b200.model.qwen2 import Qwen2ForCausalLM
    llm = Qwen2ForCausalLM(tiny_test_config(llm_layers=2).llm_cfg, device="cpu")
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for p in llm.state_dict().values():
            p.copy_(torch.randn(p.shape, generator=g) * 0.05)
    return llm


def test_set_decode_weights_arguments_and_state():
    llm = _cpu_llm()
    assert llm.decode_weights == "bf16"
    for bad in ("int8", "FP8", "e4m3", None, 8):
        with pytest.raises(ValueError):
            llm.set_decode_weights(bad)
    assert llm.decode_weights == "bf16"
    keys = list(llm.state_dict())
    before = {k: v.clone() for k, v in llm.state_dict().items()}
    llm._decoder = object()
    llm.set_decode_weights("fp8")
    assert llm.decode_weights == "fp8" and llm._decoder is None
    f = llm._fp8_weights
    layer = llm.model.layers[0]
    assert f.layers[0].gu[0].shape == layer._gu_w.shape and f.layers[0].gu[0].dtype == torch.float8_e4m3fn
    assert torch.equal(f.layers[0].qkv[1], _quant(layer._qkv_w)[1])
    assert torch.equal(f.lm_head[1], _quant(llm.lm_head.weight)[1])
    assert list(llm.state_dict()) == keys
    assert all(torch.equal(v, before[k]) for k, v in llm.state_dict().items())
    llm.set_decode_weights("bf16")
    assert llm.decode_weights == "bf16" and llm._fp8_weights is None


def test_load_pretrained_rejects_unknown_decode_weights(tmp_path):
    from vila_b200.model.loading import load_pretrained
    with pytest.raises(ValueError):
        load_pretrained(str(tmp_path), device="cpu", decode_weights="int4")


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_gemv_fp8_fails_loudly_without_gpu():
    from vila_b200 import _lib, ops
    lib = _lib.load()
    rc = lib.vila_gemv_fp8(None, None, None)
    assert rc != 0 and b"no CUDA device" in lib.vila_last_error()
    x = torch.zeros(64, dtype=torch.bfloat16)
    q = torch.zeros(8, 64, dtype=torch.float8_e4m3fn)
    with pytest.raises(RuntimeError):
        ops.gemv(x, q, w_scale=torch.ones(8))
