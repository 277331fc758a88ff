"""CPU: the W4A16 (4-bit, group-128 scale and zero point) decode-weight quantizer rule and its packed
layout, the decode-weight mode's arguments and state, and the w4a16 GEMV entry point failing loudly
without a device."""
import pytest
import torch


def _qw():
    from vila_b200.model.qwen2 import dequantize_w4_groups, quantize_w4_groups
    return quantize_w4_groups, dequantize_w4_groups


def _rule(w):
    """the quantizer rule restated plainly, one group at a time -> (q [N, K] int, s fp32 [N, G], z [N, G])"""
    N, K = w.shape
    q = torch.empty(N, K, dtype=torch.int64)
    s = torch.empty(N, K // 128)
    z = torch.empty(N, K // 128, dtype=torch.int64)
    for n in range(N):
        for g in range(K // 128):
            v = w[n, 128 * g:128 * (g + 1)].float()
            lo, hi = min(0.0, v.min().item()), max(0.0, v.max().item())
            sc = torch.tensor((hi - lo) / 15, dtype=torch.float32).to(torch.bfloat16).float().item()
            if sc == 0:
                sc = 1.0
            zp = int(min(15, max(0, torch.round(torch.tensor(-lo / sc, dtype=torch.float32)).item())))
            q[n, 128 * g:128 * (g + 1)] = (torch.round(v / sc) + zp).clamp(0, 15).long()
            s[n, g], z[n, g] = sc, zp
    return q, s, z


def _special_rows():
    g = torch.Generator().manual_seed(0)
    rows = [
        torch.rand(256, generator=g) + 0.1,             # only positive values
        -(torch.rand(256, generator=g) + 0.1),          # only negative values
        torch.zeros(256),                               # all zero
        torch.full((256,), 0.37),                       # constant
        torch.randn(256, generator=g) * 1e-3,           # rows of very different magnitude
        torch.randn(256, generator=g) * 40,
    ]
    w = torch.stack(rows)
    w[3, 128:] = -2.5  # a constant negative group
    return torch.cat([w, torch.randn(11, 256, generator=g) * torch.exp(torch.randn(11, 1, generator=g))]).to(torch.bfloat16)


def test_quantizer_rule_bit_for_bit():
    quant, deq = _qw()
    w = _special_rows()
    packed, s, z = quant(w)
    q, s_ref, z_ref = _rule(w)
    assert s.dtype == torch.bfloat16 and z.dtype == torch.uint8 and s.shape == z.shape == (w.shape[0], 2)
    assert torch.equal(s.float(), s_ref) and torch.equal(z.long(), z_ref)
    want = (q - z_ref.repeat_interleave(128, 1)).float() * s_ref.repeat_interleave(128, 1)
    assert torch.equal(deq(packed, s, z), want)
    # the all-zero group: s = 1, z = 0, dequantized zeros
    assert s[2, 0].item() == 1.0 and z[2, 0].item() == 0 and torch.equal(deq(packed, s, z)[2], torch.zeros(256))
    # zero is exact: a group of only positive values has z = 0, only negative values z = 15
    assert bool((z[0] == 0).all()) and bool((z[1] == 15).all())


def test_error_within_half_a_step():
    quant, deq = _qw()
    g = torch.Generator().manual_seed(1)
    w = torch.cat([_special_rows().float(), torch.randn(64, 512, generator=g)[:, :256]]).to(torch.bfloat16)
    packed, s, z = quant(w)
    err = (deq(packed, s, z) - w.float()).abs()
    bound = 0.55 * s.float().repeat_interleave(128, 1)
    assert bool((err <= bound).all()), (err / bound).max()


def test_grid_values_round_trip_exactly():
    quant, deq = _qw()
    g = torch.Generator().manual_seed(2)
    N, K = 24, 512
    z = torch.randint(0, 16, (N, K // 128), generator=g)
    s = 2.0 ** torch.randint(-12, 2, (N, K // 128), generator=g).float()
    q = torch.randint(0, 16, (N, K), generator=g)
    q[:, 0::128] = 0   # codes 0 and 15 in every group
    q[:, 1::128] = 15
    w = ((q - z.repeat_interleave(128, 1)).float() * s.repeat_interleave(128, 1))
    assert torch.equal(w.to(torch.bfloat16).float(), w)
    packed, s2, z2 = quant(w.to(torch.bfloat16))
    assert torch.equal(deq(packed, s2, z2), w)


def test_chunked_matches_one_pass():
    from vila_b200.model.qwen2 import quantize_w4_groups
    w = torch.randn(100, 256, generator=torch.Generator().manual_seed(3)).to(torch.bfloat16)
    a = quantize_w4_groups(w)
    b = quantize_w4_groups(w, rows_per_chunk=32)
    c = quantize_w4_groups(w, rows_per_chunk=7)  # rounded to whole 16-row tiles
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and all(torch.equal(x, y) for x, y in zip(a, c))


def test_interleaved_gate_up_rows_are_quantized_per_row():
    quant, deq = _qw()
    g = torch.Generator().manual_seed(4)
    gate = torch.randn(8, 256, generator=g).to(torch.bfloat16)
    up = (torch.randn(8, 256, generator=g) * 50).to(torch.bfloat16)
    gu = torch.stack([gate, up], dim=1).reshape(16, 256)  # rows: gate_0, up_0, gate_1, ...
    d = deq(*quant(gu))
    assert torch.equal(d[0::2], deq(*quant(gate))) and torch.equal(d[1::2], deq(*quant(up)))


@pytest.mark.parametrize("N,K", [(16, 128), (37, 512), (1003, 256), (48, 3584)])
def test_pack_unpack_round_trip(N, K):
    from vila_b200.model.qwen2 import _w4_pack, _w4_unpack
    g = torch.Generator().manual_seed(N + K)
    R = (N + 15) // 16 * 16
    q = torch.randint(0, 16, (R, K), generator=g, dtype=torch.uint8)
    packed = _w4_pack(q)
    assert packed.shape == (R // 16, 8 * K) and packed.dtype == torch.uint8
    assert torch.equal(_w4_unpack(packed, K), q)
    # through the public pair: codes of N rows, the padding rows are zero codes
    w = torch.randn(N, K, generator=g).to(torch.bfloat16)
    quant, deq = _qw()
    packed, s, z = quant(w)
    assert packed.shape == (R // 16, 8 * K) and s.shape == (N, K // 128)
    assert bool((_w4_unpack(packed, K)[N:] == 0).all())
    q_ref, s_ref, z_ref = _rule(w) if N * K <= 37 * 512 else (None, None, None)
    if q_ref is not None:
        assert torch.equal(_w4_unpack(packed, K)[:N].long(), q_ref)


def test_rejects_k_not_multiple_of_128():
    quant, _ = _qw()
    with pytest.raises(ValueError):
        quant(torch.zeros(16, 192, dtype=torch.bfloat16))


def _cpu_llm(**kw):
    from vila_b200.model import tiny_test_config
    from vila_b200.model.qwen2 import Qwen2ForCausalLM
    cfg = tiny_test_config(llm_layers=2).llm_cfg
    for k, v in kw.items():
        setattr(cfg, k, v)
    llm = Qwen2ForCausalLM(cfg, device="cpu")
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for p in llm.state_dict().values():
            p.copy_(torch.randn(p.shape, generator=g) * 0.05)
    return llm


def test_set_decode_weights_w4a16_arguments_and_state():
    from vila_b200.model.qwen2 import dequantize_w4_groups, quantize_e4m3_rows
    llm = _cpu_llm()
    for bad in ("int4", "W4A16", "w4", "awq"):
        with pytest.raises(ValueError):
            llm.set_decode_weights(bad)
    assert llm.decode_weights == "bf16"
    keys = list(llm.state_dict())
    before = {k: v.clone() for k, v in llm.state_dict().items()}
    llm._decoder = object()
    llm.set_decode_weights("w4a16")
    assert llm.decode_weights == "w4a16" and llm._decoder is None and llm._fp8_weights is None
    f = llm._w4_weights
    layer = llm.model.layers[0]
    packed, s, z = f.layers[0].gu
    assert packed.dtype == torch.uint8 and s.shape == (layer._gu_w.shape[0], layer._gu_w.shape[1] // 128)
    d = dequantize_w4_groups(*f.layers[0].down)
    assert d.shape == layer.mlp.down_proj.weight.shape
    q, sc = quantize_e4m3_rows(llm.lm_head.weight)  # lm_head stays e4m3
    assert torch.equal(f.lm_head[1], sc) and torch.equal(f.lm_head[0].float(), q.float())
    assert list(llm.state_dict()) == keys
    assert all(torch.equal(v, before[k]) for k, v in llm.state_dict().items())
    # switching frees the previous copies and drops the cached decoder
    llm._decoder = object()
    llm.set_decode_weights("fp8")
    assert llm._w4_weights is None and llm._fp8_weights is not None and llm._decoder is None
    llm.set_decode_weights("w4a16")
    assert llm._fp8_weights is None and llm._w4_weights is not None
    llm.set_decode_weights("bf16")
    assert llm.decode_weights == "bf16" and llm._fp8_weights is None and llm._w4_weights is None
    assert all(torch.equal(v, before[k]) for k, v in llm.state_dict().items())


def test_w4a16_refuses_k_not_multiple_of_128_before_quantizing():
    llm = _cpu_llm(intermediate_size=1000)  # down_proj K = 1000
    llm.set_decode_weights("fp8")
    dec = llm._decoder = object()
    with pytest.raises(ValueError, match="128"):
        llm.set_decode_weights("w4a16")
    assert llm.decode_weights == "fp8" and llm._fp8_weights is not None and llm._w4_weights is None
    assert llm._decoder is dec


def test_load_pretrained_takes_w4a16(tmp_path):
    import inspect

    from vila_b200.model.loading import load_pretrained
    with pytest.raises(ValueError):
        load_pretrained(str(tmp_path), device="cpu", decode_weights="int4")
    assert "w4a16" in inspect.getsource(load_pretrained)


def test_server_flag_accepts_w4a16():
    import inspect

    from vila_b200 import server
    assert '"w4a16"' in inspect.getsource(server.main)


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_gemv_w4a16_fails_loudly_without_gpu():
    from vila_b200 import _lib, ops
    lib = _lib.load()
    rc = lib.vila_gemv_w4a16(None, None, None, None)
    assert rc != 0 and b"no CUDA device" in lib.vila_last_error()
    x = torch.zeros(128, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError):
        ops.gemv(x, torch.zeros(1, 1024, dtype=torch.uint8), w_scale=torch.ones(8, 1, dtype=torch.bfloat16),
                 w_zero=torch.zeros(8, 1, dtype=torch.uint8))
