"""CPU: the opt-in FP8 KV cache of the batched engine without a device: the format's rule (quantize_kv_e4m3) on
hand-picked rows and the round-trip bound it implies, the pool and staging bytes per page in both formats, the
kv_cache arguments of serving.BatchedDecoder / generate_batch, the argument errors of the new ops, the loud
failure of the new entry points and the ABI struct's field order."""
import math
import re
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from vila_b200 import ops, serving
from vila_b200.model.qwen2 import quantize_kv_e4m3

ROOT = Path(__file__).resolve().parent.parent


def _codes(c):
    return c.view(torch.uint8).tolist()


def _half_ulp(c: torch.Tensor) -> torch.Tensor:
    """half the e4m3 spacing at each code (normals: 2^(e-3); subnormals and zero: 2^-9)"""
    a = c.float().abs()
    e = torch.floor(torch.log2(a.clamp(min=2.0 ** -6)))
    return torch.exp2(e - 3) / 2


def test_rule_zero_rows():
    x = torch.zeros(3, 128, dtype=torch.bfloat16)
    x[1] = -0.0
    c, s = quantize_kv_e4m3(x)
    assert c.dtype == torch.float8_e4m3fn and s.dtype == torch.float32 and s.shape == (3,)
    assert all(v == 0 for row in _codes(c) for v in row)  # no negative-zero codes either
    assert s.tolist() == [0.0, 0.0, 0.0]


def test_rule_amax_maps_to_448():
    x = torch.zeros(2, 128, dtype=torch.bfloat16)
    x[0, 5], x[0, 9] = -3.5, 1.75
    x[1, 0], x[1, 127] = 0.0078125, -0.00390625
    c, s = quantize_kv_e4m3(x)
    assert _codes(c)[0][5] == 0xFE and _codes(c)[0][9] == 0x76        # -448, 224
    assert _codes(c)[1][0] == 0x7E and _codes(c)[1][127] == 0xF6      # 448, -224
    assert s.tolist() == [float(np.float32(3.5) / np.float32(448)), float(np.float32(0.0078125) / np.float32(448))]
    assert c.float()[0, 5].item() * s[0].item() == -3.5


def test_rule_divides_in_ieee_fp32():
    """inv = 448 / amax and scale = amax / 448 are correctly rounded fp32 divisions, as in the kernels"""
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(4096, 128, generator=g) * torch.logspace(-3, 3, 4096)[:, None]).bfloat16()
    c, s = quantize_kv_e4m3(x)
    amax = x.float().abs().amax(dim=1).numpy()
    inv = np.float32(448) / amax
    assert np.array_equal(s.numpy(), amax / np.float32(448))
    ref = torch.from_numpy(np.clip(x.float().numpy() * inv[:, None], -448, 448)).to(torch.float8_e4m3fn)
    assert torch.equal(c.view(torch.uint8), ref.view(torch.uint8))


def test_rule_subnormals_round_to_nearest_even():
    x = torch.zeros(1, 128, dtype=torch.bfloat16)
    x[0, 0] = 448.0                     # inv = 1 exactly
    vals = [2.0 ** -9, 3 * 2.0 ** -9, 2.0 ** -10, 1.5 * 2.0 ** -9, 2.5 * 2.0 ** -9, 7 * 2.0 ** -9, 2.0 ** -6]
    for i, v in enumerate(vals):
        x[0, 1 + i] = v
        x[0, 64 + i] = -v
    c, s = quantize_kv_e4m3(x)
    assert s.item() == 1.0
    got = _codes(c)[0]
    # 2^-9 -> 1, 3*2^-9 -> 3, 2^-10 -> 0 (tie to even), 1.5*2^-9 -> 2, 2.5*2^-9 -> 2, 7*2^-9 -> 7, 2^-6 -> normal
    assert got[1:8] == [0x01, 0x03, 0x00, 0x02, 0x02, 0x07, 0x08]
    assert got[64:71] == [0x81, 0x83, 0x80, 0x82, 0x82, 0x87, 0x88]


def test_rule_saturates_instead_of_overflowing():
    # rows whose amax * (448 / amax) rounds above 448 in fp32: the clamp keeps the code at +-448, never NaN
    amaxes = []
    for k in range(1, 20000):
        a = torch.tensor(1.0 + k * 2.0 ** -7, dtype=torch.bfloat16).float()
        if float(np.float32(a.item()) * (np.float32(448) / np.float32(a.item()))) > 448.0:
            amaxes.append(a.item())
    assert amaxes, "no bf16 amax overshoots 448 in fp32"
    x = torch.zeros(len(amaxes), 128, dtype=torch.bfloat16)
    x[:, 3] = torch.tensor(amaxes)
    x[:, 4] = -torch.tensor(amaxes)
    c, _ = quantize_kv_e4m3(x)
    u = c.view(torch.uint8)
    assert (u[:, 3] == 0x7E).all() and (u[:, 4] == 0xFE).all()
    assert not torch.isnan(c.float()).any()


def test_round_trip_within_half_an_e4m3_ulp():
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(512, 128, generator=g) * torch.logspace(-4, 3, 512)[:, None]).bfloat16()
    x[7, :] = 0
    x[8, 17] = 1e4  # an outlier sets the row's scale
    c, s = quantize_kv_e4m3(x)
    deq = c.float() * s[:, None]
    err = (deq - x.float()).abs()
    # |code - x*inv| <= half an ulp of the code; inv * scale = 1 up to two fp32 roundings
    bound = _half_ulp(c) * s[:, None] + 2.0 ** -21 * x.float().abs().amax(dim=1, keepdim=True)
    assert (err <= bound).all(), float((err - bound).max())
    assert (deq[7] == 0).all()


def _duck_llm(L=28, Hq=28, Hkv=4):
    cfg = SimpleNamespace(num_attention_heads=Hq, num_key_value_heads=Hkv, head_dim=128, num_hidden_layers=L,
                          hidden_size=64)
    return SimpleNamespace(config=cfg, device=torch.device("cpu"), dtype=torch.bfloat16)


def test_pool_and_staging_bytes_per_page():
    L, Hkv, P = 28, 4, 3
    bf = serving.BatchedDecoder(_duck_llm(L), slots=1, max_tokens_per_slot=256, max_new=8, total_pages=P)
    f8 = serving.BatchedDecoder(_duck_llm(L), slots=1, max_tokens_per_slot=256, max_new=8, total_pages=P,
                                kv_cache="fp8")
    assert bf.kv_cache == "bf16" and bf.pool_scale is None and not hasattr(bf, "staging")
    assert bf.pool.dtype == torch.bfloat16 and f8.pool.dtype == torch.float8_e4m3fn
    assert f8.pool.shape == bf.pool.shape == (L, 2, P, 128, Hkv, 128)
    assert f8.pool_scale.shape == (L, 2, P, 128, Hkv) and f8.pool_scale.dtype == torch.float32

    def nbytes(*ts):
        return sum(t.numel() * t.element_size() for t in ts)

    per_token_bf16 = nbytes(bf.pool) // (P * 128)
    per_token_fp8 = nbytes(f8.pool, f8.pool_scale) // (P * 128)
    assert per_token_bf16 == 57_344 and per_token_fp8 == 29_568  # NVILA-8B: 28 layers, 4 KV heads, head_dim 128
    assert per_token_fp8 / per_token_bf16 == pytest.approx(0.516, abs=5e-4)
    # the bf16 staging cache holds one slot (2 pages here) with an identity page table
    assert f8.staging.shape == (L, 2, 2, 128, Hkv, 128) and f8.staging.dtype == torch.bfloat16
    assert nbytes(f8.staging) == 2 * 128 * per_token_bf16
    assert f8.staging_pages.tolist() == [0, 1]
    # the README's staging figures: one slot of bf16 K/V at 2048 and 69,632 tokens
    assert 2048 * per_token_bf16 / 1e9 == pytest.approx(0.12, abs=0.005)
    assert serving.MAX_SLOT_TOKENS * per_token_bf16 / 1e9 == pytest.approx(3.99, abs=0.005)


def test_fp8_ladder_and_configurations():
    S = serving.FP8_SPLIT_TOKENS
    assert serving.FP8_LADDER_TOKENS[-1] == serving.MAX_SLOT_TOKENS
    assert all(n % S == 0 or n == serving.MAX_SLOT_TOKENS for n in serving.FP8_LADDER_TOKENS)
    assert serving.fp8_attention_config(1) == 2048 // S
    assert serving.fp8_attention_config(2048) == 2048 // S
    assert serving.fp8_attention_config(2049) == 8192 // S
    assert serving.fp8_attention_config(16_470) == 32768 // S
    assert serving.fp8_attention_config(serving.MAX_SLOT_TOKENS) == math.ceil(serving.MAX_SLOT_TOKENS / S)
    with pytest.raises(ValueError):
        serving.fp8_attention_config(serving.MAX_SLOT_TOKENS + 1)
    small = serving.BatchedDecoder(_duck_llm(2, 4, 2), slots=2, max_tokens_per_slot=2048, max_new=8, kv_cache="fp8")
    assert small.configs == [2048 // S]
    big = serving.BatchedDecoder(_duck_llm(2, 4, 2), slots=2, max_tokens_per_slot=16_600, max_new=8, kv_cache="fp8",
                                 total_pages=4)
    assert big.configs == [serving.fp8_attention_config(n) for n in (2048, 8192, 16384, 32768)]
    assert big.ws.numel() == 2 * 4 * big.configs[-1] * 130 and big.counters.numel() == 2 * 2
    big.config = big.configs[-1]
    assert big.launches_per_step == 7 * 2 + 2  # one attention launch per layer for every slot length


def test_kv_cache_argument_validation():
    with pytest.raises(ValueError, match="kv_cache"):
        serving.BatchedDecoder(_duck_llm(2, 4, 2), slots=1, max_tokens_per_slot=256, max_new=8, kv_cache="int8")
    prompts = [torch.zeros(10, 64)]
    with pytest.raises(ValueError, match="kv_cache"):
        serving.generate_batch(_duck_llm(2, 4, 2), prompts, max_new_tokens=4, kv_cache="fp16")
    f8 = serving.BatchedDecoder(_duck_llm(2, 4, 2), slots=1, max_tokens_per_slot=256, max_new=8, kv_cache="fp8")
    bf = serving.BatchedDecoder(_duck_llm(2, 4, 2), slots=1, max_tokens_per_slot=256, max_new=8)
    with pytest.raises(ValueError, match="fp8"):
        serving.generate_batch(_duck_llm(2, 4, 2), prompts, max_new_tokens=4, decoder=f8)  # default bf16
    with pytest.raises(ValueError, match="bf16"):
        serving.generate_batch(_duck_llm(2, 4, 2), prompts, max_new_tokens=4, decoder=bf, kv_cache="fp8")


def _attn_args(Hq=28, Hkv=4, B=2, P=4, pages=4, dtype=torch.float8_e4m3fn):
    return dict(qkv=torch.zeros(B, (Hq + 2 * Hkv) * 128, dtype=torch.bfloat16),
                positions=torch.zeros(B, dtype=torch.int32),
                k_pool=torch.zeros(P, 128, Hkv, 128, dtype=dtype), v_pool=torch.zeros(P, 128, Hkv, 128, dtype=dtype),
                k_scale=torch.zeros(P, 128, Hkv), v_scale=torch.zeros(P, 128, Hkv),
                page_tables=torch.zeros(B, pages, dtype=torch.int32),
                out=torch.zeros(B, Hq * 128, dtype=torch.bfloat16), ws=torch.zeros(B * Hq * 4 * 130),
                counters=torch.zeros(B * Hkv, dtype=torch.int32), inv_freq=torch.zeros(64),
                Hq=Hq, Hkv=Hkv, num_splits=4, split_tokens=512, scale=128 ** -0.5)


def test_ops_argument_errors():
    a = _attn_args()
    with pytest.raises(ValueError, match="<= 16"):
        ops.decode_attention_fp8_batch(**{**_attn_args(Hq=34, Hkv=2), "ws": torch.zeros(2 * 34 * 4 * 130)})
    with pytest.raises(ValueError, match="head_dim"):
        ops.decode_attention_fp8_batch(**{**a, "qkv": torch.zeros(2, 36 * 64, dtype=torch.bfloat16)})
    with pytest.raises(ValueError):
        ops.decode_attention_fp8_batch(**{**a, "split_tokens": 200})
    with pytest.raises(ValueError):
        ops.decode_attention_fp8_batch(**{**a, "ws": torch.zeros(10)})
    with pytest.raises(ValueError):
        ops.decode_attention_fp8_batch(**{**a, "k_scale": torch.zeros(4, 128, 2)})
    with pytest.raises(ValueError, match="float8_e4m3fn"):  # a bf16 pool is not an e4m3 pool
        ops.decode_attention_fp8_batch(**_attn_args(dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="CUDA"):  # well-formed, but no CPU path exists
        ops.decode_attention_fp8_batch(**a)
    src = torch.zeros(2, 2, 2, 128, 4, 128, dtype=torch.bfloat16)
    dst = torch.zeros(2, 2, 5, 128, 4, 128, dtype=torch.float8_e4m3fn)
    sc = torch.zeros(2, 2, 5, 128, 4)
    row = torch.zeros(2, dtype=torch.int32)
    with pytest.raises(ValueError):
        ops.kv_quantize_fp8(src, dst, sc, row, 257)                   # more rows than the staging cache
    with pytest.raises(ValueError):
        ops.kv_quantize_fp8(src, dst, sc, row[:1], 200)               # more pages than the page row
    with pytest.raises(ValueError):
        ops.kv_quantize_fp8(src, dst[:1], sc, row, 10)                # layers do not match
    with pytest.raises(ValueError, match="float8_e4m3fn"):
        ops.kv_quantize_fp8(src, dst.view(torch.uint8), sc, row, 10)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.kv_quantize_fp8(src, dst, sc, row, 10)


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_entry_points_fail_loudly_without_gpu():
    from vila_b200 import _lib
    lib = _lib.load()
    for rc in (lib.vila_decode_attention_fp8_batch(None, None),
               lib.vila_kv_quantize_fp8(None, 0, None, None, 0, None, 0, 1, 1, 128, 0, None)):
        assert rc != 0 and b"no CUDA device" in lib.vila_last_error()


def test_struct_matches_header_field_order():
    from vila_b200 import _lib
    text = (ROOT / "include" / "vila_b200.h").read_text()
    body = re.search(r"typedef struct vila_decode_attn_fp8_params \{(.*?)\} vila_decode_attn_fp8_params;", text,
                     flags=re.S).group(1)
    fields = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        names = decl.split(",")
        fields.append(names[0].split()[-1].lstrip("*"))
        fields.extend(x.strip().lstrip("*") for x in names[1:])
    assert fields == [f[0] for f in _lib.DecodeAttnFp8Params._fields_]
    assert fields[:11] == ["qkv", "position", "k_pool", "v_pool", "k_scale", "v_scale", "page_table", "out", "ws",
                           "counters", "inv_freq"]
    for name in ("vila_kv_quantize_fp8", "vila_decode_attention_fp8_batch"):
        assert name in _lib.SIGNATURES and hasattr(_lib.load(), name)
