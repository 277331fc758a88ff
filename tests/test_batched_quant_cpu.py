"""CPU: the batched engine on the quantized decode weights (fp8 / w4a16) without a device: the argument
errors of ops.gemv_batch, the loud failure of the new entry points, the ABI struct's field order, and how
serving.BatchedDecoder / generate_batch take the LLM's decode-weight mode."""
import re
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch

from vila_b200 import ops, serving

ROOT = Path(__file__).resolve().parent.parent


def _w4(N=64, K=256):
    return (torch.zeros((N + 15) // 16, 8 * K, dtype=torch.uint8), torch.ones(N, K // 128, dtype=torch.bfloat16),
            torch.zeros(N, K // 128, dtype=torch.uint8))


def _fp8(N=64, K=256):
    return torch.zeros(N, K, dtype=torch.float8_e4m3fn), torch.ones(N, dtype=torch.float32)


def test_gemv_batch_argument_errors():
    x = torch.zeros(4, 256, dtype=torch.bfloat16)
    q, s, z = _w4()
    q8, s8 = _fp8()
    with pytest.raises(ValueError, match="ops.linear"):  # bf16 batches keep the wgmma GEMM
        ops.gemv_batch(x, torch.zeros(64, 256, dtype=torch.bfloat16), w_scale=s8)
    with pytest.raises(ValueError):
        ops.gemv_batch(x, q, w_scale=None, w_zero=z)               # scales are required
    with pytest.raises(ValueError):
        ops.gemv_batch(x, q, w_scale=s)                            # zero points are required
    with pytest.raises(ValueError):
        ops.gemv_batch(x, q, w_scale=s[:32], w_zero=z[:32])        # packed rows do not match
    with pytest.raises(ValueError):
        ops.gemv_batch(x, q, w_scale=s[:, :1], w_zero=z)           # mis-shaped scales
    with pytest.raises(ValueError):
        ops.gemv_batch(x, q8, w_scale=s8, w_zero=z)                # zero points only with 4-bit weights
    with pytest.raises(ValueError):
        ops.gemv_batch(x, q8, w_scale=s8[:32])                     # one scale per row
    with pytest.raises(ValueError):
        ops.gemv_batch(x[:, :128], q8, w_scale=s8)                 # x does not match K
    with pytest.raises(ValueError):
        ops.gemv_batch(x, q8, w_scale=s8, residual=torch.zeros(4, 64, dtype=torch.bfloat16), swiglu=True)
    with pytest.raises(ValueError):
        ops.gemv_batch(x, q8, w_scale=s8, out=torch.zeros(4, 64, dtype=torch.bfloat16), swiglu=True)  # [M, N/2]
    with pytest.raises(ValueError):
        ops.gemv_batch(x, q8, w_scale=s8, residual=torch.zeros(3, 64, dtype=torch.bfloat16))
    with pytest.raises(ValueError):
        ops.gemv_batch(x, q8, w_scale=s8, bias=torch.zeros(63, dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="CUDA"):  # well-formed, but no CPU path exists
        ops.gemv_batch(x, q8, w_scale=s8)


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_gemv_batch_entry_points_fail_loudly_without_gpu():
    from vila_b200 import _lib
    lib = _lib.load()
    for rc in (lib.vila_gemv_batch_fp8(None, None, None), lib.vila_gemv_batch_w4a16(None, None, None, None),
               lib.vila_gemv_batch_partition(4608, 3584, 0, None)):
        assert rc != 0 and b"no CUDA device" in lib.vila_last_error()
    q, s, z = _w4()
    with pytest.raises(RuntimeError):
        ops.gemv_batch(torch.zeros(2, 256, dtype=torch.bfloat16), q, w_scale=s, w_zero=z)


def test_gemv_batch_struct_matches_header_field_order():
    from vila_b200 import _lib
    text = (ROOT / "include" / "vila_b200.h").read_text()
    body = re.search(r"typedef struct vila_gemv_batch_params \{(.*?)\} vila_gemv_batch_params;", text,
                     flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        names = decl.split(",")
        fields.append(names[0].split()[-1].lstrip("*"))
        fields.extend(x.strip().lstrip("*") for x in names[1:])
    assert fields == ["x", "ldx", "w", "bias", "residual", "ld_res", "y", "ldy", "M", "N", "K", "flags"]
    assert fields == [f[0] for f in _lib.GemvBatchParams._fields_]
    for name in ("vila_gemv_batch_fp8", "vila_gemv_batch_w4a16", "vila_gemv_batch_partition"):
        assert name in _lib.SIGNATURES and hasattr(_lib.load(), name)


def _duck_llm(mode=None):
    cfg = SimpleNamespace(num_attention_heads=2, num_key_value_heads=1, head_dim=128, num_hidden_layers=2,
                          hidden_size=64)
    llm = SimpleNamespace(config=cfg, device=torch.device("cpu"), dtype=torch.bfloat16)
    if mode is not None:
        llm.decode_weights = mode
        llm._fp8_weights = SimpleNamespace(layers=["fp8 layer"], lm_head="fp8 lm_head") if mode == "fp8" else None
        llm._w4_weights = SimpleNamespace(layers=["w4 layer"], lm_head="fp8 lm_head") if mode == "w4a16" else None
    return llm


def test_batched_decoder_takes_the_llm_mode_and_copies():
    dec = serving.BatchedDecoder(_duck_llm(), slots=2, max_tokens_per_slot=256, max_new=8)
    assert dec.decode_weights == "bf16" and dec.fp8 is None and dec.w4 is None  # an LLM without the attribute
    for mode in ("bf16", "fp8", "w4a16"):
        llm = _duck_llm(mode)
        dec = serving.BatchedDecoder(llm, slots=2, max_tokens_per_slot=256, max_new=8)
        assert dec.decode_weights == mode
        assert dec.fp8 is (llm._fp8_weights if mode == "fp8" else None)
        assert dec.w4 is (llm._w4_weights if mode == "w4a16" else None)
        held = (dec.fp8, dec.w4)
        llm._fp8_weights = llm._w4_weights = None  # the LLM switches modes: the decoder keeps its copies
        llm.decode_weights = "bf16"
        assert (dec.fp8, dec.w4) == held and dec.decode_weights == mode


def test_generate_batch_refuses_a_decoder_of_another_mode():
    prompts = [torch.zeros(10, 64)]
    dec = serving.BatchedDecoder(_duck_llm("w4a16"), slots=1, max_tokens_per_slot=256, max_new=8)
    for mode in ("bf16", "fp8"):
        with pytest.raises(ValueError, match="w4a16"):
            serving.generate_batch(_duck_llm(mode), prompts, max_new_tokens=4, decoder=dec)
    bf16_dec = serving.BatchedDecoder(_duck_llm(), slots=1, max_tokens_per_slot=256, max_new=8)
    with pytest.raises(ValueError, match="fp8"):
        serving.generate_batch(_duck_llm("fp8"), prompts, max_new_tokens=4, decoder=bf16_dec)
