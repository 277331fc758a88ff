"""CPU: presence / frequency penalties of the continuous-batching engine without a device: PenaltyParams validation,
the numpy rule of vila_b200/penalties.py on hand-built rows (repeats, t = 0, t beyond the history, negative penalties,
ids outside the vocabulary, bf16 rounding against hand-computed bits), the argument errors of ops.apply_penalties, the
loud failure of the entry point, the struct's field order against the header, the host logic of BatchedDecoder and
generate_batch, and the server's penalty plumbing on a stub model (validation before batching, routing, no keyword when
nobody asked, the streaming refusal)."""
import asyncio
import inspect
import math
import re
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from vila_b200 import ops, serving
from vila_b200.penalties import PenaltyParams, reference_penalized, reference_penalized64

ROOT = Path(__file__).resolve().parent.parent


def _bits(t: torch.Tensor):
    return t.view(torch.int16).tolist()


def test_penalty_params_validation():
    assert PenaltyParams().off and PenaltyParams(0, 0.0).off
    assert not PenaltyParams(presence=0.5).off and not PenaltyParams(frequency=-2).off
    for ok in (-2, -2.0, 2.0, 1.5, np.float32(0.25)):
        PenaltyParams(presence=ok, frequency=ok)
    for bad in (2.0001, -2.5, math.inf, -math.inf, math.nan, "0.5", None, True, [1.0]):
        with pytest.raises(ValueError, match=r"\[-2, 2\]"):
            PenaltyParams(presence=bad)
        with pytest.raises(ValueError, match="frequency"):
            PenaltyParams(frequency=bad)
    with pytest.raises(Exception):
        PenaltyParams().presence = 1.0  # frozen


def test_rule_counts_frequency_per_repeat_and_presence_once():
    x = torch.tensor([1.0, 2.0, 3.0, 4.0, 5.0, 6.0], dtype=torch.bfloat16)
    hist = [2, 2, 2, 4, 0]
    y = reference_penalized(x, hist, 5, presence=0.5, frequency=0.25)
    # id 2 three times: 3 - (3 * 0.25 + 0.5) = 1.75; id 4 once: 5 - 0.75 = 4.25; id 0 once: 1 - 0.75 = 0.25
    assert y.float().tolist() == [0.25, 2.0, 1.75, 4.0, 4.25, 6.0]
    for k in (1, 3, 5):  # untouched entries are bit-identical copies
        assert _bits(y[k:k + 1]) == _bits(x[k:k + 1])
    # only the first t ids count
    assert reference_penalized(x, hist, 2, 0.5, 0.25).float().tolist() == [1.0, 2.0, 2.0, 4.0, 5.0, 6.0]
    # t = 0: an empty history, the row is returned as it is
    assert _bits(reference_penalized(x, hist, 0, 2.0, 2.0)) == _bits(x)
    # t beyond the history: every id counts
    assert torch.equal(reference_penalized(x, hist, 100, 0.5, 0.25), y)
    # penalties 0 / 0 leave every bit alone
    assert _bits(reference_penalized(x, hist, 5, 0.0, 0.0)) == _bits(x)


def test_rule_negative_penalties_and_foreign_ids():
    x = torch.tensor([1.0, -2.0, 0.0, 8.0], dtype=torch.bfloat16)
    y = reference_penalized(x, [1, 1, -1, 4, 99, 3, -7], 7, presence=-1.0, frequency=-0.5)
    # id 1 twice: -2 - (2 * -0.5 - 1) = 0; id 3 once: 8 + 1.5 = 9.5; -1, 4, 99, -7 are not ids of V = 4
    assert y.float().tolist() == [1.0, 0.0, 0.0, 9.5]
    assert _bits(y[2:3]) == _bits(x[2:3])


def test_rule_bf16_rounding_against_hand_computed_bits():
    x = torch.tensor([1.0, 20.0, 17.0, 16.0, -3.0], dtype=torch.bfloat16)
    assert [b & 0xFFFF for b in _bits(x)] == [0x3F80, 0x41A0, 0x4188, 0x4180, 0xC040]
    # 1 - 0.5 = 0.5 (0x3F00); 20 - 0.03125 = 19.96875 -> 20.0 (bf16 ulp 0.125 in [16, 32)); 17 - 0.0625 = 16.9375 is
    # the midpoint of 16.875 (mantissa 7, odd) and 17.0 (mantissa 8, even) -> 17.0; 16 - 0.0625 = 15.9375, exact in
    # [8, 16) (0x417F); -3 - 0.5 = -3.5 (0xC060)
    rows = [(0, 0.5, 0.0), (1, 0.03125, 0.0), (2, 0.0, 0.0625), (3, 0.0625, 0.0), (4, 0.25, 0.25)]
    want = [0x3F00, 0x41A0, 0x4188, 0x417F, 0xC060]
    for (j, p, f), w in zip(rows, want):
        y = reference_penalized(x, [j], 1, presence=p, frequency=f)
        assert y[j].view(torch.int16).item() & 0xFFFF == w, (j, p, f)
        assert abs(float(y[j]) - reference_penalized64(x, [j], 1, p, f)[j]) <= 0.0625


def test_rule_fp32_order_of_operations():
    """pen = fp32(fp32(c * f) + p), then fp32(x - pen), then bf16: checked against numpy fp32 step by step on a random
    row with many repeats, and within half a bf16 ulp (plus the fp32 steps) of the fp64 form"""
    g = np.random.default_rng(3)
    V = 4096
    x = torch.from_numpy(g.normal(0, 12, V).astype(np.float32)).bfloat16()
    hist = g.integers(0, 300, 2000)
    f, p = np.float32(0.3), np.float32(0.7)
    y = reference_penalized(x, hist, len(hist), float(p), float(f))
    c = np.bincount(hist, minlength=V)
    pen = (c.astype(np.float32) * f).astype(np.float32) + p
    z = torch.from_numpy((x.float().numpy() - pen).astype(np.float32)).bfloat16()
    want = torch.where(torch.from_numpy(c > 0), z, x)
    assert torch.equal(y.view(torch.int16), want.view(torch.int16))
    y64 = reference_penalized64(x, hist, len(hist), float(p), float(f))
    err = np.abs(y.double().numpy() - y64)
    assert (err <= 2.0 ** -8 * np.abs(y64) + 1e-6).all()  # half a bf16 ulp plus the fp32 steps


def _pen_args(M=3, V=100, cols=6):
    return dict(logits=torch.zeros(M, V, dtype=torch.bfloat16), history=torch.zeros(M, cols, dtype=torch.int64),
                step=torch.zeros(M, dtype=torch.int64), positions=torch.zeros(M, dtype=torch.int32),
                presence=torch.zeros(M), frequency=torch.zeros(M), out=torch.zeros(M, V, dtype=torch.bfloat16))


def test_ops_apply_penalties_rejections():
    a = _pen_args()
    with pytest.raises(ValueError, match="bfloat16"):
        ops.apply_penalties(**{**a, "logits": torch.zeros(3, 100)})
    with pytest.raises(ValueError, match="unit column stride"):
        ops.apply_penalties(**{**a, "logits": torch.zeros(100, 3, dtype=torch.bfloat16).t()})
    with pytest.raises(ValueError, match="V="):
        ops.apply_penalties(**{**a, "logits": torch.zeros(3, 8 * 40960 + 1, dtype=torch.bfloat16)})
    with pytest.raises(ValueError, match="M=0"):
        ops.apply_penalties(**{**a, "logits": torch.zeros(0, 100, dtype=torch.bfloat16)})
    with pytest.raises(ValueError, match="history"):
        ops.apply_penalties(**{**a, "history": torch.zeros(3, 6, dtype=torch.int32)})
    with pytest.raises(ValueError, match="history"):
        ops.apply_penalties(**{**a, "history": torch.zeros(6, 3, dtype=torch.int64).t()})
    with pytest.raises(ValueError, match="history"):
        ops.apply_penalties(**{**a, "history": torch.zeros(3, 0, dtype=torch.int64)})
    with pytest.raises(ValueError, match="int64"):
        ops.apply_penalties(**{**a, "step": torch.zeros(3, dtype=torch.int32)})
    with pytest.raises(ValueError, match=r"\[3\]"):
        ops.apply_penalties(**{**a, "step": torch.zeros(6, dtype=torch.int64)[::2]})
    with pytest.raises(ValueError, match="positions"):
        ops.apply_penalties(**{**a, "positions": torch.zeros(4, dtype=torch.int32)})
    with pytest.raises(ValueError, match="presence"):
        ops.apply_penalties(**{**a, "presence": torch.zeros(3, dtype=torch.float64)})
    with pytest.raises(ValueError, match="frequency"):
        ops.apply_penalties(**{**a, "frequency": torch.zeros(2)})
    with pytest.raises(ValueError, match="out"):
        ops.apply_penalties(**{**a, "out": torch.zeros(3, 101, dtype=torch.bfloat16)})
    with pytest.raises(ValueError, match="out"):
        ops.apply_penalties(**{**a, "out": torch.zeros(3, 100)})
    # a strided row layout is accepted up to the device check
    wide = torch.zeros(3, 128, dtype=torch.bfloat16)[:, :100]
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.apply_penalties(**{**a, "logits": wide})


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_entry_point_fails_loudly_without_gpu():
    from vila_b200 import _lib
    lib = _lib.load()
    assert lib.vila_apply_penalties(None, None) != 0 and b"params are required" in lib.vila_last_error()
    p = _lib.PenaltyParams()
    assert lib.vila_apply_penalties(p, None) != 0 and b"required" in lib.vila_last_error()  # checked before the device
    buf = torch.zeros(64, dtype=torch.int64)
    for name in ("logits", "history", "step", "position", "presence", "frequency", "out"):
        setattr(p, name, buf.data_ptr())
    p.ld, p.M, p.V, p.cols = 8, 2, 8, 4
    assert lib.vila_apply_penalties(p, None) != 0 and b"no CUDA device" in lib.vila_last_error()
    for field, bad, msg in (("M", 0, b"M=0"), ("M", 65536, b"M=65536"), ("V", 0, b"V=0"), ("V", 8 * 40960 + 1, b"V="),
                            ("cols", 0, b"cols=0"), ("ld", 7, b"row stride")):
        good = getattr(p, field)
        setattr(p, field, bad)
        if field == "V" and bad > 8:
            p.ld = bad
        assert lib.vila_apply_penalties(p, None) != 0 and msg in lib.vila_last_error(), field
        setattr(p, field, good)
        p.ld = 8


def test_struct_matches_header_field_order():
    from vila_b200 import _lib
    text = (ROOT / "include" / "vila_b200.h").read_text()
    body = re.search(r"typedef struct vila_penalty_params \{(.*?)\} vila_penalty_params;", text, flags=re.S).group(1)
    fields = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        names = decl.split(",")
        fields.append(names[0].split()[-1].lstrip("*"))
        fields.extend(x.strip().lstrip("*") for x in names[1:])
    assert fields == [f[0] for f in _lib.PenaltyParams._fields_]
    assert fields == ["logits", "ld", "history", "step", "position", "presence", "frequency", "out", "M", "V", "cols"]
    assert "vila_apply_penalties" in _lib.SIGNATURES and hasattr(_lib.load(), "vila_apply_penalties")
    assert "vila_apply_penalties" in (ROOT / "vila_b200" / "csrc" / "api.cu").read_text()
    assert _lib.load().vila_abi_version() == 3  # a new entry point leaves the ABI version as it is


# ------------------------------------------------------------------------------------------------
# engine host logic
# ------------------------------------------------------------------------------------------------
def _duck_llm(L=2, Hq=4, Hkv=2, V=50):
    cfg = SimpleNamespace(num_attention_heads=Hq, num_key_value_heads=Hkv, head_dim=128, num_hidden_layers=L,
                          hidden_size=64, vocab_size=V)
    return SimpleNamespace(config=cfg, device=torch.device("cpu"), dtype=torch.bfloat16)


def test_batched_decoder_penalties_state():
    plain = serving.BatchedDecoder(_duck_llm(), slots=3, max_tokens_per_slot=256, max_new=8)
    pen = serving.BatchedDecoder(_duck_llm(), slots=3, max_tokens_per_slot=256, max_new=8, penalties=True)
    assert not plain.penalties and not hasattr(plain, "pen_logits") and not hasattr(plain, "presence")
    assert pen.pen_logits.shape == (3, 50) and pen.pen_logits.dtype == torch.bfloat16
    assert pen.presence.shape == pen.frequency.shape == (3,) and pen.presence.dtype == torch.float32
    assert pen.launches_per_step == plain.launches_per_step + 1 == 7 * 2 + 3
    every = serving.BatchedDecoder(_duck_llm(), slots=3, max_tokens_per_slot=256, max_new=8, penalties=True,
                                   sampling=True, logprobs=2)
    assert every.launches_per_step == plain.launches_per_step + 3
    emb = torch.zeros(10, 64, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="penalties=True"):
        plain.admit(0, emb, penalties=PenaltyParams(0.5, 0.5))
    with pytest.raises(ValueError, match="PenaltyParams"):
        pen.admit(0, emb, penalties=(0.5, 0.5))
    # a refused admission leaves the running slot's penalties alone
    cached = serving.BatchedDecoder(_duck_llm(), slots=2, max_tokens_per_slot=256, max_new=8, penalties=True,
                                    prefix_cache=True)
    cached._pos_host[0] = 12
    cached.presence[0], cached.frequency[0] = 0.25, -0.5
    with pytest.raises(ValueError, match="still in use"):
        cached.admit(0, emb, penalties=PenaltyParams(1.0, 1.0))
    assert cached.presence[0].item() == 0.25 and cached.frequency[0].item() == -0.5


class _FakePenDecoder:
    """serving.BatchedDecoder's host surface; records the penalties each admission got"""

    def __init__(self, slots=2, penalties=True):
        self.slots, self.pages_per_slot, self.penalties = slots, 8, penalties
        self.allocator = serving.PageAllocator(64)
        self.state = [None] * slots
        self.admitted = []

    def capture(self):
        pass

    def admit(self, s, emb, params=None, **kw):
        self.admitted.append((emb.shape[0], kw))
        self.state[s] = [emb.shape[0]]

    def run(self, n):
        for st in self.state:
            if st is not None:
                st.extend(st[-1] + 1 + i for i in range(n))

    def generated(self, s):
        return list(self.state[s])

    def release(self, s):
        self.state[s] = None


def test_generate_batch_penalties_host_logic():
    prompts = [torch.zeros(n, 4) for n in (10, 20, 30)]
    dec = _FakePenDecoder()
    plain = serving.generate_batch(None, prompts, max_new_tokens=5, slots=2, check_every=4, decoder=dec)
    assert all(kw == {} for _, kw in dec.admitted)  # no penalties asked for: admit() gets no keyword
    a, b = PenaltyParams(0.5, 0.0), PenaltyParams(0.0, 1.0)
    dec = _FakePenDecoder()
    ids = serving.generate_batch(None, prompts, max_new_tokens=5, slots=2, check_every=4, decoder=dec,
                                 penalties=[a, None, b])
    assert ids == plain and sorted((n, kw["penalties"]) for n, kw in dec.admitted) == [(10, a), (20, None), (30, b)]
    dec = _FakePenDecoder()
    serving.generate_batch(None, prompts, max_new_tokens=5, slots=2, check_every=4, decoder=dec, penalties=a)
    assert [kw["penalties"] for _, kw in dec.admitted] == [a, a, a]
    for bad in ([a, b], [a, b, a, b], [a, (0.5, 0.5), b], 0.5):
        with pytest.raises(ValueError, match="one per request"):
            serving.generate_batch(None, prompts, max_new_tokens=5, decoder=_FakePenDecoder(), penalties=bad)
    with pytest.raises(ValueError, match="penalties=False"):
        serving.generate_batch(None, prompts, max_new_tokens=5, decoder=_FakePenDecoder(penalties=False), penalties=a)
    real = serving.BatchedDecoder(_duck_llm(), slots=1, max_tokens_per_slot=256, max_new=8)
    with pytest.raises(ValueError, match="penalties=False"):
        serving.generate_batch(_duck_llm(), prompts, max_new_tokens=4, decoder=real, penalties=[None, None, None])


def test_llava_generate_batch_passes_penalties_through():
    from vila_b200.model.llava_llama import LlavaLlamaModel
    sig = inspect.signature(LlavaLlamaModel.generate_batch)
    assert sig.parameters["penalties"].default is None
    src = inspect.getsource(LlavaLlamaModel.generate_batch)
    assert "penalties=penalties" in src and "key += (penalties is not None,)" in src  # the kept engine's key
    assert "sampling is not None, logprobs)" in src and "sampling=sampling" in src and "prefix_cache=prefix_cache" in src


# ------------------------------------------------------------------------------------------------
# server
# ------------------------------------------------------------------------------------------------
def _server_stub(calls):
    class Tok:
        stop_token_ids = [9]

        def decode(self, ids, skip_special_tokens=True):
            return " ".join(f"t{i}" for i in ids)

    class Stub:
        tokenizer = Tok()
        default_generation_config = SimpleNamespace(max_new_tokens=None)

        def generate_content(self, prompt, generation_config=None, response_format=None, stream=False):
            calls["single"] += 1
            return iter(["a", "b"]) if stream else "single"

        def _prepare_content(self, prompt):
            return torch.tensor([[1, 2]]), None, {}

        def generate_batch(self, requests, max_new_tokens=128, slots=8, **kw):
            calls["batch"].append((len(requests), kw))
            return [[7, 8, 9] for _ in requests]

    return Stub()


def _req(**kw):
    from vila_b200 import server as S
    return S.ChatCompletionRequest(model="m", max_tokens=kw.pop("max_tokens", 5),
                                   messages=[S.ChatMessage(role="user", content="hi")], **kw)


def test_server_penalty_validation_before_batching():
    from vila_b200 import server as S
    assert S.ChatCompletionRequest.model_fields["presence_penalty"].default == 0.0
    assert S.ChatCompletionRequest.model_fields["frequency_penalty"].default == 0.0
    calls = {"batch": [], "single": 0}
    eng = S.Engine(_server_stub(calls), "m", slots=4)
    for bad in (dict(presence_penalty=2.5), dict(frequency_penalty=-3.0), dict(frequency_penalty=math.nan),
                dict(presence_penalty=math.inf)):
        with pytest.raises(ValueError, match=r"\[-2, 2\]"):
            asyncio.run(eng.complete(_req(**bad)))
    assert calls == {"batch": [], "single": 0}  # refused before joining a batch
    no_batch = _server_stub(calls)
    del type(no_batch).generate_batch
    with pytest.raises(ValueError, match="generate_batch"):
        asyncio.run(S.Engine(no_batch, "m").complete(_req(presence_penalty=0.5)))


def test_server_routes_a_lone_penalised_request_to_the_engine():
    from vila_b200 import server as S
    calls = {"batch": [], "single": 0}
    eng = S.Engine(_server_stub(calls), "m", slots=4)
    res = asyncio.run(eng.complete(_req(presence_penalty=0.5, frequency_penalty=None)))
    assert calls["single"] == 0 and calls["batch"] == [(1, {"penalties": [PenaltyParams(0.5, 0.0)]})]
    assert res["choices"][0]["message"]["content"] == "t7 t8 t9" and "logprobs" not in res["choices"][0]
    calls["batch"].clear()

    async def mixed():
        return await asyncio.gather(eng.complete(_req(frequency_penalty=1.0)), eng.complete(_req()),
                                    eng.complete(_req(presence_penalty=-0.5, frequency_penalty=0.25)))

    asyncio.run(mixed())
    got = [p for n, kw in calls["batch"] for p in kw.get("penalties", [None] * n)]
    assert sorted(map(repr, got)) == sorted(map(repr, [PenaltyParams(0.0, 1.0), None, PenaltyParams(-0.5, 0.25)]))
    # with --sample the penalties go along with the sampling parameters
    calls = {"batch": [], "single": 0}
    asyncio.run(S.Engine(_server_stub(calls), "m", slots=4, sample=True).complete(_req(seed=1, presence_penalty=1)))
    assert calls["batch"][0][1]["penalties"] == [PenaltyParams(1.0, 0.0)] and "sampling" in calls["batch"][0][1]


def test_server_passes_no_penalties_keyword_when_nobody_asked():
    from vila_b200 import server as S
    calls = {"batch": [], "single": 0}
    eng = S.Engine(_server_stub(calls), "m", slots=4)
    lone = asyncio.run(eng.complete(_req(presence_penalty=0.0, frequency_penalty=None)))
    assert calls == {"batch": [], "single": 1} and lone["choices"][0]["message"]["content"] == "single"

    async def default():
        return await asyncio.gather(*[eng.complete(_req(presence_penalty=0)) for _ in range(3)])

    res = asyncio.run(default())
    assert calls["batch"] and all("penalties" not in kw for _, kw in calls["batch"])
    assert all(set(r["choices"][0]) == {"message"} for r in res)  # the response shape is as before
    assert all(r["choices"][0]["message"]["content"] in ("single", "t7 t8 t9") for r in res)


def test_server_refuses_penalties_when_streaming():
    from vila_b200 import server as S
    calls = {"batch": [], "single": 0}
    eng = S.Engine(_server_stub(calls), "m", slots=4)
    with pytest.raises(ValueError, match="single-stream"):
        eng._stream_config(_req(stream=True, frequency_penalty=0.5))

    async def streamed():
        return [c async for c in eng.stream(_req(stream=True, presence_penalty=-1.0))]

    with pytest.raises(ValueError, match="stream"):
        asyncio.run(streamed())
    assert calls["single"] == 0
    eng._stream_config(_req(stream=True, presence_penalty=0.0))  # zero penalties stream as before
