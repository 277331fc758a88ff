"""CPU: sampling in the continuous-batching engine without a device: Philox-4x32-10 against the Random123
known-answer vectors, the rule of vila_b200/sampling.py on hand-made rows (ties at the k-th value, a top-p boundary
just below and just above, top_k >= V, top_p = 1, tiny temperatures, the greedy equivalence of T = 0 and top_k = 1,
HF's warpers on distinct values), SamplingParams validation, the argument errors of ops.sample_batch, the loud failure
of the entry point, the struct's field order against the header, generate_batch's host logic (per-request
parameters, seed derivation, refusal of a greedy decoder) and the server's --sample plumbing."""
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
from vila_b200.sampling import (SamplingParams, gumbel_noise, kept_set, philox4x32_10, philox_words, reference_draw,
                                scaled, seed_words, signed64)

ROOT = Path(__file__).resolve().parent.parent


def _hex(words):
    return [f"{int(w):08x}" for w in words]


def test_philox_known_answers():
    assert _hex(philox4x32_10([0, 0, 0, 0], (0, 0))) == ["6627e8d5", "e169c58d", "bc57ac4c", "9b00dbd8"]
    ones = 0xFFFFFFFF
    assert _hex(philox4x32_10([ones] * 4, (ones, ones))) == ["408f276d", "41c83b0e", "a20bc7c6", "6d5451fd"]
    assert _hex(philox4x32_10([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], (0xA4093822, 0x299F31D0))) == [
        "d16cfe09", "94fdcceb", "5001e420", "24126ea1"]


def test_philox_words_layout():
    """x_i is word i % 4 of the block with counter (i // 4, t lo, t hi, 0); a prefix does not depend on V"""
    seed, t = 0x0123456789ABCDEF, (5 << 32) + 17
    x = philox_words(seed, t, 11)
    k = seed_words(seed)
    assert k == (0x89ABCDEF, 0x01234567)
    for blk in range(3):
        want = philox4x32_10([blk, 17, 5, 0], k)
        n = min(4, 11 - 4 * blk)
        assert list(x[4 * blk:4 * blk + n]) == list(want[:n])
    assert np.array_equal(gumbel_noise(seed, t, 1000)[:11], gumbel_noise(seed, t, 11))
    assert signed64(2 ** 64 - 1) == -1 and seed_words(-1) == (0xFFFFFFFF, 0xFFFFFFFF)


def test_gumbel_noise_is_finite_and_standard():
    g = gumbel_noise(1234, 0, 200_000)
    assert np.isfinite(g).all()
    assert abs(g.mean() - 0.5772156649) < 0.01 and abs(g.var() - math.pi ** 2 / 6) < 0.03


def test_topk_keeps_ties_at_the_kth_value():
    s = np.float32([3, 1, 2, 2, 0, 2, -1])
    keep, margin = kept_set(s, 2, 1.0)
    assert keep.tolist() == [True, False, True, True, False, True, False] and margin == math.inf
    assert kept_set(s, 1, 1.0)[0].sum() == 1


def test_topk_at_or_above_vocab_and_topp_one_are_off():
    s = np.float32(np.random.RandomState(0).randn(50))
    for k in (0, 50, 51, 10_000):
        assert kept_set(s, k, 1.0)[0].all()


def _boundary(s, i):
    """mass strictly above s[i] over Z, in fp64 as the rule computes it"""
    sd = s.astype(np.float64)
    p = np.exp(sd - sd.max())
    return p[sd > sd[i]].sum() / p.sum()


def test_topp_boundary_just_below_and_just_above():
    s = np.float32([2.0, 1.0, 0.0, -1.0, -3.0])
    b = _boundary(s, 2)  # value 0 is kept iff top_p > b
    above, m_above = kept_set(s, 0, b * (1 + 1e-6))
    below, m_below = kept_set(s, 0, b * (1 - 1e-6))
    assert above.tolist() == [True, True, True, False, False]
    assert below.tolist() == [True, True, False, False, False]
    assert m_above == pytest.approx(b * 1e-6, rel=1e-3) and m_below == pytest.approx(b * 1e-6, rel=1e-3)
    exact, _ = kept_set(s, 0, b)  # mass above == top_p * Z: dropped (strictly less is required)
    assert exact.tolist() == [True, True, False, False, False]


def test_topp_keeps_boundary_ties_and_the_largest():
    s = np.float32([1.0, 0.0, 0.0, -1.0])
    keep, _ = kept_set(s, 0, _boundary(s, 1) * 1.01)
    assert keep.tolist() == [True, True, True, False]
    assert kept_set(s, 0, 1e-9)[0].tolist() == [True, False, False, False]
    tie_top = np.float32([4.0, 4.0, 1.0])
    assert kept_set(tie_top, 0, 1e-9)[0].tolist() == [True, True, False]


def test_topk_then_topp_renormalises_over_the_survivors():
    s = np.float32([3.0, 2.0, 1.0, 0.0, -1.0])
    # over the top-3 survivors, value 1 has mass above (e^0 + e^-1) / Z3
    p = np.exp(s.astype(np.float64) - 3)
    b3 = (p[0] + p[1]) / p[:3].sum()
    assert kept_set(s, 3, b3 * (1 + 1e-6))[0].tolist() == [True, True, True, False, False]
    assert kept_set(s, 3, b3 * (1 - 1e-6))[0].tolist() == [True, True, False, False, False]


def _hf_top_p(scores: torch.Tensor, top_p: float) -> torch.Tensor:
    """HF TopPLogitsWarper's kept mask (sort ascending, remove cumulative probability <= 1 - top_p, keep the top)"""
    sorted_logits, sorted_idx = torch.sort(scores, descending=False)
    cum = sorted_logits.softmax(-1).cumsum(-1)
    remove = cum <= (1 - top_p)
    remove[-1] = False
    return ~remove.scatter(0, sorted_idx, remove)


def test_topp_matches_hf_on_distinct_values():
    rs = np.random.RandomState(3)
    checked = 0
    for trial in range(200):
        x = torch.from_numpy(rs.randn(300) * rs.uniform(0.5, 4)).double()
        s = scaled(x.float(), 1.0)
        top_p = float(rs.uniform(0.05, 0.99))
        keep, margin = kept_set(s, 0, top_p)
        if margin < 1e-9:
            continue
        assert keep.tolist() == _hf_top_p(torch.from_numpy(s.astype(np.float64)), top_p).tolist(), trial
        checked += 1
    assert checked >= 190


def test_greedy_equivalence_and_tiny_temperature():
    rs = np.random.RandomState(7)
    x = torch.from_numpy(rs.randn(1000)).bfloat16()
    x[17] = x[511] = x.float().max() + 1  # a tie at the maximum: the first index wins
    want = int(torch.argmax(x.float()))
    assert want == 17
    for inv_t, k in ((0.0, 0), (0.0, 50), (2.0, 1), (0.5, 1)):
        tok, keep, v, margin = reference_draw(x, inv_t, k, 0.9, seed=5, t=3)
        assert tok == want and keep.sum() == 1 and v is None
    y = torch.from_numpy(rs.randn(1000)).bfloat16()
    inv = float(np.float32(1 / 1e-4))
    for seed in range(20):  # T = 1e-4: the maximum carries all the mass
        tok, keep, _, _ = reference_draw(y, inv, 0, 0.9, seed=seed, t=seed)
        assert tok == int(torch.argmax(y.float())) and keep.sum() == 1


def test_scaling_is_fp32_and_canonicalises_negative_zero():
    x = torch.tensor([-0.0, 1.5, -2.25, 3.0], dtype=torch.bfloat16)
    s = scaled(x, float(np.float32(1 / 0.7)))
    assert s.dtype == np.float32 and np.signbit(s[0]) == False  # noqa: E712
    assert s[1] == np.float32(1.5) * np.float32(1 / 0.7)


def test_sampling_params_validation():
    for bad in (dict(temperature=-0.1), dict(temperature=float("nan")), dict(temperature=float("inf")),
                dict(top_p=0.0), dict(top_p=1.5), dict(top_p=-0.2), dict(top_k=-1), dict(top_k=2.5),
                dict(seed=2 ** 64)):
        with pytest.raises(ValueError):
            SamplingParams(**bad)
    p = SamplingParams(temperature=0.7, top_k=50, top_p=0.9, seed=3)
    assert not p.greedy and p.inv_temperature == float(np.float32(1 / 0.7))
    assert SamplingParams().greedy and SamplingParams(temperature=1.0, top_k=1).greedy
    assert SamplingParams().inv_temperature == 0.0 and SamplingParams(temperature=2.0, top_k=1).inv_temperature == 0.0
    assert serving.SamplingParams is SamplingParams


def _sample_args(M=3, V=100, dev="cpu"):
    return dict(logits=torch.zeros(M, V, dtype=torch.bfloat16, device=dev),
                inv_temperature=torch.zeros(M, device=dev), top_k=torch.zeros(M, dtype=torch.int32, device=dev),
                top_p=torch.ones(M, device=dev), seed=torch.zeros(M, dtype=torch.int64, device=dev),
                step=torch.zeros(M, dtype=torch.int64, device=dev), positions=torch.zeros(M, dtype=torch.int32, device=dev),
                out=torch.zeros(M, dtype=torch.int64, device=dev))


def test_ops_sample_batch_rejections():
    a = _sample_args()
    with pytest.raises(ValueError, match="bfloat16"):
        ops.sample_batch(**{**a, "logits": torch.zeros(3, 100)})
    with pytest.raises(ValueError, match="unit column stride"):
        ops.sample_batch(**{**a, "logits": torch.zeros(100, 3, dtype=torch.bfloat16).t()})
    with pytest.raises(ValueError):
        ops.sample_batch(**{**a, "logits": torch.zeros(3, 8 * 40960 + 1, dtype=torch.bfloat16)})
    with pytest.raises(ValueError, match="int32"):
        ops.sample_batch(**{**a, "top_k": torch.zeros(3, dtype=torch.int64)})
    with pytest.raises(ValueError, match="int64"):
        ops.sample_batch(**{**a, "seed": torch.zeros(3, dtype=torch.int32)})
    with pytest.raises(ValueError, match=r"\[3\]"):
        ops.sample_batch(**{**a, "top_p": torch.ones(4)})
    with pytest.raises(ValueError, match=r"\[3\]"):
        ops.sample_batch(**{**a, "step": torch.zeros(6, dtype=torch.int64)[::2]})
    with pytest.raises(ValueError, match="n_kept"):
        ops.sample_batch(**a, n_kept=torch.zeros(3, dtype=torch.int64))
    # a strided row layout (the engine's logits of a wider buffer) is accepted up to the device check
    wide = torch.zeros(3, 128, dtype=torch.bfloat16)[:, :100]
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.sample_batch(**{**a, "logits": wide})


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_entry_point_fails_loudly_without_gpu():
    from vila_b200 import _lib
    lib = _lib.load()
    p = _lib.SampleParams()
    for arg in (None, p):
        rc = lib.vila_sample_batch(arg, None)
        assert rc != 0 and b"no CUDA device" in lib.vila_last_error()


def test_struct_matches_header_field_order():
    from vila_b200 import _lib
    text = (ROOT / "include" / "vila_b200.h").read_text()
    body = re.search(r"typedef struct vila_sample_params \{(.*?)\} vila_sample_params;", text, flags=re.S).group(1)
    fields = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        names = decl.split(",")
        fields.append(names[0].split()[-1].lstrip("*"))
        fields.extend(x.strip().lstrip("*") for x in names[1:])
    assert fields == [f[0] for f in _lib.SampleParams._fields_]
    assert fields == ["logits", "ld", "inv_temperature", "top_k", "top_p", "seed", "step", "position", "tokens",
                      "n_kept", "M", "V"]
    assert "vila_sample_batch" in _lib.SIGNATURES and hasattr(_lib.load(), "vila_sample_batch")
    assert "vila_sample_batch" in (ROOT / "vila_b200" / "csrc" / "api.cu").read_text()


# ------------------------------------------------------------------------------------------------
# engine host logic
# ------------------------------------------------------------------------------------------------
def _duck_llm(L=2, Hq=4, Hkv=2):
    cfg = SimpleNamespace(num_attention_heads=Hq, num_key_value_heads=Hkv, head_dim=128, num_hidden_layers=L,
                          hidden_size=64)
    return SimpleNamespace(config=cfg, device=torch.device("cpu"), dtype=torch.bfloat16)


def test_batched_decoder_sampling_state():
    greedy = serving.BatchedDecoder(_duck_llm(), slots=3, max_tokens_per_slot=256, max_new=8)
    samp = serving.BatchedDecoder(_duck_llm(), slots=3, max_tokens_per_slot=256, max_new=8, sampling=True)
    assert not greedy.sampling and not hasattr(greedy, "inv_temperature")
    assert samp.sampling
    for name, dt, val in (("inv_temperature", torch.float32, 0), ("top_k", torch.int32, 0),
                          ("top_p", torch.float32, 1), ("seed", torch.int64, 0)):
        t = getattr(samp, name)
        assert t.dtype == dt and t.shape == (3,) and bool((t == val).all())
    assert samp.launches_per_step == greedy.launches_per_step + 1 == 7 * 2 + 3
    with pytest.raises(ValueError, match="sampling=True"):
        greedy.admit(0, torch.zeros(4, 64), SamplingParams(temperature=1.0, seed=1))
    with pytest.raises(ValueError, match="seed"):
        samp.admit(0, torch.zeros(4, 64), SamplingParams(temperature=1.0))


class _FakeSamplingDecoder:
    """serving.BatchedDecoder's host surface; request r emits its prompt length S, then S + 1, ..."""

    def __init__(self, slots=2, sampling=True):
        self.slots, self.pages_per_slot, self.sampling = slots, 8, sampling
        self.allocator = serving.PageAllocator(64)
        self.state = [None] * slots
        self.admitted = []

    def capture(self):
        pass

    def admit(self, s, emb, params=None):
        self.state[s] = [emb.shape[0]]
        self.admitted.append((emb.shape[0], params))

    def run(self, n):
        for st in self.state:
            if st is not None:
                last = st[-1]
                st.extend(last + 1 + i for i in range(n))

    def generated(self, s):
        return list(self.state[s])

    def release(self, s):
        self.state[s] = None


def test_generate_batch_sampling_host_logic():
    prompts = [torch.zeros(n, 4) for n in (10, 20, 30)]
    per = [SamplingParams(0.7, 0, 0.9, seed=11), SamplingParams(), SamplingParams(1.3, 40, 1.0, seed=None)]
    dec = _FakeSamplingDecoder()
    out = serving.generate_batch(None, prompts, max_new_tokens=5, slots=2, check_every=4, decoder=dec, sampling=per)
    assert out == [list(range(n, n + 5)) for n in (10, 20, 30)]
    got = {S: p for S, p in dec.admitted}
    assert got[10] == per[0] and got[20].greedy and got[20].seed is not None
    assert (got[30].temperature, got[30].top_k, got[30].top_p) == (1.3, 40, 1.0) and got[30].seed is not None
    # seeds left None come from the host default generator, in request order
    torch.manual_seed(1234)
    a = serving.sampling_for_requests(SamplingParams(temperature=1.0), 4)
    torch.manual_seed(1234)
    b = serving.sampling_for_requests([SamplingParams(temperature=1.0)] * 4, 4)
    assert [p.seed for p in a] == [p.seed for p in b] and len({p.seed for p in a}) == 4
    torch.manual_seed(1234)
    first = int(torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64))
    assert a[0].seed == first
    assert serving.sampling_for_requests(None, 3) is None
    with pytest.raises(ValueError, match="one per request"):
        serving.sampling_for_requests([SamplingParams()] * 2, 3)


def test_generate_batch_refuses_a_greedy_decoder_for_sampling():
    prompts = [torch.zeros(10, 4)]
    with pytest.raises(ValueError, match="sampling=False"):
        serving.generate_batch(None, prompts, max_new_tokens=4, decoder=_FakeSamplingDecoder(sampling=False),
                               sampling=SamplingParams(temperature=1.0, seed=0))
    real = serving.BatchedDecoder(_duck_llm(), slots=1, max_tokens_per_slot=256, max_new=8)
    with pytest.raises(ValueError, match="sampling=False"):
        serving.generate_batch(_duck_llm(), prompts, max_new_tokens=4, decoder=real, sampling=SamplingParams())
    # greedy generate_batch calls admit(slot, prompt) exactly as before
    dec = _FakeSamplingDecoder(sampling=False)
    serving.generate_batch(None, prompts, max_new_tokens=4, decoder=dec)
    assert dec.admitted == [(10, None)]


def test_llava_generate_batch_passes_sampling_through():
    from vila_b200.model.llava_llama import LlavaLlamaModel
    sig = inspect.signature(LlavaLlamaModel.generate_batch)
    assert sig.parameters["sampling"].default is None
    assert "sampling=sampling" in inspect.getsource(LlavaLlamaModel.generate_batch)


def _server_stub(calls):
    class Tok:
        def decode(self, ids, skip_special_tokens=True):
            return " ".join(str(i) for i in ids)

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


def test_server_sample_flag():
    from vila_b200 import server as S

    def req(**kw):
        return S.ChatCompletionRequest(model="m", max_tokens=2, messages=[S.ChatMessage(role="user", content="hi")],
                                       **kw)

    calls = {"batch": [], "single": 0}
    eng = S.Engine(_server_stub(calls), "m", slots=4, sample=True)

    async def scenario():
        lone = await eng.complete(req(temperature=0.7, top_p=0.8, seed=42))
        many = await asyncio.gather(eng.complete(req()), eng.complete(req(temperature=0.0, seed=5)),
                                    eng.complete(req(temperature=1.1, top_p=None)))
        chunks = [c async for c in eng.stream(req(stream=True, temperature=0.9))]
        return lone, many, chunks

    lone, many, chunks = asyncio.run(scenario())
    assert lone["choices"][0]["message"]["content"] == "7 8"
    assert calls["single"] == 1  # only the streaming request took the single-stream path
    assert len(chunks) == 3
    n0, kw0 = calls["batch"][0]
    assert n0 == 1 and kw0["sampling"] == [SamplingParams(0.7, 0, 0.8, 42)]  # a lone request is sampled too
    sent = [p for _, kw in calls["batch"][1:] for p in kw["sampling"]]
    assert (sent[0].temperature, sent[0].top_p, sent[0].seed) == (0.2, 0.9, None)  # the request's defaults
    assert sent[1].greedy and sent[1].seed == 5
    assert (sent[2].temperature, sent[2].top_p) == (1.1, 1.0)
    # bad parameters answer the request with an error instead of decoding it greedily
    with pytest.raises(ValueError):
        asyncio.run(S.Engine(_server_stub(calls), "m", sample=True).complete(req(top_p=0.0)))
    # ... and only that request: the good ones gathered with it are still served, in one batch
    calls["batch"].clear()
    eng = S.Engine(_server_stub(calls), "m", slots=8, sample=True)

    async def mixed():
        return await asyncio.gather(eng.complete(req(seed=1)), eng.complete(req(seed=2)),
                                    eng.complete(req(top_p=0.0)), eng.complete(req(temperature=-1.0)),
                                    eng.complete(req(seed=2 ** 64)), eng.complete(req(seed=3)),
                                    return_exceptions=True)

    res = asyncio.run(mixed())
    assert [type(r) for r in res[2:5]] == [ValueError] * 3
    assert [r["choices"][0]["message"]["content"] for r in res[:2] + res[5:]] == ["7 8"] * 3
    assert sorted(p.seed for _, kw in calls["batch"] for p in kw["sampling"]) == [1, 2, 3]
    # a model without the batched engine cannot sample
    no_batch = _server_stub(calls)
    del type(no_batch).generate_batch  # each _server_stub call defines its own class
    with pytest.raises(ValueError, match="generate_batch"):
        S.Engine(no_batch, "m", sample=True)
    S.Engine(no_batch, "m")  # greedy serving still falls back to generate_content
    # off by default: no new keyword reaches generate_batch
    calls = {"batch": [], "single": 0}
    eng = S.Engine(_server_stub(calls), "m", slots=4)

    async def default():
        return await asyncio.gather(*[eng.complete(req(temperature=0.9)) for _ in range(3)])

    asyncio.run(default())
    assert calls["single"] == 1 and [kw for _, kw in calls["batch"]] == [{}]
    assert "--sample" in inspect.getsource(S.main) and "greedy" in inspect.getsource(S.main)
    assert "seed" in S.ChatCompletionRequest.model_fields
