"""CPU: per-token logprobs of the continuous-batching engine without a device: the numpy rule of
vila_b200/logprobs.py against torch.log_softmax in fp64 (tied maxima, ties across the n-th place, a V that is not a
multiple of the cluster width, large logit ranges), the argument errors of ops.token_logprobs, the struct's field order
against the header, the loud failure of the entry point, generate_batch's host logic on a duck decoder (return shape,
truncation at EOS and at the budget, the decoder-mismatch ValueError) and the server's logprobs plumbing on a stub
model (validation, routing, per-request trimming, the OpenAI response shape, the streaming refusal, no keyword when
nobody asked)."""
import asyncio
import inspect
import re
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from vila_b200 import ops, serving
from vila_b200.logprobs import MAX_TOP_LOGPROBS, TokenLogprob, check_top, reference_logprobs

ROOT = Path(__file__).resolve().parent.parent


def _log_softmax64(x):
    return torch.log_softmax(torch.as_tensor(x).float().double(), dim=-1).numpy()


@pytest.mark.parametrize("V,scale", [(1003, 1.0), (152064, 4.0), (37, 300.0), (8 * 19008 + 5, 0.01)])
def test_rule_matches_log_softmax(V, scale):
    g = torch.Generator().manual_seed(V)
    x = (torch.randn(V, generator=g) * scale).bfloat16()
    ref = _log_softmax64(x)
    for t in (0, V // 2, V - 1):
        for n in (0, 1, 5, MAX_TOP_LOGPROBS):
            lp, ids, vals = reference_logprobs(x, t, n)
            assert abs(lp - ref[t]) <= 1e-12 * max(1.0, abs(ref[t]))
            assert ids.shape == (n,) and vals.shape == (n,)
            order = np.argsort(-ref, kind="stable")[:n]
            assert ids.tolist() == order.tolist()
            assert np.allclose(vals, ref[order], rtol=0, atol=1e-12 * max(1.0, np.abs(ref).max()))


def test_rule_ties_go_to_the_lower_index():
    x = torch.tensor([1.0, 3.0, 2.0, 3.0, 2.0, 2.0, -1.0, 3.0], dtype=torch.bfloat16)
    _, ids, vals = reference_logprobs(x, 3, 5)
    assert ids.tolist() == [1, 3, 7, 2, 4]  # tied maxima in index order; the 2.0 tie is cut at the 5th place
    assert vals[0] == vals[1] == vals[2]
    lp, _, _ = reference_logprobs(x, 7, 0)
    assert lp == vals[2]
    # -0 and +0 are one value: index order
    z = torch.tensor([-0.0, 0.0, -5.0], dtype=torch.bfloat16)
    assert reference_logprobs(z, 0, 2)[1].tolist() == [0, 1]


def test_rule_large_ranges_stay_finite():
    x = torch.tensor([3e38, -3e38, 0.0, 1e4, 1e4 - 64], dtype=torch.float32).bfloat16()
    lp, ids, vals = reference_logprobs(x, 1, 5)
    assert ids[0] == 0 and vals[0] == 0.0 and np.isfinite(vals).all() and np.isfinite(lp)
    assert lp == pytest.approx(float(x[1].float()) - float(x[0].float()), rel=1e-12)


def test_check_top():
    for good in (0, 1, 20):
        assert check_top(good) == good
    for bad in (-1, 21, 2.0, True, "3", None):
        with pytest.raises(ValueError, match="0..20"):
            check_top(bad)


def _lp_args(M=3, V=100, cols=6, n=4):
    return dict(logits=torch.zeros(M, V, dtype=torch.bfloat16), tokens=torch.zeros(M, dtype=torch.int64),
                step=torch.zeros(M, dtype=torch.int64), positions=torch.zeros(M, dtype=torch.int32),
                lp_hist=torch.zeros(M, cols), top_ids=torch.zeros(M, cols, n, dtype=torch.int32),
                top_lp=torch.zeros(M, cols, n))


def test_ops_token_logprobs_rejections():
    a = _lp_args()
    with pytest.raises(ValueError, match="bfloat16"):
        ops.token_logprobs(**{**a, "logits": torch.zeros(3, 100)})
    with pytest.raises(ValueError, match="unit column stride"):
        ops.token_logprobs(**{**a, "logits": torch.zeros(100, 3, dtype=torch.bfloat16).t()})
    with pytest.raises(ValueError, match="V="):
        ops.token_logprobs(**{**a, "logits": torch.zeros(3, 8 * 40960 + 1, dtype=torch.bfloat16)})
    with pytest.raises(ValueError, match="int64"):
        ops.token_logprobs(**{**a, "tokens": torch.zeros(3, dtype=torch.int32)})
    with pytest.raises(ValueError, match=r"\[3\]"):
        ops.token_logprobs(**{**a, "step": torch.zeros(6, dtype=torch.int64)[::2]})
    with pytest.raises(ValueError, match="positions"):
        ops.token_logprobs(**{**a, "positions": torch.zeros(4, dtype=torch.int32)})
    with pytest.raises(ValueError, match="lp_hist"):
        ops.token_logprobs(**{**a, "lp_hist": torch.zeros(3, 6, dtype=torch.float64)})
    with pytest.raises(ValueError, match="lp_hist"):
        ops.token_logprobs(**{**a, "lp_hist": torch.zeros(6, 3).t()})
    with pytest.raises(ValueError, match="go together"):
        ops.token_logprobs(**{**a, "top_lp": None})
    with pytest.raises(ValueError, match="top_ids"):
        ops.token_logprobs(**{**a, "top_ids": torch.zeros(3, 5, 4, dtype=torch.int32)})
    with pytest.raises(ValueError, match="int32"):
        ops.token_logprobs(**{**a, "top_ids": torch.zeros(3, 6, 4, dtype=torch.int64)})
    with pytest.raises(ValueError, match="n=21"):
        ops.token_logprobs(**{**a, "top_ids": torch.zeros(3, 6, 21, dtype=torch.int32),
                              "top_lp": torch.zeros(3, 6, 21)})
    with pytest.raises(ValueError, match="n=8"):
        ops.token_logprobs(**{**a, "logits": torch.zeros(3, 5, dtype=torch.bfloat16),
                              "top_ids": torch.zeros(3, 6, 8, dtype=torch.int32), "top_lp": torch.zeros(3, 6, 8)})
    # a strided row layout and n = 0 are accepted up to the device check
    wide = torch.zeros(3, 128, dtype=torch.bfloat16)[:, :100]
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.token_logprobs(**{**a, "logits": wide})
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.token_logprobs(**{**a, "top_ids": None, "top_lp": None})


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_entry_point_fails_loudly_without_gpu():
    from vila_b200 import _lib
    lib = _lib.load()
    assert lib.vila_token_logprobs(None, None) != 0 and b"params are required" in lib.vila_last_error()
    p = _lib.LogprobsParams()
    assert lib.vila_token_logprobs(p, None) != 0 and b"required" in lib.vila_last_error()  # checked before the device
    buf = torch.zeros(64, dtype=torch.int64)
    for name in ("logits", "tokens", "step", "position", "lp_hist"):
        setattr(p, name, buf.data_ptr())
    p.ld, p.M, p.V, p.cols, p.n = 8, 2, 8, 4, 0
    assert lib.vila_token_logprobs(p, None) != 0 and b"no CUDA device" in lib.vila_last_error()
    p.n = 21
    assert lib.vila_token_logprobs(p, None) != 0 and b"n=21" in lib.vila_last_error()


def test_struct_matches_header_field_order():
    from vila_b200 import _lib
    text = (ROOT / "include" / "vila_b200.h").read_text()
    body = re.search(r"typedef struct vila_logprobs_params \{(.*?)\} vila_logprobs_params;", text, flags=re.S).group(1)
    fields = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        names = decl.split(",")
        fields.append(names[0].split()[-1].lstrip("*"))
        fields.extend(x.strip().lstrip("*") for x in names[1:])
    assert fields == [f[0] for f in _lib.LogprobsParams._fields_]
    assert fields == ["logits", "ld", "tokens", "step", "position", "lp_hist", "top_ids", "top_lp", "M", "V", "cols",
                      "n"]
    assert "vila_token_logprobs" in _lib.SIGNATURES and hasattr(_lib.load(), "vila_token_logprobs")
    assert "vila_token_logprobs" in (ROOT / "vila_b200" / "csrc" / "api.cu").read_text()
    assert _lib.load().vila_abi_version() == 3  # a new entry point leaves the ABI version as it is


# ------------------------------------------------------------------------------------------------
# engine host logic
# ------------------------------------------------------------------------------------------------
def _duck_llm(L=2, Hq=4, Hkv=2):
    cfg = SimpleNamespace(num_attention_heads=Hq, num_key_value_heads=Hkv, head_dim=128, num_hidden_layers=L,
                          hidden_size=64)
    return SimpleNamespace(config=cfg, device=torch.device("cpu"), dtype=torch.bfloat16)


def test_batched_decoder_logprobs_state():
    plain = serving.BatchedDecoder(_duck_llm(), slots=3, max_tokens_per_slot=256, max_new=8)
    lp = serving.BatchedDecoder(_duck_llm(), slots=3, max_tokens_per_slot=256, max_new=8, logprobs=5)
    assert plain.logprobs is None and not hasattr(plain, "lp_hist") and not hasattr(plain, "_zero_step")
    assert lp.lp_hist.shape == (3, 16) and lp.lp_hist.dtype == torch.float32
    assert lp.top_ids.shape == (3, 16, 5) and lp.top_ids.dtype == torch.int32 and lp.top_lp.shape == (3, 16, 5)
    assert lp.launches_per_step == plain.launches_per_step + 1 == 7 * 2 + 3
    both = serving.BatchedDecoder(_duck_llm(), slots=3, max_tokens_per_slot=256, max_new=8, logprobs=0, sampling=True)
    assert both.launches_per_step == plain.launches_per_step + 2 and both.top_ids.shape == (3, 16, 0)
    with pytest.raises(ValueError, match="0..20"):
        serving.BatchedDecoder(_duck_llm(), slots=1, max_tokens_per_slot=256, max_new=8, logprobs=21)
    with pytest.raises(ValueError, match="logprobs=n"):
        plain.generated_logprobs(0)
    # generated_logprobs reads the history buffers up to step_idx
    lp.hist[1, :3] = torch.tensor([7, 8, 9])
    lp.lp_hist[1, :3] = torch.tensor([-0.5, -1.0, -2.0])
    lp.top_ids[1, :3] = torch.arange(15, dtype=torch.int32).view(3, 5)
    lp.top_lp[1, :3] = -torch.arange(15, dtype=torch.float32).view(3, 5)
    lp.step_idx[1, 0] = 2
    got = lp.generated_logprobs(1)
    assert got == [TokenLogprob(7, -0.5, [(0, -0.0), (1, -1.0), (2, -2.0), (3, -3.0), (4, -4.0)]),
                   TokenLogprob(8, -1.0, [(5, -5.0), (6, -6.0), (7, -7.0), (8, -8.0), (9, -9.0)])]


class _FakeLpDecoder:
    """serving.BatchedDecoder's host surface; request r emits its prompt length S, then S + 1, ...; the logprob of id
    i is -i / 1000 and its top list is (i, -i / 1000), (i + 1, ...), ... of the decoder's n"""

    def __init__(self, slots=2, logprobs=5):
        self.slots, self.pages_per_slot, self.logprobs = slots, 8, logprobs
        self.allocator = serving.PageAllocator(64)
        self.state = [None] * slots

    def capture(self):
        pass

    def admit(self, s, emb, params=None):
        self.state[s] = [emb.shape[0]]

    def run(self, n):
        for st in self.state:
            if st is not None:
                last = st[-1]
                st.extend(last + 1 + i for i in range(n))

    def generated(self, s):
        return list(self.state[s])

    def generated_logprobs(self, s):
        return [TokenLogprob(i, -i / 1000, [(i + j, -(i + j) / 1000) for j in range(self.logprobs)])
                for i in self.state[s]]

    def release(self, s):
        self.state[s] = None


def test_generate_batch_logprobs_host_logic():
    prompts = [torch.zeros(n, 4) for n in (10, 20, 30)]
    plain = serving.generate_batch(None, prompts, max_new_tokens=5, slots=2, check_every=4, decoder=_FakeLpDecoder())
    assert plain == [list(range(n, n + 5)) for n in (10, 20, 30)]  # no logprobs: the ids alone, as before
    ids, lps = serving.generate_batch(None, prompts, max_new_tokens=5, slots=2, check_every=4,
                                      decoder=_FakeLpDecoder(), logprobs=3)
    assert ids == plain and [len(x) for x in lps] == [5, 5, 5]  # cut at the budget, as the ids
    for r, row in enumerate(lps):
        assert [e.token for e in row] == ids[r]
        assert all(e.logprob == -e.token / 1000 and len(e.top) == 3 and e.top[0][0] == e.token for e in row)
    # EOS: the ids and their logprobs stop at it (included)
    ids, lps = serving.generate_batch(None, prompts, max_new_tokens=8, eos_token_ids=[22, 31], slots=2,
                                      check_every=4, decoder=_FakeLpDecoder(), logprobs=0)
    assert ids == [list(range(10, 18)), [20, 21, 22], [30, 31]]
    assert [[e.token for e in x] for x in lps] == ids and all(e.top == [] for x in lps for e in x)


def test_generate_batch_refuses_a_smaller_logprobs_decoder():
    prompts = [torch.zeros(10, 4)]
    with pytest.raises(ValueError, match="logprobs=None"):
        serving.generate_batch(None, prompts, max_new_tokens=4, decoder=_FakeLpDecoder(logprobs=None), logprobs=0)
    with pytest.raises(ValueError, match="logprobs=2"):
        serving.generate_batch(None, prompts, max_new_tokens=4, decoder=_FakeLpDecoder(logprobs=2), logprobs=3)
    real = serving.BatchedDecoder(_duck_llm(), slots=1, max_tokens_per_slot=256, max_new=8)
    with pytest.raises(ValueError, match="logprobs=None"):
        serving.generate_batch(_duck_llm(), prompts, max_new_tokens=4, decoder=real, logprobs=1)
    with pytest.raises(ValueError, match="0..20"):
        serving.generate_batch(None, prompts, max_new_tokens=4, decoder=_FakeLpDecoder(), logprobs=-1)
    # a decoder with more alternatives serves a smaller request, cut to its n
    _, lps = serving.generate_batch(None, prompts, max_new_tokens=4, decoder=_FakeLpDecoder(logprobs=5), logprobs=2)
    assert all(len(e.top) == 2 for e in lps[0])


def test_llava_generate_batch_passes_logprobs_through():
    from vila_b200.model.llava_llama import LlavaLlamaModel
    sig = inspect.signature(LlavaLlamaModel.generate_batch)
    assert sig.parameters["logprobs"].default is None
    src = inspect.getsource(LlavaLlamaModel.generate_batch)
    assert "logprobs=logprobs" in src and "sampling is not None, logprobs)" in src  # the kept engine's key


# ------------------------------------------------------------------------------------------------
# server
# ------------------------------------------------------------------------------------------------
def _server_stub(calls, stop=(9,)):
    class Tok:
        stop_token_ids = list(stop)

        def decode(self, ids, skip_special_tokens=True):
            return " ".join(f"t{i}é" for i in ids)

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
            ids = [[7, 8, 9] for _ in requests]
            if "logprobs" not in kw:
                return ids
            n = kw["logprobs"]
            lps = [[TokenLogprob(i, -i / 10, [(i + j, -(i + j) / 10) for j in range(n)]) for i in g] for g in ids]
            return ids, lps

    return Stub()


def _req(**kw):
    from vila_b200 import server as S
    return S.ChatCompletionRequest(model="m", max_tokens=kw.pop("max_tokens", 5),
                                   messages=[S.ChatMessage(role="user", content="hi")], **kw)


def test_server_logprobs_validation_and_streaming_refusal():
    from vila_b200 import server as S
    calls = {"batch": [], "single": 0}
    eng = S.Engine(_server_stub(calls), "m", slots=4)
    for bad, msg in ((dict(top_logprobs=3), "needs logprobs"), (dict(logprobs=True, top_logprobs=21), "0..20"),
                     (dict(logprobs=True, top_logprobs=-1), "0..20")):
        with pytest.raises(ValueError, match=msg):
            asyncio.run(eng.complete(_req(**bad)))
    assert calls == {"batch": [], "single": 0}  # refused before joining a batch
    with pytest.raises(ValueError, match="stream"):
        eng._stream_config(_req(stream=True, logprobs=True))

    async def streamed():
        return [c async for c in eng.stream(_req(stream=True, logprobs=True, top_logprobs=2))]

    with pytest.raises(ValueError, match="single-stream"):
        asyncio.run(streamed())
    assert "logprobs" in S.ChatCompletionRequest.model_fields and "top_logprobs" in S.ChatCompletionRequest.model_fields
    no_batch = _server_stub(calls)
    del type(no_batch).generate_batch
    with pytest.raises(ValueError, match="generate_batch"):
        asyncio.run(S.Engine(no_batch, "m").complete(_req(logprobs=True)))


def test_server_logprobs_routing_trimming_and_shape():
    from vila_b200 import server as S
    calls = {"batch": [], "single": 0}
    eng = S.Engine(_server_stub(calls), "m", slots=4)
    lone = asyncio.run(eng.complete(_req(logprobs=True, top_logprobs=2)))
    assert calls["single"] == 0 and calls["batch"] == [(1, {"logprobs": 2})]  # a lone request goes to the engine
    choice = lone["choices"][0]
    assert choice["message"]["content"] == "t7é t8é t9é"
    content = choice["logprobs"]["content"]
    assert [c["token"] for c in content] == ["t7é", "t8é"]  # the stop token 9 is excluded
    assert content[0] == {"token": "t7é", "logprob": -0.7, "bytes": list("t7é".encode("utf-8")),
                          "top_logprobs": [{"token": "t7é", "logprob": -0.7, "bytes": list("t7é".encode("utf-8"))},
                                           {"token": "t8é", "logprob": -0.8, "bytes": list("t8é".encode("utf-8"))}]}

    calls["batch"].clear()

    async def mixed():
        return await asyncio.gather(eng.complete(_req(logprobs=True, top_logprobs=5)), eng.complete(_req()),
                                    eng.complete(_req(logprobs=True)), eng.complete(_req(logprobs=True, max_tokens=1)))

    res = asyncio.run(mixed())
    n_kw = [kw for _, kw in calls["batch"]]
    assert all(kw.get("logprobs") in (5, 0, None) for kw in n_kw) and any(kw.get("logprobs") == 5 for kw in n_kw)
    assert [len(e["top_logprobs"]) for e in res[0]["choices"][0]["logprobs"]["content"]] == [5, 5]
    assert "logprobs" not in res[1]["choices"][0]  # not asked for: the response is as before
    assert [len(e["top_logprobs"]) for e in res[2]["choices"][0]["logprobs"]["content"]] == [0, 0]
    assert [e["token"] for e in res[3]["choices"][0]["logprobs"]["content"]] == ["t7é"]  # max_tokens 1
    assert res[3]["choices"][0]["message"]["content"] == "t7é"


def test_server_passes_no_logprobs_keyword_when_nobody_asked():
    from vila_b200 import server as S
    calls = {"batch": [], "single": 0}
    eng = S.Engine(_server_stub(calls), "m", slots=4)

    async def default():
        return await asyncio.gather(*[eng.complete(_req()) for _ in range(3)])

    res = asyncio.run(default())
    assert all("logprobs" not in kw for _, kw in calls["batch"])
    assert all("logprobs" not in r["choices"][0] for r in res)
    calls = {"batch": [], "single": 0}
    eng = S.Engine(_server_stub(calls), "m", slots=4, sample=True)
    asyncio.run(eng.complete(_req(seed=1)))
    assert "logprobs" not in calls["batch"][0][1]
    asyncio.run(eng.complete(_req(seed=1, logprobs=True, top_logprobs=1)))
    assert calls["batch"][1][1]["logprobs"] == 1 and "sampling" in calls["batch"][1][1]
