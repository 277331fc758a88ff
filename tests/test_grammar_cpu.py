"""CPU: grammar-constrained decoding without a device.

  * the rule of vila_b200/grammar.py on hand-built cases and against xgrammar's own apply_token_bitmask_inplace on CPU
    tensors at V in {152064, 151936, 1003, 37}, with bits at and beyond V set;
  * the pure-Python matcher of the tests and an xgrammar matcher over a toy vocabulary;
  * vila_apply_token_bitmask_row's export and its argument errors, reported before any device call;
  * the chunk loop ending when the decoder's grammar terminates; stream_content and generate_content routing a
    response_format to the graph decoder with a matcher whose stop tokens are the EOS ids;
  * the server on stubs: response_format routing for streamed and non-streamed requests, "text" is no constraint, bad
    schemas fail first, combinations with logprobs, penalties and --sample, requests without the field unchanged.
"""
import asyncio
import json
import threading
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests.grammar_support import PyMatcher, TOY_JSON, allow_all, pack, random_subsets, toy_compiler
from vila_b200.grammar import allowed_ids, any_allowed, bitmask_words, reference_masked

VOCABS = [152064, 151936, 1003, 37]


def _row(V, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(V, generator=g) * 4).to(torch.bfloat16)
    x[::97] = float("-inf")  # rows may already hold -inf
    return x


def _mask(V, seed, density):
    rng = np.random.default_rng(seed)
    w = pack(rng.random(V) < density, bitmask_words(V))
    if V % 32:
        w[-1] |= np.int32(-1 << (V % 32))  # bits at and beyond V: ignored
    return w


def test_rule_on_hand_built_cases():
    V = 37
    x = torch.arange(V, dtype=torch.float32).to(torch.bfloat16) - 3
    ones = np.full(bitmask_words(V), -1, dtype=np.int32)
    assert torch.equal(reference_masked(x, ones).view(torch.int16), x.view(torch.int16))
    none = np.zeros(2, dtype=np.int32)
    none[1] = np.int32(-1 << 5)  # only bits >= V
    y = reference_masked(x, none)
    assert bool((y.view(torch.int16) == torch.tensor(0xFF80 - 65536, dtype=torch.int16)).all())
    assert not any_allowed(none, V) and any_allowed(ones, V)
    one = np.array([0, 1 << 4], dtype=np.int32)  # token 36 alone
    assert allowed_ids(one, V).nonzero()[0].tolist() == [36] and any_allowed(one, V)
    y = reference_masked(x, one)
    assert y[36].item() == x[36].item() and torch.isinf(y[:36]).all() and (y[:36] < 0).all()
    # word 0 bit 31 is token 31 (the sign bit of the int32)
    assert allowed_ids(np.array([np.int32(-2 ** 31), 0], dtype=np.int32), V).nonzero()[0].tolist() == [31]
    assert not any_allowed(np.zeros(4752, dtype=np.int32), 152064)


@pytest.mark.parametrize("V", VOCABS)
def test_rule_matches_xgrammar_apply_token_bitmask(V):
    import xgrammar as xgr
    for seed, density in ((1, 0.5), (2, 0.01), (3, 1.0)):
        x = _row(V, seed)
        w = _mask(V, seed, density)
        want = x.float().clone()[None]
        xgr.apply_token_bitmask_inplace(want, torch.from_numpy(w)[None], vocab_size=V)
        got = reference_masked(x, w)
        assert torch.equal(got.float(), want[0]), f"V={V} density={density}"
        keep = torch.from_numpy(allowed_ids(w, V))
        assert torch.equal(got[keep].view(torch.int16), x[keep].view(torch.int16))  # bit for bit where allowed


def test_python_matcher_follows_the_interface():
    V = 70
    m = random_subsets(V, seed=4, density=0.1)
    mask = torch.zeros(1, bitmask_words(V), dtype=torch.int32)
    for t in range(5):
        m.fill_next_token_bitmask(mask)
        ok = allowed_ids(mask[0], V)
        assert ok.any() and (ok == m.allowed(t, m.history)).all()
        bad = int(np.flatnonzero(~ok)[0])
        assert not m.accept_token(bad)
        assert m.accept_token(int(np.flatnonzero(ok)[-1])) and not m.is_terminated()
    stop = PyMatcher(V, lambda t, h: np.arange(V) < 3, stop=(2,))
    assert stop.accept_token(1) and not stop.is_terminated()
    assert stop.accept_token(2) and stop.is_terminated() and not stop.accept_token(1)
    a = allow_all(V)
    a.fill_next_token_bitmask(mask)
    assert allowed_ids(mask[0], V).all()


def test_xgrammar_matcher_over_a_toy_vocabulary():
    import xgrammar as xgr
    V = 1024
    compiler, vocab = toy_compiler(V)
    m = xgr.GrammarMatcher(compiler.compile_builtin_json_grammar(), override_stop_tokens=[0])
    mask = torch.zeros(1, bitmask_words(V), dtype=torch.int32)
    out = []
    for tok in ("{", "\"a\"", ":", " ", "42", "}", "</s>"):
        m.fill_next_token_bitmask(mask)
        ok = allowed_ids(mask[0], V)
        t = vocab.index(tok)
        assert ok[t] and not ok[len(TOY_JSON):].any(), tok  # padding is never allowed
        assert m.accept_token(t)
        out.append(tok)
    assert m.is_terminated() and json.loads("".join(out[:-1])) == {"a": 42}
    # a schema: only the keys it names
    schema = json.dumps({"type": "object", "properties": {"name": {"type": "string"}}, "required": ["name"],
                         "additionalProperties": False})
    m = xgr.GrammarMatcher(compiler.compile_json_schema(schema, indent=2), override_stop_tokens=[0])
    m.fill_next_token_bitmask(mask)
    assert allowed_ids(mask[0], V)[vocab.index("{")]
    assert m.accept_token(vocab.index("{"))
    assert m.accept_token(vocab.index("\n")) and m.accept_token(vocab.index("  "))
    m.fill_next_token_bitmask(mask)
    ok = allowed_ids(mask[0], V)
    assert ok[vocab.index("\"name\"")] and not ok[vocab.index("\"a\"")]


def test_entry_point_reports_argument_errors_before_any_device_call():
    """every call below fails the argument checks, so it is safe with or without a device"""
    import ctypes

    from vila_b200 import _lib
    lib = _lib.load()
    assert "vila_apply_token_bitmask_row" in _lib.SIGNATURES
    buf = (ctypes.c_int32 * 64)()
    a = ctypes.addressof(buf)
    for args, msg in (((None, a, a + 128, 8), b"required"), ((a, a + 128, a, 0), b"vocabulary size"),
                      ((a + 1, a + 128, a + 64, 8), b"misaligned"), ((a, a + 130, a + 64, 8), b"misaligned"),
                      ((a, a + 128, a + 2, 8), b"overlap")):
        assert lib.vila_apply_token_bitmask_row(*args, None) != 0
        assert msg in lib.vila_last_error(), (args, lib.vila_last_error())


def test_ops_rejections():
    from vila_b200 import ops
    row = torch.zeros(40, dtype=torch.bfloat16)
    mask = torch.zeros(2, dtype=torch.int32)
    with pytest.raises(ValueError, match="at least 2 words"):
        ops.apply_token_bitmask_row(row, mask[:1], out=row)
    with pytest.raises(ValueError, match="int32"):
        ops.apply_token_bitmask_row(row, mask.long(), out=row)
    with pytest.raises(ValueError, match="contiguous"):
        ops.apply_token_bitmask_row(row, mask, out=torch.zeros(41, dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.apply_token_bitmask_row(row, mask, out=row)


# ------------------------------------------------------------------------------------------------
# decode loop and model routing
# ------------------------------------------------------------------------------------------------
class _StoppingDecoder:
    """a started decoder whose grammar terminates after `total` ids"""

    def __init__(self, total):
        self.total, self.done, self.log = total, 0, []

    def run(self, n):
        self.log.append(n)
        self.done = min(self.total, self.done + n)

    def read(self, n, start=0):
        ids = list(range(start, min(n, self.done)))
        return lambda: (ids, None)


def test_chunk_loop_ends_when_the_grammar_terminates():
    from vila_b200.model.qwen2 import _decode_chunks
    dec = _StoppingDecoder(10)
    assert list(_decode_chunks(dec, 64, 4, [], ahead=False)) == [([0, 1, 2, 3], None), ([4, 5, 6, 7], None),
                                                                 ([8, 9], None)]
    assert dec.log == [4, 4, 4]
    dec = _StoppingDecoder(8)  # ends on a chunk boundary: the next chunk is empty and not yielded
    assert [ids for ids, _ in _decode_chunks(dec, 64, 4, [], ahead=False)] == [[0, 1, 2, 3], [4, 5, 6, 7]]
    dec = _StoppingDecoder(100)  # EOS still cuts
    assert [ids for ids, _ in _decode_chunks(dec, 64, 4, [6], ahead=False)] == [[0, 1, 2, 3], [4, 5, 6]]


def _model_stub(calls, fail_sampled=False):
    from vila_b200.model.llava_llama import LlavaLlamaModel

    class LLM:
        def stream_tokens(self, emb, gc, chunk_tokens=8, sampling=None, logprobs=None, penalties=None, **kw):
            calls.append(dict(sampling=sampling, logprobs=logprobs, penalties=penalties, **kw))
            if fail_sampled and sampling is not None:
                raise ValueError("sampling failed")
            yield [1, 9, 2]
            yield [3]

    class Stub:
        llm = LLM()
        tokenizer = SimpleNamespace(decode=lambda ids, skip_special_tokens=True: " ".join(map(str, ids)))
        default_generation_config = SimpleNamespace(max_new_tokens=8, eos_token_id=[7, 8], do_sample=False)
        _sp_runner = staticmethod(lambda: None)
        _prepare_content = staticmethod(lambda prompt: (None, None, None))
        _embed = staticmethod(lambda *a: (torch.zeros(1, 3, 4), None, None))
        stream_content = LlavaLlamaModel.stream_content
        generate_content = LlavaLlamaModel.generate_content
        _generate_content_stream = LlavaLlamaModel._generate_content_stream

        def grammar_matcher(self, rf, stop):
            calls.append(("matcher", rf.type, stop))
            return "matcher"

    return Stub()


def test_model_routes_response_format_to_the_graph_decoder():
    from llava.model.configuration_llava import ResponseFormat
    calls = []
    m = _model_stub(calls)
    rf = ResponseFormat(type="json_object")
    chunks = list(m.stream_content(["q"], response_format=rf))
    assert chunks == [([1, 9, 2], None), ([3], None)]
    assert calls[0] == ("matcher", "json_object", [7, 8]) and calls[1]["grammar"] == "matcher"
    calls.clear()
    assert list(m.stream_content(["q"])) == chunks and "grammar" not in calls[0]  # no grammar: not passed
    calls.clear()
    assert m.generate_content(["q"], response_format=rf) == "1 9 2 3"
    assert m.generate_content(["q"], stream=True, response_format=rf) is not None
    assert list(m.generate_content(["q"], stream=True, response_format=rf)) == ["1 9 2", "3"]
    assert all(c[0] == "matcher" if isinstance(c, tuple) else c["grammar"] == "matcher" for c in calls)
    # a sampled constrained request that fails with a ValueError is retried greedily with a fresh matcher
    calls.clear()
    m = _model_stub(calls, fail_sampled=True)
    gc = SimpleNamespace(max_new_tokens=8, eos_token_id=5, do_sample=True, temperature=0.7, top_k=0, top_p=1.0,
                         seed=3)
    assert m.generate_content(["q"], gc, response_format=rf) == "1 9 2 3"
    assert gc.do_sample is False
    assert [c for c in calls if isinstance(c, tuple)] == [("matcher", "json_object", [5])] * 2
    # sequence-parallel decoding is refused
    m._sp_runner = lambda: object()
    with pytest.raises(NotImplementedError, match="response_format"):
        list(m.stream_content(["q"], response_format=rf))


def test_compile_keeps_the_reference_mapping_and_uses_the_installed_compiler():
    import xgrammar as xgr

    from llava.model.configuration_llava import JsonSchemaResponseFormat, ResponseFormat
    from vila_b200.model.llava_llama import LlavaLlamaModel
    compiler, vocab = toy_compiler(64)
    stub = SimpleNamespace(grammar_compiler=compiler)
    stub.compile_response_format = lambda rf: LlavaLlamaModel.compile_response_format(stub, rf)
    schema = json.dumps({"type": "array", "items": {"type": "integer"}})
    sch = ResponseFormat(type="json_schema", json_schema=JsonSchemaResponseFormat(schema=schema))
    mask = torch.zeros(1, 2, dtype=torch.int32)

    def first_allowed(rf):
        m = LlavaLlamaModel.grammar_matcher(stub, rf, [0])
        assert isinstance(m, xgr.GrammarMatcher)
        m.fill_next_token_bitmask(mask)
        return {vocab[j] for j in np.flatnonzero(allowed_ids(mask[0], 64))}

    assert first_allowed(sch) == {"["}
    assert first_allowed(ResponseFormat(type="json_object")) == {"{", "[", "{\""}  # the builtin JSON grammar
    assert first_allowed(ResponseFormat(type="text")) == first_allowed(ResponseFormat(type="json_object"))
    with pytest.raises(RuntimeError):
        LlavaLlamaModel.compile_response_format(stub, ResponseFormat(
            type="json_schema", json_schema=JsonSchemaResponseFormat(schema="{not json")))


# ------------------------------------------------------------------------------------------------
# server
# ------------------------------------------------------------------------------------------------
def _server_stub(calls, compile_errors=False):
    from vila_b200.logprobs import TokenLogprob

    class Tok:
        stop_token_ids = [9]

        def decode(self, ids, skip_special_tokens=True):
            return "".join(f"t{i}" for i in ids if i != 9)

    class Stub:
        tokenizer = Tok()
        default_generation_config = SimpleNamespace(max_new_tokens=None)

        def generate_content(self, prompt, generation_config=None, response_format=None, stream=False):
            calls.append(("generate_content", response_format, stream))
            return iter(["a"]) if stream else "plain"

        def generate_batch(self, requests, **kw):
            calls.append(("generate_batch", kw))
            return [[1]] * len(requests)

        def _prepare_content(self, prompt):
            return None, None, None

        def stream_content(self, prompt, generation_config=None, *, logprobs=None, penalties=None, chunk_tokens=8,
                           response_format=None):
            if response_format is not None:  # as the model: the matcher is built, and the grammar compiled, first
                self.compile_response_format(response_format)
            calls.append(("stream_content", generation_config, logprobs, penalties, response_format))
            for ids in ([7, 8], [5, 9]):
                yield ids, None if logprobs is None else [TokenLogprob(i, -i / 10, [(i, -i / 10)] * logprobs)
                                                          for i in ids]

        def compile_response_format(self, rf):
            calls.append(("compile", rf.type, threading.current_thread() is threading.main_thread()))
            if compile_errors:
                raise RuntimeError("cannot compile")

    return Stub()


def _req(**kw):
    from vila_b200 import server as S
    return S.ChatCompletionRequest(model="m", max_tokens=kw.pop("max_tokens", 5),
                                   messages=[S.ChatMessage(role="user", content="hi")], **kw)


def _events(eng, req):
    async def go():
        return [c async for c in eng.stream(req)]

    out = asyncio.run(go())
    assert out[-1] == "data: [DONE]\n\n"
    return [json.loads(c[len("data: "):]) for c in out[:-1]]


SCHEMA = json.dumps({"type": "object", "properties": {"a": {"type": "integer"}}})


def test_server_routes_response_format_through_stream_content():
    from vila_b200 import server as S
    calls = []
    eng = S.Engine(_server_stub(calls), "m")
    rf = {"type": "json_schema", "json_schema": {"schema": SCHEMA}}
    ev = _events(eng, _req(stream=True, response_format=rf))
    assert [e["choices"][0]["delta"]["content"] for e in ev] == ["t7t8", "t5"]
    sc = [c for c in calls if c[0] == "stream_content"]
    assert len(sc) == 1 and sc[0][4].type == "json_schema" and sc[0][4].json_schema.schema_ == SCHEMA
    assert sc[0][2] is None and sc[0][3] is None and sc[0][1].do_sample is False
    assert not any(c[0] in ("generate_content", "generate_batch") for c in calls)
    # non-streamed: decoded alone through stream_content, collected into one completion, never batched
    calls.clear()
    out = asyncio.run(eng.complete(_req(response_format={"type": "json_object"})))
    assert out["object"] == "chat.completion" and out["choices"][0]["message"]["content"] == "t7t8t5"
    assert "logprobs" not in out["choices"][0]
    # compiled once, in a worker thread (the decode's), not on the event loop's thread
    assert calls[0] == ("compile", "json_object", False) and len(calls) == 2
    assert calls[1][0] == "stream_content" and calls[1][4].type == "json_object"
    # a streamed request's schema is compiled in a worker thread before its stream starts
    calls.clear()
    asyncio.run(eng.check_stream(_req(stream=True, response_format=rf)))
    assert calls == [("compile", "json_schema", False)]


def test_server_text_format_is_unconstrained_and_requests_without_it_are_unchanged():
    from vila_b200 import server as S
    calls = []
    eng = S.Engine(_server_stub(calls), "m")
    out = asyncio.run(eng.complete(_req(response_format={"type": "text"})))
    assert out["choices"][0]["message"]["content"] == "plain" and calls == [("generate_content", None, False)]
    calls.clear()
    assert asyncio.run(eng.complete(_req()))["choices"][0]["message"]["content"] == "plain"
    assert calls == [("generate_content", None, False)]
    calls.clear()
    assert _events(eng, _req(stream=True, response_format={"type": "text"}))[0]["choices"][0]["delta"] == {
        "content": "a"}
    assert calls == [("generate_content", None, True)]
    # logprobs without a response_format: stream_content is called without the keyword (older stubs lack it)
    calls.clear()
    _events(eng, _req(stream=True, logprobs=True))
    assert calls[0][0] == "stream_content" and calls[0][4] is None


def test_server_response_format_combines_with_logprobs_penalties_and_sampling():
    from vila_b200 import server as S
    from vila_b200.penalties import PenaltyParams
    calls = []
    eng = S.Engine(_server_stub(calls), "m", sample=True)
    req = _req(response_format={"type": "json_object"}, logprobs=True, top_logprobs=1, presence_penalty=0.5,
               temperature=0.7, top_p=0.9, seed=4)
    out = asyncio.run(eng.complete(req))
    _, gc, top, pen, rf = calls[-1]
    assert top == 1 and pen == PenaltyParams(0.5, 0.0) and rf.type == "json_object"
    assert gc.do_sample and gc.temperature == 0.7 and gc.top_p == 0.9 and gc.seed == 4 and gc.max_new_tokens == 5
    content = out["choices"][0]["logprobs"]["content"]
    assert [x["token"] for x in content] == ["t7", "t8", "t5"]  # the stop token excluded
    assert not any(c[0] == "generate_batch" for c in calls)
    ev = _events(eng, _req(stream=True, response_format={"type": "json_object"}, logprobs=True, frequency_penalty=1.0))
    _, gc, top, pen, rf = calls[-1]
    assert top == 0 and pen.frequency == 1.0 and rf.type == "json_object"
    assert [x["token"] for e in ev for x in e["choices"][0]["logprobs"]["content"]] == ["t7", "t8", "t5"]


def test_server_bad_schemas_fail_before_streaming():
    from vila_b200 import server as S
    calls = []
    eng = S.Engine(_server_stub(calls), "m")
    for rf, msg in (({"type": "json_schema"}, "needs json_schema"),
                    ({"type": "json_schema", "json_schema": {"schema": "{not json"}}, "not valid JSON")):
        with pytest.raises(ValueError, match=msg):
            asyncio.run(eng.check_stream(_req(stream=True, response_format=rf)))
        with pytest.raises(ValueError, match=msg):
            asyncio.run(eng.complete(_req(response_format=rf)))
    eng = S.Engine(_server_stub(calls, compile_errors=True), "m")
    with pytest.raises(RuntimeError, match="cannot compile"):
        asyncio.run(eng.check_stream(_req(stream=True, response_format={"type": "json_object"})))
    with pytest.raises(RuntimeError, match="cannot compile"):
        asyncio.run(eng.complete(_req(response_format={"type": "json_object"})))
    assert not any(c[0] in ("stream_content", "generate_content", "generate_batch") for c in calls)
    # the app answers 500 before the stream starts
    from fastapi.testclient import TestClient
    app = S.create_app(_server_stub(calls), "m")
    r = TestClient(app).post("/chat/completions", json=dict(
        model="m", stream=True, messages=[{"role": "user", "content": "hi"}],
        response_format={"type": "json_schema", "json_schema": {"schema": "[1,"}}))
    assert r.status_code == 500 and "not valid JSON" in r.json()["error"]
    # a model without stream_content cannot apply a grammar
    stub = _server_stub(calls)
    del type(stub).stream_content
    with pytest.raises(ValueError, match="stream_content"):
        asyncio.run(S.Engine(stub, "m").check_stream(_req(stream=True, response_format={"type": "json_object"})))


def test_sequence_parallel_generate_refuses_a_grammar():
    from vila_b200.model.qwen2 import Qwen2ForCausalLM
    with pytest.raises(NotImplementedError, match="grammar"):
        Qwen2ForCausalLM._generate_greedy(SimpleNamespace(), torch.zeros(3, 8), 4, [], sp_runner=object(),
                                          grammar=allow_all(8))
