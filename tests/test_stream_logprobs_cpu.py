"""CPU: logprobs and presence / frequency penalties in the single-stream graph decoder without a device: the argument
errors of ops.token_logprobs_row / ops.apply_penalties_row, the structs' field order against the header, the loud
failure of both entry points, GraphDecoder's host logic on a stand-in (graph selection per mode, .off penalties on the
base graph, lazily allocated buffers, launches per step, the sequence-parallel refusal), stream_tokens' chunk shapes
and EOS truncation of the entries, and the server's streaming plumbing on stubs with and without stream_content."""
import asyncio
import json
import re
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch

from vila_b200 import ops
from vila_b200.logprobs import TokenLogprob
from vila_b200.model.qwen2 import GraphDecoder, Qwen2ForCausalLM
from vila_b200.penalties import PenaltyParams

ROOT = Path(__file__).resolve().parent.parent


def _fields(struct):
    text = (ROOT / "include" / "vila_b200.h").read_text()
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (struct, struct), text, flags=re.S).group(1)
    fields = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        names = decl.split(",")
        fields.append(names[0].split()[-1].lstrip("*"))
        fields.extend(x.strip().lstrip("*") for x in names[1:])
    return fields


def test_structs_match_the_header():
    from vila_b200 import _lib
    assert _fields("vila_logprobs_row_params") == [f[0] for f in _lib.LogprobsRowParams._fields_] == [
        "logits", "token", "step", "lp_hist", "top_ids", "top_lp", "n_used", "workspace", "workspace_bytes", "counter",
        "V", "cols", "n"]
    assert _fields("vila_penalty_row_params") == [f[0] for f in _lib.PenaltyRowParams._fields_] == [
        "logits", "history", "step", "presence", "frequency", "out", "V", "cols"]
    for name in ("vila_token_logprobs_row", "vila_apply_penalties_row"):
        assert name in _lib.SIGNATURES and hasattr(_lib.load(), name)
    assert _lib.load().vila_abi_version() == 3


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_entry_points_fail_loudly_without_gpu():
    from vila_b200 import _lib
    lib = _lib.load()
    assert lib.vila_token_logprobs_row(None, None) != 0 and b"params are required" in lib.vila_last_error()
    p = _lib.LogprobsRowParams()
    assert lib.vila_token_logprobs_row(p, None) != 0 and b"required" in lib.vila_last_error()
    buf = torch.zeros(4096, dtype=torch.int64)
    for name in ("logits", "token", "step", "lp_hist", "workspace", "counter"):
        setattr(p, name, buf.data_ptr())
    p.V, p.cols, p.n, p.workspace_bytes = 1000, 4, 0, 168
    assert lib.vila_token_logprobs_row(p, None) != 0 and b"no CUDA device" in lib.vila_last_error()
    p.n = 21
    assert lib.vila_token_logprobs_row(p, None) != 0 and b"n=21" in lib.vila_last_error()
    p.n, p.V = 0, 2000  # two chunks need 336 bytes
    assert lib.vila_token_logprobs_row(p, None) != 0 and b"workspace" in lib.vila_last_error()

    assert lib.vila_apply_penalties_row(None, None) != 0 and b"params are required" in lib.vila_last_error()
    q = _lib.PenaltyRowParams()
    assert lib.vila_apply_penalties_row(q, None) != 0 and b"required" in lib.vila_last_error()
    for name in ("logits", "history", "step", "presence", "frequency", "out"):
        setattr(q, name, buf.data_ptr())
    q.V, q.cols = 1000, 8
    assert lib.vila_apply_penalties_row(q, None) != 0 and b"no CUDA device" in lib.vila_last_error()
    q.V = 8 * 40960 + 1
    assert lib.vila_apply_penalties_row(q, None) != 0 and b"vocabulary" in lib.vila_last_error()


def _lp_args(V=100, cols=6, n=4):
    return dict(logits=torch.zeros(V, dtype=torch.bfloat16), token=torch.zeros(1, dtype=torch.int32),
                step=torch.zeros(1, dtype=torch.int32), lp_hist=torch.zeros(cols),
                workspace=torch.zeros(21, dtype=torch.int64), counter=torch.zeros(1, dtype=torch.int32),
                top_ids=torch.zeros(cols, n, dtype=torch.int32), top_lp=torch.zeros(cols, n))


def _call_lp(a):
    return ops.token_logprobs_row(a.pop("logits"), a.pop("token"), a.pop("step"), **a)


def test_ops_token_logprobs_row_rejections():
    cases = [
        (dict(logits=torch.zeros(2, 50, dtype=torch.bfloat16)), "contiguous \\[V\\] row"),
        (dict(top_lp=None), "go together"),
        (dict(lp_hist=torch.zeros(2, 3)), "lp_hist"),
        (dict(top_ids=torch.zeros(5, 4, dtype=torch.int32)), "top_ids must be"),
        (dict(top_ids=torch.zeros(6, 21, dtype=torch.int32), top_lp=torch.zeros(6, 21)), "n=21"),
        (dict(token=torch.zeros(1, dtype=torch.int64)), "token must be"),
        (dict(step=torch.zeros(2, dtype=torch.int32)), "step must be a single value"),
        (dict(workspace=torch.zeros(2, dtype=torch.int64)), "workspace"),
        (dict(counter=torch.zeros(1, dtype=torch.int64)), "counter must be"),
        (dict(n_used=torch.zeros(2, dtype=torch.int32)), "n_used must be a single value"),
        (dict(n_used=torch.zeros(1, dtype=torch.int64)), "n_used must be"),
    ]
    for change, msg in cases:
        a = _lp_args()
        a.update(change)
        with pytest.raises(ValueError, match=msg):
            _call_lp(a)
    with pytest.raises(RuntimeError, match="CUDA tensor"):  # valid arguments: no CPU fallback
        _call_lp(_lp_args())
    ws, counter = ops.logprobs_row_workspace(152064, "cpu")
    assert ws.numel() * 8 == 132 * 168 and counter.tolist() == [0]


def test_ops_apply_penalties_row_rejections():
    def args(**kw):
        a = dict(logits=torch.zeros(100, dtype=torch.bfloat16), history=torch.zeros(8, dtype=torch.int32),
                 step=torch.zeros(1, dtype=torch.int32), presence=torch.zeros(1), frequency=torch.zeros(1),
                 out=torch.zeros(100, dtype=torch.bfloat16))
        a.update(kw)
        return a

    def call(a):
        return ops.apply_penalties_row(a.pop("logits"), a.pop("history"), a.pop("step"), a.pop("presence"),
                                       a.pop("frequency"), **a)

    for change, msg in ((dict(logits=torch.zeros(2, 50, dtype=torch.bfloat16)), "contiguous \\[V\\] row"),
                        (dict(history=torch.zeros(2, 4, dtype=torch.int32)), "history must be"),
                        (dict(history=torch.zeros(8, dtype=torch.int64)), "history must be torch.int32"),
                        (dict(out=torch.zeros(99, dtype=torch.bfloat16)), "out must be"),
                        (dict(step=torch.zeros(1, dtype=torch.int64)), "step must be torch.int32"),
                        (dict(presence=torch.zeros(2)), "presence must be a single value")):
        with pytest.raises(ValueError, match=msg):
            call(args(**change))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        call(args())


# ------------------------------------------------------------------------------------------------
# GraphDecoder host logic on a stand-in (no kernels run: ops calls are recorded)
# ------------------------------------------------------------------------------------------------
class _Cfg:
    num_hidden_layers, hidden_size, num_attention_heads, num_key_value_heads, head_dim = 2, 8, 4, 2, 4
    intermediate_size, rms_norm_eps, vocab_size = 16, 1e-6, 50


def _stand_in_llm():
    emb = torch.zeros(50, 8, dtype=torch.bfloat16)
    norm = SimpleNamespace(weight=torch.ones(8, dtype=torch.bfloat16))
    return SimpleNamespace(config=_Cfg(), device=torch.device("cpu"), dtype=torch.bfloat16, _fp8_weights=None,
                           _w4_weights=None, lm_head=SimpleNamespace(weight=emb),
                           model=SimpleNamespace(embed_tokens=SimpleNamespace(weight=emb), norm=norm, layers=[]))


@pytest.fixture
def recorded(monkeypatch):
    calls = []
    for name in ("gemv", "argmax_finalize", "sample_finalize", "apply_penalties_row", "token_logprobs_row"):
        monkeypatch.setattr(ops, name, lambda *a, _n=name, **k: calls.append((_n, k)))
    monkeypatch.setattr(ops, "logprobs_row_workspace",
                        lambda V, dev: (torch.zeros(21, dtype=torch.int64), torch.zeros(1, dtype=torch.int32)))
    return calls


def _decoder():
    dec = GraphDecoder(_stand_in_llm(), 16)
    dec.cache = SimpleNamespace(length=10)
    dec._order_key = None
    return dec


def test_decoder_modes_select_their_graph_keys_and_buffers(recorded):
    from vila_b200.sampling import SamplingParams
    dec = _decoder()
    base = dec.launches_per_step
    assert base == 5 * 2 + 2

    def head(call):  # the lm_head GEMV as ops.gemv reads its arguments: (writes the row, keeps the argmax key)
        kw = call[1]
        return kw.get("out") is dec.logits and kw.get("write_out", True), kw.get("argmax_key") is dec.key

    dec.start(torch.zeros(8), dec.cache)
    assert [c[0] for c in recorded] == ["gemv", "argmax_finalize"] and head(recorded[0]) == (False, True)
    assert dec.lp_hist is None and dec.pen_logits is None  # nothing allocated without the options
    plan = (dec.num_splits, dec.split_tokens)
    assert dec._graph_key() == (False, False, False) + plan
    dec.start(torch.zeros(8), dec.cache, penalties=PenaltyParams(0.0, 0.0))  # .off: the base graph
    assert dec._graph_key() == (False, False, False) + plan and dec.pen_logits is None
    assert dec.launches_per_step == base
    recorded.clear()
    dec.start(torch.zeros(8), dec.cache, logprobs=5)
    assert [c[0] for c in recorded] == ["gemv", "argmax_finalize", "token_logprobs_row"]
    assert recorded[0][1]["argmax_key"] is dec.key and recorded[0][1]["out"] is dec.logits  # row and key together
    assert head(recorded[0]) == (True, True)
    assert dec.lp_hist.shape == (24,) and dec.top_ids.shape == (24, 20) and dec.pen_logits is None
    assert recorded[2][1]["top_ids"] is dec.top_ids and recorded[2][1]["n_used"] is dec.lp_n and dec.lp_n.item() == 5
    key = dec._graph_key()
    assert key == (False, False, True) + plan and dec.launches_per_step == base + 1
    dec.start(torch.zeros(8), dec.cache, logprobs=17)  # another n: the same graph, n is a device scalar
    assert dec._graph_key() == key and dec.lp_n.item() == 17
    recorded.clear()
    dec.inv_temperature.fill_(0.5)
    dec.start(torch.zeros(8), dec.cache, penalties=PenaltyParams(0.5, -1.0), logprobs=0)
    assert [c[0] for c in recorded] == ["gemv", "apply_penalties_row", "sample_finalize", "token_logprobs_row"]
    assert float(dec.inv_temperature) == 0.0  # greedy on the penalised row
    assert dec.presence.item() == 0.5 and dec.frequency.item() == -1.0
    assert recorded[2][0] == "sample_finalize" and head(recorded[0]) == (True, False)
    assert dec._graph_key() == (False, True, True) + plan and dec.launches_per_step == base + 2
    assert dec.lp_n.item() == 0
    recorded.clear()
    dec.start(torch.zeros(8), dec.cache, SamplingParams(0.7, seed=3), penalties=PenaltyParams(1.0, 0.0))
    assert [c[0] for c in recorded] == ["gemv", "apply_penalties_row", "sample_finalize"]
    assert head(recorded[0]) == (True, False)
    assert dec._graph_key() == (True, True, False) + plan and dec.launches_per_step == base + 1
    recorded.clear()
    dec.start(torch.zeros(8), dec.cache, SamplingParams(0.7, seed=3))
    assert [c[0] for c in recorded] == ["gemv", "sample_finalize"] and head(recorded[0]) == (True, False)
    assert dec._graph_key() == (True, False, False) + plan and dec.launches_per_step == base
    with pytest.raises(ValueError, match="started without logprobs"):
        dec.token_logprobs(3)
    with pytest.raises(ValueError, match="logprobs must be"):
        dec.start(torch.zeros(8), dec.cache, logprobs=21)


def test_decoder_refuses_options_on_a_sequence_parallel_cache(recorded):
    dec = _decoder()
    dec._order_key = ("sp", 2, 0, 256)
    dec.start(torch.zeros(8), dec.cache)  # plain greedy stays allowed
    for kw in (dict(logprobs=2), dict(penalties=PenaltyParams(0.5, 0.0))):
        with pytest.raises(NotImplementedError, match="sequence-parallel"):
            dec.start(torch.zeros(8), dec.cache, **kw)


def test_decoder_token_logprobs_reads_its_buffers(recorded):
    dec = _decoder()
    dec.start(torch.zeros(8), dec.cache, logprobs=2)
    dec.hist[:3] = torch.tensor([4, 5, 6], dtype=torch.int32)
    dec.lp_hist[:3] = torch.tensor([-0.5, -1.0, -1.5])
    dec.top_ids[:3, :2] = torch.tensor([[4, 1], [5, 2], [6, 3]], dtype=torch.int32)
    dec.top_lp[:3, :2] = torch.tensor([[-0.5, -2.0], [-1.0, -3.0], [-1.5, -4.0]])
    dec.top_ids[:3, 2:] = 99  # past n: not read
    got = dec.token_logprobs(3)
    assert got == [TokenLogprob(4, -0.5, [(4, -0.5), (1, -2.0)]), TokenLogprob(5, -1.0, [(5, -1.0), (2, -3.0)]),
                   TokenLogprob(6, -1.5, [(6, -1.5), (3, -4.0)])]
    assert dec.token_logprobs(3, start=1) == got[1:] and dec.token_logprobs(3, start=3) == []
    assert dec.read(3, start=1)() == ([5, 6], got[1:])
    dec.start(torch.zeros(8), dec.cache)  # without logprobs: the ids alone
    dec.hist[:3] = torch.tensor([4, 5, 6], dtype=torch.int32)
    assert dec.read(3, start=1)() == ([5, 6], None) and dec.read(3, start=3)() == ([], None)


# ------------------------------------------------------------------------------------------------
# stream_tokens on a stand-in decoder
# ------------------------------------------------------------------------------------------------
class _LpDecoder:
    def __init__(self):
        self.started = None
        self.log = []

    def cache_for(self, n):
        return "cache"

    def start(self, last_hidden, cache, params=None, **kw):
        self.started = kw

    def run(self, n):
        self.log.append(("run", n))

    def read(self, n, start=0):
        assert start % 4 == 0 and n - start <= 4  # only the chunk's new rows are asked for
        lp = self.started["logprobs"] is not None

        def wait():
            self.log.append(("wait", start))
            return [100 + i for i in range(start, n)], [TokenLogprob(100 + i, -i / 8, [(100 + i, -i / 8)])
                                                        for i in range(start, n)] if lp else None

        return wait


def _stream_llm():
    dec = _LpDecoder()
    return SimpleNamespace(generation_config=None, decoder=lambda n: dec, prefill_hidden_graphed=lambda e, c: e,
                           dec=dec)


def test_stream_tokens_chunk_reads_and_eos_truncation():
    llm = _stream_llm()
    gc = SimpleNamespace(max_new_tokens=10, eos_token_id=[106])
    pen = PenaltyParams(0.5, 0.5)
    out = list(Qwen2ForCausalLM.stream_tokens(llm, torch.zeros(3, 8), gc, chunk_tokens=4, logprobs=1, penalties=pen))
    assert llm.dec.started == dict(logprobs=1, penalties=pen)
    assert [ids for ids, _ in out] == [[100, 101, 102, 103], [104, 105, 106]]  # cut after the EOS id
    assert [[e.token for e in es] for _, es in out] == [ids for ids, _ in out]
    # one chunk ahead: chunk k + 1 is enqueued before the host waits for chunk k's rows
    assert llm.dec.log == [("run", 4), ("run", 4), ("wait", 0), ("run", 2), ("wait", 4)]
    llm.dec.log.clear()
    gc_all = SimpleNamespace(max_new_tokens=10, eos_token_id=[])
    out = list(Qwen2ForCausalLM.stream_tokens(llm, torch.zeros(3, 8), gc_all, chunk_tokens=4, logprobs=1))
    assert [ids for ids, _ in out] == [[100, 101, 102, 103], [104, 105, 106, 107], [108, 109]]
    assert llm.dec.log == [("run", 4), ("run", 4), ("wait", 0), ("run", 2), ("wait", 4), ("wait", 8)]
    llm.dec.log.clear()
    plain = list(Qwen2ForCausalLM.stream_tokens(llm, torch.zeros(3, 8), gc, chunk_tokens=4))
    assert plain == [[100, 101, 102, 103], [104, 105, 106]] and llm.dec.started == dict(logprobs=None, penalties=None)
    # no read-ahead without logprobs: each chunk's rows are read before the next chunk runs, none after EOS
    assert llm.dec.log == [("run", 4), ("wait", 0), ("run", 4), ("wait", 4)]
    llm.dec.log.clear()
    pen_only = list(Qwen2ForCausalLM.stream_tokens(llm, torch.zeros(3, 8), gc, chunk_tokens=4, penalties=pen))
    assert pen_only == plain and llm.dec.started == dict(logprobs=None, penalties=pen)
    assert llm.dec.log == [("run", 4), ("wait", 0), ("run", 4), ("wait", 4)]
    llm.dec.log.clear()
    plain_all = list(Qwen2ForCausalLM.stream_tokens(llm, torch.zeros(3, 8), gc_all, chunk_tokens=4))
    assert plain_all == [ids for ids, _ in out]
    assert llm.dec.log == [("run", 4), ("wait", 0), ("run", 4), ("wait", 4), ("run", 2), ("wait", 8)]
    with pytest.raises(ValueError, match="logprobs must be"):
        list(Qwen2ForCausalLM.stream_tokens(llm, torch.zeros(3, 8), gc, logprobs=30))


# ------------------------------------------------------------------------------------------------
# server
# ------------------------------------------------------------------------------------------------
def _stub(calls, stop=(9,)):
    class Tok:
        stop_token_ids = list(stop)

        def decode(self, ids, skip_special_tokens=True):
            return "".join(f"t{i}é" for i in ids if i not in (0, 9))  # id 0 decodes to no text

    class Stub:
        tokenizer = Tok()
        default_generation_config = SimpleNamespace(max_new_tokens=None)

        def generate_content(self, prompt, generation_config=None, response_format=None, stream=False):
            calls["plain"] += 1
            return iter(["a", "b"]) if stream else "single"

        def stream_content(self, prompt, generation_config=None, *, logprobs=None, penalties=None, chunk_tokens=8):
            calls["stream"].append((generation_config, logprobs, penalties))
            for ids in ([7, 8], [0, 0], [5, 9]):
                yield ids, None if logprobs is None else [
                    TokenLogprob(i, -i / 10, [(i + j, -(i + j) / 10) for j in range(logprobs)]) for i in ids]

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


def test_server_streams_logprobs_and_penalties_through_stream_content():
    from vila_b200 import server as S
    calls = {"plain": 0, "stream": []}
    eng = S.Engine(_stub(calls), "m")
    ev = _events(eng, _req(stream=True, logprobs=True, top_logprobs=2))
    gc, top, pen = calls["stream"][-1]
    assert top == 2 and pen is None and gc.do_sample is False and gc.max_new_tokens == 5
    assert [e["choices"][0]["delta"]["content"] for e in ev] == ["t7ét8é", "", "t5é"]  # the empty chunk is sent
    content = [x for e in ev for x in e["choices"][0]["logprobs"]["content"]]
    assert [x["token"] for x in content] == ["t7é", "t8é", "", "", "t5é"]  # every id once, the stop token excluded
    assert content[0] == {"token": "t7é", "logprob": -0.7, "bytes": list("t7é".encode()),
                          "top_logprobs": [{"token": "t7é", "logprob": -0.7, "bytes": list("t7é".encode())},
                                           {"token": "t8é", "logprob": -0.8, "bytes": list("t8é".encode())}]}
    assert all(e["object"] == "chat.completion.chunk" for e in ev) and calls["plain"] == 0
    # logprobs without top_logprobs: no alternatives
    ev = _events(eng, _req(stream=True, logprobs=True))
    assert all(x["top_logprobs"] == [] for e in ev for x in e["choices"][0]["logprobs"]["content"])
    # penalties alone: no logprobs field, the empty-text chunk is skipped
    ev = _events(eng, _req(stream=True, presence_penalty=0.5, frequency_penalty=-0.25))
    gc, top, pen = calls["stream"][-1]
    assert top is None and pen == PenaltyParams(0.5, -0.25)
    assert [e["choices"][0] for e in ev] == [{"delta": {"content": "t7ét8é"}}, {"delta": {"content": "t5é"}}]
    # zero penalties and no logprobs: the plain stream
    _events(eng, _req(stream=True, presence_penalty=0.0))
    assert calls["plain"] == 1 and len(calls["stream"]) == 3


def test_server_stream_passes_sampling_and_fails_bad_values_first():
    from vila_b200 import server as S
    calls = {"plain": 0, "stream": []}
    model = _stub(calls)
    type(model).generate_batch = lambda self, *a, **k: None  # Engine(sample=True) needs a model with generate_batch
    eng = S.Engine(model, "m", sample=True)
    _events(eng, _req(stream=True, logprobs=True, temperature=0.7, top_p=0.9, seed=5, frequency_penalty=1.0))
    gc, top, pen = calls["stream"][-1]
    assert gc.do_sample and gc.temperature == 0.7 and gc.top_p == 0.9 and gc.seed == 5 and pen.frequency == 1.0
    for bad, msg in ((dict(top_logprobs=3), "needs logprobs"), (dict(logprobs=True, top_logprobs=21), "0..20"),
                     (dict(presence_penalty=2.5), "presence penalty"), (dict(frequency_penalty=float("nan")), "frequency")):
        with pytest.raises(ValueError, match=msg):
            eng._stream_config(_req(stream=True, **bad))
    assert len(calls["stream"]) == 1


def test_server_without_stream_content_still_refuses():
    from vila_b200 import server as S
    calls = {"plain": 0, "stream": []}
    model = _stub(calls)
    del type(model).stream_content
    eng = S.Engine(model, "m")
    with pytest.raises(ValueError, match="logprobs are not supported with stream=true"):
        eng._stream_config(_req(stream=True, logprobs=True))
    with pytest.raises(ValueError, match="penalties are not supported with stream=true"):
        eng._stream_config(_req(stream=True, presence_penalty=0.5))
    assert _events(eng, _req(stream=True))[0]["choices"][0]["delta"]["content"] == "a"
