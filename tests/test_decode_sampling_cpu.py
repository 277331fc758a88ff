"""CPU: sampling in the single-stream graph decoder without a device: vila_sample_finalize's export, struct layout
and argument errors (reported before any device call); generate(do_sample=True) routing to the graph decoder (or to
the eager path with logits processors) with stand-in decoders; per-row seeds that replay after torch.manual_seed and
a generation config `seed` that wins; stream_tokens / stream_greedy passing the parameters to the decoder; the
server's streamed requests under --sample and without it."""
import asyncio
import ctypes as C
import re
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch

from vila_b200 import _lib
from vila_b200.model.qwen2 import Qwen2ForCausalLM, sampling_for_generate
from vila_b200.sampling import SamplingParams

ROOT = Path(__file__).resolve().parent.parent
FIELDS = ["logits", "inv_temperature", "top_k", "top_p", "seed", "step", "position", "token_out", "token_hist",
          "embed_table", "x_next", "V", "hidden"]


def test_entry_point_is_exported():
    assert "vila_sample_finalize" in _lib.SIGNATURES and hasattr(_lib.load(), "vila_sample_finalize")
    assert "vila_sample_finalize" in (ROOT / "vila_b200" / "csrc" / "api.cu").read_text()


def test_struct_matches_header():
    text = (ROOT / "include" / "vila_b200.h").read_text()
    body = re.search(r"typedef struct vila_sample_finalize_params \{(.*?)\} vila_sample_finalize_params;", text,
                     flags=re.S).group(1)
    decls = []  # (name, is_pointer)
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        names = [n.strip() for n in decl.split(",")]
        first = names[0].split()[-1]
        ptr = "*" in decl.split(",")[0]
        decls.append((first.lstrip("*"), ptr))
        decls.extend((n.lstrip("*"), n.startswith("*")) for n in names[1:])
    assert [n for n, _ in decls] == [f[0] for f in _lib.SampleFinalizeParams._fields_] == FIELDS
    # C layout: pointers 8 bytes, int32_t 4, natural alignment
    off = 0
    for (name, ptr), (fname, ftype) in zip(decls, _lib.SampleFinalizeParams._fields_):
        size = 8 if ptr else 4
        off = (off + size - 1) // size * size
        assert getattr(_lib.SampleFinalizeParams, fname).offset == off and C.sizeof(ftype) == size, name
        off += size
    assert C.sizeof(_lib.SampleFinalizeParams) == (off + 7) // 8 * 8


def _valid():
    p = _lib.SampleFinalizeParams()
    for i, name in enumerate(FIELDS[:11]):  # distinct 256-byte-aligned stand-in addresses, never dereferenced
        setattr(p, name, 0x10000 + 0x100 * i)
    p.V, p.hidden = 152064, 3584
    return p


def _rejected(p, match):
    lib = _lib.load()
    rc = lib.vila_sample_finalize(p, None)
    msg = lib.vila_last_error().decode()
    assert rc != 0 and match in msg, (rc, msg)


def test_rejections_before_any_device_call():
    lib = _lib.load()
    assert lib.vila_sample_finalize(None, None) != 0 and b"params are required" in lib.vila_last_error()
    for name in ("logits", "inv_temperature", "top_k", "top_p", "seed", "step", "token_out"):
        p = _valid()
        setattr(p, name, None)
        _rejected(p, "required")
    for V in (0, -1, 8 * 40960 + 1):
        p = _valid()
        p.V = V
        _rejected(p, "vocabulary size")
    for name, off in (("logits", 1), ("inv_temperature", 2), ("seed", 4), ("step", 2), ("token_out", 2),
                      ("token_hist", 2), ("position", 1), ("embed_table", 8), ("x_next", 8)):
        p = _valid()
        setattr(p, name, getattr(p, name) + off)
        _rejected(p, "misaligned")
    p = _valid()
    p.x_next = None
    _rejected(p, "go together")
    p = _valid()
    p.hidden = 12
    _rejected(p, "multiple of 8")


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_valid_arguments_fail_loudly_without_gpu():
    p = _valid()
    _rejected(p, "no CUDA device")
    p.token_hist = p.position = p.embed_table = p.x_next = None  # the optional pointers
    p.hidden = 0
    _rejected(p, "no CUDA device")


def test_ops_sample_finalize_rejections():
    from vila_b200 import ops
    z = dict(logits=torch.zeros(100, dtype=torch.bfloat16), inv_temperature=torch.zeros(1),
             top_k=torch.zeros(1, dtype=torch.int32), top_p=torch.ones(1), seed=torch.zeros(1, dtype=torch.int64),
             step=torch.zeros(1, dtype=torch.int32), token_out=torch.zeros(1, dtype=torch.int32))
    with pytest.raises(ValueError, match="bfloat16"):
        ops.sample_finalize(**{**z, "logits": torch.zeros(100)})
    with pytest.raises(ValueError, match=r"\[V\]"):
        ops.sample_finalize(**{**z, "logits": torch.zeros(2, 100, dtype=torch.bfloat16)})
    with pytest.raises(ValueError, match="int32"):
        ops.sample_finalize(**{**z, "step": torch.zeros(1, dtype=torch.int64)})
    with pytest.raises(ValueError, match="single value"):
        ops.sample_finalize(**{**z, "top_p": torch.ones(2)})
    with pytest.raises(ValueError, match="together"):
        ops.sample_finalize(**z, embed_table=torch.zeros(100, 64, dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.sample_finalize(**z)


# ------------------------------------------------------------------------------------------------
# generate / streaming routing with stand-in decoders
# ------------------------------------------------------------------------------------------------
class _StandInLLM:
    """Qwen2ForCausalLM's host surface for generate / stream_tokens: token i of a greedy run is 100 + i, of a
    sampled run 200 + i; every call is recorded"""

    def __init__(self, generation_config=None):
        self.generation_config = generation_config
        self.device = torch.device("cpu")
        self.calls = []
        self.dec = _StandInDecoder(self.calls)

    def _generate_greedy(self, emb, max_new, eos_ids, check_every=16, sp_runner=None, sampling=None):
        self.calls.append(("graph", emb.shape[0], sampling))
        base = 100 if sampling is None or sampling.greedy else 200
        return [base + i for i in range(max_new)]

    def _generate_eager(self, emb, max_new, eos_ids, sample, processors, temperature, top_p, top_k):
        self.calls.append(("eager", emb.shape[0], (sample, temperature, top_p, top_k)))
        return [7] * max_new

    def decoder(self, n):
        return self.dec

    def prefill_hidden_graphed(self, emb, cache):
        return emb

    stream_tokens = Qwen2ForCausalLM.stream_tokens


class _StandInDecoder:
    def __init__(self, calls):
        self.calls = calls

    def cache_for(self, n):
        return "cache"

    def start(self, last_hidden, cache, params=None, *, logprobs=None, penalties=None):
        self.calls.append(("start", params))
        self.base = 100 if params is None or params.greedy else 200

    def run(self, n):
        pass

    def read(self, n, start=0):
        return lambda: ([self.base + i for i in range(start, n)], None)


def _generate(llm, **kw):
    return Qwen2ForCausalLM.generate(llm, torch.zeros(kw.pop("rows", 1), 5, 8), max_new_tokens=4, eos_token_id=None,
                                     **kw)


def test_generate_routes_sampling_to_the_graph_decoder():
    llm = _StandInLLM()
    out = _generate(llm, do_sample=True, temperature=0.7, top_p=0.9, rows=2)
    assert out.tolist() == [[200, 201, 202, 203]] * 2
    assert [c[0] for c in llm.calls] == ["graph", "graph"]
    for _, S, p in llm.calls:
        assert S == 5 and (p.temperature, p.top_k, p.top_p) == (0.7, 0, 0.9) and p.seed is not None
    assert llm.calls[0][2].seed != llm.calls[1][2].seed  # each row its own seed
    # logits processors keep the eager path exactly as before
    llm = _StandInLLM()
    proc = [lambda ids, lg: lg]
    out = _generate(llm, do_sample=True, temperature=0.7, top_p=0.9, logits_processor=proc)
    assert out.tolist() == [[7] * 4] and llm.calls == [("eager", 5, (True, 0.7, 0.9, 0))]
    # greedy stays greedy
    llm = _StandInLLM()
    assert _generate(llm).tolist() == [[100, 101, 102, 103]] and llm.calls == [("graph", 5, None)]
    # sequence-parallel sampling is still refused
    with pytest.raises(NotImplementedError):
        _generate(_StandInLLM(), do_sample=True, sp_runner=object())


def test_generate_parameters_come_from_the_config():
    hf_like = SimpleNamespace(do_sample=True, temperature=0.6, top_k=50, top_p=0.95, max_new_tokens=4)
    llm = _StandInLLM(hf_like)
    _generate(llm)
    p = llm.calls[0][2]
    assert (p.temperature, p.top_k, p.top_p) == (0.6, 50, 0.95)  # HF's default GenerationConfig has top_k 50
    llm = _StandInLLM(hf_like)
    _generate(llm, top_k=0, temperature=1.5)  # explicit kwargs first
    assert (llm.calls[0][2].temperature, llm.calls[0][2].top_k, llm.calls[0][2].top_p) == (1.5, 0, 0.95)
    with pytest.raises(ValueError):
        _generate(_StandInLLM(), do_sample=True, top_p=0.0)


def test_row_seeds_replay_and_a_config_seed_wins():
    def seeds(gc=None, **kw):
        llm = _StandInLLM(gc)
        _generate(llm, do_sample=True, temperature=0.8, rows=3, **kw)
        return [c[2].seed for c in llm.calls]

    torch.manual_seed(5)
    a = seeds()
    torch.manual_seed(5)
    assert seeds() == a and len(set(a)) == 3
    torch.manual_seed(5)
    # the draw of serving.sampling_for_requests, in row order
    assert a == [int(torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64)) for _ in range(3)]
    assert seeds(SimpleNamespace(seed=42)) == [42, 42, 42]
    state = torch.get_rng_state()
    assert sampling_for_generate(SimpleNamespace(seed=7, temperature=0.5), 1)[0] == SamplingParams(0.5, 0, 1.0, 7)
    assert torch.equal(torch.get_rng_state(), state)  # a config seed draws nothing


def test_stream_tokens_starts_the_decoder_with_the_parameters():
    llm = _StandInLLM()
    gc = SimpleNamespace(eos_token_id=None)
    p = SamplingParams(0.9, top_p=0.8, seed=3)
    chunks = list(Qwen2ForCausalLM.stream_tokens(llm, torch.zeros(5, 8), gc, chunk_tokens=3, max_new_tokens=7,
                                                 sampling=p))
    assert chunks == [[200, 201, 202], [203, 204, 205], [206]] and llm.calls == [("start", p)]
    llm = _StandInLLM()
    chunks = list(Qwen2ForCausalLM.stream_greedy(llm, torch.zeros(5, 8), SimpleNamespace(eos_token_id=[102]),
                                                 chunk_tokens=2, max_new_tokens=7))
    assert chunks == [[100, 101], [102]] and llm.calls == [("start", None)]
    with pytest.raises(ValueError, match="seed"):
        list(Qwen2ForCausalLM.stream_tokens(_StandInLLM(), torch.zeros(5, 8), gc, sampling=SamplingParams(1.0)))


# ------------------------------------------------------------------------------------------------
# server
# ------------------------------------------------------------------------------------------------
def _server_stub(configs):
    class Tok:
        def decode(self, ids, skip_special_tokens=True):
            return " ".join(str(i) for i in ids)

    class Stub:
        tokenizer = Tok()
        # a checkpoint config that asks for sampling: streamed requests must not inherit it without --sample
        default_generation_config = SimpleNamespace(max_new_tokens=None, do_sample=True, temperature=1.0, top_k=50,
                                                    top_p=1.0)

        def generate_content(self, prompt, generation_config=None, response_format=None, stream=False):
            configs.append(generation_config)
            return iter(["a", "b"]) if stream else "single"

        def _prepare_content(self, prompt):
            return torch.tensor([[1, 2]]), None, {}

        def generate_batch(self, requests, max_new_tokens=128, slots=8, **kw):
            return [[7, 8, 9] for _ in requests]

    return Stub()


def test_server_streams_sampled_under_the_flag():
    from vila_b200 import server as S

    def req(**kw):
        return S.ChatCompletionRequest(model="m", max_tokens=5, stream=True,
                                       messages=[S.ChatMessage(role="user", content="hi")], **kw)

    async def drain(eng, r):
        return [c async for c in eng.stream(r)]

    configs = []
    stub = _server_stub(configs)
    eng = S.Engine(stub, "m", sample=True)
    assert len(asyncio.run(drain(eng, req(temperature=0.9, top_p=0.8, seed=42)))) == 3
    gc = configs[-1]
    assert (gc.do_sample, gc.temperature, gc.top_p, gc.top_k, gc.seed, gc.max_new_tokens) == (True, 0.9, 0.8, 0, 42, 5)
    assert stub.default_generation_config.top_k == 50  # a copy was changed, not the model's config
    asyncio.run(drain(eng, req()))  # the request defaults: temperature 0.2, top_p 0.9, no seed
    gc = configs[-1]
    assert (gc.do_sample, gc.temperature, gc.top_p, gc.top_k, gc.seed) == (True, 0.2, 0.9, 0, None)
    asyncio.run(drain(eng, req(temperature=0.0)))
    assert configs[-1].do_sample is False
    # an invalid top_p fails that request only
    n = len(configs)
    with pytest.raises(ValueError):
        asyncio.run(drain(eng, req(top_p=0.0)))
    assert len(configs) == n
    assert len(asyncio.run(drain(eng, req(seed=1)))) == 3 and configs[-1].seed == 1
    # without --sample: greedy, whatever the checkpoint's config says
    configs.clear()
    eng = S.Engine(_server_stub(configs), "m")
    asyncio.run(drain(eng, req(temperature=0.9, top_p=0.0)))
    assert configs[-1].do_sample is False and configs[-1].max_new_tokens == 5
