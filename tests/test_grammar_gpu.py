"""GPU: grammar-constrained decoding in the single-stream graph decoder.

  * vila_apply_token_bitmask_row bit for bit against vila_b200/grammar.py at V in {152064, 151936, 1003, 37}: masks of
    all ones (output = input), a single bit, random densities and bits beyond V; rows holding -inf; in place, out of
    place and on rows that are not 16-byte aligned; the same bits across replays of a captured graph;
  * vila_sample_finalize on masked rows (-inf entries): top-k above the allowed count, top-p, and rows whose allowed
    logits all equal the row's minimum choose an allowed id, the rule's;
  * GraphDecoder with a grammar for bf16 / fp8 / w4a16 weights x greedy / sampled, and on a split-KV prompt: every
    step's id is the rule's choice on that step's recorded raw row and mask, and allowed; an all-allowing matcher gives
    the unconstrained ids; chunk_tokens 1 and 8 agree; penalties and logprobs combine, the entries being the raw row's;
    an all-zero mask is a ValueError before the step; unconstrained requests keep their graphs, launches and ids;
  * end to end: generate_content (streamed and not) and stream_content with response_format on the tiny model and a
    toy-vocabulary compiler: the ids, mapped through the vocabulary, are JSON that satisfies the schema whenever the
    grammar terminated.
"""
import json

import numpy as np
import pytest
import torch

from tests import test_fp8_decode_gpu as T8
from tests import test_w4a16_decode_gpu as T4
from tests.grammar_support import PyMatcher, Recorder, allow_all, pack, random_subsets, toy_compiler
from tests.helpers import _record
from tests.test_decode_engines_gpu import _model, _prompt
from tests.test_kernels_gpu import _ops
from tests.test_stream_logprobs_gpu import _row_launch
from vila_b200.grammar import allowed_ids, bitmask_words, reference_masked

pytestmark = pytest.mark.gpu

VOCABS = [152064, 151936, 1003, 37]


def _masks(V, g):
    W = bitmask_words(V)
    out = {"ones": np.full(W, -1, dtype=np.int32)}
    one = np.zeros(V, dtype=bool)
    one[V // 3] = True
    out["single"] = pack(one, W)
    for d in (0.5, 0.02):
        out[f"density {d}"] = pack(g.random(V) < d, W)
    beyond = pack(g.random(V) < 0.3, W)
    if V % 32:
        beyond[-1] |= np.int32(-1 << (V % 32))
    out["bits beyond V"] = beyond
    return out


@pytest.mark.parametrize("V", VOCABS)
def test_kernel_bit_exact(cuda, V):
    ops = _ops()
    g = np.random.default_rng(V)
    gen = torch.Generator(device="cuda").manual_seed(V)
    row = (torch.randn(V, device="cuda", generator=gen) * 5).to(torch.bfloat16)
    row[::53] = float("-inf")
    cases = 0
    for name, w in _masks(V, g).items():
        mask = torch.from_numpy(w).cuda()
        want = reference_masked(row, w).view(torch.int16)
        out = torch.full((V,), 3.0, dtype=torch.bfloat16, device="cuda")
        ops.apply_token_bitmask_row(row, mask, out=out)
        assert torch.equal(out.cpu().view(torch.int16), want), f"V={V} {name}"
        if name == "ones":
            assert torch.equal(out.view(torch.int16), row.view(torch.int16))
        inplace = row.clone()
        ops.apply_token_bitmask_row(inplace, mask, out=inplace)
        assert torch.equal(inplace.cpu().view(torch.int16), want), f"V={V} {name} in place"
        # rows at a 2-byte offset: the element-wise path
        buf = torch.zeros(2 * V + 8, dtype=torch.bfloat16, device="cuda")
        src, dst = buf[1:V + 1], buf[V + 3:2 * V + 3]
        src.copy_(row)
        ops.apply_token_bitmask_row(src, mask, out=dst)
        assert torch.equal(dst.cpu().view(torch.int16), want), f"V={V} {name} unaligned"
        cases += 3
    # a captured graph gives the same bits on every replay
    w = _masks(V, g)["density 0.5"]
    mask = torch.from_numpy(w).cuda()
    out = torch.zeros(V, dtype=torch.bfloat16, device="cuda")
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.apply_token_bitmask_row(row, mask, out=out)
    for _ in range(3):
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out.cpu().view(torch.int16), reference_masked(row, w).view(torch.int16))
    _record({"name": f"apply_token_bitmask_row V={V}", "cases": cases, "ok": True})


def _finalize(row, inv_t, top_k, top_p, seed, t):
    ops = _ops()
    dev = dict(device="cuda")
    tok = torch.zeros(1, dtype=torch.int32, **dev)
    ops.sample_finalize(row, torch.tensor([inv_t], **dev), torch.tensor([top_k], dtype=torch.int32, **dev),
                        torch.tensor([top_p], **dev), torch.tensor([seed], dtype=torch.int64, **dev),
                        torch.tensor([t], dtype=torch.int32, **dev), tok)
    return int(tok.item())


def test_sample_finalize_on_masked_rows(cuda):
    from vila_b200.sampling import reference_draw
    ops = _ops()
    V = 152064
    g = np.random.default_rng(2)
    gen = torch.Generator(device="cuda").manual_seed(2)
    raw = (torch.randn(V, device="cuda", generator=gen) * 3).to(torch.bfloat16)
    few = np.zeros(V, dtype=bool)
    few[g.choice(V, 12, replace=False)] = True
    lowest = raw.clone()
    lowest[torch.from_numpy(few).cuda()] = raw.min()  # the allowed logits all equal the row's minimum
    checked = 0
    for base in (raw, lowest):
        for allowed in (few, g.random(V) < 0.01):
            mask = torch.from_numpy(pack(allowed, bitmask_words(V))).cuda()
            row = torch.empty_like(base)
            ops.apply_token_bitmask_row(base, mask, out=row)
            for inv_t, top_k, top_p in ((0.0, 0, 1.0), (1.0, 0, 1.0), (1.4, 50, 1.0), (1.4, 0, 0.9),
                                        (0.7, 4000, 0.95), (1.0, 5, 1.0)):
                for t in (0, 3):
                    tok = _finalize(row, inv_t, top_k, top_p, 9, t)
                    assert allowed[tok], (inv_t, top_k, top_p, t)
                    want, _, _, _ = reference_draw(row.cpu(), inv_t, top_k, top_p, 9, t)
                    assert tok == want, (inv_t, top_k, top_p, t)
                    if inv_t == 0:
                        assert tok == int(np.flatnonzero(allowed)[np.argmax(base.float().cpu().numpy()[allowed])])
                    checked += 1
    _record({"name": "sample_finalize on bitmask-masked rows", "draws": checked, "ok": True})


# ------------------------------------------------------------------------------------------------
# decoder
# ------------------------------------------------------------------------------------------------
def _gc(n, eos=None):
    return type("GC", (), dict(max_new_tokens=n, eos_token_id=eos))()


def _stream(llm, emb, n, chunk=8, sampling=None, logprobs=None, penalties=None, grammar=None):
    ids, entries = [], []
    kw = {} if grammar is None else {"grammar": grammar}
    for out in llm.stream_tokens(emb, _gc(n), chunk_tokens=chunk, sampling=sampling, logprobs=logprobs,
                                 penalties=penalties, **kw):
        if logprobs is None:
            ids += out
        else:
            ids += out[0]
            entries += out[1]
    return ids, entries


def _stepwise(llm, emb, n, matcher, sampling=None, logprobs=None, penalties=None):
    """the constrained decoder one token at a time -> (ids, entries, raw rows, penalised rows or None, masks)"""
    rec = Recorder(matcher)
    dec = llm.decoder(n)
    cache = dec.cache_for(emb.shape[0] + n)
    with torch.inference_mode():
        hid = llm.prefill_hidden_graphed(emb, cache)
        dec.start(hid[-1], cache, sampling, logprobs=logprobs, penalties=penalties, grammar=rec)
        raw = [dec.logits.clone()]
        pen = [dec.pen_logits.clone() if dec.penalised else None]
        dec.run(1)
        for _ in range(n - 1):
            dec.run(1)
            raw.append(dec.logits.clone())
            pen.append(dec.pen_logits.clone() if dec.penalised else None)
        torch.cuda.synchronize()
        assert dec.tokens(n) == dec.grammar_ids
        ids = dec.grammar_ids[:n]
        entries = dec.token_logprobs(n) if logprobs is not None else None
    return ids, entries, raw, pen, rec.masks


def _check_choices(ids, raw, pen, masks, sp, penalties=None):
    from vila_b200.penalties import reference_penalized
    from vila_b200.sampling import reference_draw, top2_gap
    checked = 0
    for t, tok in enumerate(ids):
        V = raw[t].numel()
        assert allowed_ids(masks[t], V)[tok], f"step {t}: id {tok} not allowed"
        row = raw[t].cpu()
        if penalties is not None:
            row = reference_penalized(row, ids, t, penalties.presence, penalties.frequency)
            assert torch.equal(pen[t].cpu().view(torch.int16), row.view(torch.int16))
        y = reference_masked(row, masks[t])
        if sp is None:
            assert tok == int(torch.argmax(y.float())), f"step {t}"
            checked += 1
            continue
        got, _, v, margin = reference_draw(y, sp.inv_temperature, sp.top_k, sp.top_p, sp.seed, t)
        if top2_gap(v) <= 1e-4 or margin < 1e-6:
            continue
        assert tok == got, f"step {t}"
        checked += 1
    assert checked >= 0.8 * len(ids)


DECODER_COMBOS = [(w, s) for w in ("bf16", "fp8", "w4a16") for s in (False, True)]


@pytest.mark.parametrize("weights,sampled", DECODER_COMBOS,
                         ids=[f"{w}-{'sampled' if s else 'greedy'}" for w, s in DECODER_COMBOS])
def test_decoder_chooses_by_the_rule_on_each_step(cuda, weights, sampled):
    from vila_b200.sampling import SamplingParams
    llm = (T8 if weights == "fp8" else T4)._model("tiny")[0].llm
    sp = SamplingParams(0.8, top_k=40, top_p=0.9, seed=3) if sampled else None
    n = 14
    with torch.inference_mode():
        llm.set_decode_weights(weights)
        try:
            V = llm.lm_head.weight.shape[0]
            for S in (300, 1500):  # 1500: the split-KV graphs
                emb = _prompt(llm, S, seed=S)
                ids, _, raw, pen, masks = _stepwise(llm, emb, n, random_subsets(V, seed=S, density=0.05), sp)
                assert len(ids) == n and len(masks) == n
                _check_choices(ids, raw, pen, masks, sp)
                # the streaming loop gives the same ids; so does another chunk size
                assert _stream(llm, emb, n, chunk=8, sampling=sp, grammar=random_subsets(V, S, 0.05))[0] == ids
                assert _stream(llm, emb, n, chunk=1, sampling=sp, grammar=random_subsets(V, S, 0.05))[0] == ids
                # an all-allowing matcher: the unconstrained ids
                plain, _ = _stream(llm, emb, n, sampling=sp)
                assert _stream(llm, emb, n, sampling=sp, grammar=allow_all(V))[0] == plain
        finally:
            llm.set_decode_weights("bf16")
            if weights == "fp8":
                T8._release()


@pytest.mark.parametrize("sampled", [False, True], ids=["greedy", "sampled"])
def test_decoder_grammar_with_penalties_and_logprobs(cuda, sampled):
    from vila_b200.penalties import PenaltyParams
    from vila_b200.sampling import SamplingParams
    llm = _model("tiny")[0].llm
    V = llm.lm_head.weight.shape[0]
    sp = SamplingParams(0.7, top_p=0.9, seed=5) if sampled else None
    pen = PenaltyParams(1.5, 1.0)
    emb = _prompt(llm, 280, seed=8)
    n = 12
    ids, entries, raw, rows, masks = _stepwise(llm, emb, n, random_subsets(V, 7, 0.2), sp, logprobs=4, penalties=pen)
    _check_choices(ids, raw, rows, masks, sp, penalties=pen)
    assert [e.token for e in entries] == ids
    for t, (e, row) in enumerate(zip(entries, raw)):  # the entries are those of the raw row
        lp, tid, top = _row_launch(row, e.token, 1, 1, 4)
        assert e.logprob == lp[0].item() and e.top == list(zip(tid[0].tolist(), top[0].tolist())), f"step {t}"
    a = _stream(llm, emb, n, chunk=1, sampling=sp, logprobs=4, penalties=pen, grammar=random_subsets(V, 7, 0.2))
    b = _stream(llm, emb, n, chunk=8, sampling=sp, logprobs=4, penalties=pen, grammar=random_subsets(V, 7, 0.2))
    assert a == b and a[0] == ids


def test_decoder_stops_refuses_and_leaves_unconstrained_requests_alone(cuda):
    llm = _model("tiny")[0].llm
    llm._decoder = None
    V = llm.lm_head.weight.shape[0]
    emb = _prompt(llm, 200, seed=3)
    plain, _ = _stream(llm, emb, 10)
    dec = llm._decoder
    base, graphs = dec.launches_per_step, dict(dec.graphs)
    assert dec.mask is None  # nothing allocated before a grammar
    # a matcher that allows 3 ids and stops at the 5th: the stream ends when it terminates
    stop_after = PyMatcher(V, lambda t, h: np.isin(np.arange(V), [5, 6, 7] if t < 4 else [9]), stop=(9,))
    ids, _ = _stream(llm, emb, 32, grammar=stop_after)
    assert len(ids) == 5 and set(ids[:4]) <= {5, 6, 7} and ids[4] == 9 and stop_after.is_terminated()
    assert dec.launches_per_step == base + 1
    constrained = [k for k in dec.graphs if k not in graphs]
    assert sorted(k[-1] for k in constrained) == ["body", "choose"]
    # an all-zero mask: a ValueError on the host, before the step runs
    with pytest.raises(ValueError, match="allows no token"):
        _stream(llm, emb, 8, grammar=PyMatcher(V, lambda t, h: np.zeros(V, dtype=bool)))
    late = PyMatcher(V, lambda t, h: np.ones(V, dtype=bool) if t < 3 else np.zeros(V, dtype=bool))
    with pytest.raises(ValueError, match="after 3 tokens"):
        _stream(llm, emb, 8, grammar=late)
    torch.cuda.synchronize()
    # unconstrained requests afterwards: the same graphs, launches and ids
    again, _ = _stream(llm, emb, 10)
    assert again == plain and dec.launches_per_step == base
    assert all(dec.graphs[k] is g for k, g in graphs.items()) and len(dec.graphs) == len(graphs) + 2


def test_generate_content_with_a_response_format_end_to_end(cuda):
    from types import SimpleNamespace

    from llava.model.configuration_llava import JsonSchemaResponseFormat, ResponseFormat
    from vila_b200.model import LlavaLlamaModel, tiny_test_config
    model = LlavaLlamaModel(tiny_test_config(), device="cuda").init_random(14)
    V = model.llm.lm_head.weight.shape[0]
    compiler, vocab = toy_compiler(V)
    forced, _ = toy_compiler(V, whitespace=False)  # no whitespace tokens: {"b": bool} must end within 8 tokens

    def schema(properties):
        return ResponseFormat(type="json_schema", json_schema=JsonSchemaResponseFormat(schema=json.dumps(
            {"type": "object", "properties": properties, "required": list(properties), "additionalProperties": False})))
    cases = [(compiler, ResponseFormat(type="json_object"), None),
             (compiler, schema({"a": {"type": "integer"}, "b": {"type": "boolean"}}), {"a": int, "b": bool}),
             (forced, schema({"b": {"type": "boolean"}}), {"b": bool})]
    prompt = ["Answer in JSON."]
    finished = 0
    for comp, rf, types in cases:
        model.grammar_compiler = comp
        for sample in (False, True):
            gc = SimpleNamespace(max_new_tokens=48, do_sample=sample, temperature=0.9, top_k=0, top_p=0.95, seed=7,
                                 eos_token_id=[0], pad_token_id=0, max_length=None)
            text = model.generate_content(prompt, generation_config=gc, response_format=rf)
            ids = [int(s) for s in text.split()]
            streamed = [int(s) for c in model.generate_content(prompt, generation_config=gc, response_format=rf,
                                                                stream=True) for s in c.split()]
            chunks = [i for c, _ in model.stream_content(prompt, gc, response_format=rf) for i in c]
            # the tokenizer's decode drops its EOS id 2, which the grammar allows inside strings
            assert ids == streamed == [i for i in chunks if i != 2]
            doc = "".join(vocab[i] for i in chunks if i != 0)
            if chunks and chunks[-1] == 0:  # the grammar terminated: a complete document
                value = json.loads(doc)
                if types is not None:
                    assert set(value) == set(types) and all(type(value[k]) is t for k, t in types.items()), doc
                finished += 1
            else:
                assert comp is not forced and len(chunks) == 48
    assert finished >= 2  # at least the two forced requests parsed and checked on the device's ids
    _record({"name": "generate_content response_format end to end", "finished": finished, "ok": True})
