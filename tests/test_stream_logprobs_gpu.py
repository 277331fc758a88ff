"""GPU: logprobs and presence / frequency penalties in the single-stream graph decoder.

  * vila_token_logprobs_row against the fp64 rule of vila_b200/logprobs.py at V in {152064, 151936, 1003, 37} and n in
    {0, 5, 20}, on random rows, rows of few distinct values (tied maxima, ties across the n-th place) and a wide-range
    row: top ids exact, values within 1e-5 + 1e-6 |lp|, the chosen token's value equal to its top entry bit for bit,
    the column min(step - 1, cols - 1), other columns untouched; the same bits on a second launch and across replays
    of a captured graph; top ids equal to vila_token_logprobs' at M = 1;
  * vila_apply_penalties_row bit for bit against vila_b200/penalties.py and vila_apply_penalties at M = 1;
  * GraphDecoder with logprobs: the ids of the plain decoder for bf16 / fp8 / w4a16 weights x greedy / sampled and a
    split-KV prompt; every entry is the row kernel's result on that step's logits row; a greedy step's top-1 is its id;
    the chosen logprob is the fp32 oracle's log_softmax on the decoder's own ids within twice the engines' logit bound;
  * GraphDecoder with penalties: zero penalties give the plain ids; every step's penalised row is the rule on its raw
    row bit for bit and the id is the greedy / sampled rule's choice on it; the fp32 oracle with the rule in fp64
    agrees wherever the penalised top-2 gap exceeds the bound; chunk_tokens 1 and 8 agree;
  * requests without options keep their launches and graphs; LlavaLlamaModel.stream_content end to end.
"""
import numpy as np
import pytest
import torch

from tests import test_fp8_decode_gpu as T8
from tests import test_w4a16_decode_gpu as T4
from tests.helpers import _record
from tests.test_decode_engines_gpu import _fp32_truth  # noqa: F401  (autouse: the fp32 oracle is really fp32)
from tests.test_decode_engines_gpu import _model, _prompt, _teacher_forced
from tests.test_kernels_gpu import _ops
from tests.test_logprobs_gpu import _rows

pytestmark = pytest.mark.gpu

ATOL, RTOL = 1e-5, 1e-6


def _row_launch(row, token, step, cols, n, ws=None):
    ops = _ops()
    lp = torch.full((cols,), -7.0, device="cuda")
    ids = torch.full((cols, n), -7, dtype=torch.int32, device="cuda")
    top = torch.full((cols, n), -7.0, device="cuda")
    ws, counter = ws or ops.logprobs_row_workspace(row.numel(), "cuda")
    ops.token_logprobs_row(row, torch.tensor([token], dtype=torch.int32, device="cuda"),
                           torch.tensor([step], dtype=torch.int32, device="cuda"), lp_hist=lp, workspace=ws,
                           counter=counter, top_ids=ids if n else None, top_lp=top if n else None)
    torch.cuda.synchronize()
    assert int(counter.item()) == 0  # the last CTA resets the arrival counter
    return lp, ids, top


@pytest.mark.parametrize("V", [152064, 151936, 1003, 37])
def test_row_kernel_against_the_fp64_rule(cuda, V):
    from vila_b200.logprobs import reference_logprobs
    worst, rows_checked = 0.0, 0
    for n in (0, 5, 20):
        if n > V:
            continue
        logits = _rows(6, V, seed=V + n)
        for r in range(6):
            row = logits[r].contiguous()
            token = int(torch.argmax(row.float())) if r % 2 == 0 else (r * 7919) % V
            cols = 6
            step = [0, 1, 3, 6, 9, 2][r]  # 0 and >= cols clamp
            lp, ids, top = _row_launch(row, token, step, cols, n)
            c = max(0, min(step - 1, cols - 1))
            others = [k for k in range(cols) if k != c]
            assert bool((lp[others] == -7.0).all()) and bool((ids[others] == -7).all())
            want_lp, want_ids, want_top = reference_logprobs(row, token, n)
            assert ids[c].tolist() == want_ids.tolist(), f"V={V} n={n} row {r}"
            got = np.array([lp[c].item()] + top[c].tolist(), dtype=np.float64)
            want = np.concatenate([[want_lp], want_top])
            err = np.abs(got - want)
            assert bool((err <= ATOL + RTOL * np.abs(want)).all()), f"V={V} n={n} row {r}: {err.max()}"
            worst = max(worst, float(err.max()))
            if token in want_ids.tolist():
                j = want_ids.tolist().index(token)
                assert lp[c].view(torch.int32).item() == top[c, j].view(torch.int32).item()
            # the batched kernel at M = 1: the same top ids
            if n:
                blp = torch.zeros(1, 1, device="cuda")
                bids = torch.zeros(1, 1, n, dtype=torch.int32, device="cuda")
                btop = torch.zeros(1, 1, n, device="cuda")
                _ops().token_logprobs(row[None], torch.tensor([token], device="cuda"),
                                      torch.zeros(1, dtype=torch.int64, device="cuda"),
                                      torch.zeros(1, dtype=torch.int32, device="cuda"), lp_hist=blp, top_ids=bids,
                                      top_lp=btop)
                assert bids[0, 0].tolist() == ids[c].tolist()
            rows_checked += 1
    _record({"name": f"token_logprobs_row V={V}", "rows": rows_checked, "worst_abs_err": worst, "ok": True})


def test_row_kernel_is_deterministic_across_launches_and_replays(cuda):
    ops = _ops()
    V, n, cols = 152064, 20, 4
    row = _rows(3, V, seed=5)[2].contiguous()
    first = _row_launch(row, 17, 2, cols, n)
    again = _row_launch(row, 17, 2, cols, n)
    for a, b in zip(first, again):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    lp = torch.zeros(cols, device="cuda")
    ids = torch.zeros(cols, n, dtype=torch.int32, device="cuda")
    top = torch.zeros(cols, n, device="cuda")
    ws, counter = ops.logprobs_row_workspace(V, "cuda")
    tok = torch.tensor([17], dtype=torch.int32, device="cuda")
    step = torch.tensor([2], dtype=torch.int32, device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(3):
            ops.token_logprobs_row(row, tok, step, lp_hist=lp, workspace=ws, counter=counter, top_ids=ids, top_lp=top)
    for _ in range(4):
        lp.zero_(); ids.zero_(); top.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert int(counter.item()) == 0
        for a, b in zip(first, (lp, ids, top)):
            assert torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))
    # n_used: one captured launch with row stride 20 serves every k <= 20; entries past k are not written
    k_dev = torch.tensor([0], dtype=torch.int32, device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.token_logprobs_row(row, tok, step, lp_hist=lp, workspace=ws, counter=counter, top_ids=ids, top_lp=top,
                               n_used=k_dev)
    for k in (0, 1, 5, 20, 25):
        lp.zero_(); ids.fill_(-7); top.fill_(-7.0)
        k_dev.fill_(k)
        g.replay()
        torch.cuda.synchronize()
        kk = min(k, n)
        want = _row_launch(row, 17, 2, cols, kk)
        assert lp[1].view(torch.int32).item() == want[0][1].view(torch.int32).item()
        assert torch.equal(ids[1, :kk], want[1][1]) and torch.equal(top[1, :kk].view(torch.int32),
                                                                    want[2][1].view(torch.int32))
        assert bool((ids[1, kk:] == -7).all()) and bool((top[1, kk:] == -7.0).all())


@pytest.mark.parametrize("V", [152064, 1003])
def test_penalties_row_kernel_bit_exact(cuda, V):
    from vila_b200.penalties import reference_penalized
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(V)
    row = (torch.randn(V, device="cuda", generator=g) * 6).to(torch.bfloat16)
    cols = 40
    hist = torch.randint(0, V, (cols,), device="cuda", generator=g, dtype=torch.int64)
    hist[5:15] = hist[0]  # repeats
    hist[20] = V + 3      # outside the vocabulary: ignored
    for t, p, f in ((0, 1.0, 0.5), (7, 0.5, 0.5), (25, -0.5, 2.0), (cols + 5, 2.0, -1.25)):
        pres = torch.tensor([p], device="cuda")
        freq = torch.tensor([f], device="cuda")
        out = torch.full((V,), 7.0, dtype=torch.bfloat16, device="cuda")
        ops.apply_penalties_row(row, hist.to(torch.int32), torch.tensor([t], dtype=torch.int32, device="cuda"), pres,
                                freq, out=out)
        want = reference_penalized(row, hist, t, p, f)
        assert torch.equal(out.cpu().view(torch.int16), want.view(torch.int16)), f"t={t}"
        batched = torch.zeros(1, V, dtype=torch.bfloat16, device="cuda")
        ops.apply_penalties(row[None], hist[None].contiguous(), torch.tensor([t], device="cuda"),
                            torch.zeros(1, dtype=torch.int32, device="cuda"), pres, freq, out=batched)
        assert torch.equal(batched[0].view(torch.int16), out.view(torch.int16))


# ------------------------------------------------------------------------------------------------
# decoder
# ------------------------------------------------------------------------------------------------
def _stream(llm, emb, n, chunk=8, sampling=None, logprobs=None, penalties=None):
    ids, entries = [], []
    gc = type("GC", (), dict(max_new_tokens=n, eos_token_id=None))()
    for out in llm.stream_tokens(emb, gc, chunk_tokens=chunk, sampling=sampling, logprobs=logprobs,
                                 penalties=penalties):
        if logprobs is None:
            ids += out
        else:
            ids += out[0]
            entries += out[1]
            assert [e.token for e in out[1]] == out[0]
    return ids, entries


def _stepwise(llm, emb, n, sampling=None, logprobs=None, penalties=None):
    """the decoder one token at a time: -> (ids, entries, raw rows, penalised rows) of every step"""
    dec = llm.decoder(n)
    cache = dec.cache_for(emb.shape[0] + n)
    with torch.inference_mode():
        hid = llm.prefill_hidden_graphed(emb, cache)
        dec.start(hid[-1], cache, sampling, logprobs=logprobs, penalties=penalties)
        raw = [dec.logits.clone()]
        pen = [dec.pen_logits.clone() if dec.penalised else None]
        dec.run(1)  # the first token came from start()
        for _ in range(n - 1):
            dec.run(1)
            raw.append(dec.logits.clone())
            pen.append(dec.pen_logits.clone() if dec.penalised else None)
        torch.cuda.synchronize()
        ids = dec.tokens(n)
        entries = dec.token_logprobs(n) if logprobs is not None else None
    return ids, entries, raw, pen


DECODER_COMBOS = [(w, s) for w in ("bf16", "fp8", "w4a16") for s in (False, True)]


@pytest.mark.parametrize("weights,sampled", DECODER_COMBOS,
                         ids=[f"{w}-{'sampled' if s else 'greedy'}" for w, s in DECODER_COMBOS])
def test_decoder_ids_unchanged_by_logprobs(cuda, weights, sampled):
    from vila_b200.sampling import SamplingParams
    model = (T8 if weights == "fp8" else T4)._model("tiny")[0]
    llm = model.llm
    sp = SamplingParams(0.8, top_k=40, top_p=0.9, seed=3) if sampled else None
    with torch.inference_mode():
        llm.set_decode_weights(weights)
        try:
            for S in (300, 1500):  # 1500: the split-KV graph
                emb = _prompt(llm, S, seed=S)
                plain, _ = _stream(llm, emb, 24, sampling=sp)
                ids, entries = _stream(llm, emb, 24, sampling=sp, logprobs=5)
                assert ids == plain, f"{weights} S={S}"
                assert all(len(e.top) == 5 and e.logprob <= 0 for e in entries)
                if not sampled:
                    assert all(e.top[0][0] == e.token for e in entries)
        finally:
            llm.set_decode_weights("bf16")
            if weights == "fp8":
                T8._release()


@pytest.mark.parametrize("weights,sampled", DECODER_COMBOS,
                         ids=[f"{w}-{'sampled' if s else 'greedy'}" for w, s in DECODER_COMBOS])
def test_decoder_entries_are_the_row_kernel_on_each_step(cuda, weights, sampled):
    """the row each entry was computed from is the row the token was chosen from: in greedy + logprobs the lm_head
    GEMV writes it next to its fused argmax key, in every weight mode"""
    from vila_b200.logprobs import reference_logprobs
    from vila_b200.sampling import SamplingParams
    llm = (T8 if weights == "fp8" else T4)._model("tiny")[0].llm
    sp = SamplingParams(0.7, top_p=0.9, seed=11) if sampled else None
    emb = _prompt(llm, 260, seed=4)
    n = 12
    with torch.inference_mode():
        llm.set_decode_weights(weights)
        try:
            ids, entries, raw, _ = _stepwise(llm, emb, n, sampling=sp, logprobs=5)
        finally:
            llm.set_decode_weights("bf16")
            if weights == "fp8":
                T8._release()
    assert [e.token for e in entries] == ids
    for t, (e, row) in enumerate(zip(entries, raw)):
        lp, tid, top = _row_launch(row, e.token, 1, 1, 5)
        assert e.logprob == lp[0].item() and e.top == list(zip(tid[0].tolist(), top[0].tolist())), f"step {t}"
        want_lp, want_ids, _ = reference_logprobs(row, e.token, 5)
        assert [i for i, _ in e.top] == want_ids.tolist()
        assert abs(e.logprob - want_lp) <= ATOL + RTOL * abs(want_lp)
        if not sampled:
            assert e.top[0][0] == e.token
            assert e.token == int(torch.argmax(row.float()))  # the greedy id is the arg-max of the written row


@pytest.mark.parametrize("kind", ["tiny", "8b-shallow"])
def test_decoder_logprobs_against_the_oracle(cuda, kind):
    model, o32, _ = _model(kind)
    llm = model.llm
    worst = 0.0
    for S in (250, 1100):
        emb = _prompt(llm, S, seed=S + 1)
        ids, entries = _stream(llm, emb, 16, logprobs=3)
        with torch.no_grad():
            truth, _ = _teacher_forced(o32, emb, ids)
        ref = torch.log_softmax(truth.double(), dim=-1)
        bound = 2 * 3 * 2 ** -8 * truth.abs().max().item()
        for t, e in enumerate(entries):
            err = abs(e.logprob - ref[t, e.token].item())
            worst = max(worst, err)
            assert err <= bound, f"{kind} S={S} step {t}: {e.logprob} vs {ref[t, e.token].item()} ({bound})"
    _record({"name": f"graph decoder logprobs vs fp32 oracle {kind}", "worst_abs_err": worst, "ok": True})


@pytest.mark.parametrize("sampled", [False, True], ids=["greedy", "sampled"])
def test_decoder_chooses_from_the_penalised_row(cuda, sampled):
    from vila_b200.penalties import PenaltyParams, reference_penalized
    from vila_b200.sampling import SamplingParams, reference_draw, top2_gap
    llm = _model("tiny")[0].llm
    sp = SamplingParams(0.7, top_p=0.9, seed=5) if sampled else None
    emb = _prompt(llm, 300, seed=8)
    n = 16
    pen = PenaltyParams(1.5, 1.0)
    plain, _ = _stream(llm, emb, n, sampling=sp)
    assert _stream(llm, emb, n, sampling=sp, penalties=PenaltyParams(0.0, 0.0))[0] == plain  # off is off
    ids, _, raw, rows = _stepwise(llm, emb, n, sampling=sp, penalties=pen)
    checked, changed = 0, 0
    for t in range(n):
        want = reference_penalized(raw[t], ids, t, pen.presence, pen.frequency)
        assert torch.equal(rows[t].cpu().view(torch.int16), want.view(torch.int16)), f"t={t}"
        changed += int((want.view(torch.int16) != raw[t].cpu().view(torch.int16)).sum())
        if not sampled:
            assert ids[t] == int(torch.argmax(want.float())), f"t={t}"
            checked += 1
            continue
        got, _, v, margin = reference_draw(want, sp.inv_temperature, sp.top_k, sp.top_p, sp.seed, t)
        if top2_gap(v) <= 1e-4 or margin < 1e-6:
            continue
        assert ids[t] == got, f"t={t}"
        checked += 1
    assert changed > 0 and checked >= 0.8 * n
    if not sampled:
        assert ids != plain  # the penalties changed the greedy run
    # chunk sizes do not matter
    a = _stream(llm, emb, n, chunk=1, sampling=sp, logprobs=4, penalties=pen)
    b = _stream(llm, emb, n, chunk=8, sampling=sp, logprobs=4, penalties=pen)
    assert a == b and a[0] == ids


def test_decoder_greedy_penalised_ids_against_the_oracle(cuda):
    from vila_b200.penalties import PenaltyParams, reference_penalized64
    model, o32, _ = _model("8b-shallow")
    llm = model.llm
    pen = PenaltyParams(0.5, 0.5)
    emb = _prompt(llm, 280, seed=2)
    n = 32
    ids, _ = _stream(llm, emb, n, penalties=pen)
    with torch.no_grad():
        truth, _ = _teacher_forced(o32, emb, ids)
    bound = 3 * 2 ** -8 * truth.abs().max().item() + 0.0625  # logit bound + the rule's final bf16 rounding
    compared = 0
    for t in range(n):
        y = reference_penalized64(truth[t], ids, t, pen.presence, pen.frequency)
        order = np.argsort(-y, kind="stable")
        if y[order[0]] - y[order[1]] <= 2 * bound:
            continue
        assert ids[t] == int(order[0]), f"step {t}"
        compared += 1
    assert compared >= 4  # the steps whose penalised top-2 gap exceeds twice the bound on both sides
    _record({"name": "graph decoder penalised greedy ids vs fp32 oracle", "steps": n, "compared": compared,
             "ok": True})


def test_requests_without_options_replay_their_graph(cuda):
    from vila_b200.penalties import PenaltyParams
    from vila_b200.sampling import SamplingParams
    llm = _model("tiny")[0].llm
    llm._decoder = None
    emb = _prompt(llm, 200, seed=3)
    plain, _ = _stream(llm, emb, 10)
    dec = llm._decoder
    base = dec.launches_per_step
    assert base == 5 * llm.config.num_hidden_layers + 2
    plan = (dec.num_splits, dec.split_tokens)
    assert list(dec.graphs) == [(False, False, False) + plan]
    plain_graph = dec.graphs[(False, False, False) + plan]
    assert dec.lp_hist is None and dec.pen_logits is None  # nothing allocated for the options
    _stream(llm, emb, 10, logprobs=2, penalties=PenaltyParams(0.5, 0.5))
    assert dec.launches_per_step == base + 2 and list(dec.graphs)[1:] == [(False, True, True) + plan]
    _stream(llm, emb, 10, sampling=SamplingParams(0.7, seed=1), logprobs=2)
    assert dec.launches_per_step == base + 1 and list(dec.graphs)[2:] == [(True, False, True) + plan]
    a = _stream(llm, emb, 10, logprobs=7)  # another top count: the greedy + logprobs graph is reused
    b = _stream(llm, emb, 10, logprobs=3)
    assert list(dec.graphs)[3:] == [(False, False, True) + plan] and a[0] == b[0] == plain
    assert [e.top[:3] for e in a[1]] == [e.top for e in b[1]] and all(len(e.top) == 7 for e in a[1])
    again, _ = _stream(llm, emb, 10)
    # the plain request after the option requests replays the graph it replayed first: no greedy or sampled recapture
    assert again == plain and dec.launches_per_step == base and len(dec.graphs) == 4
    assert dec.graphs[(False, False, False) + plan] is plain_graph


def test_llava_stream_content_end_to_end(cuda):
    from types import SimpleNamespace

    from vila_b200.model import LlavaLlamaModel, tiny_test_config
    from vila_b200.penalties import PenaltyParams
    model = LlavaLlamaModel(tiny_test_config(), device="cuda").init_random(14)
    prompt = ["Describe the scene."]
    for sample in (False, True):
        gc = SimpleNamespace(max_new_tokens=16, do_sample=sample, temperature=0.9, top_k=0, top_p=0.95, seed=77,
                             eos_token_id=None, pad_token_id=0, max_length=None)
        streamed = list(model.generate_content(prompt, generation_config=gc, stream=True))
        chunks = list(model.stream_content(prompt, generation_config=gc, logprobs=3))
        assert sum(len(i) for i, _ in chunks) == 16 and all([e.token for e in es] == i for i, es in chunks)
        texts = [model.tokenizer.decode(i, skip_special_tokens=True) for i, _ in chunks]
        assert " ".join(t for t in texts if t).split() == " ".join(streamed).split()
        pen = list(model.stream_content(prompt, generation_config=gc, logprobs=2, penalties=PenaltyParams(1.0, 1.0)))
        assert sum(len(i) for i, _ in pen) == 16 and all(len(e) == len(i) for i, e in pen)
        plain = list(model.stream_content(prompt, generation_config=gc))
        assert [i for i, _ in plain] == [i for i, _ in chunks] and all(e is None for _, e in plain)
