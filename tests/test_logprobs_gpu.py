"""GPU: vila_token_logprobs against the fp64 rule of vila_b200/logprobs.py, and logprobs in the continuous-batching
engine.

  * kernel: at V in {152064, 1003, 37} and M in {1, 8, 32}, n in {0, 5, 20}, on random rows, rows of few distinct
    values (tied maxima, ties across the n-th place) and a wide-range row: top ids equal the rule's, values are within
    1e-5 + 1e-6 |lp| of the rule in fp64, the chosen token's value equals its entry in top bit for bit, idle rows and
    other columns are untouched, the column is min(step, cols - 1), and a row's bits do not change with M, its index
    or its neighbours;
  * engine: ids with logprobs=5 equal ids without, for bf16 / fp8 / w4a16 weights x bf16 / fp8 K/V x greedy /
    sampled, and with prefix caching; entry 0 is the kernel's result on the admission logits, bit for bit; a greedy
    slot's top-1 id is its chosen id; the chosen logprob matches the fp32 oracle's log_softmax fed the engine's own ids
    within twice the greedy engines' logit bound (3 bf16 ulps at the logit scale, test_decode_engines_gpu), since a
    log-probability moves by at most twice the largest logit error; LlavaLlamaModel.generate_batch(logprobs=3) end to
    end.
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

pytestmark = pytest.mark.gpu

ATOL, RTOL = 1e-5, 1e-6


def _rows(M, V, seed):
    """random rows at several scales, rows of few distinct values (ties at the maximum and across the n-th place) and
    a wide-range row"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(M, V, device="cuda", generator=g) * torch.linspace(0.5, 8, M, device="cuda")[:, None]
    for r in range(1, M, 3):
        x[r] = torch.round(x[r] / 4)  # a handful of values, each repeated many times
    if M > 2:
        x[2] = torch.randn(V, device="cuda", generator=g) * 200
        x[2, V // 3] = 1e4
    return x.to(torch.bfloat16)


def _launch(logits, tokens, step, pos, cols, n):
    M = logits.shape[0]
    lp = torch.full((M, cols), -7.0, device="cuda")
    ids = torch.full((M, cols, n), -7, dtype=torch.int32, device="cuda")
    top = torch.full((M, cols, n), -7.0, device="cuda")
    _ops().token_logprobs(logits, tokens, step, pos, lp_hist=lp, top_ids=ids if n else None, top_lp=top if n else None)
    torch.cuda.synchronize()
    return lp, ids, top


@pytest.mark.parametrize("V", [152064, 1003, 37])
def test_kernel_against_the_fp64_rule(cuda, V):
    from vila_b200.logprobs import reference_logprobs
    worst, rows_checked = 0.0, 0
    for M in (1, 8, 32):
        for n in (0, 5, 20):
            logits = _rows(M, V, seed=V + M + n)
            g = torch.Generator(device="cuda").manual_seed(M * 7 + n)
            tokens = torch.randint(0, V, (M,), device="cuda", generator=g)
            tokens[0] = int(torch.argmax(logits[0].float()))  # a chosen token that is in top
            cols = 6
            step = torch.randint(0, cols + 3, (M,), device="cuda", generator=g)  # >= cols: the last column
            pos = torch.arange(M, dtype=torch.int32, device="cuda")
            if M > 1:
                pos[M // 2] = -1  # idle
            lp, ids, top = _launch(logits, tokens, step, pos, cols, n)
            for m in range(M):
                c = min(int(step[m]), cols - 1)
                others = [k for k in range(cols) if k != c or int(pos[m]) < 0]
                assert bool((lp[m, others] == -7.0).all()) and bool((ids[m, others] == -7).all())
                if int(pos[m]) < 0:
                    continue
                want_lp, want_ids, want_top = reference_logprobs(logits[m], int(tokens[m]), n)
                assert ids[m, c].tolist() == want_ids.tolist(), f"V={V} M={M} n={n} row {m}"
                got = np.array([lp[m, c].item()] + top[m, c].tolist(), dtype=np.float64)
                want = np.concatenate([[want_lp], want_top])
                err = np.abs(got - want)
                assert bool((err <= ATOL + RTOL * np.abs(want)).all()), f"V={V} M={M} n={n} row {m}: {err.max()}"
                worst = max(worst, float(err.max()))
                if int(tokens[m]) in want_ids.tolist():
                    j = want_ids.tolist().index(int(tokens[m]))
                    assert lp[m, c].view(torch.int32).item() == top[m, c, j].view(torch.int32).item()
                rows_checked += 1
    _record({"name": f"token_logprobs V={V}", "rows": rows_checked, "worst_abs_err": worst, "ok": True})


def test_kernel_bits_do_not_depend_on_the_batch(cuda):
    V, n, cols = 152064, 20, 4
    logits = _rows(32, V, seed=11)
    tokens = torch.randint(0, V, (32,), device="cuda")
    step = torch.full((32,), 2, dtype=torch.int64, device="cuda")
    pos = torch.zeros(32, dtype=torch.int32, device="cuda")
    full = _launch(logits, tokens, step, pos, cols, n)
    again = _launch(logits, tokens, step, pos, cols, n)
    for a, b in zip(full, again):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    for r in (0, 1, 2, 17, 31):
        one = _launch(logits[r:r + 1].clone(), tokens[r:r + 1], step[:1], pos[:1], cols, n)
        # the row at index 5 of an 8-row batch, among rows scaled by 1e3 (other maxima and sums)
        other = torch.randn(8, V, device="cuda").mul(1e3).to(torch.bfloat16)
        other[5] = logits[r]
        tok8 = torch.randint(0, V, (8,), device="cuda")
        tok8[5] = tokens[r]
        eight = _launch(other, tok8, step[:8], pos[:8], cols, n)
        for a, b, c in zip(full, one, eight):
            assert torch.equal(a[r].view(torch.int32), b[0].view(torch.int32))
            assert torch.equal(a[r].view(torch.int32), c[5].view(torch.int32))


# ------------------------------------------------------------------------------------------------
# engine
# ------------------------------------------------------------------------------------------------
COMBOS = [(w, kv, s) for w in ("bf16", "fp8", "w4a16") for kv in ("bf16", "fp8") for s in (False, True)]


@pytest.mark.parametrize("weights,kv,sampled", COMBOS,
                         ids=[f"{w}-{kv}-{'sampled' if s else 'greedy'}" for w, kv, s in COMBOS])
def test_engine_ids_unchanged_by_logprobs(cuda, weights, kv, sampled):
    from vila_b200 import serving
    from vila_b200.sampling import SamplingParams
    model = (T8 if weights == "fp8" else T4)._model("tiny")[0]
    llm = model.llm
    prompts = [_prompt(llm, S, seed=S) for S in (120, 333, 57, 410)]
    sampling = [SamplingParams(0.8, top_k=40, top_p=0.9, seed=i + 1) for i in range(4)] if sampled else None
    with torch.inference_mode():
        llm.set_decode_weights(weights)
        try:
            plain = serving.generate_batch(llm, prompts, max_new_tokens=20, slots=3, kv_cache=kv, sampling=sampling)
            ids, lps = serving.generate_batch(llm, prompts, max_new_tokens=20, slots=3, kv_cache=kv, sampling=sampling,
                                              logprobs=5)
        finally:
            llm.set_decode_weights("bf16")
            if weights == "fp8":
                T8._release()
    assert ids == plain
    for r, row in enumerate(lps):
        assert [e.token for e in row] == ids[r] and all(len(e.top) == 5 for e in row)
        assert all(e.logprob <= 0 and all(v <= 0 for _, v in e.top) for e in row)
        assert all(e.top[j][1] >= e.top[j + 1][1] for e in row for j in range(4))
        if not sampled:
            assert all(e.top[0][0] == e.token for e in row)  # greedy: top-1 is the chosen id


def test_engine_ids_unchanged_by_logprobs_with_prefix_cache(cuda):
    from vila_b200 import serving
    llm = _model("tiny")[0].llm
    shared = _prompt(llm, 300, seed=1)
    prompts = [torch.cat([shared, _prompt(llm, n, seed=n)]) for n in (20, 45, 7)] + [_prompt(llm, 200, seed=9)]
    with torch.inference_mode():
        plain = serving.generate_batch(llm, prompts, 12, slots=2, max_tokens_per_slot=1024, prefix_cache=True)
        ids, lps = serving.generate_batch(llm, prompts, 12, slots=2, max_tokens_per_slot=1024, prefix_cache=True,
                                          logprobs=5)
    assert ids == plain and [[e.token for e in r] for r in lps] == ids


@pytest.mark.parametrize("kind", ["tiny", "8b-shallow"])
def test_engine_logprobs_against_the_oracle(cuda, kind, monkeypatch):
    """entry 0 is the kernel on the admission logits (bit for bit) and the rule on them; every chosen logprob is the
    fp32 oracle's log_softmax on the engine's own ids within twice the greedy engines' logit bound"""
    from vila_b200 import ops, serving
    from vila_b200.logprobs import reference_logprobs
    model, o32, _ = _model(kind)
    llm = model.llm
    admitted = []
    orig = llm.logits_from_hidden

    def spy(h):
        out = orig(h)
        admitted.append(out.clone())
        return out

    monkeypatch.setattr(llm, "logits_from_hidden", spy)
    lens = (250, 700, 90)
    prompts = [_prompt(llm, S, seed=S) for S in lens]
    n = 16
    with torch.inference_mode():
        dec = serving.BatchedDecoder(llm, slots=4, max_tokens_per_slot=2048, max_new=n + 8, logprobs=5)
        dec.capture()
        for s, emb in zip((0, 1, 3), prompts):  # slot 2 stays idle
            dec.admit(s, emb)
        dec.run(n - 1)
        assert dec.launches_per_step == 7 * llm.config.num_hidden_layers + 3
        got = {s: dec.generated_logprobs(s) for s in (0, 1, 3)}
        assert dec.generated(2) == [] and float(dec.lp_hist[2].abs().sum()) == 0.0
        for k, s in enumerate((0, 1, 3)):
            row = admitted[k]
            e0 = got[s][0]
            tok = torch.tensor([e0.token], dtype=torch.int64, device="cuda")
            lp = torch.zeros(1, 1, device="cuda")
            ids = torch.zeros(1, 1, 5, dtype=torch.int32, device="cuda")
            top = torch.zeros(1, 1, 5, device="cuda")
            ops.token_logprobs(row, tok, torch.zeros(1, dtype=torch.int64, device="cuda"),
                               torch.zeros(1, dtype=torch.int32, device="cuda"), lp_hist=lp, top_ids=ids, top_lp=top)
            assert e0.logprob == lp.item() and e0.top == list(zip(ids[0, 0].tolist(), top[0, 0].tolist()))
            want_lp, want_ids, want_top = reference_logprobs(row[0], e0.token, 5)
            assert [i for i, _ in e0.top] == want_ids.tolist()
            assert abs(e0.logprob - want_lp) <= ATOL + RTOL * abs(want_lp)
    worst = 0.0
    for s, emb in zip((0, 1, 3), prompts):
        ids = [e.token for e in got[s]]
        assert len(ids) == n and all(e.top[0][0] == e.token for e in got[s])  # greedy
        with torch.no_grad():
            truth, _ = _teacher_forced(o32, emb, ids)
        ref = torch.log_softmax(truth.double(), dim=-1)
        bound = 2 * 3 * 2 ** -8 * truth.abs().max().item()
        for t, e in enumerate(got[s]):
            err = abs(e.logprob - ref[t, e.token].item())
            worst = max(worst, err)
            assert err <= bound, f"{kind} slot {s} step {t}: {e.logprob} vs oracle {ref[t, e.token].item()} ({bound})"
    _record({"name": f"engine logprobs vs fp32 oracle {kind}", "worst_abs_err": worst, "ok": True})


def test_llava_generate_batch_logprobs_end_to_end(cuda):
    from tests.test_model_gpu import build, synth_inputs
    from vila_b200.model import tiny_test_config
    cfg = tiny_test_config(llm_layers=3)
    model = build(cfg, seed=15)
    reqs = []
    for i, n_text in enumerate([5, 12, 3]):
        ids, images = synth_inputs(cfg, n_images=1 if i % 2 == 0 else 0, n_text=n_text, seed=20 + i)
        reqs.append({"input_ids": ids, "media": {"image": [im.cuda() for im in images]} if images else None})
    plain = model.generate_batch(reqs, max_new_tokens=10, slots=2, max_tokens_per_slot=256, eos_token_id=[])
    ids, lps = model.generate_batch(reqs, max_new_tokens=10, slots=2, max_tokens_per_slot=256, eos_token_id=[],
                                    logprobs=3)
    assert ids == plain and all(len(r) == 10 for r in lps)
    for r, row in enumerate(lps):
        assert [e.token for e in row] == ids[r]
        assert all(len(e.top) == 3 and e.top[0][0] == e.token and e.top[0][1] == e.logprob for e in row)
    eos = ids[0][3]
    cut, cut_lp = model.generate_batch(reqs[:1], max_new_tokens=10, slots=2, max_tokens_per_slot=256,
                                       eos_token_id=[eos], logprobs=3)
    assert cut[0] == ids[0][:ids[0].index(eos) + 1] and [e.token for e in cut_lp[0]] == cut[0]
