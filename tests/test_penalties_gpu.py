"""GPU: vila_apply_penalties against the rule of vila_b200/penalties.py, and presence / frequency penalties in the
continuous-batching engine.

  * kernel: at V in {152064, 1003, 37} and M in {1, 8, 32}, with histories full of repeats and of ids outside
    [0, V), t = 0, t >= cols, strided (and misaligned) logits rows and idle rows, the output equals reference_penalized
    bit for bit; unpenalised entries are exact copies, idle output rows are untouched, and a row's bits do not change
    with M, its index or its neighbours;
  * engine, off is off: a penalties=True decoder whose requests all have 0 / 0 gives the ids of a decoder without
    penalties, for bf16 / fp8 / w4a16 weights x bf16 / fp8 K/V x greedy / sampled, and with prefix caching;
  * engine, on is right: in eager steps, the row the greedy arg-max and vila_sample_batch read is reference_penalized
    of the lm_head row over the slot's own ids, bit for bit, and the chosen id is its arg-max or reference_draw on it;
    through the step graphs, the engine's greedy ids fed to the fp32 oracle (_teacher_forced) are the arg-max of the
    fp64 rule at every step whose penalised top-2 gap exceeds the engines' logit bound plus a bf16 ulp;
  * a slot's ids do not depend on its neighbours or the slot count; with logprobs=5 the ids are unchanged and each
    chosen logprob is the oracle's raw log_softmax within test_logprobs_gpu's bound (a penalty of 1 would break it if
    the penalised row leaked into logprobs); LlavaLlamaModel.generate_batch(penalties=...) end to end.
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

SENTINEL = 0x7E7E  # bf16 bits of a value the kernel never writes in these tests (a large finite number)


def _problem(M, V, cols, seed, stride_pad=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    big = (torch.randn(M, V + stride_pad, device="cuda", generator=g) * 12).to(torch.bfloat16)
    logits = big[:, :V]
    # repeats: ids from a handful of values, from the first 64 ids, from the whole row, and ids outside [0, V)
    hist = torch.randint(0, V, (M, cols), device="cuda", generator=g)
    hist[:, ::3] = torch.randint(0, min(V, 64), (M, (cols + 2) // 3), device="cuda", generator=g)
    hist[:, 1::7] = torch.randint(0, min(V, 5), (M, (cols + 5) // 7), device="cuda", generator=g)
    hist[:, 2::11] = torch.tensor([-1, V, V + 5, -(2 ** 40)], device="cuda")[
        torch.randint(0, 4, (M, (cols + 8) // 11), device="cuda", generator=g)]
    if M > 1:
        hist[1] = V // 2  # one id, repeated cols times
    step = torch.randint(0, cols + 6, (M,), device="cuda", generator=g)  # beyond cols: every column counts
    step[0] = 0 if M > 2 else step[0]
    if M > 3:
        step[3] = cols
    pos = torch.arange(M, dtype=torch.int32, device="cuda")
    if M > 1:
        pos[M // 2] = -1  # idle
    presence = (torch.rand(M, device="cuda", generator=g) * 4 - 2)
    frequency = (torch.rand(M, device="cuda", generator=g) * 4 - 2)
    return logits, hist.contiguous(), step, pos, presence, frequency


def _launch(logits, hist, step, pos, presence, frequency):
    M, V = logits.shape
    out = torch.full((M, V), SENTINEL, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    _ops().apply_penalties(logits, hist, step, pos, presence, frequency, out=out)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("V", [152064, 1003, 37])
def test_kernel_bit_exact_against_the_rule(cuda, V):
    from vila_b200.penalties import reference_penalized
    rows, penalised = 0, 0
    for M in (1, 8, 32):
        for pad, cols in ((0, 40), (3, 40), (8, 1), (1, 300)):  # pad 3 / 1: odd row strides, rows misaligned
            logits, hist, step, pos, pres, freq = _problem(M, V, cols, seed=V + M + 7 * pad + cols, stride_pad=pad)
            out = _launch(logits, hist, step, pos, pres, freq)
            for m in range(M):
                if int(pos[m]) < 0:
                    assert bool((out[m].view(torch.int16) == SENTINEL).all()), f"idle row {m} written"
                    continue
                want = reference_penalized(logits[m], hist[m], int(step[m]), pres[m].item(), freq[m].item())
                got = out[m].cpu()
                assert torch.equal(got.view(torch.int16), want.view(torch.int16)), \
                    f"V={V} M={M} pad={pad} cols={cols} row {m} step {int(step[m])}"
                same = want.view(torch.int16) == logits[m].cpu().view(torch.int16)
                penalised += int((~same).sum())
                rows += 1
            if M > 2:
                assert torch.equal(out[0].cpu().view(torch.int16), logits[0].cpu().view(torch.int16))  # t = 0
    assert penalised > 0
    _record({"name": f"apply_penalties V={V}", "rows": rows, "entries_penalised": penalised, "ok": True})


def test_kernel_bits_do_not_depend_on_the_batch(cuda):
    V, cols = 152064, 64
    logits, hist, step, pos, pres, freq = _problem(32, V, cols, seed=5)
    pos[:] = 0
    full = _launch(logits, hist, step, pos, pres, freq)
    assert torch.equal(full.view(torch.int16), _launch(logits, hist, step, pos, pres, freq).view(torch.int16))
    for r in (0, 1, 2, 17, 31):
        one = _launch(logits[r:r + 1].clone(), hist[r:r + 1].clone(), step[r:r + 1].clone(), pos[:1],
                      pres[r:r + 1].clone(), freq[r:r + 1].clone())
        o_logits, o_hist, o_step, o_pos, o_pres, o_freq = _problem(8, V, cols, seed=100 + r)
        o_pos[:] = 0
        o_logits = o_logits.clone()
        o_logits[5], o_hist[5], o_step[5], o_pres[5], o_freq[5] = logits[r], hist[r], step[r], pres[r], freq[r]
        eight = _launch(o_logits, o_hist, o_step, o_pos, o_pres, o_freq)
        assert torch.equal(full[r].view(torch.int16), one[0].view(torch.int16))
        assert torch.equal(full[r].view(torch.int16), eight[5].view(torch.int16))


# ------------------------------------------------------------------------------------------------
# engine
# ------------------------------------------------------------------------------------------------
COMBOS = [(w, kv, s) for w in ("bf16", "fp8", "w4a16") for kv in ("bf16", "fp8") for s in (False, True)]


@pytest.mark.parametrize("weights,kv,sampled", COMBOS,
                         ids=[f"{w}-{kv}-{'sampled' if s else 'greedy'}" for w, kv, s in COMBOS])
def test_engine_off_is_off(cuda, weights, kv, sampled):
    from vila_b200 import serving
    from vila_b200.penalties import PenaltyParams
    from vila_b200.sampling import SamplingParams
    model = (T8 if weights == "fp8" else T4)._model("tiny")[0]
    llm = model.llm
    prompts = [_prompt(llm, S, seed=S) for S in (120, 333, 57, 410)]
    sampling = [SamplingParams(0.8, top_k=40, top_p=0.9, seed=i + 1) for i in range(4)] if sampled else None
    with torch.inference_mode():
        llm.set_decode_weights(weights)
        try:
            plain = serving.generate_batch(llm, prompts, max_new_tokens=20, slots=3, kv_cache=kv, sampling=sampling)
            dec = serving.BatchedDecoder(llm, slots=3, max_tokens_per_slot=2048, max_new=20, kv_cache=kv,
                                         sampling=sampled, penalties=True)
            zero = serving.generate_batch(llm, prompts, max_new_tokens=20, slots=3, kv_cache=kv, sampling=sampling,
                                          decoder=dec, penalties=[PenaltyParams(), None, PenaltyParams(0, 0), None])
            assert dec.launches_per_step == 7 * llm.config.num_hidden_layers + 3 + (1 if sampled else 0)
        finally:
            llm.set_decode_weights("bf16")
            if weights == "fp8":
                T8._release()
    assert zero == plain


def test_engine_off_is_off_with_prefix_cache(cuda):
    from vila_b200 import serving
    from vila_b200.penalties import PenaltyParams
    llm = _model("tiny")[0].llm
    shared = _prompt(llm, 300, seed=1)
    prompts = [torch.cat([shared, _prompt(llm, n, seed=n)]) for n in (20, 45, 7)] + [_prompt(llm, 200, seed=9)]
    with torch.inference_mode():
        plain = serving.generate_batch(llm, prompts, 12, slots=2, max_tokens_per_slot=1024, prefix_cache=True)
        zero = serving.generate_batch(llm, prompts, 12, slots=2, max_tokens_per_slot=1024, prefix_cache=True,
                                      penalties=PenaltyParams())
    assert zero == plain


def _record_steps(monkeypatch):
    """spies on ops.apply_penalties, ops.sample_batch and torch.argmax of eager steps: -> list of dicts per step"""
    from vila_b200 import ops
    calls = []
    orig_pen, orig_sample = ops.apply_penalties, ops.sample_batch

    def pen_spy(logits, hist, step, pos, presence, frequency, *, out):
        rec = dict(raw=logits.clone(), hist=hist.clone(), step=step.clone(), pos=pos.clone(),
                   presence=presence.clone(), frequency=frequency.clone())
        res = orig_pen(logits, hist, step, pos, presence, frequency, out=out)
        rec["pen"] = out.clone()
        rec["out_ptr"] = out.data_ptr()
        calls.append(rec)
        return res

    def sample_spy(logits, inv, k, p, seed, step, pos, *, out, n_kept=None):
        res = orig_sample(logits, inv, k, p, seed, step, pos, out=out, n_kept=n_kept)
        if calls and "read_ptr" not in calls[-1] and logits.shape[0] == calls[-1]["raw"].shape[0]:
            calls[-1].update(read_ptr=logits.data_ptr(), inv=inv.clone(), k=k.clone(), p=p.clone(), seed=seed.clone(),
                             tok=out.clone())
        return res

    monkeypatch.setattr(ops, "apply_penalties", pen_spy)
    monkeypatch.setattr(ops, "sample_batch", sample_spy)
    return calls


@pytest.mark.parametrize("sampled", [False, True], ids=["greedy", "sampled"])
def test_engine_chooses_from_the_penalised_row(cuda, sampled, monkeypatch):
    """Eager steps (the kernels the step graph replays): the row the token is chosen from is reference_penalized of
    the lm_head row over the slot's own ids, bit for bit, and the token is its arg-max (greedy) or reference_draw on it
    (sampled, where the sampler's stated margins allow)"""
    from vila_b200 import serving
    from vila_b200.penalties import PenaltyParams, reference_penalized
    from vila_b200.sampling import SamplingParams, reference_draw, top2_gap
    llm = _model("tiny")[0].llm
    calls = _record_steps(monkeypatch)
    pens = [PenaltyParams(1.0, 0.7), PenaltyParams(0.0, 2.0), PenaltyParams(-0.5, 0.3)]
    sp = [SamplingParams(0.7, top_p=0.9, seed=1), SamplingParams(0.7, top_k=50, seed=2), None]
    n = 14
    with torch.inference_mode():
        dec = serving.BatchedDecoder(llm, slots=4, max_tokens_per_slot=2048, max_new=n + 8, sampling=sampled,
                                     penalties=True)
        for s, (S, pen, p) in enumerate(zip((250, 700, 90), pens, sp)):
            if sampled:
                dec.admit(s if s < 2 else 3, _prompt(llm, S, seed=S), p, penalties=pen)  # slot 2 stays idle
            else:
                dec.admit(s if s < 2 else 3, _prompt(llm, S, seed=S), penalties=pen)
        for _ in range(n - 1):
            dec._step(None)
    assert len(calls) == n - 1
    checked, changed = 0, 0
    for c in calls:
        assert c["out_ptr"] == dec.pen_logits.data_ptr()
        if sampled:
            assert c["read_ptr"] == dec.pen_logits.data_ptr()  # the sampler reads the penalised buffer
        for m in range(4):
            if int(c["pos"][m]) < 0:
                continue
            t = int(c["step"][m])
            want = reference_penalized(c["raw"][m], c["hist"][m], t, c["presence"][m].item(), c["frequency"][m].item())
            assert torch.equal(c["pen"][m].cpu().view(torch.int16), want.view(torch.int16)), f"slot {m} t={t}"
            changed += int((want.view(torch.int16) != c["raw"][m].cpu().view(torch.int16)).sum())
            tok = dec.hist[m, t].item()
            if not sampled or c["inv"][m].item() == 0:
                assert tok == int(torch.argmax(want.float())), f"slot {m} t={t}"
                checked += 1
                continue
            got, keep, v, margin = reference_draw(want, c["inv"][m].item(), int(c["k"][m]), c["p"][m].item(),
                                                  int(c["seed"][m]), t)
            if top2_gap(v) <= 1e-4 or margin < 1e-6:
                continue
            assert tok == got, f"slot {m} t={t}: {tok} != {got}"
            checked += 1
    assert changed > 0 and checked >= 0.9 * 3 * (n - 1)
    for s in (0, 1, 3):
        assert len(dec.generated(s)) == n
    assert dec.generated(2) == []


@pytest.mark.parametrize("kind", ["tiny", "8b-shallow"])
def test_engine_greedy_penalised_ids_against_the_oracle(cuda, kind):
    """the engine's own greedy ids (step graphs) fed to the fp32 oracle: where the fp64 rule's penalised top-2 gap
    exceeds the engines' logit bound (3 bf16 ulps of the logit scale, test_decode_engines_gpu) plus a bf16 ulp of the
    penalised scale, the engine's id is the rule's arg-max"""
    from vila_b200 import serving
    from vila_b200.penalties import PenaltyParams, reference_penalized64
    model, o32, _ = _model(kind)
    llm = model.llm
    lens = (250, 700, 90)
    prompts = [_prompt(llm, S, seed=S) for S in lens]
    pens = [PenaltyParams(1.0, 0.7), PenaltyParams(0.3, 1.5), PenaltyParams(0.0, 0.4)]
    n = 24
    with torch.inference_mode():
        ids = serving.generate_batch(llm, prompts, max_new_tokens=n, slots=3, penalties=pens)
        plain = serving.generate_batch(llm, prompts, max_new_tokens=n, slots=3)
    steps, compared = 0, 0
    for r, (emb, pen) in enumerate(zip(prompts, pens)):
        assert len(ids[r]) == n
        with torch.no_grad():
            truth, _ = _teacher_forced(o32, emb, ids[r])
        bound = 3 * 2 ** -8 * truth.abs().max().item()
        for t, got in enumerate(ids[r]):
            steps += 1
            y = reference_penalized64(truth[t], ids[r], t, pen.presence, pen.frequency)
            top2 = np.partition(y, -2)[-2:]
            if top2[1] - top2[0] <= bound + 2 ** -8 * np.abs(y).max():
                continue
            compared += 1
            assert got == int(np.argmax(y)), f"{kind} request {r} step {t}: engine {got}, rule {int(np.argmax(y))}"
    _record({"name": f"penalised greedy engine vs fp32 oracle {kind}", "steps": steps, "compared": compared,
             "ok": compared >= 2 * steps / 3})
    assert compared >= 2 * steps / 3
    if kind == "tiny":  # its small vocabulary repeats ids when decoded plainly; the 8B vocabulary may not in 24 steps
        assert ids != plain


def test_engine_penalised_ids_are_slot_independent(cuda):
    from vila_b200 import serving
    from vila_b200.penalties import PenaltyParams
    from vila_b200.sampling import SamplingParams
    llm = _model("tiny")[0].llm
    lens = (120, 333, 57, 410, 260)
    prompts = [_prompt(llm, S, seed=S) for S in lens]
    pens = [PenaltyParams(1.0, 0.7), None, PenaltyParams(-0.5, 1.0), PenaltyParams(2.0, 0.0), PenaltyParams(0.0, 2.0)]
    sampling = [SamplingParams(0.7, top_p=0.9, seed=10 + i) for i in range(len(lens))]
    with torch.inference_mode():
        for sp in (None, sampling):
            runs = {slots: serving.generate_batch(llm, prompts, max_new_tokens=24, slots=slots, penalties=pens,
                                                  sampling=sp, max_tokens_per_slot=4096)
                    for slots in (1, 3, 8)}
            order = [4, 2, 0, 3, 1]
            rev = serving.generate_batch(llm, [prompts[i] for i in order], max_new_tokens=24, slots=3,
                                         penalties=[pens[i] for i in order],
                                         sampling=None if sp is None else [sp[i] for i in order],
                                         max_tokens_per_slot=4096)
            assert runs[1] == runs[3] == runs[8]
            assert [rev[order.index(i)] for i in range(len(lens))] == runs[1]


@pytest.mark.parametrize("kind", ["tiny", "8b-shallow"])
def test_engine_logprobs_stay_raw_with_penalties(cuda, kind):
    """ids with logprobs=5 equal ids without; each chosen logprob is the fp32 oracle's raw log_softmax on the engine's
    own ids within twice the greedy engines' logit bound (test_logprobs_gpu)"""
    from vila_b200 import serving
    from vila_b200.penalties import PenaltyParams
    model, o32, _ = _model(kind)
    llm = model.llm
    prompts = [_prompt(llm, S, seed=S) for S in (250, 700, 90)]
    pens = PenaltyParams(1.5, 1.0)
    n = 16
    with torch.inference_mode():
        ids = serving.generate_batch(llm, prompts, max_new_tokens=n, slots=3, penalties=pens)
        ids_lp, lps = serving.generate_batch(llm, prompts, max_new_tokens=n, slots=3, penalties=pens, logprobs=5)
    assert ids_lp == ids
    worst = 0.0
    for r, emb in enumerate(prompts):
        with torch.no_grad():
            truth, _ = _teacher_forced(o32, emb, ids[r])
        ref = torch.log_softmax(truth.double(), dim=-1)
        bound = 2 * 3 * 2 ** -8 * truth.abs().max().item()
        for t, e in enumerate(lps[r]):
            assert e.token == ids[r][t]
            err = abs(e.logprob - ref[t, e.token].item())
            worst = max(worst, err)
            assert err <= bound, f"{kind} request {r} step {t}: {e.logprob} vs raw oracle {ref[t, e.token].item()}"
    _record({"name": f"penalised engine logprobs vs raw fp32 oracle {kind}", "worst_abs_err": worst, "ok": True})


def test_llava_generate_batch_penalties_end_to_end(cuda):
    from tests.test_model_gpu import build, synth_inputs
    from vila_b200.model import tiny_test_config
    from vila_b200.penalties import PenaltyParams
    cfg = tiny_test_config(llm_layers=3)
    model = build(cfg, seed=15)
    reqs = []
    for i, n_text in enumerate([5, 12, 3]):
        ids, images = synth_inputs(cfg, n_images=1 if i % 2 == 0 else 0, n_text=n_text, seed=20 + i)
        reqs.append({"input_ids": ids, "media": {"image": [im.cuda() for im in images]} if images else None})
    plain = model.generate_batch(reqs, max_new_tokens=10, slots=2, max_tokens_per_slot=256, eos_token_id=[])
    zero = model.generate_batch(reqs, max_new_tokens=10, slots=2, max_tokens_per_slot=256, eos_token_id=[],
                                penalties=PenaltyParams())
    pen = model.generate_batch(reqs, max_new_tokens=10, slots=2, max_tokens_per_slot=256, eos_token_id=[],
                               penalties=[PenaltyParams(2.0, 2.0), None, PenaltyParams(1.0, 0.5)])
    assert zero == plain and all(len(r) == 10 for r in pen) and pen[1] == plain[1]
    # the kept prefix-caching engine is rebuilt when the penalty setting changes
    kw = dict(max_new_tokens=10, slots=2, max_tokens_per_slot=256, eos_token_id=[], prefix_cache=True)
    a = model.generate_batch(reqs, **kw)
    engine = model._prefix_engine[1]
    b = model.generate_batch(reqs, penalties=PenaltyParams(2.0, 2.0), **kw)
    assert model._prefix_engine[1] is not engine and model._prefix_engine[1].penalties
    assert a == plain and len(b) == 3
