"""GPU: temperature / top-k / top-p sampling in the single-stream graph decoder (vila_sample_finalize).

  * kernel: sample_finalize gives sample_batch's token at M = 1 on every KINDS row of test_sampling_gpu, at V in
    {152064, 151936, 1003} and t in {0, 1, 2^31 - 1}; its side effects are argmax_finalize's (hist[t], step + 1,
    position + 1, x = the token's embedding row bit for bit);
  * every draw of the sampled decoder, step by step, is the rule's draw on the exact logits row it received (tiny and
    8B-shallow; bf16, fp8 and w4a16 decode weights; a prompt over 1024 tokens takes the split-KV graph path), except
    where the fp64 rule's top-2 gap is <= 1e-4 or its top-p margin < 1e-6; at least 90 % of the draws are compared;
  * teacher-forced against the fp32 oracle with test_sampling_gpu._uncertain's tolerance (two thirds compared);
  * the same ids from generate(do_sample=True), the sampled stream at chunk_tokens 1 and 8, the decoder driven
    directly and a second run, EOS cutting at the same token; greedy parameters give stream_greedy's ids; one
    sampled graph per configuration; equal launches per step in both modes; an eager sampled step calls
    sample_finalize once and neither argmax_finalize nor sample_batch;
  * LlavaLlamaModel.generate_content with a sampling config and a seed: the same text streamed and not.
"""
from types import SimpleNamespace

import pytest
import torch

from tests.helpers import _record
from tests.test_decode_engines_gpu import _fp32_truth  # noqa: F401  (autouse: the fp32 oracle is really fp32)
from tests.test_decode_engines_gpu import _model, _prompt, _teacher_forced
from tests.test_kernels_gpu import _ops
from tests.test_sampling_gpu import KINDS, _logits, _params, _uncertain

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("V", [152064, 151936, 1003])
def test_finalize_equals_sample_batch(cuda, V):
    ops = _ops()
    logits = _logits(1, V, seed=V)
    row = logits[0].contiguous()
    checked = 0
    for i, kind in enumerate(KINDS):
        prm = _params(1, seed0=i, kinds=[kind])
        for t in (0, 1, 2 ** 31 - 1):
            prm[4] = torch.tensor([t], dtype=torch.int64, device="cuda")
            out = torch.full((1,), -7, dtype=torch.int64, device="cuda")
            ops.sample_batch(row[None], *prm, torch.zeros(1, dtype=torch.int32, device="cuda"), out=out)
            step = torch.tensor([t], dtype=torch.int32, device="cuda")
            tok = torch.full((1,), -7, dtype=torch.int32, device="cuda")
            ops.sample_finalize(row, *prm[:4], step, tok)
            assert tok.item() == out.item(), f"V={V} kind {kind} t={t}: finalize {tok.item()} != batch {out.item()}"
            assert step.item() == (t + 1 if t < 2 ** 31 - 1 else -2 ** 31)
            checked += 1
    # argmax_finalize's side effects
    hidden = 256
    table = torch.randn(V, hidden, device="cuda").to(torch.bfloat16)
    for i, kind in enumerate(KINDS[:5]):
        prm = _params(1, seed0=i, kinds=[kind])
        prm[4] = torch.tensor([5], dtype=torch.int64, device="cuda")
        out = torch.zeros(1, dtype=torch.int64, device="cuda")
        ops.sample_batch(row[None], *prm, torch.zeros(1, dtype=torch.int32, device="cuda"), out=out)
        step = torch.tensor([5], dtype=torch.int32, device="cuda")
        pos = torch.tensor([100], dtype=torch.int32, device="cuda")
        hist = torch.full((8,), -1, dtype=torch.int32, device="cuda")
        tok = torch.zeros(1, dtype=torch.int32, device="cuda")
        x = torch.zeros(hidden, dtype=torch.bfloat16, device="cuda")
        ops.sample_finalize(row, *prm[:4], step, tok, hist, pos, table, x)
        t = out.item()
        assert tok.item() == t and hist.tolist() == [-1] * 5 + [t, -1, -1]
        assert step.item() == 6 and pos.item() == 101
        assert torch.equal(x.view(torch.int16), table[t].view(torch.int16))
    _record({"name": f"sample_finalize == sample_batch V={V}", "draws": checked, "ok": True})


def _draw_calls(monkeypatch):
    """spy on ops.sample_finalize: (logits, inv, k, p, seed, t, token) of every call"""
    from vila_b200 import ops
    calls, orig = [], ops.sample_finalize

    def spy(logits, inv, k, p, seed, step, token_out, *rest):
        rec = [logits.clone(), inv.item(), k.item(), p.item(), seed.item(), step.item()]
        orig(logits, inv, k, p, seed, step, token_out, *rest)
        calls.append(rec + [token_out.item()])

    monkeypatch.setattr(ops, "sample_finalize", spy)
    return calls


WEIGHTS = [(k, w) for k in ("tiny", "8b-shallow") for w in ("bf16", "fp8", "w4a16")]


@pytest.mark.parametrize("kind,weights", WEIGHTS, ids=[f"{k}-{w}" for k, w in WEIGHTS])
def test_decoder_draws_follow_the_rule_on_its_own_logits(cuda, kind, weights, monkeypatch):
    """start() and each eager decode step (the kernels the sampled graph replays) draw the rule's token on the exact
    logits row sample_finalize received, at t = 0, 1, ..."""
    from vila_b200.sampling import SamplingParams, reference_draw, top2_gap
    model = _model(kind)[0]
    llm = model.llm
    calls = _draw_calls(monkeypatch)
    n = 10
    params = [SamplingParams(0.7, top_p=0.9, seed=11), SamplingParams(0.5, top_k=50, top_p=0.9, seed=12)]
    with torch.inference_mode():
        llm.set_decode_weights(weights)
        try:
            for S, p in zip((250, 1500), params):  # 1500 > LONG_CTX: the split-KV step
                emb = _prompt(llm, S, seed=S)
                dec = llm.decoder(n)
                cache = dec.cache_for(S + n)
                assert (dec.split_tokens > 0) == (S > dec.LONG_CTX)
                dec.start(llm.prefill_hidden_graphed(emb, cache)[-1], cache, p)
                for _ in range(n - 1):
                    dec._step()
                assert dec.tokens(n) == [c[-1] for c in calls[-n:]]
        finally:
            llm.set_decode_weights("bf16")
    assert len(calls) == 2 * n
    checked = 0
    for j, (logits, inv, k, p, seed, t, tok) in enumerate(calls):
        assert t == j % n
        want, keep, v, margin = reference_draw(logits, inv, k, p, seed, t)
        if top2_gap(v) <= 1e-4 or margin < 1e-6:
            continue
        checked += 1
        assert tok == want, f"{kind} {weights}: call {j} (t={t}): {tok} != {want}"
    _record({"name": f"sampled decoder draws {kind} {weights}", "draws": len(calls), "compared": checked,
             "ok": checked >= 0.9 * len(calls)})
    assert checked >= 0.9 * len(calls)


@pytest.mark.parametrize("kind", ["tiny", "8b-shallow"])
def test_decoder_sampled_teacher_forced(cuda, kind):
    from vila_b200.sampling import SamplingParams
    model, o32, _ = _model(kind)
    llm = model.llm
    params = [SamplingParams(0.7, top_p=0.9, seed=1), SamplingParams(0.7, top_k=50, seed=2),
              SamplingParams(0.5, top_k=20, top_p=0.8, seed=3)]
    n = 24
    steps, compared, left_out = 0, 0, {"top-2 margin": 0, "kept-set membership": 0}
    for S, p in zip((250, 700, 90), params):  # test_engine_sampled_teacher_forced's requests
        emb = _prompt(llm, S, seed=S)
        with torch.inference_mode():
            ids = llm._generate_greedy(emb, n, [], sampling=p)
        with torch.no_grad():
            truth, _ = _teacher_forced(o32, emb, ids)
        tol = 3 * 2 ** -8 * truth.abs().max().item() * p.inv_temperature
        for t, got in enumerate(ids):
            steps += 1
            want, why = _uncertain(truth[t], p, t, tol)
            if why is not None:
                left_out[why] += 1
                continue
            compared += 1
            assert got == want, f"{kind} S={S} step {t}: decoder {got}, oracle draw {want}"
    _record({"name": f"sampled graph decoder teacher-forced {kind}", "steps": steps, "compared": compared,
             "left_out": left_out, "ok": compared >= 2 * steps / 3})
    assert compared >= 2 * steps / 3


def test_same_ids_and_graphs_on_every_route(cuda, monkeypatch):
    from vila_b200 import _lib, ops
    from vila_b200.sampling import SamplingParams
    model = _model("tiny")[0]
    llm = model.llm
    emb = _prompt(llm, 300, seed=300)
    n = 40
    p = SamplingParams(0.8, top_k=40, top_p=0.95, seed=1234)
    kw = dict(do_sample=True, temperature=0.8, top_k=40, top_p=0.95)

    def gen(eos):
        return llm.generate(inputs_embeds=emb[None], max_new_tokens=n, eos_token_id=eos,
                            generation_config=SimpleNamespace(seed=1234), **kw)[0].tolist()

    def stream(eos, chunk):
        gc = SimpleNamespace(eos_token_id=eos)
        return [t for c in llm.stream_tokens(emb, gc, chunk_tokens=chunk, max_new_tokens=n, sampling=p) for t in c]

    def direct():
        dec = llm.decoder(n)
        cache = dec.cache_for(300 + n)
        dec.start(llm.prefill_hidden_graphed(emb, cache)[-1], cache, p)
        dec.run(n)
        return dec.tokens(n)

    with torch.inference_mode():
        llm.set_decode_weights("bf16")  # a fresh decoder: its graphs are only this test's
        ref = gen(None)
        assert len(ref) == n and direct() == ref and gen(None) == ref
        assert stream(None, 1) == ref and stream(None, 8) == ref
        # an EOS id whose first occurrence is inside the sequence: every route stops there
        cut = next(i for i in range(5, n) if ref[i] not in ref[:i])
        eos = ref[cut]
        assert gen(eos) == stream(eos, 1) == stream(eos, 8) == ref[:cut + 1]
        # greedy parameters: exactly the greedy decoder
        greedy = list(llm.stream_greedy(emb, SimpleNamespace(eos_token_id=None), max_new_tokens=n))
        greedy = [t for c in greedy for t in c]
        assert greedy != ref
        assert stream(None, 8) == ref
        via_greedy_params = [t for c in llm.stream_tokens(emb, SimpleNamespace(eos_token_id=None), max_new_tokens=n,
                                                          sampling=SamplingParams(0.0, seed=5)) for t in c]
        assert via_greedy_params == greedy
        assert llm.generate(inputs_embeds=emb[None], max_new_tokens=n, eos_token_id=None)[0].tolist() == greedy
        # three requests with different parameters replay one sampled graph per configuration
        dec = llm.decoder(n)
        for q in (SamplingParams(1.1, seed=1), SamplingParams(0.6, top_p=0.8, seed=2),
                  SamplingParams(0.9, top_k=5, seed=3)):
            got = [t for c in llm.stream_tokens(emb, SimpleNamespace(eos_token_id=None), max_new_tokens=n,
                                                 sampling=q) for t in c]
            assert len(got) == n and got != ref
        modes = [k[:3] for k in dec.graphs]  # one greedy and one sampled graph
        assert llm.decoder(n) is dec and sorted(modes) == [(False, False, False), (True, False, False)]
        long_emb = _prompt(llm, 700, seed=700)
        list(llm.stream_tokens(long_emb, SimpleNamespace(eos_token_id=None), max_new_tokens=n, sampling=p))
        assert [k[:3] for k in dec.graphs].count((True, False, False)) == 2 and len(dec.graphs) == 3
        # launches per step and the finalize kernel of each mode
        names = {"sample_finalize": 0, "argmax_finalize": 0, "sample_batch": 0}
        for name in names:
            orig = getattr(ops, name)

            def counted(*a, _orig=orig, _name=name, **k):
                names[_name] += 1
                return _orig(*a, **k)

            monkeypatch.setattr(ops, name, counted)
        launches = {}
        for mode in (None, p):
            cache = dec.cache_for(300 + n)
            dec.start(llm.prefill_hidden_graphed(emb, cache)[-1], cache, mode)
            for k in names:
                names[k] = 0
            before = _lib.LAUNCHES
            dec._step()
            launches[mode is None] = _lib.LAUNCHES - before
            if mode is not None:
                assert names == {"sample_finalize": 1, "argmax_finalize": 0, "sample_batch": 0}
            else:
                assert names == {"sample_finalize": 0, "argmax_finalize": 1, "sample_batch": 0}
        assert launches[True] == launches[False] == dec.launches_per_step
    torch.manual_seed(99)
    with torch.inference_mode():
        a = llm.generate(inputs_embeds=emb[None], max_new_tokens=12, eos_token_id=None, **kw)
    torch.manual_seed(99)
    with torch.inference_mode():
        b = llm.generate(inputs_embeds=emb[None], max_new_tokens=12, eos_token_id=None, **kw)
    assert torch.equal(a, b)


def test_generate_content_stream_equals_whole(cuda):
    from vila_b200.model import LlavaLlamaModel, tiny_test_config
    model = LlavaLlamaModel(tiny_test_config(), device="cuda").init_random(14)
    gc = SimpleNamespace(max_new_tokens=16, do_sample=True, temperature=0.9, top_k=0, top_p=0.95, seed=77,
                         eos_token_id=None, pad_token_id=0, max_length=None)
    whole = model.generate_content(["Describe the scene."], generation_config=gc)
    chunks = list(model.generate_content(["Describe the scene."], generation_config=gc, stream=True))
    assert len(chunks) >= 2 and " ".join(chunks).split() == whole.split()
    greedy = model.generate_content(["Describe the scene."],
                                    generation_config=SimpleNamespace(**{**vars(gc), "do_sample": False}))
    assert greedy != whole
