"""Grammar-constrained decoding (response_format) in the single-stream graph decoder: what it costs.

  * kernel: vila_apply_token_bitmask_row at V = 152,064 (half the ids allowed): CUDA events around --launches launches
    captured in one graph, median of --reps rounds;
  * step: NVILA-8B (random init) ms/token for a 279-token and a 16,470-token prompt with bf16 and w4a16 decode weights,
    in four conditions alternated over --reps rounds (median, min, max): unconstrained greedy (the graph decoder),
    JSON greedy and JSON at T 0.7 (the graph decoder with an xgrammar matcher: two graphs and one host round trip per
    token), and the eager logits_processor path (Qwen2ForCausalLM.generate(logits_processor=...)) with xgrammar's HF
    processor for the same grammar.  Host clock around GraphDecoder.run, which ends in a device synchronisation in
    every condition; the eager path's time per token is (T(n) - T(1)) / (n - 1), so its prefill is not counted.
  * grammar: a JSON schema, an object whose one required property is a string of at least 8 (--steps + 8) characters.
    No token is longer than 8 characters, so no document can end within a timed run and every run makes exactly
    --steps tokens: the per-token cost in steady state, not a run cut short by the grammar's stop token.  Inside the
    string nearly every id is allowed; the matcher's cost at structural positions (fewer allowed ids) is not separated.
  * profile (--profile, a run of its own after the timed rounds): torch.profiler with CUDA activities around one
    unconstrained greedy run and one constrained greedy run of the 279-token prompt per weight mode.  Their device
    timelines are split per token into busy time (the union of every kernel and copy), the mask kernel's and the two
    copies' durations, and the device's idle time, which is attributed to what ends it: the mask copy / choose graph (the gap
    between the body and choose), the token copy, or the next body (the host's synchronisation and body launch).  The
    traces are written under --out-dir.
  * vocabulary: no tokenizer files ship with the project, so the production-size vocabulary (152,064 entries) is built
    from a seeded generator: the 256 single bytes, then random strings of 2 to 8 printable ASCII characters.  The
    matcher's host cost on the real Qwen2 vocabulary is not measured.  The weights are random, so EOS is off.
Reads the card (name, power limit, max SM clock) with a read-only nvidia-smi query in the same run, prints markdown
tables and writes constrained.json under --out-dir.

    python tools/bench_constrained.py [--reps 5] [--steps 64] [--eager-steps 16] [--launches 2000] [--profile]
"""
import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from vila_b200 import ops  # noqa: E402
from vila_b200.sampling import SamplingParams  # noqa: E402

V = 152064
PROMPTS = {"image-279": 279, "video-16470": 16470}
MODES = ("bf16", "w4a16")
CONDITIONS = ("greedy", "json greedy", "json T 0.7", "eager logits_processor")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit not read"


def stats(xs):
    return {"median": round(statistics.median(xs), 4), "min": round(min(xs), 4), "max": round(max(xs), 4)}


def vocabulary(seed=0):
    rng = np.random.default_rng(seed)
    chars = np.array([chr(c) for c in range(32, 127)])
    vocab = [bytes([i]) for i in range(256)]
    seen = set(vocab)
    while len(vocab) < V:
        s = "".join(rng.choice(chars, int(rng.integers(2, 9)))).encode()
        if s not in seen:
            seen.add(s)
            vocab.append(s)
    return vocab


class HostIds(list):
    """the eager loop's id history as xgrammar's HF processor reads it: rows of Python ints (xgrammar 0.2's
    accept_token takes an int, not the 0-d tensor that indexing a torch tensor gives)"""

    @property
    def shape(self):
        return (len(self),)


def device_breakdown(trace: Path, tokens):
    """µs per token of the device timeline of a profiled run (its exported chrome trace): the time the device is busy,
    the mask kernel's and the two copies' durations, and the idle time by what ends it"""
    evs = sorted((e["ts"], e["ts"] + e["dur"], e["name"]) for e in json.loads(trace.read_text())["traceEvents"]
                 if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset"))

    def kind(name):
        if name.startswith("Memcpy HtoD"):
            return "mask copy"
        if name.startswith("Memcpy DtoH"):
            return "token copy"
        if "token_bitmask" in name:
            return "mask kernel"
        return None

    # kernels launched with PDL start before their predecessor ends, so their durations overlap: "busy" is the union
    out = {k: 0.0 for k in ("busy", "mask kernel", "mask copy", "token copy", "idle before choose",
                            "idle before token copy", "idle before body")}
    end = None
    for a, b, name in evs:
        k = kind(name)
        if k is not None:
            out[k] += b - a
        if end is not None and a > end:
            gap = "idle before choose" if k in ("mask copy", "mask kernel") else (
                "idle before token copy" if k == "token copy" else "idle before body")
            out[gap] += a - end
        out["busy"] += max(0.0, b - max(a, end if end is not None else a))
        end = b if end is None else max(end, b)
    out["span"] = (evs[-1][1] - evs[0][0]) if evs else 0.0
    return {k: round(v / tokens, 2) for k, v in out.items()}


def bench_kernel(launches, reps):
    g = torch.Generator(device="cuda").manual_seed(0)
    row = (torch.randn(V, device="cuda", generator=g) * 4).to(torch.bfloat16)
    mask = torch.randint(-2 ** 31, 2 ** 31 - 1, ((V + 31) // 32,), device="cuda", generator=g, dtype=torch.int32)
    out = torch.empty_like(row)
    ops.apply_token_bitmask_row(row, mask, out=out)
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        for _ in range(launches):
            ops.apply_token_bitmask_row(row, mask, out=out)
    gr.replay()
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        gr.replay()
        b.record()
        torch.cuda.synchronize()
        t.append(a.elapsed_time(b) * 1e3 / launches)
    return stats(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed rounds (every condition once per round)")
    ap.add_argument("--steps", type=int, default=64, help="tokens per graph-decoder run")
    ap.add_argument("--eager-steps", type=int, default=16, help="tokens per eager run")
    ap.add_argument("--launches", type=int, default=2000, help="kernel launches per timed graph")
    ap.add_argument("--out-dir", type=str, default="bench_results")
    ap.add_argument("--kernel-only", action="store_true")
    ap.add_argument("--profile", action="store_true", help="also the torch.profiler breakdown (a run of its own)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    ops.ensure_workspace("cuda")
    Path(args.out_dir).mkdir(parents=True, exist_ok=True)
    who = card()
    res = {"card": who, "kernel_us": bench_kernel(args.launches, args.reps)}
    print(f"card: {who}")
    k = res["kernel_us"]
    print(f"vila_apply_token_bitmask_row V={V}: {k['median']:.2f} us/launch ({k['min']:.2f}-{k['max']:.2f})")
    if not args.kernel_only:
        import xgrammar as xgr

        from vila_b200.model import GraphDecoder, LlavaLlamaModel, nvila_8b
        t0 = time.perf_counter()
        stop = V - 1
        compiler = xgr.GrammarCompiler(xgr.TokenizerInfo(vocabulary(), vocab_size=V, stop_token_ids=[stop]))
        schema = {"type": "object", "properties": {"text": {"type": "string", "minLength": 8 * (args.steps + 8)}},
                  "required": ["text"], "additionalProperties": False}
        grammar = compiler.compile_json_schema(json.dumps(schema))
        res["grammar_compile_s"] = round(time.perf_counter() - t0, 2)
        model = LlavaLlamaModel(nvila_8b(), device="cuda").init_random(0, device_rng=True)
        llm = model.llm
        res.update(model="NVILA-8B LLM, random init", steps=args.steps, eager_steps=args.eager_steps, reps=args.reps,
                   schema=schema, decode={}, tokens={}, profile={})
        t07 = SamplingParams(0.7, seed=1)
        with torch.inference_mode():
            g = torch.Generator(device="cuda").manual_seed(1)
            ids = torch.randint(0, llm.config.vocab_size, (max(PROMPTS.values()),), device="cuda", generator=g)
            emb_all = llm.model.embed_tokens(ids)
            for mode in MODES:
                llm.set_decode_weights(mode)
                for pname, S in PROMPTS.items():
                    dec = GraphDecoder(llm, args.steps + 8)
                    cache = dec.cache_for(S + args.steps + 1)
                    last = llm.prefill_hidden(emb_all[:S].clone(), cache)[-1].clone()
                    emb = emb_all[:S].clone()

                    def graph_run(params, constrained):
                        cache.length = S
                        m = xgr.GrammarMatcher(grammar, override_stop_tokens=[stop]) if constrained else None
                        dec.start(last, cache, params, **({"grammar": m} if constrained else {}))
                        torch.cuda.synchronize()
                        t = time.perf_counter()
                        dec.run(args.steps + 1)  # the first token came from start()
                        torch.cuda.synchronize()
                        made = len(dec.grammar_ids) - 1 if constrained else args.steps
                        assert made == args.steps, f"the grammar ended a run after {made} tokens"
                        return (time.perf_counter() - t) * 1e3 / made, made

                    def eager_once(n):
                        proc = xgr.contrib.hf.LogitsProcessor(grammar)
                        torch.cuda.synchronize()
                        t = time.perf_counter()
                        out = llm._generate_eager(emb, n, [], False, [lambda h, lg: proc(HostIds(h.tolist()), lg)],
                                                  1.0, 1.0, 0)
                        torch.cuda.synchronize()
                        return time.perf_counter() - t, len(out)

                    def eager_run():
                        t1, _ = eager_once(1)
                        tn, made = eager_once(args.eager_steps)
                        return (tn - t1) * 1e3 / max(made - 1, 1), made

                    runs = {"greedy": lambda: graph_run(None, False), "json greedy": lambda: graph_run(None, True),
                            "json T 0.7": lambda: graph_run(t07, True), "eager logits_processor": eager_run}
                    for fn in runs.values():  # warm-up: captures every graph the timed runs replay
                        fn()
                    ms = {c: [] for c in CONDITIONS}
                    made = {}
                    for _ in range(args.reps):
                        for c in CONDITIONS:
                            t, made[c] = runs[c]()
                            ms[c].append(t)
                    res["decode"].setdefault(pname, {})[mode] = {c: stats(v) for c, v in ms.items()}
                    res["tokens"].setdefault(pname, {})[mode] = made
                    if args.profile and pname == "image-279":
                        from torch.profiler import ProfilerActivity, profile
                        for c, constrained in (("greedy", False), ("json greedy", True)):
                            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                                graph_run(None, constrained)
                            trace = Path(args.out_dir) / f"trace_{mode}_{c.replace(' ', '_')}.json"
                            prof.export_chrome_trace(str(trace))
                            res["profile"].setdefault(mode, {})[c] = device_breakdown(trace, args.steps)
                    del dec, cache
                    torch.cuda.empty_cache()
            llm.set_decode_weights("bf16")
        print("ms/token (median, min-max); tokens made per timed run in brackets")
        print("| prompt | weights | " + " | ".join(CONDITIONS) + " |")
        print("|" + "---|" * (2 + len(CONDITIONS)))
        for pname, per_mode in res["decode"].items():
            for mode, row in per_mode.items():
                made = res["tokens"][pname][mode]
                print(f"| {pname} | {mode} | " + " | ".join(
                    f"{row[c]['median']:.3f} ({row[c]['min']:.3f}-{row[c]['max']:.3f}) [{made[c]}]"
                    for c in CONDITIONS) + " |")
        for mode, per in res["profile"].items():
            print(f"device timeline, 279-token prompt, {mode}, µs/token (profiled run):")
            print("| | " + " | ".join(per["greedy"]) + " |\n|" + "---|" * (1 + len(per["greedy"])))
            for c, row in per.items():
                print(f"| {c} | " + " | ".join(f"{v:.1f}" for v in row.values()) + " |")
            print("| difference | " + " | ".join(f"{per['json greedy'][k] - per['greedy'][k]:+.1f}"
                                               for k in per["greedy"]) + " |")
    out = Path(args.out_dir)
    out.mkdir(parents=True, exist_ok=True)
    (out / "constrained.json").write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
