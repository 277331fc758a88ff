"""Logprobs and presence / frequency penalties in the single-stream graph decoder: what they cost.

  * kernel: vila_token_logprobs_row (one CTA per 1152 entries) against vila_token_logprobs at M = 1 (one 8-CTA
    cluster), V = 152,064, n in {0, 5, 20}: CUDA events around --launches launches captured in one graph, the two
    kernels alternated over --reps rounds, median and spread;
  * step: NVILA-8B (random init) GraphDecoder ms/token for a 279-token and a 16,470-token prompt with bf16, fp8 and
    w4a16 decode weights, in the settings greedy, greedy + logprobs 5, greedy + presence 0.5 / frequency 0.5, greedy
    + both, T 0.7 and T 0.7 + logprobs 5: --steps tokens per run with EOS off, CUDA events around the graph replays,
    every setting once per round (alternated), the median of --reps rounds with min / max;
  * whole stream: Qwen2ForCausalLM.stream_tokens as the server drives it (chunks of 8, the host reading each chunk's
    ids and entries back), --stream-tokens tokens from the 279-token prompt with w4a16 and bf16 weights, without
    options, with logprobs 5, with logprobs 20 and with penalties: host clock around the whole call (prefill
    included; each chunk ends in a device-to-host copy), alternated, median of --stream-reps rounds.
Reads the card (name, power limit, max SM clock) with a read-only nvidia-smi query in the same run, prints markdown
tables and writes stream_logprobs.json under --out-dir.

    python tools/bench_stream_logprobs.py [--reps 5] [--steps 128] [--launches 2000] [--out-dir bench_results]
"""
import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from vila_b200 import ops  # noqa: E402
from vila_b200.penalties import PenaltyParams  # noqa: E402
from vila_b200.sampling import SamplingParams  # noqa: E402

PROMPTS = {"image-279": 279, "video-16470": 16470}
MODES = ("bf16", "fp8", "w4a16")
PEN = PenaltyParams(0.5, 0.5)
T07 = SamplingParams(0.7, seed=1)
SETTINGS = {"greedy": (None, None, None), "greedy + logprobs 5": (None, 5, None), "greedy + penalties": (None, None, PEN),
            "greedy + both": (None, 5, PEN), "T 0.7": (T07, None, None), "T 0.7 + logprobs 5": (T07, 5, None)}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit not read"


def stats(xs):
    return {"median": round(statistics.median(xs), 4), "min": round(min(xs), 4), "max": round(max(xs), 4)}


def bench_kernels(launches, reps):
    """µs per launch of the row kernel and of the cluster kernel at M = 1"""
    V = 152064
    g = torch.Generator(device="cuda").manual_seed(0)
    row = (torch.randn(V, device="cuda", generator=g) * 4).to(torch.bfloat16)
    tok32 = torch.tensor([7], dtype=torch.int32, device="cuda")
    step32 = torch.tensor([1], dtype=torch.int32, device="cuda")
    tok64 = torch.tensor([7], dtype=torch.int64, device="cuda")
    step64 = torch.zeros(1, dtype=torch.int64, device="cuda")
    pos = torch.zeros(1, dtype=torch.int32, device="cuda")
    ws, counter = ops.logprobs_row_workspace(V, "cuda")
    out = {}
    for n in (0, 5, 20):
        lp = torch.zeros(4, device="cuda")
        ids = torch.zeros(4, max(n, 1), dtype=torch.int32, device="cuda")[:, :n].contiguous()
        top = torch.zeros(4, max(n, 1), device="cuda")[:, :n].contiguous()
        lp2 = torch.zeros(1, 4, device="cuda")
        ids2 = torch.zeros(1, 4, max(n, 1), dtype=torch.int32, device="cuda")[:, :, :n].contiguous()
        top2 = torch.zeros(1, 4, max(n, 1), device="cuda")[:, :, :n].contiguous()

        def row_k():
            ops.token_logprobs_row(row, tok32, step32, lp_hist=lp, workspace=ws, counter=counter,
                                   top_ids=ids if n else None, top_lp=top if n else None)

        def cluster_k():
            ops.token_logprobs(row[None], tok64, step64, pos, lp_hist=lp2, top_ids=ids2 if n else None,
                               top_lp=top2 if n else None)

        graphs = {}
        for name, fn in (("row", row_k), ("cluster", cluster_k)):
            fn()
            torch.cuda.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                for _ in range(launches):
                    fn()
            gr.replay()
            graphs[name] = gr
        torch.cuda.synchronize()
        t = {"row": [], "cluster": []}
        for _ in range(reps):
            for name, gr in graphs.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                gr.replay()
                b.record()
                torch.cuda.synchronize()
                t[name].append(a.elapsed_time(b) * 1e3 / launches)
        assert torch.equal(ids, ids2[0]), "the two kernels disagree on the top ids"
        out[n] = {k: stats(v) for k, v in t.items()}
        del graphs
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed rounds (every setting once per round)")
    ap.add_argument("--steps", type=int, default=128, help="tokens per timed run")
    ap.add_argument("--launches", type=int, default=2000, help="kernel launches per timed graph")
    ap.add_argument("--out-dir", type=str, default="bench_results")
    ap.add_argument("--kernels-only", action="store_true")
    ap.add_argument("--stream-tokens", type=int, default=1024, help="tokens per whole-stream run")
    ap.add_argument("--stream-reps", type=int, default=3, help="timed rounds of the whole-stream runs")
    ap.add_argument("--stream-only", action="store_true", help="only the whole-stream runs")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    ops.ensure_workspace("cuda")
    who = card()
    res = {"card": who, "kernels_us": {} if args.stream_only else bench_kernels(args.launches, args.reps)}
    print(f"card: {who}")
    print("| n | vila_token_logprobs_row (µs) | vila_token_logprobs M=1 (µs) |\n|---|---|---|")
    for n, r in res["kernels_us"].items():
        print(f"| {n} | {r['row']['median']:.2f} ({r['row']['min']:.2f}-{r['row']['max']:.2f}) | "
              f"{r['cluster']['median']:.2f} ({r['cluster']['min']:.2f}-{r['cluster']['max']:.2f}) |")
    if not args.kernels_only:
        from vila_b200.model import GraphDecoder, LlavaLlamaModel, nvila_8b
        model = LlavaLlamaModel(nvila_8b(), device="cuda").init_random(0, device_rng=True)
        llm = model.llm
        res.update(model="NVILA-8B LLM, random init", steps=args.steps, reps=args.reps, decode={})
        with torch.inference_mode():
            g = torch.Generator(device="cuda").manual_seed(1)
            ids = torch.randint(0, llm.config.vocab_size, (max(PROMPTS.values()),), device="cuda", generator=g)
            emb_all = llm.model.embed_tokens(ids)
            decs = {}
            for mode in () if args.stream_only else MODES:
                llm.set_decode_weights(mode)
                for pname, S in PROMPTS.items():
                    dec = GraphDecoder(llm, args.steps + 8)
                    cache = dec.cache_for(S + args.steps + 1)
                    last = llm.prefill_hidden(emb_all[:S].clone(), cache)[-1].clone()
                    decs[mode, pname] = (dec, cache, S, last)
            llm.set_decode_weights("bf16")

            def run(mode, pname, setting):
                dec, cache, S, last = decs[mode, pname]
                params, lp, pen = setting
                cache.length = S
                dec.start(last, cache, params, logprobs=lp, penalties=pen)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                dec.run(args.steps + 1)  # the first token came from start(): args.steps graph replays
                b.record()
                torch.cuda.synchronize()
                return a.elapsed_time(b) / args.steps

            for key in decs:  # warm-up: captures every graph the timed runs replay
                for setting in SETTINGS.values():
                    run(*key, setting)
            for pname in () if args.stream_only else PROMPTS:
                ms = {(mode, name): [] for mode in MODES for name in SETTINGS}
                for _ in range(args.reps):
                    for mode in MODES:
                        for name, setting in SETTINGS.items():
                            ms[mode, name].append(run(mode, pname, setting))
                res["decode"][pname] = {mode: {name: stats(ms[mode, name]) for name in SETTINGS} for mode in MODES}
            # the whole stream, host work included
            del decs
            torch.cuda.empty_cache()
            emb = emb_all[:PROMPTS["image-279"]].clone()
            gc = type("GC", (), dict(max_new_tokens=args.stream_tokens, eos_token_id=None))()
            streams = {"plain": {}, "logprobs 5": dict(logprobs=5), "logprobs 20": dict(logprobs=20),
                       "penalties": dict(penalties=PEN)}
            res["stream"] = {"tokens": args.stream_tokens, "chunk_tokens": 8}
            for mode in ("w4a16", "bf16"):
                llm.set_decode_weights(mode)

                def whole(kw):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    n = sum(len(c if not isinstance(c, tuple) else c[0])
                            for c in llm.stream_tokens(emb, gc, chunk_tokens=8, **kw))
                    torch.cuda.synchronize()
                    assert n == args.stream_tokens
                    return (time.perf_counter() - t0) * 1e3 / n

                for kw in streams.values():
                    whole(kw)  # warm-up: captures the graphs
                t = {name: [] for name in streams}
                for _ in range(args.stream_reps):
                    for name, kw in streams.items():
                        t[name].append(whole(kw))
                res["stream"][mode] = {name: stats(v) for name, v in t.items()}
            llm.set_decode_weights("bf16")
        print("| prompt | weights | " + " | ".join(SETTINGS) + " |")
        print("|" + "---|" * (2 + len(SETTINGS)))
        for pname, per_mode in res["decode"].items():
            for mode, row in per_mode.items():
                print(f"| {pname} | {mode} | " + " | ".join(
                    f"{row[n]['median']:.4f} ({row[n]['min']:.4f}-{row[n]['max']:.4f})" for n in SETTINGS) + " |")
        names = list(res["stream"]["w4a16"])
        print(f"whole stream_tokens, 279-token prompt, {args.stream_tokens} tokens, ms/token:")
        print("| weights | " + " | ".join(names) + " |\n|" + "---|" * (1 + len(names)))
        for mode in ("w4a16", "bf16"):
            row = res["stream"][mode]
            print(f"| {mode} | " + " | ".join(
                f"{row[n]['median']:.4f} ({row[n]['min']:.4f}-{row[n]['max']:.4f})" for n in names) + " |")
    out = Path(args.out_dir)
    out.mkdir(parents=True, exist_ok=True)
    (out / "stream_logprobs.json").write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
