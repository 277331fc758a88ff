"""Logprobs in the continuous-batching engine (serving.BatchedDecoder(logprobs=n)) of NVILA-8B (random init).

  * the kernel alone: vila_token_logprobs at V = 152,064, M = 1 / 8 / 32 rows and n = 0 / 5 / 20 alternatives;
    --kernel-reps launches captured in CUDA graphs, CUDA events around their replays, µs per launch;
  * the whole engine step: the decoder without logprobs against the decoder with logprobs=5 (greedy) at 8 x 300 and
    32 x 300 tokens with bf16 and w4a16 weights; the decoders alternated, median of --reps runs of --steps steps after
    a warm-up; the logprobs cost is the difference of the medians.
Reads the card (name, power limit, max SM clock) with a read-only nvidia-smi query in the same run, prints a summary
and writes batched_logprobs.json under --out-dir.

    python tools/bench_batched_logprobs.py [--reps 5] [--steps 32] [--kernel-reps 2000] [--out-dir bench_results]
"""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from vila_b200 import ops, serving  # noqa: E402

V = 152_064
ROWS = (1, 8, 32)
TOPS = (0, 5, 20)
MIXES = {"8x300": [300] * 8, "32x300": [300] * 32}
ENGINE_TOP = 5


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit not read"



def kernel_table(launches):
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    cols = 64
    for M in ROWS:
        logits = (torch.randn(M, V, device="cuda", generator=g) * 3).to(torch.bfloat16)
        tokens = torch.randint(0, V, (M,), device="cuda", generator=g)
        step = torch.full((M,), 3, dtype=torch.int64, device="cuda")
        pos = torch.zeros(M, dtype=torch.int32, device="cuda")
        lp = torch.zeros(M, cols, device="cuda")
        for n in TOPS:
            top = dict(top_ids=torch.zeros(M, cols, n, dtype=torch.int32, device="cuda"),
                       top_lp=torch.zeros(M, cols, n, device="cuda")) if n else {}
            per_graph = 50
            ops.token_logprobs(logits, tokens, step, pos, lp_hist=lp, **top)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(per_graph):
                    ops.token_logprobs(logits, tokens, step, pos, lp_hist=lp, **top)
            graph.replay()
            torch.cuda.synchronize()
            replays = max(1, launches // per_graph)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(replays):
                graph.replay()
            b.record()
            torch.cuda.synchronize()
            rows.append({"M": M, "n": n, "us_per_launch": round(a.elapsed_time(b) * 1e3 / (replays * per_graph), 2)})
    return rows


def engine_table(llm, reps, steps):
    g = torch.Generator(device="cuda").manual_seed(1)
    rows = []
    for w in ("bf16", "w4a16"):
        llm.set_decode_weights(w)
        for mix, ctxs in MIXES.items():
            ids = torch.randint(0, llm.config.vocab_size, (max(ctxs),), device="cuda", generator=g)
            emb = llm.model.embed_tokens(ids)
            tokens = (max(ctxs) + (reps + 1) * steps + 8 + 127) // 128 * 128
            decs = {}
            for top in (None, ENGINE_TOP):
                dec = serving.BatchedDecoder(llm, len(ctxs), tokens, max_new=(reps + 1) * steps + 8, logprobs=top)
                dec.capture()
                for s, c in enumerate(ctxs):
                    dec.admit(s, emb[:c].clone())
                dec.run(steps)  # warm-up
                decs[top] = dec
            times = {None: [], ENGINE_TOP: []}
            for _ in range(reps):
                for top in (None, ENGINE_TOP):  # alternated
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    decs[top].run(steps)
                    b.record()
                    torch.cuda.synchronize()
                    times[top].append(a.elapsed_time(b) / steps)
            assert decs[None].generated(0) == decs[ENGINE_TOP].generated(0)  # logprobs change no token
            plain, with_lp = statistics.median(times[None]), statistics.median(times[ENGINE_TOP])
            rows.append({"mix": mix, "weights": w, "plain_step_ms": round(plain, 3),
                         "logprobs_step_ms": round(with_lp, 3), "cost_ms": round(with_lp - plain, 4),
                         "cost_frac": round((with_lp - plain) / plain, 4),
                         "plain_all": [round(t, 3) for t in times[None]],
                         "logprobs_all": [round(t, 3) for t in times[ENGINE_TOP]]})
            del decs, emb
            torch.cuda.empty_cache()
    llm.set_decode_weights("bf16")
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed engine runs per decoder (alternated)")
    ap.add_argument("--steps", type=int, default=32, help="decode steps per timed engine run")
    ap.add_argument("--kernel-reps", type=int, default=2000, help="timed vila_token_logprobs launches per case")
    ap.add_argument("--skip-engine", action="store_true", help="the kernel alone only")
    ap.add_argument("--out-dir", type=str, default="bench_results")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    ops.ensure_workspace("cuda")
    who = card()
    with torch.inference_mode():
        kern = kernel_table(args.kernel_reps)
        eng = []
        if not args.skip_engine:
            from vila_b200.model import LlavaLlamaModel, nvila_8b
            model = LlavaLlamaModel(nvila_8b(), device="cuda").init_random(0, device_rng=True)
            eng = engine_table(model.llm, args.reps, args.steps)
    res = {"card": who, "model": "NVILA-8B LLM, random init", "vocab": V, "kernel": kern, "engine": eng,
           "engine_top": ENGINE_TOP, "steps": args.steps, "reps": args.reps, "kernel_reps": args.kernel_reps}
    print(f"card: {who}\n")
    print("| M | " + " | ".join(f"n = {n}" for n in TOPS) + " |\n|---|" + "---|" * len(TOPS))
    for M in ROWS:
        us = {r["n"]: r["us_per_launch"] for r in kern if r["M"] == M}
        print(f"| {M} | " + " | ".join(f"{us[n]}" for n in TOPS) + " |")
    print("\n| mix | weights | step ms | step ms, logprobs=5 | cost ms | cost |\n|---|---|---|---|---|---|")
    for r in eng:
        print(f"| {r['mix']} | {r['weights']} | {r['plain_step_ms']} | {r['logprobs_step_ms']} | {r['cost_ms']} | "
              f"{r['cost_frac']:.2%} |")
    out = Path(args.out_dir)
    out.mkdir(parents=True, exist_ok=True)
    (out / "batched_logprobs.json").write_text(json.dumps(res, indent=1))
    print(json.dumps({"card": who, "kernel": kern, "engine": eng}))


if __name__ == "__main__":
    main()
