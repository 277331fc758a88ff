"""Sampling in the continuous-batching engine (serving.BatchedDecoder(sampling=True)) of NVILA-8B (random init).

  * the kernel alone: vila_sample_batch at V = 152,064 and M = 1 / 8 / 16 / 32 rows for greedy, T only, top-k 50,
    top-p 0.9 and top-k 50 + top-p 0.9 rows (T 0.7); --kernel-reps launches captured in one CUDA graph, CUDA events
    around its replays, µs per launch;
  * the whole engine step: the greedy decoder against the sampling decoder (T 0.7, top-p 0.9) at 8 x 300 and
    32 x 300 tokens with bf16 and w4a16 weights; the decoders alternated, median of --reps runs of --steps steps
    after a warm-up; the sampling cost is the difference of the medians.
Reads the card (name, power limit, max SM clock) with a read-only nvidia-smi query in the same run, prints a summary
and writes batched_sampling.json under --out-dir.

    python tools/bench_batched_sampling.py [--reps 5] [--steps 32] [--kernel-reps 2000] [--out-dir bench_results]
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
from vila_b200.sampling import SamplingParams  # noqa: E402

V = 152_064
ROW_KINDS = {"greedy": SamplingParams(), "T only": SamplingParams(0.7),
             "top-k 50": SamplingParams(0.7, top_k=50), "top-p 0.9": SamplingParams(0.7, top_p=0.9),
             "top-k 50 + top-p 0.9": SamplingParams(0.7, top_k=50, top_p=0.9)}
MIXES = {"8x300": [300] * 8, "32x300": [300] * 32}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit not read"


def kernel_table(launches):
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    for M in (1, 8, 16, 32):
        logits = (torch.randn(M, V, device="cuda", generator=g) * 3).to(torch.bfloat16)
        for kind, p in ROW_KINDS.items():
            args = [torch.full((M,), v, device="cuda", dtype=dt) for v, dt in
                    ((p.inv_temperature, torch.float32), (p.top_k, torch.int32), (p.top_p, torch.float32),
                     (7, torch.int64), (3, torch.int64), (0, torch.int32))]
            out = torch.zeros(M, dtype=torch.int64, device="cuda")
            per_graph = 50
            ops.sample_batch(logits, *args, out=out)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(per_graph):
                    ops.sample_batch(logits, *args, out=out)
            graph.replay()
            torch.cuda.synchronize()
            replays = max(1, launches // per_graph)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(replays):
                graph.replay()
            b.record()
            torch.cuda.synchronize()
            rows.append({"M": M, "rows": kind, "us_per_launch": round(a.elapsed_time(b) * 1e3 / (replays * per_graph), 2)})
    return rows


def engine_table(llm, reps, steps):
    g = torch.Generator(device="cuda").manual_seed(1)
    rows = []
    samp = SamplingParams(0.7, top_p=0.9)
    for w in ("bf16", "w4a16"):
        llm.set_decode_weights(w)
        for mix, ctxs in MIXES.items():
            ids = torch.randint(0, llm.config.vocab_size, (max(ctxs),), device="cuda", generator=g)
            emb = llm.model.embed_tokens(ids)
            tokens = (max(ctxs) + (reps + 1) * steps + 8 + 127) // 128 * 128
            decs = {}
            for sampling in (False, True):
                dec = serving.BatchedDecoder(llm, len(ctxs), tokens, max_new=(reps + 1) * steps + 8, sampling=sampling)
                dec.capture()
                for s, c in enumerate(ctxs):
                    if sampling:
                        dec.admit(s, emb[:c].clone(), SamplingParams(samp.temperature, samp.top_k, samp.top_p, seed=s))
                    else:
                        dec.admit(s, emb[:c].clone())
                dec.run(steps)  # warm-up
                decs[sampling] = dec
            times = {False: [], True: []}
            for _ in range(reps):
                for sampling in (False, True):  # alternated
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    decs[sampling].run(steps)
                    b.record()
                    torch.cuda.synchronize()
                    times[sampling].append(a.elapsed_time(b) / steps)
            greedy, sampled = statistics.median(times[False]), statistics.median(times[True])
            rows.append({"mix": mix, "weights": w, "greedy_step_ms": round(greedy, 3),
                         "sampling_step_ms": round(sampled, 3), "cost_ms": round(sampled - greedy, 4),
                         "cost_frac": round((sampled - greedy) / greedy, 4),
                         "greedy_all": [round(t, 3) for t in times[False]],
                         "sampling_all": [round(t, 3) for t in times[True]]})
            del decs, emb
            torch.cuda.empty_cache()
    llm.set_decode_weights("bf16")
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed engine runs per decoder (alternated)")
    ap.add_argument("--steps", type=int, default=32, help="decode steps per timed engine run")
    ap.add_argument("--kernel-reps", type=int, default=2000, help="timed vila_sample_batch launches per case")
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
           "steps": args.steps, "reps": args.reps, "kernel_reps": args.kernel_reps}
    print(f"card: {who}\n")
    kinds = list(ROW_KINDS)
    print("| M | " + " | ".join(kinds) + " |\n|---|" + "---|" * len(kinds))
    for M in (1, 8, 16, 32):
        us = {r["rows"]: r["us_per_launch"] for r in kern if r["M"] == M}
        print(f"| {M} | " + " | ".join(f"{us[k]}" for k in kinds) + " |")
    print("\n| mix | weights | greedy step ms | sampling step ms | cost ms | cost |\n|---|---|---|---|---|---|")
    for r in eng:
        print(f"| {r['mix']} | {r['weights']} | {r['greedy_step_ms']} | {r['sampling_step_ms']} | {r['cost_ms']} | "
              f"{r['cost_frac']:.2%} |")
    out = Path(args.out_dir)
    out.mkdir(parents=True, exist_ok=True)
    (out / "batched_sampling.json").write_text(json.dumps(res, indent=1))
    print(json.dumps({"card": who, "kernel": kern, "engine": eng}))


if __name__ == "__main__":
    main()
