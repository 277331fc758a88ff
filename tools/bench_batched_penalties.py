"""Presence / frequency penalties in the continuous-batching engine (serving.BatchedDecoder(penalties=True)) of NVILA-8B
(random init).

  * the kernel alone: vila_apply_penalties at V = 152,064, M = 1 / 8 / 32 rows and t = 0 / 128 / 1024 generated ids
    per row (history ids drawn from the first 4096 ids, so that they repeat); --kernel-reps launches captured in CUDA
    graphs, CUDA events around their replays, µs per launch, and the bytes the kernel must move (one read and one
    write of each row, plus the history) over that time against the H100 SXM data sheet's 3.35 TB/s;
  * the whole engine step: the decoder without penalties against the decoder with penalties=True and every slot at
    presence 0.5 / frequency 0.5 (greedy) at 8 x 300 and 32 x 300 tokens with bf16 and w4a16 weights; the decoders
    alternated, median of --reps runs of --steps steps after a warm-up; the penalty cost is the difference of the
    medians.
Reads the card (name, power limit, max SM clock) with a read-only nvidia-smi query in the same run, prints a summary
and writes batched_penalties.json under --out-dir.

    python tools/bench_batched_penalties.py [--reps 5] [--steps 32] [--kernel-reps 2000] [--out-dir bench_results]
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
from vila_b200.penalties import PenaltyParams  # noqa: E402

V = 152_064
ROWS = (1, 8, 32)
STEPS_T = (0, 128, 1024)
MIXES = {"8x300": [300] * 8, "32x300": [300] * 32}
ENGINE_PENALTIES = PenaltyParams(presence=0.5, frequency=0.5)
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit not read"


def kernel_table(launches):
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    cols = max(STEPS_T) + 8
    for M in ROWS:
        logits = (torch.randn(M, V, device="cuda", generator=g) * 3).to(torch.bfloat16)
        hist = torch.randint(0, 4096, (M, cols), device="cuda", generator=g)
        pos = torch.zeros(M, dtype=torch.int32, device="cuda")
        presence = torch.full((M,), 0.5, device="cuda")
        frequency = torch.full((M,), 0.5, device="cuda")
        out = torch.empty(M, V, dtype=torch.bfloat16, device="cuda")
        for t in STEPS_T:
            step = torch.full((M,), t, dtype=torch.int64, device="cuda")
            per_graph = 50
            ops.apply_penalties(logits, hist, step, pos, presence, frequency, out=out)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(per_graph):
                    ops.apply_penalties(logits, hist, step, pos, presence, frequency, out=out)
            graph.replay()
            torch.cuda.synchronize()
            replays = max(1, launches // per_graph)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(replays):
                graph.replay()
            b.record()
            torch.cuda.synchronize()
            us = a.elapsed_time(b) * 1e3 / (replays * per_graph)
            nbytes = 2 * M * V * 2 + M * t * 8
            rows.append({"M": M, "t": t, "us_per_launch": round(us, 2), "bytes": nbytes,
                         "share_of_hbm_peak": round(nbytes / HBM_BYTES_PER_S / (us * 1e-6), 3)})
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
            for pen in (False, True):
                dec = serving.BatchedDecoder(llm, len(ctxs), tokens, max_new=(reps + 1) * steps + 8, penalties=pen)
                dec.capture()
                for s, c in enumerate(ctxs):
                    dec.admit(s, emb[:c].clone(), **({"penalties": ENGINE_PENALTIES} if pen else {}))
                dec.run(steps)  # warm-up
                decs[pen] = dec
            times = {False: [], True: []}
            for _ in range(reps):
                for pen in (False, True):  # alternated
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    decs[pen].run(steps)
                    b.record()
                    torch.cuda.synchronize()
                    times[pen].append(a.elapsed_time(b) / steps)
            plain, with_pen = statistics.median(times[False]), statistics.median(times[True])
            rows.append({"mix": mix, "weights": w, "plain_step_ms": round(plain, 3),
                         "penalties_step_ms": round(with_pen, 3), "cost_ms": round(with_pen - plain, 4),
                         "cost_frac": round((with_pen - plain) / plain, 4),
                         "plain_all": [round(t, 3) for t in times[False]],
                         "penalties_all": [round(t, 3) for t in times[True]]})
            del decs, emb
            torch.cuda.empty_cache()
    llm.set_decode_weights("bf16")
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed engine runs per decoder (alternated)")
    ap.add_argument("--steps", type=int, default=32, help="decode steps per timed engine run")
    ap.add_argument("--kernel-reps", type=int, default=2000, help="timed vila_apply_penalties launches per case")
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
           "engine_penalties": [ENGINE_PENALTIES.presence, ENGINE_PENALTIES.frequency], "steps": args.steps,
           "reps": args.reps, "kernel_reps": args.kernel_reps}
    print(f"card: {who}\n")
    print("| M | " + " | ".join(f"t = {t}: µs (share of 3.35 TB/s)" for t in STEPS_T) + " |\n|---|"
          + "---|" * len(STEPS_T))
    for M in ROWS:
        cell = {r["t"]: f"{r['us_per_launch']} ({r['share_of_hbm_peak']:.0%})" for r in kern if r["M"] == M}
        print(f"| {M} | " + " | ".join(cell[t] for t in STEPS_T) + " |")
    print("\n| mix | weights | step ms | step ms, penalties | cost ms | cost |\n|---|---|---|---|---|---|")
    for r in eng:
        print(f"| {r['mix']} | {r['weights']} | {r['plain_step_ms']} | {r['penalties_step_ms']} | {r['cost_ms']} | "
              f"{r['cost_frac']:.2%} |")
    out = Path(args.out_dir)
    out.mkdir(parents=True, exist_ok=True)
    (out / "batched_penalties.json").write_text(json.dumps(res, indent=1))
    print(json.dumps({"card": who, "kernel": kern, "engine": eng}))


if __name__ == "__main__":
    main()
