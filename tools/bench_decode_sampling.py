"""Single-stream decode of NVILA-8B (random init), greedy against sampled on the device (vila_sample_finalize).

  * for a 279-token prompt (one image) and a 16,470-token prompt (64-frame video), with bf16, fp8 and w4a16 decode
    weights: ms/token of the GraphDecoder greedy and sampled with T 0.7, T 0.7 + top-p 0.9 and T 0.7 + top-k 50 +
    top-p 0.9; --steps tokens per run with EOS off, CUDA events around the graph replays, the runs alternated
    (every mode and parameter set once per round) and the median of --reps rounds taken;
  * once, for comparison, the eager path generate(do_sample=True) ran before the graph decoder could sample
    (Qwen2ForCausalLM._generate_eager: an un-graphed prefill_hidden per token and a host-side draw), --eager-steps
    tokens at the 279-token prompt, host clock around work that ends in a synchronise.
Reads the card (name, power limit, max SM clock) with a read-only nvidia-smi query in the same run, prints a
markdown table and writes decode_sampling.json under --out-dir.

    python tools/bench_decode_sampling.py [--reps 5] [--steps 128] [--eager-steps 32] [--out-dir bench_results]
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
from vila_b200.sampling import SamplingParams  # noqa: E402

PROMPTS = {"image-279": 279, "video-16470": 16470}
MODES = ("bf16", "fp8", "w4a16")
PARAMS = {"greedy": None, "T 0.7": SamplingParams(0.7, seed=1), "T 0.7, top-p 0.9": SamplingParams(0.7, top_p=0.9, seed=2),
          "T 0.7, top-k 50, top-p 0.9": SamplingParams(0.7, top_k=50, top_p=0.9, seed=3)}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit not read"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed rounds (every mode and parameter set once per round)")
    ap.add_argument("--steps", type=int, default=128, help="tokens per timed run")
    ap.add_argument("--eager-steps", type=int, default=32, help="tokens of the one eager do_sample run")
    ap.add_argument("--out-dir", type=str, default="bench_results")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from vila_b200.model import GraphDecoder, LlavaLlamaModel, nvila_8b
    ops.ensure_workspace("cuda")
    who = card()
    model = LlavaLlamaModel(nvila_8b(), device="cuda").init_random(0, device_rng=True)
    llm = model.llm
    res = {"card": who, "model": "NVILA-8B LLM, random init", "steps": args.steps, "reps": args.reps, "decode": {}}
    with torch.inference_mode():
        g = torch.Generator(device="cuda").manual_seed(1)
        ids = torch.randint(0, llm.config.vocab_size, (max(PROMPTS.values()),), device="cuda", generator=g)
        emb_all = llm.model.embed_tokens(ids)
        decs = {}  # one decoder per (mode, prompt) with its own prefilled cache, holding its mode's weights
        for mode in MODES:
            llm.set_decode_weights(mode)
            for pname, S in PROMPTS.items():
                dec = GraphDecoder(llm, args.steps + 8)
                cache = dec.cache_for(S + args.steps + 1)
                last = llm.prefill_hidden(emb_all[:S].clone(), cache)[-1].clone()
                decs[mode, pname] = (dec, cache, S, last)
        llm.set_decode_weights("bf16")

        def run(mode, pname, params):
            dec, cache, S, last = decs[mode, pname]
            cache.length = S
            dec.start(last, cache, params)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            dec.run(args.steps + 1)  # the first token came from start(): args.steps graph replays
            b.record()
            torch.cuda.synchronize()
            return a.elapsed_time(b) / args.steps

        for key in decs:  # warm-up: captures every graph the timed runs replay
            for params in PARAMS.values():
                run(*key, params)
        for pname in PROMPTS:
            ms = {(mode, name): [] for mode in MODES for name in PARAMS}
            for _ in range(args.reps):
                for mode in MODES:
                    for name, params in PARAMS.items():
                        ms[mode, name].append(run(mode, pname, params))
            res["decode"][pname] = {mode: {name: {"ms_per_token": round(statistics.median(ms[mode, name]), 4),
                                                  "min": round(min(ms[mode, name]), 4),
                                                  "max": round(max(ms[mode, name]), 4)} for name in PARAMS}
                                    for mode in MODES}
        del decs
        torch.cuda.empty_cache()
        # the path do_sample=True took before: eager, one prefill_hidden per token and a host-side draw
        emb = emb_all[:PROMPTS["image-279"]].clone()
        llm._generate_eager(emb, 4, [], True, None, 0.7, 1.0, 0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        llm._generate_eager(emb, args.eager_steps, [], True, None, 0.7, 1.0, 0)
        torch.cuda.synchronize()
        res["eager_do_sample_279"] = {"tokens": args.eager_steps,
                                      "ms_per_token": round((time.perf_counter() - t0) * 1e3 / args.eager_steps, 3)}
    print(f"card: {who}")
    head = "| prompt | weights | " + " | ".join(PARAMS) + " |"
    print(head)
    print("|" + "---|" * (2 + len(PARAMS)))
    for pname, per_mode in res["decode"].items():
        for mode, row in per_mode.items():
            print(f"| {pname} | {mode} | " + " | ".join(f"{row[n]['ms_per_token']:.3f}" for n in PARAMS) + " |")
    print(f"eager generate(do_sample=True), 279-token prompt, bf16: {res['eager_do_sample_279']['ms_per_token']} "
          f"ms/token over {args.eager_steps} tokens")
    out = Path(args.out_dir)
    out.mkdir(parents=True, exist_ok=True)
    (out / "decode_sampling.json").write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
