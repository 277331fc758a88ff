"""The continuous-batching engine (serving.BatchedDecoder) of NVILA-8B (random init) with the bf16 and the opt-in
FP8 (e4m3, one fp32 scale per token and KV head) KV cache.

  * attention alone, per layer: the bf16 kernels as the engine calls them (decode_attn_head_kernel for slots of
    at most 2048 tokens, the batched split-KV kernel beside it for longer ones) and vila_decode_attention_fp8_batch
    at split sizes of 256, 512 and 1024 tokens, each with the ladder entry the engine would launch; 28 layers'
    pools in one CUDA graph (so K/V stream from HBM), replayed until >= --kernel-reps launches, CUDA events
    around the replays; K/V bytes (codes and scales) over time as a share of 3.35 TB/s;
  * engine step: ms per step and aggregate decode tok/s for bf16 / fp8 KV under bf16 and w4a16 weights, the
    four configurations alternated, median of --reps runs of --steps steps after a warm-up.
Mixes: 8 x 300, 8 x 2048, 8 x 16,470 and 2 x 16,470 + 6 x 300 tokens.  Reads the card (name, power limit, max SM
clock) with a read-only nvidia-smi query in the same run, prints a summary and writes batched_kv_fp8.json under
--out-dir.

    python tools/bench_batched_kv_fp8.py [--reps 5] [--steps 32] [--kernel-reps 224] [--out-dir bench_results]
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
from vila_b200.model.qwen2 import quantize_kv_e4m3  # noqa: E402

HBM_DATASHEET_GBS = 3350.0  # H100 SXM data sheet
MIXES = {"8x300": [300] * 8, "8x2048": [2048] * 8, "8x16470": [16470] * 8, "2x16470+6x300": [16470] * 2 + [300] * 6}
SPLITS = (256, 512, 1024)
PAGE, D = 128, 128


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit not read"


def graph_us(launch, n_layers, launches):
    """µs per launch of `launch(li)` over n_layers pools captured in one graph and replayed"""
    for li in range(n_layers):
        launch(li)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for li in range(n_layers):
            launch(li)
    graph.replay()
    torch.cuda.synchronize()
    replays = max(1, (launches + n_layers - 1) // n_layers)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(replays):
        graph.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / (replays * n_layers)


def attention_table(cfg, inv_freq, launches):
    L, Hq, Hkv = cfg.num_hidden_layers, cfg.num_attention_heads, cfg.num_key_value_heads
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    for mix, ctxs in MIXES.items():
        B = len(ctxs)
        pages_per_slot = (max(ctxs) + 1 + PAGE - 1) // PAGE
        P = B * pages_per_slot
        pt = torch.arange(P, dtype=torch.int32, device="cuda").view(B, pages_per_slot)
        pos = torch.tensor(ctxs, dtype=torch.int32, device="cuda")  # ctx cached tokens, the new one at ctx
        qkv = torch.randn(B, (Hq + 2 * Hkv) * D, device="cuda", generator=g).to(torch.bfloat16)
        out = torch.empty(B, Hq * D, dtype=torch.bfloat16, device="cuda")
        tokens = sum(c + 1 for c in ctxs)
        # bf16 pools [L, 2, P, 128, Hkv, D] and their e4m3 forms
        pool = torch.empty(L, 2, P, PAGE, Hkv, D, device="cuda", dtype=torch.bfloat16)
        codes = torch.empty(L, 2, P, PAGE, Hkv, D, device="cuda", dtype=torch.float8_e4m3fn)
        scales = torch.empty(L, 2, P, PAGE, Hkv, device="cuda")
        for li in range(L):  # layer by layer: bounds the fp32 temporaries
            pool[li] = torch.randn(2, P, PAGE, Hkv, D, device="cuda", generator=g).to(torch.bfloat16)
            codes[li], scales[li] = quantize_kv_e4m3(pool[li])
        longest = max(ctxs) + 1
        # bf16: the engine's pair of kernels
        n_bf = serving.attention_config(longest)
        long = pos >= serving.HEAD_KERNEL_TOKENS
        pos_head, pos_split = pos.masked_fill(long, -1), pos.masked_fill(~long, -1)
        if n_bf is not None:
            o_partial = torch.zeros(B * n_bf * Hq * D, device="cuda")
            lse = torch.zeros(B * n_bf * Hq, device="cuda")
            cnt = torch.zeros(B * Hkv, dtype=torch.int32, device="cuda")

        def bf16(li):
            ops.decode_attention_batch(qkv, pos_head if n_bf else pos, pool[li, 0], pool[li, 1], pt, out, inv_freq,
                                       Hq, Hkv, D, D ** -0.5)
            if n_bf is not None:
                ops.decode_attention_split_batch(qkv, pos_split, pool[li, 0], pool[li, 1], pt, out, o_partial, lse,
                                                 cnt, inv_freq, Hq, Hkv, D, n_bf, serving.SPLIT_TOKENS, D ** -0.5)
        bytes_bf16 = tokens * Hkv * D * 2 * 2
        qkv_copy = qkv.clone()

        def restore():
            qkv.copy_(qkv_copy)  # the bf16 split path rotates q / k in place
        us = graph_us(bf16, L, launches)
        restore()
        rows.append({"mix": mix, "kv": "bf16", "split_tokens": serving.SPLIT_TOKENS if n_bf else None,
                     "splits": n_bf, "us_per_layer": round(us, 2), "kv_bytes": bytes_bf16,
                     "frac_of_datasheet_hbm": round(bytes_bf16 / us / 1e3 / HBM_DATASHEET_GBS, 4)})
        bytes_fp8 = tokens * Hkv * 2 * (D + 4)
        for split in SPLITS:
            ladder = next(n for n in serving.FP8_LADDER_TOKENS if n >= longest)
            n = (ladder + split - 1) // split
            ws = torch.zeros(B * Hq * n * (D + 2), device="cuda")
            cnt8 = torch.zeros(B * Hkv, dtype=torch.int32, device="cuda")

            def fp8(li, n=n, split=split, ws=ws, cnt8=cnt8):
                ops.decode_attention_fp8_batch(qkv, pos, codes[li, 0], codes[li, 1], scales[li, 0], scales[li, 1], pt,
                                               out, ws, cnt8, inv_freq, Hq, Hkv, n, split, D ** -0.5)
            us = graph_us(fp8, L, launches)
            rows.append({"mix": mix, "kv": "fp8", "split_tokens": split, "splits": n, "us_per_layer": round(us, 2),
                         "kv_bytes": bytes_fp8,
                         "frac_of_datasheet_hbm": round(bytes_fp8 / us / 1e3 / HBM_DATASHEET_GBS, 4)})
        del pool, codes, scales
        torch.cuda.empty_cache()
    return rows


def engine_table(llm, reps, steps):
    g = torch.Generator(device="cuda").manual_seed(1)
    rows = []
    combos = [(w, kv) for w in ("bf16", "w4a16") for kv in ("bf16", "fp8")]
    for mix, ctxs in MIXES.items():
        ids = torch.randint(0, llm.config.vocab_size, (max(ctxs),), device="cuda", generator=g)
        emb = llm.model.embed_tokens(ids)
        tokens = (max(ctxs) + (reps + 1) * steps + 8 + 127) // 128 * 128
        decs = {}
        for w, kv in combos:
            llm.set_decode_weights(w)
            dec = serving.BatchedDecoder(llm, len(ctxs), tokens, max_new=(reps + 1) * steps + 8, kv_cache=kv)
            dec.capture()
            for s, c in enumerate(ctxs):
                dec.admit(s, emb[:c].clone())
            dec.run(steps)  # warm-up
            decs[(w, kv)] = dec
        llm.set_decode_weights("bf16")
        times = {c: [] for c in combos}
        for _ in range(reps):
            for c in combos:  # alternated: every configuration sees the same contexts and the same card state
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                decs[c].run(steps)
                b.record()
                torch.cuda.synchronize()
                times[c].append(a.elapsed_time(b) / steps)
        for (w, kv) in combos:
            med = statistics.median(times[(w, kv)])
            dec = decs[(w, kv)]
            pool_bytes = sum(t.numel() * t.element_size() for t in (dec.pool, dec.pool_scale) if t is not None)
            rows.append({"mix": mix, "weights": w, "kv": kv, "attention": dec.config, "step_ms": round(med, 3),
                         "step_ms_all": [round(t, 3) for t in times[(w, kv)]],
                         "decode_tok_s": round(len(ctxs) / med * 1e3, 1), "pool_gb": round(pool_bytes / 1e9, 3)})
        del decs, emb
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed engine runs per configuration (alternated)")
    ap.add_argument("--steps", type=int, default=32, help="decode steps per timed engine run")
    ap.add_argument("--kernel-reps", type=int, default=224, help="timed attention launches (whole graph replays)")
    ap.add_argument("--skip-engine", action="store_true", help="attention alone only")
    ap.add_argument("--out-dir", type=str, default="bench_results")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from vila_b200.model import LlavaLlamaModel, nvila_8b
    ops.ensure_workspace("cuda")
    who = card()
    cfg8 = nvila_8b()
    with torch.inference_mode():
        model = LlavaLlamaModel(cfg8, device="cuda").init_random(0, device_rng=True)
        llm = model.llm
        attn = attention_table(llm.config, llm.inv_freq, args.kernel_reps)
        eng = [] if args.skip_engine else engine_table(llm, args.reps, args.steps)
    res = {"card": who, "model": "NVILA-8B LLM, random init", "attention": attn, "engine": eng, "steps": args.steps,
           "reps": args.reps, "kernel_reps": args.kernel_reps}
    print(f"card: {who}\n")
    print("| mix | KV | split tokens | splits | us / layer | K/V MB | share of 3.35 TB/s |\n|---|---|---|---|---|---|---|")
    for r in attn:
        print(f"| {r['mix']} | {r['kv']} | {r['split_tokens']} | {r['splits']} | {r['us_per_layer']} | "
              f"{r['kv_bytes'] / 1e6:.1f} | {r['frac_of_datasheet_hbm']:.1%} |")
    print("\n| mix | weights | KV | step ms (median) | decode tok/s | pool GB | all |\n|---|---|---|---|---|---|---|")
    for r in eng:
        print(f"| {r['mix']} | {r['weights']} | {r['kv']} | {r['step_ms']} | {r['decode_tok_s']} | {r['pool_gb']} | "
              f"{r['step_ms_all']} |")
    out = Path(args.out_dir)
    out.mkdir(parents=True, exist_ok=True)
    (out / "batched_kv_fp8.json").write_text(json.dumps(res, indent=1))
    print(json.dumps({"card": who, "engine": eng}))


if __name__ == "__main__":
    main()
