"""Continuous batching at video-length contexts on NVILA-8B (random init), 8 slots:

  * attention alone: vila_decode_attention_split_batch for every ladder entry of vila_b200.serving, and
    vila_decode_attention_batch (the head kernel) where it applies, on one layer's pool; K/V bytes over
    kernel time;
  * whole engine: BatchedDecoder step time and aggregate tok/s, against the same requests served one
    after another by LlavaLlamaModel.llm.generate (CUDA-graph decoder);
  * bytes per step (weights + K/V read) over the 3.35 TB/s HBM3 figure of the H100 SXM data sheet.

Mixes: all slots at 16,470 tokens (64-frame NVILA-Video prompt); 2 such slots + 6 slots of ~300 tokens;
all slots at ~300 tokens; attention alone also at 1,024, 2,048 and 4,096 tokens per slot (the crossover
between the two kernels).
Prints the card (name, power limit, max SM clock), a markdown table and one JSON line.

    python tools/bench_batched_decode_long.py [--steps 128] [--reps 200]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from vila_b200 import ops, serving  # noqa: E402
from vila_b200.serving import PAGE, SPLIT_LADDER, SPLIT_TOKENS  # noqa: E402

HBM_DATASHEET_GBS = 3350.0  # H100 SXM data sheet
SLOTS = 8
VIDEO, SHORT = 16470, 300
ENGINE_MIXES = {
    "8 x 16470": [VIDEO] * SLOTS,
    "2 x 16470 + 6 x 300": [VIDEO] * 2 + [SHORT] * 6,
    "8 x 300": [SHORT] * SLOTS,
}
# attention alone also at the lengths that place the crossover (n - 1 cached + the new token = n attended)
MIXES = dict(ENGINE_MIXES, **{f"8 x {n}": [n - 1] * SLOTS for n in (1024, 2048, 4096)})


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit not read"


def events_ms(fn, reps, warm=10):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def attention_alone(llm, reps):
    lc = llm.config
    Hq, Hkv, D = lc.num_attention_heads, lc.num_key_value_heads, lc.head_dim
    inv = llm.inv_freq
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    for name, ctxs in MIXES.items():
        pages = [(c + 1 + PAGE - 1) // PAGE for c in ctxs]
        stride = max(pages)
        n_pages = sum(pages)
        kp = torch.randn(n_pages, PAGE, Hkv, D, device="cuda", generator=g).to(torch.bfloat16)
        vp = torch.randn_like(kp)
        perm = torch.randperm(n_pages, device="cuda", generator=g).to(torch.int32)
        pt = torch.zeros(SLOTS, stride, dtype=torch.int32, device="cuda")
        o = 0
        for s, n in enumerate(pages):
            pt[s, :n] = perm[o:o + n]
            o += n
        pos = torch.tensor(ctxs, dtype=torch.int32, device="cuda")
        qkv = torch.randn(SLOTS, (Hq + 2 * Hkv) * D, device="cuda", generator=g).to(torch.bfloat16)
        out = torch.empty(SLOTS, Hq * D, device="cuda", dtype=torch.bfloat16)
        kv_bytes = sum(c + 1 for c in ctxs) * Hkv * D * 2 * 2
        longest = max(ctxs) + 1
        cands = []
        if longest <= 32 * PAGE:  # the head kernel's page table holds 32 pages
            cands.append(("head kernel", lambda: ops.decode_attention_batch(
                qkv, pos, kp, vp, pt, out, inv, Hq, Hkv, D, D ** -0.5)))
        counters = torch.zeros(SLOTS * Hkv, dtype=torch.int32, device="cuda")
        for n in SPLIT_LADDER:
            if n * SPLIT_TOKENS < longest:
                continue
            op = torch.empty(SLOTS * n * Hq * D, device="cuda", dtype=torch.float32)
            lse = torch.empty(SLOTS * n * Hq, device="cuda", dtype=torch.float32)
            cands.append((f"split {n} x {SPLIT_TOKENS}", lambda n=n, op=op, lse=lse: ops.decode_attention_split_batch(
                qkv, pos, kp, vp, pt, out, op, lse, counters, inv, Hq, Hkv, D, n, SPLIT_TOKENS, D ** -0.5)))
        for kname, fn in cands:
            ms = events_ms(fn, reps)
            rows.append({"mix": name, "kernel": kname, "us": round(ms * 1e3, 2), "kv_bytes": kv_bytes,
                         "kv_gbs": round(kv_bytes / ms / 1e6, 1),
                         "kv_frac_of_datasheet_hbm": round(kv_bytes / ms / 1e6 / HBM_DATASHEET_GBS, 4)})
        del kp, vp
        torch.cuda.empty_cache()
    return rows


def prompts_for(llm, ctxs, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ids = torch.randint(0, llm.config.vocab_size, (max(ctxs),), device="cuda", generator=g)
    emb = llm.model.embed_tokens(ids)
    return [emb[:c].clone() for c in ctxs]


def weight_bytes(llm):
    return sum(p.numel() * p.element_size() for n, p in llm.named_parameters() if "embed_tokens" not in n)


def engine(llm, steps, wbytes):
    lc = llm.config
    kv_tok = lc.num_hidden_layers * lc.num_key_value_heads * lc.head_dim * 2 * 2
    rows = []
    for name, ctxs in ENGINE_MIXES.items():
        prompts = prompts_for(llm, ctxs, seed=len(name))
        tokens, pool = serving.slot_geometry(ctxs, steps + 1, 8, SLOTS)
        dec = serving.BatchedDecoder(llm, SLOTS, tokens, max_new=steps + 8, total_pages=pool)
        dec.capture()
        times = []
        for rep in range(2):  # the first pass warms the configurations the timed one uses
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for s, p in enumerate(prompts):
                dec.admit(s, p)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            dec.run(steps)
            b.record()
            torch.cuda.synchronize()
            times.append((t1 - t0, a.elapsed_time(b) / steps))
            config = dec.config
            for s in range(SLOTS):
                dec.release(s)
        prefill_s, step_ms = times[-1]
        kv = sum(c + steps / 2 for c in ctxs) * kv_tok
        byts = wbytes + kv
        del dec
        torch.cuda.empty_cache()
        # the same requests one after another (one of each distinct length, timed warm)
        seq_s = 0.0
        for c in sorted(set(ctxs)):
            p = prompts[ctxs.index(c)]
            llm.generate(inputs_embeds=p, max_new_tokens=steps, eos_token_id=None)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            llm.generate(inputs_embeds=p, max_new_tokens=steps, eos_token_id=None)
            torch.cuda.synchronize()
            seq_s += (time.perf_counter() - t0) * ctxs.count(c)
        batched_s = prefill_s + step_ms * steps / 1e3
        rows.append({"mix": name, "config": "head kernel" if config is None else f"split {config} x {SPLIT_TOKENS}",
                     "step_ms": round(step_ms, 3), "decode_tok_s": round(SLOTS / step_ms * 1e3, 1),
                     "bytes_per_step": int(byts), "gbs": round(byts / step_ms / 1e6, 1),
                     "frac_of_datasheet_hbm": round(byts / step_ms / 1e6 / HBM_DATASHEET_GBS, 4),
                     "batched_end_to_end_s": round(batched_s, 3),
                     "sequential_end_to_end_s": round(seq_s, 3),
                     "batched_tok_s_end_to_end": round(SLOTS * steps / batched_s, 1),
                     "sequential_tok_s_end_to_end": round(SLOTS * steps / seq_s, 1)})
        del prompts
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=128, help="decode steps per timed engine run (>= 100)")
    ap.add_argument("--reps", type=int, default=200, help="timed launches per attention configuration")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from vila_b200.model import LlavaLlamaModel, nvila_8b
    ops.ensure_workspace("cuda")
    who = card()
    model = LlavaLlamaModel(nvila_8b(), device="cuda").init_random(0, device_rng=True)
    llm = model.llm
    with torch.inference_mode():
        att = attention_alone(llm, args.reps)
        eng = engine(llm, args.steps, weight_bytes(llm))
    print(f"card: {who}\n")
    print("attention alone (one layer, 8 slots, CUDA events over %d launches)\n" % args.reps)
    print("| mix | kernel | us | K/V GB/s | share of 3.35 TB/s (data sheet) |\n|---|---|---|---|---|")
    for r in att:
        print(f"| {r['mix']} | {r['kernel']} | {r['us']} | {r['kv_gbs']} | {r['kv_frac_of_datasheet_hbm']:.1%} |")
    print(f"\nwhole engine (NVILA-8B, 8 slots, {args.steps} steps; sequential = llm.generate one request at a time)\n")
    print("| mix | attention | step ms | decode tok/s | GB/s (weights + K/V) | share of 3.35 TB/s (data sheet) "
          "| batched end-to-end s | sequential end-to-end s |\n|---|---|---|---|---|---|---|---|")
    for r in eng:
        print(f"| {r['mix']} | {r['config']} | {r['step_ms']} | {r['decode_tok_s']} | {r['gbs']} | "
              f"{r['frac_of_datasheet_hbm']:.1%} | {r['batched_end_to_end_s']} | {r['sequential_end_to_end_s']} |")
    print(json.dumps({"card": who, "attention": att, "engine": eng, "steps": args.steps}))


if __name__ == "__main__":
    main()
