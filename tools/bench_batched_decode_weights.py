"""The continuous-batching engine (serving.BatchedDecoder) of NVILA-8B (random init) with bf16, FP8 (e4m3,
per-row scale) and W4A16 (4-bit, group-128 scale and zero point; lm_head e4m3) decode weights.

  * per-GEMM kernel time of qkv, o, gate/up, down and lm_head at M = 1, 8, 16 and 32 (two launch groups) in
    every mode, called as the engine calls them (bf16: ops.linear; fp8 / w4a16: ops.gemv_batch), and of the
    single-stream decoder's one-row GEMV (ops.gemv) as the M = 1 baseline: each captured in a CUDA graph
    over all layers' weights (so the weights stream from HBM and no host enqueue is timed), replayed until
    about --kernel-reps launches, CUDA events around the replays; bytes from shapes (weights, their scales
    and zero points, x, y and the residual read) and their share of 3.35 TB/s; the x bytes re-read from
    L2 and the DSMEM bytes of the partition vila_gemv_batch_* use, with its cluster size and the
    cudaOccupancyMaxActiveClusters result for it;
  * engine step: ms per step and aggregate decode tok/s in each mode, modes alternated, median of --reps
    runs of --steps steps after a warm-up, for 8 slots x 300 tokens, 32 slots x 300 tokens and 8 slots x
    16,470 tokens.
Reads the card (name, power limit, max SM clock) with a read-only nvidia-smi query in the same run, prints a
summary and writes batched_decode_weights.json under --out-dir.

    python tools/bench_batched_decode_weights.py [--reps 5] [--steps 64] [--kernel-reps 560] [--out-dir bench_results]
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

HBM_DATASHEET_GBS = 3350.0  # H100 SXM data sheet
MODES = ("bf16", "fp8", "w4a16")
MIXES = {"8x300": (8, [300] * 8), "32x300": (32, [300] * 32), "8x16470": (8, [16470] * 8)}
M_VALUES = (1, 8, 16, 32)


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


def weight_bytes(N, K, fmt):
    if fmt == "bf16":
        return 2 * N * K
    if fmt == "fp8":
        return N * K + 4 * N
    return (N + 15) // 16 * 8 * K + 3 * N * (K // 128)


def graph_us(launch, n_layers, replays):
    """µs per launch: `launch(li)` for every layer li captured in one CUDA graph (no host enqueue in the
    timed window; consecutive launches overlap under PDL as in the engine's graph), replayed `replays`
    times.  Every layer has its own weights, > 50 MB of L2 in all, so each launch streams from HBM."""
    for li in range(n_layers):  # eager warm-up: function attributes, partitions
        launch(li)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for li in range(n_layers):
            launch(li)
    graph.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(replays):
        graph.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / (replays * n_layers)


def gemm_table(llm, copies, launches_per_gemm):
    """Each GEMM as the engine calls it (bf16: ops.linear; fp8 / w4a16: ops.gemv_batch), cycling over all
    layers' weights (lm_head: 8 back-to-back launches of the one head, 0.55-1.1 GB), at every M; and, as the
    M = 1 baseline, the single-row GEMV kernels of the single-stream decoder (ops.gemv) on the same weights."""
    cfg, layers = llm.config, list(llm.model.layers)
    L = len(layers)
    g = torch.Generator(device="cuda").manual_seed(0)
    Hd, I = cfg.hidden_size, cfg.intermediate_size
    xh = torch.randn(max(M_VALUES), Hd, device="cuda", generator=g).to(torch.bfloat16)
    xi = torch.randn(max(M_VALUES), I, device="cuda", generator=g).to(torch.bfloat16)
    res = torch.randn(max(M_VALUES), Hd, device="cuda", generator=g).to(torch.bfloat16)
    bf16_w = {"qkv": lambda l: l._qkv_w, "o": lambda l: l.self_attn.o_proj.weight, "gu": lambda l: l._gu_w,
              "down": lambda l: l.mlp.down_proj.weight}
    cases = [("qkv", "qkv", xh, "bias"), ("o", "o", xh, "residual"), ("gate_up", "gu", xh, "swiglu"),
             ("down", "down", xi, "residual"), ("lm_head", None, xh, "none")]
    rows, fit = [], {}
    for name, key, xx, fusion in cases:
        w0 = llm.lm_head.weight if key is None else bf16_w[key](layers[0])
        N, K = w0.shape
        n_out = N // 2 if fusion == "swiglu" else N
        n_launch = 8 if key is None else L
        replays = max(1, launches_per_gemm // n_launch)
        for mode in MODES:
            fmt = "bf16" if mode == "bf16" else "w4a16" if mode == "w4a16" and key is not None else "fp8"

            def weights(li, mode=mode):  # gemv / gemv_batch weight arguments of layer li (or lm_head)
                if mode == "bf16":
                    return dict(w=w0 if key is None else bf16_w[key](layers[li]))
                q = copies[mode].lm_head if key is None else getattr(copies[mode].layers[li], key)
                return dict(zip(("w", "w_scale", "w_zero"), q))
            part = None if fmt == "bf16" else ops.gemv_batch_partition(N, K, fmt == "fp8")
            if part is not None:
                fit[f"{fmt} N={N} K={K}"] = part
            bias = (lambda li: layers[li]._qkv_b) if fusion == "bias" else (lambda li: None)
            for M in ("gemv",) + M_VALUES:
                m = 1 if M == "gemv" else M
                out = torch.empty(m, n_out, dtype=torch.bfloat16, device="cuda")
                r = res[:m].clone()
                kw = {"residual": dict(residual=r, out=r), "swiglu": dict(swiglu=True, out=out)}.get(
                    fusion, dict(out=out))
                if M == "gemv":  # the single-stream decoder's kernels, one row
                    kw1 = {k: (v[0] if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}
                    launch = (lambda li, kw1=kw1: ops.gemv(xx[0], bias=bias(li), static_w=True, **weights(li), **kw1))
                elif fmt == "bf16":
                    launch = (lambda li, m=m, kw=kw: ops.linear(xx[:m], static_w=True, bias=bias(li),
                                                                **weights(li), **kw))
                else:
                    launch = (lambda li, m=m, kw=kw: ops.gemv_batch(xx[:m], static_w=True, bias=bias(li),
                                                                    **weights(li), **kw))
                us = graph_us(launch, n_launch, replays)
                launches = (m + 15) // 16 if fmt != "bf16" and M != "gemv" else 1
                byts = (weight_bytes(N, K, fmt) * launches + 2 * m * K + 2 * m * n_out
                        + (2 * m * N if fusion == "residual" else 0) + (2 * N if fusion == "bias" else 0))
                row = {"gemm": name, "mode": mode, "format": fmt, "N": N, "K": K, "M": M, "launches": launches,
                       "us": round(us, 2), "bytes": byts, "gbs": round(byts / us / 1e3, 1),
                       "frac_of_datasheet_hbm": round(byts / us / 1e3 / HBM_DATASHEET_GBS, 4)}
                if part is not None and M != "gemv":
                    clusters = part["ctas"] // part["cluster"]
                    row.update(cluster=part["cluster"], ctas=part["ctas"],
                               x_reread_bytes=clusters * 2 * m * K,  # each cluster stages every x row once
                               dsmem_bytes=4 * m * N * part["cluster"] if part["cluster"] > 1 else 0)
                rows.append(row)
    return rows, fit


def engine_table(llm, reps, steps):
    g = torch.Generator(device="cuda").manual_seed(1)
    rows = []
    for mix, (slots, ctxs) in MIXES.items():
        ids = torch.randint(0, llm.config.vocab_size, (max(ctxs),), device="cuda", generator=g)
        emb = llm.model.embed_tokens(ids)
        tokens = (max(ctxs) + (reps + 1) * steps + 8 + 127) // 128 * 128
        decs = {}
        for mode in MODES:  # one decoder per mode, every slot admitted; each holds its mode's copies
            llm.set_decode_weights(mode)
            dec = serving.BatchedDecoder(llm, slots, tokens, max_new=(reps + 1) * steps + 8)
            dec.capture()
            for s, c in enumerate(ctxs):
                dec.admit(s, emb[:c].clone())
            dec.run(steps)  # warm-up
            decs[mode] = dec
        llm.set_decode_weights("bf16")
        times = {m: [] for m in MODES}
        for _ in range(reps):
            for mode in MODES:  # alternated: every mode sees the same contexts and the same card state
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                decs[mode].run(steps)
                b.record()
                torch.cuda.synchronize()
                times[mode].append(a.elapsed_time(b) / steps)
        for mode in MODES:
            med = statistics.median(times[mode])
            rows.append({"mix": mix, "slots": slots, "mode": mode, "attention": decs[mode].config,
                         "step_ms": round(med, 3), "step_ms_all": [round(t, 3) for t in times[mode]],
                         "decode_tok_s": round(len(ctxs) / med * 1e3, 1)})
        del decs, emb
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed engine runs per mode (alternated)")
    ap.add_argument("--steps", type=int, default=64, help="decode steps per timed engine run")
    ap.add_argument("--kernel-reps", type=int, default=560, help="timed launches per GEMM (whole graph replays)")
    ap.add_argument("--out-dir", type=str, default="bench_results")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from vila_b200.model import LlavaLlamaModel, nvila_8b
    ops.ensure_workspace("cuda")
    who = card()
    model = LlavaLlamaModel(nvila_8b(), device="cuda").init_random(0, device_rng=True)
    llm = model.llm
    with torch.inference_mode():
        copies = {}
        for mode in ("fp8", "w4a16"):
            llm.set_decode_weights(mode)
            copies[mode] = llm._fp8_weights if mode == "fp8" else llm._w4_weights
        llm.set_decode_weights("bf16")
        gemms, fit = gemm_table(llm, copies, args.kernel_reps)
        del copies
        torch.cuda.empty_cache()
        eng = engine_table(llm, args.reps, args.steps)
    res = {"card": who, "model": "NVILA-8B LLM, random init", "gemm": gemms, "partition": fit, "engine": eng,
           "steps": args.steps, "reps": args.reps, "kernel_reps": args.kernel_reps}
    print(f"card: {who}\n")
    print("| gemm | mode | M | us | GB/s | share of 3.35 TB/s | cluster | x re-read MB | DSMEM MB |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in gemms:
        print(f"| {r['gemm']} | {r['mode']} | {r['M']} | {r['us']} | {r['gbs']} | {r['frac_of_datasheet_hbm']:.1%} | "
              f"{r.get('cluster', '-')} | {r.get('x_reread_bytes', 0) / 1e6:.2f} | {r.get('dsmem_bytes', 0) / 1e6:.2f} |")
    print("\npartition (cluster, CTAs, tiles per cluster, k-parts, max active clusters, smem):")
    for k, v in fit.items():
        print(f"  {k}: {v}")
    print("\n| mix | mode | step ms (median) | decode tok/s | all |\n|---|---|---|---|---|")
    for r in eng:
        print(f"| {r['mix']} | {r['mode']} | {r['step_ms']} | {r['decode_tok_s']} | {r['step_ms_all']} |")
    out = Path(args.out_dir)
    out.mkdir(parents=True, exist_ok=True)
    (out / "batched_decode_weights.json").write_text(json.dumps(res, indent=1))
    print(json.dumps({"card": who, "engine": eng}))


if __name__ == "__main__":
    main()
