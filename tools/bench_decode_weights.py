"""Single-stream greedy decode of NVILA-8B (random init) with bf16, FP8 (e4m3, per-row scale) and W4A16 (4-bit,
group-128 scale and zero point; lm_head e4m3) decode weights.

  * decode speed: GraphDecoder in each mode, alternating bf16 / fp8 / w4a16 for --reps repeats after a
    warm-up, after a 279-token prompt (one image) and a 16,470-token prompt (64-frame video), --steps tokens
    each; CUDA events around the graph replays -> ms/token and tok/s, with the spread over the repeats;
  * per-GEMV kernel time (CUDA events over --kernel-reps back-to-back launches) of layer 0's qkv, o,
    gate/up, down and of lm_head in every mode; achieved bytes/s from the bytes the kernel must read
    (the weights, their scales and zero points, and 2K bytes of x) and its share of 3.35 TB/s;
  * weight bytes per token and the HBM bound they imply; peak allocated memory of llm.generate at the
    long prompt in each mode;
  * for information: the first step where the bf16 greedy ids and each quantized mode's part.
Reads the card (name, power limit, max SM clock) with a read-only nvidia-smi query in the same run, prints a
summary and writes decode_weights.json under --out-dir.

    python tools/bench_decode_weights.py [--reps 5] [--steps 128] [--kernel-reps 200] [--out-dir bench_results]
"""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from vila_b200 import ops  # noqa: E402

HBM_DATASHEET_GBS = 3350.0  # H100 SXM data sheet
PROMPTS = {"image-279": 279, "video-16470": 16470}
MODES = ("bf16", "fp8", "w4a16")


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


def spread(xs):
    return {"median": round(statistics.median(xs), 4), "min": round(min(xs), 4), "max": round(max(xs), 4),
            "all": [round(x, 4) for x in xs]}


def weight_bytes(N, K, mode):
    """bytes of an [N, K] weight in a mode: bf16; e4m3 + fp32 row scales; 4-bit codes (16-row tiles) + bf16
    scales and uint8 zero points per group of 128"""
    if mode == "bf16":
        return 2 * N * K
    if mode == "fp8":
        return N * K + 4 * N
    return (N + 15) // 16 * 8 * K + 3 * N * (K // 128)


def decode_weight_bytes(llm, mode):
    """weight bytes one decode token streams: every layer's qkv, o, gate/up, down and lm_head (e4m3 in the
    w4a16 mode)"""
    mats = []
    for layer in llm.model.layers:
        mats += [layer._qkv_w, layer.self_attn.o_proj.weight, layer._gu_w, layer.mlp.down_proj.weight]
    head = tuple(llm.lm_head.weight.shape)
    return (sum(weight_bytes(*m.shape, mode) for m in mats)
            + weight_bytes(*head, "bf16" if mode == "bf16" else "fp8"))


def copy_bytes(copies):
    """bytes held by a mode's quantized copies (every tensor in them)"""
    ts = list(copies.lm_head) + [x for f in copies.layers for w in (f.qkv, f.o, f.gu, f.down) for x in w]
    return sum(t.numel() * t.element_size() for t in ts)


def gemv_table(llm, fp8, w4, reps):
    """layer 0's GEMVs and lm_head alone, each mode (fp8, w4: the copies of those modes)"""
    cfg, layer = llm.config, llm.model.layers[0]
    g = torch.Generator(device="cuda").manual_seed(0)
    Hd, I = cfg.hidden_size, cfg.intermediate_size
    x = torch.randn(Hd, device="cuda", generator=g).to(torch.bfloat16)
    xi = torch.randn(I, device="cuda", generator=g).to(torch.bfloat16)
    key = torch.zeros(1, dtype=torch.int64, device="cuda")
    nrm = dict(norm_w=layer.input_layernorm.weight, norm_eps=cfg.rms_norm_eps)
    l8, l4 = fp8.layers[0], w4.layers[0]
    cases = [  # (name, bf16 weight, fp8 (q, s), w4a16 (packed, s, z) or e4m3 for lm_head, x, kwargs)
        ("qkv", layer._qkv_w, l8.qkv, l4.qkv, x, dict(bias=layer._qkv_b, **nrm)),
        ("o", layer.self_attn.o_proj.weight, l8.o, l4.o, x, dict(residual=x)),
        ("gate_up", layer._gu_w, l8.gu, l4.gu, x, dict(swiglu=True, **nrm)),
        ("down", layer.mlp.down_proj.weight, l8.down, l4.down, xi, dict(residual=x)),
        ("lm_head", llm.lm_head.weight, fp8.lm_head, w4.lm_head, x,
         dict(argmax_key=key, write_out=False, norm_w=llm.model.norm.weight, norm_eps=cfg.rms_norm_eps)),
    ]
    rows = []
    for name, w, q8, q4, xx, kw in cases:
        N, K = w.shape
        for mode in MODES:
            if mode == "bf16":
                wk, fmt = dict(w=w), "bf16"
            elif mode == "fp8" or name == "lm_head":  # the w4a16 mode's lm_head is e4m3
                wk, fmt = dict(zip(("w", "w_scale"), q8 if mode == "fp8" else q4)), "fp8"
            else:
                wk, fmt = dict(zip(("w", "w_scale", "w_zero"), q4)), "w4a16"
            out = None if kw.get("write_out") is False else torch.empty(
                N // 2 if kw.get("swiglu") else N, dtype=torch.bfloat16, device="cuda")
            ms = events_ms(lambda: ops.gemv(xx, out=out, static_w=True, **wk, **kw), reps)
            byts = weight_bytes(N, K, fmt) + 2 * K
            rows.append({"gemv": name, "mode": mode, "format": fmt, "N": N, "K": K, "us": round(ms * 1e3, 2), "bytes": byts,
                         "gbs": round(byts / ms / 1e6, 1),
                         "frac_of_datasheet_hbm": round(byts / ms / 1e6 / HBM_DATASHEET_GBS, 4)})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed bf16 / fp8 / w4a16 alternations per prompt")
    ap.add_argument("--steps", type=int, default=128, help="greedy tokens per timed run")
    ap.add_argument("--kernel-reps", type=int, default=200, help="timed launches per GEMV")
    ap.add_argument("--out-dir", type=str, default="bench_results")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from vila_b200.model import GraphDecoder, LlavaLlamaModel, nvila_8b
    ops.ensure_workspace("cuda")
    who = card()
    model = LlavaLlamaModel(nvila_8b(), device="cuda").init_random(0, device_rng=True)
    llm = model.llm
    res = {"card": who, "model": "NVILA-8B LLM, random init", "steps": args.steps, "reps": args.reps,
           "launches_per_token": None, "decode": {}, "first_divergence": {}}
    with torch.inference_mode():
        g = torch.Generator(device="cuda").manual_seed(1)
        ids = torch.randint(0, llm.config.vocab_size, (max(PROMPTS.values()),), device="cuda", generator=g)
        emb_all = llm.model.embed_tokens(ids)
        # one decoder per (mode, prompt), each with its own prefilled cache; a GraphDecoder keeps the
        # weights of the mode it was built in
        decs = {}
        copies = {}
        for mode in MODES:
            llm.set_decode_weights(mode)
            copies[mode] = llm._fp8_weights if mode == "fp8" else llm._w4_weights
            for pname, S in PROMPTS.items():
                dec = GraphDecoder(llm, args.steps + 8)
                cache = dec.cache_for(S + args.steps + 1)
                last = llm.prefill_hidden(emb_all[:S].clone(), cache)[-1].clone()
                decs[mode, pname] = (dec, cache, S, last)
        llm.set_decode_weights("bf16")  # the decoders of the quantized modes hold their copies

        def run(mode, pname):
            dec, cache, S, last = decs[mode, pname]
            cache.length = S
            dec.start(last, cache)
            dec.run(1)  # the first token came from start()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            dec.run(args.steps)
            b.record()
            torch.cuda.synchronize()
            return a.elapsed_time(b) / args.steps, dec.tokens(args.steps + 1)

        for key in decs:  # warm-up: captures every graph the timed runs replay
            run(*key)
        res["launches_per_token"] = decs["bf16", "image-279"][0].launches_per_step
        for pname in PROMPTS:
            ms = {mode: [] for mode in MODES}
            toks = {}
            for _ in range(args.reps):
                for mode in MODES:
                    t, toks[mode] = run(mode, pname)
                    ms[mode].append(t)
            row = {}
            for mode in MODES:
                row[mode] = {"ms_per_token": spread(ms[mode]),
                             "tok_s": spread([1e3 / t for t in ms[mode]]),
                             "splits": [decs[mode, pname][0].num_splits, decs[mode, pname][0].split_tokens],
                             "speedup_over_bf16": round(statistics.median(ms["bf16"]) / statistics.median(ms[mode]), 3)}
            row["w4a16_over_fp8"] = round(statistics.median(ms["fp8"]) / statistics.median(ms["w4a16"]), 3)
            res["decode"][pname] = row
            res["first_divergence"][pname] = {
                mode: next((i for i, (a, b) in enumerate(zip(toks["bf16"], toks[mode])) if a != b), None)
                for mode in MODES[1:]}
        res["gemv"] = gemv_table(llm, copies["fp8"], copies["w4a16"], args.kernel_reps)
        for mode in MODES:
            byts = decode_weight_bytes(llm, mode)
            ms_med = res["decode"]["image-279"][mode]["ms_per_token"]["median"]
            res.setdefault("weights", {})[mode] = {
                "bytes_per_token": byts, "hbm_bound_tok_s": round(HBM_DATASHEET_GBS * 1e9 / byts, 1),
                "achieved_gbs_image_279": round(byts / ms_med / 1e6, 1)}
        res["copy_bytes"] = {mode: copy_bytes(copies[mode]) for mode in MODES[1:]}
        decs.clear()
        copies.clear()
        torch.cuda.empty_cache()
        S = PROMPTS["video-16470"]
        peaks = {}
        for mode in MODES:
            llm.set_decode_weights(mode)
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            llm.generate(inputs_embeds=emb_all[:S], max_new_tokens=args.steps, eos_token_id=None)
            torch.cuda.synchronize()
            peaks[mode] = torch.cuda.max_memory_allocated()
        res["peak_allocated_bytes_generate_video_16470"] = peaks
        llm.set_decode_weights("bf16")

    print(f"card: {who}")
    print(f"launches per token: {res['launches_per_token']}")
    print("\n| prompt | mode | ms/token (median, min-max) | tok/s (median) | over bf16 |\n|---|---|---|---|---|")
    for pname, row in res["decode"].items():
        for mode in MODES:
            m = row[mode]["ms_per_token"]
            print(f"| {pname} | {mode} | {m['median']:.3f} ({m['min']:.3f}-{m['max']:.3f}) | "
                  f"{row[mode]['tok_s']['median']:.1f} | {row[mode]['speedup_over_bf16']} |")
        print(f"| {pname} | w4a16 over fp8 | | | {row['w4a16_over_fp8']} |")
    print("\n| gemv | mode | format | N x K | us | GB/s | share of 3.35 TB/s |\n|---|---|---|---|---|---|---|")
    for r in res["gemv"]:
        print(f"| {r['gemv']} | {r['mode']} | {r['format']} | {r['N']} x {r['K']} | {r['us']} | {r['gbs']} | "
              f"{r['frac_of_datasheet_hbm']:.1%} |")
    print(f"\nweights: {json.dumps(res['weights'])}")
    print(f"peak allocated (generate, 16470-token prompt): {json.dumps(peaks)}; copies {json.dumps(res['copy_bytes'])}")
    print(f"first step where bf16 ids and each mode's part: {json.dumps(res['first_divergence'])}")
    out = Path(args.out_dir)
    out.mkdir(parents=True, exist_ok=True)
    (out / "decode_weights.json").write_text(json.dumps(res, indent=1))
    print(json.dumps({k: res[k] for k in ("card", "decode", "weights")}))


if __name__ == "__main__":
    main()
