"""Prefix caching in the continuous-batching engine on NVILA-8B (random init), 8 slots, 128 new tokens, EOS off.

Each workload is served with and without prefix caching, alternated, median of --reps runs; the prefix-caching
engine's cache is cleared before every run, so the first request of a run is always prefilled in full.  Per workload:
end-to-end time, admission time per request (host clock around BatchedDecoder.admit with a device synchronise on
both sides), the time per request of the digests that generate_batch computes before admit (prefix_digests: one hash
launch and the copy to the host, timed the same way) and the tokens served from the cache.  Workloads:

  * video QA    8 prompts of 16,470 tokens sharing the first 16,384 (8 questions on one 64-frame video);
  * image QA    8 prompts of 300 tokens sharing the first 256;
  * no sharing  8 distinct 16,470-token prompts: the cost of hashing and bookkeeping when nothing hits;
  * the hash kernel alone at 16,470 x 3584 (CUDA events): time, GB/s and its share of the 3.35 TB/s of the H100 SXM
    data sheet;
  * model level: 8 questions on one 64-frame video through LlavaLlamaModel.generate_batch, with the time of
    _embed (vision tower + projector + splice, run for every request) reported on its own.

Prints the card (name, power limit, max SM clock), a markdown table and one JSON line.

    python tools/bench_prefix_cache.py [--reps 5] [--new 128]
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
from vila_b200 import ops, serving  # noqa: E402
from vila_b200.serving import PAGE  # noqa: E402

HBM_DATASHEET_GBS = 3350.0  # H100 SXM data sheet
SLOTS, CHECK = 8, 8
VIDEO, VIDEO_SHARED = 16470, 16384
IMAGE, IMAGE_SHARED = 300, 256


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit not read"


def embeddings(llm, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ids = torch.randint(0, llm.config.vocab_size, (n,), device="cuda", generator=g)
    return llm.model.embed_tokens.weight[ids].clone()


def sharing(llm, total, shared, seed):
    head = embeddings(llm, shared, seed)
    return [torch.cat([head, embeddings(llm, total - shared, seed + 1 + k)]) for k in range(SLOTS)]


class Timed:
    """wraps a decoder method with a host clock between two device synchronises"""

    def __init__(self, dec, name):
        self.inner, self.times = getattr(dec, name), []
        setattr(dec, name, self)

    def __call__(self, *args, **kw):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = self.inner(*args, **kw)
        torch.cuda.synchronize()
        self.times.append(time.perf_counter() - t0)
        return r


def serve(llm, dec, prompts, new, prefix):
    if prefix:
        dec.clear_prefix_cache()
    before = dec.prefix_stats["hit_tokens"] if prefix else 0
    timer = dec.admit
    timer.times.clear()
    hashing = dec.prefix_digests if prefix else None
    if prefix:
        hashing.times.clear()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = serving.generate_batch(llm, prompts, new, (), check_every=CHECK, decoder=dec, prefix_cache=prefix)
    torch.cuda.synchronize()
    e2e = time.perf_counter() - t0
    assert all(len(o) == new for o in out)
    hit = (dec.prefix_stats["hit_tokens"] - before) if prefix else 0
    return e2e, statistics.mean(timer.times), hit, sum(hashing.times) / len(prompts) if prefix else 0.0


def workload(llm, decs, prompts, new, reps):
    res = {True: [], False: []}
    for prefix in (True, False):  # warm-up
        serve(llm, decs[prefix], prompts, new, prefix)
    for _ in range(reps):
        for prefix in (True, False):
            res[prefix].append(serve(llm, decs[prefix], prompts, new, prefix))
    row = {}
    for prefix, runs in res.items():
        e2e = [r[0] for r in runs]
        row["on" if prefix else "off"] = dict(e2e_s=statistics.median(e2e), e2e_min_s=min(e2e), e2e_max_s=max(e2e),
                                             admit_ms=1e3 * statistics.median(r[1] for r in runs),
                                             digest_ms=1e3 * statistics.median(r[3] for r in runs),
                                             cached_tokens=runs[0][2])
    row["speedup"] = row["off"]["e2e_s"] / row["on"]["e2e_s"]
    return row


def hash_kernel(llm, reps=200):
    x = embeddings(llm, VIDEO, 99)
    for _ in range(10):
        ops.prefix_block_hash(x, 1, 2)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        ops.prefix_block_hash(x, 1, 2)
    b.record()
    torch.cuda.synchronize()
    us = 1e3 * a.elapsed_time(b) / reps
    nbytes = (VIDEO // PAGE) * PAGE * x.shape[1] * 2
    gbs = nbytes / us / 1e3
    return dict(us=us, bytes=nbytes, gbs=gbs, share_of_hbm=gbs / HBM_DATASHEET_GBS)


def model_level(model, new, reps):
    cfg = model.config
    g = torch.Generator(device="cuda").manual_seed(7)
    frames = torch.randn(64, 3, 448, 448, device="cuda", generator=g).to(torch.bfloat16)
    reqs = []
    for k in range(SLOTS):
        q = torch.randint(100, 20000, (60 + k,), generator=torch.Generator().manual_seed(k)).tolist()
        ids = torch.tensor([[100, 101, 102, cfg.video_token_id] + q])
        reqs.append({"input_ids": ids, "media": {"video": [frames]}, "media_config": {"video": {}}})
    # _embed alone, per request
    for r in reqs[:1]:
        model._embed(r["input_ids"], r["media"], r["media_config"], None, None)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for r in reqs:
        emb, _, _ = model._embed(r["input_ids"], r["media"], r["media_config"], None, None)
    torch.cuda.synchronize()
    embed_s = (time.perf_counter() - t0) / len(reqs)
    S = emb.shape[1]
    tokens = (S + SLOTS + new + CHECK + PAGE - 1) // PAGE * PAGE
    res = {True: [], False: []}
    for prefix in (True, False, True, False):  # the first pair warms up
        model.generate_batch(reqs, new, slots=SLOTS, max_tokens_per_slot=tokens, eos_token_id=[], prefix_cache=prefix)
    for _ in range(reps):
        for prefix in (True, False):
            if prefix:
                model._prefix_engine[1].clear_prefix_cache()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model.generate_batch(reqs, new, slots=SLOTS, max_tokens_per_slot=tokens, eos_token_id=[],
                                 prefix_cache=prefix)
            torch.cuda.synchronize()
            res[prefix].append(time.perf_counter() - t0)
    st = model._prefix_engine[1].prefix_stats
    on, off = statistics.median(res[True]), statistics.median(res[False])
    return dict(prompt_tokens=S, embed_s_per_request=embed_s, on_e2e_s=on, off_e2e_s=off, speedup=off / on,
                on_spread_s=max(res[True]) - min(res[True]), off_spread_s=max(res[False]) - min(res[False]),
                hit_tokens_last_run=st["hit_tokens"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--new", type=int, default=128)
    ap.add_argument("--skip-model-level", action="store_true")
    args = ap.parse_args()
    from vila_b200.model import LlavaLlamaModel, nvila_video_8b
    info = card()
    print(f"card: {info}", flush=True)
    model = LlavaLlamaModel(nvila_video_8b(), device="cuda").init_random(0, device_rng=True)
    llm = model.llm
    tokens = (VIDEO + args.new + CHECK + PAGE - 1) // PAGE * PAGE
    decs = {}
    for prefix in (True, False):
        decs[prefix] = serving.BatchedDecoder(llm, SLOTS, tokens, max_new=args.new, prefix_cache=prefix)
        decs[prefix].capture()
        Timed(decs[prefix], "admit")
        if prefix:
            Timed(decs[prefix], "prefix_digests")
    rows = {
        "video QA 8 x 16470 (16384 shared)": workload(llm, decs, sharing(llm, VIDEO, VIDEO_SHARED, 1), args.new,
                                                       args.reps),
        "image QA 8 x 300 (256 shared)": workload(llm, decs, sharing(llm, IMAGE, IMAGE_SHARED, 2), args.new,
                                                   args.reps),
        "no sharing 8 x 16470": workload(llm, decs, [embeddings(llm, VIDEO, 300 + k) for k in range(SLOTS)],
                                         args.new, args.reps),
    }
    hk = hash_kernel(llm)
    decs.clear()
    torch.cuda.empty_cache()
    ml = None if args.skip_model_level else model_level(model, args.new, max(3, args.reps - 2))
    print(f"\nNVILA-8B random init, {SLOTS} slots, {args.new} new tokens, EOS off; median of {args.reps} "
          f"(alternated); card: {info}\n")
    print("| workload | e2e off (s) | e2e on (s) | speedup | admit/request off (ms) | admit/request on (ms) "
          "| digests/request on (ms) | tokens from cache | off min..max (s) | on min..max (s) |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for name, r in rows.items():
        print(f"| {name} | {r['off']['e2e_s']:.3f} | {r['on']['e2e_s']:.3f} | {r['speedup']:.2f}x | "
              f"{r['off']['admit_ms']:.1f} | {r['on']['admit_ms']:.1f} | {r['on']['digest_ms']:.2f} | "
              f"{r['on']['cached_tokens']} | "
              f"{r['off']['e2e_min_s']:.3f}..{r['off']['e2e_max_s']:.3f} | "
              f"{r['on']['e2e_min_s']:.3f}..{r['on']['e2e_max_s']:.3f} |")
    print(f"\nhash kernel at {VIDEO} x 3584: {hk['us']:.1f} us, {hk['gbs']:.0f} GB/s = "
          f"{100 * hk['share_of_hbm']:.1f}% of {HBM_DATASHEET_GBS:.0f} GB/s")
    if ml:
        print(f"model level, 8 questions on one 64-frame video ({ml['prompt_tokens']} tokens): off "
              f"{ml['off_e2e_s']:.3f} s, on {ml['on_e2e_s']:.3f} s ({ml['speedup']:.2f}x); _embed "
              f"{ml['embed_s_per_request'] * 1e3:.1f} ms per request (8 per call)")
    print(json.dumps({"card": info, "workloads": rows, "hash_kernel": hk, "model_level": ml}))


if __name__ == "__main__":
    main()
