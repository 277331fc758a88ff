"""Times every vila_linear tile configuration at the Qwen2-7B projection shapes for a few token counts
(decode batches and a one-image prefill) and at two ViT shapes, and prints a markdown table of
microseconds per call (CUDA events, warm, weights static).  `auto` is the dispatcher's own choice.

    python tools/bench_gemm_dispatch.py [M ...]
"""
import math
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from vila_b200 import ops  # noqa: E402

CONFIGS = [None, 64, 128, 256, 1064, 1128, 1256, 5128]
LLM = {"qkv": (4608, 3584), "o": (3584, 3584), "gate/up": (37888, 3584), "down": (3584, 18944)}
VIT = [("ViT qkv, 1 image", 1024, 3456, 1152), ("ViT fc1, 64 frames", 65536, 4304, 1152)]


def time_us(x, w, bn, reps):
    out = ops.linear(x, w, block_n=bn, static_w=True)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        ops.linear(x, w, block_n=bn, static_w=True, out=out)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / reps


def main():
    ms = [int(v) for v in sys.argv[1:]] or [8, 32, 279]
    ops.ensure_workspace("cuda")
    p = torch.cuda.get_device_properties(0)
    print(f"{p.name}, {p.multi_processor_count} SMs; us per call (auto = default dispatch)\n")
    print("| shape | M | N | K | " + " | ".join("auto" if c is None else str(c) for c in CONFIGS) + " |")
    print("|---|---|---|---|" + "---|" * len(CONFIGS))
    rows = [(f"{n}", m, N, K) for m in ms for n, (N, K) in LLM.items()] + VIT
    for name, M, N, K in rows:
        g = torch.Generator(device="cuda").manual_seed(1)
        x = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
        w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(torch.bfloat16)
        cells = []
        for bn in CONFIGS:
            try:
                cells.append("%.1f" % time_us(x, w, bn, 20 if M < 4096 else 5))
            except RuntimeError:
                cells.append("-")
        print(f"| {name} | {M} | {N} | {K} | " + " | ".join(cells) + " |")
        del x, w


if __name__ == "__main__":
    main()
