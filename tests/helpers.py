"""Shared helpers for the parity tests (oracle side only — never imported by vila_b200)."""
from __future__ import annotations

import json
import os
from typing import Dict, List

import torch

from oracle import vila_oracle as O


def oracle_from_state_dict(sd: Dict[str, torch.Tensor], cfg, dtype=torch.float32,
                           device="cpu") -> O.VilaOracleModel:
    """Build the oracle from a reference-named state dict (values are bf16 on any device).
    device="cpu" (default) is the plain CPU oracle; device="cuda" evaluates the SAME plain-PyTorch
    restatement with torch's own fp32 / bf16 library kernels on the GPU, which is what makes the
    full-size BASELINE configurations checkable (fp32 on the host would take minutes per case)."""
    def sub(prefix):
        return {k[len(prefix):]: v.detach().to(device).to(dtype) for k, v in sd.items()
                if k.startswith(prefix)}

    v, l = cfg.vision_tower_cfg, cfg.llm_cfg
    return O.VilaOracleModel(
        vcfg=O.SiglipCfg(v.hidden_size, v.intermediate_size, v.num_hidden_layers, v.num_attention_heads,
                         v.image_size, v.patch_size, v.num_channels, v.layer_norm_eps),
        lcfg=O.Qwen2Cfg(l.hidden_size, l.intermediate_size, l.num_hidden_layers, l.num_attention_heads,
                        l.num_key_value_heads, l.vocab_size, l.rms_norm_eps, l.rope_theta, l.head_dim),
        projector_type=cfg.mm_projector_type,
        vision=sub("vision_tower.vision_tower."), proj=sub("mm_projector."), llm=sub("llm."),
        image_token_id=cfg.image_token_id, newline_token_ids=tuple(cfg.newline_token_ids),
        dynamic_s2=cfg.dynamic_s2, s2_scales=tuple(sorted(cfg.s2_scales)),
        s2_resize_output_to_scale_idx=cfg.s2_resize_output_to_scale_idx)


PARITY_ROWS: List[dict] = []  # every check_close / report_rel call of this process (see conftest.py)


def _record(row: dict) -> None:
    """Keep and print one parity measurement, and append it to $VILA_PARITY_REPORT (default:
    gpurun_out/parity_report.jsonl when that directory exists) so the table can be committed."""
    PARITY_ROWS.append(row)
    print("[parity] " + json.dumps(row))
    out = os.environ.get("VILA_PARITY_REPORT")
    if out is None and os.path.isdir("gpurun_out"):
        out = "gpurun_out/parity_report.jsonl"
    if out:
        try:
            with open(out, "a") as f:
                f.write(json.dumps(row) + "\n")
        except OSError:
            pass


def check_close(name: str, got: torch.Tensor, truth: torch.Tensor, ref_lowp: torch.Tensor = None,
                rel_floor: float = 1e-3, factor: float = 1.6) -> float:
    """Tolerance model for bf16 kernels (stated once here, used by every e2e parity test):

        err(got) <= factor * err(reference's own bf16 path) + rel_floor * max|truth|

    `truth` is the oracle in fp32 on bf16-rounded weights; `ref_lowp` is the oracle run in bf16 with
    the reference's rounding points (unfused torch ops).  I.e. the CUDA path may not be further from
    the fp32 truth than `factor` x the reference's own bf16 noise (+1e-3 relative).  Without `ref_lowp`
    the bound is 2^-7 relative (one bf16 ulp of the largest value) + rel_floor.
    factor: 1.6 by default (the tiny test architecture has few elements, so its max is noisy); the
    full-size tests pass factor=1.3.
    Every call prints and records err, ref_err and their ratio (north_star's "1e-3" is not reachable
    by ANY bf16 pipeline — the reference's own bf16 path misses it — so the ratio to the reference's
    noise is the number to watch: 1.0 = as close to the fp32 truth as the reference itself)."""
    got, truth = got.detach().float().cpu(), truth.detach().float().cpu()
    scale = truth.abs().max().item()
    err = (got - truth).abs().max().item()
    rms = (got - truth).pow(2).mean().sqrt().item()
    row = {"name": name, "scale": round(scale, 5), "err": err, "rel_err": err / max(scale, 1e-30),
           "rms_err": rms}
    if ref_lowp is not None:
        ref = ref_lowp.detach().float().cpu()
        ref_err = (ref - truth).abs().max().item()
        ref_rms = (ref - truth).pow(2).mean().sqrt().item()
        bound = factor * ref_err + rel_floor * scale
        row.update({"ref_err": ref_err, "ref_rel_err": ref_err / max(scale, 1e-30),
                    "ratio_max": err / max(ref_err, 1e-30), "ref_rms_err": ref_rms,
                    "ratio_rms": rms / max(ref_rms, 1e-30), "factor": factor})
    else:
        bound = (2 ** -7 + rel_floor) * scale
    row["bound"] = bound
    row["ok"] = bool(err <= bound)
    _record(row)
    assert err <= bound, f"{name}: err {err:.4e} > bound {bound:.4e} (scale {scale:.3e})"
    return err


def report_rel(name: str, got: torch.Tensor, ref: torch.Tensor, tol: float) -> float:
    """Kernel-level check: max|got - ref| <= tol * max|ref| (ref = fp32 math on bf16-rounded inputs);
    recorded like check_close."""
    got, ref = got.detach().float(), ref.detach().float()
    scale = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    rms = (got - ref).pow(2).mean().sqrt().item()
    rel = err / max(scale, 1e-30)
    _record({"name": name, "scale": round(scale, 5), "err": err, "rel_err": rel, "rms_err": rms,
             "tol": tol, "ok": bool(rel <= tol)})
    assert rel <= tol, f"{name}: rel err {rel:.4e} > {tol:.1e}"
    return rel


def _cdiv(a: int, b: int) -> int:
    return -(-a // b)


# ------------------------------------------------------------------------------------------------
# bf16 projections: a mirror of gemm_bf16's dispatch, the fp64 reference epilogue, the bf16 checker
# ------------------------------------------------------------------------------------------------
GEMM_COUNTER_BYTES = 64 * 1024  # stream-K tile counters at the head of the workspace (16,384 ints)
REGIME = {5128: "splitk-pair", 1128: "stream-k", 128: "tile128", 256: "tile256", 64: "tile64"}


def streamk_fits(M: int, N: int, K: int, sms: int, ws_bytes: int) -> bool:
    """launch_gemm's rule (gemm_wgmma.cu) for running 128 x 128 stream-K: the registered workspace holds
    the tile counters plus (k-iteration slots per tile) fp32 partial tiles of every tile, and there are
    at most 16,384 tiles (one counter each)."""
    tiles = _cdiv(M, 128) * _cdiv(N, 128)
    nkb = _cdiv(K, 64)
    total = tiles * nkb
    ipc = total // min(total, sms)  # k-iterations per CTA (floor)
    slots = _cdiv(nkb, ipc) + 1
    need = GEMM_COUNTER_BYTES + tiles * slots * 128 * 128 * 4
    return ws_bytes >= need and tiles <= 16384


def dispatch_flavour(M: int, N: int, K: int, sms: int, ws_bytes: int) -> int:
    """The kernel gemm_bf16 (vila_linear) picks for an M x N x K problem on `sms` SMs with a registered
    stream-K workspace of ws_bytes, as the vila_linear_cfg code of the same kernel: 5128 split-K CTA
    pairs, 1128 stream-K, 256 / 128 / 64 data-parallel tiles of that width.  Keep it in step with
    gemm_bf16: tests/test_projections_gpu.py checks the two agree bit for bit at every boundary."""
    mb = _cdiv(M, 128)
    tiles128 = mb * _cdiv(N, 128)
    if tiles128 <= sms // 2 and K >= 2048 and M * 10 >= mb * 128 * 9:
        return 5128
    if K >= 8192 and tiles128 < sms:
        if tiles128 * 2 <= sms:  # stream-K when the workspace holds the partials, else plain tiles
            return 1128 if streamk_fits(M, N, K, sms, ws_bytes) else 128
        return 5128
    if mb * _cdiv(N, 256) * 10 >= 7 * sms:
        return 256
    return 64 if N < 128 else 128


def _rb64(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.bfloat16).to(torch.float64)


def linear_reference(P: torch.Tensor, *, bias=None, act: str = None, residual=None,
                     swiglu: bool = False) -> torch.Tensor:
    """The output of one projection in fp64 BEFORE its final bf16 rounding, from the product P = x W^T
    (fp64), rounding to bf16 where the reference's unfused bf16 ops do (and the GEMM epilogue with them):
      * product + bias is rounded before an activation or the residual add;
      * SwiGLU on interleaved (gate, up) columns rounds gate, up and silu(gate);
      * the residual (per output row) is added to the rounded product.
    act: None, "gelu_tanh" or "gelu_erf"."""
    import torch.nn.functional as F
    if swiglu:
        g, u = _rb64(P[:, 0::2]), _rb64(P[:, 1::2])
        return _rb64(F.silu(g)) * u
    t = P if bias is None else P + bias.to(torch.float64)
    if act is not None:
        t = F.gelu(_rb64(t), approximate="tanh" if act == "gelu_tanh" else "none")
    if residual is not None:
        t = _rb64(t) + residual.to(torch.float64)
    return t


def bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    """spacing of bf16 numbers at |x| (8 significant bits): 2^(e-7) for |x| in [2^e, 2^(e+1)); fp64"""
    x = x.to(torch.float64).abs()
    _, e = torch.frexp(x)
    ulp = torch.ldexp(torch.ones_like(x), e - 8)
    return torch.where(x > 0, ulp, torch.full_like(x, 2.0 ** -133))


class Bf16Errors:
    """Per-element, per-row and rounding-bias check of a bf16 output `got` against ref_final, the fp64
    value before its final rounding (linear_reference), with ref = bf16(ref_final).  Fed in row blocks
    (add), so a 16k x 38k output never needs a full fp64 copy.

    The kernel accumulates in fp32, which differs from fp64 by ~1e-6 of the row rms (K <= 19k); that
    alone is far below the tolerance, but where a value lies that close to a bf16 rounding tie, the
    kernel's rounding may go the other way.  Such a flip moves the rounded value by one bf16 ulp, i.e.
    by <= 2^-7 of its magnitude, and one per element is all these inputs produce.
    1. per element:  |got - ref| <= A_ULP * ulp_bf16(ref) + B_RMS * rms(ref row)
       A_ULP = 6: the final rounding (1 ulp), plus one flipped intermediate that scales with the
         output: SwiGLU's rounded up or silu(gate) (<= 2^-7 |out| < 2 ulp(out)), or its rounded
         gate > 0, which moves silu(gate) by <= 1.3 * 2^-7 |silu(gate)| and, through silu(gate)'s own
         rounding, the output by < 2.3 * 2^-7 |out| < 5 ulp(out).
       B_RMS = 2^-4: one flipped intermediate that does NOT scale with the output: the product before
         a residual add (it may cancel against the residual), before GELU, or a negative gate (silu
         near 0); one ulp <= 2^-7 |t|, and |t| stays below 8x the output row's rms for these inputs.
       A fault confined to one tile (a k-block dropped or summed twice: sqrt(64/K) of the row rms per
       element, a residual or bias added wrongly: O(rms)) exceeds this in most of its elements.
    2. per row:  rms(got - ref) over the row <= ROW_RMS * rms(ref row), ROW_RMS = 2^-7.  With correct
       rounding got == ref except at rare flips, so every row is far below; a zeroed, copied or slightly
       wrong tail row fails however small its magnitude is.
    3. rounding bias:  mean over all elements of clamp(sign(ref_final) (got - ref_final) / ulp(ref_final),
       -1, 1) within +-BIAS_ULP = 0.1.  Round-to-nearest gives ~0 (+-0.29/sqrt(n)); round-toward-zero
       or truncation gives ~-0.5, which no max bound sees.  The clamp keeps the rare intermediate flips
       at a cancelling residual (many ulps of a small output, either sign) from dominating the mean."""
    A_ULP = 6.0
    B_RMS = 2.0 ** -4
    ROW_RMS = 2.0 ** -7
    BIAS_ULP = 0.1

    def __init__(self):
        self.excess = 0.0    # max |got - ref| / tolerance
        self.where = None    # (row, col) of that maximum
        self.max_ulps = 0.0  # max |got - ref| / ulp_bf16(max(|ref|, rms(ref row))): ulps of the value,
        #                     or of the row rms where the value is smaller (a cancelling residual)
        self.worst_row = 0.0  # max over rows of rms(got - ref) / rms(ref row)
        self.worst_row_at = None
        self._bias_sum = 0.0
        self.n = 0

    def add(self, got: torch.Tensor, ref_final: torch.Tensor, row0: int = 0) -> "Bf16Errors":
        got = got.to(torch.float64).reshape(-1, ref_final.shape[-1])
        ref_final = ref_final.to(torch.float64).reshape(got.shape)
        ref = _rb64(ref_final)
        diff = got - ref
        ulp = bf16_ulp(ref)
        rms = ref.pow(2).mean(dim=1, keepdim=True).sqrt().clamp_min(1e-30)
        ratio = diff.abs() / (self.A_ULP * ulp + self.B_RMS * rms)
        i = int(ratio.argmax())
        v = ratio.view(-1)[i].item()
        if self.where is None or not v <= self.excess:  # (a NaN sticks)
            self.excess, self.where = v, (row0 + i // got.shape[1], i % got.shape[1])
        self.max_ulps = max(self.max_ulps, (diff.abs() / bf16_ulp(torch.maximum(ref.abs(), rms))).max().item())
        rows = diff.pow(2).mean(dim=1).sqrt() / rms[:, 0]
        r = int(rows.argmax())
        if self.worst_row_at is None or not rows[r].item() <= self.worst_row:
            self.worst_row, self.worst_row_at = rows[r].item(), row0 + r
        signed = torch.sign(ref_final) * (got - ref_final) / bf16_ulp(ref_final)
        self._bias_sum += signed.clamp(-1.0, 1.0).sum().item()
        self.n += signed.numel()
        return self

    @property
    def bias(self) -> float:
        return self._bias_sum / max(self.n, 1)

    def failures(self) -> List[str]:
        out = []
        if not self.excess <= 1.0:
            out.append(f"element {self.where}: error {self.excess:.2f}x the tolerance")
        if not self.worst_row <= self.ROW_RMS:
            out.append(f"row {self.worst_row_at}: rms error {self.worst_row:.3e} of the row rms > {self.ROW_RMS:.3e}")
        if not abs(self.bias) <= self.BIAS_ULP:
            out.append(f"rounding bias {self.bias:+.3f} ulp (|bias| > {self.BIAS_ULP})")
        return out

    def summary(self) -> dict:
        return {"max_ulps": round(self.max_ulps, 2), "excess": round(self.excess, 3),
                "worst_row": float(f"{self.worst_row:.3e}"), "bias_ulp": round(self.bias, 4), "n": self.n}

    def check(self, name: str) -> None:
        bad = self.failures()
        assert not bad, f"{name}: " + "; ".join(bad)


def greedy_ids_match(got: List[int], oracle_ids: List[int], oracle_logits: torch.Tensor,
                     margin: float) -> None:
    """Greedy token ids must be identical, except that the comparison stops at the first step where
    the oracle's own top-2 logit margin is below `margin` (a bf16-level tie: either choice is a
    faithful greedy decode and the continuations legitimately differ)."""
    for i, (a, b) in enumerate(zip(got, oracle_ids)):
        if a == b:
            continue
        top2 = torch.topk(oracle_logits[i].float(), 2).values
        gap = (top2[0] - top2[1]).item()
        assert gap < margin, f"token {i}: got {a}, oracle {b}, oracle top-2 margin {gap:.4f} >= {margin}"
        return
