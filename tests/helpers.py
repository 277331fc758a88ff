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
