"""Shared helpers for the parity tests (oracle side only — never imported by vila_b200)."""
from __future__ import annotations

import json
import math
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

    def add(self, got: torch.Tensor, ref_final: torch.Tensor, row0: int = 0, allow: torch.Tensor = None,
            row_scale: torch.Tensor = None) -> "Bf16Errors":
        """allow: per-element allowance that replaces B_RMS * rms(ref row) in check 1 (shape of got);
        row_scale: per-row scale that replaces rms(ref row) in check 2 (one value per row)."""
        got = got.to(torch.float64).reshape(-1, ref_final.shape[-1])
        ref_final = ref_final.to(torch.float64).reshape(got.shape)
        ref = _rb64(ref_final)
        diff = got - ref
        ulp = bf16_ulp(ref)
        rms = ref.pow(2).mean(dim=1, keepdim=True).sqrt().clamp_min(1e-30)
        extra = self.B_RMS * rms if allow is None else allow.to(torch.float64).reshape(got.shape)
        ratio = diff.abs() / (self.A_ULP * ulp + extra)
        i = int(ratio.argmax())
        v = ratio.view(-1)[i].item()
        if self.where is None or not v <= self.excess:  # (a NaN sticks)
            self.excess, self.where = v, (row0 + i // got.shape[1], i % got.shape[1])
        self.max_ulps = max(self.max_ulps, (diff.abs() / bf16_ulp(torch.maximum(ref.abs(), rms))).max().item())
        scale = rms[:, 0] if row_scale is None else row_scale.to(torch.float64).reshape(-1)
        rows = diff.pow(2).mean(dim=1).sqrt() / scale
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
            out.append(f"row {self.worst_row_at}: rms error {self.worst_row:.3e} x the row scale > {self.ROW_RMS:.3e}")
        if not abs(self.bias) <= self.BIAS_ULP:
            out.append(f"rounding bias {self.bias:+.3f} ulp (|bias| > {self.BIAS_ULP})")
        return out

    def summary(self) -> dict:
        return {"max_ulps": round(self.max_ulps, 2), "excess": round(self.excess, 3),
                "worst_row": float(f"{self.worst_row:.3e}"), "bias_ulp": round(self.bias, 4), "n": self.n}

    def check(self, name: str) -> None:
        bad = self.failures()
        assert not bad, f"{name}: " + "; ".join(bad)


# ------------------------------------------------------------------------------------------------
# prefill attention: the fp64 reference, the checker, and the three input families
# ------------------------------------------------------------------------------------------------
class AttnErrors(Bf16Errors):
    """Bf16Errors for one attention output [Sq, Hq, D] against the fp64 reference of attention_reference.
    A row is one (query, head) pair: rows are numbered query * Hq + head.

    The kernel (fmha_wgmma.cu) computes, per row, o = sum_j bf16(p_j) v_j / l with p_j = exp2(s_j *
    scale*log2(e) - m) for a running maximum m, l = sum_j p_j summed from the UNROUNDED p_j, and rounds
    o / l to bf16 once.  Every common factor of p (the stale maxima, the alpha rescales) cancels between
    the numerator and l, so the only error that does not cancel is the rounding of each p_j to bf16,
    relative error delta_j with |delta_j| <= 2^-8 (the bf16 unit roundoff; p >= 2^-126 stays normal):
        e_d = sum_j delta_j p_j v_jd / l,   |e_d| <= 2^-8 * A_d,   A_d = sum_j p_j |v_jd| / l.
    1. per element:  |got - bf16(ref_final)| <= A_ULP * ulp_bf16(ref) + P_ROUND * A_d
       A_ULP = 1: the output's own rounding, which may go the other way at a tie once e_d moves the
         value across it (|got - ref| <= |e_d| + 1 ulp).
       P_ROUND = 2^-7, twice the bound on e_d: the factor 2 absorbs the fp32 score accumulation, the
         fp32 products s * scale*log2(e), ex2.approx (relative error ~2^-22) and the fp32 alpha
         products, each below 2^-11 of p for scores within a few thousand of the row maximum.
         tests/test_attention_cpu.py checks this on an emulation of that arithmetic.
    2. per row:  rms_d(got - ref) <= ROW_RMS * sqrt(mean_d(2^-16 * S2_d + ulp_d^2 / 4)),
       S2_d = sum_j p_j^2 v_jd^2 / l^2.  The delta_j are independent, so e_d has a standard deviation
       of at most 2^-8 sqrt(S2_d); rounding then adds E[(got - ref)^2] <= e_d^2 + ulp^2 / 4.  The bound
       falls as attention spreads over more keys (S2 ~ |v|^2 / n_keys), so one leaked or dropped key
       still shows in a long row where the per-element bound (~ 2^-7 |v|) would not see it.
       ROW_RMS = 3: elementwise |got - ref| <= |e_d| + ulp_d, so rms(got - ref)^2 <= 2 rms(e)^2 +
       2 mean(ulp^2), which is within 9 x (2^-16 mean(S2) + mean(ulp^2) / 4) as long as rms(e) stays
       within 2.1 x its bound 2^-8 sqrt(mean(S2)) (a row of only 72 elements may sample it high).  A row
       in which every element is one ulp off and e is negligible sits at 2.
    3. rounding bias: as Bf16Errors.  Truncating P or the output moves every value toward zero by a
       fraction of an ulp; only the mean sees it."""
    A_ULP = 1.0
    P_ROUND = 2.0 ** -7
    ROW_RMS = 3.0

    def add_attention(self, got: torch.Tensor, ref_final: torch.Tensor, A: torch.Tensor, S2: torch.Tensor,
                      row0: int = 0) -> "AttnErrors":
        D = ref_final.shape[-1]
        ulp = bf16_ulp(_rb64(ref_final.to(torch.float64)))
        row_scale = (2.0 ** -16 * S2.to(torch.float64) + ulp.pow(2) / 4).reshape(-1, D).mean(dim=1).sqrt()
        return self.add(got, ref_final, row0, allow=self.P_ROUND * A, row_scale=row_scale)


def attention_reference(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, *, causal: bool, scale: float,
                        budget: int = 1 << 27):
    """Prefill attention in fp64 on q's device, in blocks of query rows (never Sq x Sk x Hq at once).
    q [Sq, Hq, D], k / v [Sk, Hkv, D] (the kernel's bf16 inputs: q after RoPE, K/V as stored in the pool,
    in token order); query head h reads KV head h // (Hq / Hkv); causal: query i sees keys j <= i + Sk - Sq.
    Yields (r0, r1, ref_final, A, S2), each [r1 - r0, Hq, D] in fp64:
      ref_final = sum_j p_ij v_jd / l_i,  A = sum_j p_ij |v_jd| / l_i,  S2 = sum_j p_ij^2 v_jd^2 / l_i^2,
    with p_ij = exp(s_ij - max_j s_ij), s_ij = scale * q_i . k_j, l_i = sum_j p_ij.
    budget: fp64 elements of one block's scores."""
    Sq, Hq, D = q.shape
    Sk, Hkv = k.shape[0], k.shape[1]
    G, off = Hq // Hkv, Sk - Sq
    kd = k.to(torch.float64).permute(1, 2, 0)         # [Hkv, D, Sk]
    vd = v.to(torch.float64).permute(1, 0, 2)[:, None]  # [Hkv, 1, Sk, D]
    step = max(1, min(Sq, budget // (Hq * Sk)))
    for r0 in range(0, Sq, step):
        r1 = min(Sq, r0 + step)
        n = r1 - r0
        kv = min(Sk, r1 + off) if causal else Sk
        qd = q[r0:r1].to(torch.float64).reshape(n, Hkv, G, D).permute(1, 2, 0, 3)  # [Hkv, G, n, D]
        s = torch.matmul(qd, kd[:, None, :, :kv]).mul_(scale)                      # [Hkv, G, n, kv]
        if causal:
            i = torch.arange(r0, r1, device=q.device)[:, None]
            j = torch.arange(kv, device=q.device)[None, :]
            s.masked_fill_(j > i + off, float("-inf"))
        p = s.sub_(s.amax(dim=-1, keepdim=True)).exp_()
        del s
        l = p.sum(dim=-1, keepdim=True)
        vk = vd[:, :, :kv]
        ref = torch.matmul(p, vk) / l
        A = torch.matmul(p, vk.abs()) / l
        S2 = torch.matmul(p.mul_(p), vk * vk) / (l * l)
        del p

        def out(t):
            return t.permute(2, 0, 1, 3).reshape(n, Hq, D)
        yield r0, r1, out(ref), out(A), out(S2)


def attention_errors(got: torch.Tensor, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, *, causal: bool,
                     scale: float, into: AttnErrors = None, row0: int = 0) -> AttnErrors:
    """AttnErrors of the kernel output got [Sq, Hq, D] against attention_reference(q, k, v), added to
    `into` (a new AttnErrors by default) with row numbers from row0 (several sequences in one checker)."""
    e = AttnErrors() if into is None else into
    Hq = q.shape[1]
    for r0, r1, ref, A, S2 in attention_reference(q, k, v, causal=causal, scale=scale):
        e.add_attention(got[r0:r1], ref, A, S2, row0 + r0 * Hq)
    return e


ATTN_FAMILIES = ("random", "sink", "probe")
SENTINEL_V = 256.0  # V of every garbage key slot: large, finite (the kernel multiplies a masked P = 0 by it)
PROBE_C = 4.0       # probe: q . k = PROBE_C * (key position - query position) on the position channels


def attention_inputs(family: str, q_pos: torch.Tensor, key_pos: torch.Tensor, Hq: int, Hkv: int, D: int,
                     scale: float, *, sink: torch.Tensor = None, garbage: torch.Tensor = None, seed: int = 0):
    """q [nq, Hq, D] and k, v [N, Hkv, D] (bf16, on key_pos's device) for queries at global token positions
    q_pos [nq] and N key slots at positions key_pos [N].  sink [N]: the first key of each sequence;
    garbage [N]: slots no query may see (past Sk in the last page, unused pages).  Their V is SENTINEL_V.
      random: scores scale * q.k with standard deviation ~1; three V channels 16x larger.
      sink:   scores with standard deviation ~3, and the sink keys ~12 above the rest: P spans many
              binades and the running maximum jumps.
      probe:  score = scale * PROBE_C * (key position - query position) + noise of deviation ~0.3, so every
              row is dominated by its last visible keys; garbage slots sit 256 positions past the last
              real key.  A key leaked past the causal diagonal or the end of the sequence then changes the
              output by O(1).  The position channels hold exact bf16 integers: key channel 0 = pos // 256,
              1 = pos % 256, 2 = 3 = 1; query channel 0 = 256 c, 1 = c, 2 = -256 c (qpos // 256),
              3 = -c (qpos % 256); the noise lives in channels >= 16 (its own k16 wgmma step)."""
    dev = key_pos.device
    g = torch.Generator(device=dev).manual_seed(seed)
    nq, N = q_pos.numel(), key_pos.numel()
    garbage = torch.zeros(N, dtype=torch.bool, device=dev) if garbage is None else garbage
    v = torch.randn(N, Hkv, D, device=dev, generator=g)
    if family == "random":
        q = torch.randn(nq, Hq, D, device=dev, generator=g)
        k = torch.randn(N, Hkv, D, device=dev, generator=g) / (scale * math.sqrt(D))
        v[:, :, [3, D // 2, D - 5]] *= 16.0
    elif family == "sink":
        sd = math.sqrt(3.0 / (scale * math.sqrt(D - 1)))
        q = torch.randn(nq, Hq, D, device=dev, generator=g) * sd
        k = torch.randn(N, Hkv, D, device=dev, generator=g) * sd
        q[:, :, 0] = 4.0
        k[:, :, 0] = 0.0
        if sink is not None:
            k[sink, :, 0] = 12.0 / (4.0 * scale)
    elif family == "probe":
        sd = math.sqrt(0.3 / (scale * math.sqrt(D - 16)))
        q = torch.zeros(nq, Hq, D, device=dev)
        k = torch.zeros(N, Hkv, D, device=dev)
        q[:, :, 16:] = torch.randn(nq, Hq, D - 16, device=dev, generator=g) * sd
        k[:, :, 16:] = torch.randn(N, Hkv, D - 16, device=dev, generator=g) * sd
        kp = torch.where(garbage, key_pos[~garbage].max() + 256, key_pos) if bool((~garbage).any()) else key_pos
        assert int(kp.max()) < 65536 and int(q_pos.max()) < 65536
        c = PROBE_C
        k[:, :, 0] = (kp // 256).to(k.dtype)[:, None]
        k[:, :, 1] = (kp % 256).to(k.dtype)[:, None]
        k[:, :, 2:4] = 1.0
        q[:, :, 0], q[:, :, 1] = 256 * c, c
        q[:, :, 2] = (-256 * c * (q_pos // 256)).to(q.dtype)[:, None]
        q[:, :, 3] = (-c * (q_pos % 256)).to(q.dtype)[:, None]
    else:
        raise ValueError(family)
    v[garbage] = SENTINEL_V
    return q.to(torch.bfloat16), k.to(torch.bfloat16), v.to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------
# decode attention: one new token at position pos over the keys 0..pos (Sq = 1, non-causal)
# ------------------------------------------------------------------------------------------------
DECODE_FAMILIES = ("random", "sink", "leak")
LEAK_EDGE = 6.0      # leak: score of an edge key above the rest
LEAK_GARBAGE = 30.0  # leak: score of every garbage slot (>= 16 above every visible key)
LEAK_Q = 4.0         # leak: the query heads' shared component along u (rotated space)


class DecodeInputs:
    """One decode step's inputs (decode_attention_inputs); every tensor bf16 on the device.
      qkv     [(Hq + 2 Hkv) D]  the projection row before RoPE: q, k_new, v_new
      q       [Hq, D]           q after RoPE at pos (HF's bf16 op order), what the reference uses
      k_new   [Hkv, D]          k_new after RoPE: the K row the kernel must append at pos
      v_new   [Hkv, D]          the V row it must append (not rotated)
      k_hist, v_hist [pos, Hkv, D]  the cached keys 0..pos-1 as prefill leaves them (after RoPE)
      k_garbage [Hkv, D]        K of every slot no query may see; its V is SENTINEL_V"""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    def keys(self):
        """K and V of the keys 0..pos in token order: the reference's inputs"""
        return torch.cat([self.k_hist, self.k_new[None]]), torch.cat([self.v_hist, self.v_new[None]])


def _rope_pair(pos: int, D: int, theta: float = 1e6):
    """bf16 cos / sin of position pos, [1, D] on the CPU: O.rope_cos_sin (what the kernels' sincosf matches)"""
    return O.rope_cos_sin(torch.tensor([pos]), D, theta, torch.bfloat16)


def rope_rotate(x: torch.Tensor, pos: int) -> torch.Tensor:
    """x [H, D] bf16 rotated to position pos in HF's bf16 op order (O.apply_rope)"""
    cos, sin = _rope_pair(pos, x.shape[-1])
    r, _ = O.apply_rope(x.cpu()[:, None], x.cpu()[:, None], cos, sin)
    return r[:, 0].to(x.device)


def _rope_preimage(y: torch.Tensor, pos: int) -> torch.Tensor:
    """bf16 x whose rotation to pos is close to y (fp32 [H, D]): the inverse rotation in fp64, rounded"""
    D = y.shape[-1]
    inv = O.rope_inv_freq(D, 1e6).double()
    ang = torch.tensor(float(pos), dtype=torch.float32).double() * inv
    c, s = ang.cos(), ang.sin()
    y = y.double().cpu()
    y0, y1 = y[:, :D // 2], y[:, D // 2:]
    return torch.cat([y0 * c + y1 * s, -y0 * s + y1 * c], dim=1).to(torch.bfloat16)


def decode_edges(pos: int, chunks) -> torch.Tensor:
    """bool [pos + 1]: the keys at the edges of every chunk size in `chunks` (pages, splits), pos - 1 and pos"""
    t = torch.arange(pos + 1)
    e = (t == pos) | (t == pos - 1)
    for c in chunks:
        e |= (t % c == 0) | (t % c == c - 1)
    return e


def decode_attention_inputs(family: str, pos: int, Hq: int, Hkv: int, D: int, scale: float, seed: int, *,
                            chunks=(128,), device="cpu") -> DecodeInputs:
    """The inputs of one decode step at position pos (the new token; keys 0..pos-1 are cached).  q and the
    new k are drawn after RoPE and mapped back to a bf16 pre-RoPE row, so every family's score pattern holds
    for the rotated values the kernels see; the history is drawn directly as cached (after RoPE).
      random: scores with standard deviation ~1; three V channels 16x larger.
      sink:   key 0 scores ~12 above the rest, which have standard deviation ~3.
      leak:   the G query heads of a KV group share a component LEAK_Q u (u a unit vector per KV head, the
              rest of q orthogonal to it); visible keys score with deviation ~0.3, and the edge keys (the
              new token, pos - 1, the first and last key of every chunk size in `chunks`) LEAK_EDGE above;
              k_garbage = c u scores LEAK_GARBAGE for every head.  u depends on the shape only, so the
              slots of one pool share k_garbage (random / sink: any slot's k_garbage will do).  Attending a garbage slot changes the
              output by O(SENTINEL_V); dropping or double-counting one edge key by O(|v| / edge keys)."""
    G = Hq // Hkv
    g = torch.Generator(device=device).manual_seed(seed)
    gc = torch.Generator().manual_seed(seed)
    n = pos + 1
    v = torch.randn(n, Hkv, D, device=device, generator=g)
    if family == "random":
        qr = torch.randn(Hq, D, generator=gc)
        k = torch.randn(n, Hkv, D, device=device, generator=g) / (scale * math.sqrt(D))
        kg = torch.randn(Hkv, D, generator=gc) / (scale * math.sqrt(D))
        v[:, :, [3, D // 2, D - 5]] *= 16.0
    elif family == "sink":
        sd = math.sqrt(3.0 / (scale * math.sqrt(D - 1)))
        qr = torch.randn(Hq, D, generator=gc) * sd
        k = torch.randn(n, Hkv, D, device=device, generator=g) * sd
        kg = torch.randn(Hkv, D, generator=gc) * sd
        qr[:, 0] = 4.0
        k[:, :, 0] = 0.0
        kg[:, 0] = 0.0
        k[0, :, 0] = 12.0 / (4.0 * scale)
    elif family == "leak":
        u = torch.randn(Hkv, D, generator=torch.Generator().manual_seed(Hkv * D))  # one per shape: slots
        u /= u.norm(dim=1, keepdim=True)  # sharing a pool share k_garbage
        nq = torch.randn(Hq, D, generator=gc)
        uq = u.repeat_interleave(G, dim=0)
        nq -= (nq * uq).sum(dim=1, keepdim=True) * uq
        qr = LEAK_Q * uq + nq
        sd = 0.3 / (scale * math.sqrt(D))
        k = torch.randn(n, Hkv, D, device=device, generator=g) * sd
        ud = u.to(device)
        k -= (k * ud).sum(dim=-1, keepdim=True) * ud
        edge = decode_edges(pos, chunks).to(device)
        k[edge] += (LEAK_EDGE / (scale * LEAK_Q)) * ud
        kg = (LEAK_GARBAGE / (scale * LEAK_Q)) * u
    else:
        raise ValueError(family)
    q_pre = _rope_preimage(qr, pos)
    k_pre = _rope_preimage(k[pos].float().cpu(), pos)
    q = rope_rotate(q_pre, pos)
    k_new = rope_rotate(k_pre, pos)
    v = v.to(torch.bfloat16)
    qkv = torch.cat([q_pre.reshape(-1), k_pre.reshape(-1), v[pos].cpu().reshape(-1)]).to(device)
    inp = DecodeInputs(qkv=qkv, q=q.to(device), k_new=k_new.to(device), v_new=v[pos].clone(),
                       k_hist=k[:pos].to(torch.bfloat16), v_hist=v[:pos], k_garbage=kg.to(torch.bfloat16).to(device),
                       pos=pos, family=family)
    if family == "leak":  # the family's promise, on the values the kernels see
        kq = inp.keys()[0].double()
        hk = torch.arange(Hq, device=device) // G
        s = scale * torch.einsum("hd,thd->ht", q.double().to(device), kq[:, hk])
        sg = scale * (q.double().to(device) * inp.k_garbage.double()[hk]).sum(dim=1)
        assert bool((sg >= s.amax(dim=1) + 16.0).all()), "leak: a garbage slot scores too close to a visible key"
    return inp


# The fp8 decode kernel rounds p * vscale once per (token, KV head): that rounding is shared by the G * 128
# outputs of the group, so when a few keys carry a row the group's outputs move together and the mean signed
# error is a mean of a few shifts, not of independent roundings (tests/test_decode_attention_cpu.py::
# test_fp8_sink_bias_is_one_shared_rounding).  Its rounding bias is checked only over contexts of at least this
# many keys and away from the sink family; the element and row checks apply everywhere.
FP8_BIAS_MIN_KEYS = 128


def check_decode_attention(name: str, got: torch.Tensor, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor,
                           scale: float, bias: bool = True) -> AttnErrors:
    """AttnErrors of one decode output got [Hq, D] against the fp64 reference over the keys k, v [pos + 1, Hkv,
    D] (non-causal) for the rotated q [Hq, D]; recorded like report_rel and asserted (bias False: the element
    and row checks only)."""
    e = attention_errors(got.reshape(1, *q.shape[-2:]), q.reshape(1, *q.shape[-2:]), k, v, causal=False,
                         scale=scale)
    _record({"name": name, "bias_checked": bias, **e.summary()})
    bad = [f for f in e.failures() if bias or not f.startswith("rounding bias")]
    assert not bad, f"{name}: " + "; ".join(bad)
    return e


def scatter_tokens(pool: torch.Tensor, pages, rows: torch.Tensor) -> None:
    """rows [n, ...] (token t of a sequence) into pool [P, 128, ...] at page pages[t // 128], row t % 128"""
    n = rows.shape[0]
    if n == 0:
        return
    pages = torch.as_tensor(pages, device=pool.device).long()
    full = n // 128
    if full:
        pool[pages[:full]] = rows[:full * 128].reshape(full, 128, *rows.shape[1:]).to(pool.dtype)
    if n % 128:
        pool[pages[full], :n % 128] = rows[full * 128:].to(pool.dtype)


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


# ------------------------------------------------------------------------------------------------
# decode GEMV: mirrors of the launch plans, independent quantizers, the fp64 reference and GemvErrors
# ------------------------------------------------------------------------------------------------
W4_GROUP = 128
W4_TILE = 16


def gemv_tma_plan(N: int, K: int, fp8: bool, swiglu: bool, norm: bool, sms: int):
    """gemv_tma_launch's choice (gemv_tma.cu) for the bf16 (fp8=False) or e4m3 TMA-ring kernel: a dict with
    rows_per_block, grid, ksplit, chunk_elems and stages, or None where the launcher returns -1 (bf16: the
    register-staged kernel runs instead)."""
    max_stages, eb = (12, 1) if fp8 else (6, 2)
    align = 16 // eb
    rpb = _cdiv(N, sms)
    if swiglu and rpb % 2:
        rpb += 1
    x1 = _cdiv(K * 2, 128) * 128
    xb = x1 * (2 if norm else 1)
    scb = rpb * 4 if fp8 else 0
    bars = (8 * max_stages + 2) * 8
    ksplit = -1
    for ks in range(1, 129):
        if K % ks:
            continue
        ce = K // ks
        if ce % align:
            continue
        cb = ce * eb
        if cb > 8192:
            continue
        if cb < 512:
            break
        acc = _cdiv(rpb * ks * 4 + scb, 128) * 128
        st = min(max_stages, (220 * 1024 - xb - acc - bars - 256) // (8 * cb))
        if st < 3:
            continue
        ksplit = ks
        if rpb * ks >= 6 * 8:
            break
    if ksplit < 0:
        return None
    ce = K // ksplit
    ring_off = _cdiv(xb + rpb * ksplit * 4 + scb, 128) * 128
    st = min(max_stages, (220 * 1024 - ring_off - bars - 256) // (8 * ce * eb))
    if st < 2:
        return None
    return dict(rows_per_block=rpb, grid=_cdiv(N, rpb), ksplit=ksplit, chunk_elems=ce, stages=st)


def gemv_reg_plan(N: int, K: int, swiglu: bool, sms: int) -> dict:
    """gemv_bf16's register-staged kernel (decode.cu, variant 1): rows per block, k-parts, 256-k chunks per part"""
    rpb = _cdiv(N, sms)
    if swiglu and rpb % 2:
        rpb += 1
    nchunks = _cdiv(K // 8, 32)
    ks = 1
    while rpb * ks < 3 * 8 and ks * 2 <= nchunks and ks < 16:
        ks *= 2
    return dict(rows_per_block=rpb, grid=_cdiv(N, rpb), ksplit=ks, chunks_per_part=_cdiv(nchunks, ks))


def gemv_w4_plan(N: int, K: int, norm: bool, sms: int):
    """gemv_w4_launch's choice for the single-stream W4A16 kernel: tiles_per_block, rows_per_block, grid,
    ksplit, chunk_groups, stages (None: the launcher refuses the shape)"""
    tiles = _cdiv(N, W4_TILE)
    tpb = _cdiv(tiles, sms)
    rpb = tpb * W4_TILE
    G = K // W4_GROUP
    x1 = _cdiv(K * 2, 128) * 128
    xb = x1 * (2 if norm else 1)
    gp = _cdiv(rpb * G * 3, 128) * 128
    bars = (8 * 12 + 2) * 8
    ksplit = -1
    for ks in range(1, G + 1):
        if G % ks:
            continue
        cb = G // ks * 1024
        if cb > 8192:
            continue
        acc = _cdiv(rpb * ks * 4, 128) * 128
        if (220 * 1024 - xb - acc - gp - bars - 256) // (8 * cb) < 3:
            continue
        ksplit = ks
        if tpb * ks >= 6 * 8:
            break
    if ksplit < 0:
        return None
    cg = G // ksplit
    ring_off = xb + _cdiv(rpb * ksplit * 4, 128) * 128 + gp
    st = min(12, (220 * 1024 - ring_off - bars - 256) // (8 * cg * 1024))
    return dict(tiles_per_block=tpb, rows_per_block=rpb, grid=_cdiv(tiles, tpb), ksplit=ksplit, chunk_groups=cg,
                stages=st)


def batch_partition(N: int, K: int, fp8: bool, sms: int, max_active_clusters=None):
    """batch_partition (gemv_tma.cu) for gemv_batch_*: max_active_clusters(cluster) is what
    cudaOccupancyMaxActiveClusters reports for that cluster size (default: sms // cluster).  -> dict with
    cluster, ctas, tiles_per_cluster, unit, units, max_units, parts, stages, slices [(u0, nu)] and, per slice,
    its k-parts [(pu0, pu)] as part_range cuts them; None where the launcher refuses the shape."""
    active = max_active_clusters or (lambda cl: sms // cl)
    tiles = _cdiv(N, W4_TILE)
    unit = 16 if fp8 else W4_GROUP
    units = K // unit

    def x_pitch(cl):
        return _cdiv(_cdiv(units, cl) * unit * 2, 128) * 128 + 16

    def tpc(cl):
        a = active(cl)
        n = max(1, min(sms // cl, a if a > 0 else sms // cl))
        return _cdiv(tiles, n)

    cluster = 0
    cl = 1
    while cl <= 8:
        if units < 4 * cl:
            break
        xb = 16 * x_pitch(cl)
        pb = tpc(cl) * W4_TILE * 16 * 4 if cl > 1 else 0
        if xb + pb <= 100 * 1024:
            cluster = cl
            break
        cl *= 2
    if cluster == 0:
        if 16 * x_pitch(1) > 120 * 1024:
            return None
        cluster = 1
    t = tpc(cluster)
    max_units = _cdiv(units, cluster)
    rows = t * W4_TILE
    part_off = 16 * x_pitch(cluster)
    gs_off = part_off + (rows * 16 * 4 if cluster > 1 else 0)
    gz_off = gs_off + (rows * 4 if fp8 else rows * max_units * 2)
    ring_off = _cdiv(gz_off + (0 if fp8 else rows * max_units), 128) * 128
    bars = (8 * 12 + 1) * 8
    max_chunk = 32 if fp8 else 8
    parts, stages = _cdiv(max_units, max_chunk), 0
    while parts <= max_units:
        chunk = _cdiv(max_units, parts)
        slot = 16 * (_cdiv(chunk * unit, 128) * 128 + 64) if fp8 else chunk * 1024
        stages = min(12, (220 * 1024 - ring_off - bars) // (8 * slot))
        if stages >= 3:
            break
        parts += 1
    if parts > max_units or stages < 3:
        return None
    slices = [(r * units // cluster, (r + 1) * units // cluster - r * units // cluster) for r in range(cluster)]
    kparts = [[(q * nu // parts, (q + 1) * nu // parts - q * nu // parts) for q in range(parts)] for _, nu in slices]
    return dict(cluster=cluster, ctas=_cdiv(tiles, t) * cluster, tiles_per_cluster=t, unit=unit, units=units,
                max_units=max_units, parts=parts, stages=stages, slices=slices, kparts=kparts)


def gemv_depth(kind: str, K: int, plan: dict) -> int:
    """The deepest fp32 summation chain of one output (additions a product passes through before the epilogue,
    the epilogue's scale and bias included), for GemvErrors' accumulation term.  An mma.sync step is counted
    as 16 additions; kind: "tma-bf16", "tma-fp8", "reg-bf16", "w4", "batch-fp8", "batch-w4"."""
    if kind in ("tma-bf16", "tma-fp8"):
        per_vec = 16 if kind == "tma-fp8" else 8
        vecs = plan["chunk_elems"] * (1 if kind == "tma-fp8" else 2) // 16
        return per_vec * _cdiv(vecs, 64) + 1 + 5 + plan["ksplit"] + 2
    if kind == "reg-bf16":
        return 8 * plan["chunks_per_part"] + 5 + plan["ksplit"] + 2
    if kind == "w4":
        return 4 * 16 + 1 + plan["chunk_groups"] + plan["ksplit"] + 2
    if kind == "batch-w4":
        return 4 * 16 + 1 + plan["max_units"] + plan["cluster"] + 2
    if kind == "batch-fp8":
        chunk = _cdiv(plan["max_units"], plan["parts"]) * plan["unit"]
        return 4 * 16 * _cdiv(chunk, 128) + 1 + plan["parts"] + plan["cluster"] + 2
    raise ValueError(kind)


# --- the quantizers, re-derived from their docstrings and gemv_tma.cu's layout comment -------------------------
def _bf16_rne(t: torch.Tensor) -> torch.Tensor:
    """fp32 -> the nearest bf16 (ties to even), returned as fp32; finite inputs"""
    u = t.to(torch.float32).contiguous().view(torch.int32).to(torch.int64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & ~0xFFFF
    return u.to(torch.int32).view(torch.float32)  # int64 -> int32 wraps the sign bit back


def e4m3_values() -> torch.Tensor:
    """the value of each e4m3fn code 0..255 (fp64; 0x7f and 0xff are NaN): sign, 4 exponent bits (bias 7),
    3 mantissa bits; exponent 0 is subnormal (m / 8 * 2^-6)"""
    c = torch.arange(256, dtype=torch.int64)
    e, m = (c >> 3) & 15, (c & 7).to(torch.float64)
    mag = torch.where(e == 0, m / 8 * 2.0 ** -6, (1 + m / 8) * torch.pow(2.0, (e - 7).to(torch.float64)))
    mag = torch.where((c & 127) == 127, torch.full_like(mag, float("nan")), mag)
    return torch.where(c >= 128, -mag, mag)


def e4m3_encode(t: torch.Tensor) -> torch.Tensor:
    """fp32 values with |t| <= 464 -> e4m3fn codes (uint8), round to nearest, ties to the even code (the
    even mantissa); the sign bit follows t's sign, so a negative value that rounds to 0 is -0 (0x80)"""
    pos = e4m3_values()[:127].to(t.device)  # codes 0..126: 0 .. 448, increasing
    a = t.to(torch.float64).abs()
    assert bool((a <= 464).all()), "e4m3_encode: |t| > 464 overflows"
    hi = torch.searchsorted(pos, a).clamp(max=126)
    lo = (hi - 1).clamp(min=0)
    dlo, dhi = a - pos[lo], pos[hi] - a
    code = torch.where(dlo < dhi, lo, torch.where(dhi < dlo, hi, torch.where(lo % 2 == 0, lo, hi)))
    code = torch.where(a > 448, torch.full_like(code, 126), code)
    return (code | (torch.signbit(t).to(torch.int64) << 7)).to(torch.uint8)


REF_ROWS = 4096  # rows per chunk of the reference quantizers: an lm_head's fp64 temporaries stay ~100 MB each


def ref_quantize_e4m3_rows(w: torch.Tensor):
    """quantize_e4m3_rows' docstring: s_n = amax_n / 448 in fp32 (1 for an all-zero row), code =
    e4m3(W / s_n) with the division in fp32.  -> (codes uint8 [N, K], s fp32 [N]), in chunks of rows"""
    N = w.shape[0]
    codes = torch.empty(w.shape, dtype=torch.uint8, device=w.device)
    s = torch.empty(N, dtype=torch.float32, device=w.device)
    for r0 in range(0, N, REF_ROWS):
        wf = w[r0:r0 + REF_ROWS].to(torch.float32)
        amax = wf.abs().amax(dim=1)
        sc = torch.where(amax > 0, amax / torch.tensor(448.0, device=w.device), torch.ones_like(amax))
        codes[r0:r0 + REF_ROWS] = e4m3_encode(wf / sc[:, None])
        s[r0:r0 + REF_ROWS] = sc
    return codes, s


def ref_quantize_w4(w: torch.Tensor):
    """quantize_w4_groups' docstring, per row and group of 128 k in fp32: lo = min(0, min w), hi = max(0, max w),
    s = bf16((hi - lo) / 15) or 1, z = clamp(rint(-lo / s), 0, 15), q = clamp(rint(w / s) + z, 0, 15) (rint:
    half to even).  -> (codes uint8 [N, K], s fp32 [N, G] (bf16 values), z uint8 [N, G]), in chunks of rows"""
    N, K = w.shape
    G = K // W4_GROUP
    q = torch.empty(N, K, dtype=torch.uint8, device=w.device)
    s = torch.empty(N, G, dtype=torch.float32, device=w.device)
    z = torch.empty(N, G, dtype=torch.uint8, device=w.device)
    for r0 in range(0, N, REF_ROWS):
        wf = w[r0:r0 + REF_ROWS].to(torch.float32).reshape(-1, G, W4_GROUP)
        lo = wf.amin(dim=2).clamp(max=0)
        hi = wf.amax(dim=2).clamp(min=0)
        sc = _bf16_rne((hi - lo) / torch.tensor(15.0, device=w.device))
        sc = torch.where(sc == 0, torch.ones_like(sc), sc)
        zp = torch.round(-lo / sc).clamp(0, 15)  # torch.round: half to even
        q[r0:r0 + REF_ROWS] = (torch.round(wf / sc[..., None]) + zp[..., None]).clamp(0, 15).reshape(-1, K)
        s[r0:r0 + REF_ROWS], z[r0:r0 + REF_ROWS] = sc, zp.to(torch.uint8)
    return q, s, z


# nibble p of a packed u32 (bits 4p .. 4p+3): (row offset 0 / 8 within the lane's pair g, g + 8; k offset from k0)
W4_NIBBLES = ((0, 0), (8, 0), (0, 2), (8, 2), (0, 1), (8, 1), (0, 3), (8, 3))


def ref_w4_pack(q: torch.Tensor) -> torch.Tensor:
    """codes uint8 [N, K] -> the packed bytes [ceil(N/16), 8 K] as gemv_tma.cu's comment above w4_pair lays them
    out: rows in tiles of 16 (padded with zero codes), per tile [K/64 blocks][32 lanes][4 u32], lane = 4 g + c,
    u32 j of block b holding rows g, g + 8 at k0 = b + 16 c + 4 j .. k0 + 3, nibble p as W4_NIBBLES; u32s little
    endian; in chunks of tiles"""
    N, K = q.shape
    T = _cdiv(N, W4_TILE)
    out = torch.empty(T, 8 * K, dtype=torch.uint8, device=q.device)
    step = REF_ROWS // W4_TILE
    for t0 in range(0, T, step):
        t1 = min(T, t0 + step)
        qp = torch.zeros((t1 - t0) * W4_TILE, K, dtype=torch.int64, device=q.device)
        rows = q[t0 * W4_TILE:t1 * W4_TILE]
        qp[:rows.shape[0]] = rows.to(torch.int64)
        t = qp.view(t1 - t0, W4_TILE, K // 64, 4, 4, 4)  # [tile, row, b, c, j, kk]
        word = torch.zeros(t1 - t0, K // 64, 8, 4, 4, dtype=torch.int64, device=q.device)  # [tile, b, g, c, j]
        for p, (dr, dk) in enumerate(W4_NIBBLES):
            word |= t[:, dr:dr + 8, :, :, :, dk].permute(0, 2, 1, 3, 4) << (4 * p)
        by = torch.stack([(word >> (8 * i)) & 255 for i in range(4)], dim=-1)  # [tile, b, g, c, j, byte]
        out[t0:t1] = by.reshape(t1 - t0, 8 * K).to(torch.uint8)
    return out


def ref_w4_unpack(packed: torch.Tensor, N: int, K: int) -> torch.Tensor:
    """the inverse of ref_w4_pack (the same layout read back): codes uint8 [N, K]"""
    T = packed.shape[0]
    by = packed.to(torch.int64).view(T, K // 64, 8, 4, 4, 4)
    word = by[..., 0] | (by[..., 1] << 8) | (by[..., 2] << 16) | (by[..., 3] << 24)  # [tile, b, g, c, j]
    q = torch.zeros(T, W4_TILE, K // 64, 4, 4, 4, dtype=torch.int64, device=packed.device)
    for p, (dr, dk) in enumerate(W4_NIBBLES):
        q[:, dr:dr + 8, :, :, :, dk] = ((word >> (4 * p)) & 15).permute(0, 2, 1, 3, 4)
    return q.reshape(T * W4_TILE, K)[:N].to(torch.uint8)


# --- the reference and the checker ---------------------------------------------------------------------------
def gemv_xn(x: torch.Tensor, norm_w=None, eps: float = 1e-6) -> torch.Tensor:
    """x as the GEMV multiplies it: bf16(bf16(x * rstd) * norm_w) with rstd in fp32 (the fused RMSNorm
    prologue), or x itself"""
    return x if norm_w is None else O.rms_norm(x, norm_w, eps)


def gemv_reference(x: torch.Tensor, w, N: int, *, block_rows: int = 8192, need_E: bool = True):
    """x [M, K] (bf16, already as the kernel multiplies it); w(r0, r1) -> the weight rows r0..r1 in fp64, or
    an [N, K] tensor.  -> (P, A, E) fp64 [M, N]: P = x W^T, A = |x| |W|^T (what bounds the fp32 accumulation),
    E = max_k |W_nk x_mk| (one flipped element of x; left unset without need_E).  Row blocks: no full fp64
    copy of a large W."""
    rows = w if callable(w) else (lambda r0, r1: w[r0:r1].to(torch.float64))
    xd = x.to(torch.float64)
    M = xd.shape[0]
    P = torch.empty(M, N, dtype=torch.float64, device=x.device)
    A, E = torch.empty_like(P), torch.empty_like(P)
    xa = xd.abs()
    for r0 in range(0, N, block_rows):
        r1 = min(N, r0 + block_rows)
        wb = rows(r0, r1)
        P[:, r0:r1] = xd @ wb.t()
        wa = wb.abs()
        A[:, r0:r1] = xa @ wa.t()
        for m in range(M if need_E else 0):
            E[m, r0:r1] = (wa * xa[m]).amax(dim=1)
        del wb, wa
    return P, A, E


class GemvErrors(Bf16Errors):
    """Bf16Errors for a decode GEMV output [M, N or N/2] with a per-element allowance derived from the kernel's
    arithmetic, in place of the blanket B_RMS * rms(row).  From gemv_reference's P, A, E and the depth d of the
    deepest fp32 summation chain (gemv_depth):
      e_P = ACC * d * A  +  ACC * |bias|  [+ NORM_FLIP * E with the fused RMSNorm]
    bounds how far the kernel's fp32 value before the epilogue may lie from P (+ bias):
      * fp32 accumulation: recursive summation of products that enter a chain of d additions errs by at most
        d * u * sum|products| (u = 2^-24 with round to nearest).  ACC = 2^-23 = 2u: the tensor cores' fp32
        accumulation inside an mma.sync is not round-to-nearest (it may truncate), which at most doubles u.
        The chain counts lane terms, the warp tree (5), the k-parts, the cluster ranks, the fp32 row or group
        scale and the bias add (bounded by u |bias|, the ACC |bias| term).
      * the fused RMSNorm: the kernel's rstd (rsqrtf of a differently ordered fp32 sum) is not torch's, so
        an element of bf16(x * rstd) near a rounding tie may round the other way: one ulp, <= 2^-7 of the
        element, moves P by <= 2^-7 max_k |W_nk x_nk| (NORM_FLIP = 2^-7; the later * norm_w is exact in fp32).
    Every other operation is an exact fp32 product of bf16 / e4m3 / 4-bit values.  Then, per epilogue:
      1. per element:  |got - bf16(ref_final)| <= A_ULP * ulp(ref) + allow,  A_ULP = 1, the final rounding
         (e_P may carry the value across a rounding tie), and allow =
         * plain, bias, arg-max:  e_P;
         * residual:  e_P + ulp(bf16(P + bias)): the rounded product before the add may flip (it may cancel
           against the residual, so this does not scale with the output);
         * SwiGLU, g = bf16(P_gate), u = bf16(P_up), s = bf16(silu(g)), out = bf16(s u):
           |g' - g| <= e_g + ulp(g),  |u' - u| <= e_u + ulp(u) = du,  |s' - s| <= 1.1 |g' - g| + ulp(s) = ds
           (|silu'| <= 1.1), so allow = ds (|u| + du) + |s| du.
       At K = 18944, d * ACC * A is ~1e-3 of an output's rms, far below its ulp: the element check is as tight as
       the output's own rounding.  One wrong (row, group) zero point or scale moves its output by s * (sum of the
       group's x), which is under one ulp for about a quarter of the groups; tests/test_gemv_cpu.py measures 73 %
       of such faults rejected (57 to 62 % when a residual as large as the output is added).
    2. per row and 3. rounding bias: as Bf16Errors (ROW_RMS = 2^-7 of the row rms, |bias| <= 0.1 ulp)."""
    A_ULP = 1.0
    ACC = 2.0 ** -23
    NORM_FLIP = 2.0 ** -7

    @classmethod
    def allowance(cls, P, A, E, *, depth: int, bias=None, residual=False, swiglu=False, norm=False):
        """-> (ref_final without the residual's values, allow): see the class docstring"""
        t = P if bias is None else P + bias.to(torch.float64)
        e = cls.ACC * depth * A
        if bias is not None:
            e = e + cls.ACC * bias.to(torch.float64).abs()
        if norm:
            e = e + cls.NORM_FLIP * E
        if swiglu:
            g, u = _rb64(t[:, 0::2]), _rb64(t[:, 1::2])
            s = _rb64(torch.nn.functional.silu(g))
            du = e[:, 1::2] + bf16_ulp(u)
            ds = 1.1 * (e[:, 0::2] + bf16_ulp(g)) + bf16_ulp(s)
            return ds * (u.abs() + du) + s.abs() * du
        if residual:
            return e + bf16_ulp(_rb64(t))
        return e

    def add_gemv(self, got, P, A, E, *, depth: int, bias=None, residual=None, swiglu=False, norm=False,
                 row0: int = 0) -> "GemvErrors":
        """got [M, N or N/2] against (P, A, E) of gemv_reference; residual [M, N] (the values before the add)"""
        allow = self.allowance(P, A, E, depth=depth, bias=bias, residual=residual is not None, swiglu=swiglu,
                               norm=norm)
        ref_final = linear_reference(P, bias=bias, residual=residual, swiglu=swiglu)
        return self.add(got, ref_final, row0, allow=allow)


def gemv_plan(fmt: str, N: int, K: int, fusion: str, sms: int, *, variant: int = 0, batched: bool = False):
    """-> (plan, depth, regime label) of the kernel that runs (fmt, N, K, fusion) on `sms` SMs: the single-stream
    bf16 (variant 0: TMA ring, else register-staged), e4m3 or W4A16 kernel, or (batched) gemv_batch_*"""
    swiglu, norm = "swiglu" in fusion, "norm" in fusion
    if batched:
        p = batch_partition(N, K, fmt == "fp8", sms)
        kind = "batch-fp8" if fmt == "fp8" else "batch-w4"
        return p, gemv_depth(kind, K, p), f"cluster {p['cluster']} x {p['tiles_per_cluster']} tiles, {p['parts']} parts"
    if fmt == "w4a16":
        p = gemv_w4_plan(N, K, norm, sms)
        return p, gemv_depth("w4", K, p), f"w4 ksplit {p['ksplit']} x {p['chunk_groups']} groups, {p['tiles_per_block']} tiles/block"
    p = gemv_tma_plan(N, K, fmt == "fp8", swiglu, norm, sms) if variant == 0 else None
    if p is None:
        assert fmt == "bf16", (fmt, N, K)
        p = gemv_reg_plan(N, K, swiglu, sms)
        return p, gemv_depth("reg-bf16", K, p), f"register-staged ksplit {p['ksplit']}"
    kind = "tma-fp8" if fmt == "fp8" else "tma-bf16"
    return p, gemv_depth(kind, K, p), f"tma ksplit {p['ksplit']}, {p['rows_per_block']} rows/block, {p['stages']} stages"


def check_gemv(name: str, got: torch.Tensor, x: torch.Tensor, w, N: int, *, depth: int, norm_w=None, eps=1e-6,
               bias=None, residual=None, swiglu=False, record: dict = None) -> GemvErrors:
    """GemvErrors of a GEMV output got [M, N or N/2] for the input rows x [M, K] (before the fused RMSNorm with
    norm_w) and the weight rows w (gemv_reference), recorded like report_rel; the caller asserts e.failures()"""
    x = x.reshape(-1, x.shape[-1])
    P, A, E = gemv_reference(gemv_xn(x, norm_w, eps), w, N, need_E=norm_w is not None)
    e = GemvErrors().add_gemv(got.reshape(P.shape[0], -1), P, A, E, depth=depth, bias=bias,
                              residual=None if residual is None else residual.reshape(P.shape[0], -1),
                              swiglu=swiglu, norm=norm_w is not None)
    _record({"name": name, **(record or {}), **e.summary()})
    return e


def e4m3_rows(codes: torch.Tensor, s: torch.Tensor):
    """weight rows in fp64 of ref_quantize_e4m3_rows' (codes, s), for gemv_reference"""
    vals = e4m3_values().to(codes.device)
    return lambda r0, r1: vals[codes[r0:r1].long()] * s[r0:r1, None].to(torch.float64)


def w4_rows(q: torch.Tensor, s: torch.Tensor, z: torch.Tensor):
    """weight rows (q - z) * s in fp64 of ref_quantize_w4's (q, s, z), for gemv_reference"""
    def rows(r0, r1):
        zz = z[r0:r1].to(torch.float64).repeat_interleave(W4_GROUP, 1)
        return (q[r0:r1].to(torch.float64) - zz) * s[r0:r1].to(torch.float64).repeat_interleave(W4_GROUP, 1)
    return rows


# ------------------------------------------------------------------------------------------------
# norms and media data movement: exact outside bf16 rounding ties
# ------------------------------------------------------------------------------------------------
U32 = 2.0 ** -24  # fp32 unit roundoff (round to nearest)


def bf16_rounding_tie_distance(x64: torch.Tensor) -> torch.Tensor:
    """distance of fp64 x from the nearest bf16 rounding boundary (midpoint of two bf16 neighbours), in
    fp32 ulps of x (2^-16 of its bf16 ulp)"""
    a = x64.abs()
    _, e = torch.frexp(a)
    ulp = torch.ldexp(torch.ones_like(a), e - 8)  # bf16 ulp of |x| in [2^(e-1), 2^e)
    frac = torch.remainder(a / ulp, 1.0)
    return ((frac - 0.5).abs() * 2.0 ** 16).where(a > 0, torch.full_like(a, float("inf")))


def bf16_rne64(x: torch.Tensor) -> torch.Tensor:
    """fp64 -> the nearest bf16 value (ties to even) in ONE rounding, as fp64 (torch's double -> bf16 cast
    goes through fp32, which double-rounds next to a tie); normal range"""
    x = x.to(torch.float64)
    ulp = bf16_ulp(x)
    return torch.round(x / ulp) * ulp  # x / ulp and the product are exact (powers of two); round: half to even


class TieErrors:
    """Exact-or-tie check of a bf16 output.  Each element comes with ref_final, the fp64 value before the
    last rounding, and eps, a bound on how far the kernel's fp32 value before that rounding can lie from
    ref_final.  Rounding is monotone, so the kernel's output lies in [bf16(ref_final - eps), bf16(ref_final +
    eps)]; where ref_final is further than eps from a bf16 rounding boundary that interval is the one value
    bf16(ref_final), and the output must equal it bit for bit.  Inside the window either neighbour is accepted,
    and nothing more, except where eps spans several bf16 values (`wide`: a cancellation), where any of them is.
    With `then`, the rounding checked is an intermediate one (RMSNorm's bf16(x * rstd)) and the output is
    then(intermediate): the output must be then(lo) or then(hi).
    Recorded: n, the elements in a tie window, the flips among them (output != the correctly rounded one),
    and `needed`, the largest |ref_final - crossed boundary| / eps over the flips: the part of eps the kernel
    actually used (a lower bound on its error).  failures() rejects a window covering more than
    max_window of the elements, so a too generous eps fails instead of quietly weakening the check."""

    def __init__(self, max_window: float = 0.02):
        self.max_window = max_window
        self.n = self.window = self.wide = self.flips = self.bad = 0
        self.first_bad = None
        self.needed = 0.0

    def add(self, got: torch.Tensor, ref_final: torch.Tensor, eps, then=None, where: str = "") -> "TieErrors":
        got = got.to(torch.float64).reshape(-1)
        r = ref_final.to(torch.float64).reshape(-1)
        e = torch.as_tensor(eps, dtype=torch.float64, device=r.device).expand(ref_final.shape).reshape(-1)
        lo, hi, want = bf16_rne64(r - e), bf16_rne64(r + e), bf16_rne64(r)
        win = lo != hi
        # more than two values: a cancellation (LayerNorm's + b near -x_hat w) leaves an absolute fp32 error
        # larger than the bf16 spacing of the small result; every value in [lo, hi] is then reachable
        wide = hi > lo + bf16_ulp(torch.minimum(lo.abs(), hi.abs())) * 1.0001
        self.wide += int(wide.sum())
        if then is None:
            ok = (got >= lo) & (got <= hi)
            flip = got != want
            mid = (got + want) / 2
        else:
            out_lo, out_hi, out_want = (then(t).reshape(-1) for t in (lo, hi, want))
            ok = (got == out_lo) | (got == out_hi) | (wide & (got >= torch.minimum(out_lo, out_hi))
                                                     & (got <= torch.maximum(out_lo, out_hi)))
            flip = got != out_want
            mid = (lo + hi) / 2
        self.n += got.numel()
        self.window += int(win.sum())
        self.flips += int(flip.sum())
        nb = int((~ok).sum())
        if nb and self.first_bad is None:
            i = int((~ok).nonzero()[0])
            self.first_bad = (where, i, got[i].item(), want[i].item() if then is None else None, r[i].item())
        self.bad += nb
        if bool((flip & ok).any()):
            used = ((r - mid).abs() / e.clamp_min(1e-300))[flip & ok]
            self.needed = max(self.needed, float(used.max()))
        return self

    @property
    def window_fraction(self) -> float:
        return self.window / max(self.n, 1)

    def failures(self) -> List[str]:
        out = []
        if self.bad:
            out.append(f"{self.bad} elements outside their exact-or-tie set (first: {self.first_bad})")
        if self.window_fraction > self.max_window:
            out.append(f"tie window covers {self.window_fraction:.2%} of the elements > {self.max_window:.2%}")
        return out

    def summary(self) -> dict:
        return {"n": self.n, "window": self.window, "window_frac": float(f"{self.window_fraction:.3e}"),
                "wide": self.wide, "flips": self.flips, "needed": float(f"{self.needed:.3e}")}

    def check(self, name: str) -> None:
        bad = self.failures()
        assert not bad, f"{name}: " + "; ".join(bad)


NORM_FAMILIES = ("random", "offset", "outlier", "small")


def norm_inputs(family: str, rows: int, cols: int, seed: int, device="cpu", rms: bool = False):
    """bf16 rows [rows, cols] and LayerNorm weight / bias [cols] (RMSNorm uses w only):
      random:  N(0.3, 2^2);
      offset:  256 + N(0, 4^2): the mean far above the spread (a residual stream with large offsets), so the
               fp32 mean's error is what the eps of the check has to cover;
      outlier: N(0, 1) with three channels at +-300 (alternating sign per row): outlier-dominated statistics;
      small:   N(0, 1e-3^2): the variance (mean square) is the size of the norm's eps, so a wrong eps moves
               every element;
      constant (not in NORM_FAMILIES, checked exactly): every row one value (LayerNorm) or zero (RMSNorm)."""
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn(rows, cols, generator=g, device=device)
    if family == "random":
        x = x * 2 + 0.3
    elif family == "offset":
        x = 256 + 4 * x
    elif family == "outlier":
        sign = 1 - 2 * (torch.arange(rows, device=device) % 2).to(x.dtype)
        for c in (3, cols // 2, cols - 5):
            x[:, c] = 300 * sign
    elif family == "small":
        x = x * 1e-3
    elif family == "constant":
        x = torch.zeros_like(x) if rms else torch.randn(rows, 1, generator=g, device=device).expand(rows, cols) * 8
    else:
        raise ValueError(family)
    w = 1 + 0.25 * torch.randn(cols, generator=g, device=device)
    b = 0.5 * torch.randn(cols, generator=g, device=device)
    bf = torch.bfloat16
    return x.to(bf).contiguous(), w.to(bf), b.to(bf)


NORM_THREADS = 256
WARP_ROW_MIN_ROWS = 8192  # norm.cu kWarpRowMinRows
WARP_ROW_MAX_COLS = 8 * 256  # the warp-per-row kernels hold 8 vectors of 8 per lane


def norm_plan(rows: int, cols: int) -> dict:
    """layernorm_bf16 / rmsnorm_bf16's choice (norm.cu): the warp-per-row kernel for rows >= 8192 and cols <=
    2048, else one CTA of 256 threads per row.  chain: fp32 additions a value passes through in one thread's
    partial sum (8 per 16-byte vector: 7 inside the vector's expression, 1 into the sum, times the vectors a
    thread or lane owns); warp: the xor-shuffle tree (5); block: the tree over the 8 warps' partials (5, a
    warp_sum with zeros).  depth = their sum, the deepest summation chain of the row sum."""
    nvec = cols // 8
    if rows >= WARP_ROW_MIN_ROWS and cols <= WARP_ROW_MAX_COLS:
        regime, chain, block = "warp", 8 * _cdiv(nvec, 32), 0
    else:
        regime, chain, block = "cta", 8 * _cdiv(nvec, NORM_THREADS), 5
    return dict(regime=regime, chain=chain, warp=5, block=block, depth=chain + 5 + block)


def _gamma(n) -> float:
    return n * U32 / (1 - n * U32)


def _row_blocks(rows: int, cols: int, budget: int = 1 << 24):
    step = max(1, budget // max(cols, 1))
    for r0 in range(0, rows, step):
        yield r0, min(rows, r0 + step)


def layernorm_reference(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float, depth: int):
    """nn.LayerNorm in fp64 (one rounding, at the output), in row blocks: yields (r0, r1, ref_final, eps_elem).
    eps_elem bounds |the kernel's fp32 value before its bf16 rounding - ref_final| (u = 2^-24, gamma_n = n u /
    (1 - n u), d = depth of norm_plan, m the exact mean, v the exact variance, rstd = 1 / sqrt(v + eps)):
      * the mean: the fp32 row sum errs by <= gamma_d sum|x|, the division by cols by u |m|:
            delta = gamma_d sum|x| / cols + u |m|;
        unless the sum is exact (every partial sum a multiple of the row's smallest bf16 ulp below 2^24 of
        them, see mean_eps), when delta is the division's own error, computed exactly;
      * the variance: the centred values are (x_i - m - delta)(1 + theta_i), |theta_i| <= u; the cross term of
        delta sums to zero (sum(x - m) = 0), so the sum of their squares is within (1 + 2u)^2 of v cols +
        delta^2 cols, and the fp32 sum of squares adds gamma_d; the division by cols and the + eps round once
        each:  rel_var = (gamma_(d+3) v + delta^2) / (v + eps) + 2 u;
      * rsqrtf: 2 ulps, <= 2^-22 relative; rsqrt halves the relative error of its argument:
            rel_rstd = rel_var / 2 + 2^-22;
      * the epilogue: x - mean, * rstd and * w round once each (u of |x - m| rstd |w|, whether or not the last
        product is fused into the + b), the + b once (u of the result):
            eps_elem = |w| rstd (delta + |x - m| (rel_rstd + 3 u)) (1 + 4 u) + u |ref_final| (1 + u).
    The mean term matters when the mean is much larger than the spread (delta grows with sum|x|, rstd with
    1 / spread)."""
    cols = x.shape[-1]
    x2 = x.reshape(-1, cols)
    wd, bd = w.to(torch.float64), b.to(torch.float64)
    for r0, r1 in _row_blocks(x2.shape[0], cols):
        xd = x2[r0:r1].to(torch.float64)
        m = xd.mean(dim=1, keepdim=True)
        c = xd - m
        v = c.pow(2).mean(dim=1, keepdim=True)
        rstd = (v + eps).rsqrt()
        ref = c * rstd * wd + bd
        sa = xd.abs().sum(dim=1, keepdim=True)
        delta = torch.where(sa < 2.0 ** 24 * _min_ulp(xd).amin(dim=1, keepdim=True),  # exact fp32 sum
                            ((xd.sum(dim=1, keepdim=True).float() / cols).double() - m).abs(),
                            _gamma(depth) * sa / cols + U32 * m.abs())
        rel_var = (_gamma(depth + 3) * v + delta.pow(2)) / (v + eps) + 2 * U32
        rel_rstd = rel_var / 2 + 2.0 ** -22
        e = wd.abs() * rstd * (delta + c.abs() * (rel_rstd + 3 * U32)) * (1 + 4 * U32) + U32 * ref.abs() * (1 + U32)
        yield r0, r1, ref, e


def rmsnorm_reference(x: torch.Tensor, eps: float, depth: int):
    """Qwen2RMSNorm's first rounding point in fp64, in row blocks: yields (r0, r1, t, eps_elem) with t = x rstd,
    rstd = 1 / sqrt(mean(x^2) + eps).  The output is bf16(w * bf16(t)): w * bf16(t) is a product of two bf16
    values, exact in fp32, so its rounding is exact too and the only inexact step is t.  eps_elem bounds |the
    kernel's fp32 x * rstd' - t|: the sum of squares (every term >= 0) errs by gamma_(d+1) relative, the division
    and + eps by u each, rsqrtf by 2^-22 and halves its argument's error, the product by u:
        eps_elem = |t| ((gamma_(d+1) + 2 u) / 2 + 2^-22 + u) (1 + u).
    A flip of bf16(t) inside that window moves the output by |w| ulp(bf16(t)) before its own rounding."""
    cols = x.shape[-1]
    x2 = x.reshape(-1, cols)
    for r0, r1 in _row_blocks(x2.shape[0], cols):
        xd = x2[r0:r1].to(torch.float64)
        t = xd * (xd.pow(2).mean(dim=1, keepdim=True) + eps).rsqrt()
        rel = (_gamma(depth + 1) + 2 * U32) / 2 + 2.0 ** -22 + U32
        yield r0, r1, t, t.abs() * rel * (1 + U32)


def rmsnorm_then(w: torch.Tensor):
    """the output as a function of the intermediate bf16(x rstd) [rows, cols] (flattened): bf16(w * m)"""
    wd = w.to(torch.float64)
    return lambda m: bf16_rne64(m.reshape(-1, wd.shape[0]) * wd)


def mean_eps(n, sum_abs: torch.Tensor, mean: torch.Tensor, inv: bool, min_ulp: torch.Tensor) -> torch.Tensor:
    """bound on |fp32 mean of n bf16 values - exact mean| (n a number or a tensor of window sizes):
      * the sequential sum: every value, so every partial sum, is a multiple of the smallest bf16 ulp among
        them (min_ulp), and a multiple of it below 2^24 min_ulp in magnitude is an fp32 number: where sum|v| is
        below that, the sum is exact; elsewhere it errs by <= gamma_(n-1) sum|v|;
      * then either a division by n (u |mean|) or (inv) a product with fl(1 / n) (u for the reciprocal, u for
        the product).  After an exact sum that last step is one fp32 operation on known values, so its
        error is computed exactly instead of bounded.
    This matters: the mean of two bf16 values of one binade is a bf16 rounding tie half the time, and fp32
    computes it exactly, so round-to-nearest-even decides it, with no tie window."""
    n = torch.as_tensor(n, dtype=torch.float64, device=mean.device)
    exact_sum = sum_abs < 2.0 ** 24 * min_ulp
    e_sum = torch.where(exact_sum, torch.zeros_like(sum_abs), (n - 1) * U32 / (1 - (n - 1) * U32) * sum_abs / n)
    # with an exact sum s the last step is one known fp32 operation: its result is computed exactly here
    s = torch.round(mean * n / min_ulp.clamp(max=1e300)) * min_ulp  # the sum, snapped to its grid
    if inv:
        r = (1.0 / n).to(torch.float32).to(torch.float64)
        one = (s * r).to(torch.float32).to(torch.float64)  # s * fl(1/n): 48 bits, exact in fp64
    else:
        one = (s / n).to(torch.float32).to(torch.float64)  # fp32 division: correctly rounded
    e_exact = (one - mean).abs()
    e_div = torch.where(exact_sum & torch.isfinite(e_exact), e_exact,
                        (2 if inv else 1) * U32 * mean.abs() * (1 + U32))
    return e_sum + e_div


def _min_ulp(v: torch.Tensor) -> torch.Tensor:
    """bf16 ulp of each value, +inf at zeros (which are multiples of anything)"""
    return torch.where(v != 0, bf16_ulp(v), torch.full_like(v, float("inf")))


def s2_merge_reference(tiles: torch.Tensor, splits_h, splits_w, out_bh: int, out_bw: int, share_tile=False):
    """the dynamic-S2 merge of ONE image in fp64, as the reference composes it (oracle.merge_chessboard per scale,
    F.interpolate(mode="area") == F.adaptive_avg_pool2d, the channel concatenation, oracle.split_chessboard),
    plus the fp32 bound of the kernel's windowed mean (mean_eps with the reciprocal).  tiles [n, side^2, C]
    -> (ref_final, eps) [out_bh * out_bw, side^2, n_scales * C]."""
    import torch.nn.functional as F
    n, N, C = tiles.shape
    side = int(round(N ** 0.5))
    t = tiles.to(torch.float64)
    OH, OW = out_bh * side, out_bw * side
    refs, epss = [], []
    cnt = 0
    for sh, sw in zip(splits_h, splits_w):
        k = sh * sw
        src = t[0:1] if share_tile else t[cnt:cnt + k]
        if not share_tile:
            cnt += k
        fmap = O.merge_chessboard(src, sh, sw) if not share_tile else \
            src.reshape(1, side, side, C).permute(0, 3, 1, 2)
        ref = F.adaptive_avg_pool2d(fmap, (OH, OW))
        sa = F.adaptive_avg_pool2d(fmap.abs(), (OH, OW))
        mu = -F.adaptive_max_pool2d(-_min_ulp(fmap), (OH, OW))
        # window sizes: [floor(o I / O), ceil((o + 1) I / O))
        IH, IW = fmap.shape[-2:]
        oy, ox = torch.arange(OH), torch.arange(OW)
        ny = (((oy + 1) * IH + OH - 1) // OH - (oy * IH) // OH).to(torch.float64)
        nx = (((ox + 1) * IW + OW - 1) // OW - (ox * IW) // OW).to(torch.float64)
        nwin = (ny[:, None] * nx[None, :]).to(t.device)
        e = mean_eps(nwin, sa * nwin, ref, inv=True, min_ulp=mu)
        refs.append(ref)
        epss.append(e)

    def split(m):
        return O.split_chessboard(torch.cat(m, dim=1), out_bh, out_bw).flatten(2).transpose(1, 2)
    return split(refs), split(epss)


def tsp_pool_reference(x: torch.Tensor, pt: int, ph: int, pw: int):
    """TSP pooling in fp64 with the reference's three bf16 rounding points (t-mean, then h-mean, then w-mean,
    each rounded: three chained .mean() on bf16 tensors).  x [T, h, w, C] -> (ref_final, eps) of the last
    rounding, [T/pt, h/ph, w/pw, C].  An earlier rounding that lies within its own eps of a tie may go either
    way in fp32; each such possible flip widens the next stage's eps by its ulp / pool (so the window of the
    final rounding includes every value a flipped intermediate can lead to)."""
    T, h, w, C = x.shape
    v = x.to(torch.float64)
    extra = torch.zeros_like(v)
    for dim, p in ((0, pt), (1, ph), (2, pw)):
        shp = v.shape[:dim] + (v.shape[dim] // p, p) + v.shape[dim + 1:]
        grp = v.reshape(shp)
        mean = grp.mean(dim + 1)
        e = mean_eps(p, grp.abs().sum(dim + 1), mean, inv=False, min_ulp=_min_ulp(grp).amin(dim + 1)) \
            + extra.reshape(shp).sum(dim + 1) / p
        if dim == 2:
            return mean, e
        v = bf16_rne64(mean)
        win = bf16_rne64(mean - e) != bf16_rne64(mean + e)
        extra = torch.where(win, bf16_ulp(v), torch.zeros_like(v))
