"""Temperature / top-k / top-p sampling of the continuous-batching engine: the parameters and the rule.

The rule, for a request with temperature T, top_k, top_p and a 64-bit seed, drawing its token at index t (t = 0 is
the token chosen from the prefill logits), on one row of bf16 logits of V entries:

  1. greedy   T == 0 or top_k == 1: the first index of max float(logit) (torch.argmax(logits.float())).
  2. scaling  s_i = float(logit_i) * inv_T in fp32, inv_T = fp32(1 / T) computed once on the host.
  3. top-k    top_k == 0 or top_k >= V: off.  Else keep s_i >= s_(k), the k-th largest value (ties kept, as HF
              TopKLogitsWarper).
  4. top-p    top_p == 1: off.  Else p_i = exp(s_i - max s), Z = sum of p over the top-k survivors; keep survivor i iff
              the mass of survivors with a strictly larger s is < top_p * Z.  For distinct values this is HF
              TopPLogitsWarper after the temperature and top-k warpers; ties at the boundary are all kept and the
              largest value always is.
  5. draw     the Gumbel-max over the kept set: argmax_i (s_i + g_i), ties to the lowest index.
              Philox-4x32-10 with key (seed & 0xffffffff, seed >> 32) and counter (i // 4, t & 0xffffffff, t >> 32, 0)
              gives four words; word i % 4 is x_i; u_i = (x_i + 0.5) * 2^-32; g_i = -log(-log1p(-u_i)).
              The draw of (request, t) depends only on the seed, t and the logits row.

csrc/sample.cu (vila_sample_batch) implements it with two stated differences, which the tests bound: the top-p masses
are summed as integers floor(fp32 exp(s_i - m) * 2^40), and g_i is computed in fp32 from u_i rounded to fp32 (exact
for the small u that win) and added to s_i in fp64.  The functions below state the rule in numpy, in fp64 where the
rule has real numbers: philox4x32_10 (the generator's words), kept_set (the kept mask) and reference_draw.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np
import torch

_M0, _M1 = 0xD2511F53, 0xCD9E8D57
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_MASK32 = 0xFFFFFFFF


@dataclass(frozen=True)
class SamplingParams:
    """One request's sampling parameters.  temperature 0 (or top_k 1) is greedy; top_k 0 and top_p 1 are off;
    seed None: generate_batch draws one from the host torch default generator (so torch.manual_seed reproduces
    a run).  Out-of-range values are ValueErrors."""
    temperature: float = 0.0
    top_k: int = 0
    top_p: float = 1.0
    seed: Optional[int] = None

    def __post_init__(self):
        t, p = self.temperature, self.top_p
        if not isinstance(t, (int, float)) or not math.isfinite(t) or t < 0:
            raise ValueError(f"temperature must be finite and >= 0, got {t!r}")
        if not isinstance(p, (int, float)) or not (0.0 < p <= 1.0):
            raise ValueError(f"top_p must be in (0, 1], got {p!r}")
        if not isinstance(self.top_k, int) or isinstance(self.top_k, bool) or self.top_k < 0:
            raise ValueError(f"top_k must be an integer >= 0, got {self.top_k!r}")
        if self.seed is not None and (not isinstance(self.seed, int) or not -2 ** 63 <= self.seed < 2 ** 64):
            raise ValueError(f"seed must be a 64-bit integer or None, got {self.seed!r}")

    @property
    def greedy(self) -> bool:
        return self.temperature == 0 or self.top_k == 1

    @property
    def inv_temperature(self) -> float:
        """the kernel's inv_T: fp32(1 / T), 0 for greedy"""
        return 0.0 if self.greedy else float(np.float32(1.0 / self.temperature))


def seed_words(seed: int) -> Tuple[int, int]:
    """a 64-bit seed (signed or not) -> Philox key (low 32 bits, high 32 bits)"""
    s = seed & 0xFFFFFFFFFFFFFFFF
    return s & _MASK32, s >> 32


def signed64(seed: int) -> int:
    """the seed as the int64 the device array holds"""
    s = seed & 0xFFFFFFFFFFFFFFFF
    return s - (1 << 64) if s >= 1 << 63 else s


def philox4x32_10(ctr, key) -> np.ndarray:
    """Philox-4x32-10 (Random123): ctr uint32 [..., 4], key (k0, k1) -> uint32 [..., 4]"""
    c = np.array(ctr, dtype=np.uint64).reshape(-1, 4) & _MASK32
    k0, k1 = int(key[0]) & _MASK32, int(key[1]) & _MASK32
    for r in range(10):
        if r:
            k0, k1 = (k0 + _W0) & _MASK32, (k1 + _W1) & _MASK32
        p0 = c[:, 0] * np.uint64(_M0)
        p1 = c[:, 2] * np.uint64(_M1)
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(_MASK32)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(_MASK32)
        c = np.stack([hi1 ^ c[:, 1] ^ np.uint64(k0), lo1, hi0 ^ c[:, 3] ^ np.uint64(k1), lo0], axis=1)
    return c.astype(np.uint32).reshape(np.shape(ctr))


def philox_words(seed: int, t: int, V: int) -> np.ndarray:
    """x_i for i in [0, V): uint32 [V]"""
    n = (V + 3) // 4
    ctr = np.zeros((n, 4), dtype=np.uint64)
    ctr[:, 0] = np.arange(n)
    ctr[:, 1] = t & _MASK32
    ctr[:, 2] = (t >> 32) & _MASK32
    return philox4x32_10(ctr, seed_words(seed)).reshape(-1)[:V]


def gumbel_noise(seed: int, t: int, V: int) -> np.ndarray:
    """g_i in fp64 [V]"""
    u = (philox_words(seed, t, V).astype(np.float64) + 0.5) * 2.0 ** -32
    return -np.log(-np.log1p(-u))


def scaled(logits, inv_temperature: float) -> np.ndarray:
    """s = float(logit) * inv_T in fp32 (-0 -> +0); logits: a bf16 / fp32 row"""
    x = torch.as_tensor(logits).float().cpu().numpy()
    s = (x * np.float32(inv_temperature)).astype(np.float32)
    s[s == 0] = 0.0
    return s


def kept_set(s: np.ndarray, top_k: int, top_p: float) -> Tuple[np.ndarray, float]:
    """The kept mask of fp32 scores s [V] (rules 3 and 4, fp64 masses) and the top-p decision margin: min over the
    survivors' distinct values v of |M(v) - top_p Z| / Z, M(v) the mass of survivors above v (inf when top-p is off).
    A row with a margin below the kernel's mass error may keep one value more or less there."""
    V = s.shape[0]
    keep = np.ones(V, dtype=bool)
    if 0 < top_k < V:
        kth = np.sort(s)[::-1][top_k - 1]
        keep = s >= kth
    if top_p >= 1.0:
        return keep, math.inf
    sd = s.astype(np.float64)
    p = np.where(keep, np.exp(sd - sd.max()), 0.0)
    Z = p.sum()
    vals, inv = np.unique(sd[keep], return_inverse=True)  # ascending
    mass_at = np.bincount(inv, weights=p[keep])
    above = np.concatenate([np.cumsum(mass_at[::-1])[::-1][1:], [0.0]])  # mass strictly above each value
    ok = above < top_p * Z
    thr = vals[ok].min()
    margin = float(np.min(np.abs(above - top_p * Z)) / Z)
    return keep & (sd >= thr), margin


def reference_draw(logits, inv_temperature: float, top_k: int, top_p: float, seed: int, t: int):
    """The rule on one row.  -> (token, kept mask [V], perturbed scores s + g in fp64 over the kept set (-inf
    elsewhere), top-p margin of kept_set); greedy rows: (argmax, one-hot mask, None, inf)"""
    x = torch.as_tensor(logits).float().cpu()
    V = x.shape[0]
    if inv_temperature == 0 or top_k == 1:
        tok = int(torch.argmax(x))
        mask = np.zeros(V, dtype=bool)
        mask[tok] = True
        return tok, mask, None, math.inf
    s = scaled(x, inv_temperature)
    keep, margin = kept_set(s, top_k, top_p)
    v = np.where(keep, s.astype(np.float64) + gumbel_noise(seed, t, V), -np.inf)
    return int(np.argmax(v)), keep, v, margin


def top2_gap(v: np.ndarray) -> float:
    """difference of the two largest perturbed scores (inf with one kept value)"""
    f = v[np.isfinite(v)]
    if f.size < 2:
        return math.inf
    a = np.partition(f, -2)[-2:]
    return float(a[1] - a[0])
