"""OpenAI presence and frequency penalties of the continuous-batching engine: the parameters and the rule.

A request has a presence penalty p and a frequency penalty f, both finite and in [-2, 2] (OpenAI's range), held as
fp32.  It draws its token at index t (t = 0 is the token chosen from the prefill logits).  Let c_j be the number of
times id j occurs among the ids the request generated at indices 0..t-1.  Only generated ids count, not the prompt's
(OpenAI's definition; the batched engine sees the prompt as embeddings only).  On the bf16 logits row x:

  pen_j = fp32(fp32(c_j) * f) + p            (IEEE fp32, round to nearest at each operation, no FMA contraction)
  y_j   = bf16_rn(fp32(x_j) - pen_j)         if c_j > 0
  y_j   = x_j                                otherwise (bit-identical copy)

Greedy decoding and temperature / top-k / top-p sampling (vila_b200/sampling.py) then apply to y instead of x.  Token 0
has an empty history, so it is never penalised.  Logprobs (vila_b200/logprobs.py) stay those of the raw row x.

The bf16 rounding of y adds at most half a bf16 ulp of |y| to the exact x_j - pen_j: 0.0625 for |y| in [16, 32), the
same order as the logit error the decode engines already carry.

csrc/penalties.cu (vila_apply_penalties) implements the rule bit for bit.  reference_penalized states it in numpy;
reference_penalized64 is the same rule in fp64 without the final rounding, for comparisons against the fp32 oracle.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

PENALTY_LIMIT = 2.0  # OpenAI's range for both penalties: [-2, 2]


@dataclass(frozen=True)
class PenaltyParams:
    """One request's presence and frequency penalties, each a finite number in [-2, 2] (ValueError otherwise).
    Both 0 is `off`: the request decodes as without penalties."""
    presence: float = 0.0
    frequency: float = 0.0

    def __post_init__(self):
        for name in ("presence", "frequency"):
            v = getattr(self, name)
            if (not isinstance(v, (int, float, np.integer, np.floating)) or isinstance(v, bool)
                    or not math.isfinite(v) or not -PENALTY_LIMIT <= v <= PENALTY_LIMIT):
                raise ValueError(f"{name} penalty must be a finite number in [-2, 2], got {v!r}")

    @property
    def off(self) -> bool:
        return self.presence == 0 and self.frequency == 0


def counts(history, t: int, V: int) -> np.ndarray:
    """c [V] int64: occurrences of each id in [0, V) among history[0 : min(t, len(history))]"""
    h = np.asarray(torch.as_tensor(history).cpu(), dtype=np.int64).reshape(-1)[:max(0, min(t, len(history)))]
    h = h[(h >= 0) & (h < V)]
    return np.bincount(h, minlength=V).astype(np.int64)


def reference_penalized(row, history, t: int, presence: float, frequency: float) -> torch.Tensor:
    """The rule on one bf16 row (V values), bit for bit.  history: the request's generated ids (int, any length; the
    first min(t, len) count, ids outside [0, V) are ignored).  -> bf16 [V]"""
    x = torch.as_tensor(row).cpu()
    assert x.dtype == torch.bfloat16, "the rule is stated on a bf16 row"
    V = x.shape[0]
    c = counts(history, t, V)
    hit = c > 0
    pen = (c[hit].astype(np.float32) * np.float32(frequency)).astype(np.float32) + np.float32(presence)
    y = x.clone()
    xf = x.float().numpy()[hit]
    y[torch.from_numpy(hit)] = torch.from_numpy((xf - pen.astype(np.float32)).astype(np.float32)).to(torch.bfloat16)
    return y


def reference_penalized64(row, history, t: int, presence: float, frequency: float) -> np.ndarray:
    """The rule in fp64 without any rounding: x_j - (c_j f + p) where c_j > 0, x_j elsewhere.  row: bf16 / fp32 /
    fp64 values [V] (the fp32 oracle's logits).  -> fp64 [V]"""
    x = torch.as_tensor(row).double().cpu().numpy().copy()
    c = counts(history, t, x.shape[0])
    hit = c > 0
    x[hit] -= c[hit] * float(np.float32(frequency)) + float(np.float32(presence))
    return x
