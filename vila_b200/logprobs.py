"""Per-token log-probabilities of the continuous-batching engine: the result type and the rule.

The rule, for one row x of bf16 logits (length V, the row the engine chose the token from), the chosen token t and
n in 0..20:

  1. m = max_i float(x_i), Z = sum_i exp(float(x_i) - m), lse = m + log Z.
  2. logprob(t) = float(x_t) - lse.
  3. top = the first n indices of a stable sort by float(x_i) descending (ties to the lower index), each with its
     value float(x_j) - lse.

The distribution is the raw model distribution: temperature 1, no top-k or top-p filtering, whatever the request was
sampled with (OpenAI's meaning of `logprobs`).  In the fp8 and w4a16 decode-weight modes the row is the one the mode's
e4m3 lm_head produced, since that is the row the engine chose from.

csrc/sample.cu (vila_token_logprobs) computes (float(x_j) - m) - log Z in fp32 with expf / logf and fixed-order sums;
its top ids equal the rule's, and its values are within VALUE_ATOL + VALUE_RTOL * |lp| of reference_logprobs (fp64).
"""
from __future__ import annotations

from typing import List, NamedTuple, Tuple

import numpy as np
import torch

MAX_TOP_LOGPROBS = 20  # OpenAI's top_logprobs limit, and the kernel's
VALUE_ATOL, VALUE_RTOL = 1e-5, 1e-6


class TokenLogprob(NamedTuple):
    """one generated token: its id, its log-probability and the `top` most likely ids with theirs, best first"""
    token: int
    logprob: float
    top: List[Tuple[int, float]]


def check_top(n) -> int:
    """a top-alternatives count: an integer in 0..MAX_TOP_LOGPROBS, else a ValueError"""
    if not isinstance(n, (int, np.integer)) or isinstance(n, bool) or not 0 <= n <= MAX_TOP_LOGPROBS:
        raise ValueError(f"logprobs must be an integer in 0..{MAX_TOP_LOGPROBS} (top alternatives per token), got {n!r}")
    return int(n)


def reference_logprobs(logits, token: int, n: int) -> Tuple[float, np.ndarray, np.ndarray]:
    """The rule on one row, in fp64.  logits: a bf16 / fp32 row of V values.
    -> (logprob of token, top ids int64 [n], top values fp64 [n])"""
    x = torch.as_tensor(logits).float().double().cpu().numpy()
    m = x.max()
    lse = m + np.log(np.exp(x - m).sum())
    top = np.argsort(-x, kind="stable")[:n]
    return float(x[token] - lse), top.astype(np.int64), x[top] - lse
