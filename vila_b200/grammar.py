"""Grammar-constrained decoding (structured output: `response_format` json_object / json_schema) in the single-stream
graph decoder: the rule.

A grammar matcher (xgrammar's GrammarMatcher, or any object with its fill_next_token_bitmask / accept_token /
is_terminated methods) fills, before each token, an int32 bitmask of ceil(V / 32) words in xgrammar's layout:

  allowed(j) = bit j % 32 of word j // 32 is set      (bits at or above V are ignored)

On the bf16 logits row x [V]:

  y_j = x_j      if allowed(j)   (bit-identical copy)
  y_j = -inf     otherwise

The token is chosen from the row as processors before warpers (HF's order): presence / frequency penalties when on
(vila_b200/penalties.py), then the mask, then vila_sample_finalize (vila_b200/sampling.py) on y.  Greedy (inv_T = 0) is
the first index of the max over the allowed ids; otherwise temperature, top-k and top-p apply to y, where the -inf
entries carry no mass and never win the draw.  Logprobs (vila_b200/logprobs.py) stay those of the raw row x.  A mask
that allows no id below V is refused on the host (ValueError) before the step runs.

csrc/token_bitmask.cu (vila_apply_token_bitmask_row) implements the mask bit for bit; reference_masked states it in
numpy.
"""
from __future__ import annotations

import numpy as np
import torch

NEG_INF_BF16 = 0xFF80


def bitmask_words(V: int) -> int:
    """int32 words of a token bitmask over V ids"""
    return (V + 31) // 32


def allowed_ids(bitmask, V: int) -> np.ndarray:
    """bool [V]: allowed(j) for j < V.  bitmask: int32 values (any shape, at least ceil(V / 32) of them)"""
    w = np.asarray(torch.as_tensor(bitmask).cpu(), dtype=np.int32).reshape(-1)[:bitmask_words(V)].view(np.uint32)
    j = np.arange(V)
    return ((w[j >> 5] >> (j & 31).astype(np.uint32)) & 1).astype(bool)


def any_allowed(bitmask: np.ndarray, V: int) -> bool:
    """whether an int32 bitmask [>= ceil(V / 32)] allows any id below V (the host's check before a constrained step)"""
    w = bitmask.reshape(-1).view(np.uint32)
    full, rem = divmod(V, 32)
    return bool(w[:full].any()) or (rem > 0 and bool(w[full] & np.uint32((1 << rem) - 1)))


def reference_masked(row, bitmask) -> torch.Tensor:
    """The rule on one bf16 row [V], bit for bit.  -> bf16 [V]"""
    x = torch.as_tensor(row).cpu()
    assert x.dtype == torch.bfloat16, "the rule is stated on a bf16 row"
    keep = torch.from_numpy(allowed_ids(bitmask, x.shape[0]))
    bits = torch.where(keep, x.view(torch.int16), torch.tensor(NEG_INF_BF16 - (1 << 16), dtype=torch.int16))
    return bits.view(torch.bfloat16)
