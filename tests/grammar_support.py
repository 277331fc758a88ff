"""Grammar matchers for the constrained-decoding tests: a pure-Python matcher with xgrammar's GrammarMatcher interface
(fill_next_token_bitmask, accept_token, is_terminated), a recorder of the masks a matcher fills, and an xgrammar
compiler over a toy JSON vocabulary padded to a model's V."""
from __future__ import annotations

import numpy as np
import torch

from vila_b200.grammar import bitmask_words


def pack(allowed: np.ndarray, words: int) -> np.ndarray:
    """bool [V] -> int32 [words] in xgrammar's layout (bits at or above V clear)"""
    bits = np.zeros(words * 32, dtype=np.uint64)
    bits[:allowed.shape[0]] = allowed
    return (bits.reshape(-1, 32) << np.arange(32, dtype=np.uint64)).sum(axis=1).astype(np.uint32).view(np.int32)


class PyMatcher:
    """allowed(step, history) -> bool [V] gives each step's allowed ids; accepting an id of `stop` terminates"""

    def __init__(self, V: int, allowed, stop=()):
        self.V, self.allowed, self.stop = V, allowed, set(stop)
        self.history, self.terminated = [], False

    def fill_next_token_bitmask(self, mask, index: int = 0) -> bool:
        mask[index] = torch.from_numpy(pack(self.allowed(len(self.history), self.history), bitmask_words(self.V)))
        return True

    def accept_token(self, token: int) -> bool:
        if self.terminated or not self.allowed(len(self.history), self.history)[token]:
            return False
        self.history.append(token)
        self.terminated = token in self.stop
        return True

    def is_terminated(self) -> bool:
        return self.terminated


def allow_all(V: int) -> PyMatcher:
    return PyMatcher(V, lambda t, h: np.ones(V, dtype=bool))


def random_subsets(V: int, seed: int, density: float = 0.05) -> PyMatcher:
    """each step its own seeded random subset of about density * V ids (at least one)"""
    def allowed(t, h):
        rng = np.random.default_rng((seed, t))
        a = rng.random(V) < density
        a[rng.integers(V)] = True
        return a
    return PyMatcher(V, allowed)


class Recorder:
    """a matcher's proxy that keeps a copy of every mask it fills and every id it accepts"""

    def __init__(self, m):
        self.m, self.masks, self.accepted = m, [], []

    def fill_next_token_bitmask(self, mask, index: int = 0):
        r = self.m.fill_next_token_bitmask(mask, index)
        self.masks.append(mask[index].clone())
        return r

    def accept_token(self, token: int) -> bool:
        self.accepted.append(token)
        return self.m.accept_token(token)

    def is_terminated(self) -> bool:
        return self.m.is_terminated()


# a toy vocabulary for JSON: id 0 is the stop token; id 2 and the ids past the list are padding, which a JSON grammar
# allows only inside strings
TOY_JSON = ["</s>", "{", "<unused>", "}", "[", "]", ":", ",", " ", "\"", "\"a\"", "\"b\"", "\"name\"", "\"age\"", "0", "1", "2",
            "7", "42", "true", "false", "null", "\"x\"", "\"hi\"", "a", "b", "-", ".", "e", "\n", "  ", "{\"", "\"}"]


def toy_compiler(V: int, stop=(0,), whitespace: bool = True):
    """an xgrammar GrammarCompiler over TOY_JSON padded to V entries -> (compiler, vocabulary).  whitespace=False
    turns the whitespace tokens into padding, so a schema without strings leaves the model no way to delay the end."""
    import xgrammar as xgr
    vocab = [t if whitespace or t.strip() else f"<ws{i}>" for i, t in enumerate(TOY_JSON)]
    vocab += [f"<pad{i}>" for i in range(V - len(TOY_JSON))]
    return xgr.GrammarCompiler(xgr.TokenizerInfo(vocab, vocab_size=V, stop_token_ids=list(stop))), vocab
