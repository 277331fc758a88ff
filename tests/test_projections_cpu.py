"""CPU: the tools of tests/test_projections_gpu.py, checked without a GPU.

  * the bf16 checker (tests.helpers.Bf16Errors) accepts a GEMM output that differs from the fp64
    reference only by fp32 accumulation and bf16 rounding, and rejects each fault a tiled GEMM could make
    that a loose global bound lets through: a k-block dropped or summed twice in one tile, the residual
    added twice, the bias missing from one column group, gate and up swapped in one SwiGLU group, the last
    row of a partial M tile zeroed or copied, round-toward-zero instead of round-to-nearest;
  * the dispatch mirror (tests.helpers.dispatch_flavour) against the regimes of gemm_bf16 worked out by
    hand for 132 SMs and a 96 MiB workspace, and its stream-K fallback when the workspace is too small.
"""
import math

import pytest
import torch

from tests.helpers import Bf16Errors, bf16_ulp, dispatch_flavour, linear_reference, streamk_fits

M, N, K = 130, 256, 1088  # two M tiles (the second holds 2 rows), two 128-wide N tiles, 17 k-blocks
TILE = (slice(0, 128), slice(128, 256))  # the 128 x 128 tile the faults are planted in
KB = slice(5 * 64, 6 * 64)               # one 64-wide k-block


def _problem(seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g)
    x[:, [3, 500, 1000]] = 50.0 * torch.sign(torch.randn(M, 3, generator=g))  # outlier channels
    x = x.to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(torch.bfloat16)
    b = torch.randn(N, generator=g).to(torch.bfloat16)
    r = torch.randn(M, N, generator=g).to(torch.bfloat16)
    return x, w, b, r


def _product(x, w, dtype):
    return (x.to(dtype) @ w.to(dtype).t()).to(torch.float64)


def _errors(got, ref_final):
    return Bf16Errors().add(got, ref_final)


def _rz(t):
    """bf16 by truncation (round toward zero)"""
    bits = t.to(torch.float32).view(torch.int32) & -65536
    return bits.view(torch.float32).to(torch.bfloat16)


EPILOGUES = {
    "plain": dict(),
    "bias": dict(bias=True),
    "residual": dict(residual=True),
    "bias+residual": dict(bias=True, residual=True),
    "bias+gelu_tanh": dict(bias=True, act="gelu_tanh"),
    "bias+gelu_erf": dict(bias=True, act="gelu_erf"),
    "swiglu": dict(swiglu=True),
}


def _ref(P, b, r, spec):
    return linear_reference(P, bias=b if spec.get("bias") else None, act=spec.get("act"),
                            residual=r if spec.get("residual") else None, swiglu=spec.get("swiglu", False))


@pytest.mark.parametrize("epi", list(EPILOGUES))
def test_checker_accepts_fp32_accumulation_and_rounding(epi):
    """A GEMM that accumulates in fp32 (another summation order than fp64) and rounds to nearest passes,
    also where its final rounding goes the other way (planted here in 3 % of the outputs: an fp32 sum
    that lands on the other side of a rounding boundary)."""
    x, w, b, r = _problem(1)
    spec = EPILOGUES[epi]
    r = r[:, :N // 2] if spec.get("swiglu") else r
    truth = _ref(_product(x, w, torch.float64), b, r, spec)
    got = _ref(_product(x, w, torch.float32), b, r, spec).to(torch.bfloat16).double()
    flip = torch.rand(got.shape, generator=torch.Generator().manual_seed(3)) < 0.03
    other = got + torch.sign(truth - got) * bf16_ulp(got)  # the other bf16 neighbour of truth
    got = torch.where(flip & (truth != got), other, got).to(torch.bfloat16)
    assert (got != truth.to(torch.bfloat16)).sum().item() > 0.01 * got.numel()  # (a residual sum is often exact)
    e = _errors(got, truth)
    assert not e.failures(), (epi, e.summary())
    assert e.max_ulps >= 0.5, e.summary()


def _faulty_products():
    x, w, b, r = _problem(2)
    P = _product(x, w, torch.float64)
    kblk = torch.zeros_like(P)
    kblk[TILE] = _product(x[TILE[0], KB], w[TILE[1], KB], torch.float64)
    return x, w, b, r, P, kblk


FAULTS = ["kblock_dropped", "kblock_twice", "residual_twice", "bias_missing_group", "swiglu_swapped_group",
          "tail_row_zeroed", "tail_row_copied", "round_toward_zero"]


@pytest.mark.parametrize("fault", FAULTS)
def test_checker_rejects_planted_fault(fault):
    x, w, b, r, P, kblk = _faulty_products()
    spec = EPILOGUES["swiglu" if fault == "swiglu_swapped_group" else "bias+residual"]
    rr = r[:, :N // 2] if spec.get("swiglu") else r
    truth = _ref(P, b, rr, spec)
    got = None
    if fault == "kblock_dropped":
        got = _ref(P - kblk, b, rr, spec)
    elif fault == "kblock_twice":
        got = _ref(P + kblk, b, rr, spec)
    elif fault == "residual_twice":
        got = truth.clone()
        got[TILE] += r[TILE].double()
    elif fault == "bias_missing_group":
        bb = b.clone()
        bb[136:144] = 0
        got = _ref(P, bb, rr, spec)
    elif fault == "swiglu_swapped_group":
        Ps = P.clone()
        Ps[:, 136:144] = P[:, 136:144].view(M, 4, 2).flip(-1).reshape(M, 8)  # (gate, up) -> (up, gate)
        got = _ref(Ps, b, rr, spec)
    elif fault == "tail_row_zeroed":
        got = truth.clone()
        got[M - 1] = 0
    elif fault == "tail_row_copied":
        got = truth.clone()
        got[M - 1] = got[M - 2]
    if fault == "round_toward_zero":
        got = _rz(truth)
    else:
        got = got.to(torch.bfloat16)
    e = _errors(got, truth)
    assert e.failures(), (fault, e.summary())
    if fault == "round_toward_zero":  # only the bias check sees it: every element is within 1 ulp
        assert e.max_ulps <= 1.0 and e.bias < -0.3, e.summary()


# ------------------------------------------------------------------------------------------------
# dispatch mirror
# ------------------------------------------------------------------------------------------------
SMS, WS = 132, 96 << 20
DOWN, QKV, GATE_UP = (3584, 18944), (4608, 3584), (37888, 3584)  # NVILA-8B (N, K)

# gemm_bf16 by hand, 8B down projection (28 n-blocks of 128, 296 k-blocks):
#   split-K pairs when the 128 x 128 grid fits one wave of pairs (<= 66 tiles: 1-2 m-blocks) and the
#   last m-block is >= 90 % full (M 116-128, 231-256); else long K under one wave: stream-K up to 66
#   tiles (M <= 256), split-K pairs up to 131 tiles (M 257-512); then 128-wide tiles until the 256-wide
#   grid fills 70 % of the SMs (7 m-blocks x 14 = 98 >= 92.4: M >= 769)
MIRROR_CASES = [
    (DOWN, 8, 1128), (DOWN, 115, 1128), (DOWN, 116, 5128), (DOWN, 120, 5128), (DOWN, 128, 5128),
    (DOWN, 129, 1128), (DOWN, 200, 1128), (DOWN, 230, 1128), (DOWN, 231, 5128), (DOWN, 300, 5128),
    (DOWN, 512, 5128), (DOWN, 513, 128), (DOWN, 600, 128), (DOWN, 768, 128), (DOWN, 769, 256),
    (DOWN, 1000, 256), (DOWN, 16470, 256),
    # q/k/v: 36 n-blocks; split-K pairs only for one near-full m-block; 256-wide from 6 m-blocks (108)
    (QKV, 100, 128), (QKV, 120, 5128), (QKV, 279, 128), (QKV, 640, 128), (QKV, 641, 256), (QKV, 700, 256),
    # gate/up: 148 tiles of 256 at M = 1 already fill the SMs
    (GATE_UP, 1, 256), (GATE_UP, 279, 256), (GATE_UP, 16470, 256),
    # 8B projector at one image (256 tokens): 2 x 28 tiles, K >= 2048 -> split-K pairs
    ((3584, 4608), 256, 5128), ((3584, 3584), 256, 5128),
    # ViT fc2 at one image (1024 x 1152 x 4304): 8 x 9 = 72 tiles > 66 -> 128-wide tiles
    ((1152, 4304), 1024, 128),
]


@pytest.mark.parametrize("NK,M,want", MIRROR_CASES)
def test_dispatch_mirror_by_hand(NK, M, want):
    N, K = NK
    assert dispatch_flavour(M, N, K, SMS, WS) == want


def test_dispatch_streamk_falls_back_without_workspace():
    N, K = DOWN
    # M = 200: 56 tiles, 296 k-blocks over 132 CTAs -> 125 per CTA -> 4 slots per tile:
    # 64 KiB of counters + 56 * 4 fp32 128 x 128 tiles
    need = 64 * 1024 + 56 * 4 * 128 * 128 * 4
    assert streamk_fits(200, N, K, SMS, need) and not streamk_fits(200, N, K, SMS, need - 1)
    assert dispatch_flavour(200, N, K, SMS, need) == 1128
    assert dispatch_flavour(200, N, K, SMS, need - 1) == 128
    assert dispatch_flavour(8, N, K, SMS, 0) == 128  # no workspace registered
    # the other regimes do not depend on the workspace
    for M, want in ((120, 5128), (300, 5128), (600, 128), (1000, 256)):
        assert dispatch_flavour(M, N, K, SMS, 0) == want
