"""CPU: the prefill-attention checker of tests/test_attention_gpu.py, checked without a GPU.

emulate_fmha restates the arithmetic of fmha_fwd_kernel (fmha_wgmma.cu) in fp32: 128-row query tiles,
128-token KV blocks, fp32 scores times scale*log2(e) with a running maximum, P rounded to bf16 before the
PV product while the row sum l adds the unrounded P, the fp32 alpha rescale, one final bf16 rounding.
  * tests.helpers.AttnErrors accepts it, with margin, on the three input families of
    tests.helpers.attention_inputs, at D = 72 (non-causal, two sequences back to back as SigLIP lays them
    out) and D = 128 (causal GQA, Sq < Sk), Sq and Sk not multiples of 128;
  * it rejects each fault the kernel could make that the loose global bound of test_kernels_gpu.py lets
    through, planted into the emulation where the kernel would make it, and the check that targets the
    fault is the one that fails:
      diag_off_by_one  the causal mask lets row i see key i + off + 1           probe, per element
      tail_unmasked    the last KV block's slots past Sk are not masked         probe, per element
      block_skipped    a KV block left out                                       random, per element
      block_twice      a KV block summed twice                                   random, per element
      alpha_missing    O not rescaled when the running maximum grows             random, per element
      p_truncated      P rounded toward zero before the PV product               random, rounding bias
      gqa_mod          query head h reads KV head h % Hkv in the last query tile random, per element
      wg2_zeroed       rows 64..127 of one query tile left at zero               random, per element
"""
import pytest
import torch

from tests.helpers import ATTN_FAMILIES, AttnErrors, attention_errors, attention_inputs

BQ = BKV = 128
LOG2E = 1.4426950408889634


def _cdiv(a, b):
    return -(-a // b)


def _bf16_rz(t):
    """bf16 by truncation (round toward zero)"""
    return (t.to(torch.float32).view(torch.int32) & -65536).view(torch.float32).to(torch.bfloat16)


def emulate_fmha(q, k, v, Sk, *, causal, scale, fault=None):
    """fmha_fwd_kernel for one sequence, in fp32 on the CPU.  q [Sq, Hq, D] bf16; k, v [>= 128 *
    ceil(Sk / 128), Hkv, D] bf16: every key slot the kernel's TMA loads, the ones at and past Sk included
    (the next sequence's rows, or a page's unused tail).  Returns the bf16 output [Sq, Hq, D]."""
    Sq, Hq, D = q.shape
    Hkv = k.shape[1]
    off = Sk - Sq
    sl2 = torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)
    out = torch.empty(Sq, Hq, D, dtype=torch.bfloat16)
    ntile = _cdiv(Sq, BQ)
    for h in range(Hq):
        for qt in range(ntile):
            hk = h % Hkv if fault == "gqa_mod" and qt == ntile - 1 else h // (Hq // Hkv)
            r0, r1 = qt * BQ, min(Sq, (qt + 1) * BQ)
            Q = q[r0:r1, h].float()
            rows = torch.arange(r0, r1)[:, None]
            kv_end = min(Sk, r1 + off) if causal else Sk
            blocks = list(range(_cdiv(kv_end, BKV)))
            if fault in ("block_skipped", "block_twice") and len(blocks) > 2:
                blocks.insert(2, 1) if fault == "block_twice" else blocks.remove(1)
            m = torch.full((r1 - r0,), float("-inf"))
            l = torch.zeros(r1 - r0)
            O = torch.zeros(r1 - r0, D)
            for j in blocks:
                kv0 = j * BKV
                K, V = k[kv0:kv0 + BKV, hk].float(), v[kv0:kv0 + BKV, hk].float()
                S = Q @ K.t()
                tail = kv0 + BKV > Sk and fault != "tail_unmasked"
                if tail or (causal and kv0 + BKV - 1 > r0 + off):
                    lim = Sk - 1
                    if causal:
                        lim = torch.clamp(rows + off + (1 if fault == "diag_off_by_one" else 0), max=Sk - 1)
                    S = S.masked_fill(kv0 + torch.arange(BKV)[None, :] > lim, float("-inf"))
                m_new = torch.maximum(m, S.amax(dim=1) * sl2)
                m_use = torch.where(m_new == float("-inf"), torch.zeros_like(m_new), m_new)
                alpha = torch.exp2(m - m_use)
                P = torch.exp2(S * sl2 - m_use[:, None])
                l = l * alpha + P.sum(dim=1)
                Pb = _bf16_rz(P) if fault == "p_truncated" else P.to(torch.bfloat16)
                if fault != "alpha_missing":
                    O = O * alpha[:, None]
                O = O + Pb.float() @ V
                m = m_new
            res = O * (1.0 / l)[:, None]
            if fault == "wg2_zeroed" and qt == 0:
                res[64:] = 0.0
            out[r0:r1, h] = res.to(torch.bfloat16)
    return out


# causal GQA at D = 128: 200 queries at positions 133..332 against 333 keys (3 KV blocks, the last one
# 77 tokens), 2 query tiles (128 + 72 rows); the slots 333..383 of the last block hold garbage
CAUSAL = dict(Sq=200, Sk=333, Hq=4, Hkv=2, D=128)
# SigLIP layout at D = 72: B = 2 sequences of 200 tokens back to back; sequence 0's last KV block reads
# sequence 1's first 56 keys, sequence 1's reads past the buffer (TMA fills zeros)
NONCAUSAL = dict(B=2, S=200, H=2, D=72)


def _causal_case(family, fault=None, seed=0):
    c = CAUSAL
    Sq, Sk, D = c["Sq"], c["Sk"], c["D"]
    scale = D ** -0.5
    slots = _cdiv(Sk, BKV) * BKV
    pos = torch.arange(slots)
    q, k, v = attention_inputs(family, torch.arange(Sk - Sq, Sk), pos, c["Hq"], c["Hkv"], D, scale,
                               sink=pos == 0, garbage=pos >= Sk, seed=seed)
    got = emulate_fmha(q, k, v, Sk, causal=True, scale=scale, fault=fault)
    return attention_errors(got, q, k[:Sk], v[:Sk], causal=True, scale=scale), got


def _noncausal_case(family, fault=None, seed=0):
    c = NONCAUSAL
    B, S, H, D = c["B"], c["S"], c["H"], c["D"]
    scale = D ** -0.5
    pos = torch.arange(B * S)
    q, k, v = attention_inputs(family, pos, pos, H, H, D, scale, sink=pos % S == 0, seed=seed)
    pad = _cdiv(S, BKV) * BKV - S
    kz = torch.cat([k, torch.zeros(pad, H, D, dtype=k.dtype)])  # TMA's out-of-bounds fill
    vz = torch.cat([v, torch.zeros(pad, H, D, dtype=v.dtype)])
    e = AttnErrors()
    outs = []
    for b in range(B):
        sl = slice(b * S, (b + 1) * S)
        got = emulate_fmha(q[sl], kz[b * S:b * S + S + pad], vz[b * S:b * S + S + pad], S, causal=False,
                           scale=scale, fault=fault)
        attention_errors(got, q[sl], k[sl], v[sl], causal=False, scale=scale, into=e, row0=b * S * H)
        outs.append(got)
    return e, torch.cat(outs)


CASES = {"causal-d128": _causal_case, "noncausal-d72": _noncausal_case}


def _caught(e):
    """the checks of AttnErrors that fail"""
    out = set()
    if not e.excess <= 1.0:
        out.add("element")
    if not e.worst_row <= e.ROW_RMS:
        out.add("row")
    if not abs(e.bias) <= e.BIAS_ULP:
        out.add("bias")
    return out


@pytest.mark.parametrize("family", ATTN_FAMILIES)
@pytest.mark.parametrize("case", list(CASES))
def test_checker_accepts_kernel_arithmetic(case, family):
    """The emulated kernel passes every check with margin: no element uses more than 0.6 of its bound
    (1 ulp + 2^-7 A; a single flipped rounding costs at most 0.5 of it), with the fp32 scores, running
    maxima and alpha products in place; no row exceeds 2 of the per-row bound's 3 (2 is a row whose every
    element is one ulp off); the rounding bias stays within 0.05 ulp."""
    for seed in range(3):
        e, _ = CASES[case](family, seed=seed)
        assert not e.failures(), (case, family, seed, e.summary())
        assert e.excess <= 0.6 and e.worst_row <= 2.0 and abs(e.bias) <= 0.05, (case, family, seed, e.summary())


# fault -> (case, family, the check that must catch it)
FAULTS = {
    "diag_off_by_one": ("causal-d128", "probe", "element"),
    "tail_unmasked": ("noncausal-d72", "probe", "element"),
    "block_skipped": ("causal-d128", "random", "element"),
    "block_twice": ("causal-d128", "random", "element"),
    "alpha_missing": ("causal-d128", "random", "element"),
    "p_truncated": ("causal-d128", "random", "bias"),
    "gqa_mod": ("causal-d128", "random", "element"),
    "wg2_zeroed": ("causal-d128", "random", "element"),
}


@pytest.mark.parametrize("fault", list(FAULTS))
def test_checker_rejects_planted_fault(fault):
    case, family, check = FAULTS[fault]
    e, got = CASES[case](family, fault=fault)
    assert check in _caught(e), (fault, e.summary())
    if fault == "p_truncated":  # every element stays within its bound: only the mean sees it
        assert _caught(e) == {"bias"} and e.bias < -0.2, e.summary()


@pytest.mark.parametrize("fault", list(FAULTS))
def test_planted_fault_changes_the_output(fault):
    """each planted fault really changes the emulated output (the fault is not a no-op at these shapes)"""
    case, family, _ = FAULTS[fault]
    _, clean = CASES[case](family)
    _, bad = CASES[case](family, fault=fault)
    assert not torch.equal(clean, bad)
