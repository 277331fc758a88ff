"""CPU: the decode GEMV checker (tests.helpers.GemvErrors), the independent quantizers and the launch-plan mirrors,
proven without a GPU.

  * quantize_e4m3_rows and quantize_w4_groups agree bit for bit with their re-derivation in tests.helpers
    (codes, scales, zero points, packed bytes), on edge rows and groups;
  * fp32 emulations of the kernels' arithmetic (gemv_tma.cu) pass GemvErrors with margin at K = 512, 3584 and
    18944 for every fusion: gemv_tma_kernel (bf16 and e4m3: two interleaved lane accumulators, the warp tree,
    the k-parts in order, then the row scale), gemv_w4_kernel (a fresh fp32 sum per group, times s, added to the
    row sum) and gemv_batch_kernel (per slice and part, then the cluster ranks in order);
  * each planted fault is rejected, through the check named in the test;
  * batch_partition's mirror, checked by hand at NVILA-8B's and Lite's shapes: no slice and no k-part is empty
    at any shape of the GPU table.
"""
import math

import pytest
import torch

from tests.helpers import (GemvErrors, W4_GROUP, W4_NIBBLES, batch_partition, e4m3_values, gemv_depth,
                           gemv_reference, gemv_tma_plan, gemv_w4_plan, gemv_xn, ref_quantize_e4m3_rows,
                           ref_quantize_w4, ref_w4_pack, ref_w4_unpack)
from tests.test_gemv_gpu import BATCH_TABLE, SINGLE_TABLE, SMS_H100, edge_groups

F32 = torch.float32


def rb(t):
    return t.to(torch.bfloat16).to(F32)


def rtz(t):
    """fp32 -> bf16 by truncation (round toward zero), as fp32"""
    return (t.contiguous().view(torch.int32) & ~0xFFFF).view(F32)


def _weights(N, K, seed, edges=False):
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(N, K, generator=g) / math.sqrt(K) * torch.exp(torch.randn(N, 1, generator=g))
         * torch.exp(0.5 * torch.randn(N, K // 128, generator=g)).repeat_interleave(128, 1))
    if edges:
        edge_groups(w)
    return w.to(torch.bfloat16)


def _row_scale(M):
    """batched x rows: 2^-8, 1 and 2^8 in turn"""
    return torch.tensor([2.0 ** (8 * (m % 3 - 1)) for m in range(M)])


def _x(M, K, seed, outliers=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g) * (_row_scale(M)[:, None] if M > 1 else 1.0)
    for m in range(M):  # outliers in every fifth row from row 3
        if outliers and m % 5 == 3:
            x[m, torch.randperm(K, generator=g)[:6]] = torch.tensor([1e4, -1e4] * 3)
    return x.to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------
# §1 the quantizers against their re-derivation
# ------------------------------------------------------------------------------------------------
def test_e4m3_value_table():
    v = e4m3_values()
    assert v[0x7E] == 448 and v[0xFE] == -448 and math.isnan(v[0x7F]) and math.isnan(v[0xFF])
    assert v[1] == 2.0 ** -9 and v[7] == 7 * 2.0 ** -9 and v[8] == 2.0 ** -6  # subnormals, then the first normal
    assert bool((v[1:127] > v[0:126]).all())
    ref = torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn).to(torch.float64)
    assert torch.equal(torch.nan_to_num(v, 7.0), torch.nan_to_num(ref, 7.0))


def test_quantize_e4m3_rows_bit_exact():
    from vila_b200.model.qwen2 import quantize_e4m3_rows
    w = _weights(1003, 512, seed=1).float()  # N not a multiple of 16
    w[3] = 0                                   # an all-zero row: s = 1, codes 0
    w[5] = w[5] * 1e-3
    w[5, 17] = 1.0                             # a large maximum: the rest of the row lands on subnormal codes
    w[6, 9], w[6, 10] = 2.5, -2.5              # codes at +-448
    w = w.to(torch.bfloat16)
    q, s = quantize_e4m3_rows(w, rows_per_chunk=256)
    rq, rs = ref_quantize_e4m3_rows(w)
    assert torch.equal(q.view(torch.uint8), rq) and torch.equal(s, rs)
    assert bool((rq[3] == 0).all()) and rs[3] == 1
    sub = (rq[5] & 0x78) == 0
    assert int((sub & ((rq[5] & 7) != 0)).sum()) > 100, "too few subnormal codes in row 5"
    assert int(rq[6, 9]) == 0x7E and int(rq[6, 10]) == 0xFE


def test_quantize_w4_groups_bit_exact():
    from vila_b200.model.qwen2 import quantize_w4_groups
    w = _weights(1003, 1024, seed=2, edges=True)  # N not a multiple of 16: the last tile is padded
    packed, s, z = quantize_w4_groups(w, rows_per_chunk=256)
    rq, rs, rz = ref_quantize_w4(w)
    assert torch.equal(s.float(), rs) and torch.equal(z, rz)
    assert torch.equal(packed, ref_w4_pack(rq))
    assert torch.equal(ref_w4_unpack(packed, 1003, 1024), rq)
    # the edge groups of edge_groups(): all zero (s = 1, z = 0, codes 0), all positive (z = 0), all negative (z = 15)
    assert rs[0, 0] == 1 and rz[0, 0] == 0 and bool((rq[0, :128] == 0).all())
    assert rz[1, 1] == 0 and rz[2, 2] == 15 and bool((rq[2, 256:384] <= 15).all())
    assert bool((rz[1:, 0] >= 0).all())
    # the layout comment: nibble 0 of the first u32 of tile 0 is row 0, k 0; nibble 1 row 8, k 0; nibble 4 row 0, k 1
    word = int(packed[0, 0]) | int(packed[0, 1]) << 8 | int(packed[0, 2]) << 16 | int(packed[0, 3]) << 24
    for p, (dr, dk) in enumerate(W4_NIBBLES):
        assert (word >> 4 * p) & 15 == int(rq[dr, dk])
    # lane 5 (g = 1, c = 1), u32 j = 2 of block 64: rows 1 and 9 at k0 = 64 + 16 + 8
    off = 1 * 512 + 5 * 16 + 2 * 4
    word = int.from_bytes(bytes(packed[0, off:off + 4].tolist()), "little")
    assert (word & 15) == int(rq[1, 88]) and (word >> 4 & 15) == int(rq[9, 88]) and (word >> 24 & 15) == int(rq[1, 91])


# ------------------------------------------------------------------------------------------------
# §3 fp32 emulations of the kernels
# ------------------------------------------------------------------------------------------------
def prologue(x, nw, eps=1e-6, shift=0):
    """the fused RMSNorm in fp32 (its own summation order); shift: the norm weight read `shift` elements off"""
    xf = x.float()
    rstd = torch.rsqrt((xf * xf).sum(dim=1, keepdim=True, dtype=F32) / x.shape[1] + eps)
    nwf = nw.float().roll(-shift) if shift else nw.float()
    return rb(rb(xf * rstd) * nwf).to(torch.bfloat16)


def emu_tma(wf, x, ksplit, per_vec, twice=None):
    """gemv_tma_kernel's row sums (before the row scale) for one x row: fp32 [N].  wf fp32 [N, K] (bf16 or e4m3
    values), per_vec = 8 (bf16) or 16 (e4m3) elements per 16-byte vector; twice: a k-part added twice"""
    N, K = wf.shape
    cv = K // ksplit // per_vec
    W = wf.view(N, ksplit, cv, per_vec)
    X = x.float().view(ksplit, cv, per_vec)
    lanes = torch.arange(32)
    s0, s1 = torch.zeros(N, ksplit, 32), torch.zeros(N, ksplit, 32)
    done = torch.zeros(32, dtype=torch.bool)
    i = 0
    while not bool(done.all()):
        v = lanes + 64 * i
        pair = ~done & (v + 32 < cv)
        leave = ~done & ~pair
        tail = leave & (v < cv)
        for e in range(per_vec):
            if bool(pair.any()):
                a, b = v[pair], v[pair] + 32
                s0[:, :, pair] = s0[:, :, pair] + W[:, :, a, e] * X[:, a, e]
                s1[:, :, pair] = s1[:, :, pair] + W[:, :, b, e] * X[:, b, e]
            if bool(tail.any()):
                a = v[tail]
                s0[:, :, tail] = s0[:, :, tail] + W[:, :, a, e] * X[:, a, e]
        done |= leave
        i += 1
    t = s0 + s1
    for o in (16, 8, 4, 2, 1):
        t = t + t[:, :, lanes ^ o]
    acc = t[:, :, 0]
    tot = torch.zeros(N)
    for q in range(ksplit):
        tot = tot + acc[:, q]
        if q == twice:
            tot = tot + acc[:, q]
    return tot


def _mma_chain(prods, d=None):
    """prods fp32 [..., 64]: one 64-k block as 4 mma.sync steps (step j: k = 16 c + 4 j + e), each adding its 16
    products to the running fp32 fragment d"""
    st = prods.view(*prods.shape[:-1], 4, 4, 4).sum(dim=(-3, -1), dtype=F32)  # [..., j]
    d = torch.zeros(prods.shape[:-1]) if d is None else d
    for j in range(4):
        d = d + st[..., j]
    return d


def _fma(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def w4_deq_codes(packed, N, K):
    return ref_w4_unpack(packed, N, K).float()


def emu_w4(q, s, z, x, ksplit):
    """gemv_w4_kernel's row sums for one x row: fp32 [N].  q codes fp32 [N, K], s fp32 [N, G], z fp32 [N, G]:
    per group two chains of 4 mma (its two 64-k blocks), d0 + d1, times s into the part's sum; parts in order"""
    N, K = q.shape
    G = K // W4_GROUP
    prods = (q - z.repeat_interleave(W4_GROUP, 1)) * x.float().view(1, K)  # exact: small integers x bf16
    d = prods.view(N, G, 2, 64)
    dd = _mma_chain(d)  # [N, G, 2]
    grp = dd[..., 0] + dd[..., 1]
    cg = G // ksplit
    tot = torch.zeros(N)
    for part in range(ksplit):
        sg = torch.zeros(N)
        for gi in range(part * cg, (part + 1) * cg):
            sg = _fma(s[:, gi], grp[:, gi], sg)
        tot = tot + sg
    return tot


def emu_batch(fmt, wq, s, z, x, plan, *, drop_short=False, row_from_next=None):
    """gemv_batch_kernel's fp32 sums before the epilogue, [M, N].  w4: wq codes [N, K], s / z [N, G]; e4m3: wq the
    code values [N, K] (the row scale is the epilogue's).  Per rank (slice u0, nu) and per part: w4 adds each
    group's s * (d0 + d1) to the slice's running sum; e4m3 runs two chains of mma over the part's even / odd
    64-k blocks (lanes past the part's end feed zeros) and adds d0 + d1 per part; the ranks' sums are then added
    in rank order.  drop_short: the last unit of the first shorter slice is skipped; row_from_next: output row m
    uses x row m + 1 (a column-tile index fault)."""
    M, K = x.shape
    xf = x.float()
    if row_from_next is not None:
        xf = xf.clone()
        xf[row_from_next] = xf[row_from_next + 1]
    N = wq.shape[0]
    unit = plan["unit"]
    short = min(nu for _, nu in plan["slices"])
    dropped = False
    ranks = []
    for (u0, nu), parts in zip(plan["slices"], plan["kparts"]):
        run = torch.zeros(M, N)
        for pu0, pu in parts:
            if pu == 0:
                continue
            units = range(u0 + pu0, u0 + pu0 + pu)
            if drop_short and not dropped and nu == short and nu < plan["max_units"] and pu0 + pu == nu:
                units, dropped = units[:-1], True
            if fmt == "w4a16":
                for u in units:
                    k = slice(u * 128, (u + 1) * 128)
                    prods = (wq[None, :, k] - z[None, :, u, None]) * xf[:, None, k]
                    dd = _mma_chain(prods.view(M, N, 2, 64))
                    run = _fma(s[None, :, u], dd[..., 0] + dd[..., 1], run)
            else:
                k0, kq = units.start * unit, len(units) * unit
                dh = [torch.zeros(M, N), torch.zeros(M, N)]
                for kb in range(0, kq, 128):
                    for h in range(2):
                        kk = kb + 64 * h
                        if kk >= kq:
                            continue
                        blk = torch.zeros(M, N, 64)
                        n = min(64, kq - kk)  # a part ends on a 16-k boundary: lanes c past it read zeros
                        blk[..., :n] = wq[None, :, k0 + kk:k0 + kk + n] * xf[:, None, k0 + kk:k0 + kk + n]
                        dh[h] = _mma_chain(blk, dh[h])
                run = run + (dh[0] + dh[1])
        ranks.append(run)
    if len(ranks) == 1:
        return ranks[0]
    tot = torch.zeros(M, N)
    for r in ranks:
        tot = tot + r
    return tot


def epilogue(v, *, sc=None, bias=None, residual=None, swiglu=False, round_fn=rb, residual_twice=False,
             swap_pair=None):
    """gemv_epilogue / batch_finish in fp32: row scale, bias, bf16, residual (or SwiGLU); -> bf16 values [M, n_out]"""
    if sc is not None:
        v = v * sc
    if bias is not None:
        v = v + bias.float()
    if swiglu:
        g, u = v[:, 0::2].clone(), v[:, 1::2].clone()
        if swap_pair is not None:
            g[:, swap_pair], u[:, swap_pair] = v[:, 2 * swap_pair + 1], v[:, 2 * swap_pair]
        g, u = rb(g), rb(u)
        return round_fn(rb(g / (1.0 + torch.exp(-g))) * u)
    if residual is None:
        return round_fn(v)
    v = rb(v)
    v = rb(v + residual.float()) if residual_twice else v
    return round_fn(v + residual.float())


def check(got, P, A, E, depth, *, bias=None, residual=None, swiglu=False, norm=False):
    return GemvErrors().add_gemv(got, P, A, E, depth=depth, bias=bias, residual=residual, swiglu=swiglu, norm=norm)


# ------------------------------------------------------------------------------------------------
# emulation cases: a slice of rows of the production shape, with that shape's plan
# ------------------------------------------------------------------------------------------------
N_PROD = {512: 1024, 3584: 4608, 18944: 3584}   # the production N whose plan each K runs under (tiny / 8B)
ROWS = 256                                      # rows emulated (single stream)
BATCH_ROWS = 32                                 # rows emulated (batched), M = 16
SS_FUSIONS = ("bias+norm", "residual", "swiglu+norm", "argmax+norm")
BATCH_FUSIONS = ("bias", "residual", "swiglu", "none")


class _Problem:
    def __init__(self, fmt, K, rows, M, seed):
        self.fmt, self.K = fmt, K
        w = _weights(rows, K, seed, edges=fmt == "w4a16")
        g = torch.Generator().manual_seed(seed + 1)
        self.bias = torch.randn(rows, generator=g).to(torch.bfloat16)
        self.nw = (1 + 0.1 * torch.randn(K, generator=g)).to(torch.bfloat16)
        self.x = _x(M, K, seed + 2, outliers=M > 1)
        self.res = (torch.randn(M, rows, generator=g) * (_row_scale(M)[:, None] if M > 1 else 1.0)).to(torch.bfloat16)
        if fmt == "bf16":
            self.wf, self.sc = w.float(), None
            self.w64 = w.double()
        elif fmt == "fp8":
            codes, self.sc = ref_quantize_e4m3_rows(w)
            self.wf = e4m3_values()[codes.long()].float()
            self.w64 = self.wf.double() * self.sc.double()[:, None]
        else:
            self.q, self.s, self.z = ref_quantize_w4(w)
            self.packed, self.zf, self.sc = ref_w4_pack(self.q), self.z.float(), None
            self.w64 = ((self.q.double() - self.zf.double().repeat_interleave(128, 1))
                        * self.s.double().repeat_interleave(128, 1))

    def reference(self, norm, x=None):
        x = self.x if x is None else x
        return gemv_reference(gemv_xn(x, self.nw if norm else None), self.w64, self.w64.shape[0])

    def check(self, got, fusion, depth, P, A, E):
        return check(got, P, A, E, depth, bias=self.bias if fusion.startswith("bias") else None,
                     residual=self.res[:got.shape[0]] if fusion.startswith("residual") else None,
                     swiglu=fusion.startswith("swiglu"), norm="norm" in fusion)

    def finish(self, acc, fusion, **kw):
        return epilogue(acc, sc=self.sc, bias=self.bias if fusion.startswith("bias") else None,
                        residual=self.res[:acc.shape[0]] if fusion.startswith("residual") else None,
                        swiglu=fusion.startswith("swiglu"), **kw)


def single_plan(fmt, K, swiglu=False, norm=True):
    N = N_PROD[K]
    if fmt == "w4a16":
        p = gemv_w4_plan(N, K, norm, SMS_H100)
        return p, gemv_depth("w4", K, p)
    p = gemv_tma_plan(N, K, fmt == "fp8", swiglu, norm, SMS_H100)
    return p, gemv_depth("tma-fp8" if fmt == "fp8" else "tma-bf16", K, p)


def emu_single(prob, plan, x, **faults):
    if prob.fmt == "w4a16":
        q = w4_deq_codes(faults.get("packed", prob.packed), prob.q.shape[0], prob.K)
        return emu_w4(q, faults.get("s", prob.s), faults.get("z", prob.zf), x[0], plan["ksplit"])[None]
    return emu_tma(prob.wf, x[0], plan["ksplit"], 16 if prob.fmt == "fp8" else 8, faults.get("twice"))[None]


SINGLE_EMU = [(fmt, K) for fmt in ("bf16", "fp8", "w4a16") for K in (512, 3584, 18944)]


@pytest.mark.parametrize("fmt,K", SINGLE_EMU, ids=[f"{f}-K{K}" for f, K in SINGLE_EMU])
def test_single_stream_emulation_passes(fmt, K):
    prob = _Problem(fmt, K, ROWS, 1, seed=K + len(fmt))
    plan, depth = single_plan(fmt, K)
    worst = {}
    for norm in (False, True):
        x = prologue(prob.x, prob.nw) if norm else prob.x
        acc = emu_single(prob, plan, x)
        P, A, E = prob.reference(norm)
        for fusion in SS_FUSIONS:
            if ("norm" in fusion) != norm:
                continue
            e = prob.check(prob.finish(acc, fusion), fusion, depth, P, A, E)
            assert not e.failures(), (fusion, e.failures(), e.summary())
            assert e.excess < 0.75 and abs(e.bias) < 0.05, (fusion, e.summary())
            worst[fusion] = e.summary()
    print(fmt, K, plan, worst)


BATCH_EMU = [(fmt, K) for fmt in ("fp8", "w4a16") for K in (512, 3584, 18944)]


@pytest.mark.parametrize("fmt,K", BATCH_EMU, ids=[f"{f}-K{K}" for f, K in BATCH_EMU])
def test_batched_emulation_passes(fmt, K):
    prob = _Problem(fmt, K, BATCH_ROWS, 16, seed=K + 7)
    plan = batch_partition(N_PROD[K], K, fmt == "fp8", SMS_H100)
    depth = gemv_depth("batch-fp8" if fmt == "fp8" else "batch-w4", K, plan)
    acc = emu_batch(fmt, prob.wf if fmt == "fp8" else prob.q.float(), prob.s if fmt == "w4a16" else None,
                    prob.zf if fmt == "w4a16" else None, prob.x, plan)
    P, A, E = prob.reference(False)
    for fusion in BATCH_FUSIONS:
        e = prob.check(prob.finish(acc, fusion), fusion, depth, P, A, E)
        assert not e.failures(), (fusion, e.failures(), e.summary())
        assert e.excess < 0.75 and abs(e.bias) < 0.05, (fusion, e.summary())
    print(fmt, K, {k: plan[k] for k in ("cluster", "parts", "max_units")}, e.summary())


# ------------------------------------------------------------------------------------------------
# planted faults: each must be rejected by the named check
# ------------------------------------------------------------------------------------------------
def _rejected(e, check_name):
    return any(f.startswith(check_name) for f in e.failures())


def _w4_fault_rate(fault, fusion):
    """W4A16 at K = 18944 (8B down_proj's plan): a fault in one (row, group) of every row, each row checked on its
    own element; -> (checker rejects, fraction of the faulted elements over their allowance)"""
    K = 18944
    prob = _Problem("w4a16", K, ROWS, 1, seed=99)
    plan, depth = single_plan("w4a16", K, norm=False)
    g = torch.Generator().manual_seed(5)
    grp = torch.randint(1, K // 128 - 1, (ROWS,), generator=g)
    s, z = prob.s.clone(), prob.zf.clone()
    rows = torch.arange(ROWS)
    if fault == "zero":
        z[rows, grp] = torch.where(z[rows, grp] < 15, z[rows, grp] + 1, z[rows, grp] - 1)
    else:
        s[rows, grp] = s[rows, grp + 1]
    acc = emu_single(prob, plan, prob.x, s=s, z=z)
    P, A, E = prob.reference(False)
    got = prob.finish(acc, fusion)
    e = prob.check(got, fusion, depth, P, A, E)
    res = prob.res if fusion == "residual" else None
    allow = GemvErrors.allowance(P, A, E, depth=depth, residual=res is not None)
    from tests.helpers import _rb64, bf16_ulp, linear_reference
    ref = _rb64(linear_reference(P, residual=res))
    over = (got.double() - ref).abs() > GemvErrors.A_ULP * bf16_ulp(ref) + allow
    return e, float(over.float().mean())


# A wrong zero point or scale moves its output by s * sum of the group's x (times 1 or the scale's change): for
# about a quarter of the groups that sum is small enough that the output moves by less than one ulp, which no
# bound on a bf16 output can see.  Measured: 73 % of the faulted elements are rejected with a plain epilogue,
# 57 % (zero point) and 62 % (scale) when a residual of the output's size is added.
@pytest.mark.parametrize("fusion,rate_min", [("argmax", 0.65), ("residual", 0.5)])
def test_fault_w4_zero_point_off_by_one(fusion, rate_min):
    e, rate = _w4_fault_rate("zero", fusion)
    print("zero point off by one:", fusion, "faulted elements rejected", rate)
    assert _rejected(e, "element") and rate >= rate_min


@pytest.mark.parametrize("fusion,rate_min", [("argmax", 0.65), ("residual", 0.5)])
def test_fault_w4_neighbour_group_scale(fusion, rate_min):
    e, rate = _w4_fault_rate("scale", fusion)
    print("neighbouring group's scale:", fusion, "faulted elements rejected", rate)
    assert _rejected(e, "element") and rate >= rate_min


def test_fault_w4_rows_swapped_in_one_word():
    K = 3584
    prob = _Problem("w4a16", K, ROWS, 1, seed=11)
    plan, depth = single_plan("w4a16", K, norm=False)
    P, A, E = prob.reference(False)
    bad = prob.packed.clone()
    off = 4 * 512 + 6 * 16  # tile 3, 64-k block 4, lane 6 (g = 1, c = 2: rows 49 and 57), u32 0: k 288 .. 291
    word = bad[3, off:off + 4].clone()
    bad[3, off:off + 4] = (word >> 4) | ((word & 15) << 4)  # nibbles 2i and 2i + 1 of a byte: rows g and g + 8
    assert int((ref_w4_unpack(bad, ROWS, K) != prob.q).sum()) == 8
    got = prob.finish(emu_single(prob, plan, prob.x, packed=bad), "bias")
    e = prob.check(got, "bias", depth, P, A, E)
    assert _rejected(e, "element"), e.summary()


def test_fault_tma_kpart_twice():
    K = 3584
    prob = _Problem("bf16", K, ROWS, 1, seed=12)
    plan, depth = single_plan("bf16", K, norm=False)
    assert plan["ksplit"] > 1
    P, A, E = prob.reference(False)
    got = prob.finish(emu_single(prob, plan, prob.x, twice=plan["ksplit"] - 1), "bias")
    e = prob.check(got, "bias", depth, P, A, E)
    assert _rejected(e, "element"), e.summary()


def test_fault_batch_short_slice_unit_dropped():
    K = 18944
    prob = _Problem("w4a16", K, BATCH_ROWS, 16, seed=13)
    plan = batch_partition(3584, K, False, SMS_H100)
    assert len({nu for _, nu in plan["slices"]}) == 2  # slices of 18 and 19 groups
    depth = gemv_depth("batch-w4", K, plan)
    acc = emu_batch("w4a16", prob.q.float(), prob.s, prob.zf, prob.x, plan, drop_short=True)
    P, A, E = prob.reference(False)
    e = prob.check(prob.finish(acc, "residual"), "residual", depth, P, A, E)
    assert _rejected(e, "element"), e.summary()


def test_fault_batch_e4m3_neighbour_row_scale():
    K = 3584
    prob = _Problem("fp8", K, BATCH_ROWS, 16, seed=14)
    plan = batch_partition(4608, K, True, SMS_H100)
    depth = gemv_depth("batch-fp8", K, plan)
    acc = emu_batch("fp8", prob.wf, None, None, prob.x, plan)
    P, A, E = prob.reference(False)
    sc = prob.sc.clone()
    sc[21] = prob.sc[22]  # rows 21, 22: one tile
    got = epilogue(acc, sc=sc, bias=prob.bias)
    e = prob.check(got, "bias", depth, P, A, E)
    assert _rejected(e, "element"), e.summary()


def test_fault_batch_ntile2_row_from_next():
    K = 3584
    prob = _Problem("w4a16", K, BATCH_ROWS, 16, seed=15)
    plan = batch_partition(4608, K, False, SMS_H100)
    depth = gemv_depth("batch-w4", K, plan)
    acc = emu_batch("w4a16", prob.q.float(), prob.s, prob.zf, prob.x, plan, row_from_next=12)
    P, A, E = prob.reference(False)
    e = prob.check(prob.finish(acc, "bias"), "bias", depth, P, A, E)
    assert _rejected(e, "element") and _rejected(e, "row"), e.summary()


def test_fault_swiglu_gate_up_swapped():
    K = 3584
    prob = _Problem("fp8", K, ROWS, 1, seed=16)
    plan, depth = single_plan("fp8", K, swiglu=True)
    x = prologue(prob.x, prob.nw)
    P, A, E = prob.reference(True)
    got = prob.finish(emu_single(prob, plan, x), "swiglu+norm", swap_pair=37)
    e = prob.check(got, "swiglu+norm", depth, P, A, E)
    assert _rejected(e, "element"), e.summary()


def test_fault_residual_added_twice():
    K = 18944
    prob = _Problem("fp8", K, ROWS, 1, seed=17)
    plan, depth = single_plan("fp8", K, norm=False)
    P, A, E = prob.reference(False)
    got = prob.finish(emu_single(prob, plan, prob.x), "residual", residual_twice=True)
    e = prob.check(got, "residual", depth, P, A, E)
    assert _rejected(e, "element"), e.summary()


def test_fault_round_toward_zero():
    K = 3584
    prob = _Problem("bf16", K, ROWS, 1, seed=18)
    plan, depth = single_plan("bf16", K, norm=False)
    P, A, E = prob.reference(False)
    got = prob.finish(emu_single(prob, plan, prob.x), "bias", round_fn=rtz)
    e = prob.check(got, "bias", depth, P, A, E)
    assert _rejected(e, "rounding bias"), e.summary()


def test_fault_norm_weight_one_vector_off():
    K = 3584
    prob = _Problem("w4a16", K, ROWS, 1, seed=19)
    plan, depth = single_plan("w4a16", K)
    P, A, E = prob.reference(True)
    got = prob.finish(emu_single(prob, plan, prologue(prob.x, prob.nw, shift=8)), "bias+norm")
    e = prob.check(got, "bias+norm", depth, P, A, E)
    assert _rejected(e, "element"), e.summary()


# ------------------------------------------------------------------------------------------------
# the launch-plan mirrors
# ------------------------------------------------------------------------------------------------
def test_batch_partition_by_hand():
    """worked through from batch_partition's rules with 132 SMs and sms / cluster resident clusters"""
    p = batch_partition(3584, 18944, False, 132)  # 8B down_proj, W4A16: 148 groups
    # x slice per cluster size: 16 rows x (148 / cl groups x 256 B + 16): cl = 8 is the first under 100 KB with
    # 14 tiles x 1 KB of partial sums (224 tiles over 16 clusters)
    assert (p["cluster"], p["tiles_per_cluster"], p["ctas"], p["max_units"]) == (8, 14, 128, 19)
    assert [nu for _, nu in p["slices"]] == [18, 19] * 4
    assert p["parts"] == 5 and p["stages"] == 3  # 3 or 4 parts leave < 3 stages of 7 / 5 KB slots
    assert [pu for _, pu in p["kparts"][0]] == [3, 4, 3, 4, 4] and [pu for _, pu in p["kparts"][1]] == [3, 4, 4, 4, 4]
    p = batch_partition(2048, 11008, False, 132)  # Lite down_proj, W4A16: 86 groups
    assert (p["cluster"], p["tiles_per_cluster"], p["ctas"], p["max_units"], p["parts"]) == (4, 4, 128, 22, 5)
    assert [nu for _, nu in p["slices"]] == [21, 22, 21, 22]
    p = batch_partition(4608, 3584, True, 132)  # 8B qkv, e4m3: 224 units of 16 k
    assert (p["cluster"], p["max_units"]) == (2, 112) and p["tiles_per_cluster"] == 5  # 288 tiles / 66
    p = batch_partition(1024, 512, True, 132)  # tiny qkv, e4m3: 32 units, x of 1 KB per row
    assert p["cluster"] == 1 and p["tiles_per_cluster"] == 1 and p["ctas"] == 64
    # fewer resident clusters than SMs / cluster: more tiles per cluster
    assert batch_partition(3584, 18944, False, 132, lambda cl: 12)["tiles_per_cluster"] == 19


def test_tma_and_w4_plans_by_hand():
    p = gemv_tma_plan(3584, 18944, False, False, False, 132)  # 8B down_proj, bf16: 28 rows per block
    assert (p["rows_per_block"], p["grid"], p["ksplit"], p["chunk_elems"]) == (28, 128, 8, 2368)
    p = gemv_tma_plan(37888, 3584, True, True, True, 132)  # 8B gate_up, e4m3: 288 rows (even)
    assert p["rows_per_block"] == 288 and p["ksplit"] == 1 and p["stages"] == 7  # 3,584-byte chunks
    p = gemv_w4_plan(3584, 18944, False, 132)  # 224 tiles: 2 per block, 148 groups in 37 parts of 4
    assert (p["tiles_per_block"], p["grid"], p["ksplit"], p["chunk_groups"]) == (2, 112, 37, 4)


def test_partitions_of_the_gpu_table():
    """every batched shape of the GPU table: no slice and no k-part is empty; the table reaches clusters of 1, 2,
    4 and 8, slices of different sizes and k-parts of different sizes"""
    clusters, uneven_slices, uneven_parts = set(), False, False
    for row in BATCH_TABLE:
        p = batch_partition(row["N"], row["K"], row["fmt"] == "fp8", SMS_H100)
        assert p is not None, row
        assert all(nu >= 1 for _, nu in p["slices"]), (row, p["slices"])
        assert all(pu >= 1 for parts in p["kparts"] for _, pu in parts), (row, p["kparts"])
        clusters.add(p["cluster"])
        uneven_slices |= len({nu for _, nu in p["slices"]}) > 1
        uneven_parts |= any(len({pu for _, pu in parts}) > 1 for parts in p["kparts"])
    assert clusters == {1, 2, 4, 8} and uneven_slices and uneven_parts, clusters
    for row in SINGLE_TABLE:
        if row["fmt"] == "w4a16":
            assert gemv_w4_plan(row["N"], row["K"], "norm" in row["fusion"], SMS_H100) is not None, row
        elif row["fmt"] == "fp8":
            assert gemv_tma_plan(row["N"], row["K"], True, "swiglu" in row["fusion"], "norm" in row["fusion"],
                                 SMS_H100) is not None, row
