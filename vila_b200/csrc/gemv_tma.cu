// Weight-streaming GEMV with TMA bulk copies into per-warp shared-memory rings (sm_90a).
//
//   y = W x  (M == 1 decode):  every byte of W is read exactly once from HBM, so the kernel is a pure
//   bandwidth problem.  Instead of register-staged LDG (in-flight bytes limited by registers) each of
//   the 8 consumer warps owns a ring of kStages shared-memory slots that its lane 0 keeps filled with
//   cp.async.bulk (1-D TMA) copies of (row, k-part) chunks; completion is signalled on per-slot
//   mbarriers.  ~100-190 KB of weight data are in flight per SM with zero address arithmetic on the
//   load path, and — because the weights are parameters — the first kStages chunks are issued BEFORE
//   the programmatic-dependent-launch wait, overlapping the predecessor kernel's tail and this
//   kernel's own RMSNorm prologue.
//
//   Fusions: RMSNorm(x) prologue, bias, residual, SwiGLU (interleaved gate/up rows), greedy argmax.
//   Partial sums of the k-parts of a row are parked in slots and added in a fixed order.
//
//   FP8 form (gemv_tma_fp8): W is e4m3 [N, K] with one fp32 scale per row.  The row sum is
//   acc_n = sum_k float(q[n,k]) * float(x[k]) in fp32 (cvt.rn.f16x2.e4m3x2 is exact: every e4m3 value
//   is an f16 value), the k-parts are added in the same fixed order, and v = acc_n * w_scale[n] enters
//   the bf16 kernel's epilogue unchanged.  Half the bytes per row: the ring holds twice the stages.
//
//   W4A16 form (gemv_tma_w4a16, gemv_w4_kernel below): 4-bit codes with a bf16 scale and a uint8 zero
//   point per group of 128 k; its own main loop runs mma.sync on 16-row tiles, the prologue and the
//   epilogue are those of the bf16 form.
//
// Replaces cuBLAS GEMV behind nn.Linear + ATen RMSNorm / SiLU / mul / add / argmax at decode time
// (modeling_qwen2.py:81-95,164-176,223-226; HF lm_head + greedy argmax).
#include "common.cuh"
#include "kernels.h"

namespace vb {
namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
// ring slots per warp: 6 for bf16 weights; 12 for e4m3, whose chunks of the same rows are half as long
template <bool kFp8>
constexpr int max_stages() { return kFp8 ? 12 : 6; }


__device__ __forceinline__ float dot8(const uint4& w, const uint4& x, float acc) {
  acc = fmaf(bf_lo(w.x), bf_lo(x.x), acc);
  acc = fmaf(bf_hi(w.x), bf_hi(x.x), acc);
  acc = fmaf(bf_lo(w.y), bf_lo(x.y), acc);
  acc = fmaf(bf_hi(w.y), bf_hi(x.y), acc);
  acc = fmaf(bf_lo(w.z), bf_lo(x.z), acc);
  acc = fmaf(bf_hi(w.z), bf_hi(x.z), acc);
  acc = fmaf(bf_lo(w.w), bf_lo(x.w), acc);
  acc = fmaf(bf_hi(w.w), bf_hi(x.w), acc);
  return acc;
}

// two e4m3 (low byte = lower k) -> two floats, exactly
__device__ __forceinline__ float2 e4m3x2_to_float2(uint32_t v) {
  uint32_t h;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h) : "h"(static_cast<uint16_t>(v)));
  __half2 hh;
  memcpy(&hh, &h, sizeof(h));
  return __half22float2(hh);
}

// 16 e4m3 weights against 16 bf16 activations (xa: k 0..7, xb: k 8..15)
__device__ __forceinline__ float dot16_e4m3(const uint4& w, const uint4& xa, const uint4& xb, float acc) {
  const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
  const uint32_t xs[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 a = e4m3x2_to_float2(ws[i]), b = e4m3x2_to_float2(ws[i] >> 16);
    acc = fmaf(a.x, bf_lo(xs[2 * i]), acc);
    acc = fmaf(a.y, bf_hi(xs[2 * i]), acc);
    acc = fmaf(b.x, bf_lo(xs[2 * i + 1]), acc);
    acc = fmaf(b.y, bf_hi(xs[2 * i + 1]), acc);
  }
  return acc;
}

// one 16-byte weight vector v of a chunk against the matching activations xv (of that chunk)
template <bool kFp8>
__device__ __forceinline__ float dot_vec(const uint4& w, const uint4* xv, int v, float acc) {
  if constexpr (kFp8) return dot16_e4m3(w, xv[2 * v], xv[2 * v + 1], acc);
  else return dot8(w, xv[v], acc);
}

__device__ __forceinline__ uint32_t float_order(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// 1-D bulk copy global -> shared, completion on an mbarrier (complete_tx::bytes)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

struct TmaGemvLayout {
  int chunk_elems;   // K / ksplit
  int stages;
  int x_off, nw_off, acc_off, sc_off, ring_off, bar_off, total;  // sc: row scales (fp8 only)
};

// Fused RMSNorm prologue, in place on x in shared memory (every thread of the block takes part):
// x <- bf16(bf16(x * rstd) * norm_w), the norm weight arriving on nw_bar.
__device__ __forceinline__ void rmsnorm_x_in_smem(const GemvParams& p, uint4* xs, const uint4* nws, int nvec,
                                                  float* red, uint64_t* nw_bar) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float s = 0.f;
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
    const uint4 v = xs[i];
    float t;
    t = bf_lo(v.x); s += t * t;
    t = bf_hi(v.x); s += t * t;
    t = bf_lo(v.y); s += t * t;
    t = bf_hi(v.y); s += t * t;
    t = bf_lo(v.z); s += t * t;
    t = bf_hi(v.z); s += t * t;
    t = bf_lo(v.w); s += t * t;
    t = bf_hi(v.w); s += t * t;
  }
  s = warp_sum(s);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  float t = lane < kWarps ? red[lane] : 0.f;
  t = warp_sum(t);
  const float rstd = rsqrtf(t / p.K + p.norm_eps);
  mbar_wait(nw_bar, 0);
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) {  // each thread rewrites only its own slots
    const uint4 v = xs[i], g = nws[i];
    uint4 o;
    o.x = pack_bf16(bf16_round(bf_lo(v.x) * rstd) * bf_lo(g.x), bf16_round(bf_hi(v.x) * rstd) * bf_hi(g.x));
    o.y = pack_bf16(bf16_round(bf_lo(v.y) * rstd) * bf_lo(g.y), bf16_round(bf_hi(v.y) * rstd) * bf_hi(g.y));
    o.z = pack_bf16(bf16_round(bf_lo(v.z) * rstd) * bf_lo(g.z), bf16_round(bf_hi(v.z) * rstd) * bf_hi(g.z));
    o.w = pack_bf16(bf16_round(bf_lo(v.w) * rstd) * bf_lo(g.w), bf16_round(bf_hi(v.w) * rstd) * bf_hi(g.w));
    xs[i] = o;
  }
}

// Fixed-order reduction of the k-parts, in place: acc[i] <- sum_q acc[i*ksplit + q].  Rows are processed
// in phases of blockDim.x; writing row i only overwrites slots of rows <= i, which have been read in this
// or an earlier phase.
__device__ __forceinline__ void reduce_kparts(float* acc, int nrows, int ksplit) {
  if (ksplit > 1) {
    for (int base = 0; base < nrows; base += blockDim.x) {
      const int i = base + threadIdx.x;
      float tot = 0.f;
      if (i < nrows)
        for (int q = 0; q < ksplit; ++q) tot += acc[i * ksplit + q];
      __syncthreads();
      if (i < nrows) acc[i] = tot;
      __syncthreads();
    }
  }
}

// Epilogue on the row sums acc[0, nrows) (times the row scales sc with kScaled): bias, residual, SwiGLU
// (interleaved gate / up rows), greedy argmax.
template <bool kScaled>
__device__ __forceinline__ void gemv_epilogue(const GemvParams& p, const float* acc, const float* sc, int row0,
                                              int nrows, unsigned long long* best_s) {
  const int lane = threadIdx.x & 31;
  if (p.flags & 1) {
    for (int j = threadIdx.x; j < (nrows >> 1); j += blockDim.x) {
      float g = acc[2 * j], u = acc[2 * j + 1];
      if constexpr (kScaled) {
        g *= sc[2 * j];
        u *= sc[2 * j + 1];
      }
      if (p.bias) {
        g += __bfloat162float(p.bias[row0 + 2 * j]);
        u += __bfloat162float(p.bias[row0 + 2 * j + 1]);
      }
      g = bf16_round(g);
      u = bf16_round(u);
      p.y[(row0 >> 1) + j] = __float2bfloat16(bf16_round(silu_f(g)) * u);
    }
    return;
  }
  unsigned long long best = 0ull;
  for (int r = threadIdx.x; r < nrows; r += blockDim.x) {
    float v = acc[r];
    if constexpr (kScaled) v *= sc[r];
    if (p.bias) v += __bfloat162float(p.bias[row0 + r]);
    v = bf16_round(v);
    if (p.residual) v = bf16_round(v + __bfloat162float(p.residual[row0 + r]));
    if (p.y) p.y[row0 + r] = __float2bfloat16(v);
    if (p.argmax_key) {
      const unsigned long long key =
          (static_cast<unsigned long long>(float_order(v)) << 32) |
          static_cast<unsigned long long>(0xffffffffu - static_cast<uint32_t>(row0 + r));
      best = key > best ? key : best;
    }
  }
  if (p.argmax_key) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
      best = other > best ? other : best;
    }
    if (lane == 0) atomicMax(best_s, best);
    __syncthreads();
    if (threadIdx.x == 0) atomicMax(p.argmax_key, *best_s);
  }
}

template <bool kFp8>
__global__ void __launch_bounds__(kThreads, 1)
gemv_tma_kernel(GemvParams p, int rows_per_block, int ksplit, TmaGemvLayout L) {
  constexpr int kMaxStages = max_stages<kFp8>();
  constexpr int kElemBytes = kFp8 ? 1 : 2;
  extern __shared__ __align__(128) uint8_t smem[];
  uint4* xs = reinterpret_cast<uint4*>(smem + L.x_off);
  float* acc = reinterpret_cast<float*>(smem + L.acc_off);
  float* sc = reinterpret_cast<float*>(smem + L.sc_off);
  uint8_t* ring = smem + L.ring_off;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.bar_off);
  __shared__ float red[32];
  __shared__ unsigned long long best_s;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row0 = blockIdx.x * rows_per_block;
  const int nrows = min(rows_per_block, p.N - row0);
  if (nrows <= 0) return;
  const int nvec = p.K >> 3;
  const int chunk_bytes = L.chunk_elems * kElemBytes;
  const int chunk_vecs = chunk_bytes >> 4;  // 16-byte weight vectors per chunk
  const int items = nrows * ksplit;
  const int n_my = items > warp ? (items - warp + kWarps - 1) / kWarps : 0;
  uint8_t* my_ring = ring + static_cast<size_t>(warp) * L.stages * chunk_bytes;
  uint64_t* my_bars = bars + warp * kMaxStages;

  uint64_t* x_bar = bars + kWarps * kMaxStages;  // [0]: x arrived, [1]: norm weight arrived
  if (lane == 0) {
    for (int s = 0; s < L.stages; ++s) mbar_init(&my_bars[s], 1);
    if (warp == 0) {
      mbar_init(&x_bar[0], 1);
      mbar_init(&x_bar[1], 1);
    }
    fence_barrier_init();
  }
  __syncwarp();
  griddep_launch_dependents();

  auto issue = [&](int j) {  // lane 0 only: copy item j of this warp into slot j % stages
    const int item = warp + j * kWarps;
    const int r = item / ksplit, part = item - r * ksplit;
    const uint8_t* src = reinterpret_cast<const uint8_t*>(p.w) +
                         (static_cast<size_t>(row0 + r) * p.K + part * L.chunk_elems) * kElemBytes;
    const int s = j % L.stages;
    mbar_arrive_expect_tx(&my_bars[s], chunk_bytes);
    bulk_g2s(my_ring + static_cast<size_t>(s) * chunk_bytes, src, chunk_bytes, &my_bars[s]);
  };

  const bool early = (p.flags & 2) != 0;  // static weights: stream before the dependency wait
  const uint32_t x_bytes = static_cast<uint32_t>(p.K) * 2;
  uint4* nws = reinterpret_cast<uint4*>(smem + L.nw_off);
  int issued = 0;
  if (early && lane == 0) {
    for (; issued < L.stages && issued < n_my; ++issued) issue(issued);
    if (warp == 0 && p.norm_w != nullptr) {  // the norm weight is a parameter as well
      mbar_arrive_expect_tx(&x_bar[1], x_bytes);
      bulk_g2s(nws, p.norm_w, x_bytes, &x_bar[1]);
    }
  }
  if constexpr (kFp8) {  // row scales are parameters too (plain loads: a row block need not be 16-byte aligned)
    if (early)
      for (int i = threadIdx.x; i < nrows; i += kThreads) sc[i] = p.w_scale[row0 + i];
  }
  griddep_wait();
  if constexpr (kFp8) {
    if (!early)
      for (int i = threadIdx.x; i < nrows; i += kThreads) sc[i] = p.w_scale[row0 + i];
  }
  // ---- prologue: x arrives as ONE bulk copy (a register-staged loop of dependent LDG -> STS round
  // trips per slice would stall the full weight rings, and with them the HBM stream) ----
  if (lane == 0) {
    if (warp == 0) {
      mbar_arrive_expect_tx(&x_bar[0], x_bytes);
      bulk_g2s(xs, p.x, x_bytes, &x_bar[0]);
      if (!early && p.norm_w != nullptr) {
        mbar_arrive_expect_tx(&x_bar[1], x_bytes);
        bulk_g2s(nws, p.norm_w, x_bytes, &x_bar[1]);
      }
    }
    if (!early)
      for (; issued < L.stages && issued < n_my; ++issued) issue(issued);
  }
  if (threadIdx.x == 0) best_s = 0ull;
  __syncthreads();  // barrier initialisation by warp 0 is visible to every warp
  mbar_wait(&x_bar[0], 0);
  if (p.norm_w != nullptr) rmsnorm_x_in_smem(p, xs, nws, nvec, red, &x_bar[1]);
  __syncthreads();

  // ---- main loop: consume this warp's ring ----
  for (int j = 0; j < n_my; ++j) {
    const int s = j % L.stages;
    const int item = warp + j * kWarps;
    const int r = item / ksplit, part = item - r * ksplit;
    mbar_wait(&my_bars[s], (j / L.stages) & 1);
    const uint4* wv = reinterpret_cast<const uint4*>(my_ring + static_cast<size_t>(s) * chunk_bytes);
    const uint4* xv = xs + part * (L.chunk_elems >> 3);
    float s0 = 0.f, s1 = 0.f;
    int v = lane;
    for (; v + 32 < chunk_vecs; v += 64) {
      const uint4 a = wv[v], b = wv[v + 32];
      s0 = dot_vec<kFp8>(a, xv, v, s0);
      s1 = dot_vec<kFp8>(b, xv, v + 32, s1);
    }
    if (v < chunk_vecs) s0 = dot_vec<kFp8>(wv[v], xv, v, s0);
    const float tot = warp_sum(s0 + s1);
    __syncwarp();  // every lane is done reading slot s
    if (lane == 0) {
      acc[item] = tot;  // slot = row * ksplit + part
      if (j + L.stages < n_my) issue(j + L.stages);
    }
  }
  __syncthreads();
  reduce_kparts(acc, nrows, ksplit);
  gemv_epilogue<kFp8>(p, acc, sc, row0, nrows, &best_s);
}

template <bool kFp8>
int gemv_tma_launch(const GemvParams& p, cudaStream_t stream) {
  constexpr int kMaxStages = max_stages<kFp8>();
  constexpr int kElemBytes = kFp8 ? 1 : 2;
  constexpr int kElemAlign = 16 / kElemBytes;  // chunk elements per 16-byte weight vector
  const int sms = num_sms();
  int rows_per_block = (p.N + sms - 1) / sms;
  if ((p.flags & 1) && (rows_per_block & 1)) rows_per_block += 1;
  const int grid = (p.N + rows_per_block - 1) / rows_per_block;
  // Shared-memory budget: (almost) the whole SM (227 KB per block on H100).  Under a saturated HBM
  // pipe the load latency is a few microseconds, so ~100+ KB must be in flight per SM to sustain the
  // full rate; the rings are not halved to let the next kernel's CTA co-reside.
  constexpr int kSmemBudget = 220 * 1024;
  // x and the norm weight arrive by bulk copy: 16-byte aligned sources (else: register-staged kernel)
  if ((reinterpret_cast<uintptr_t>(p.x) & 15) || (p.norm_w && (reinterpret_cast<uintptr_t>(p.norm_w) & 15)))
    return -1;
  const int x1_bytes = (p.K * 2 + 127) / 128 * 128;
  const int x_bytes = x1_bytes * (p.norm_w ? 2 : 1);  // x (+ norm weight staging)
  const int sc_bytes = kFp8 ? rows_per_block * 4 : 0;  // row scales
  TmaGemvLayout L;
  int ksplit = -1;
  for (int ks = 1; ks <= 128; ++ks) {
    if (p.K % ks) continue;
    const int ce = p.K / ks;
    if (ce % kElemAlign) continue;
    const int cb = ce * kElemBytes;
    if (cb > 8192) continue;
    if (cb < 512) break;
    const int acc_bytes = (rows_per_block * ks * 4 + sc_bytes + 127) / 128 * 128;
    const int ring_budget = kSmemBudget - x_bytes - acc_bytes - (kWarps * kMaxStages + 2) * 8 - 256;
    int st = ring_budget / (kWarps * cb);
    if (st > kMaxStages) st = kMaxStages;
    if (st < 3) continue;  // need a few chunks in flight per warp
    ksplit = ks;
    L.stages = st;
    if (static_cast<long>(rows_per_block) * ks >= 6L * kWarps) break;  // enough items per warp
  }
  if (ksplit < 0) return -1;
  L.chunk_elems = p.K / ksplit;
  const int chunk_bytes = L.chunk_elems * kElemBytes;
  L.x_off = 0;
  L.nw_off = x1_bytes;
  L.acc_off = x_bytes;
  L.sc_off = L.acc_off + rows_per_block * ksplit * 4;
  L.ring_off = (L.sc_off + sc_bytes + 127) / 128 * 128;
  {
    // recompute stages for the final ksplit (the loop may have broken on an earlier candidate)
    const int ring_budget = kSmemBudget - L.ring_off - (kWarps * kMaxStages + 2) * 8 - 256;
    int st = ring_budget / (kWarps * chunk_bytes);
    if (st > kMaxStages) st = kMaxStages;
    if (st < 2) return -1;
    L.stages = st;
  }
  L.bar_off = (L.ring_off + kWarps * L.stages * chunk_bytes + 127) / 128 * 128;
  L.total = L.bar_off + (kWarps * kMaxStages + 2) * 8;
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    VB_CUDA(cudaFuncSetAttribute(gemv_tma_kernel<kFp8>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 224 * 1024));
  }
  VB_CUDA(launch_pdl(gemv_tma_kernel<kFp8>, dim3(grid), dim3(kThreads), static_cast<size_t>(L.total), stream,
                     p, rows_per_block, ksplit, L));
  return 0;
}

// ---------------------------------------------------------------------------------------------------
// W4A16 form (gemv_tma_w4a16): 4-bit codes q in groups of 128 consecutive k of a row, each group with a
// bf16 scale s and a uint8 zero point z, w = (q - z) * s.  The products run on the tensor cores:
// mma.sync m16n8k16 (bf16 in, fp32 accumulate) with a 16-row weight tile as A and x as B, broadcast to
// all 8 columns (so every column of D holds the same row sums).  Dequantisation to the A fragment is
// exact and cheap: 0x4300 | q is the bf16 value 128 + q, and subtracting the bf16 128 + z leaves q - z.
// Each group's 8 mma steps accumulate into a fresh fragment, which is scaled by s in fp32 and added to
// the row sum; the k-parts of a row are then added in a fixed order, as in the bf16 and fp8 forms.
//
// Packed code layout (written by quantize_w4_groups, vila_b200/model/qwen2.py): rows in tiles of 16
// (N padded with zero codes), each tile's K/2 * 16 bytes contiguous, as [K/64][32 lanes][4 u32].  In the
// 64-k block at k = b, lane (g = lane / 4, c = lane % 4) owns u32 j (mma step j) holding rows g and g + 8
// at k0 = b + 16c + 4j .. k0 + 3, nibble i + 4m of it in bf16x2 register i, half m:
//   nibble 0 / 4: row g, k0 / k0+1      nibble 1 / 5: row g+8, k0 / k0+1
//   nibble 2 / 6: row g, k0+2 / k0+3    nibble 3 / 7: row g+8, k0+2 / k0+3
// which is the A fragment of m16n8k16 with mma k index (2c, 2c+1, 2c+8, 2c+9) mapped to k0 + (0, 1, 2, 3);
// x's B fragment under the same mapping is x[k0 .. k0+3], so a lane reads its x as two plain 16-byte words
// per 64-k block.
constexpr int kW4TileRows = 16;
constexpr int kW4Group = 128;
constexpr int kW4GroupBytes = kW4TileRows * kW4Group / 2;  // one group of one tile: 1 KB
constexpr int kW4MaxStages = 12;

__device__ __forceinline__ void mma_bf16_m16n8k16(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2,
                                                  uint32_t a3, uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// bf16x2 {128 + nibble i, 128 + nibble i + 4} of w, minus the bf16x2 {128 + z, 128 + z}: exactly q - z
__device__ __forceinline__ uint32_t w4_pair(uint32_t w, int i, uint32_t zz) {
  uint32_t v;  // (w >> 4i) & 0x000f000f | 0x43004300 as one LOP3 (the compiler splits the C form in two)
  asm("lop3.b32 %0, %1, %2, %3, 0xea;" : "=r"(v) : "r"(w >> (4 * i)), "n"(0x000f000f), "n"(0x43004300));
  __nv_bfloat162 a, b;
  memcpy(&a, &v, 4);
  memcpy(&b, &zz, 4);
  const __nv_bfloat162 d = __hsub2(a, b);
  uint32_t r;
  memcpy(&r, &d, 4);
  return r;
}

// one 64-k block: 4 mma steps on the weight word wq (u32 j = step j) and this lane's x words xa, xb
__device__ __forceinline__ void w4_block(float (&d)[4], const uint4& wq, const uint4& xa, const uint4& xb,
                                         uint32_t zg, uint32_t zg8) {
  const uint32_t ws[4] = {wq.x, wq.y, wq.z, wq.w};
  const uint32_t xw[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
#pragma unroll
  for (int j = 0; j < 4; ++j)
    mma_bf16_m16n8k16(d, w4_pair(ws[j], 0, zg), w4_pair(ws[j], 1, zg8), w4_pair(ws[j], 2, zg),
                      w4_pair(ws[j], 3, zg8), xw[2 * j], xw[2 * j + 1]);
}

struct W4GemvLayout {
  int chunk_groups;  // groups per (tile, k-part) item: G / ksplit
  int stages;
  int x_off, nw_off, acc_off, gs_off, gz_off, ring_off, bar_off, total;  // gs / gz: group scales / zeros
};

__global__ void __launch_bounds__(kThreads, 1)
gemv_w4_kernel(GemvParams p, const __nv_bfloat16* __restrict__ w_gscale, const uint8_t* __restrict__ w_zero,
               int rows_per_block, int ksplit, W4GemvLayout L) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint4* xs = reinterpret_cast<uint4*>(smem + L.x_off);
  float* acc = reinterpret_cast<float*>(smem + L.acc_off);
  __nv_bfloat16* gs = reinterpret_cast<__nv_bfloat16*>(smem + L.gs_off);  // [rows_per_block][G]
  uint8_t* gz = smem + L.gz_off;                                           // [rows_per_block][G]
  uint8_t* ring = smem + L.ring_off;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.bar_off);
  __shared__ float red[32];
  __shared__ unsigned long long best_s;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row0 = blockIdx.x * rows_per_block;
  const int nrows = min(rows_per_block, p.N - row0);
  if (nrows <= 0) return;
  const int ntiles = (nrows + kW4TileRows - 1) / kW4TileRows;
  const int G = p.K / kW4Group;
  const int nvec = p.K >> 3;
  const int chunk_bytes = L.chunk_groups * kW4GroupBytes;
  const int items = ntiles * ksplit;
  const int n_my = items > warp ? (items - warp + kWarps - 1) / kWarps : 0;
  uint8_t* my_ring = ring + static_cast<size_t>(warp) * L.stages * chunk_bytes;
  uint64_t* my_bars = bars + warp * kW4MaxStages;

  uint64_t* x_bar = bars + kWarps * kW4MaxStages;  // [0]: x arrived, [1]: norm weight arrived
  if (lane == 0) {
    for (int s = 0; s < L.stages; ++s) mbar_init(&my_bars[s], 1);
    if (warp == 0) {
      mbar_init(&x_bar[0], 1);
      mbar_init(&x_bar[1], 1);
    }
    fence_barrier_init();
  }
  __syncwarp();
  griddep_launch_dependents();

  const size_t tile_bytes = static_cast<size_t>(p.K) * (kW4TileRows / 2);
  auto issue = [&](int j) {  // lane 0 only: copy item j of this warp into slot j % stages
    const int item = warp + j * kWarps;
    const int t = item / ksplit, part = item - t * ksplit;
    const uint8_t* src = reinterpret_cast<const uint8_t*>(p.w) +
                         static_cast<size_t>(row0 / kW4TileRows + t) * tile_bytes +
                         static_cast<size_t>(part) * chunk_bytes;
    const int s = j % L.stages;
    mbar_arrive_expect_tx(&my_bars[s], chunk_bytes);
    bulk_g2s(my_ring + static_cast<size_t>(s) * chunk_bytes, src, chunk_bytes, &my_bars[s]);
  };
  // group parameters of the block's rows (rows past N of the last tile: s = 0, z = 0)
  auto load_params = [&]() {
    for (int i = threadIdx.x; i < ntiles * kW4TileRows * G; i += kThreads) {
      const bool in = i < nrows * G;
      gs[i] = in ? w_gscale[static_cast<size_t>(row0) * G + i] : __float2bfloat16(0.f);
      gz[i] = in ? w_zero[static_cast<size_t>(row0) * G + i] : 0;
    }
  };

  const bool early = (p.flags & 2) != 0;  // static weights: stream before the dependency wait
  const uint32_t x_bytes = static_cast<uint32_t>(p.K) * 2;
  uint4* nws = reinterpret_cast<uint4*>(smem + L.nw_off);
  int issued = 0;
  if (early && lane == 0) {
    for (; issued < L.stages && issued < n_my; ++issued) issue(issued);
    if (warp == 0 && p.norm_w != nullptr) {
      mbar_arrive_expect_tx(&x_bar[1], x_bytes);
      bulk_g2s(nws, p.norm_w, x_bytes, &x_bar[1]);
    }
  }
  if (early) load_params();  // parameters too
  griddep_wait();
  if (!early) load_params();
  if (lane == 0) {
    if (warp == 0) {
      mbar_arrive_expect_tx(&x_bar[0], x_bytes);
      bulk_g2s(xs, p.x, x_bytes, &x_bar[0]);
      if (!early && p.norm_w != nullptr) {
        mbar_arrive_expect_tx(&x_bar[1], x_bytes);
        bulk_g2s(nws, p.norm_w, x_bytes, &x_bar[1]);
      }
    }
    if (!early)
      for (; issued < L.stages && issued < n_my; ++issued) issue(issued);
  }
  if (threadIdx.x == 0) best_s = 0ull;
  __syncthreads();  // barrier initialisation and the group parameters are visible to every warp
  mbar_wait(&x_bar[0], 0);
  if (p.norm_w != nullptr) rmsnorm_x_in_smem(p, xs, nws, nvec, red, &x_bar[1]);
  __syncthreads();

  // ---- main loop: consume this warp's ring; item = (16-row tile, k-part of chunk_groups groups) ----
  const int g = lane >> 2, c = lane & 3;
  for (int j = 0; j < n_my; ++j) {
    const int s = j % L.stages;
    const int item = warp + j * kWarps;
    const int t = item / ksplit, part = item - t * ksplit;
    mbar_wait(&my_bars[s], (j / L.stages) & 1);
    const uint4* wv = reinterpret_cast<const uint4*>(my_ring + static_cast<size_t>(s) * chunk_bytes) + lane;
    const int grp0 = part * L.chunk_groups;
    const int pr = (t * kW4TileRows + g) * G + grp0;  // parameters of row g; row g + 8 at pr + 8 * G
    const uint4* xv = xs + grp0 * (kW4Group / 8) + 2 * c;
    float sum_g = 0.f, sum_g8 = 0.f;
    for (int q = 0; q < L.chunk_groups; ++q) {
      const uint32_t zg = (0x4300u | gz[pr + q]) * 0x10001u;
      const uint32_t zg8 = (0x4300u | gz[pr + 8 * G + q]) * 0x10001u;
      float d0[4] = {0.f, 0.f, 0.f, 0.f}, d1[4] = {0.f, 0.f, 0.f, 0.f};  // two chains of 4 dependent mma
      w4_block(d0, wv[64 * q], xv[16 * q], xv[16 * q + 1], zg, zg8);
      w4_block(d1, wv[64 * q + 32], xv[16 * q + 8], xv[16 * q + 9], zg, zg8);
      sum_g = fmaf(__bfloat162float(gs[pr + q]), d0[0] + d1[0], sum_g);
      sum_g8 = fmaf(__bfloat162float(gs[pr + 8 * G + q]), d0[2] + d1[2], sum_g8);
    }
    __syncwarp();  // every lane is done reading slot s
    if (c == 0) {  // lanes 4g .. 4g+3 hold the same sums (the 8 columns of D are equal)
      acc[(t * kW4TileRows + g) * ksplit + part] = sum_g;  // slot = row * ksplit + part
      acc[(t * kW4TileRows + g + 8) * ksplit + part] = sum_g8;
    }
    if (lane == 0 && j + L.stages < n_my) issue(j + L.stages);
  }
  __syncthreads();
  reduce_kparts(acc, nrows, ksplit);
  gemv_epilogue<false>(p, acc, nullptr, row0, nrows, &best_s);
}

int gemv_w4_launch(const GemvParams& p, const __nv_bfloat16* w_gscale, const uint8_t* w_zero, cudaStream_t stream) {
  const int sms = num_sms();
  const int tiles = (p.N + kW4TileRows - 1) / kW4TileRows;
  const int tiles_per_block = (tiles + sms - 1) / sms;
  const int rows_per_block = tiles_per_block * kW4TileRows;  // even: a SwiGLU pair never straddles blocks
  const int grid = (tiles + tiles_per_block - 1) / tiles_per_block;
  const int G = p.K / kW4Group;
  constexpr int kSmemBudget = 220 * 1024;
  const int x1_bytes = (p.K * 2 + 127) / 128 * 128;
  const int x_bytes = x1_bytes * (p.norm_w ? 2 : 1);
  const int gp_bytes = (rows_per_block * G * 3 + 127) / 128 * 128;  // bf16 scales + uint8 zeros
  const int bar_bytes = (kWarps * kW4MaxStages + 2) * 8;
  // k-parts: whole groups per item; the largest chunk (<= 8 KB) with >= 3 stages per warp, unless the
  // block then has fewer than 6 items per warp (a block's rows are few: split K further)
  W4GemvLayout L;
  int ksplit = -1;
  for (int ks = 1; ks <= G; ++ks) {
    if (G % ks) continue;
    const int cb = G / ks * kW4GroupBytes;
    if (cb > 8192) continue;
    const int acc_bytes = (rows_per_block * ks * 4 + 127) / 128 * 128;
    const int st = (kSmemBudget - x_bytes - acc_bytes - gp_bytes - bar_bytes - 256) / (kWarps * cb);
    if (st < 3) continue;
    ksplit = ks;
    if (static_cast<long>(tiles_per_block) * ks >= 6L * kWarps) break;
  }
  if (ksplit < 0) return -1;
  L.chunk_groups = G / ksplit;
  const int chunk_bytes = L.chunk_groups * kW4GroupBytes;
  L.x_off = 0;
  L.nw_off = x1_bytes;
  L.acc_off = x_bytes;
  L.gs_off = L.acc_off + (rows_per_block * ksplit * 4 + 127) / 128 * 128;
  L.gz_off = L.gs_off + rows_per_block * G * 2;
  L.ring_off = L.gs_off + gp_bytes;
  L.stages = std::min(kW4MaxStages, (kSmemBudget - L.ring_off - bar_bytes - 256) / (kWarps * chunk_bytes));
  L.bar_off = (L.ring_off + kWarps * L.stages * chunk_bytes + 127) / 128 * 128;
  L.total = L.bar_off + bar_bytes;
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    VB_CUDA(cudaFuncSetAttribute(gemv_w4_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
  }
  VB_CUDA(launch_pdl(gemv_w4_kernel, dim3(grid), dim3(kThreads), static_cast<size_t>(L.total), stream, p,
                     w_gscale, w_zero, rows_per_block, ksplit, L));
  return 0;
}

// ---------------------------------------------------------------------------------------------------
// Batched form (gemv_batch_kernel): y[m, :] = epilogue(W x[m, :]) for M <= 16 activation rows, on the
// quantized copies of the W4A16 and FP8 forms, unchanged.  The mma.sync m16n8k16 of the W4A16 form takes
// x as its B operand; here column g of B column tile t is x row 8t + g, so one A fragment serves 8 (kNT =
// 1) or 16 (kNT = 2) rows of x and every weight byte is still read once per launch.
//   * w4a16: A fragments from w4_pair as in gemv_w4_kernel; each group's fp32 fragment is scaled by s.
//   * e4m3: an item is a 16-row tile x k-part copied as 16 row segments; in the ring the rows are
//     padded to a pitch of 64 mod 128 bytes, so lanes g = 0, 1 of a quarter-warp read different banks.
//     Lane (g, c) reads 16 contiguous bytes of rows g and g + 8 at k0 = b + 16c of the 64-k block b, the
//     W4 layout's k order, so the x words are those of the W4 path.  e4m3 -> f16 -> f32 -> bf16 is exact.
//     The row scale, staged in shared memory with the weights' parameters, multiplies the finished row sum.
// K is cut into `cluster` slices (whole units: groups of 128 k, or 16 k for e4m3) streamed by the CTAs of
// one thread-block cluster, which share a row block: each rank stages only its slice of the x rows.  The
// ranks' fp32 partial sums are added through DSMEM in rank order, each rank finishing a share of the rows.
// The partition (cluster size, row blocks, k-parts) follows from (N, K, format) and the device only, and
// every sum runs in a fixed order: an output row depends on its own x row alone, for any M.
constexpr int kBatchMaxStages = 12;
constexpr int kBatchMaxRows = 16;
constexpr int kBatchSmemBudget = 220 * 1024;
constexpr int kBatchXBudget = 100 * 1024;     // x slice + cluster partial sums, per CTA
constexpr int kBatchXBudgetOne = 120 * 1024;  // x of a cluster of one (no partial sums)

struct BatchLayout {
  int cluster;            // CTAs per cluster, each streaming one k-slice of the cluster's row block
  int tiles_per_cluster;  // 16-row tiles per row block
  int unit;               // k per slice unit: 128 (one w4 group) or 16 (e4m3)
  int units;              // K / unit
  int max_units;          // units of the largest slice
  int parts;              // k-parts per slice: items per tile
  int slot_bytes;         // ring slot (one item)
  int row_pitch;          // e4m3: bytes per weight row in a slot
  int x_pitch;            // bytes per x row in shared memory
  int stages;
  int x_off, part_off, gs_off, gz_off, ring_off, bar_off, total;  // gs: w4 group scales or e4m3 row scales
};

// two e4m3 (low byte = lower k) -> bf16x2, exactly
__device__ __forceinline__ uint32_t e4m3x2_to_bf16x2(uint32_t v) {
  const float2 f = e4m3x2_to_float2(v);
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(f.y), "f"(f.x));
  return r;
}

__device__ __forceinline__ float ld_dsmem_f32(uint32_t cluster_addr) {
  float v;
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(cluster_addr));
  return v;
}

// epilogue of one output element (row n, x row m), with the rounding points of gemv_epilogue; sc: the row
// scales of the row block staged in shared memory, row n at sc[n - row0]
template <bool kFp8>
__device__ __forceinline__ void batch_finish(const GemvBatchArgs& p, const float* sc, int row0, int n, int m,
                                             float v) {
  if constexpr (kFp8) v *= sc[n - row0];
  if (p.bias) v += __bfloat162float(p.bias[n]);
  v = bf16_round(v);
  if (p.residual) v = bf16_round(v + __bfloat162float(p.residual[m * p.ld_res + n]));
  p.y[m * p.ldy + n] = __float2bfloat16(v);
}
template <bool kFp8>
__device__ __forceinline__ void batch_finish_swiglu(const GemvBatchArgs& p, const float* sc, int row0, int n,
                                                    int m, float g, float u) {  // n even: gate n, up n + 1
  if constexpr (kFp8) {
    g *= sc[n - row0];
    u *= sc[n + 1 - row0];
  }
  if (p.bias) {
    g += __bfloat162float(p.bias[n]);
    u += __bfloat162float(p.bias[n + 1]);
  }
  g = bf16_round(g);
  u = bf16_round(u);
  p.y[m * p.ldy + (n >> 1)] = __float2bfloat16(bf16_round(silu_f(g)) * u);
}

template <bool kFp8, int kNT>
__global__ void __launch_bounds__(kThreads, 1)
gemv_batch_kernel(GemvBatchArgs p, const void* __restrict__ w_scale, const uint8_t* __restrict__ w_zero,
                  BatchLayout L) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* xs = smem + L.x_off;                                             // [16][x_pitch]
  float* part = reinterpret_cast<float*>(smem + L.part_off);                // [tiles * 16][16] (cluster > 1)
  __nv_bfloat16* gs = reinterpret_cast<__nv_bfloat16*>(smem + L.gs_off);  // w4: [tiles * 16][max_units]
  float* sc = reinterpret_cast<float*>(smem + L.gs_off);                    // e4m3: [tiles * 16] row scales
  uint8_t* gz = smem + L.gz_off;
  uint8_t* ring = smem + L.ring_off;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.bar_off);
  const float* row_scale = static_cast<const float*>(w_scale);
  const __nv_bfloat16* gscale = static_cast<const __nv_bfloat16*>(w_scale);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rank = L.cluster > 1 ? static_cast<int>(cluster_ctarank()) : 0;
  const int tile0 = static_cast<int>(blockIdx.x) / L.cluster * L.tiles_per_cluster;
  const int ntiles = min(L.tiles_per_cluster, (p.N + 15) / 16 - tile0);  // the same on every rank
  const int u0 = rank * L.units / L.cluster, nu = (rank + 1) * L.units / L.cluster - u0;  // this slice
  const int k0 = u0 * L.unit;
  const int my_tiles = ntiles > warp ? (ntiles - warp + kWarps - 1) / kWarps : 0;
  const int n_my = my_tiles * L.parts;  // items (tile, part), the parts of a tile consecutive
  uint8_t* my_ring = ring + static_cast<size_t>(warp) * L.stages * L.slot_bytes;
  uint64_t* my_bars = bars + warp * kBatchMaxStages;
  uint64_t* x_bar = bars + kWarps * kBatchMaxStages;

  if (lane == 0) {
    for (int s = 0; s < L.stages; ++s) mbar_init(&my_bars[s], 1);
    if (warp == 0) mbar_init(x_bar, 1);
    fence_barrier_init();
  }
  __syncwarp();
  griddep_launch_dependents();

  auto part_range = [&](int q, int& pu0) {  // units [pu0, pu0 + return) of the slice
    pu0 = q * nu / L.parts;
    return (q + 1) * nu / L.parts - pu0;
  };
  auto issue = [&](int j) {  // whole warp: copy item j of this warp into slot j % stages
    const int t = tile0 + warp + (j / L.parts) * kWarps;
    int pu0;
    const int pu = part_range(j % L.parts, pu0);
    const int s = j % L.stages;
    uint8_t* dst = my_ring + static_cast<size_t>(s) * L.slot_bytes;
    if constexpr (kFp8) {
      const int rows = min(kW4TileRows, p.N - t * kW4TileRows), bytes = pu * L.unit;
      if (lane == 0) mbar_arrive_expect_tx(&my_bars[s], rows * bytes);
      __syncwarp();
      if (lane < rows)
        bulk_g2s(dst + lane * L.row_pitch,
                 static_cast<const uint8_t*>(p.w) + static_cast<size_t>(t * kW4TileRows + lane) * p.K + k0 +
                     pu0 * L.unit,
                 bytes, &my_bars[s]);
    } else {
      if (lane == 0) {
        const uint8_t* src = static_cast<const uint8_t*>(p.w) +
                             static_cast<size_t>(t) * p.K * (kW4TileRows / 2) +
                             static_cast<size_t>(u0 + pu0) * kW4GroupBytes;
        mbar_arrive_expect_tx(&my_bars[s], pu * kW4GroupBytes);
        bulk_g2s(dst, src, pu * kW4GroupBytes, &my_bars[s]);
      }
    }
  };
  auto load_params = [&]() {  // e4m3: row scales of the row block; w4: group scales / zeros of the slice
    if constexpr (kFp8) {       // (rows past N: s = 0, z = 0)
      for (int r = threadIdx.x; r < ntiles * kW4TileRows; r += kThreads) {
        const int n = tile0 * kW4TileRows + r;
        sc[r] = n < p.N ? row_scale[n] : 0.f;
      }
      return;
    }
    const int G = p.K / kW4Group;
    for (int i = threadIdx.x; i < ntiles * kW4TileRows * nu; i += kThreads) {
      const int r = i / nu, q = i - r * nu, n = tile0 * kW4TileRows + r;
      const bool in = n < p.N;
      gs[r * L.max_units + q] = in ? gscale[static_cast<size_t>(n) * G + u0 + q] : __float2bfloat16(0.f);
      gz[r * L.max_units + q] = in ? w_zero[static_cast<size_t>(n) * G + u0 + q] : 0;
    }
  };

  const bool early = (p.flags & 2) != 0;  // static weights: stream before the dependency wait
  int issued = 0;
  if (early) {
    for (; issued < L.stages && issued < n_my; ++issued) issue(issued);
    load_params();  // parameters too
  }
  griddep_wait();
  if (!early) {
    for (; issued < L.stages && issued < n_my; ++issued) issue(issued);
    load_params();
  }
  // x rows of the slice: one bulk copy per row < M, rows M .. 8 kNT - 1 zero
  const uint32_t x_bytes = static_cast<uint32_t>(nu * L.unit) * 2;
  if (warp == 0) {
    if (lane == 0) mbar_arrive_expect_tx(x_bar, p.M * x_bytes);
    __syncwarp();
    if (lane < p.M) bulk_g2s(xs + lane * L.x_pitch, p.x + lane * p.ldx + k0, x_bytes, x_bar);
  }
  for (int i = threadIdx.x; i < (8 * kNT - p.M) * (L.x_pitch >> 4); i += kThreads)
    reinterpret_cast<uint4*>(xs + p.M * L.x_pitch)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();  // barrier initialisation, group parameters and zero rows are visible to every warp
  mbar_wait(x_bar, 0);

  // ---- main loop; lane (g, c) sums rows g, g + 8 of its tile for x rows 8t + 2c, 8t + 2c + 1 ----
  const int g = lane >> 2, c = lane & 3;
  const uint8_t* xl = xs + g * L.x_pitch + 32 * c;  // + 8 x_pitch per column tile
  float run[kNT][2][2];
#pragma unroll
  for (int t = 0; t < kNT; ++t) run[t][0][0] = run[t][0][1] = run[t][1][0] = run[t][1][1] = 0.f;
  for (int j = 0; j < n_my; ++j) {
    const int s = j % L.stages, q = j % L.parts;
    const int tl = warp + (j / L.parts) * kWarps;  // tile of the row block
    int pu0;
    const int pu = part_range(q, pu0);
    mbar_wait(&my_bars[s], (j / L.stages) & 1);
    const uint8_t* slot = my_ring + static_cast<size_t>(s) * L.slot_bytes;
    if constexpr (kFp8) {
      float d[2][kNT][4];  // two chains: even and odd 64-k blocks
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int t = 0; t < kNT; ++t) d[h][t][0] = d[h][t][1] = d[h][t][2] = d[h][t][3] = 0.f;
      const int kq = pu * L.unit;
      const uint8_t* xq = xl + pu0 * L.unit * 2;
      for (int kb = 0; kb < kq; kb += 128) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int k = kb + 64 * h;
          const bool in = k + 16 * c < kq;  // a part ends on a 16-k boundary
          const uint4 z4 = make_uint4(0, 0, 0, 0);
          const uint4 wa = in ? *reinterpret_cast<const uint4*>(slot + g * L.row_pitch + k + 16 * c) : z4;
          const uint4 wb = in ? *reinterpret_cast<const uint4*>(slot + (g + 8) * L.row_pitch + k + 16 * c) : z4;
          uint32_t xw[kNT][8];
#pragma unroll
          for (int t = 0; t < kNT; ++t) {
            const uint8_t* xp = xq + t * 8 * L.x_pitch + 2 * k;
            const uint4 xa = in ? *reinterpret_cast<const uint4*>(xp) : z4;
            const uint4 xb = in ? *reinterpret_cast<const uint4*>(xp + 16) : z4;
            xw[t][0] = xa.x; xw[t][1] = xa.y; xw[t][2] = xa.z; xw[t][3] = xa.w;
            xw[t][4] = xb.x; xw[t][5] = xb.y; xw[t][6] = xb.z; xw[t][7] = xb.w;
          }
          const uint32_t ra[4] = {wa.x, wa.y, wa.z, wa.w}, rb[4] = {wb.x, wb.y, wb.z, wb.w};
#pragma unroll
          for (int s4 = 0; s4 < 4; ++s4) {
            const uint32_t a0 = e4m3x2_to_bf16x2(ra[s4]), a1 = e4m3x2_to_bf16x2(rb[s4]);
            const uint32_t a2 = e4m3x2_to_bf16x2(ra[s4] >> 16), a3 = e4m3x2_to_bf16x2(rb[s4] >> 16);
#pragma unroll
            for (int t = 0; t < kNT; ++t)
              mma_bf16_m16n8k16(d[h][t], a0, a1, a2, a3, xw[t][2 * s4], xw[t][2 * s4 + 1]);
          }
        }
      }
#pragma unroll
      for (int t = 0; t < kNT; ++t) {
        run[t][0][0] += d[0][t][0] + d[1][t][0];
        run[t][0][1] += d[0][t][1] + d[1][t][1];
        run[t][1][0] += d[0][t][2] + d[1][t][2];
        run[t][1][1] += d[0][t][3] + d[1][t][3];
      }
    } else {
      const uint4* wv = reinterpret_cast<const uint4*>(slot) + lane;
      const int pr = (tl * kW4TileRows + g) * L.max_units + pu0;  // row g; row g + 8 at + 8 max_units
      const uint8_t* xq = xl + pu0 * kW4Group * 2;
      for (int gq = 0; gq < pu; ++gq) {
        const uint32_t zg = (0x4300u | gz[pr + gq]) * 0x10001u;
        const uint32_t zg8 = (0x4300u | gz[pr + 8 * L.max_units + gq]) * 0x10001u;
        const float sg = __bfloat162float(gs[pr + gq]), sg8 = __bfloat162float(gs[pr + 8 * L.max_units + gq]);
        float d[2][kNT][4];  // two chains of 4 dependent mma per column tile: the two 64-k blocks
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint4 wq = wv[64 * gq + 32 * h];
          uint32_t xw[kNT][8];
#pragma unroll
          for (int t = 0; t < kNT; ++t) {
            const uint8_t* xp = xq + t * 8 * L.x_pitch + gq * kW4Group * 2 + 128 * h;
            const uint4 xa = *reinterpret_cast<const uint4*>(xp), xb = *reinterpret_cast<const uint4*>(xp + 16);
            xw[t][0] = xa.x; xw[t][1] = xa.y; xw[t][2] = xa.z; xw[t][3] = xa.w;
            xw[t][4] = xb.x; xw[t][5] = xb.y; xw[t][6] = xb.z; xw[t][7] = xb.w;
            d[h][t][0] = d[h][t][1] = d[h][t][2] = d[h][t][3] = 0.f;
          }
          const uint32_t ws[4] = {wq.x, wq.y, wq.z, wq.w};
#pragma unroll
          for (int s4 = 0; s4 < 4; ++s4) {
            const uint32_t a0 = w4_pair(ws[s4], 0, zg), a1 = w4_pair(ws[s4], 1, zg8);
            const uint32_t a2 = w4_pair(ws[s4], 2, zg), a3 = w4_pair(ws[s4], 3, zg8);
#pragma unroll
            for (int t = 0; t < kNT; ++t)
              mma_bf16_m16n8k16(d[h][t], a0, a1, a2, a3, xw[t][2 * s4], xw[t][2 * s4 + 1]);
          }
        }
#pragma unroll
        for (int t = 0; t < kNT; ++t) {
          run[t][0][0] = fmaf(sg, d[0][t][0] + d[1][t][0], run[t][0][0]);
          run[t][0][1] = fmaf(sg, d[0][t][1] + d[1][t][1], run[t][0][1]);
          run[t][1][0] = fmaf(sg8, d[0][t][2] + d[1][t][2], run[t][1][0]);
          run[t][1][1] = fmaf(sg8, d[0][t][3] + d[1][t][3], run[t][1][1]);
        }
      }
    }
    __syncwarp();  // every lane is done reading slot s
    if (j + L.stages < n_my) issue(j + L.stages);
    if (q == L.parts - 1) {  // the tile's slice is summed
      const int n0 = (tile0 + tl) * kW4TileRows + g;
#pragma unroll
      for (int t = 0; t < kNT; ++t)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int n = n0 + 8 * h, m = 8 * t + 2 * c + e;
            const float v = run[t][h][e];
            run[t][h][e] = 0.f;
            if (L.cluster > 1) {
              part[((tl * kW4TileRows) + g + 8 * h) * kBatchMaxRows + m] = v;
            } else if (p.flags & 1) {
              const float u = __shfl_down_sync(0xffffffffu, v, 4);  // row n + 1: lane g + 1
              if (!(g & 1) && n < p.N && m < p.M) batch_finish_swiglu<kFp8>(p, sc, tile0 * kW4TileRows, n, m, v, u);
            } else if (n < p.N && m < p.M) {
              batch_finish<kFp8>(p, sc, tile0 * kW4TileRows, n, m, v);
            }
          }
    }
  }
  if (L.cluster > 1) {
    cluster_sync_all();  // every rank's partial sums are written
    const int rows = ntiles * kW4TileRows;
    const int share = ((rows + L.cluster - 1) / L.cluster + 1) & ~1;  // even: SwiGLU pairs stay together
    const int r0 = rank * share, r1 = min(rows, r0 + share);
    const uint32_t part_addr = smem_u32(part);
    const bool swiglu = (p.flags & 1) != 0;
    const int per = swiglu ? 2 : 1;
    for (int i = threadIdx.x; i < (r1 - r0) / per * p.M; i += kThreads) {
      const int r = r0 + i / p.M * per, m = i % p.M, n = tile0 * kW4TileRows + r;
      if (n >= p.N) continue;
      float v = 0.f, u = 0.f;
      for (int k = 0; k < L.cluster; ++k) {  // ranks in order
        const uint32_t a = mapa_u32(part_addr + (r * kBatchMaxRows + m) * 4, k);
        v += ld_dsmem_f32(a);
        if (swiglu) u += ld_dsmem_f32(a + kBatchMaxRows * 4);
      }
      if (swiglu) batch_finish_swiglu<kFp8>(p, sc, tile0 * kW4TileRows, n, m, v, u);
      else batch_finish<kFp8>(p, sc, tile0 * kW4TileRows, n, m, v);
    }
    cluster_sync_all();  // no CTA leaves while its partial sums are read
  }
}

template <bool kFp8, int kNT>
int batch_set_smem_attr() {
  static PerDeviceOnce once;
  if (once.first()) {
    VB_CUDA(cudaFuncSetAttribute(gemv_batch_kernel<kFp8, kNT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 224 * 1024));
  }
  return 0;
}

// clusters of `cluster` CTAs that can be resident at once with one CTA per SM (from the device only)
int batch_max_active_clusters(int cluster) {
  static int cache[64][4] = {};
  int dev = 0;
  VB_CUDA(cudaGetDevice(&dev));
  int ci = cluster == 1 ? 0 : cluster == 2 ? 1 : cluster == 4 ? 2 : 3;
  int& v = cache[dev & 63][ci];
  if (v == 0) {
    if (batch_set_smem_attr<false, 2>() != 0) return -1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(cluster);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = 224 * 1024;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = cluster;
    attr.val.clusterDim.y = attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    int n = 0;
    VB_CUDA(cudaOccupancyMaxActiveClusters(&n, gemv_batch_kernel<false, 2>, &cfg));
    v = n > 0 ? n : -1;
  }
  return v;
}

// The partition of one (N, K, format) on this device: the smallest cluster whose x slice and partial sums
// fit kBatchXBudget (else a cluster of one, if its x fits kBatchXBudgetOne), then the fewest k-parts per
// slice that leave >= 3 ring stages per warp.  -1: no partition fits.
int batch_partition(int N, int K, bool fp8, BatchLayout& L) {
  const int sms = num_sms();
  const int tiles = (N + kW4TileRows - 1) / kW4TileRows;
  L.unit = fp8 ? 16 : kW4Group;
  L.units = K / L.unit;
  auto x_pitch = [&](int cl) { return ((L.units + cl - 1) / cl * L.unit * 2 + 127) / 128 * 128 + 16; };
  auto tpc = [&](int cl) {
    int active = batch_max_active_clusters(cl);
    int n = std::max(1, std::min(sms / cl, active > 0 ? active : sms / cl));
    return (tiles + n - 1) / n;
  };
  L.cluster = 0;
  for (int cl = 1; cl <= 8; cl *= 2) {
    if (L.units < 4 * cl) break;
    const int xb = kBatchMaxRows * x_pitch(cl), pb = cl > 1 ? tpc(cl) * kW4TileRows * kBatchMaxRows * 4 : 0;
    if (xb + pb <= kBatchXBudget) {
      L.cluster = cl;
      break;
    }
  }
  if (L.cluster == 0) {
    if (kBatchMaxRows * x_pitch(1) > kBatchXBudgetOne) return -1;
    L.cluster = 1;
  }
  L.tiles_per_cluster = tpc(L.cluster);
  L.max_units = (L.units + L.cluster - 1) / L.cluster;
  L.x_pitch = x_pitch(L.cluster);
  const int rows = L.tiles_per_cluster * kW4TileRows;
  L.x_off = 0;
  L.part_off = kBatchMaxRows * L.x_pitch;
  L.gs_off = L.part_off + (L.cluster > 1 ? rows * kBatchMaxRows * 4 : 0);
  L.gz_off = L.gs_off + (fp8 ? rows * 4 : rows * L.max_units * 2);  // e4m3 row scales / w4 group scales
  L.ring_off = (L.gz_off + (fp8 ? 0 : rows * L.max_units) + 127) / 128 * 128;
  const int bar_bytes = (kWarps * kBatchMaxStages + 1) * 8;
  const int max_chunk = fp8 ? 32 : 8;  // units per item: <= 512 bytes per e4m3 row, <= 8 w4 groups
  for (L.parts = (L.max_units + max_chunk - 1) / max_chunk; L.parts <= L.max_units; ++L.parts) {
    const int chunk = (L.max_units + L.parts - 1) / L.parts;
    L.row_pitch = fp8 ? (chunk * L.unit + 127) / 128 * 128 + 64 : 0;
    L.slot_bytes = fp8 ? kW4TileRows * L.row_pitch : chunk * kW4GroupBytes;
    L.stages = std::min(kBatchMaxStages, (kBatchSmemBudget - L.ring_off - bar_bytes) / (kWarps * L.slot_bytes));
    if (L.stages >= 3) break;
  }
  if (L.parts > L.max_units || L.stages < 3) return -1;
  L.bar_off = (L.ring_off + kWarps * L.stages * L.slot_bytes + 127) / 128 * 128;
  L.total = L.bar_off + bar_bytes;
  return 0;
}

template <bool kFp8, int kNT>
int gemv_batch_launch(const GemvBatchArgs& p, const void* w_scale, const uint8_t* w_zero, const BatchLayout& L,
                      cudaStream_t stream) {
  if (batch_set_smem_attr<kFp8, kNT>() != 0) return 2;
  const int tiles = (p.N + kW4TileRows - 1) / kW4TileRows;
  const int grid = (tiles + L.tiles_per_cluster - 1) / L.tiles_per_cluster * L.cluster;
  VB_CUDA(launch_pdl_cluster(gemv_batch_kernel<kFp8, kNT>, dim3(grid), dim3(kThreads),
                             static_cast<size_t>(L.total), stream, dim3(L.cluster, 1, 1), p, w_scale, w_zero, L));
  return 0;
}

int gemv_batch(const GemvBatchArgs& p, const void* w_scale, const uint8_t* w_zero, bool fp8, cudaStream_t stream) {
  const char* name = fp8 ? "gemv_batch_fp8" : "gemv_batch_w4a16";
  const int unit = fp8 ? 16 : kW4Group;
  VB_CHECK(p.M >= 1 && p.M <= kBatchMaxRows, "%s: M=%d outside 1..%d", name, p.M, kBatchMaxRows);
  VB_CHECK(p.N > 0 && p.K > 0 && p.K % unit == 0, "%s: bad shape N=%d K=%d (K %% %d == 0)", name, p.N, p.K, unit);
  VB_CHECK(!(p.flags & ~3), "%s: unknown flags 0x%x", name, p.flags);
  VB_CHECK(!(p.flags & 1) || p.N % 2 == 0, "%s: swiglu needs even N", name);
  VB_CHECK(w_scale != nullptr && (fp8 || w_zero != nullptr),
           fp8 ? "%s: w_scale is required" : "%s: group scales and zero points are required", name);
  VB_CHECK(p.x != nullptr && p.w != nullptr && p.y != nullptr, "%s: x, w and y are required", name);
  const int n_out = (p.flags & 1) ? p.N / 2 : p.N;
  VB_CHECK(!(reinterpret_cast<uintptr_t>(p.w) & 15) && !(reinterpret_cast<uintptr_t>(p.x) & 15) &&
               !(reinterpret_cast<uintptr_t>(p.y) & 15) &&
               !(p.residual && (reinterpret_cast<uintptr_t>(p.residual) & 15)),
           "%s: w, x, y and residual must be 16-byte aligned", name);
  VB_CHECK(p.ldx % 8 == 0 && p.ldy % 8 == 0 && (!p.residual || p.ld_res % 8 == 0),
           "%s: row strides must be 16-byte multiples (ldx=%lld ldy=%lld ld_res=%lld)", name,
           static_cast<long long>(p.ldx), static_cast<long long>(p.ldy), static_cast<long long>(p.ld_res));
  VB_CHECK((p.M == 1 || p.ldx >= p.K) && (p.M == 1 || p.ldy >= n_out) && (!p.residual || p.M == 1 || p.ld_res >= p.N),
           "%s: row strides shorter than a row", name);
  BatchLayout L;
  VB_CHECK(batch_partition(p.N, p.K, fp8, L) == 0, "%s: N=%d K=%d does not fit the TMA rings", name, p.N, p.K);
  const int nt = p.M > 8 ? 2 : 1;
  if (fp8) return nt == 1 ? gemv_batch_launch<true, 1>(p, w_scale, w_zero, L, stream)
                          : gemv_batch_launch<true, 2>(p, w_scale, w_zero, L, stream);
  return nt == 1 ? gemv_batch_launch<false, 1>(p, w_scale, w_zero, L, stream)
                 : gemv_batch_launch<false, 2>(p, w_scale, w_zero, L, stream);
}

}  // namespace

// returns 0 on launch, -1 if the shape does not fit this kernel (caller falls back to the LSU kernel)
int gemv_tma_bf16(const GemvParams& p, cudaStream_t stream) { return gemv_tma_launch<false>(p, stream); }

// e4m3 weights: this kernel or an error, never a fallback
int gemv_tma_fp8(const GemvParams& p, cudaStream_t stream) {
  VB_CHECK(p.N > 0 && p.K > 0 && p.K % 16 == 0, "gemv_fp8: bad shape N=%d K=%d (K %% 16 == 0)", p.N, p.K);
  VB_CHECK(!(p.flags & 1) || p.N % 2 == 0, "gemv_fp8: swiglu needs even N");
  VB_CHECK(!(p.flags & 4), "gemv_fp8: there is no register-staged variant for e4m3 weights");
  VB_CHECK(p.w_scale != nullptr, "gemv_fp8: w_scale is required");
  VB_CHECK(!(reinterpret_cast<uintptr_t>(p.w) & 15) && !(reinterpret_cast<uintptr_t>(p.x) & 15) &&
               !(p.norm_w && (reinterpret_cast<uintptr_t>(p.norm_w) & 15)),
           "gemv_fp8: w, x and norm_w must be 16-byte aligned");
  const int rc = gemv_tma_launch<true>(p, stream);
  VB_CHECK(rc >= 0, "gemv_fp8: N=%d K=%d does not fit the TMA ring (K / ksplit >= 512 bytes)", p.N, p.K);
  return rc;
}

// 4-bit weights with group-128 scales and zero points: this kernel or an error, never a fallback
int gemv_tma_w4a16(const GemvParams& p, const __nv_bfloat16* w_gscale, const uint8_t* w_zero, cudaStream_t stream) {
  VB_CHECK(p.N > 0 && p.K > 0 && p.K % kW4Group == 0, "gemv_w4a16: bad shape N=%d K=%d (K %% 128 == 0)", p.N,
           p.K);
  VB_CHECK(!(p.flags & 1) || p.N % 2 == 0, "gemv_w4a16: swiglu needs even N");
  VB_CHECK(!(p.flags & 4), "gemv_w4a16: there is no register-staged variant for 4-bit weights");
  VB_CHECK(w_gscale != nullptr && w_zero != nullptr, "gemv_w4a16: group scales and zero points are required");
  VB_CHECK(!(reinterpret_cast<uintptr_t>(p.w) & 15) && !(reinterpret_cast<uintptr_t>(p.x) & 15) &&
               !(p.norm_w && (reinterpret_cast<uintptr_t>(p.norm_w) & 15)),
           "gemv_w4a16: w, x and norm_w must be 16-byte aligned");
  const int rc = gemv_w4_launch(p, w_gscale, w_zero, stream);
  VB_CHECK(rc >= 0, "gemv_w4a16: N=%d K=%d does not fit the TMA ring", p.N, p.K);
  return rc;
}

// batched forms: this kernel or an error, never a fallback
int gemv_batch_fp8(const GemvBatchArgs& p, const float* w_scale, cudaStream_t stream) {
  return gemv_batch(p, w_scale, nullptr, true, stream);
}
int gemv_batch_w4a16(const GemvBatchArgs& p, const __nv_bfloat16* w_gscale, const uint8_t* w_zero,
                     cudaStream_t stream) {
  return gemv_batch(p, w_gscale, w_zero, false, stream);
}
int gemv_batch_partition(int N, int K, int fp8, int32_t* out) {
  VB_CHECK(out != nullptr && N > 0 && K > 0 && K % (fp8 ? 16 : kW4Group) == 0, "gemv_batch_partition: bad shape");
  BatchLayout L;
  VB_CHECK(batch_partition(N, K, fp8 != 0, L) == 0, "gemv_batch_partition: N=%d K=%d does not fit", N, K);
  const int tiles = (N + kW4TileRows - 1) / kW4TileRows;
  out[0] = L.cluster;
  out[1] = (tiles + L.tiles_per_cluster - 1) / L.tiles_per_cluster * L.cluster;
  out[2] = L.tiles_per_cluster;
  out[3] = L.parts;
  out[4] = batch_max_active_clusters(L.cluster);
  out[5] = L.total;
  return 0;
}

}  // namespace vb
