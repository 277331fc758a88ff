// Temperature / top-k / top-p sampling of the continuous-batching engine (vila_b200/serving.py, sampling=True).
//
// The rule (stated in torch / numpy by vila_b200/sampling.py, which the tests use) for a row of bf16 logits with
// inv_T, top_k, top_p, a 64-bit seed and the token index t of the request:
//   greedy   inv_T == 0 or top_k == 1: the first index of max float(logit) (torch.argmax)
//   scaling  s_i = float(logit_i) * inv_T (fp32; -0 becomes +0)
//   top-k    top_k in (1, V): keep s_i >= s_(k), the k-th largest value (ties kept)
//   top-p    top_p < 1: p_i = exp(s_i - max s), Z = sum of p over the top-k survivors; keep survivor i iff the mass of
//            survivors with a strictly larger s is < top_p * Z (ties at the boundary kept, the largest always kept)
//   draw     argmax over the kept set of s_i + g_i (ties to the lowest index), g_i = -log(-log1p(-u_i)),
//            u_i = (x_i + 0.5) * 2^-32, x_i word i % 4 of Philox-4x32-10 with key (seed lo, seed hi) and counter
//            (i / 4, t lo, t hi, 0)
//
// sample_kernel: one cluster of kSampCluster CTAs per row.  Each CTA keeps its contiguous slice of s in shared
// memory as fp32, so the row is read once.  The k-th largest value and the top-p boundary are found by radix selects
// on the order-preserving 32-bit key of s (digits of 11, 11 and 10 bits); each round's histogram counts keys (top-k)
// or sums the fixed-point masses floor(p_i * 2^40) (top-p) with integer shared-memory atomics, so the kept set does
// not depend on thread order.  Histograms and arg-maxes are merged through DSMEM.  Greedy rows run one max pass,
// "T only" rows one draw pass.  A row's token depends only on its own logits and parameters.
//
// Replaces HF TemperatureLogitsWarper / TopKLogitsWarper / TopPLogitsWarper + torch.multinomial in
// GenerationMixin._sample, reached from llava_arch.py:823-833.
#include <math.h>

#include "common.cuh"
#include "kernels.h"

namespace vb {
namespace {

constexpr int kSampThreads = 256;
constexpr int kSampWarps = kSampThreads / 32;
constexpr int kSampCluster = 8;
constexpr int kSampMaxSlice = 40960;  // fp32 values per CTA: V <= 327,680
constexpr int kHistBins = 2048;       // radix digits: bits [21, 32), [10, 21), [0, 10)
constexpr float kMassScale = 1099511627776.f;  // 2^40: fixed-point unit of the top-p masses

struct SampleArgs {
  const __nv_bfloat16* logits;
  int64_t ld;
  const float* inv_t;
  const int32_t* top_k;
  const float* top_p;
  const int64_t* seed;
  const int64_t* step;
  const int32_t* position;
  int64_t* tokens;
  int32_t* n_kept;
  int V, slice;  // slice: values per CTA, a multiple of 4
};

struct SampleScratch {
  unsigned long long hist[2][kHistBins];  // double-buffered: round r writes hist[r & 1]
  unsigned long long warp_sum[kSampWarps];
  double warp_v[kSampWarps];
  int warp_i[kSampWarps];
  double cta_v[2];  // this CTA's arg-max: [0] max pass, [1] draw pass (each slot written once per launch)
  int cta_i[2];
  unsigned long long cta_n;  // this CTA's kept count
  unsigned long long found_above;
  uint32_t found_bin;
};

__device__ __forceinline__ uint32_t order_key(float s) {
  const uint32_t b = __float_as_uint(s);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

// u = fp32((x + 0.5) * 2^-32) correctly rounded; g = -log(-log1p(-u)) in fp32.  The winners come from small u,
// where u is exact.
__device__ __forceinline__ float gumbel(uint32_t x) {
  const float u = __double2float_rn((static_cast<double>(x) + 0.5) * 2.3283064365386962890625e-10);
  return -logf(-log1pf(-u));
}

__device__ __forceinline__ unsigned long long ld_dsmem_u64(const void* p, uint32_t rank) {
  unsigned long long v;
  asm volatile("ld.shared::cluster.u64 %0, [%1];" : "=l"(v) : "r"(mapa_u32(smem_u32(p), rank)));
  return v;
}
__device__ __forceinline__ double ld_dsmem_f64(const void* p, uint32_t rank) {
  double v;
  asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(mapa_u32(smem_u32(p), rank)));
  return v;
}
__device__ __forceinline__ int ld_dsmem_s32(const void* p, uint32_t rank) {
  int v;
  asm volatile("ld.shared::cluster.s32 %0, [%1];" : "=r"(v) : "r"(mapa_u32(smem_u32(p), rank)));
  return v;
}

__device__ __forceinline__ bool better(double v, int i, double bv, int bi) {
  return v > bv || (v == bv && i < bi);
}

// block arg-max of (v, i) -> sc.cta_v[slot] / sc.cta_i[slot]; then cluster_sync, after which every CTA may read
// every CTA's entry
__device__ void cta_argmax(SampleScratch& sc, double v, int i, int slot) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (better(ov, oi, v, i)) v = ov, i = oi;
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) sc.warp_v[w] = v, sc.warp_i[w] = i;
  __syncthreads();
  if (threadIdx.x == 0) {
    double bv = sc.warp_v[0];
    int bi = sc.warp_i[0];
    for (int k = 1; k < kSampWarps; ++k)
      if (better(sc.warp_v[k], sc.warp_i[k], bv, bi)) bv = sc.warp_v[k], bi = sc.warp_i[k];
    sc.cta_v[slot] = bv;
    sc.cta_i[slot] = bi;
  }
  cluster_sync_all();
}

// cluster arg-max of slot `slot` (after cta_argmax), read from every rank in rank order
__device__ void cluster_argmax(SampleScratch& sc, int slot, double* v, int* i) {
  double bv = ld_dsmem_f64(&sc.cta_v[slot], 0);
  int bi = ld_dsmem_s32(&sc.cta_i[slot], 0);
  for (uint32_t r = 1; r < kSampCluster; ++r) {
    const double ov = ld_dsmem_f64(&sc.cta_v[slot], r);
    const int oi = ld_dsmem_s32(&sc.cta_i[slot], r);
    if (better(ov, oi, bv, bi)) bv = ov, bi = oi;
  }
  *v = bv;
  *i = bi;
}

// One radix-select round.  hist[round & 1] gets, for every key of this CTA with key >= lo_key and (key & mask) ==
// prefix, a count of 1 (mass == false) or its fixed-point mass floor(exp(s - m) * 2^40), in bin (key >> shift) &
// (bins - 1).  The cluster's histogram is merged and scanned from the top bin down; the first bin whose inclusive
// sum reaches the target is returned (*bin_out) with the sum strictly above it (*above_out).  target_p > 0
// replaces the target by clamp(ceil(target_p * total), 1, total), total being this round's whole sum; *target_out
// gets the target used.  Every thread of every CTA of the cluster calls it.
__device__ void radix_round(SampleScratch& sc, const float* s_sh, int n_local, int round, bool mass, float m,
                            uint32_t lo_key, uint32_t mask, uint32_t prefix, int shift, int bins,
                            unsigned long long target, double target_p, uint32_t* bin_out,
                            unsigned long long* above_out, unsigned long long* target_out) {
  unsigned long long* h = sc.hist[round & 1];  // last read in round - 2, before round - 1's cluster barrier
  for (int b = threadIdx.x; b < bins; b += kSampThreads) h[b] = 0;
  __syncthreads();
  for (int j = threadIdx.x; j < n_local; j += kSampThreads) {
    const float s = s_sh[j];
    const uint32_t key = order_key(s);
    if (key >= lo_key && (key & mask) == prefix) {
      const unsigned long long add = mass ? __float2ull_rz(expf(s - m) * kMassScale) : 1ull;
      atomicAdd(&h[(key >> shift) & (bins - 1)], add);
    }
  }
  cluster_sync_all();
  // thread t owns `per` consecutive bins, walking down from the top bin
  const int per = bins / kSampThreads;  // 8 or 4
  unsigned long long vals[kHistBins / kSampThreads];
  unsigned long long tot = 0;
#pragma unroll
  for (int j = 0; j < kHistBins / kSampThreads; ++j) {
    vals[j] = 0;
    if (j < per) {
      const int b = bins - 1 - (threadIdx.x * per + j);
      for (uint32_t r = 0; r < kSampCluster; ++r) vals[j] += ld_dsmem_u64(&h[b], r);
      tot += vals[j];
    }
  }
  // exclusive scan of tot over the block (thread order = bins from the top)
  unsigned long long incl = tot;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xffffffffu, incl, o);
    if ((threadIdx.x & 31) >= o) incl += y;
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 31) sc.warp_sum[w] = incl;
  __syncthreads();
  unsigned long long excl = incl - tot, total = 0;
  for (int k = 0; k < kSampWarps; ++k) {
    if (k < w) excl += sc.warp_sum[k];
    total += sc.warp_sum[k];
  }
  if (target_p > 0.0) {
    const double x = ceil(target_p * static_cast<double>(total));
    target = x < 1.0 ? 1ull : static_cast<unsigned long long>(x);
    if (target > total) target = total;
  }
  if (excl < target && excl + tot >= target) {  // exactly one thread (1 <= target <= total)
    unsigned long long run = excl;
    bool found = false;
#pragma unroll
    for (int j = 0; j < kHistBins / kSampThreads; ++j) {
      if (j < per && !found && run + vals[j] >= target) {
        sc.found_bin = static_cast<uint32_t>(bins - 1 - (threadIdx.x * per + j));
        sc.found_above = run;
        found = true;
      }
      run += vals[j];
    }
  }
  __syncthreads();
  *bin_out = sc.found_bin;
  *above_out = sc.found_above;
  *target_out = target;
}

// Three rounds: the key at which the inclusive (count or mass) sum from the top first reaches the target.
__device__ uint32_t radix_select(SampleScratch& sc, const float* s_sh, int n_local, int* round, bool mass, float m,
                                 uint32_t lo_key, unsigned long long target, double target_p) {
  uint32_t prefix = 0, mask = 0;
#pragma unroll 1
  for (int r = 0; r < 3; ++r) {
    const int shift = r == 0 ? 21 : r == 1 ? 10 : 0;
    const int bins = r == 2 ? 1024 : 2048;
    uint32_t bin;
    unsigned long long above, used;
    radix_round(sc, s_sh, n_local, (*round)++, mass, m, lo_key, mask, prefix, shift, bins, target,
                r == 0 ? target_p : 0.0, &bin, &above, &used);
    prefix |= bin << shift;
    mask |= static_cast<uint32_t>(bins - 1) << shift;
    target = used - above;
  }
  return prefix;
}

__global__ void __launch_bounds__(kSampThreads, 2) sample_kernel(SampleArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  SampleScratch& sc = *reinterpret_cast<SampleScratch*>(smem);
  float* s_sh = reinterpret_cast<float*>(smem + ((sizeof(SampleScratch) + 15) & ~size_t(15)));
  griddep_wait();
  griddep_launch_dependents();
  const int row = blockIdx.y;
  if (a.position[row] < 0) return;  // idle slot: the whole cluster leaves, its token is untouched
  const uint32_t rank = cluster_ctarank();
  const int base = static_cast<int>(rank) * a.slice;
  const int n_local = max(0, min(a.slice, a.V - base));
  const float inv_t = a.inv_t[row];
  const int top_k = a.top_k[row];
  const float top_p = a.top_p[row];
  const bool greedy = !(inv_t > 0.f) || top_k == 1;
  const bool use_k = !greedy && top_k > 1 && top_k < a.V;
  const bool use_p = !greedy && top_p < 1.f;
  const float mul = greedy ? 1.f : inv_t;

  // pass 1: s into shared memory, and the slice's first arg-max
  const __nv_bfloat16* lrow = a.logits + static_cast<int64_t>(row) * a.ld + base;
  const bool vec = (reinterpret_cast<uintptr_t>(lrow) & 7) == 0;
  float best = -INFINITY;
  int best_i = INT_MAX;
  for (int j = threadIdx.x * 4; j < n_local; j += kSampThreads * 4) {
    float v[4];
    if (vec && j + 4 <= n_local) {
      const uint2 w = *reinterpret_cast<const uint2*>(lrow + j);
      v[0] = bf_lo(w.x); v[1] = bf_hi(w.x); v[2] = bf_lo(w.y); v[3] = bf_hi(w.y);
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] = j + e < n_local ? __bfloat162float(lrow[j + e]) : 0.f;
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float s = v[e] * mul;
      if (s == 0.f) s = 0.f;  // -0 -> +0: one key per value
      v[e] = s;
      if (j + e < n_local && (s > best || (best_i == INT_MAX && s == s))) best = s, best_i = base + j + e;
    }
    *reinterpret_cast<float4*>(s_sh + j) = make_float4(v[0], v[1], v[2], v[3]);
  }

  if (greedy) {
    cta_argmax(sc, best, best_i, 0);
    if (rank == 0 && threadIdx.x == 0) {
      double v;
      int i;
      cluster_argmax(sc, 0, &v, &i);
      a.tokens[row] = i;
      if (a.n_kept) a.n_kept[row] = 1;
    }
    cluster_sync_all();  // no CTA leaves while rank 0 reads its shared memory
    return;
  }

  float m = 0.f;
  if (use_p) {
    cta_argmax(sc, best, best_i, 0);
    double v;
    int i;
    cluster_argmax(sc, 0, &v, &i);
    m = static_cast<float>(v);
  }
  int round = 0;
  uint32_t lo_key = 0;  // kept: key >= lo_key
  if (use_k) lo_key = radix_select(sc, s_sh, n_local, &round, false, 0.f, 0u, static_cast<unsigned long long>(top_k), 0.0);
  if (use_p) lo_key = radix_select(sc, s_sh, n_local, &round, true, m, lo_key, 0ull, static_cast<double>(top_p));

  // pass 2: Gumbel-max over the kept set
  const uint64_t seed = static_cast<uint64_t>(a.seed[row]);
  const uint64_t t = static_cast<uint64_t>(a.step[row]);
  const uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
  double bv = -INFINITY;
  int bi = INT_MAX;
  unsigned cnt = 0;
  for (int j = threadIdx.x * 4; j < n_local; j += kSampThreads * 4) {
    const float4 s4 = *reinterpret_cast<const float4*>(s_sh + j);
    const float s[4] = {s4.x, s4.y, s4.z, s4.w};
    bool keep[4], any = false;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      keep[e] = j + e < n_local && order_key(s[e]) >= lo_key;
      any |= keep[e];
    }
    if (!any) continue;
    const uint4 x = philox4x32_10(
        make_uint4(static_cast<uint32_t>((base + j) >> 2), static_cast<uint32_t>(t), static_cast<uint32_t>(t >> 32), 0u),
        k0, k1);
    const uint32_t xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (!keep[e]) continue;
      ++cnt;
      const double v = static_cast<double>(s[e]) + static_cast<double>(gumbel(xs[e]));
      if (better(v, base + j + e, bv, bi)) bv = v, bi = base + j + e;
    }
  }
  if (a.n_kept) {
    const unsigned wc = __reduce_add_sync(0xffffffffu, cnt);
    if ((threadIdx.x & 31) == 0) sc.warp_sum[threadIdx.x >> 5] = wc;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long c = 0;
      for (int k = 0; k < kSampWarps; ++k) c += sc.warp_sum[k];
      sc.cta_n = c;
    }
  }
  cta_argmax(sc, bv, bi, 1);  // its cluster barrier also publishes cta_n
  if (rank == 0 && threadIdx.x == 0) {
    double v;
    int i;
    cluster_argmax(sc, 1, &v, &i);
    a.tokens[row] = i;
    if (a.n_kept) {
      unsigned long long c = 0;
      for (uint32_t r = 0; r < kSampCluster; ++r) c += ld_dsmem_u64(&sc.cta_n, r);
      a.n_kept[row] = static_cast<int32_t>(c);
    }
  }
  cluster_sync_all();
}

size_t sample_smem_bytes(int slice) {
  return ((sizeof(SampleScratch) + 15) & ~size_t(15)) + static_cast<size_t>(slice) * sizeof(float);
}

}  // namespace

int sample_batch(const SampleParams& p, cudaStream_t stream) {
  VB_CHECK(p.logits && p.inv_temperature && p.top_k && p.top_p && p.seed && p.step && p.position && p.tokens,
           "sample_batch: logits, the five parameter arrays, position and tokens are required");
  VB_CHECK(p.M >= 1 && p.M <= 65535, "sample_batch: bad row count M=%d (1..65535)", p.M);
  VB_CHECK(p.V >= 1 && p.V <= kSampCluster * kSampMaxSlice, "sample_batch: bad vocabulary size V=%d (1..%d)", p.V,
           kSampCluster * kSampMaxSlice);
  VB_CHECK(p.ld >= p.V, "sample_batch: row stride %lld is smaller than V=%d", (long long)p.ld, p.V);
  VB_CHECK((reinterpret_cast<uintptr_t>(p.logits) & 1) == 0 && (reinterpret_cast<uintptr_t>(p.inv_temperature) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.top_k) & 3) == 0 && (reinterpret_cast<uintptr_t>(p.top_p) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.seed) & 7) == 0 && (reinterpret_cast<uintptr_t>(p.step) & 7) == 0 &&
               (reinterpret_cast<uintptr_t>(p.position) & 3) == 0 && (reinterpret_cast<uintptr_t>(p.tokens) & 7) == 0 &&
               (reinterpret_cast<uintptr_t>(p.n_kept) & 3) == 0,
           "sample_batch: misaligned pointer");
  const int slice = ((p.V + kSampCluster - 1) / kSampCluster + 3) & ~3;
  SampleArgs a{p.logits, p.ld, p.inv_temperature, p.top_k, p.top_p, p.seed, p.step, p.position, p.tokens, p.n_kept,
               p.V, slice};
  static PerDeviceOnce attr_once;
  if (attr_once.first())
    VB_CUDA(cudaFuncSetAttribute(sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)sample_smem_bytes(kSampMaxSlice)));
  VB_CUDA(launch_pdl_cluster(sample_kernel, dim3(kSampCluster, p.M), dim3(kSampThreads), sample_smem_bytes(slice),
                             stream, dim3(kSampCluster, 1, 1), a));
  return 0;
}

}  // namespace vb
