// Temperature / top-k / top-p sampling on the device: vila_sample_batch for the continuous-batching engine
// (vila_b200/serving.py, sampling=True) and vila_sample_finalize for the single-stream graph decoder
// (GraphDecoder's sampled step, vila_b200/model/qwen2.py).
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
// Both kernels run the same selection code (draw_row), templated on the cluster width.  Every quantity it decides on
// is independent of how the row is cut into slices (integer histograms and masses summed over the whole cluster,
// exact arg-maxes with ties to the lowest index, Philox counters from the global index), so a wider cluster draws
// the same token.  sample_finalize_kernel serves one row; its width is kFinCluster.
//
// Replaces HF TemperatureLogitsWarper / TopKLogitsWarper / TopPLogitsWarper + torch.multinomial in
// GenerationMixin._sample, reached from llava_arch.py:823-833.
//
// vila_token_logprobs (token_logprobs_kernel, below the samplers so that it shares their cluster helpers) gives the
// batched engine each chosen token's log-probability and its top alternatives under the raw model distribution.
#include <math.h>

#include "common.cuh"
#include "kernels.h"

namespace vb {
namespace {

constexpr int kSampThreads = 256;
constexpr int kSampWarps = kSampThreads / 32;
constexpr int kSampCluster = 8;   // vila_sample_batch: one 8-CTA cluster per row
// vila_sample_finalize serves one row, so a wider (non-portable) 16-CTA cluster was timed against 8 on an H100 SXM
// (700 W) at V = 152,064, back-to-back launches: 16 CTAs won for greedy (5.6 vs 7.6 us) and T only (14.6 vs 25.0 us)
// but lost for top-p 0.9 (196 vs 167 us) and top-k 50 + top-p 0.9 (327 vs 220 us), where every radix round merges one
// histogram per CTA through DSMEM.  Top-p is the common request (the server's default is top_p 0.9), so: 8.
constexpr int kFinCluster = 8;
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
template <int kC>
__device__ void cluster_argmax(SampleScratch& sc, int slot, double* v, int* i) {
  double bv = ld_dsmem_f64(&sc.cta_v[slot], 0);
  int bi = ld_dsmem_s32(&sc.cta_i[slot], 0);
  for (uint32_t r = 1; r < kC; ++r) {
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
// gets the target used.  Every thread of every CTA of the kC-CTA cluster calls it.
template <int kC>
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
      for (uint32_t r = 0; r < kC; ++r) vals[j] += ld_dsmem_u64(&h[b], r);
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
template <int kC>
__device__ uint32_t radix_select(SampleScratch& sc, const float* s_sh, int n_local, int* round, bool mass, float m,
                                 uint32_t lo_key, unsigned long long target, double target_p) {
  uint32_t prefix = 0, mask = 0;
#pragma unroll 1
  for (int r = 0; r < 3; ++r) {
    const int shift = r == 0 ? 21 : r == 1 ? 10 : 0;
    const int bins = r == 2 ? 1024 : 2048;
    uint32_t bin;
    unsigned long long above, used;
    radix_round<kC>(sc, s_sh, n_local, (*round)++, mass, m, lo_key, mask, prefix, shift, bins, target,
                r == 0 ? target_p : 0.0, &bin, &above, &used);
    prefix |= bin << shift;
    mask |= static_cast<uint32_t>(bins - 1) << shift;
    target = used - above;
  }
  return prefix;
}

// One row's draw: its logits, parameters, seed and token index t.
struct RowDraw {
  const __nv_bfloat16* logits;  // the row
  int V, slice;                 // slice: values per CTA, a multiple of 4
  float inv_t;
  int top_k;
  float top_p;
  uint64_t seed, t;
};

// The rule on one row.  Every thread of every CTA of the kC-CTA cluster calls it.  Returns the slot whose per-CTA
// arg-maxes decide the token (0: greedy max pass, 1: draw pass); on return they are published by a cluster barrier,
// so any CTA may merge them with cluster_argmax<kC>.  With count, sc.cta_n holds the CTA's kept count (draw pass).
template <int kC>
__device__ int draw_row(SampleScratch& sc, float* s_sh, const RowDraw& d, bool count) {
  const uint32_t rank = cluster_ctarank();
  const int base = static_cast<int>(rank) * d.slice;
  const int n_local = max(0, min(d.slice, d.V - base));
  const bool greedy = !(d.inv_t > 0.f) || d.top_k == 1;
  const bool use_k = !greedy && d.top_k > 1 && d.top_k < d.V;
  const bool use_p = !greedy && d.top_p < 1.f;
  const float mul = greedy ? 1.f : d.inv_t;

  // pass 1: s into shared memory, and the slice's first arg-max
  const __nv_bfloat16* lrow = d.logits + base;
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
    return 0;
  }

  float m = 0.f;
  if (use_p) {
    cta_argmax(sc, best, best_i, 0);
    double v;
    int i;
    cluster_argmax<kC>(sc, 0, &v, &i);
    m = static_cast<float>(v);
  }
  int round = 0;
  uint32_t lo_key = 0;  // kept: key >= lo_key
  if (use_k)
    lo_key = radix_select<kC>(sc, s_sh, n_local, &round, false, 0.f, 0u, static_cast<unsigned long long>(d.top_k), 0.0);
  if (use_p) lo_key = radix_select<kC>(sc, s_sh, n_local, &round, true, m, lo_key, 0ull, static_cast<double>(d.top_p));

  // pass 2: Gumbel-max over the kept set
  const uint32_t k0 = static_cast<uint32_t>(d.seed), k1 = static_cast<uint32_t>(d.seed >> 32);
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
    const uint4 x = philox4x32_10(make_uint4(static_cast<uint32_t>((base + j) >> 2), static_cast<uint32_t>(d.t),
                                             static_cast<uint32_t>(d.t >> 32), 0u),
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
  if (count) {
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
  return 1;
}

__global__ void __launch_bounds__(kSampThreads, 2) sample_kernel(SampleArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  SampleScratch& sc = *reinterpret_cast<SampleScratch*>(smem);
  float* s_sh = reinterpret_cast<float*>(smem + ((sizeof(SampleScratch) + 15) & ~size_t(15)));
  griddep_wait();
  griddep_launch_dependents();
  const int row = blockIdx.y;
  if (a.position[row] < 0) return;  // idle slot: the whole cluster leaves, its token is untouched
  const RowDraw d{a.logits + static_cast<int64_t>(row) * a.ld, a.V, a.slice, a.inv_t[row], a.top_k[row],
                  a.top_p[row], static_cast<uint64_t>(a.seed[row]), static_cast<uint64_t>(a.step[row])};
  const int slot = draw_row<kSampCluster>(sc, s_sh, d, a.n_kept != nullptr);
  if (cluster_ctarank() == 0 && threadIdx.x == 0) {
    double v;
    int i;
    cluster_argmax<kSampCluster>(sc, slot, &v, &i);
    a.tokens[row] = i;
    if (a.n_kept) {
      unsigned long long c = 1;  // greedy rows keep one value
      if (slot == 1) {
        c = 0;
        for (uint32_t r = 0; r < kSampCluster; ++r) c += ld_dsmem_u64(&sc.cta_n, r);
      }
      a.n_kept[row] = static_cast<int32_t>(c);
    }
  }
  cluster_sync_all();  // no CTA leaves while rank 0 reads its shared memory
}

struct FinalizeArgs {
  const __nv_bfloat16* logits;
  const float* inv_t;
  const int32_t* top_k;
  const float* top_p;
  const int64_t* seed;
  int32_t* step;
  int32_t* position;
  int32_t* token_out;
  int32_t* token_hist;
  const uint4* embed_table;
  uint4* x_next;
  int hidden_vec;  // 16-byte vectors per embedding row
  int V, slice;
};

// The decoder's end of step: token = the rule's draw on the logits row at t = *step; token_out = token;
// token_hist[t] = token; step and position + 1; x_next = embed_table[token], each CTA copying its share.
template <int kC>
__global__ void __launch_bounds__(kSampThreads, 2) sample_finalize_kernel(FinalizeArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  SampleScratch& sc = *reinterpret_cast<SampleScratch*>(smem);
  float* s_sh = reinterpret_cast<float*>(smem + ((sizeof(SampleScratch) + 15) & ~size_t(15)));
  __shared__ int tok_s;
  griddep_wait();
  griddep_launch_dependents();
  const int32_t t = *a.step;  // read by every CTA before rank 0 advances it (after the draw's cluster barriers)
  const RowDraw d{a.logits, a.V, a.slice, *a.inv_t, *a.top_k, *a.top_p, static_cast<uint64_t>(*a.seed),
                  static_cast<uint64_t>(static_cast<int64_t>(t))};
  const int slot = draw_row<kC>(sc, s_sh, d, false);
  if (threadIdx.x == 0) {  // every CTA merges the cluster's arg-maxes itself
    double v;
    int i;
    cluster_argmax<kC>(sc, slot, &v, &i);
    tok_s = i;
  }
  __syncthreads();
  const int tok = tok_s;
  const uint32_t rank = cluster_ctarank();
  if (rank == 0 && threadIdx.x == 0) {
    *a.token_out = tok;
    if (a.token_hist) a.token_hist[t] = tok;
    *a.step = static_cast<int32_t>(static_cast<uint32_t>(t) + 1u);
    if (a.position) *a.position = *a.position + 1;
  }
  if (a.x_next) {
    const uint4* src = a.embed_table + static_cast<size_t>(tok) * a.hidden_vec;
    for (int i = static_cast<int>(rank) * kSampThreads + threadIdx.x; i < a.hidden_vec; i += kC * kSampThreads)
      a.x_next[i] = src[i];
  }
  cluster_sync_all();  // no CTA leaves while another reads its shared memory
}

// ---- vila_token_logprobs ----------------------------------------------------------------------------------------
// The rule (vila_b200/logprobs.py states it in numpy): m = max float(x), Z = sum exp(float(x_i) - m); the chosen
// token's value and those of the first n indices of a stable descending sort (ties to the lower index) are
// (float(x_j) - m) - log Z.  One cluster of kSampCluster CTAs per row, each holding its slice of float(x) in shared
// memory: a max pass (cta_argmax / cluster_argmax), a fixed-order fp32 exp-sum per CTA added in rank order, n rounds of
// a CTA arg-max over the slice that excludes the winners already taken, then a rank-ordered merge of the cluster's
// kC * n candidates on rank 0.  The slice of a row follows from V alone and every sum runs in a fixed order, so a
// row's bits depend on that row only.

constexpr int kLpMaxTop = 20;

struct LogprobArgs {
  const __nv_bfloat16* logits;
  int64_t ld;
  const int64_t* tokens;
  const int64_t* step;
  const int32_t* position;
  float* lp_hist;
  int32_t* top_ids;
  float* top_lp;
  int V, slice, cols, n;
};

struct LogprobScratch {
  SampleScratch s;  // first: cta_argmax / cluster_argmax work on it
  float warp_z[kSampWarps];
  double cta_z;               // this CTA's exp-sum (fp32 value), read by rank 0 through DSMEM
  float round_v[2][kSampWarps];  // per-warp winners of a top-n round, double-buffered by round parity
  int round_i[2][kSampWarps];
  double cand_v[kLpMaxTop];   // this CTA's top-n, best first (index INT_MAX: the slice ran out)
  int cand_i[kLpMaxTop];
  float all_v[kSampCluster * kLpMaxTop];  // rank 0: every CTA's candidates
  int all_i[kSampCluster * kLpMaxTop];
  float log_z;
};

// the best (value, index) of this thread's elements of the slice (NaN marks a value already taken)
__device__ __forceinline__ void thread_best(const float* s_sh, int n_local, int base, float* bv, int* bi) {
  float v = -INFINITY;
  int i = INT_MAX;
  for (int j = threadIdx.x * 4; j < n_local; j += kSampThreads * 4) {
    const float4 s4 = *reinterpret_cast<const float4*>(s_sh + j);
    const float s[4] = {s4.x, s4.y, s4.z, s4.w};
#pragma unroll
    for (int e = 0; e < 4; ++e)
      if (j + e < n_local && (s[e] > v || (s[e] == v && base + j + e < i))) v = s[e], i = base + j + e;
  }
  *bv = v;
  *bi = i;
}

__global__ void __launch_bounds__(kSampThreads, 2) token_logprobs_kernel(LogprobArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  LogprobScratch& sc = *reinterpret_cast<LogprobScratch*>(smem);
  float* s_sh = reinterpret_cast<float*>(smem + ((sizeof(LogprobScratch) + 15) & ~size_t(15)));
  griddep_wait();
  griddep_launch_dependents();
  const int row = blockIdx.y;
  if (a.position[row] < 0) return;  // idle row: the whole cluster leaves, nothing is written
  const uint32_t rank = cluster_ctarank();
  const int base = static_cast<int>(rank) * a.slice;
  const int n_local = max(0, min(a.slice, a.V - base));
  const __nv_bfloat16* lrow = a.logits + static_cast<int64_t>(row) * a.ld + base;
  const bool vec = (reinterpret_cast<uintptr_t>(lrow) & 7) == 0;

  // pass 1: float(x) into shared memory and the slice's first arg-max
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
    for (int e = 0; e < 4; ++e)
      if (j + e < n_local && (v[e] > best || (best_i == INT_MAX && v[e] == v[e]))) best = v[e], best_i = base + j + e;
    *reinterpret_cast<float4*>(s_sh + j) = make_float4(v[0], v[1], v[2], v[3]);
  }
  cta_argmax(sc.s, best, best_i, 0);
  float m;
  {
    double v;
    int i;
    cluster_argmax<kSampCluster>(sc.s, 0, &v, &i);
    m = static_cast<float>(v);
  }

  // pass 2: this CTA's exp-sum, each thread over its elements in order, then lane 0's butterfly, then warps in order
  float z = 0.f;
  for (int j = threadIdx.x * 4; j < n_local; j += kSampThreads * 4) {
    const float4 s4 = *reinterpret_cast<const float4*>(s_sh + j);
    const float s[4] = {s4.x, s4.y, s4.z, s4.w};
#pragma unroll
    for (int e = 0; e < 4; ++e)
      if (j + e < n_local) z += expf(s[e] - m);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) sc.warp_z[w] = z;

  // top-n: each round the best value not yet taken; only the elements of the thread that held it are rescanned
  float tv;
  int ti;
  if (a.n > 0) thread_best(s_sh, n_local, base, &tv, &ti);
#pragma unroll 1
  for (int r = 0; r < a.n; ++r) {
    float v = tv;
    int i = ti;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, v, o);
      const int oi = __shfl_xor_sync(0xffffffffu, i, o);
      if (ov > v || (ov == v && oi < i)) v = ov, i = oi;
    }
    if ((threadIdx.x & 31) == 0) sc.round_v[r & 1][w] = v, sc.round_i[r & 1][w] = i;
    __syncthreads();  // round r + 1 writes the other buffer; round r + 2 this one, after round r + 1's barrier
    v = sc.round_v[r & 1][0];
    i = sc.round_i[r & 1][0];
    for (int k = 1; k < kSampWarps; ++k) {
      const float ov = sc.round_v[r & 1][k];
      const int oi = sc.round_i[r & 1][k];
      if (ov > v || (ov == v && oi < i)) v = ov, i = oi;
    }
    if (threadIdx.x == 0) sc.cand_v[r] = v, sc.cand_i[r] = i;
    const int owner = ((i - base) >> 2) & (kSampThreads - 1);  // the thread whose elements held the winner
    if (i != INT_MAX && (owner >> 5) == w) {
      // the owner's warp takes the value out and finds the owner's next best: lane l reads the owner's float4s
      // l, l + 32, ... (a serial rescan by the owner alone took ~3 us a round on an H100)
      if (static_cast<int>(threadIdx.x) == owner) s_sh[i - base] = __int_as_float(0x7fffffff);
      __syncwarp();
      float bv = -INFINITY;
      int bi = INT_MAX;
      for (int j = owner * 4 + (threadIdx.x & 31) * (kSampThreads * 4); j < n_local; j += 32 * kSampThreads * 4) {
        const float4 s4 = *reinterpret_cast<const float4*>(s_sh + j);
        const float sv[4] = {s4.x, s4.y, s4.z, s4.w};
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (j + e < n_local && (sv[e] > bv || (sv[e] == bv && base + j + e < bi))) bv = sv[e], bi = base + j + e;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) bv = ov, bi = oi;
      }
      if (static_cast<int>(threadIdx.x) == owner) tv = bv, ti = bi;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float cz = 0.f;
    for (int k = 0; k < kSampWarps; ++k) cz += sc.warp_z[k];
    sc.cta_z = cz;
  }
  cluster_sync_all();  // publishes cta_z and the candidates

  if (rank == 0) {
    const int nc = kSampCluster * a.n;
    if (static_cast<int>(threadIdx.x) < nc) {
      const uint32_t src = threadIdx.x / a.n;
      const int k = threadIdx.x % a.n;
      sc.all_v[threadIdx.x] = static_cast<float>(ld_dsmem_f64(&sc.cand_v[k], src));
      sc.all_i[threadIdx.x] = ld_dsmem_s32(&sc.cand_i[k], src);
    }
    if (threadIdx.x == kSampThreads - 1) {
      float zz = 0.f;
      for (uint32_t q = 0; q < kSampCluster; ++q) zz += static_cast<float>(ld_dsmem_f64(&sc.cta_z, q));
      sc.log_z = logf(zz);
    }
    __syncthreads();
    const float log_z = sc.log_z;
    const int64_t col = max(int64_t(0), min(a.step[row], static_cast<int64_t>(a.cols - 1)));
    const int64_t at = static_cast<int64_t>(row) * a.cols + col;
    if (threadIdx.x == 0) {
      const int64_t t = a.tokens[row];
      a.lp_hist[at] = t >= 0 && t < a.V
                          ? (__bfloat162float(a.logits[static_cast<int64_t>(row) * a.ld + t]) - m) - log_z
                          : __int_as_float(0x7fffffff);  // not a token of this vocabulary
    }
    if (static_cast<int>(threadIdx.x) < nc) {
      const float v = sc.all_v[threadIdx.x];
      const int i = sc.all_i[threadIdx.x];
      if (i != INT_MAX) {
        int place = 0;  // candidates ahead of this one in (value descending, index ascending) order
        for (int k = 0; k < nc; ++k) {
          const float ov = sc.all_v[k];
          const int oi = sc.all_i[k];
          place += oi != INT_MAX && (ov > v || (ov == v && oi < i));
        }
        if (place < a.n) {
          a.top_ids[at * a.n + place] = i;
          a.top_lp[at * a.n + place] = (v - m) - log_z;
        }
      }
    }
  }
  cluster_sync_all();  // no CTA leaves while rank 0 reads its shared memory
}

size_t sample_smem_bytes(int slice) {
  return ((sizeof(SampleScratch) + 15) & ~size_t(15)) + static_cast<size_t>(slice) * sizeof(float);
}

size_t logprob_smem_bytes(int slice) {
  return ((sizeof(LogprobScratch) + 15) & ~size_t(15)) + static_cast<size_t>(slice) * sizeof(float);
}

// values per CTA when a cluster of `cluster` CTAs splits a row of V: a multiple of 4
int slice_for(int V, int cluster) { return ((V + cluster - 1) / cluster + 3) & ~3; }

}  // namespace

int sample_batch(const vila_sample_params& p, cudaStream_t stream) {
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
  const int slice = slice_for(p.V, kSampCluster);
  SampleArgs a{static_cast<const __nv_bfloat16*>(p.logits), p.ld, p.inv_temperature, p.top_k, p.top_p, p.seed, p.step,
               p.position, p.tokens, p.n_kept, p.V, slice};
  static PerDeviceOnce attr_once;
  if (attr_once.first())
    VB_CUDA(cudaFuncSetAttribute(sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)sample_smem_bytes(kSampMaxSlice)));
  VB_CUDA(launch_pdl_cluster(sample_kernel, dim3(kSampCluster, p.M), dim3(kSampThreads), sample_smem_bytes(slice),
                             stream, dim3(kSampCluster, 1, 1), a));
  return 0;
}

int sample_finalize_check(const vila_sample_finalize_params& p) {
  VB_CHECK(p.logits && p.inv_temperature && p.top_k && p.top_p && p.seed && p.step && p.token_out,
           "sample_finalize: logits, the four parameter scalars, step and token_out are required");
  VB_CHECK(p.V >= 1 && p.V <= kSampCluster * kSampMaxSlice, "sample_finalize: bad vocabulary size V=%d (1..%d)", p.V,
           kSampCluster * kSampMaxSlice);
  VB_CHECK((p.embed_table == nullptr) == (p.x_next == nullptr),
           "sample_finalize: embed_table and x_next go together");
  VB_CHECK(p.x_next == nullptr || (p.hidden > 0 && p.hidden % 8 == 0),
           "sample_finalize: hidden=%d must be a positive multiple of 8", p.hidden);
  VB_CHECK((reinterpret_cast<uintptr_t>(p.logits) & 1) == 0 && (reinterpret_cast<uintptr_t>(p.inv_temperature) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.top_k) & 3) == 0 && (reinterpret_cast<uintptr_t>(p.top_p) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.seed) & 7) == 0 && (reinterpret_cast<uintptr_t>(p.step) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.position) & 3) == 0 && (reinterpret_cast<uintptr_t>(p.token_out) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.token_hist) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.embed_table) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.x_next) & 15) == 0,
           "sample_finalize: misaligned pointer");
  return 0;
}

int sample_finalize(const vila_sample_finalize_params& p, cudaStream_t stream) {
  if (int rc = sample_finalize_check(p)) return rc;
  const int slice = slice_for(p.V, kFinCluster);
  FinalizeArgs a{static_cast<const __nv_bfloat16*>(p.logits), p.inv_temperature, p.top_k, p.top_p, p.seed, p.step,
                 p.position, p.token_out, p.token_hist, static_cast<const uint4*>(p.embed_table),
                 static_cast<uint4*>(p.x_next), p.hidden / 8, p.V, slice};
  auto kern = sample_finalize_kernel<kFinCluster>;
  static PerDeviceOnce attr_once;
  if (attr_once.first())
    VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)sample_smem_bytes(slice_for(kSampCluster * kSampMaxSlice, kFinCluster))));
  VB_CUDA(launch_pdl_cluster(kern, dim3(kFinCluster), dim3(kSampThreads), sample_smem_bytes(slice), stream,
                             dim3(kFinCluster, 1, 1), a));
  return 0;
}

int token_logprobs_check(const vila_logprobs_params& p) {
  VB_CHECK(p.logits && p.tokens && p.step && p.position && p.lp_hist,
           "token_logprobs: logits, tokens, step, position and lp_hist are required");
  VB_CHECK(p.M >= 1 && p.M <= 65535, "token_logprobs: bad row count M=%d (1..65535)", p.M);
  VB_CHECK(p.V >= 1 && p.V <= kSampCluster * kSampMaxSlice, "token_logprobs: bad vocabulary size V=%d (1..%d)", p.V,
           kSampCluster * kSampMaxSlice);
  VB_CHECK(p.ld >= p.V, "token_logprobs: row stride %lld is smaller than V=%d", (long long)p.ld, p.V);
  VB_CHECK(p.cols >= 1, "token_logprobs: cols=%d must be >= 1", p.cols);
  VB_CHECK(p.n >= 0 && p.n <= kLpMaxTop && p.n <= p.V, "token_logprobs: n=%d must be in 0..%d and <= V=%d", p.n,
           kLpMaxTop, p.V);
  VB_CHECK(p.n == 0 || (p.top_ids && p.top_lp), "token_logprobs: n=%d needs top_ids and top_lp", p.n);
  VB_CHECK((reinterpret_cast<uintptr_t>(p.logits) & 1) == 0 && (reinterpret_cast<uintptr_t>(p.tokens) & 7) == 0 &&
               (reinterpret_cast<uintptr_t>(p.step) & 7) == 0 && (reinterpret_cast<uintptr_t>(p.position) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.lp_hist) & 3) == 0 && (reinterpret_cast<uintptr_t>(p.top_ids) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.top_lp) & 3) == 0,
           "token_logprobs: misaligned pointer");
  return 0;
}

int token_logprobs(const vila_logprobs_params& p, cudaStream_t stream) {
  if (int rc = token_logprobs_check(p)) return rc;
  const int slice = slice_for(p.V, kSampCluster);
  LogprobArgs a{static_cast<const __nv_bfloat16*>(p.logits), p.ld, p.tokens, p.step, p.position, p.lp_hist, p.top_ids,
                p.top_lp, p.V, slice, p.cols, p.n};
  static PerDeviceOnce attr_once;
  if (attr_once.first())
    VB_CUDA(cudaFuncSetAttribute(token_logprobs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)logprob_smem_bytes(kSampMaxSlice)));
  VB_CUDA(launch_pdl_cluster(token_logprobs_kernel, dim3(kSampCluster, p.M), dim3(kSampThreads),
                             logprob_smem_bytes(slice), stream, dim3(kSampCluster, 1, 1), a));
  return 0;
}

}  // namespace vb
