// Log-probabilities of one row for the single-stream graph decoder (GraphDecoder with logprobs, vila_b200/model/
// qwen2.py): vila_token_logprobs_row.
//
// The rule is vila_token_logprobs' (vila_b200/logprobs.py states it in numpy).  vila_token_logprobs gives each row one
// 8-CTA cluster, which at M = 1 leaves most of the GPU idle; this kernel spreads the one row over the whole GPU:
//
//   1. One CTA per chunk of kRowChunk entries (the chunk size is a constant, so the cut depends on V only).  Each
//      thread holds 4 consecutive entries.  The CTA computes the chunk's max m_c, its fp32 s_c = sum exp(x - m_c) in a
//      fixed order (each thread's 4 in order, a warp butterfly, the warps in order) and its top n, and writes them
//      to the workspace.
//   2. The top n use 64-bit keys (order-preserving bits of the value << 32 | ~index): larger key = larger value, or
//      the same value at a lower index, so "the n largest keys" is the rule's stable descending order.  -0 counts as
//      +0.  Each warp takes its n largest keys in n shuffle rounds, then the CTA places the 9 warps' candidates by
//      rank (the number of larger candidates).
//   3. The last CTA to arrive (an arrival counter, reset by that CTA so that graph replays need no memset) combines
//      the chunks in chunk order: M = max m_c, Z = sum s_c exp(m_c - M) (one chunk per thread, then the same fixed
//      reduction), log Z, and the n largest of every chunk's keys (warp rounds over slices of them, then the rank
//      placement).  It writes lp_hist[col], top_ids[col, :k] and top_lp[col, :k], col = min(step - 1, cols - 1), where
//      k = min(*n_used, n) alternatives (all n without n_used) and n is the row stride of top_ids / top_lp: a
//      captured graph serves every k up to n.
//
// Every sum runs in an order fixed by V, and which CTA arrives last does not change what it reads, so the bits do not
// depend on scheduling or on the device.  The chosen token's value and the top values are both (x - M) - log Z from
// the same M and log Z: the token's value equals its top entry bit for bit.
#include <math.h>

#include "common.cuh"
#include "kernels.h"

namespace vb {
namespace {

constexpr int kRowThreads = 288;                 // 9 warps
constexpr int kRowWarps = kRowThreads / 32;
constexpr int kRowChunk = kRowThreads * 4;       // 1152 entries per CTA: 132 CTAs at V = 152,064
constexpr int kRowMaxTop = 20;
constexpr int kRowMaxVocab = 8 * 40960;          // as vila_token_logprobs
constexpr int kRowMaxChunks = (kRowMaxVocab + kRowChunk - 1) / kRowChunk;  // 285: at most one chunk per thread
static_assert(kRowMaxChunks <= kRowThreads, "the last CTA combines one chunk per thread");

typedef unsigned long long u64;

struct RowArgs {
  const __nv_bfloat16* logits;
  const int32_t* token;
  const int32_t* step;
  float* lp_hist;
  int32_t* top_ids;
  float* top_lp;
  const int32_t* n_used;
  u64* ws_keys;      // [chunks, kRowMaxTop]
  float2* ws_ms;     // [chunks] (m_c, s_c)
  unsigned int* counter;
  int V, cols, n, chunks;
};

__device__ __forceinline__ u64 lp_key(float v, int idx) {
  if (v == 0.f) v = 0.f;  // -0 -> +0: equal values differ by index only
  const uint32_t b = __float_as_uint(v);
  const uint32_t o = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
  return (static_cast<u64>(o) << 32) | static_cast<u64>(0xffffffffu - static_cast<uint32_t>(idx));
}
__device__ __forceinline__ float key_value(u64 k) {
  const uint32_t o = static_cast<uint32_t>(k >> 32);
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}
__device__ __forceinline__ int key_index(u64 k) { return static_cast<int>(0xffffffffu - static_cast<uint32_t>(k)); }

__device__ __forceinline__ u64 warp_max_u64(u64 v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const u64 w = __shfl_xor_sync(0xffffffffu, v, o);
    v = w > v ? w : v;
  }
  return v;
}

// fixed-order block sum: lane butterfly, then the warps in order (thread 0's result, broadcast through red[])
__device__ __forceinline__ float block_sum(float z, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = z;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int k = 0; k < kRowWarps; ++k) t += red[k];
    red[kRowWarps] = t;
  }
  __syncthreads();
  return red[kRowWarps];
}

__device__ __forceinline__ float block_max(float m, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  float r = red[0];
  for (int k = 1; k < kRowWarps; ++k) r = fmaxf(r, red[k]);
  __syncthreads();  // red[] is reused next
  return r;
}

// Rank placement of the warps' candidates cand[0, kRowWarps * n) (distinct keys, 0 = none): top[p] = the key with p
// larger candidates, for p < n; places with no key stay 0 (top[] is zeroed by the caller before its last barrier).
__device__ __forceinline__ void place_by_rank(const u64* cand, int n, u64* top) {
  const int nc = kRowWarps * n;
  if (static_cast<int>(threadIdx.x) < nc) {
    const u64 k = cand[threadIdx.x];
    if (k != 0ull) {
      int place = 0;
      for (int j = 0; j < nc; ++j) place += cand[j] > k;
      if (place < n) top[place] = k;
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kRowThreads) token_logprobs_row_kernel(RowArgs a) {
  extern __shared__ u64 all_keys[];  // last CTA: every chunk's top n
  __shared__ u64 cand[kRowWarps * kRowMaxTop];
  __shared__ u64 top[kRowMaxTop];
  __shared__ float red[kRowWarps + 1];
  __shared__ bool last;
  griddep_wait();
  griddep_launch_dependents();
  const int c = blockIdx.x;
  const int base = c * kRowChunk;
  const int j0 = base + static_cast<int>(threadIdx.x) * 4;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int n = a.n_used ? max(0, min(*a.n_used, a.n)) : a.n;  // alternatives this launch; a.n is the row stride

  float v[4];
  if (j0 + 4 <= a.V && (reinterpret_cast<uintptr_t>(a.logits + j0) & 7) == 0) {
    const uint2 u = *reinterpret_cast<const uint2*>(a.logits + j0);
    v[0] = bf_lo(u.x); v[1] = bf_hi(u.x); v[2] = bf_lo(u.y); v[3] = bf_hi(u.y);
  } else {
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = j0 + e < a.V ? __bfloat162float(a.logits[j0 + e]) : -INFINITY;
  }
  if (static_cast<int>(threadIdx.x) < kRowMaxTop) top[threadIdx.x] = 0ull;

  // the chunk's max and exp-sum
  float m = fmaxf(fmaxf(v[0], v[1]), fmaxf(v[2], v[3]));
  m = block_max(m, red);
  float z = 0.f;
#pragma unroll
  for (int e = 0; e < 4; ++e)
    if (j0 + e < a.V) z += expf(v[e] - m);
  z = block_sum(z, red);

  // the chunk's top n: each warp's n largest keys, best first, then the rank placement
  if (n > 0) {
    u64 k[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) k[e] = j0 + e < a.V ? lp_key(v[e], j0 + e) : 0ull;
    u64 prev = ~0ull;
    for (int r = 0; r < n; ++r) {
      u64 b = 0ull;
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (k[e] < prev && k[e] > b) b = k[e];
      b = warp_max_u64(b);
      if (lane == 0) cand[w * n + r] = b;
      prev = b;
    }
    __syncthreads();
    place_by_rank(cand, n, top);
    if (static_cast<int>(threadIdx.x) < n) a.ws_keys[static_cast<int64_t>(c) * kRowMaxTop + threadIdx.x] = top[threadIdx.x];
  }
  if (threadIdx.x == 0) a.ws_ms[c] = make_float2(m, z);

  // arrival: the last CTA combines
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    last = atomicAdd(a.counter, 1u) == static_cast<unsigned int>(a.chunks - 1);
  }
  __syncthreads();
  if (!last) return;
  __threadfence();

  // M, then Z = sum_c s_c exp(m_c - M): chunk c on thread c, then the fixed-order block sum
  float2 ms = make_float2(-INFINITY, 0.f);
  if (static_cast<int>(threadIdx.x) < a.chunks) ms = __ldcg(a.ws_ms + threadIdx.x);
  const float M = block_max(ms.x, red);
  const float Z = block_sum(static_cast<int>(threadIdx.x) < a.chunks ? ms.y * expf(ms.x - M) : 0.f, red);
  const float log_z = logf(Z);
  const int32_t st = *a.step;
  const int col = max(0, min(st - 1, a.cols - 1));

  if (n > 0) {
    if (static_cast<int>(threadIdx.x) < kRowMaxTop) top[threadIdx.x] = 0ull;
    const int total = a.chunks * n;
    for (int i = threadIdx.x; i < total; i += kRowThreads)
      all_keys[i] = __ldcg(a.ws_keys + static_cast<int64_t>(i / n) * kRowMaxTop + i % n);
    __syncthreads();
    // warp w: the n largest keys of slice w of all_keys
    const int per = (total + kRowWarps - 1) / kRowWarps;
    const int lo = w * per, hi = min(total, lo + per);
    u64 prev = ~0ull;
    for (int r = 0; r < n; ++r) {
      u64 b = 0ull;
      for (int i = lo + lane; i < hi; i += 32) {
        const u64 k = all_keys[i];
        if (k < prev && k > b) b = k;
      }
      b = warp_max_u64(b);
      if (lane == 0) cand[w * n + r] = b;
      prev = b;
    }
    __syncthreads();
    place_by_rank(cand, n, top);
    if (static_cast<int>(threadIdx.x) < n) {
      const u64 k = top[threadIdx.x];
      if (k != 0ull) {
        a.top_ids[col * a.n + threadIdx.x] = key_index(k);
        a.top_lp[col * a.n + threadIdx.x] = (key_value(k) - M) - log_z;
      }
    }
  }
  if (threadIdx.x == 0) {
    const int32_t t = *a.token;
    a.lp_hist[col] = t >= 0 && t < a.V ? (__bfloat162float(a.logits[t]) - M) - log_z
                                       : __int_as_float(0x7fffffff);  // not a token of this vocabulary
    *a.counter = 0u;  // every CTA has arrived: ready for the next launch
  }
}

}  // namespace

int64_t token_logprobs_row_workspace_bytes(int V) {
  const int64_t chunks = (static_cast<int64_t>(V) + kRowChunk - 1) / kRowChunk;
  return chunks * (kRowMaxTop * static_cast<int64_t>(sizeof(u64)) + static_cast<int64_t>(sizeof(float2)));
}

int token_logprobs_row_check(const vila_logprobs_row_params& p) {
  VB_CHECK(p.logits && p.token && p.step && p.lp_hist && p.workspace && p.counter,
           "token_logprobs_row: logits, token, step, lp_hist, workspace and counter are required");
  VB_CHECK(p.V >= 1 && p.V <= kRowMaxVocab, "token_logprobs_row: bad vocabulary size V=%d (1..%d)", p.V,
           kRowMaxVocab);
  VB_CHECK(p.cols >= 1, "token_logprobs_row: cols=%d must be >= 1", p.cols);
  VB_CHECK(p.n >= 0 && p.n <= kRowMaxTop && p.n <= p.V, "token_logprobs_row: n=%d must be in 0..%d and <= V=%d", p.n,
           kRowMaxTop, p.V);
  VB_CHECK(p.n == 0 || (p.top_ids && p.top_lp), "token_logprobs_row: n=%d needs top_ids and top_lp", p.n);
  VB_CHECK(p.workspace_bytes >= token_logprobs_row_workspace_bytes(p.V),
           "token_logprobs_row: workspace of %lld bytes is smaller than the %lld V=%d needs",
           (long long)p.workspace_bytes, (long long)token_logprobs_row_workspace_bytes(p.V), p.V);
  VB_CHECK((reinterpret_cast<uintptr_t>(p.logits) & 1) == 0 && (reinterpret_cast<uintptr_t>(p.token) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.step) & 3) == 0 && (reinterpret_cast<uintptr_t>(p.lp_hist) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.top_ids) & 3) == 0 && (reinterpret_cast<uintptr_t>(p.top_lp) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.workspace) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.counter) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.n_used) & 3) == 0,
           "token_logprobs_row: misaligned pointer");
  return 0;
}

int token_logprobs_row(const vila_logprobs_row_params& p, cudaStream_t stream) {
  if (int rc = token_logprobs_row_check(p)) return rc;
  const int chunks = (p.V + kRowChunk - 1) / kRowChunk;
  u64* keys = static_cast<u64*>(p.workspace);
  RowArgs a{static_cast<const __nv_bfloat16*>(p.logits), p.token, p.step, p.lp_hist, p.top_ids, p.top_lp, p.n_used,
            keys, reinterpret_cast<float2*>(keys + static_cast<int64_t>(chunks) * kRowMaxTop), p.counter, p.V, p.cols,
            p.n, chunks};
  // at most 285 x 20 keys = 45,600 bytes: within the default dynamic shared-memory limit (sized for n, the most
  // alternatives a launch may compute)
  const size_t smem = static_cast<size_t>(chunks) * p.n * sizeof(u64);
  VB_CUDA(launch_pdl(token_logprobs_row_kernel, dim3(chunks), dim3(kRowThreads), smem, stream, a));
  return 0;
}

}  // namespace vb
