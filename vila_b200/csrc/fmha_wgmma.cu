// Flash-attention forward for sm_90a with wgmma tensor cores and register accumulators.
//
// One CTA = one 128-row query tile of one (batch, head).  Warp roles:
//   warps 0-7 : two consumer warpgroups, 64 query rows each
//   warp  8   : TMA producer (Q once, then K/V blocks of 128 tokens, double buffered)
// Per KV block j, in each consumer warpgroup:
//   S_j = Q K_j^T          wgmma, A = Q and B = K straight from 128B/64B-swizzled shared memory
//   P_j = exp2(S_j*scale - m), online softmax on the register fragments (a row lives in 4 lanes)
//   O  = O * alpha + P_j V_j   wgmma with A = P_j from registers (bf16) and B = V as the MN-major
//                              operand straight from its [tok, d] layout
// The two warpgroups run independently, so one's softmax overlaps the other's tensor-core work.
// Head dims that are not a multiple of the swizzle chunk (SigLIP d=72) are zero-padded for free
// by TMA out-of-bounds fill (72 -> 96 = 3 x 32-column SW64 chunks); the LLM d=128 uses 2 x SW128.
//
// Replaces flash_attn_func in SiglipFlashAttention2 (modeling_siglip.py:583-585, non-causal,
// scale 72^-0.5) and HF _flash_attention_forward for Qwen2 (modeling_qwen2.py:191-310; causal GQA).
#include <math.h>
#include <stdlib.h>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace vb {

namespace {

constexpr int BQ = 128;   // query rows per CTA
constexpr int BKV = 128;  // kv rows per block (== KV page size)
constexpr int kConsumerThreads = 256;
constexpr int kThreads = kConsumerThreads + 32;

template <int DP, int CW>
struct FmhaCfg {
  static_assert(DP % CW == 0, "");
  static constexpr int kChunks = DP / CW;
  static constexpr int kChunkBytes = 128 * CW * 2;  // [128 rows][CW] bf16
  static constexpr int kTileBytes = kChunks * kChunkBytes;
  static constexpr uint32_t kLayout = CW == 64 ? kWgmmaSW128 : kWgmmaSW64;
  static constexpr int kSwizzleBytes = CW * 2;
  static constexpr int kSBO = 8 * CW * 2;  // 8-row group pitch
  static constexpr int kNumBars = 9;
  static constexpr int kSmem = kTileBytes * 5 + kNumBars * 8 + 16 + 1024;
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// exp2 on the FMA pipe (Cody-Waite split + degree-3 minimax polynomial, max relative error 7.5e-5,
// far below the bf16 rounding P gets anyway): moves part of the exponentials off the MUFU unit.
__device__ __forceinline__ float ex2_poly(float x) {
  x = fmaxf(x, -125.f);
  const float xf = x + 12582912.f;          // 1.5 * 2^23: rounds x to an integer in the low mantissa bits
  const float fr = x - (xf - 12582912.f);   // fractional part in [-0.5, 0.5]
  float p = fmaf(fr, 0.0551716685f, 0.2426111251f);
  p = fmaf(fr, p, 0.6932609677f);
  p = fmaf(fr, p, 0.9999280572f);
  return __int_as_float(__float_as_int(p) + (__float_as_int(xf) << 23));
}

struct FmhaKernelArgs {
  __nv_bfloat16* o;
  int64_t o_tok_stride, o_head_stride;
  const int32_t* page_table;
  int page_table_stride;
  int Sq, Sk, Hq, Hkv, D, causal, paged;
  float scale_log2;
  // split-KV decode mode (fmha_decode_split): blockIdx.z is a KV split of ONE sequence, not a batch
  // entry.  Split z covers tokens [z*split_tokens, min(Sk_total, (z+1)*split_tokens)); Sk_total is read
  // from device memory (*sk_dev + 1: the position of the token being decoded), the partial outputs go
  // to o_partial (fp32, normalised per split) with their log2-sum-exp in lse_out.
  const int32_t* sk_dev;
  int split_tokens;
  float* o_partial;  // [splits][Hq][Sq][D]
  float* lse_out;    // [splits][Hq][Sq]
  int* split_counters;  // [Hq] zero-initialised, self-cleaning; non-null: the last CTA of a head combines into o
  // batched split mode (fmha_decode_split with batch > 0): blockIdx.x is the sequence.  Sequence s reads
  // sk_dev[s] (< 0: idle, every CTA exits), the page-table row page_table + s*page_table_stride and the
  // Q rows at 4th tensor-map coordinate s; its partials, lse and counters are the s-th [splits][Hq][Sq]
  // block, its output starts at o + s*o_seq_stride.  Split CTAs past the sequence's length exit without
  // writing anything and the combine reads only the splits that hold tokens (the skipped ones would add
  // exact zeros: same bits as the single-sequence combine over all splits).
  int batched;
  int64_t o_seq_stride;
};

// kPolyEvery: every n-th exponential of a thread's row values uses ex2_poly (0: none)
template <int DP, int CW, int kPolyEvery>
__global__ void __launch_bounds__(kThreads, 1)
fmha_fwd_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                const __grid_constant__ CUtensorMap tm_v, FmhaKernelArgs a) {
  using C = FmhaCfg<DP, CW>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* q_s = smem;
  uint8_t* k_s = q_s + C::kTileBytes;       // 2 stages
  uint8_t* v_s = k_s + 2 * C::kTileBytes;   // 2 stages
  uint64_t* bars = reinterpret_cast<uint64_t*>(v_s + 2 * C::kTileBytes);
  uint64_t* q_full = bars + 0;
  uint64_t* k_full = bars + 1;   // [2]
  uint64_t* k_empty = bars + 3;  // [2]
  uint64_t* v_full = bars + 5;   // [2]
  uint64_t* v_empty = bars + 7;  // [2]
  int* is_last_s = reinterpret_cast<int*>(bars + 9);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // causal: heaviest (last) query tiles first
  const int qt = a.batched ? 0
                 : a.causal ? static_cast<int>(gridDim.x) - 1 - static_cast<int>(blockIdx.x)
                            : static_cast<int>(blockIdx.x);
  const int seq = a.batched ? static_cast<int>(blockIdx.x) : 0;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int hk = h / (a.Hq / a.Hkv);
  const bool split_mode = a.split_tokens > 0;
  // the second warpgroup only works when the tile has rows beyond the first 64 (decode: 7 rows)
  const int n_wg = (a.Sq - qt * BQ > 64) ? 2 : 1;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 4 * n_wg);  // one arrival per consumer warp
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 4 * n_wg);
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_launch_dependents();
  griddep_wait();  // Q/K/V come from the predecessor; O may alias memory it still reads

  // KV extent of this CTA (after the dependency wait: in split mode it comes from device memory)
  int Sk = a.Sk;
  int blk0 = 0;              // first KV block (page-table index) of this CTA
  const int qb = split_mode ? 0 : b;  // batch entry the queries / outputs belong to
  const int32_t* page_table = a.page_table;
  int total = 0;             // split mode: tokens of the sequence, the new one included
  if (split_mode) {
    total = a.sk_dev[seq] + 1;
    const int start = b * a.split_tokens;
    if (a.batched) {
      if (start >= total) return;  // idle sequence (total <= 0) or split past its length (block-uniform)
      page_table += static_cast<int64_t>(seq) * a.page_table_stride;
    }
    blk0 = start / BKV;
    Sk = max(0, min(a.split_tokens, total - start));
  }
  const int off = Sk - a.Sq;  // causal diagonal offset
  int kv_end = Sk;
  if (a.causal) {
    int q_last = min((qt + 1) * BQ, a.Sq) - 1;
    kv_end = min(Sk, q_last + off + 1);
  }
  const int nblk = (kv_end + BKV - 1) / BKV;

  if (warp == kConsumerThreads / 32) {
    // ===================== TMA producer =====================
    if (lane == 0 && nblk > 0) {
      tma_prefetch_desc(&tm_q);
      tma_prefetch_desc(&tm_k);
      tma_prefetch_desc(&tm_v);
      mbar_arrive_expect_tx(q_full, C::kTileBytes);
#pragma unroll
      for (int c = 0; c < C::kChunks; ++c)
        tma_load_4d(q_s + c * C::kChunkBytes, &tm_q, q_full, c * CW, h, qb * a.Sq + qt * BQ, seq);
      for (int j = 0; j < nblk; ++j) {
        const int s = j & 1;
        const uint32_t par = ((j >> 1) & 1) ^ 1;
        int tok, page;
        if (a.paged) {
          tok = 0;
          page = page_table ? page_table[split_mode ? blk0 + j : b * a.page_table_stride + j] : blk0 + j;
        } else {
          tok = b * a.Sk + j * BKV;
          page = 0;
        }
        mbar_wait(&k_empty[s], par);
        mbar_arrive_expect_tx(&k_full[s], C::kTileBytes);
#pragma unroll
        for (int c = 0; c < C::kChunks; ++c)
          tma_load_4d(k_s + s * C::kTileBytes + c * C::kChunkBytes, &tm_k, &k_full[s], c * CW, hk,
                      tok, page);
        mbar_wait(&v_empty[s], par);
        mbar_arrive_expect_tx(&v_full[s], C::kTileBytes);
#pragma unroll
        for (int c = 0; c < C::kChunks; ++c)
          tma_load_4d(v_s + s * C::kTileBytes + c * C::kChunkBytes, &tm_v, &v_full[s], c * CW, hk,
                      tok, page);
      }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  const int wg = warp >> 2;
  if (wg >= n_wg) return;
  const int ctid = threadIdx.x;
  // this thread's two rows (fragment rows r and r + 8) and first column within each n8 group
  const int r_loc = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int col0 = (lane & 3) * 2;
  const int q_idx0 = qt * BQ + r_loc;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};  // l: this thread's partial row sums
  float o_acc[DP / 2];
#pragma unroll
  for (int i = 0; i < DP / 2; ++i) o_acc[i] = 0.f;
  float s_acc[BKV / 2];
  uint32_t p_frag[BKV / 16][4];

  if (nblk > 0) mbar_wait(q_full, 0);
  for (int j = 0; j < nblk; ++j) {
    const int s = j & 1;
    const uint32_t par = (j >> 1) & 1;
    // ---- S = Q K^T ----
    mbar_wait(&k_full[s], par);
    wgmma_fence_operand<BKV / 2>(s_acc);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < C::kChunks; ++c) {
#pragma unroll
      for (int k = 0; k < CW / 16; ++k) {
        const uint64_t ad = make_wgmma_desc(
            smem_u32(q_s + c * C::kChunkBytes + wg * 64 * CW * 2) + k * 32, 16, C::kSBO, C::kLayout);
        const uint64_t bd = make_wgmma_desc(
            smem_u32(k_s + s * C::kTileBytes + c * C::kChunkBytes) + k * 32, 16, C::kSBO, C::kLayout);
        Wgmma<BKV>::ss(s_acc, ad, bd, (c | k) != 0 ? 1u : 0u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operand<BKV / 2>(s_acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&k_empty[s]);

    // ---- online softmax on the fragment ----
    const int kv0 = j * BKV;
    const bool need_mask = (kv0 + BKV > Sk) || (a.causal && (kv0 + BKV - 1 > qt * BQ + off));
    float alpha[2], m_use[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int kv_lim = a.causal ? min(Sk - 1, q_idx0 + 8 * hh + off) : Sk - 1;  // last valid kv index
      float mx = -INFINITY;
#pragma unroll
      for (int n = 0; n < BKV / 8; ++n) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& v = s_acc[4 * n + 2 * hh + e];
          if (need_mask && kv0 + 8 * n + col0 + e > kv_lim) v = -INFINITY;
          mx = fmaxf(mx, v);
        }
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m[hh], mx * a.scale_log2);
      m_use[hh] = (m_new == -INFINITY) ? 0.f : m_new;
      alpha[hh] = ex2(m[hh] - m_use[hh]);  // m == -inf -> 0
      m[hh] = m_new;
    }
    float rowsum[2] = {0.f, 0.f};
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float p2[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float x = s_acc[4 * n + 2 * hh + e] * a.scale_log2 - m_use[hh];  // -inf for masked
          const int i = 2 * n + e;
          p2[e] = (kPolyEvery > 0 && (i % (kPolyEvery > 0 ? kPolyEvery : 1)) == kPolyEvery - 1) ? (x == -INFINITY ? 0.f : ex2_poly(x))
                                                                          : ex2(x);
          rowsum[hh] += p2[e];
        }
        // accumulator n8 groups 2kk, 2kk+1 form the k16 A fragment kk
        p_frag[n >> 1][(n & 1) * 2 + hh] = pack_bf16(p2[0], p2[1]);
      }
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) l[hh] = l[hh] * alpha[hh] + rowsum[hh];
#pragma unroll
    for (int n = 0; n < DP / 8; ++n) {
      o_acc[4 * n + 0] *= alpha[0];
      o_acc[4 * n + 1] *= alpha[0];
      o_acc[4 * n + 2] *= alpha[1];
      o_acc[4 * n + 3] *= alpha[1];
    }

    // ---- O += P V ----
    mbar_wait(&v_full[s], par);
    wgmma_fence_operand<DP / 2>(o_acc);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
      // B = V (MN-major): N spans the d-chunks (LBO = chunk pitch), K = 16 token rows per MMA
      const uint64_t bd = make_wgmma_desc(smem_u32(v_s + s * C::kTileBytes) + kk * 16 * (CW * 2),
                                          C::kChunkBytes, C::kSBO, C::kLayout);
      Wgmma<DP>::rs_bt(o_acc, p_frag[kk], bd);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operand<DP / 2>(o_acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&v_empty[s]);
  }

  // full row sums (a row's values are spread over the 4 lanes of a quad)
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
  }

  if (split_mode) {
    const int64_t seq_rows = static_cast<int64_t>(seq) * gridDim.z * a.Hq * a.Sq;
    float* lse_out = a.lse_out + seq_rows;
    float* o_partial = a.o_partial + seq_rows * a.D;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int q_idx = q_idx0 + 8 * hh;
      if (q_idx >= a.Sq) continue;
      const float inv = l[hh] > 0.f ? 1.f / l[hh] : 0.f;
      const int64_t r = (static_cast<int64_t>(b) * a.Hq + h) * a.Sq + q_idx;
      if ((lane & 3) == 0) lse_out[r] = l[hh] > 0.f ? m[hh] + log2f(l[hh]) : -INFINITY;
      float* dst = o_partial + r * a.D;
#pragma unroll
      for (int n = 0; n < DP / 8; ++n) {
        const int d = 8 * n + col0;
        if (d < a.D)
          *reinterpret_cast<float2*>(dst + d) =
              make_float2(o_acc[4 * n + 2 * hh] * inv, o_acc[4 * n + 2 * hh + 1] * inv);
      }
    }
    if (a.split_counters != nullptr) {
      // Fused combine: the LAST split CTA of this head to finish merges all partials (fixed split
      // order -> deterministic) and writes the bf16 output, saving the separate combine launch.
      const int nthr = 128 * n_wg;
      // splits taking part: all of them, or (batched) those holding tokens of this sequence
      const int nsp = a.batched ? min(static_cast<int>(gridDim.z), (total + a.split_tokens - 1) / a.split_tokens)
                                : static_cast<int>(gridDim.z);
      int* counter = a.split_counters + static_cast<int64_t>(seq) * a.Hq + h;
      __threadfence();                  // this thread's partial rows are visible device-wide
      named_bar_sync(1, nthr);
      if (ctid == 0) {
        const int prev = atomicAdd(counter, 1);
        *is_last_s = (prev == nsp - 1);
        if (*is_last_s) *counter = 0;  // re-arm for the next launch / graph replay
      }
      named_bar_sync(1, nthr);
      if (*is_last_s && ctid < 128) {
        __threadfence();
        const int d = ctid;                         // 128 threads <-> D = 128 columns
        __nv_bfloat16* o = a.o + static_cast<int64_t>(seq) * a.o_seq_stride;
        for (int g = 0; g < a.Sq; ++g) {
          float mx = -INFINITY;
          for (int s = 0; s < nsp; ++s)
            mx = fmaxf(mx, __ldcg(&lse_out[(static_cast<int64_t>(s) * a.Hq + h) * a.Sq + g]));
          float den = 0.f, acc = 0.f;
          for (int s = 0; s < nsp; ++s) {
            const int64_t r = (static_cast<int64_t>(s) * a.Hq + h) * a.Sq + g;
            const float v = __ldcg(&lse_out[r]);
            const float w = (v == -INFINITY) ? 0.f : exp2f(v - mx);
            den += w;
            acc += w * __ldcg(&o_partial[r * a.D + d]);
          }
          const float inv_den = den > 0.f ? 1.f / den : 0.f;  // same arithmetic as decode_combine_kernel
          o[static_cast<int64_t>(g) * a.o_tok_stride + static_cast<int64_t>(h) * a.o_head_stride + d] =
              __float2bfloat16(acc * inv_den);
        }
      }
    }
    return;
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int q_idx = q_idx0 + 8 * hh;
    if (q_idx >= a.Sq) continue;
    const float inv = l[hh] > 0.f ? 1.f / l[hh] : 0.f;
    __nv_bfloat16* dst = a.o + static_cast<int64_t>(b * a.Sq + q_idx) * a.o_tok_stride +
                         static_cast<int64_t>(h) * a.o_head_stride;
#pragma unroll
    for (int n = 0; n < DP / 8; ++n) {
      const int d = 8 * n + col0;
      if (d < a.D)
        *reinterpret_cast<uint32_t*>(dst + d) =
            pack_bf16(o_acc[4 * n + 2 * hh] * inv, o_acc[4 * n + 2 * hh + 1] * inv);
    }
  }
}

struct SplitArgs {
  const int32_t* sk_dev;
  int split_tokens;
  float* o_partial;
  float* lse_out;
  int* counters;
  int batch;              // > 0: batched split mode, one sequence per blockIdx.x
  int64_t q_seq_stride;   // elements between the query rows of consecutive sequences
  int64_t o_seq_stride;
};

template <int DP, int CW, int kPolyEvery = 0>
int launch_fmha(const vila_fmha_params& p, cudaStream_t stream, const SplitArgs* split = nullptr) {
  using C = FmhaCfg<DP, CW>;
  CUtensorMap tq, tk, tv;
  const int batch = split ? split->batch : 0;
  {
    // split mode: the queries are ONE set of Sq rows shared by all splits (blockIdx.z); batched: one
    // such set per sequence along the 4th dimension
    const uint64_t q_rows = (uint64_t)(split ? 1 : p.B) * p.Sq;
    uint64_t dims[4] = {(uint64_t)p.D, (uint64_t)p.Hq, q_rows, batch > 0 ? (uint64_t)batch : 1};
    uint64_t str[3] = {(uint64_t)p.q_head_stride, (uint64_t)p.q_tok_stride,
                       batch > 0 ? (uint64_t)split->q_seq_stride : (uint64_t)p.q_tok_stride * q_rows};
    uint32_t box[4] = {CW, 1, BQ, 1};
    if (make_tmap_nd_bf16(&tq, p.q, 4, dims, str, box, C::kSwizzleBytes)) return 1;
  }
  const bool paged = p.kv_page_stride != 0;
  {
    uint64_t dims[4], str[3];
    if (paged) {
      dims[0] = p.D; dims[1] = p.Hkv; dims[2] = BKV; dims[3] = p.kv_num_pages;
      str[0] = p.kv_head_stride; str[1] = p.kv_tok_stride; str[2] = p.kv_page_stride;
    } else {
      dims[0] = p.D; dims[1] = p.Hkv; dims[2] = (uint64_t)p.B * p.Sk; dims[3] = 1;
      str[0] = p.kv_head_stride; str[1] = p.kv_tok_stride;
      str[2] = (uint64_t)p.kv_tok_stride * p.B * p.Sk;
    }
    uint32_t box[4] = {CW, 1, BKV, 1};
    if (make_tmap_nd_bf16(&tk, p.k, 4, dims, str, box, C::kSwizzleBytes)) return 1;
    if (make_tmap_nd_bf16(&tv, p.v, 4, dims, str, box, C::kSwizzleBytes)) return 1;
  }
  FmhaKernelArgs a;
  a.o = static_cast<__nv_bfloat16*>(p.o);
  a.o_tok_stride = p.o_tok_stride;
  a.o_head_stride = p.o_head_stride;
  a.page_table = p.page_table;
  a.page_table_stride = p.page_table_stride;
  a.Sq = p.Sq; a.Sk = p.Sk; a.Hq = p.Hq; a.Hkv = p.Hkv; a.D = p.D;
  a.causal = p.causal;
  a.paged = paged ? 1 : 0;
  a.scale_log2 = p.scale * 1.4426950408889634f;
  a.sk_dev = split ? split->sk_dev : nullptr;
  a.split_tokens = split ? split->split_tokens : 0;
  a.o_partial = split ? split->o_partial : nullptr;
  a.lse_out = split ? split->lse_out : nullptr;
  a.split_counters = split ? split->counters : nullptr;
  a.batched = batch > 0 ? 1 : 0;
  a.o_seq_stride = batch > 0 ? split->o_seq_stride : 0;
  auto kern = fmha_fwd_kernel<DP, CW, kPolyEvery>;
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmem));
  }
  dim3 grid(batch > 0 ? batch : (p.Sq + BQ - 1) / BQ, p.Hq, p.B);
  VB_CUDA(launch_pdl(kern, grid, dim3(kThreads), C::kSmem, stream, tq, tk, tv, a));
  return 0;
}

template <int kPolyEvery>
int launch_fmha_for_head_dim(const vila_fmha_params& p, cudaStream_t stream) {
  if (p.D == 128) return launch_fmha<128, 64, kPolyEvery>(p, stream);
  if (p.D <= 96 && p.D > 64) return launch_fmha<96, 32, kPolyEvery>(p, stream);
  if (p.D == 64) return launch_fmha<64, 64, kPolyEvery>(p, stream);
  set_last_error("fmha: unsupported head dim %d (supported: 64, 65..96, 128)", p.D);
  return 1;
}

}  // namespace

int fmha_prefill(const vila_fmha_params& p, cudaStream_t stream) { return fmha_prefill_cfg(0, p, stream); }

// Split-KV attention of ONE long sequence for a handful of query rows (decode: the G query heads of a
// KV group are the "rows" of the 128-row tile, the KV heads are the "heads"): p.B = number of KV
// splits of split_tokens tokens each, the sequence length is *n_tok_minus_1 + 1 (device memory, read
// after the dependency wait, so one captured graph serves every decode position), K/V paged.  Writes
// normalised fp32 partials [B][Hq][Sq][D] and their log2-sum-exp [B][Hq][Sq]; non-causal.
//
// batch > 0: `batch` sequences in one launch (blockIdx.x), sequence s with length n_tok_minus_1[s] + 1
// (< 0: idle), queries at p.q + s*q_seq_stride, page-table row p.page_table + s*p.page_table_stride,
// partials / lse / counters the s-th block of [B][Hq][Sq][D] / [B][Hq][Sq] / [Hq], output at
// p.o + s*o_seq_stride; the fused combine (counters) is required.
int fmha_decode_split(const vila_fmha_params& p, const int32_t* n_tok_minus_1, int split_tokens,
                      float* o_partial, float* lse, int* counters, cudaStream_t stream,
                      int batch, int64_t q_seq_stride, int64_t o_seq_stride) {
  VB_CHECK(p.D == 128, "fmha_decode_split: head dim must be 128");
  VB_CHECK(p.kv_page_stride != 0 && p.page_table != nullptr, "fmha_decode_split: K/V must be paged");
  VB_CHECK(split_tokens > 0 && split_tokens % BKV == 0, "fmha_decode_split: split_tokens %% 128 != 0");
  VB_CHECK(p.Sq >= 1 && p.Sq <= BQ && !p.causal, "fmha_decode_split: 1..128 query rows, non-causal");
  VB_CHECK(n_tok_minus_1 && o_partial && lse, "fmha_decode_split: null output / length pointer");
  VB_CHECK(counters == nullptr || p.o != nullptr, "fmha_decode_split: fused combine needs the output pointer");
  VB_CHECK(batch == 0 || (counters != nullptr && q_seq_stride % 8 == 0 && q_seq_stride > 0),
           "fmha_decode_split: a batch needs counters and a query stride that is a positive multiple of 8");
  VB_CHECK(p.B >= 1 && p.B <= 65535, "fmha_decode_split: 1..65535 splits (got %d)", p.B);
  SplitArgs sa{n_tok_minus_1, split_tokens, o_partial, lse, counters, batch, q_seq_stride, o_seq_stride};
  return launch_fmha<128, 64>(p, stream, &sa);
}

// variant: 0 = default, 1 / 2 = the wgmma kernel (kept as separate selectors so callers can pin a
// kernel), 3 / 4 = the same kernel with every 4th / 2nd exp2 computed by the FMA-pipe polynomial.
int fmha_prefill_cfg(int variant, const vila_fmha_params& p, cudaStream_t stream) {
  VB_CHECK(variant >= 0 && variant <= 4, "fmha: unknown variant %d", variant);
  VB_CHECK(p.B > 0 && p.Sq > 0 && p.Sk > 0, "fmha: empty problem");
  VB_CHECK(p.Hq % p.Hkv == 0, "fmha: Hq (%d) must be a multiple of Hkv (%d)", p.Hq, p.Hkv);
  VB_CHECK(p.D % 8 == 0, "fmha: head dim must be a multiple of 8 (got %d)", p.D);
  VB_CHECK(p.q_tok_stride % 8 == 0 && p.q_head_stride % 8 == 0 && p.kv_tok_stride % 8 == 0 &&
               p.kv_head_stride % 8 == 0 && p.o_tok_stride % 8 == 0 && p.o_head_stride % 8 == 0,
           "fmha: strides must be multiples of 8 elements (16 bytes)");
  VB_CHECK(!p.causal || p.Sk >= p.Sq, "fmha: causal needs Sk >= Sq");
  if (variant == 3) return launch_fmha_for_head_dim<4>(p, stream);
  if (variant == 4) return launch_fmha_for_head_dim<2>(p, stream);
  return launch_fmha_for_head_dim<0>(p, stream);
}

}  // namespace vb
