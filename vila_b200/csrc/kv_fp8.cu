// Opt-in FP8 (e4m3) KV cache of the continuous-batching engine (vila_b200/serving.py, kv_cache="fp8").
//
// Format (one rule, shared by both kernels below and by vila_b200.model.qwen2.quantize_kv_e4m3):
//   codes  e4m3 [L, 2, P, 128, Hkv, 128]  (the bf16 pool's layout with 1-byte elements; K after RoPE)
//   scales fp32 [L, 2, P, 128, Hkv]       one per (layer, K|V, token, KV head) row of 128 values
//   amax = max|x|;  inv = 448 / amax (fp32, IEEE division);  code = e4m3(rn, satfinite)(x * inv);
//   scale = amax / 448;  amax == 0: codes and scale 0.  Dequantised value: float(code) * scale.
//
//  kv_quantize_kernel      rows [0, S) of every layer's K and V of a bf16 staging cache (identity pages)
//                          -> the slot's e4m3 pages through its page-table row; one warp per row.
//  decode_attn_fp8_kernel  one decode step of every slot: RoPE of q and of the new k (the rounding points
//                          of decode_attn_head_kernel), e4m3 append of the new k / v row at `pos`, and
//                          attention over [0, pos] on the dequantised rows.  Grid (split, KV head, slot);
//                          a CTA serves the G query heads of its KV group, so every K/V byte is read once.
//                          Split j covers tokens [j*split_tokens, (j+1)*split_tokens) for every slot length;
//                          the last CTA of a (slot, KV head) combines the splits that hold tokens in index
//                          order (self-cleaning counters).  A slot's result depends on that slot only.
// Both replace DynamicCache.update + flash-attn decode (modeling_qwen2.py:99-160,262-310) for this format.
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"
#include "kernels.h"

namespace vb {
namespace {

constexpr float kE4m3Max = 448.f;
constexpr int kFaThreads = 256;
constexpr int kFaWarps = kFaThreads / 32;
constexpr int kFaChunk = 128;         // tokens per inner-loop chunk (= one page)
constexpr int kFaMaxSplitPages = 16;  // split_tokens <= 2048
constexpr int kQPad = 68;             // q_s row half stride (floats): the two d halves sit in other banks

// four e4m3 (low byte = lowest index) -> four floats, exactly (every e4m3 value is an f16 value)
__device__ __forceinline__ void e4m3x4_to_float(uint32_t w, float* f) {
  uint32_t lo, hi;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(lo) : "h"(static_cast<uint16_t>(w)));
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(hi) : "h"(static_cast<uint16_t>(w >> 16)));
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&lo));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
}

// The format's rule on one 128-value row held by a warp, four values per lane (lane j: 4j .. 4j+3).
// Returns the lane's four codes (lowest index in the low byte); *scale gets the row's scale.
__device__ __forceinline__ uint32_t quantize_row_warp(const float x[4], float* scale) {
  float amax = fmaxf(fmaxf(fabsf(x[0]), fabsf(x[1])), fmaxf(fabsf(x[2]), fabsf(x[3])));
  amax = warp_max(amax);
  if (amax == 0.f) {
    *scale = 0.f;
    return 0u;
  }
  const float inv = __fdiv_rn(kE4m3Max, amax);
  uint16_t lo, hi;  // cvt ... d, a, b: a -> upper byte, b -> lower byte
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(__fmul_rn(x[1], inv)), "f"(__fmul_rn(x[0], inv)));
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(__fmul_rn(x[3], inv)), "f"(__fmul_rn(x[2], inv)));
  *scale = __fdiv_rn(amax, kE4m3Max);
  return static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
}

struct KvQuantArgs {
  const __nv_bfloat16* src;  // staging [L, 2, src_tokens, Hkv, 128]
  int64_t src_tokens;
  uint8_t* dst;              // codes [L, 2, dst_pages, 128, Hkv, 128]
  float* dst_scale;          // [L, 2, dst_pages, 128, Hkv]
  int64_t dst_pages;
  const int32_t* page_table; // the slot's row
  int L, Hkv, S;
};

__global__ void __launch_bounds__(256) kv_quantize_kernel(KvQuantArgs a) {
  griddep_launch_dependents();
  griddep_wait();
  const int64_t rows = static_cast<int64_t>(a.L) * 2 * a.S * a.Hkv;
  const int64_t row = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;  // warp-uniform
  const int lane = threadIdx.x & 31;
  const int h = static_cast<int>(row % a.Hkv);
  const int64_t rest = row / a.Hkv;
  const int t = static_cast<int>(rest % a.S);
  const int64_t lj = rest / a.S;  // layer * 2 + (K|V)
  const uint2 v = *reinterpret_cast<const uint2*>(a.src + ((lj * a.src_tokens + t) * a.Hkv + h) * 128 + lane * 4);
  const float x[4] = {bf_lo(v.x), bf_hi(v.x), bf_lo(v.y), bf_hi(v.y)};
  float scale;
  const uint32_t codes = quantize_row_warp(x, &scale);
  const int64_t drow = ((lj * a.dst_pages + a.page_table[t >> 7]) * 128 + (t & 127)) * a.Hkv + h;
  reinterpret_cast<uint32_t*>(a.dst + drow * 128)[lane] = codes;
  if (lane == 0) a.dst_scale[drow] = scale;
}

// Inner loop, per 128-token chunk of the split (every sum in a fixed order):
//   A  thread (token r = tid / 2, d half = tid % 2): s_g = sum_d q_g[d] * float(kcode[d]) in fp32 (64 fmas per
//      half, halves added with one shuffle), then score = (s_g * kscale) * scale * log2(e)
//   B  warp per head: chunk max, m_new = max(m, chunk max), p = exp2(score - m_new), l = l * alpha + sum p;
//      the v scale is folded into the probability before its bf16 rounding: pb = bf16(p * vscale)
//   C  thread (4 d = tid % 32, token group = warp): o_g[d] = o_g[d] * alpha + sum_r pb_g[r] * float(vcode[r, d])
//      over tokens r = warp, warp + 8, ...; the 8 token groups are added in order after the last chunk.
// K / V are read with plain L2 loads: the CTA that holds `pos` writes the new row first and reads it back.
template <int G>
__global__ void __launch_bounds__(kFaThreads, G <= 8 ? 2 : 1) decode_attn_fp8_kernel(DecodeAttnFp8Params p) {
  constexpr int D = 128;
  constexpr int GP = (G + 3) & ~3;  // pb_s row width (float4 reads)
  extern __shared__ __align__(16) float fa_smem[];
  float* q_s = fa_smem;                        // [G][2][kQPad]
  float* sc_s = q_s + G * 2 * kQPad;           // [G][128] scores (log2 domain)
  float* pb_s = sc_s + G * kFaChunk;           // [128][GP] bf16-rounded, v-scaled probabilities
  float* vs_s = pb_s + kFaChunk * GP;          // [128] v scales of the chunk
  float* red = vs_s + kFaChunk;                // [8][G][128] token-group partials
  __shared__ float m_s[G], l_s[G], alpha_s[G];
  __shared__ int pages_s[kFaMaxSplitPages];
  __shared__ __align__(16) __nv_bfloat16 knew_s[D];
  __shared__ int is_last_s;

  const int split = blockIdx.x, hk = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int t0 = split * p.split_tokens;
  const int npg = p.split_tokens / kFaChunk;
  const int32_t* pt = p.page_table + static_cast<int64_t>(b) * p.pt_stride;
  if (tid < npg && (t0 >> 7) + tid < p.pt_stride) pages_s[tid] = pt[(t0 >> 7) + tid];  // static: before the wait
  griddep_launch_dependents();
  griddep_wait();
  const int pos = p.position[b];
  if (pos < 0 || t0 > pos) return;  // idle slot, or a split past the slot's length (block-uniform)
  const int t1 = min(pos + 1, t0 + p.split_tokens);
  const int n_used = min(pos / p.split_tokens + 1, static_cast<int>(gridDim.x));
  const __nv_bfloat16* qkv = p.qkv + static_cast<int64_t>(b) * p.qkv_stride;

  // ---- RoPE on the G query heads (and on the new key in the CTA that holds pos) ----
  const bool owner = pos < t1;
  for (int idx = tid; idx < (G + 1) * (D / 2); idx += kFaThreads) {
    const int hh = idx / (D / 2), i = idx % (D / 2);
    if (hh == G && !owner) break;
    const __nv_bfloat16* src = hh < G ? qkv + (hk * G + hh) * D : qkv + (p.Hq + hk) * D;
    const float x0 = __bfloat162float(src[i]), x1 = __bfloat162float(src[i + D / 2]);
    float sn, cs;
    sincosf((float)pos * p.inv_freq[i], &sn, &cs);
    cs = bf16_round(cs);
    sn = bf16_round(sn);
    const float y0 = bf16_round(bf16_round(x0 * cs) + bf16_round(-x1 * sn));
    const float y1 = bf16_round(bf16_round(x1 * cs) + bf16_round(x0 * sn));
    if (hh < G) {
      q_s[hh * 2 * kQPad + i] = y0;
      q_s[hh * 2 * kQPad + kQPad + i] = y1;
    } else {
      knew_s[i] = __float2bfloat16(y0);
      knew_s[i + D / 2] = __float2bfloat16(y1);
    }
  }
  if (tid < G) {
    m_s[tid] = -INFINITY;
    l_s[tid] = 0.f;
  }
  __syncthreads();
  if (owner && warp < 2) {  // e4m3 append of the new row: warp 0 K, warp 1 V
    float x[4];
    if (warp == 0) {
      const uint2 v = *reinterpret_cast<const uint2*>(knew_s + lane * 4);
      x[0] = bf_lo(v.x); x[1] = bf_hi(v.x); x[2] = bf_lo(v.y); x[3] = bf_hi(v.y);
    } else {
      const uint2 v = *reinterpret_cast<const uint2*>(qkv + (p.Hq + p.Hkv + hk) * D + lane * 4);
      x[0] = bf_lo(v.x); x[1] = bf_hi(v.x); x[2] = bf_lo(v.y); x[3] = bf_hi(v.y);
    }
    float scale;
    const uint32_t codes = quantize_row_warp(x, &scale);
    const int64_t row = (static_cast<int64_t>(pages_s[(pos - t0) >> 7]) * 128 + (pos & 127)) * p.Hkv + hk;
    reinterpret_cast<uint32_t*>((warp == 0 ? p.k_pool : p.v_pool) + row * D)[lane] = codes;
    if (lane == 0) (warp == 0 ? p.k_scale : p.v_scale)[row] = scale;
  }
  __syncthreads();  // the new row is visible to the loads below

  const float sl2 = p.scale * 1.4426950408889634f;
  const int ra = tid >> 1, half = tid & 1;  // phase A: token, d half
  const int dq = lane;                      // phase C: d quad, token group = warp
  float acc[G][4];
#pragma unroll
  for (int g = 0; g < G; ++g)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[g][e] = 0.f;

  for (int c0 = t0; c0 < t1; c0 += kFaChunk) {
    const int n = min(kFaChunk, t1 - c0);
    const int64_t prow = static_cast<int64_t>(pages_s[(c0 - t0) >> 7]) * 128 * p.Hkv + hk;  // row of token 0
    // ---- this thread's K half-row ----
    uint4 kr[4];
    float ks = 0.f;
    if (ra < n) {
      const uint4* src = reinterpret_cast<const uint4*>(p.k_pool + (prow + static_cast<int64_t>(ra) * p.Hkv) * D + half * 64);
#pragma unroll
      for (int c = 0; c < 4; ++c) kr[c] = __ldcg(src + c);
      if (half == 0) {
        ks = __ldcg(p.k_scale + prow + static_cast<int64_t>(ra) * p.Hkv);
        vs_s[ra] = __ldcg(p.v_scale + prow + static_cast<int64_t>(ra) * p.Hkv);
      }
    } else {
#pragma unroll
      for (int c = 0; c < 4; ++c) kr[c] = make_uint4(0, 0, 0, 0);
      if (half == 0) vs_s[ra] = 0.f;
    }
    // ---- A: scores ----
    float s[G];
#pragma unroll
    for (int g = 0; g < G; ++g) s[g] = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const uint32_t w4[4] = {kr[c].x, kr[c].y, kr[c].z, kr[c].w};
#pragma unroll
      for (int wi = 0; wi < 4; ++wi) {
        float f[4];
        e4m3x4_to_float(w4[wi], f);
#pragma unroll
        for (int g = 0; g < G; ++g) {
          const float4 q4 = *reinterpret_cast<const float4*>(q_s + g * 2 * kQPad + half * kQPad + c * 16 + wi * 4);
          s[g] = fmaf(q4.x, f[0], s[g]);
          s[g] = fmaf(q4.y, f[1], s[g]);
          s[g] = fmaf(q4.z, f[2], s[g]);
          s[g] = fmaf(q4.w, f[3], s[g]);
        }
      }
    }
#pragma unroll
    for (int g = 0; g < G; ++g) {
      s[g] += __shfl_xor_sync(0xffffffffu, s[g], 1);
      if (half == 0) sc_s[g * kFaChunk + ra] = ra < n ? (s[g] * ks) * sl2 : -INFINITY;
    }
    // V words of this thread's token group, in flight during the softmax: the first kVPre of its 16 tokens, the
    // rest loaded in C.  Fewer for G > 12, whose accumulators leave no room for all 16 without spilling.
    constexpr int kVPre = G > 14 ? 4 : G > 12 ? 8 : kFaChunk / kFaWarps;
    auto v_word = [&](int r) {
      return __ldcg(reinterpret_cast<const uint32_t*>(p.v_pool + (prow + static_cast<int64_t>(r) * p.Hkv) * D) + dq);
    };
    uint32_t vw[kVPre];
#pragma unroll
    for (int i = 0; i < kVPre; ++i) {
      const int r = warp + kFaWarps * i;
      vw[i] = r < n ? v_word(r) : 0u;
    }
    __syncthreads();
    // ---- B: online softmax, one warp per head ----
    for (int g = warp; g < G; g += kFaWarps) {
      float v[4], cm = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        v[j] = sc_s[g * kFaChunk + lane + 32 * j];
        cm = fmaxf(cm, v[j]);
      }
      cm = warp_max(cm);
      const float m_old = m_s[g];
      const float m_new = fmaxf(m_old, cm);
      const float alpha = exp2f(m_old - m_new);  // m_old == -inf -> 0
      float ps = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int r = lane + 32 * j;
        const float pe = exp2f(v[j] - m_new);  // -inf (past the chunk's tokens) -> 0
        ps += pe;
        pb_s[r * GP + g] = bf16_round(pe * vs_s[r]);
      }
      ps = warp_sum(ps);
      __syncwarp();
      if (lane == 0) {
        l_s[g] = l_s[g] * alpha + ps;
        m_s[g] = m_new;
        alpha_s[g] = alpha;
      }
    }
    __syncthreads();
    // ---- C: P.V ----
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const float al = alpha_s[g];
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[g][e] *= al;
    }
#pragma unroll
    for (int i = 0; i < kFaChunk / kFaWarps; ++i) {
      const int r = warp + kFaWarps * i;
      if (r < n) {  // warp-uniform
        float f[4];
        e4m3x4_to_float(i < kVPre ? vw[i] : v_word(r), f);
        float pb[GP];
#pragma unroll
        for (int g4 = 0; g4 < GP; g4 += 4) {
          const float4 t = *reinterpret_cast<const float4*>(pb_s + r * GP + g4);
          pb[g4] = t.x; pb[g4 + 1] = t.y; pb[g4 + 2] = t.z; pb[g4 + 3] = t.w;
        }
#pragma unroll
        for (int g = 0; g < G; ++g)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[g][e] = fmaf(pb[g], f[e], acc[g][e]);
      }
    }
  }

  // ---- the split's result: token groups added in order ----
#pragma unroll
  for (int g = 0; g < G; ++g)
    *reinterpret_cast<float4*>(red + (warp * G + g) * D + dq * 4) = make_float4(acc[g][0], acc[g][1], acc[g][2], acc[g][3]);
  __syncthreads();
  __nv_bfloat16* out = p.out + static_cast<int64_t>(b) * p.out_stride + hk * G * D;
  const size_t blk = static_cast<size_t>(G) * (D + 2);  // one split's record: o [G][D], m [G], l [G]
  float* ws = p.ws + (static_cast<size_t>(b) * p.Hkv + hk) * gridDim.x * blk;
  for (int idx = tid; idx < G * D; idx += kFaThreads) {
    const int g = idx / D, d = idx % D;
    float o = 0.f;
#pragma unroll
    for (int w = 0; w < kFaWarps; ++w) o += red[(w * G + g) * D + d];
    if (n_used == 1) {
      out[idx] = __float2bfloat16(o / l_s[g]);
    } else {
      float* rec = ws + split * blk;
      rec[idx] = o;
      if (d == 0) {
        rec[G * D + g] = m_s[g];
        rec[G * D + G + g] = l_s[g];
      }
    }
  }
  if (n_used == 1) return;
  __threadfence();
  __syncthreads();
  int32_t* counter = p.counters + b * p.Hkv + hk;
  if (tid == 0) {
    const int prev = atomicAdd(counter, 1);
    is_last_s = prev == n_used - 1;
    if (is_last_s) *counter = 0;  // re-armed for the next launch (CUDA-graph replay)
  }
  __syncthreads();
  if (!is_last_s) return;
  __threadfence();
  for (int idx = tid; idx < G * D; idx += kFaThreads) {
    const int g = idx / D;
    float mm = -INFINITY;
    for (int sp = 0; sp < n_used; ++sp) mm = fmaxf(mm, __ldcg(ws + sp * blk + G * D + g));
    float ll = 0.f, oo = 0.f;
    for (int sp = 0; sp < n_used; ++sp) {
      const float* rec = ws + sp * blk;
      const float w = exp2f(__ldcg(rec + G * D + g) - mm);
      ll += __ldcg(rec + G * D + G + g) * w;
      oo += __ldcg(rec + idx) * w;
    }
    out[idx] = __float2bfloat16(oo / ll);
  }
}

template <int G>
size_t fa_smem_bytes() {
  constexpr int GP = (G + 3) & ~3;
  return sizeof(float) * (G * 2 * kQPad + G * kFaChunk + kFaChunk * GP + kFaChunk + kFaWarps * G * 128);
}

template <int G>
int launch_fa(const DecodeAttnFp8Params& p, cudaStream_t stream) {
  auto kern = decode_attn_fp8_kernel<G>;
  const size_t smem = fa_smem_bytes<G>();
  static PerDeviceOnce attr_once;
  if (attr_once.first()) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  VB_CUDA(launch_pdl(kern, dim3(p.num_splits, p.Hkv, p.batch), dim3(kFaThreads), smem, stream, p));
  return 0;
}

}  // namespace

int kv_quantize_fp8(const __nv_bfloat16* src, int64_t src_tokens, uint8_t* dst, float* dst_scale, int64_t dst_pages,
                    const int32_t* page_table, int pt_len, int L, int Hkv, int D, int S, cudaStream_t stream) {
  VB_CHECK(D == 128, "kv_quantize_fp8: head_dim must be 128 (got %d)", D);
  VB_CHECK(src && dst && dst_scale && page_table, "kv_quantize_fp8: src, dst, dst_scale and page_table are required");
  VB_CHECK((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0 &&
               (reinterpret_cast<uintptr_t>(dst_scale) & 3) == 0 && (reinterpret_cast<uintptr_t>(page_table) & 3) == 0,
           "kv_quantize_fp8: misaligned pointer (src and dst 16-byte, dst_scale and page_table 4-byte)");
  VB_CHECK(L >= 1 && Hkv >= 1 && dst_pages >= 1, "kv_quantize_fp8: bad shape L=%d Hkv=%d pages=%lld", L, Hkv,
           (long long)dst_pages);
  VB_CHECK(S >= 0 && S <= src_tokens && (S + 127) / 128 <= pt_len,
           "kv_quantize_fp8: S=%d exceeds the staging cache (%lld tokens) or the page-table row (%d pages)", S,
           (long long)src_tokens, pt_len);
  if (S == 0) return 0;
  KvQuantArgs a{src, src_tokens, dst, dst_scale, dst_pages, page_table, L, Hkv, S};
  const int64_t rows = static_cast<int64_t>(L) * 2 * S * Hkv;
  const int64_t blocks = (rows + 7) / 8;
  VB_CHECK(blocks <= 0x7fffffffLL, "kv_quantize_fp8: too many rows (%lld)", (long long)rows);
  VB_CUDA(launch_pdl(kv_quantize_kernel, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, stream, a));
  return 0;
}

int decode_attention_fp8_batch(const DecodeAttnFp8Params& p, cudaStream_t stream) {
  VB_CHECK(p.D == 128, "decode_attention_fp8_batch: head_dim must be 128 (got %d)", p.D);
  VB_CHECK(p.Hq >= 1 && p.Hkv >= 1 && p.Hq % p.Hkv == 0, "decode_attention_fp8_batch: Hq %d is not a multiple of Hkv %d",
           p.Hq, p.Hkv);
  const int G = p.Hq / p.Hkv;
  VB_CHECK(G <= 16, "decode_attention_fp8_batch: at most 16 query heads per KV head (got %d)", G);
  VB_CHECK(p.qkv && p.position && p.k_pool && p.v_pool && p.k_scale && p.v_scale && p.page_table && p.out && p.ws &&
               p.counters && p.inv_freq,
           "decode_attention_fp8_batch: every pointer is required");
  VB_CHECK((reinterpret_cast<uintptr_t>(p.qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.k_pool) & 15) == 0 &&
               (reinterpret_cast<uintptr_t>(p.v_pool) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.out) & 3) == 0,
           "decode_attention_fp8_batch: misaligned qkv / pools (16-byte) or out (4-byte)");
  VB_CHECK(p.batch >= 1 && p.batch <= 65535, "decode_attention_fp8_batch: bad batch %d", p.batch);
  VB_CHECK(p.qkv_stride >= (p.Hq + 2 * p.Hkv) * p.D && p.qkv_stride % 8 == 0 && p.out_stride >= p.Hq * p.D &&
               p.out_stride % 2 == 0 && p.pt_stride >= 1,
           "decode_attention_fp8_batch: bad strides (qkv %d, out %d, page table %d)", p.qkv_stride, p.out_stride,
           p.pt_stride);
  VB_CHECK(p.split_tokens >= kFaChunk && p.split_tokens % kFaChunk == 0 &&
               p.split_tokens <= kFaMaxSplitPages * kFaChunk && p.num_splits >= 1 && p.num_splits <= 65535,
           "decode_attention_fp8_batch: bad split configuration (%d x %d; split_tokens a multiple of 128, <= %d)",
           p.num_splits, p.split_tokens, kFaMaxSplitPages * kFaChunk);
  switch (G) {
#define VB_FA_CASE(GG) \
  case GG:             \
    return launch_fa<GG>(p, stream);
    VB_FA_CASE(1) VB_FA_CASE(2) VB_FA_CASE(3) VB_FA_CASE(4) VB_FA_CASE(5) VB_FA_CASE(6) VB_FA_CASE(7) VB_FA_CASE(8)
    VB_FA_CASE(9) VB_FA_CASE(10) VB_FA_CASE(11) VB_FA_CASE(12) VB_FA_CASE(13) VB_FA_CASE(14) VB_FA_CASE(15)
    VB_FA_CASE(16)
#undef VB_FA_CASE
  }
  return 1;  // unreachable: 1 <= G <= 16
}

}  // namespace vb
