// Decode-time (one new token, batch 1) kernels: everything is HBM-bound weight / KV streaming.
//
//  gemv_kernel       y = W x (+bias)(+residual)(SwiGLU)(argmax) with a fused RMSNorm prologue.
//                    One CTA per SM, 16 warps; each warp streams whole (row, k-part) items with
//                    UNROLL independent 128-bit loads in flight per lane; x lives in shared memory.
//                    Replaces cuBLAS GEMV behind nn.Linear + ATen RMSNorm/SiLU/mul/add/argmax
//                    (modeling_qwen2.py:81-95,164-176,223-226 ; HF lm_head + greedy argmax).
//  decode_attn_kernel  split-KV paged attention for GQA (7 query heads share one KV head), with
//                    RoPE of q / new k and the KV append fused in (replaces apply_rotary_pos_emb,
//                    DynamicCache.update (torch.cat) and flash_attn decode).
#include <cooperative_groups.h>
#include <math.h>

#include "common.cuh"
#include "kernels.h"

namespace vb {
namespace {

constexpr int kGemvThreads = 512;
constexpr int kGemvWarps = kGemvThreads / 32;
constexpr size_t kGemvPrefetchBytes = 256 * 1024;  // per-CTA L2 prefetch before the PDL wait


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

// order-preserving float -> uint32 map (for atomicMax on packed keys)
__device__ __forceinline__ uint32_t float_order(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

template <int UNROLL>
__global__ void __launch_bounds__(kGemvThreads, 2)
gemv_kernel(GemvParams p, int rows_per_block, int ksplit) {
  extern __shared__ uint4 smem_v[];
  uint4* xs = smem_v;                                              // K/8 vectors (bf16 x)
  float* acc = reinterpret_cast<float*>(xs + ((p.K + 7) >> 3));    // rows_per_block floats
  __shared__ float red[32];
  __shared__ unsigned long long best_s;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row0 = blockIdx.x * rows_per_block;
  const int nrows = min(rows_per_block, p.N - row0);
  if (nrows <= 0) return;
  const int nvec = p.K >> 3;

  // ---- PDL prologue: let the next kernel become resident, and pull the head of this CTA's
  // (static) weight slab into L2 while the predecessor kernel is still draining ----
  griddep_launch_dependents();
  if (p.flags & 2) {
    const char* slab = reinterpret_cast<const char*>(p.w + static_cast<size_t>(row0) * p.K);
    const size_t slab_bytes = static_cast<size_t>(nrows) * p.K * 2;
    const size_t cap = slab_bytes < kGemvPrefetchBytes ? slab_bytes : kGemvPrefetchBytes;
    for (size_t off = static_cast<size_t>(threadIdx.x) * 2048; off < cap;
         off += static_cast<size_t>(kGemvThreads) * 2048) {
      const size_t n = cap - off < 2048 ? cap - off : 2048;
      prefetch_l2_bulk(slab + off, static_cast<uint32_t>(n & ~static_cast<size_t>(15)));
    }
  }
  griddep_wait();

  // ---- prologue: stage x (optionally RMS-normalised) in shared memory ----
  const uint4* xg = reinterpret_cast<const uint4*>(p.x);
  if (p.norm_w != nullptr) {
    float s = 0.f;
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
      const uint4 v = ldg_v4(xg + i);
      xs[i] = v;
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
    float t = lane < kGemvWarps ? red[lane] : 0.f;
    t = warp_sum(t);
    const float rstd = rsqrtf(t / p.K + p.norm_eps);
    const uint4* wv = reinterpret_cast<const uint4*>(p.norm_w);
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
      const uint4 v = xs[i], g = ldg_v4(wv + i);
      uint4 o;
      o.x = pack_bf16(bf16_round(bf_lo(v.x) * rstd) * bf_lo(g.x), bf16_round(bf_hi(v.x) * rstd) * bf_hi(g.x));
      o.y = pack_bf16(bf16_round(bf_lo(v.y) * rstd) * bf_lo(g.y), bf16_round(bf_hi(v.y) * rstd) * bf_hi(g.y));
      o.z = pack_bf16(bf16_round(bf_lo(v.z) * rstd) * bf_lo(g.z), bf16_round(bf_hi(v.z) * rstd) * bf_hi(g.z));
      o.w = pack_bf16(bf16_round(bf_lo(v.w) * rstd) * bf_lo(g.w), bf16_round(bf_hi(v.w) * rstd) * bf_hi(g.w));
      xs[i] = o;
    }
  } else {
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) xs[i] = ldg_v4(xg + i);
  }
  if (threadIdx.x == 0) best_s = 0ull;
  __syncthreads();

  // ---- main loop: this warp's (row, k-part) items form ONE flat stream of 512-byte row chunks;
  // UNROLL independent 128-bit loads per lane stay in flight across item boundaries.  Item/chunk
  // indices advance incrementally (no divisions on the load path).  Partial sums of the k-parts of a
  // row go to separate slots and are added in a fixed order (deterministic). ----
  const int nchunks = (nvec + 31) >> 5;             // 32 vectors (256 elements) per chunk
  const int cpi = (nchunks + ksplit - 1) / ksplit;  // chunks per item
  const int items = nrows * ksplit;
  {
    int item = warp;                 // item being LOADED
    int ch = 0;                      // chunk of that item
    int r = item / ksplit, part = item - r * ksplit;
    const uint4* wrow = reinterpret_cast<const uint4*>(p.w + static_cast<size_t>(row0 + r) * p.K);
    int vbase = part * cpi * 32 + lane;
    float sum = 0.f;
    while (item < items) {
      uint4 wv[UNROLL];
      int xo[UNROLL];    // smem vector index of the matching x chunk, -1: nothing loaded
      int fin[UNROLL];   // >= 0: this chunk closes an item -> slot index to publish
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const bool live = item < items;
        const int vi = vbase + ch * 32;
        const bool ok = live && vi < nvec;
        xo[u] = ok ? vi : -1;
        wv[u] = ok ? ldg_stream(wrow + vi) : make_uint4(0, 0, 0, 0);
        fin[u] = (live && ch == cpi - 1) ? item : -1;
        if (live) {
          if (++ch == cpi) {
            ch = 0;
            item += kGemvWarps;
            if (item < items) {
              r = item / ksplit;
              part = item - r * ksplit;
              wrow = reinterpret_cast<const uint4*>(p.w + static_cast<size_t>(row0 + r) * p.K);
              vbase = part * cpi * 32 + lane;
            }
          }
        }
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        if (xo[u] >= 0) sum = dot8(wv[u], xs[xo[u]], sum);
        if (fin[u] >= 0) {  // warp-uniform
          const float tot = warp_sum(sum);
          sum = 0.f;
          if (lane == 0) acc[fin[u]] = tot;  // slot = row * ksplit + part
        }
      }
    }
  }
  __syncthreads();
  if (ksplit > 1) {  // fixed-order reduction of the k-parts
    float tot[4];
    int nmine = 0;
    for (int i = threadIdx.x; i < nrows; i += blockDim.x) {
      float t = 0.f;
      for (int q = 0; q < ksplit; ++q) t += acc[i * ksplit + q];
      if (nmine < 4) tot[nmine] = t;
      ++nmine;
    }
    __syncthreads();
    nmine = 0;
    for (int i = threadIdx.x; i < nrows; i += blockDim.x) {
      if (nmine < 4) acc[i] = tot[nmine];
      ++nmine;
    }
    __syncthreads();
  }

  // ---- epilogue ----
  if (p.flags & 1) {
    for (int j = threadIdx.x; j < (nrows >> 1); j += blockDim.x) {
      float g = acc[2 * j], u = acc[2 * j + 1];
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
    if (lane == 0) atomicMax(&best_s, best);
    __syncthreads();
    if (threadIdx.x == 0) atomicMax(p.argmax_key, best_s);
  }
}

// token = argmax; append to history; bump position / step; fetch the token's embedding as the next x.
__global__ void argmax_finalize_kernel(unsigned long long* key, int32_t* token_out,
                                       int32_t* token_hist, int32_t* step_counter,
                                       int32_t* position, const uint4* __restrict__ embed_table,
                                       uint4* __restrict__ x_next, int hidden_vec) {
  __shared__ int32_t tok_s;
  griddep_launch_dependents();
  griddep_wait();
  if (threadIdx.x == 0) {
    const unsigned long long k = *key;
    const int32_t tok = static_cast<int32_t>(0xffffffffu - static_cast<uint32_t>(k & 0xffffffffull));
    *token_out = tok;
    if (token_hist && step_counter) {
      const int32_t st = *step_counter;
      token_hist[st] = tok;
      *step_counter = st + 1;
    }
    if (position) *position = *position + 1;
    *key = 0ull;
    tok_s = tok;
  }
  __syncthreads();
  if (embed_table != nullptr && x_next != nullptr) {
    const uint4* src = embed_table + static_cast<size_t>(tok_s) * hidden_vec;
    for (int i = threadIdx.x; i < hidden_vec; i += blockDim.x) x_next[i] = src[i];
  }
}

// ------------------------------------------------------------------------------------------------
// decode attention
// ------------------------------------------------------------------------------------------------
constexpr int kDaThreads = 256;
constexpr int kDaWarps = 8;
constexpr int kMaxG = 8;  // query heads per kv head

template <int D, int G, bool kCluster>
__global__ void __launch_bounds__(kDaThreads)
decode_attn_kernel(vila_decode_attn_params p) {
  const float* __restrict__ inv_freq = p.inv_freq;
  __nv_bfloat16* qkv = static_cast<__nv_bfloat16*>(p.qkv);
  __nv_bfloat16* k_pool = static_cast<__nv_bfloat16*>(p.k_pool);
  __nv_bfloat16* v_pool = static_cast<__nv_bfloat16*>(p.v_pool);
  __nv_bfloat16* out = static_cast<__nv_bfloat16*>(p.out);
  static_assert(D == 128, "decode attention is specialised for head_dim 128");
  constexpr int VPT = 8;             // elements per lane (16 bytes)
  constexpr int LPT = D / VPT;       // lanes per token (16)
  const int hk = blockIdx.x, split = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sub = lane / LPT;        // which of the 2 tokens this half-warp handles
  const int dl = lane % LPT;         // d-slice index
  griddep_launch_dependents();
  griddep_wait();
  const int pos = *p.position;       // index of the new token == number of cached tokens
  const int n_tok = pos + 1;

  // ---- this split's token range; the first batch of K/V rows is requested BEFORE the RoPE
  // prologue so that its HBM latency overlaps the prologue (K/V do not depend on q) ----
  constexpr int TB = 4;  // tokens per half-warp per batch
  const int per = (n_tok + p.num_splits - 1) / p.num_splits;
  const int t0 = split * per, t1 = min(n_tok, t0 + per);
  const int hw = warp * 2 + sub;
  uint4 kreg[TB], vreg[TB];
  auto load_batch = [&](int base) {
#pragma unroll
    for (int i = 0; i < TB; ++i) {
      const int t = base + hw + 16 * i;
      kreg[i] = make_uint4(0, 0, 0, 0);
      vreg[i] = make_uint4(0, 0, 0, 0);
      if (t < t1 && t != pos) {
        const int page = p.page_table[t >> 7];
        const size_t o = ((static_cast<size_t>(page) * 128 + (t & 127)) * p.Hkv + hk) * D + dl * VPT;
        kreg[i] = ldg_v4(k_pool + o);
        vreg[i] = ldg_v4(v_pool + o);
      }
    }
  };
  load_batch(t0);

  __shared__ float q_s[G][D];
  __shared__ __align__(16) __nv_bfloat16 knew_s[D];
  __shared__ __align__(16) __nv_bfloat16 vnew_s[D];
  extern __shared__ float da_smem[];
  float (*red_o)[G][D] = reinterpret_cast<float (*)[G][D]>(da_smem);             // [16][G][D]
  float (*red_m)[G] = reinterpret_cast<float (*)[G]>(da_smem + kDaWarps * 2 * G * D);  // [16][G]
  float (*red_l)[G] = red_m + kDaWarps * 2;                                       // [16][G]
  __shared__ int is_last_s;

  // ---- RoPE on the G query heads and the new key; stage in smem ----
  const int Ht = p.Hq + 2 * p.Hkv;
  (void)Ht;
  for (int idx = threadIdx.x; idx < (G + 1) * (D / 2); idx += blockDim.x) {
    const int hh = idx / (D / 2), i = idx % (D / 2);
    const __nv_bfloat16* src =
        hh < G ? qkv + (hk * G + hh) * D : qkv + (p.Hq + hk) * D;
    const float x0 = __bfloat162float(src[i]), x1 = __bfloat162float(src[i + D / 2]);
    const float ang = (float)pos * inv_freq[i];
    float sn, cs;
    sincosf(ang, &sn, &cs);
    cs = bf16_round(cs);
    sn = bf16_round(sn);
    const float y0 = bf16_round(bf16_round(x0 * cs) + bf16_round(-x1 * sn));
    const float y1 = bf16_round(bf16_round(x1 * cs) + bf16_round(x0 * sn));
    if (hh < G) {
      q_s[hh][i] = y0;
      q_s[hh][i + D / 2] = y1;
    } else {
      knew_s[i] = __float2bfloat16(y0);
      knew_s[i + D / 2] = __float2bfloat16(y1);
    }
  }
  for (int i = threadIdx.x; i < D; i += blockDim.x) vnew_s[i] = qkv[(p.Hq + p.Hkv + hk) * D + i];
  __syncthreads();
  if (split == 0) {  // KV append (DynamicCache.update)
    const int page = p.page_table[pos >> 7];
    const size_t o = ((static_cast<size_t>(page) * 128 + (pos & 127)) * p.Hkv + hk) * D;
    for (int i = threadIdx.x; i < D; i += blockDim.x) {
      k_pool[o + i] = knew_s[i];
      v_pool[o + i] = vnew_s[i];
    }
  }

  float qreg[G][VPT];
#pragma unroll
  for (int g = 0; g < G; ++g)
#pragma unroll
    for (int e = 0; e < VPT; ++e) qreg[g][e] = q_s[g][dl * VPT + e];

  float m[G], l[G], o_acc[G][VPT];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    m[g] = -INFINITY;
    l[g] = 0.f;
#pragma unroll
    for (int e = 0; e < VPT; ++e) o_acc[g][e] = 0.f;
  }
  const float sl2 = p.scale * 1.4426950408889634f;

  for (int base = t0; base < t1; base += 16 * TB) {  // block-uniform trip count
    if (base != t0) load_batch(base);
#pragma unroll
    for (int i = 0; i < TB; ++i) {
      const int t = base + hw + 16 * i;
      const bool valid = t < t1;
      uint4 kv = kreg[i], vv = vreg[i];
      if (valid && t == pos) {
        kv = *reinterpret_cast<const uint4*>(knew_s + dl * VPT);
        vv = *reinterpret_cast<const uint4*>(vnew_s + dl * VPT);
      }
      const float kf[VPT] = {bf_lo(kv.x), bf_hi(kv.x), bf_lo(kv.y), bf_hi(kv.y),
                             bf_lo(kv.z), bf_hi(kv.z), bf_lo(kv.w), bf_hi(kv.w)};
      const float vf[VPT] = {bf_lo(vv.x), bf_hi(vv.x), bf_lo(vv.y), bf_hi(vv.y),
                             bf_lo(vv.z), bf_hi(vv.z), bf_lo(vv.w), bf_hi(vv.w)};
#pragma unroll
      for (int g = 0; g < G; ++g) {
        float s = 0.f;
#pragma unroll
        for (int e = 0; e < VPT; ++e) s = fmaf(qreg[g][e], kf[e], s);
        // reduce over the 16 lanes of this half-warp
#pragma unroll
        for (int o = LPT / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (valid) {
          s *= sl2;
          const float m_new = fmaxf(m[g], s);
          const float alpha = exp2f(m[g] - m_new);  // m == -inf -> 0
          const float pexp = exp2f(s - m_new);
          l[g] = l[g] * alpha + pexp;
          // the reference's attention kernels cast probabilities to bf16 before P.V
          const float pb = bf16_round(pexp);
#pragma unroll
          for (int e = 0; e < VPT; ++e) o_acc[g][e] = o_acc[g][e] * alpha + pb * vf[e];
          m[g] = m_new;
        }
      }
    }
  }

  // ---- block combine: 16 half-warp partials per head ----
  const int slot = hw;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    if (dl == 0) {
      red_m[slot][g] = m[g];
      red_l[slot][g] = l[g];
    }
#pragma unroll
    for (int e = 0; e < VPT; ++e) red_o[slot][g][dl * VPT + e] = o_acc[g][e];
  }
  __syncthreads();
  // ---- cross-split combine ----
  if constexpr (kCluster) {
    // All splits of this KV head form one thread-block cluster: block partials stay in shared
    // memory and are combined through DSMEM (no global workspace / atomics / fences).
    namespace cg = cooperative_groups;
    __shared__ float part_m[G], part_l[G];
    __shared__ float part_o[G][D];
    for (int idx = threadIdx.x; idx < G * D; idx += blockDim.x) {
      const int g = idx / D, d = idx % D;
      float mm = -INFINITY;
      for (int s = 0; s < kDaWarps * 2; ++s) mm = fmaxf(mm, red_m[s][g]);
      float ll = 0.f, oo = 0.f;
      for (int s = 0; s < kDaWarps * 2; ++s) {
        const float w = (red_m[s][g] == -INFINITY) ? 0.f : exp2f(red_m[s][g] - mm);
        ll += red_l[s][g] * w;
        oo += red_o[s][g][d] * w;
      }
      if (d == 0) {
        part_m[g] = mm;
        part_l[g] = ll;
      }
      part_o[g][d] = oo;
    }
    cg::cluster_group cluster = cg::this_cluster();
    cluster.sync();
    const int nr = static_cast<int>(cluster.num_blocks());
    const int rank = static_cast<int>(cluster.block_rank());
    for (int idx = rank * blockDim.x + threadIdx.x; idx < G * D; idx += nr * blockDim.x) {
      const int g = idx / D, d = idx % D;
      float mm = -INFINITY;
      for (int s = 0; s < nr; ++s) mm = fmaxf(mm, cluster.map_shared_rank(&part_m[0], s)[g]);
      float ll = 0.f, oo = 0.f;
      for (int s = 0; s < nr; ++s) {
        const float ms = cluster.map_shared_rank(&part_m[0], s)[g];
        const float w = (ms == -INFINITY) ? 0.f : exp2f(ms - mm);
        ll += cluster.map_shared_rank(&part_l[0], s)[g] * w;
        oo += cluster.map_shared_rank(&part_o[0][0], s)[g * D + d] * w;
      }
      out[(hk * G + g) * D + d] = __float2bfloat16(oo / ll);
    }
    cluster.sync();  // peers may still be reading this CTA's shared memory
    return;
  }
  // thread -> (g, d) pairs
  float* ws_m = p.ws;                                             // [Hkv][splits][G]
  float* ws_l = ws_m + p.Hkv * p.num_splits * G;                  // [Hkv][splits][G]
  float* ws_o = ws_l + p.Hkv * p.num_splits * G;                  // [Hkv][splits][G][D]
  for (int idx = threadIdx.x; idx < G * D; idx += blockDim.x) {
    const int g = idx / D, d = idx % D;
    float mm = -INFINITY;
    for (int s = 0; s < kDaWarps * 2; ++s) mm = fmaxf(mm, red_m[s][g]);
    float ll = 0.f, oo = 0.f;
    for (int s = 0; s < kDaWarps * 2; ++s) {
      const float w = (red_m[s][g] == -INFINITY) ? 0.f : exp2f(red_m[s][g] - mm);
      ll += red_l[s][g] * w;
      oo += red_o[s][g][d] * w;
    }
    const size_t base = (static_cast<size_t>(hk) * p.num_splits + split) * G + g;
    if (d == 0) {
      ws_m[base] = mm;
      ws_l[base] = ll;
    }
    ws_o[base * D + d] = oo;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int prev = atomicAdd(&p.counters[hk], 1);
    is_last_s = (prev == p.num_splits - 1);
    if (is_last_s) p.counters[hk] = 0;  // re-arm for the next launch (CUDA-graph replay)
  }
  __syncthreads();
  if (!is_last_s) return;
  __threadfence();
  for (int idx = threadIdx.x; idx < G * D; idx += blockDim.x) {
    const int g = idx / D, d = idx % D;
    float mm = -INFINITY;
    for (int s = 0; s < p.num_splits; ++s)
      mm = fmaxf(mm, ws_m[(static_cast<size_t>(hk) * p.num_splits + s) * G + g]);
    float ll = 0.f, oo = 0.f;
    for (int s = 0; s < p.num_splits; ++s) {
      const size_t base = (static_cast<size_t>(hk) * p.num_splits + s) * G + g;
      const float ms = ws_m[base];
      const float w = (ms == -INFINITY) ? 0.f : exp2f(ms - mm);
      ll += ws_l[base] * w;
      oo += ws_o[base * D + d] * w;
    }
    out[(hk * G + g) * D + d] = __float2bfloat16(oo / ll);
  }
}


// ------------------------------------------------------------------------------------------------
// decode attention, short contexts (<= 1024 cached tokens): ONE CTA per QUERY head over all tokens.
// At the headline context (~300-400 tokens) the whole K/V of a layer is 0.6 MB: the op is a pure
// latency chain, and the split-KV kernel above spends most of it combining partials (shared-memory
// combine of 16 half-warps x 7 heads, two cluster barriers and a DSMEM pass).  Here a CTA owns one
// query head: no cross-CTA combine, no cluster launch; the 7 heads of a GQA group re-read the same
// K/V rows (L2 hits).  Token batches are register double-buffered so one L2 latency is exposed, not
// one per batch; the page table (static across decode steps) is fetched before the PDL wait.
// Same arithmetic as decode_attn_kernel (RoPE rounding points, bf16 probabilities, fp32 combine).
// ------------------------------------------------------------------------------------------------
constexpr int kDhThreads = 256;
constexpr int kDhMaxPages = 32;  // <= 4096 tokens per sequence

// Batched form (continuous batching over ONE shared paged pool, vila_b200/serving.py): blockIdx.y is
// the sequence; each has its own row of qkv / out, its own position and its own page-table row.
// positions[b] < 0 marks an idle slot (the CTA exits).  The single-sequence entry point is batch 1.
// The kernel reads vila_decode_attn_params through typed pointers, in a struct of the same layout filled by
// head_args(): offsetting the C-ABI struct's void pointers inside the kernel compiles to different code.
struct DecodeAttnHeadParams {
  __nv_bfloat16* qkv;
  const int32_t* position;
  __nv_bfloat16* k_pool;
  __nv_bfloat16* v_pool;
  const int32_t* page_table;
  __nv_bfloat16* out;
  float* ws;
  int32_t* counters;
  const float* inv_freq;
  int Hq, Hkv, D, num_splits;
  float scale;
};
struct DecodeAttnBatchArgs {
  DecodeAttnHeadParams p;  // qkv / out / position / page_table point at sequence 0
  int batch;
  int qkv_stride, out_stride, pt_stride;  // elements between consecutive sequences
  int max_pages;                          // valid entries per page-table row (<= kDhMaxPages)
};

template <int D, int TB>
__global__ void __launch_bounds__(kDhThreads)
decode_attn_head_kernel(DecodeAttnBatchArgs args) {
  static_assert(D == 128, "head_dim 128");
  constexpr int VPT = 8, LPT = D / VPT;
  DecodeAttnHeadParams p = args.p;
  {
    const int b = blockIdx.y;
    p.qkv += static_cast<size_t>(b) * args.qkv_stride;
    p.out += static_cast<size_t>(b) * args.out_stride;
    p.position += b;
    p.page_table += static_cast<size_t>(b) * args.pt_stride;
  }
  const int h = blockIdx.x;
  const int ratio = p.Hq / p.Hkv;
  const int hk = h / ratio;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int sub = lane / LPT, dl = lane % LPT;
  const int hw = warp * 2 + sub;  // 16 half-warps, one token each per step

  __shared__ int pages_s[kDhMaxPages];
  __shared__ float q_s[D];
  __shared__ __align__(16) __nv_bfloat16 knew_s[D];
  __shared__ __align__(16) __nv_bfloat16 vnew_s[D];
  __shared__ float red_m[16], red_l[16];
  __shared__ float red_o[16][D];

  if (threadIdx.x < args.max_pages) pages_s[threadIdx.x] = p.page_table[threadIdx.x];  // static: before the wait
  griddep_launch_dependents();
  griddep_wait();
  const int pos = *p.position;
  if (pos < 0) return;  // idle slot (block-uniform)
  const int n_tok = pos + 1;
  __syncthreads();

  auto load_batch = [&](int base, uint4* kr, uint4* vr) {
#pragma unroll
    for (int i = 0; i < TB; ++i) {
      const int t = base + hw + 16 * i;
      kr[i] = make_uint4(0, 0, 0, 0);
      vr[i] = make_uint4(0, 0, 0, 0);
      if (t < n_tok && t != pos) {
        const size_t o = ((static_cast<size_t>(pages_s[t >> 7]) * 128 + (t & 127)) * p.Hkv + hk) * D + dl * VPT;
        kr[i] = ldg_v4(p.k_pool + o);
        vr[i] = ldg_v4(p.v_pool + o);
      }
    }
  };
  uint4 kA[TB], vA[TB], kB[TB], vB[TB];
  load_batch(0, kA, vA);

  // ---- RoPE of this query head and of the new key; stage in shared memory ----
  if (threadIdx.x < D) {
    const int i = threadIdx.x & (D / 2 - 1);
    const bool is_k = threadIdx.x >= D / 2;
    const __nv_bfloat16* src = is_k ? p.qkv + (p.Hq + hk) * D : p.qkv + h * D;
    const float x0 = __bfloat162float(src[i]), x1 = __bfloat162float(src[i + D / 2]);
    float sn, cs;
    sincosf((float)pos * p.inv_freq[i], &sn, &cs);
    cs = bf16_round(cs);
    sn = bf16_round(sn);
    const float y0 = bf16_round(bf16_round(x0 * cs) + bf16_round(-x1 * sn));
    const float y1 = bf16_round(bf16_round(x1 * cs) + bf16_round(x0 * sn));
    if (is_k) {
      knew_s[i] = __float2bfloat16(y0);
      knew_s[i + D / 2] = __float2bfloat16(y1);
    } else {
      q_s[i] = y0;
      q_s[i + D / 2] = y1;
    }
  } else {
    const int i = threadIdx.x - D;
    vnew_s[i] = p.qkv[(p.Hq + p.Hkv + hk) * D + i];
  }
  __syncthreads();
  if (h % ratio == 0) {  // KV append (DynamicCache.update), once per KV head
    const size_t o = ((static_cast<size_t>(pages_s[pos >> 7]) * 128 + (pos & 127)) * p.Hkv + hk) * D;
    if (threadIdx.x < D) p.k_pool[o + threadIdx.x] = knew_s[threadIdx.x];
    else p.v_pool[o + threadIdx.x - D] = vnew_s[threadIdx.x - D];
  }
  float qreg[VPT];
#pragma unroll
  for (int e = 0; e < VPT; ++e) qreg[e] = q_s[dl * VPT + e];

  float m = -INFINITY, l = 0.f, o_acc[VPT];
#pragma unroll
  for (int e = 0; e < VPT; ++e) o_acc[e] = 0.f;
  const float sl2 = p.scale * 1.4426950408889634f;

  auto consume = [&](int base, const uint4* kr, const uint4* vr) {
#pragma unroll
    for (int i = 0; i < TB; ++i) {
      const int t = base + hw + 16 * i;
      const bool valid = t < n_tok;
      uint4 kv = kr[i], vv = vr[i];
      if (valid && t == pos) {
        kv = *reinterpret_cast<const uint4*>(knew_s + dl * VPT);
        vv = *reinterpret_cast<const uint4*>(vnew_s + dl * VPT);
      }
      const float kf[VPT] = {bf_lo(kv.x), bf_hi(kv.x), bf_lo(kv.y), bf_hi(kv.y),
                             bf_lo(kv.z), bf_hi(kv.z), bf_lo(kv.w), bf_hi(kv.w)};
      const float vf[VPT] = {bf_lo(vv.x), bf_hi(vv.x), bf_lo(vv.y), bf_hi(vv.y),
                             bf_lo(vv.z), bf_hi(vv.z), bf_lo(vv.w), bf_hi(vv.w)};
      float sc = 0.f;
#pragma unroll
      for (int e = 0; e < VPT; ++e) sc = fmaf(qreg[e], kf[e], sc);
#pragma unroll
      for (int o = LPT / 2; o > 0; o >>= 1) sc += __shfl_xor_sync(0xffffffffu, sc, o);
      if (valid) {
        sc *= sl2;
        const float m_new = fmaxf(m, sc);
        const float alpha = exp2f(m - m_new);
        const float pexp = exp2f(sc - m_new);
        l = l * alpha + pexp;
        const float pb = bf16_round(pexp);  // probabilities are cast to bf16 before P.V
#pragma unroll
        for (int e = 0; e < VPT; ++e) o_acc[e] = o_acc[e] * alpha + pb * vf[e];
        m = m_new;
      }
    }
  };
  constexpr int STEP = 16 * TB;
  for (int base = 0; base < n_tok; base += 2 * STEP) {  // block-uniform trip count
    if (base + STEP < n_tok) load_batch(base + STEP, kB, vB);
    consume(base, kA, vA);
    if (base + STEP < n_tok) {
      if (base + 2 * STEP < n_tok) load_batch(base + 2 * STEP, kA, vA);
      consume(base + STEP, kB, vB);
    }
  }

  // ---- combine the 16 half-warp partials (fixed order) ----
  if (dl == 0) {
    red_m[hw] = m;
    red_l[hw] = l;
  }
#pragma unroll
  for (int e = 0; e < VPT; ++e) red_o[hw][dl * VPT + e] = o_acc[e];
  __syncthreads();
  if (threadIdx.x < D) {
    const int d = threadIdx.x;
    float mm = -INFINITY;
#pragma unroll
    for (int s = 0; s < 16; ++s) mm = fmaxf(mm, red_m[s]);
    float ll = 0.f, oo = 0.f;
#pragma unroll
    for (int s = 0; s < 16; ++s) {
      const float w = (red_m[s] == -INFINITY) ? 0.f : exp2f(red_m[s] - mm);
      ll += red_l[s] * w;
      oo += red_o[s][d] * w;
    }
    p.out[h * D + d] = __float2bfloat16(oo / ll);
  }
}

// ------------------------------------------------------------------------------------------------
// long-context decode attention: combine of the split-KV partials written by fmha_decode_split
// (wgmma FMHA kernel in split mode).  out[h, :] = sum_s w_s * O_s[h, :], w_s = 2^(lse_s - max) / sum.
// Splits are summed in index order (deterministic).
// ------------------------------------------------------------------------------------------------
// The split weights are computed once per CTA from lse values fetched in parallel, and the partial rows are
// fetched 16 at a time, instead of walking the splits three times with one dependent load per step (a
// chain of DRAM latencies).  Same summation order -> same result.
constexpr int kCombineMaxSplits = 256;
__global__ void decode_combine_kernel(const float* __restrict__ o_partial, const float* __restrict__ lse,
                                      __nv_bfloat16* __restrict__ out, int Hq, int D, int splits) {
  __shared__ float w_s[kCombineMaxSplits];
  griddep_launch_dependents();
  griddep_wait();
  const int h = blockIdx.x;  // query head (= kv head * G + g, the layout of the partials' [Hkv][G])
  for (int s = threadIdx.x; s < splits; s += blockDim.x) w_s[s] = __ldcg(lse + (long)s * Hq + h);
  __syncthreads();
  float mx = -INFINITY;
  for (int s = 0; s < splits; ++s) mx = fmaxf(mx, w_s[s]);
  __syncthreads();
  for (int s = threadIdx.x; s < splits; s += blockDim.x) {
    const float v = w_s[s];
    w_s[s] = (v == -INFINITY) ? 0.f : exp2f(v - mx);
  }
  __syncthreads();
  float den = 0.f;
  for (int s = 0; s < splits; ++s) den += w_s[s];
  const float inv = den > 0.f ? 1.f / den : 0.f;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float acc = 0.f;
    const float* src = o_partial + (long)h * D + d;
    for (int s0 = 0; s0 < splits; s0 += 16) {
      float o[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) o[j] = (s0 + j < splits) ? __ldcg(src + (long)(s0 + j) * Hq * D) : 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (s0 + j < splits) acc += w_s[s0 + j] * o[j];
    }
    out[(long)h * D + d] = __float2bfloat16(acc * inv);
  }
}

DecodeAttnBatchArgs head_args(const vila_decode_attn_params& p, int batch, int qkv_stride, int out_stride,
                              int pt_stride, int max_pages) {
  using bf = __nv_bfloat16;
  return {{static_cast<bf*>(p.qkv), p.position, static_cast<bf*>(p.k_pool), static_cast<bf*>(p.v_pool), p.page_table,
           static_cast<bf*>(p.out), p.ws, p.counters, p.inv_freq, p.Hq, p.Hkv, p.D, p.num_splits, p.scale},
          batch, qkv_stride, out_stride, pt_stride, max_pages};
}

}  // namespace

int gemv_bf16(const GemvParams& p, cudaStream_t stream) {
  VB_CHECK(p.N > 0 && p.K > 0 && p.K % 8 == 0, "gemv: bad shape N=%d K=%d (K %% 8 == 0)", p.N, p.K);
  VB_CHECK(!(p.flags & 1) || p.N % 2 == 0, "gemv: swiglu needs even N");
  if (!(p.flags & 4)) {  // default: TMA-ring kernel; flag 4 selects the register-staged variant
    const int rc = gemv_tma_bf16(p, stream);
    if (rc >= 0) return rc;
  }
  const int sms = num_sms();
  int rows_per_block = (p.N + sms - 1) / sms;
  if ((p.flags & 1) && (rows_per_block & 1)) rows_per_block += 1;
  const int grid = (p.N + rows_per_block - 1) / rows_per_block;
  const int nchunks = ((p.K >> 3) + 31) >> 5;
  int ksplit = 1;
  while (rows_per_block * ksplit < 3 * kGemvWarps && ksplit * 2 <= nchunks && ksplit < 16) ksplit *= 2;
  const size_t smem = static_cast<size_t>((p.K + 7) / 8) * 16 + static_cast<size_t>(rows_per_block) * ksplit * 4;
  VB_CHECK(smem <= 200 * 1024, "gemv: K=%d / rows_per_block=%d exceed shared memory", p.K,
           rows_per_block);
  auto kern = gemv_kernel<8>;
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  }
  VB_CUDA(launch_pdl(kern, dim3(grid), dim3(kGemvThreads), smem, stream, p, rows_per_block, ksplit));
  return 0;
}

int argmax_finalize(unsigned long long* key, int32_t* token_out, int32_t* token_hist,
                       int32_t* step_counter, int32_t* position, const __nv_bfloat16* embed_table,
                       __nv_bfloat16* x_next, int hidden, cudaStream_t stream) {
  VB_CHECK(hidden % 8 == 0, "argmax_finalize: hidden must be a multiple of 8");
  VB_CUDA(launch_pdl(argmax_finalize_kernel, dim3(1), dim3(256), 0, stream, key, token_out, token_hist,
                     step_counter, position, reinterpret_cast<const uint4*>(embed_table),
                     reinterpret_cast<uint4*>(x_next), hidden / 8));
  return 0;
}

int decode_attention(const vila_decode_attn_params& p, cudaStream_t stream) {
  VB_CHECK(p.D == 128, "decode_attention: head_dim must be 128 (got %d)", p.D);
  VB_CHECK(p.Hq % p.Hkv == 0, "decode_attention: Hq %% Hkv != 0");
  VB_CHECK(p.num_splits >= 0 && p.num_splits <= 64, "decode_attention: bad num_splits %d",
           p.num_splits);
  if (p.num_splits == 0) {
    // one CTA per query head, no split: contexts of at most 1024 tokens (8 pages), see the kernel
    const DecodeAttnBatchArgs a = head_args(p, 1, 0, 0, 0, 8);
    VB_CUDA(launch_pdl(decode_attn_head_kernel<128, 4>, dim3(p.Hq), dim3(kDhThreads), 0, stream, a));
    return 0;
  }
  const int G = p.Hq / p.Hkv;
  dim3 grid(p.Hkv, p.num_splits);
#define VB_DA_CASE(GG)                                                                          \
  case GG: {                                                                                    \
    const bool use_cluster = p.num_splits <= 8;                                                 \
    auto kern = use_cluster ? decode_attn_kernel<128, GG, true> : decode_attn_kernel<128, GG, false>; \
    const size_t smem = (size_t)kDaWarps * 2 * GG * (128 + 2) * sizeof(float);                  \
    static PerDeviceOnce attr_once[2];                                                          \
    if (attr_once[use_cluster].first()) {                                                       \
      VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    }                                                                                           \
    VB_CUDA(launch_pdl_cluster(kern, grid, dim3(kDaThreads), smem, stream,                      \
                               dim3(1, use_cluster ? p.num_splits : 1, 1), p));                 \
    break;                                                                                      \
  }
  switch (G) {
    VB_DA_CASE(1)
    VB_DA_CASE(2)
    VB_DA_CASE(4)
    VB_DA_CASE(7)
    VB_DA_CASE(8)
    default:
      set_last_error("decode_attention: unsupported GQA group size %d", G);
      return 1;
  }
#undef VB_DA_CASE
  return 0;
}


// Long-context decode attention in two launches (three without `counters`; all PDL, graph-capturable,
// position on the device):
//   1. rope_kv_append on the one new token: RoPE(q, k_new) in place, k/v appended at slot = position
//   2. fmha_decode_split: the wgmma FMHA kernel with the G query heads of a KV group as its query
//      rows and the KV splits as blockIdx.z: K/V pages stream through TMA into the warp-specialised
//      producer / MMA / softmax pipeline on every SM
//   3. the combine: by the last split CTA of every KV head inside (2) when `counters` is given, else
//      decode_combine_kernel
int decode_attention_split(const vila_decode_attn_split_params& p, cudaStream_t stream) {
  VB_CHECK(p.D == 128, "decode_attention_split: head_dim must be 128 (got %d)", p.D);
  VB_CHECK(p.Hq % p.Hkv == 0, "decode_attention_split: Hq %% Hkv != 0");
  VB_CHECK(p.num_splits >= 1 && p.split_tokens > 0 && p.split_tokens % 128 == 0,
           "decode_attention_split: bad split configuration (%d x %d)", p.num_splits, p.split_tokens);
  const int G = p.Hq / p.Hkv;
  int rc = rope_kv_append(static_cast<__nv_bfloat16*>(p.qkv), p.position, 1, p.Hq, p.Hkv, p.D, p.inv_freq,
                          static_cast<__nv_bfloat16*>(p.k_pool), static_cast<__nv_bfloat16*>(p.v_pool),
                          p.page_table, -1, stream);
  if (rc) return rc;
  vila_fmha_params f;
  f.q = p.qkv;
  f.q_tok_stride = p.D;                       // "token" = query head g of the group
  f.q_head_stride = static_cast<int64_t>(G) * p.D;   // "head" = KV head
  f.k = p.k_pool;
  f.v = p.v_pool;
  f.kv_page_stride = static_cast<int64_t>(128) * p.Hkv * p.D;
  f.kv_tok_stride = static_cast<int64_t>(p.Hkv) * p.D;
  f.kv_head_stride = p.D;
  f.kv_num_pages = p.kv_num_pages;
  f.page_table = p.page_table;
  f.page_table_stride = 0;
  f.o = p.counters ? p.out : nullptr;   // fused combine writes out[(hk*G + g)*D + d]
  f.o_tok_stride = p.D;
  f.o_head_stride = static_cast<int64_t>(G) * p.D;
  f.B = p.num_splits;
  f.Sq = G;
  f.Sk = p.split_tokens;
  f.Hq = p.Hkv;
  f.Hkv = p.Hkv;
  f.D = p.D;
  f.causal = 0;
  f.scale = p.scale;
  rc = fmha_decode_split(f, p.position, p.split_tokens, p.o_partial, p.lse, p.counters, stream);
  if (rc) return rc;
  if (p.counters != nullptr) return 0;  // combined by the last split CTA of every KV head
  VB_CHECK(p.num_splits <= kCombineMaxSplits, "decode_attention_split: at most %d splits", kCombineMaxSplits);
  VB_CUDA(launch_pdl(decode_combine_kernel, dim3(p.Hq), dim3(128), 0, stream,
                     static_cast<const float*>(p.o_partial), static_cast<const float*>(p.lse),
                     static_cast<__nv_bfloat16*>(p.out), p.Hq, p.D, p.num_splits));
  return 0;
}


// Batched long-context decode attention (continuous batching at video contexts): the two launches of
// decode_attention_split with the fused combine, over `batch` sequences at once.  Sequence b's output is
// bit-identical to decode_attention_split on that sequence alone with the same split configuration.
int decode_attention_split_batch(const vila_decode_attn_split_params& p, int batch, int qkv_stride, int out_stride,
                                 int pt_stride, cudaStream_t stream) {
  VB_CHECK(p.D == 128, "decode_attention_split_batch: head_dim must be 128 (got %d)", p.D);
  VB_CHECK(p.Hq % p.Hkv == 0, "decode_attention_split_batch: Hq %% Hkv != 0");
  VB_CHECK(batch >= 1, "decode_attention_split_batch: bad batch %d", batch);
  VB_CHECK(p.num_splits >= 1 && p.split_tokens > 0 && p.split_tokens % 128 == 0,
           "decode_attention_split_batch: bad split configuration (%d x %d)", p.num_splits, p.split_tokens);
  VB_CHECK(p.counters != nullptr, "decode_attention_split_batch: counters are required");
  VB_CHECK(qkv_stride >= (p.Hq + 2 * p.Hkv) * p.D && qkv_stride % 8 == 0 && out_stride >= p.Hq * p.D &&
               pt_stride >= 1,
           "decode_attention_split_batch: bad strides (qkv %d, out %d, page table %d)", qkv_stride, out_stride,
           pt_stride);
  const int G = p.Hq / p.Hkv;
  int rc = rope_kv_append_decode_batch(static_cast<__nv_bfloat16*>(p.qkv), qkv_stride, p.position, batch, p.Hq,
                                       p.Hkv, p.D, p.inv_freq, static_cast<__nv_bfloat16*>(p.k_pool),
                                       static_cast<__nv_bfloat16*>(p.v_pool), p.page_table, pt_stride, stream);
  if (rc) return rc;
  vila_fmha_params f;
  f.q = p.qkv;
  f.q_tok_stride = p.D;
  f.q_head_stride = static_cast<int64_t>(G) * p.D;
  f.k = p.k_pool;
  f.v = p.v_pool;
  f.kv_page_stride = static_cast<int64_t>(128) * p.Hkv * p.D;
  f.kv_tok_stride = static_cast<int64_t>(p.Hkv) * p.D;
  f.kv_head_stride = p.D;
  f.kv_num_pages = p.kv_num_pages;
  f.page_table = p.page_table;
  f.page_table_stride = pt_stride;
  f.o = p.out;
  f.o_tok_stride = p.D;
  f.o_head_stride = static_cast<int64_t>(G) * p.D;
  f.B = p.num_splits;
  f.Sq = G;
  f.Sk = p.split_tokens;
  f.Hq = p.Hkv;
  f.Hkv = p.Hkv;
  f.D = p.D;
  f.causal = 0;
  f.scale = p.scale;
  return fmha_decode_split(f, p.position, p.split_tokens, p.o_partial, p.lse, p.counters, stream, batch,
                           qkv_stride, out_stride);
}

int decode_attention_batch(const vila_decode_attn_params& p, int batch, int qkv_stride, int out_stride,
                           int pt_stride, int max_pages, cudaStream_t stream) {
  VB_CHECK(p.D == 128, "decode_attention_batch: head_dim must be 128 (got %d)", p.D);
  VB_CHECK(p.Hq % p.Hkv == 0, "decode_attention_batch: Hq %% Hkv != 0");
  VB_CHECK(batch >= 1 && batch <= 65535, "decode_attention_batch: bad batch %d", batch);
  VB_CHECK(max_pages >= 1 && max_pages <= kDhMaxPages && max_pages <= pt_stride,
           "decode_attention_batch: 1 <= max_pages (%d) <= min(%d, pt_stride %d)", max_pages, kDhMaxPages, pt_stride);
  const DecodeAttnBatchArgs a = head_args(p, batch, qkv_stride, out_stride, pt_stride, max_pages);
  VB_CUDA(launch_pdl(decode_attn_head_kernel<128, 4>, dim3(p.Hq, batch), dim3(kDhThreads), 0, stream, a));
  return 0;
}

}  // namespace vb
