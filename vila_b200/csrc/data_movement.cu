// Pure HBM-bound permutation / gather kernels of the hot path (bf16, 128-bit vectors, coalesced
// along the channel dimension, grids sized in multiples of the SM count with grid-stride loops).
#include "common.cuh"
#include "kernels.h"

namespace vb {
namespace {

inline int grid_for(long total_items, int threads, int items_per_thread = 1) {
  long blocks = (total_items + (long)threads * items_per_thread - 1) / ((long)threads * items_per_thread);
  const long cap = (long)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

// ------------------------------------------------------------------------------------------------
// im2col for the 14x14/s14 patch-embed conv (modeling_siglip.py:269-275,322): row = (b, py, px),
// col = (c, ky, kx) matching Conv2d weight.view(1152, 588); columns [588, k_pad) are zero.
// ------------------------------------------------------------------------------------------------
__global__ void im2col_kernel(const __nv_bfloat16* __restrict__ pix, __nv_bfloat16* __restrict__ out,
                              int B, int C, int H, int W, int P, int k_pad) {
  griddep_launch_dependents();
  griddep_wait();
  const int gh = H / P, gw = W / P;
  const int kk = C * P * P;
  // one thread handles one (row, c, ky) strip of P contiguous pixels (28 bytes for P=14)
  const long strips = (long)B * gh * gw * C * P;
  for (long s = blockIdx.x * (long)blockDim.x + threadIdx.x; s < strips;
       s += (long)gridDim.x * blockDim.x) {
    int ky = s % P;
    long t = s / P;
    int c = t % C;
    t /= C;
    int px = t % gw;
    t /= gw;
    int py = t % gh;
    int b = t / gh;
    const __nv_bfloat16* src =
        pix + (((long)b * C + c) * H + (py * P + ky)) * W + px * P;
    long row = ((long)b * gh + py) * gw + px;
    __nv_bfloat16* dst = out + row * k_pad + (c * P + ky) * P;
    // P is even (14): copy as 32-bit pairs (source/dest are 4-byte aligned when W, P even)
    const uint32_t* s32 = reinterpret_cast<const uint32_t*>(src);
    uint32_t* d32 = reinterpret_cast<uint32_t*>(dst);
#pragma unroll 7
    for (int i = 0; i < P / 2; ++i) d32[i] = s32[i];
    if (c == C - 1 && ky == P - 1) {
      for (int i = kk; i < k_pad; ++i) out[row * k_pad + i] = __float2bfloat16(0.f);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// space-to-depth (DownSampleBlock.flat_square / flat_square_2x2 / _3x3, base_projector.py:58-123):
// out[b, i, j, (q*r + p)*C + ch] = x[b, r*i+q, r*j+p, ch], zero beyond the (odd) border.
// ------------------------------------------------------------------------------------------------
__global__ void s2d_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, int B, int h, int w,
                           int Cv, int r) {
  griddep_launch_dependents();
  griddep_wait();
  const int ho = (h + r - 1) / r, wo = (w + r - 1) / r;
  const long total = (long)B * ho * wo * r * r * Cv;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total;
       idx += (long)gridDim.x * blockDim.x) {
    int cv = idx % Cv;
    long t = idx / Cv;
    int p = t % r;
    t /= r;
    int q = t % r;
    t /= r;
    int j = t % wo;
    t /= wo;
    int i = t % ho;
    int b = t / ho;
    const int yi = r * i + q, xj = r * j + p;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (yi < h && xj < w) v = ldg_stream(x + (((long)b * h + yi) * w + xj) * Cv + cv);
    out[idx] = v;
  }
}

// ------------------------------------------------------------------------------------------------
// dynamic-S2 merge for ONE image (llava_arch.py:298-364 + split_chessboard :282-296):
//   per scale s: tiles stitched to a (side*sh) x (side*sw) map (merge_chessboard :255-280),
//   F.interpolate(mode="area") to the output map (== adaptive average pooling, fp32 accumulate),
//   channel-concatenated over scales, then re-split into out_bh x out_bw tiles of side x side.
// ------------------------------------------------------------------------------------------------
struct S2Args {
  int n_scales, side, C;
  int sh[4], sw[4], tile0[4];
  int out_bh, out_bw;
};
// I = index type: uint32_t whenever the item count fits (always for real images) — the 64-bit divisions
// of the generic version made the kernel instruction-issue bound
template <typename I>
__global__ void s2_merge_kernel(const __nv_bfloat16* __restrict__ tiles,
                                __nv_bfloat16* __restrict__ out, S2Args a) {
  griddep_launch_dependents();
  griddep_wait();
  const I Cv = a.C / 8;
  const I OH = a.out_bh * a.side, OW = a.out_bw * a.side;
  const I total = OH * OW * (I)a.n_scales * Cv;
  const I side = a.side;
  for (I idx = blockIdx.x * (I)blockDim.x + threadIdx.x; idx < total; idx += (I)gridDim.x * blockDim.x) {
    const I cv = idx % Cv;
    I t = idx / Cv;
    const int s = (int)(t % (I)a.n_scales);
    t /= (I)a.n_scales;
    const I ox = t % OW;
    const I oy = t / OW;
    const I IH = a.sh[s] * a.side, IW = a.sw[s] * a.side;
    // adaptive_avg_pool window: [floor(o*I/O), ceil((o+1)*I/O))
    const I y0 = (oy * IH) / OH, y1 = ((oy + 1) * IH + OH - 1) / OH;
    const I x0 = (ox * IW) / OW, x1 = ((ox + 1) * IW + OW - 1) / OW;
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (I y = y0; y < y1; ++y) {
      for (I x = x0; x < x1; ++x) {
        const I tile = a.tile0[s] + (y / side) * a.sw[s] + (x / side);
        const I tok = (y % side) * side + (x % side);
        const uint4 v = ldg_v4(reinterpret_cast<const uint4*>(
                                   tiles + ((size_t)tile * side * side + tok) * a.C) + cv);
        acc[0] += bf_lo(v.x); acc[1] += bf_hi(v.x); acc[2] += bf_lo(v.y); acc[3] += bf_hi(v.y);
        acc[4] += bf_lo(v.z); acc[5] += bf_hi(v.z); acc[6] += bf_lo(v.w); acc[7] += bf_hi(v.w);
      }
    }
    const float inv = 1.f / (float)((y1 - y0) * (x1 - x0));
    uint4 o;
    o.x = pack_bf16(acc[0] * inv, acc[1] * inv);
    o.y = pack_bf16(acc[2] * inv, acc[3] * inv);
    o.z = pack_bf16(acc[4] * inv, acc[5] * inv);
    o.w = pack_bf16(acc[6] * inv, acc[7] * inv);
    const I otile = (oy / side) * a.out_bw + (ox / side);
    const I otok = (oy % side) * side + (ox % side);
    uint4* dst = reinterpret_cast<uint4*>(
        out + ((size_t)otile * side * side + otok) * ((size_t)a.n_scales * a.C) + (size_t)s * a.C);
    dst[cv] = o;
  }
}

// merge_chessboard + "1 c h w -> (h w) c" (llava_arch.py:384-390): tiles [bh*bw, s*s, C] ->
// out [(bh*s) * (bw*s), C]
__global__ void chessboard_kernel(const uint4* __restrict__ tiles, uint4* __restrict__ out, int bh,
                                  int bw, int s, int Cv) {
  griddep_launch_dependents();
  griddep_wait();
  const long total = (long)bh * s * bw * s * Cv;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total;
       idx += (long)gridDim.x * blockDim.x) {
    int cv = idx % Cv;
    long t = idx / Cv;
    int x = t % (bw * s);
    int y = t / (bw * s);
    const int tile = (y / s) * bw + (x / s);
    const int tok = (y % s) * s + (x % s);
    out[idx] = ldg_stream(tiles + ((long)tile * s * s + tok) * Cv + cv);
  }
}

// TSP pooling (encoders/video/tsp.py:11-12,28-51): mean over (pt, ph, pw) groups, fp32 accumulate.
// The reference chains three .mean() calls each rounding to bf16; we follow the same order of
// roundings: t-pool -> bf16 -> h-pool -> bf16 -> w-pool -> bf16.
__global__ void tsp_pool_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ out,
                                int T, int h, int w, int C, int pt, int ph, int pw) {
  griddep_launch_dependents();
  griddep_wait();
  const int To = T / pt, ho = h / ph, wo = w / pw;
  const long total = (long)To * ho * wo * C;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total;
       idx += (long)gridDim.x * blockDim.x) {
    int c = idx % C;
    long t = idx / C;
    int xo = t % wo;
    t /= wo;
    int yo = t % ho;
    int to = t / ho;
    float sw_acc = 0.f;
    for (int c3 = 0; c3 < pw; ++c3) {
      float sh_acc = 0.f;
      for (int c2 = 0; c2 < ph; ++c2) {
        float st = 0.f;
        for (int c1 = 0; c1 < pt; ++c1) {
          st += __bfloat162float(
              x[((((long)(to * pt + c1)) * h + (yo * ph + c2)) * w + (xo * pw + c3)) * C + c]);
        }
        sh_acc += bf16_round(st / pt);
      }
      sw_acc += bf16_round(sh_acc / ph);
    }
    out[idx] = __float2bfloat16(sw_acc / pw);
  }
}

// the same pooling, 8 channels per thread (16-byte loads / stores, 32-bit index math): the scalar version
// above moves 2 bytes per load, too few to keep HBM busy.  Same order of roundings per channel.
__global__ void tsp_pool_v8_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, int T, int h,
                                   int w, int Cv, int pt, int ph, int pw) {
  griddep_launch_dependents();
  griddep_wait();
  const uint32_t ho = h / ph, wo = w / pw;
  const uint32_t total = (uint32_t)(T / pt) * ho * wo * Cv;
  for (uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const uint32_t cv = idx % Cv;
    uint32_t t = idx / Cv;
    const uint32_t xo = t % wo;
    t /= wo;
    const uint32_t yo = t % ho, to = t / ho;
    float sw_acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int c3 = 0; c3 < pw; ++c3) {
      float sh_acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      for (int c2 = 0; c2 < ph; ++c2) {
        float st[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        const size_t row0 = ((size_t)(to * pt) * h + (yo * ph + c2)) * w + (xo * pw + c3);
#pragma unroll 4
        for (int c1 = 0; c1 < pt; ++c1) {
          const uint4 v = ldg_stream(x + (row0 + (size_t)c1 * h * w) * Cv + cv);
          st[0] += bf_lo(v.x); st[1] += bf_hi(v.x); st[2] += bf_lo(v.y); st[3] += bf_hi(v.y);
          st[4] += bf_lo(v.z); st[5] += bf_hi(v.z); st[6] += bf_lo(v.w); st[7] += bf_hi(v.w);
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) sh_acc[k] += bf16_round(st[k] / pt);
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) sw_acc[k] += bf16_round(sh_acc[k] / ph);
    }
    uint4 o;
    o.x = pack_bf16(sw_acc[0] / pw, sw_acc[1] / pw);
    o.y = pack_bf16(sw_acc[2] / pw, sw_acc[3] / pw);
    o.z = pack_bf16(sw_acc[4] / pw, sw_acc[5] / pw);
    o.w = pack_bf16(sw_acc[6] / pw, sw_acc[7] / pw);
    out[idx] = o;
  }
}

// text/media embedding splice (llava_arch.py:429,457-479): one gather driven by a host-built table
__global__ void embed_splice_kernel(const uint4* __restrict__ table, const uint4* __restrict__ media,
                                    const int32_t* __restrict__ src, uint4* __restrict__ out,
                                    int rows, int Cv) {
  griddep_launch_dependents();
  griddep_wait();
  const long total = (long)rows * Cv;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total;
       idx += (long)gridDim.x * blockDim.x) {
    const int r = idx / Cv, cv = idx % Cv;
    const int sidx = src[r];
    const uint4* p = sidx >= 0 ? table + (long)sidx * Cv : media + (long)(-(sidx + 1)) * Cv;
    out[idx] = ldg_stream(p + cv);
  }
}

// RoPE (rotate-half, HF apply_rotary_pos_emb, modeling_qwen2.py:99-160) in place on the q and k
// heads of a fused [S, (Hq+2Hkv)*D] buffer + KV append into the paged pool.
// cos/sin are computed in fp32 and rounded to bf16 like HF (cos.to(dtype)); products are rounded
// to bf16 before the sum as the reference's bf16 tensor ops do.
// Row s of qkv starts at qkv + s*row_stride.  Decode (cache_pos0 < 0) of a batch of sequences: row s
// uses the page-table row page_table + s*pt_stride, and a negative position marks an idle row that is
// left untouched.
__global__ void rope_kv_kernel(__nv_bfloat16* __restrict__ qkv, const int32_t* __restrict__ pos,
                               int S, int Hq, int Hkv, int D,
                               const float* __restrict__ inv_freq_tab,
                               __nv_bfloat16* __restrict__ k_pool,
                               __nv_bfloat16* __restrict__ v_pool,
                               const int32_t* __restrict__ page_table, int cache_pos0,
                               long row_stride, int pt_stride) {
  griddep_launch_dependents();
  griddep_wait();
  const int half = D / 2;
  const int Ht = Hq + 2 * Hkv;
  const long total = (long)S * Ht * half;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total;
       idx += (long)gridDim.x * blockDim.x) {
    const int i = idx % half;
    long t = idx / half;
    const int hh = t % Ht;
    const int s = t / Ht;
    if (cache_pos0 < 0 && pos[s] < 0) continue;  // idle decode row
    __nv_bfloat16* base = qkv + (long)s * row_stride + (long)hh * D;
    float x0 = __bfloat162float(base[i]), x1 = __bfloat162float(base[i + half]);
    if (hh < Hq + Hkv) {
      const float ang = (float)pos[s] * inv_freq_tab[i];
      float sn, cs;
      sincosf(ang, &sn, &cs);
      cs = bf16_round(cs);
      sn = bf16_round(sn);
      const float y0 = bf16_round(x0 * cs) + bf16_round(-x1 * sn);
      const float y1 = bf16_round(x1 * cs) + bf16_round(x0 * sn);
      x0 = bf16_round(y0);
      x1 = bf16_round(y1);
      base[i] = __float2bfloat16(x0);
      base[i + half] = __float2bfloat16(x1);
    }
    if (hh >= Hq && k_pool != nullptr) {
      // cache_pos0 < 0: the cache slot is the position id itself (decode: the position lives in
      // device memory so that one captured graph serves every step)
      const int cpos = cache_pos0 < 0 ? pos[s] : cache_pos0 + s;
      const int page = page_table[(long)s * pt_stride + (cpos >> 7)];
      const int hk = (hh - Hq) % Hkv;
      __nv_bfloat16* pool = (hh < Hq + Hkv) ? k_pool : v_pool;
      __nv_bfloat16* dst = pool + (((long)page * 128 + (cpos & 127)) * Hkv + hk) * D;
      dst[i] = __float2bfloat16(x0);
      dst[i + half] = __float2bfloat16(x1);
    }
  }
}

// Table-driven, vectorised variant for long prefills: cos / sin come from rope_table() (computed once
// per request instead of once per head: 36x fewer sincosf), every thread rotates 8 + 8 elements with
// 16-byte accesses.  Bit-identical to rope_kv_kernel (same cos/sin rounding, same product rounding).
__global__ void rope_kv_table_kernel(__nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ table,
                                     int S, int Hq, int Hkv, int D, __nv_bfloat16* __restrict__ k_pool,
                                     __nv_bfloat16* __restrict__ v_pool,
                                     const int32_t* __restrict__ page_table, int cache_pos0) {
  griddep_launch_dependents();
  griddep_wait();
  const int half = D / 2;
  const int vph = half / 8;  // 16-byte vectors per half head
  const int Ht = Hq + 2 * Hkv;
  const long total = (long)S * Ht * vph;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total;
       idx += (long)gridDim.x * blockDim.x) {
    const int vi = idx % vph;
    long t = idx / vph;
    const int hh = t % Ht;
    const int s = t / Ht;
    __nv_bfloat16* base = qkv + ((long)s * Ht + hh) * D + vi * 8;
    uint4 a = *reinterpret_cast<const uint4*>(base);
    uint4 b = *reinterpret_cast<const uint4*>(base + half);
    if (hh < Hq + Hkv) {
      const uint4 cv = ldg_v4(table + (long)s * D + vi * 8);
      const uint4 sv = ldg_v4(table + (long)s * D + half + vi * 8);
      auto rot = [](uint32_t x0p, uint32_t x1p, uint32_t cp, uint32_t sp, uint32_t& y0p, uint32_t& y1p) {
        const float x0l = bf_lo(x0p), x0h = bf_hi(x0p), x1l = bf_lo(x1p), x1h = bf_hi(x1p);
        const float cl = bf_lo(cp), ch = bf_hi(cp), sl = bf_lo(sp), sh = bf_hi(sp);
        y0p = pack_bf16(bf16_round(x0l * cl) + bf16_round(-x1l * sl), bf16_round(x0h * ch) + bf16_round(-x1h * sh));
        y1p = pack_bf16(bf16_round(x1l * cl) + bf16_round(x0l * sl), bf16_round(x1h * ch) + bf16_round(x0h * sh));
      };
      uint4 ya, yb;
      rot(a.x, b.x, cv.x, sv.x, ya.x, yb.x);
      rot(a.y, b.y, cv.y, sv.y, ya.y, yb.y);
      rot(a.z, b.z, cv.z, sv.z, ya.z, yb.z);
      rot(a.w, b.w, cv.w, sv.w, ya.w, yb.w);
      a = ya;
      b = yb;
      *reinterpret_cast<uint4*>(base) = a;
      *reinterpret_cast<uint4*>(base + half) = b;
    }
    if (hh >= Hq && k_pool != nullptr) {
      const int cpos = cache_pos0 + s;
      const int page = page_table[cpos >> 7];
      const int hk = (hh - Hq) % Hkv;
      __nv_bfloat16* pool = (hh < Hq + Hkv) ? k_pool : v_pool;
      __nv_bfloat16* dst = pool + (((long)page * 128 + (cpos & 127)) * Hkv + hk) * D + vi * 8;
      *reinterpret_cast<uint4*>(dst) = a;
      *reinterpret_cast<uint4*>(dst + half) = b;
    }
  }
}

// cos / sin of HF Qwen2RotaryEmbedding for a request, computed once and shared by all layers and
// heads: table[s] = bf16(cos(pos[s] * inv_freq[i])) for i < D/2, then bf16(sin(...)).
__global__ void rope_table_kernel(const int32_t* __restrict__ pos, int S, int half,
                                  const float* __restrict__ inv_freq_tab,
                                  __nv_bfloat16* __restrict__ table) {
  griddep_launch_dependents();
  griddep_wait();
  const long total = (long)S * half;
  for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total;
       idx += (long)gridDim.x * blockDim.x) {
    const int i = idx % half;
    const int s = idx / half;
    const float ang = (float)pos[s] * inv_freq_tab[i];
    float sn, cs;
    sincosf(ang, &sn, &cs);
    table[(long)s * 2 * half + i] = __float2bfloat16(cs);
    table[(long)s * 2 * half + half + i] = __float2bfloat16(sn);
  }
}


// ------------------------------------------------------------------------------------------------
// Image preprocessing (SURVEY §8 f2): PIL's 8-bit bicubic resampler (Pillow src/libImaging/Resample.c:
// 22-bit fixed-point separable convolution, uint8 after each pass) + SiglipImageProcessor's rescale
// (1/255) and normalise ((x - mean) / std) + tiling, i.e. what processor.preprocess does to every tile
// in mm_utils.process_image (llava/mm_utils.py:476,480,505,518) — bit-identical by construction: the
// integer filter taps come from the host exactly as precompute_coeffs / normalize_coeffs_8bpc make them.
// ------------------------------------------------------------------------------------------------
constexpr int kResampleBits = 32 - 8 - 2;

__device__ __forceinline__ uint8_t clip8(int v) {
  v >>= kResampleBits;  // arithmetic shift, like Pillow's clip8 lookup
  return static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// src [H][W][3] uint8 -> tmp [H][out_w][3] uint8
__global__ void resize_h_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ tmp, int H, int W,
                                int out_w, const int32_t* __restrict__ coef,
                                const int32_t* __restrict__ bounds, int ksize) {
  griddep_launch_dependents();
  griddep_wait();
  const long total = (long)H * out_w;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int X = static_cast<int>(i % out_w);
    const int y = static_cast<int>(i / out_w);
    const int xmin = bounds[2 * X], n = bounds[2 * X + 1];
    const int32_t* k = coef + (long)X * ksize;
    const uint8_t* p = src + ((long)y * W + xmin) * 3;
    int a0 = 1 << (kResampleBits - 1), a1 = a0, a2 = a0;
    for (int x = 0; x < n; ++x) {
      const int kk = k[x];
      a0 += p[3 * x] * kk;
      a1 += p[3 * x + 1] * kk;
      a2 += p[3 * x + 2] * kk;
    }
    uint8_t* d = tmp + i * 3;
    d[0] = clip8(a0);
    d[1] = clip8(a1);
    d[2] = clip8(a2);
  }
}

// tmp [H][out_w][3] uint8 -> tiles [n][3][tile][tile] bf16 of the resized (out_h x out_w) image
__global__ void resize_v_norm_kernel(const uint8_t* __restrict__ tmp, __nv_bfloat16* __restrict__ out,
                                     int out_w, int out_h, const int32_t* __restrict__ coef,
                                     const int32_t* __restrict__ bounds, int ksize, int tile, int tile0,
                                     float mean, float stdv) {
  griddep_launch_dependents();
  griddep_wait();
  const long total = (long)out_h * out_w;
  const int per_row = out_w / tile;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int X = static_cast<int>(i % out_w);
    const int Y = static_cast<int>(i / out_w);
    const int ymin = bounds[2 * Y], n = bounds[2 * Y + 1];
    const int32_t* k = coef + (long)Y * ksize;
    const uint8_t* p = tmp + ((long)ymin * out_w + X) * 3;
    int a[3] = {1 << (kResampleBits - 1), 1 << (kResampleBits - 1), 1 << (kResampleBits - 1)};
    for (int y = 0; y < n; ++y) {
      const int kk = k[y];
      const uint8_t* q = p + (long)y * out_w * 3;
      a[0] += q[0] * kk;
      a[1] += q[1] * kk;
      a[2] += q[2] * kk;
    }
    const int t = tile0 + (Y / tile) * per_row + X / tile;
    const int ly = Y % tile, lx = X % tile;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      // fp32 like the processor: x / 255 (IEEE division), then (x - mean) / std; bf16 RN like .to(bf16)
      const float v = __fdiv_rn(static_cast<float>(clip8(a[c])), 255.0f);
      out[(((long)t * 3 + c) * tile + ly) * tile + lx] = __float2bfloat16(__fdiv_rn(v - mean, stdv));
    }
  }
}

}  // namespace

int rope_table(const int32_t* positions, int S, int D, const float* inv_freq, __nv_bfloat16* table,
               cudaStream_t stream) {
  VB_CHECK(D % 2 == 0, "rope_table: head dim must be even");
  if (S == 0) return 0;
  const long total = (long)S * (D / 2);
  VB_CUDA(launch_pdl(rope_table_kernel, dim3(grid_for(total, 256)), dim3(256), 0, stream, positions, S, D / 2,
                     inv_freq, table));
  return 0;
}

int im2col_patch14(const __nv_bfloat16* pixels, __nv_bfloat16* out, int B, int C, int H, int W,
                   int patch, int k_pad, cudaStream_t stream) {
  VB_CHECK(H % patch == 0 && W % patch == 0, "im2col: image %dx%d not divisible by patch %d", H, W,
           patch);
  VB_CHECK(patch % 2 == 0 && W % 2 == 0, "im2col: patch and width must be even");
  VB_CHECK(k_pad >= C * patch * patch && k_pad % 8 == 0, "im2col: bad k_pad %d", k_pad);
  const long strips = (long)B * (H / patch) * (W / patch) * C * patch;
  if (strips == 0) return 0;
  VB_CUDA(launch_pdl(im2col_kernel, dim3(grid_for(strips, 256)), dim3(256), 0, stream, pixels, out, B, C, H, W, patch, k_pad));
  return 0;
}

int space_to_depth(const __nv_bfloat16* x, __nv_bfloat16* out, int B, int h, int w, int C, int r,
                   cudaStream_t stream) {
  VB_CHECK(C % 8 == 0, "space_to_depth: C must be a multiple of 8 (got %d)", C);
  VB_CHECK(r == 2 || r == 3, "space_to_depth: r must be 2 or 3 (got %d)", r);
  const long total = (long)B * ((h + r - 1) / r) * ((w + r - 1) / r) * r * r * (C / 8);
  if (total == 0) return 0;
  VB_CUDA(launch_pdl(s2d_kernel, dim3(grid_for(total, 256)), dim3(256), 0, stream, reinterpret_cast<const uint4*>(x),
                                                      reinterpret_cast<uint4*>(out), B, h, w, C / 8, r));
  return 0;
}

int s2_merge(const __nv_bfloat16* tiles, __nv_bfloat16* out, int side, int C, int n_scales,
             const int* scale_splits_h, const int* scale_splits_w, int out_bh, int out_bw,
             int share_tile, cudaStream_t stream) {
  VB_CHECK(n_scales >= 1 && n_scales <= 4, "s2_merge: 1..4 scales supported (got %d)", n_scales);
  VB_CHECK(C % 8 == 0, "s2_merge: C must be a multiple of 8");
  S2Args a;
  a.n_scales = n_scales;
  a.side = side;
  a.C = C;
  a.out_bh = out_bh;
  a.out_bw = out_bw;
  int t0 = 0;
  for (int s = 0; s < n_scales; ++s) {
    a.sh[s] = scale_splits_h[s];
    a.sw[s] = scale_splits_w[s];
    a.tile0[s] = t0;
    if (!share_tile) t0 += a.sh[s] * a.sw[s];
  }
  const long total = (long)out_bh * side * out_bw * side * n_scales * (C / 8);
  if (total < (1L << 31)) {
    VB_CUDA(launch_pdl(s2_merge_kernel<uint32_t>, dim3(grid_for(total, 256)), dim3(256), 0, stream, tiles, out, a));
  } else {
    VB_CUDA(launch_pdl(s2_merge_kernel<long>, dim3(grid_for(total, 256)), dim3(256), 0, stream, tiles, out, a));
  }
  return 0;
}

int chessboard_merge(const __nv_bfloat16* tiles, __nv_bfloat16* out, int bh, int bw, int s, int C,
                     cudaStream_t stream) {
  VB_CHECK(C % 8 == 0, "chessboard_merge: C must be a multiple of 8");
  const long total = (long)bh * s * bw * s * (C / 8);
  if (total == 0) return 0;
  VB_CUDA(launch_pdl(chessboard_kernel, dim3(grid_for(total, 256)), dim3(256), 0, stream, 
      reinterpret_cast<const uint4*>(tiles), reinterpret_cast<uint4*>(out), bh, bw, s, C / 8));
  return 0;
}

int tsp_pool(const __nv_bfloat16* x, __nv_bfloat16* out, int T, int h, int w, int C, int pt, int ph,
             int pw, cudaStream_t stream) {
  VB_CHECK(pt > 0 && ph > 0 && pw > 0 && T % pt == 0 && h % ph == 0 && w % pw == 0,
           "tsp_pool: pool sizes (%d,%d,%d) must divide (%d,%d,%d)", pt, ph, pw, T, h, w);
  const long total = (long)(T / pt) * (h / ph) * (w / pw) * C;
  if (total == 0) return 0;
  if (C % 8 == 0 && total / 8 < (1L << 31) && (long)T * h * w < (1L << 31) &&
      ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15) == 0) {
    VB_CUDA(launch_pdl(tsp_pool_v8_kernel, dim3(grid_for(total / 8, 256)), dim3(256), 0, stream,
                       reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(out), T, h, w, C / 8, pt, ph, pw));
    return 0;
  }
  VB_CUDA(launch_pdl(tsp_pool_kernel, dim3(grid_for(total, 256)), dim3(256), 0, stream, x, out, T, h, w, C, pt, ph, pw));
  return 0;
}

int embed_splice(const __nv_bfloat16* table, const __nv_bfloat16* media, const int32_t* src,
                 __nv_bfloat16* out, int rows, int cols, cudaStream_t stream) {
  VB_CHECK(cols % 8 == 0, "embed_splice: cols must be a multiple of 8");
  if (rows == 0) return 0;
  const long total = (long)rows * (cols / 8);
  VB_CUDA(launch_pdl(embed_splice_kernel, dim3(grid_for(total, 256)), dim3(256), 0, stream, 
      reinterpret_cast<const uint4*>(table), reinterpret_cast<const uint4*>(media), src,
      reinterpret_cast<uint4*>(out), rows, cols / 8));
  return 0;
}

int rope_kv_append(__nv_bfloat16* qkv, const int32_t* positions, int S, int Hq, int Hkv, int D,
                   const float* inv_freq, __nv_bfloat16* k_pool, __nv_bfloat16* v_pool,
                   const int32_t* page_table, int cache_pos0, cudaStream_t stream) {
  VB_CHECK(D % 2 == 0, "rope: head dim must be even");
  VB_CHECK(k_pool == nullptr || page_table != nullptr, "rope_kv_append: page_table required");
  if (S == 0) return 0;
  const long total = (long)S * (Hq + 2 * Hkv) * (D / 2);
  VB_CUDA(launch_pdl(rope_kv_kernel, dim3(grid_for(total, 256)), dim3(256), 0, stream, qkv, positions, S, Hq, Hkv, D, inv_freq,
                                                          k_pool, v_pool, page_table, cache_pos0,
                     (long)(Hq + 2 * Hkv) * D, 0));
  return 0;
}

int rope_kv_append_decode_batch(__nv_bfloat16* qkv, long qkv_stride, const int32_t* positions, int batch,
                                int Hq, int Hkv, int D, const float* inv_freq, __nv_bfloat16* k_pool,
                                __nv_bfloat16* v_pool, const int32_t* page_table, int pt_stride,
                                cudaStream_t stream) {
  VB_CHECK(D % 2 == 0, "rope: head dim must be even");
  VB_CHECK(k_pool != nullptr && v_pool != nullptr && page_table != nullptr,
           "rope_kv_append_decode_batch: pools and page table required");
  VB_CHECK(batch >= 1 && qkv_stride >= (long)(Hq + 2 * Hkv) * D && pt_stride >= 1,
           "rope_kv_append_decode_batch: bad batch %d / strides", batch);
  const long total = (long)batch * (Hq + 2 * Hkv) * (D / 2);
  VB_CUDA(launch_pdl(rope_kv_kernel, dim3(grid_for(total, 256)), dim3(256), 0, stream, qkv, positions, batch, Hq,
                     Hkv, D, inv_freq, k_pool, v_pool, page_table, -1, qkv_stride, pt_stride));
  return 0;
}


int rope_kv_append_table(__nv_bfloat16* qkv, const __nv_bfloat16* table, int S, int Hq, int Hkv, int D,
                         __nv_bfloat16* k_pool, __nv_bfloat16* v_pool, const int32_t* page_table,
                         int cache_pos0, cudaStream_t stream) {
  VB_CHECK(D % 16 == 0, "rope_kv_append_table: head dim must be a multiple of 16");
  VB_CHECK(k_pool == nullptr || page_table != nullptr, "rope_kv_append_table: page_table required");
  VB_CHECK(cache_pos0 >= 0, "rope_kv_append_table: cache_pos0 must be >= 0");
  if (S == 0) return 0;
  const long total = (long)S * (Hq + 2 * Hkv) * (D / 16);
  VB_CUDA(launch_pdl(rope_kv_table_kernel, dim3(grid_for(total, 256)), dim3(256), 0, stream, qkv, table, S, Hq,
                     Hkv, D, k_pool, v_pool, page_table, cache_pos0));
  return 0;
}

int resize_bicubic_tiles(const uint8_t* src, int H, int W, int out_w, int out_h, const int32_t* coef_x,
                         const int32_t* bounds_x, int ksize_x, const int32_t* coef_y,
                         const int32_t* bounds_y, int ksize_y, uint8_t* tmp, __nv_bfloat16* out_tiles,
                         int tile, int tile_index0, float mean, float stdv, cudaStream_t stream) {
  VB_CHECK(H > 0 && W > 0 && out_w > 0 && out_h > 0, "resize_bicubic_tiles: empty image");
  VB_CHECK(tile > 0 && out_w % tile == 0 && out_h % tile == 0,
           "resize_bicubic_tiles: output %dx%d is not a grid of %d-pixel tiles", out_w, out_h, tile);
  VB_CHECK(stdv != 0.f, "resize_bicubic_tiles: std must be non-zero");
  VB_CUDA(launch_pdl(resize_h_kernel, dim3(grid_for((long)H * out_w, 256)), dim3(256), 0, stream, src, tmp,
                     H, W, out_w, coef_x, bounds_x, ksize_x));
  VB_CUDA(launch_pdl(resize_v_norm_kernel, dim3(grid_for((long)out_h * out_w, 256)), dim3(256), 0, stream,
                     static_cast<const uint8_t*>(tmp), out_tiles, out_w, out_h, coef_y, bounds_y, ksize_y,
                     tile, tile_index0, mean, stdv));
  return 0;
}

}  // namespace vb
