// HBM-bound row normalisations: one CTA per row, 128-bit vector loads, row cached in shared
// memory so global memory is read exactly once, warp-shuffle + smem block reductions.
//   LayerNorm : nn.LayerNorm(1152, eps=1e-6) in SigLIP (modeling_siglip.py:723,725,746,755) and the
//               projector LayerNorm(4C / 9C / 3C) (base_projector.py:147,166,170)
//   RMSNorm   : Qwen2RMSNorm (modeling_qwen2.py:81-95): fp32 variance, x*rsqrt -> bf16, then * weight
#include "common.cuh"
#include "kernels.h"

namespace vb {
namespace {

constexpr int kNormThreads = 256;

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();  // protect red[] reuse
  if (l == 0) red[w] = v;
  __syncthreads();
  float t = (l < (blockDim.x >> 5)) ? red[l] : 0.f;
  t = warp_sum(t);
  return t;
}

__global__ void __launch_bounds__(kNormThreads)
layernorm_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                 const __nv_bfloat16* __restrict__ b, __nv_bfloat16* __restrict__ out, int cols,
                 float eps) {
  extern __shared__ uint4 row_s[];  // cols/8 vectors
  __shared__ float red[32];
  griddep_launch_dependents();
  griddep_wait();
  const int row = blockIdx.x;
  const int nvec = cols >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + static_cast<size_t>(row) * cols);
  float s = 0.f;
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
    const uint4 v = ldg_stream(xr + i);
    row_s[i] = v;
    s += bf_lo(v.x) + bf_hi(v.x) + bf_lo(v.y) + bf_hi(v.y) + bf_lo(v.z) + bf_hi(v.z) + bf_lo(v.w) +
         bf_hi(v.w);
  }
  const float mean = block_sum(s, red) / cols;
  float q = 0.f;
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
    const uint4 v = row_s[i];
    float d;
    d = bf_lo(v.x) - mean; q += d * d;
    d = bf_hi(v.x) - mean; q += d * d;
    d = bf_lo(v.y) - mean; q += d * d;
    d = bf_hi(v.y) - mean; q += d * d;
    d = bf_lo(v.z) - mean; q += d * d;
    d = bf_hi(v.z) - mean; q += d * d;
    d = bf_lo(v.w) - mean; q += d * d;
    d = bf_hi(v.w) - mean; q += d * d;
  }
  const float rstd = rsqrtf(block_sum(q, red) / cols + eps);
  uint4* orow = reinterpret_cast<uint4*>(out + static_cast<size_t>(row) * cols);
  const uint4* wv = reinterpret_cast<const uint4*>(w);
  const uint4* bv = reinterpret_cast<const uint4*>(b);
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
    const uint4 v = row_s[i], g = ldg_v4(wv + i), be = ldg_v4(bv + i);
    uint4 o;
    o.x = pack_bf16((bf_lo(v.x) - mean) * rstd * bf_lo(g.x) + bf_lo(be.x),
                    (bf_hi(v.x) - mean) * rstd * bf_hi(g.x) + bf_hi(be.x));
    o.y = pack_bf16((bf_lo(v.y) - mean) * rstd * bf_lo(g.y) + bf_lo(be.y),
                    (bf_hi(v.y) - mean) * rstd * bf_hi(g.y) + bf_hi(be.y));
    o.z = pack_bf16((bf_lo(v.z) - mean) * rstd * bf_lo(g.z) + bf_lo(be.z),
                    (bf_hi(v.z) - mean) * rstd * bf_hi(g.z) + bf_hi(be.z));
    o.w = pack_bf16((bf_lo(v.w) - mean) * rstd * bf_lo(g.w) + bf_lo(be.w),
                    (bf_hi(v.w) - mean) * rstd * bf_hi(g.w) + bf_hi(be.w));
    orow[i] = o;
  }
}

__device__ __forceinline__ uint32_t rms_pair(uint32_t xv, uint32_t gv, float rstd) {
  // Qwen2RMSNorm: weight * (x * rsqrt(var+eps)).to(bf16)   (product rounded to bf16 again)
  const float a = bf16_round(bf_lo(xv) * rstd) * bf_lo(gv);
  const float c = bf16_round(bf_hi(xv) * rstd) * bf_hi(gv);
  return pack_bf16(a, c);
}

__global__ void __launch_bounds__(kNormThreads)
rmsnorm_kernel(__nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res_add,
               const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ out, int cols,
               float eps) {
  extern __shared__ uint4 row_s[];
  __shared__ float red[32];
  griddep_launch_dependents();
  griddep_wait();
  const int row = blockIdx.x;
  const int nvec = cols >> 3;
  uint4* xr = reinterpret_cast<uint4*>(x + static_cast<size_t>(row) * cols);
  const uint4* rr =
      res_add ? reinterpret_cast<const uint4*>(res_add + static_cast<size_t>(row) * cols) : nullptr;
  float s = 0.f;
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
    uint4 v = ldg_v4(xr + i);
    if (rr) {
      const uint4 r = ldg_stream(rr + i);
      v.x = pack_bf16(bf_lo(v.x) + bf_lo(r.x), bf_hi(v.x) + bf_hi(r.x));
      v.y = pack_bf16(bf_lo(v.y) + bf_lo(r.y), bf_hi(v.y) + bf_hi(r.y));
      v.z = pack_bf16(bf_lo(v.z) + bf_lo(r.z), bf_hi(v.z) + bf_hi(r.z));
      v.w = pack_bf16(bf_lo(v.w) + bf_lo(r.w), bf_hi(v.w) + bf_hi(r.w));
      xr[i] = v;
    }
    row_s[i] = v;
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
  const float rstd = rsqrtf(block_sum(s, red) / cols + eps);
  uint4* orow = reinterpret_cast<uint4*>(out + static_cast<size_t>(row) * cols);
  const uint4* wv = reinterpret_cast<const uint4*>(w);
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
    const uint4 v = row_s[i], g = ldg_v4(wv + i);
    uint4 o;
    o.x = rms_pair(v.x, g.x, rstd);
    o.y = rms_pair(v.y, g.y, rstd);
    o.z = rms_pair(v.z, g.z, rstd);
    o.w = rms_pair(v.w, g.w, rstd);
    orow[i] = o;
  }
}


// ---- warp-per-row variants for LARGE row counts (batched video frames, long prefill) --------------
// One CTA per row keeps only rows_per_SM * row_bytes = 8 * 2.3 KB = 18 KB of loads in flight per SM
// for SigLIP's 1152-wide rows, too little to cover the HBM latency.  Here a warp owns a
// row, holds it in registers (no shared memory, no block barrier), and 64 resident warps per SM keep
// ~150 KB in flight.  Same arithmetic as the CTA-per-row kernels (two-pass variance in fp32).
constexpr int kWarpRowThreads = 256;
constexpr int kWarpRowMinRows = 8192;  // below: one CTA per row (more CTAs -> lower latency)

template <int VPL>  // 16-byte vectors per lane: cols <= VPL * 256
__global__ void __launch_bounds__(kWarpRowThreads, 4)
layernorm_warp_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                      const __nv_bfloat16* __restrict__ b, __nv_bfloat16* __restrict__ out, int rows,
                      int cols, float eps) {
  griddep_launch_dependents();
  griddep_wait();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (kWarpRowThreads / 32) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nvec = cols >> 3;
  const uint4* xr = reinterpret_cast<const uint4*>(x + static_cast<size_t>(row) * cols);
  uint4 v[VPL];
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    const int i = lane + 32 * j;
    v[j] = i < nvec ? ldg_stream(xr + i) : make_uint4(0, 0, 0, 0);
    s += bf_lo(v[j].x) + bf_hi(v[j].x) + bf_lo(v[j].y) + bf_hi(v[j].y) + bf_lo(v[j].z) + bf_hi(v[j].z) +
         bf_lo(v[j].w) + bf_hi(v[j].w);
  }
  const float mean = warp_sum(s) / cols;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    if (lane + 32 * j < nvec) {
      float d;
      d = bf_lo(v[j].x) - mean; q += d * d;
      d = bf_hi(v[j].x) - mean; q += d * d;
      d = bf_lo(v[j].y) - mean; q += d * d;
      d = bf_hi(v[j].y) - mean; q += d * d;
      d = bf_lo(v[j].z) - mean; q += d * d;
      d = bf_hi(v[j].z) - mean; q += d * d;
      d = bf_lo(v[j].w) - mean; q += d * d;
      d = bf_hi(v[j].w) - mean; q += d * d;
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / cols + eps);
  uint4* orow = reinterpret_cast<uint4*>(out + static_cast<size_t>(row) * cols);
  const uint4* wv = reinterpret_cast<const uint4*>(w);
  const uint4* bv = reinterpret_cast<const uint4*>(b);
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    const int i = lane + 32 * j;
    if (i < nvec) {
      const uint4 g = ldg_v4(wv + i), be = ldg_v4(bv + i);
      uint4 o;
      o.x = pack_bf16((bf_lo(v[j].x) - mean) * rstd * bf_lo(g.x) + bf_lo(be.x),
                      (bf_hi(v[j].x) - mean) * rstd * bf_hi(g.x) + bf_hi(be.x));
      o.y = pack_bf16((bf_lo(v[j].y) - mean) * rstd * bf_lo(g.y) + bf_lo(be.y),
                      (bf_hi(v[j].y) - mean) * rstd * bf_hi(g.y) + bf_hi(be.y));
      o.z = pack_bf16((bf_lo(v[j].z) - mean) * rstd * bf_lo(g.z) + bf_lo(be.z),
                      (bf_hi(v[j].z) - mean) * rstd * bf_hi(g.z) + bf_hi(be.z));
      o.w = pack_bf16((bf_lo(v[j].w) - mean) * rstd * bf_lo(g.w) + bf_lo(be.w),
                      (bf_hi(v[j].w) - mean) * rstd * bf_hi(g.w) + bf_hi(be.w));
      orow[i] = o;
    }
  }
}

template <int VPL>
__global__ void __launch_bounds__(kWarpRowThreads, 4)
rmsnorm_warp_kernel(__nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res_add,
                    const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ out, int rows,
                    int cols, float eps) {
  griddep_launch_dependents();
  griddep_wait();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (kWarpRowThreads / 32) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nvec = cols >> 3;
  uint4* xr = reinterpret_cast<uint4*>(x + static_cast<size_t>(row) * cols);
  const uint4* rr =
      res_add ? reinterpret_cast<const uint4*>(res_add + static_cast<size_t>(row) * cols) : nullptr;
  uint4 v[VPL];
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    const int i = lane + 32 * j;
    v[j] = make_uint4(0, 0, 0, 0);
    if (i < nvec) {
      v[j] = ldg_v4(xr + i);
      if (rr) {
        const uint4 r = ldg_stream(rr + i);
        v[j].x = pack_bf16(bf_lo(v[j].x) + bf_lo(r.x), bf_hi(v[j].x) + bf_hi(r.x));
        v[j].y = pack_bf16(bf_lo(v[j].y) + bf_lo(r.y), bf_hi(v[j].y) + bf_hi(r.y));
        v[j].z = pack_bf16(bf_lo(v[j].z) + bf_lo(r.z), bf_hi(v[j].z) + bf_hi(r.z));
        v[j].w = pack_bf16(bf_lo(v[j].w) + bf_lo(r.w), bf_hi(v[j].w) + bf_hi(r.w));
        xr[i] = v[j];
      }
    }
    float t;
    t = bf_lo(v[j].x); s += t * t;
    t = bf_hi(v[j].x); s += t * t;
    t = bf_lo(v[j].y); s += t * t;
    t = bf_hi(v[j].y); s += t * t;
    t = bf_lo(v[j].z); s += t * t;
    t = bf_hi(v[j].z); s += t * t;
    t = bf_lo(v[j].w); s += t * t;
    t = bf_hi(v[j].w); s += t * t;
  }
  const float rstd = rsqrtf(warp_sum(s) / cols + eps);
  uint4* orow = reinterpret_cast<uint4*>(out + static_cast<size_t>(row) * cols);
  const uint4* wv = reinterpret_cast<const uint4*>(w);
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    const int i = lane + 32 * j;
    if (i < nvec) {
      const uint4 g = ldg_v4(wv + i);
      uint4 o;
      o.x = rms_pair(v[j].x, g.x, rstd);
      o.y = rms_pair(v[j].y, g.y, rstd);
      o.z = rms_pair(v[j].z, g.z, rstd);
      o.w = rms_pair(v[j].w, g.w, rstd);
      orow[i] = o;
    }
  }
}

}  // namespace

int layernorm_bf16(const __nv_bfloat16* x, const __nv_bfloat16* w, const __nv_bfloat16* b,
                   __nv_bfloat16* out, int rows, int cols, float eps, cudaStream_t stream) {
  VB_CHECK(cols % 8 == 0, "layernorm: cols must be a multiple of 8 (got %d)", cols);
  VB_CHECK(cols * 2 <= 96 * 1024, "layernorm: row too long (%d)", cols);
  if (rows == 0) return 0;
  if (rows >= kWarpRowMinRows && cols <= 8 * 256) {  // many short rows: warp per row (see above)
    VB_CUDA(launch_pdl(layernorm_warp_kernel<8>, dim3((rows + 7) / 8), dim3(kWarpRowThreads), 0, stream, x, w,
                       b, out, rows, cols, eps));
    return 0;
  }
  const size_t smem = static_cast<size_t>(cols) * 2;
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    VB_CUDA(cudaFuncSetAttribute(layernorm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 96 * 1024));
  }
  VB_CUDA(launch_pdl(layernorm_kernel, dim3(rows), dim3(kNormThreads), smem, stream, x, w, b, out, cols, eps));
  return 0;
}

int rmsnorm_bf16(__nv_bfloat16* x_inout, const __nv_bfloat16* residual_add,
                 const __nv_bfloat16* w, __nv_bfloat16* out, int rows, int cols, float eps,
                 cudaStream_t stream) {
  VB_CHECK(cols % 8 == 0, "rmsnorm: cols must be a multiple of 8 (got %d)", cols);
  VB_CHECK(cols * 2 <= 96 * 1024, "rmsnorm: row too long (%d)", cols);
  if (rows == 0) return 0;
  // rows of up to 2048 elements only: at 3584 (Qwen2-7B) the 14 vectors per lane cost 128 registers,
  // i.e. fewer resident warps than one CTA per row keeps busy
  if (rows >= kWarpRowMinRows && cols <= 8 * 256) {
    VB_CUDA(launch_pdl(rmsnorm_warp_kernel<8>, dim3((rows + 7) / 8), dim3(kWarpRowThreads), 0, stream,
                       x_inout, residual_add, w, out, rows, cols, eps));
    return 0;
  }
  const size_t smem = static_cast<size_t>(cols) * 2;
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    VB_CUDA(cudaFuncSetAttribute(rmsnorm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 96 * 1024));
  }
  VB_CUDA(launch_pdl(rmsnorm_kernel, dim3(rows), dim3(kNormThreads), smem, stream, x_inout, residual_add, w,
                     out, cols, eps));
  return 0;
}

}  // namespace vb
