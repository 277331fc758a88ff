// vila_b200 — sm_90a PTX helper layer (mbarrier / TMA / clusters / wgmma descriptors).
// Everything in this file is hand-written inline PTX for Hopper (H100, sm_90a).
// No CUTLASS / CuTe / Triton. Bit layouts of the matrix descriptors follow the PTX ISA
// "wgmma matrix descriptor" table.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vb {

// ----------------------------------------------------------------------------------------------
// error handling (C-ABI returns int error codes; message retrievable via vila_last_error())
// ----------------------------------------------------------------------------------------------
void set_last_error(const char* fmt, ...);

#define VB_CHECK(cond, ...)                       \
  do {                                            \
    if (!(cond)) {                                \
      ::vb::set_last_error(__VA_ARGS__);          \
      return 1;                                   \
    }                                             \
  } while (0)

#define VB_CUDA(expr)                                                                   \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      ::vb::set_last_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),      \
                           __FILE__, __LINE__);                                         \
      (void)cudaGetLastError(); /* do not leave a stale error for the caller's runtime */ \
      return 2;                                                                         \
    }                                                                                   \
  } while (0)

// ----------------------------------------------------------------------------------------------
// small device utilities
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- activations (shared by the GEMM / GEMV epilogues).  The division is the fast one
// (MUFU.RCP + FMUL, ~1 ulp): the IEEE fp32 division's slow path cost ~20 instructions per element
// in the epilogues, and every result is rounded to bf16 right after.
__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
__device__ __forceinline__ float gelu_tanh_f(float x) {
  // gelu_pytorch_tanh: 0.5 x (1 + tanh( sqrt(2/pi) (x + 0.044715 x^3) ))
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float u = k0 * (x + k1 * x * x * x);
  const float t = 1.0f - __fdividef(2.0f, __expf(2.0f * u) + 1.0f);
  return 0.5f * x * (1.0f + t);
}
__device__ __forceinline__ float gelu_erf_f(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.7071067811865476f));
}

// ---- programmatic dependent launch (PDL) device side ----
// wait: all prerequisite grids have completed and their memory is visible (no-op without PDL)
__device__ __forceinline__ void griddep_wait() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
// allow the dependent grid to start launching as SM resources free up
__device__ __forceinline__ void griddep_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
// asynchronous bulk prefetch of [p, p+bytes) into L2 (bytes % 16 == 0)
__device__ __forceinline__ void prefetch_l2_bulk(const void* p, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}

// streaming 128-bit global load (read once: do not allocate in L1)
__device__ __forceinline__ uint4 ldg_stream(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ uint4 ldg_v4(const void* p) {
  return *reinterpret_cast<const uint4*>(p);
}
__device__ __forceinline__ void stg_v4(void* p, uint4 v) { *reinterpret_cast<uint4*>(p) = v; }

__device__ __forceinline__ float bf_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf_hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_round(float x) {
  return __bfloat162float(__float2bfloat16_rn(x));
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// make generic-proxy smem writes visible to the async proxy (TMA / wgmma)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) — loads arrive on an mbarrier with complete_tx::bytes
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0),
        "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int32_t c0, int32_t c1, int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0),
        "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int32_t c0, int32_t c1, int32_t c2, int32_t c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0),
        "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ----------------------------------------------------------------------------------------------
// TMA multicast and thread-block clusters
// ----------------------------------------------------------------------------------------------
// 2D TMA load delivered to the same shared-memory offset in every CTA of `cta_mask` (this cluster);
// each destination CTA's mbarrier at the offset of `bar` receives the complete_tx of its copy
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                                      int32_t c0, int32_t c1, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0),
        "r"(c1), "h"(cta_mask)
      : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of the same shared-memory offset in CTA `rank` of this cluster
__device__ __forceinline__ uint32_t mapa_u32(uint32_t smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ float2 ld_dsmem_v2f(uint32_t cluster_addr) {
  float2 v;
  asm volatile("ld.shared::cluster.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(cluster_addr));
  return v;
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr)
               : "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor (sm_90a), 64-bit:
//   [0,14) start_address>>4  [16,30) leading_byte_offset>>4  [32,46) stride_byte_offset>>4
//   [49,52) base_offset (0: every swizzle atom here is 1024-byte aligned)  [62,64) layout
// K-major swizzled operands: SBO = pitch of 8-row groups, LBO unused; a k-step inside the swizzle
// row advances the start address.  MN-major: LBO = pitch of swizzle-width column blocks along MN,
// SBO = pitch of 8-row groups along K.
// ----------------------------------------------------------------------------------------------
enum : uint32_t { kWgmmaSW128 = 1, kWgmmaSW64 = 2, kWgmmaSW32 = 3 };
__device__ __forceinline__ uint64_t make_wgmma_desc(uint32_t smem_addr, uint32_t lbo_bytes,
                                                    uint32_t sbo_bytes, uint32_t layout) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3ffffu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3fffu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3fffu) << 32;
  d |= static_cast<uint64_t>(layout) << 62;
  return d;
}
// named barrier over `count` threads (id 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}


// ----------------------------------------------------------------------------------------------
// host: TMA descriptor encoding through the driver entry point (no link-time libcuda dependency)
// ----------------------------------------------------------------------------------------------
// 2D bf16 row-major tensor [rows, cols] with row pitch `ld_elems`; box = [box_rows, box_cols].
// swizzle_bytes in {0, 32, 64, 128}; box_cols*2 must be <= swizzle_bytes when swizzled.
int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                      uint64_t ld_elems, uint32_t box_rows, uint32_t box_cols,
                      uint32_t swizzle_bytes);
// 3D bf16 tensor: dims (fastest first) d0,d1,d2 with strides (elements) s1,s2; box b0,b1,b2
int make_tmap_3d_bf16(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2,
                      uint64_t s1_elems, uint64_t s2_elems, uint32_t b0, uint32_t b1, uint32_t b2,
                      uint32_t swizzle_bytes);
int make_tmap_nd_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                      const uint64_t* strides_elems, const uint32_t* box, uint32_t swizzle_bytes);
int num_sms();
bool pdl_enabled();  // programmatic dependent launch on unless VILA_B200_NO_PDL=1

// Launch with programmatic stream serialization (PDL): the kernel may become resident while its
// predecessor in the stream is still draining; it must execute griddep_wait() before touching
// anything the predecessor produced (or that the predecessor still reads). Works inside CUDA-graph
// capture (programmatic dependency edges).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_cluster(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                      cudaStream_t stream, dim3 cluster, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster.x * cluster.y * cluster.z > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster.x;
    attr[n].val.clusterDim.y = cluster.y;
    attr[n].val.clusterDim.z = cluster.z;
    ++n;
  }
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem,
                              cudaStream_t stream, Args... args) {
  return launch_pdl_cluster(kern, grid, block, smem, stream, dim3(1, 1, 1), args...);
}
const char* last_error();

// One-time per-DEVICE setup guard (cudaFuncSetAttribute is per device; a process may drive several).
struct PerDeviceOnce {
  bool done[64] = {};
  bool first() {
    int d = 0;
    cudaGetDevice(&d);
    if (d < 0 || d >= 64) d = 0;
    if (done[d]) return false;
    done[d] = true;
    return true;
  }
};

}  // namespace vb
