// Host-side support: error string, SM count, TMA descriptor encoding via the driver entry point.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "common.cuh"

namespace vb {

static thread_local char g_last_error[1024] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_last_error; }

bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("VILA_B200_NO_PDL");
    v = (e != nullptr && e[0] == '1') ? 0 : 1;
  }
  return v == 1;
}

int num_sms() {
  static int cached[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (cached[dev] == 0) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cached[dev] = n > 0 ? n : 132;
  }
  return cached[dev];
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e =
        cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = (EncodeTiledFn)p;
  });
  return fn;
}

static CUtensorMapSwizzle swz(uint32_t bytes) {
  switch (bytes) {
    case 32: return CU_TENSOR_MAP_SWIZZLE_32B;
    case 64: return CU_TENSOR_MAP_SWIZZLE_64B;
    case 128: return CU_TENSOR_MAP_SWIZZLE_128B;
    default: return CU_TENSOR_MAP_SWIZZLE_NONE;
  }
}

int make_tmap_nd_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                      const uint64_t* strides_elems /* rank-1 entries, for dims 1.. */,
                      const uint32_t* box, uint32_t swizzle_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  VB_CHECK(fn != nullptr, "cuTensorMapEncodeTiled driver entry point not available");
  cuuint64_t gdim[5];
  cuuint64_t gstride[4];
  cuuint32_t bdim[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    if (i > 0) gstride[i - 1] = strides_elems[i - 1] * 2;
  }
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), gdim,
                  gstride, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz(swizzle_bytes),
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  VB_CHECK(r == CUDA_SUCCESS,
           "cuTensorMapEncodeTiled failed (%d): rank=%d dims=[%llu,%llu,%llu,%llu] box=[%u,%u,%u,%u] "
           "stride1=%llu swizzle=%u base=%p",
           (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
           (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0),
           box[0], rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0,
           (unsigned long long)(rank > 1 ? strides_elems[0] : 0), swizzle_bytes, base);
  return 0;
}

int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                      uint64_t ld_elems, uint32_t box_rows, uint32_t box_cols,
                      uint32_t swizzle_bytes) {
  uint64_t dims[2] = {cols, rows};
  uint64_t strides[1] = {ld_elems};
  uint32_t box[2] = {box_cols, box_rows};
  return make_tmap_nd_bf16(out, base, 2, dims, strides, box, swizzle_bytes);
}

int make_tmap_3d_bf16(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2,
                      uint64_t s1_elems, uint64_t s2_elems, uint32_t b0, uint32_t b1, uint32_t b2,
                      uint32_t swizzle_bytes) {
  uint64_t dims[3] = {d0, d1, d2};
  uint64_t strides[2] = {s1_elems, s2_elems};
  uint32_t box[3] = {b0, b1, b2};
  return make_tmap_nd_bf16(out, base, 3, dims, strides, box, swizzle_bytes);
}

}  // namespace vb
