// Grammar-constrained decoding on the device: vila_apply_token_bitmask_row masks the single-stream graph decoder's
// logits row with the token bitmask of a grammar matcher (GraphDecoder with a grammar, vila_b200/model/qwen2.py).
//
// The rule (stated in numpy by vila_b200/grammar.py, which the tests use), for a bf16 row x [V] and an int32 bitmask
// in xgrammar's layout (token j is allowed iff bit j % 32 of word j / 32 is set; bits at or above V are ignored):
//   allowed j:     y_j = x_j, bit for bit
//   not allowed j: y_j = -inf (0xFF80)
//
// One thread per 8 consecutive entries (one byte of the mask), 256 threads per CTA: 75 CTAs at V = 152,064.  Each
// entry is read and written by the thread that owns it, so in == out (in place) is safe.  Rows that are not 16-byte
// aligned, and the tail of a row whose V is not a multiple of 8, take the element-wise path.  Bytes: one read and one
// write of the row and one read of the mask (~0.6 MB per token at V = 152,064).
#include "common.cuh"
#include "kernels.h"

namespace vb {
namespace {

constexpr int kMaskThreads = 256;
constexpr int kMaskPerThread = 8;
constexpr int kMaskChunk = kMaskThreads * kMaskPerThread;
constexpr unsigned short kNegInf = 0xFF80u;

__global__ void __launch_bounds__(kMaskThreads) token_bitmask_row_kernel(const unsigned short* in,
                                                                         const int32_t* bitmask,
                                                                         unsigned short* out, int V, bool vec) {
  griddep_wait();
  griddep_launch_dependents();
  const int64_t j = (static_cast<int64_t>(blockIdx.x) * kMaskThreads + threadIdx.x) * kMaskPerThread;
  if (j >= V) return;
  const uint32_t bits = (static_cast<uint32_t>(bitmask[j >> 5]) >> (j & 31)) & 0xffu;
  if (vec && j + kMaskPerThread <= V) {
    uint4 v = *reinterpret_cast<const uint4*>(in + j);
    uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const uint32_t keep = (bits >> (2 * e)) & 3u;  // bit 0: the low half (entry 2e), bit 1: the high half
      w[e] = (keep & 1u ? w[e] & 0x0000ffffu : static_cast<uint32_t>(kNegInf)) |
             (keep & 2u ? w[e] & 0xffff0000u : static_cast<uint32_t>(kNegInf) << 16);
    }
    *reinterpret_cast<uint4*>(out + j) = make_uint4(w[0], w[1], w[2], w[3]);
  } else {
    const int n = static_cast<int>(min(static_cast<int64_t>(kMaskPerThread), V - j));
    for (int e = 0; e < n; ++e) out[j + e] = (bits >> e) & 1u ? in[j + e] : kNegInf;
  }
}

}  // namespace

int apply_token_bitmask_row_check(const void* logits, const int32_t* bitmask, const void* out, int V) {
  VB_CHECK(logits && bitmask && out, "apply_token_bitmask_row: logits, bitmask and out are required");
  VB_CHECK(V >= 1, "apply_token_bitmask_row: bad vocabulary size V=%d (>= 1)", V);
  const uintptr_t in = reinterpret_cast<uintptr_t>(logits), o = reinterpret_cast<uintptr_t>(out);
  VB_CHECK((in & 1) == 0 && (o & 1) == 0 && (reinterpret_cast<uintptr_t>(bitmask) & 3) == 0,
           "apply_token_bitmask_row: misaligned pointer");
  const uintptr_t bytes = static_cast<uintptr_t>(V) * 2;
  VB_CHECK(in == o || in + bytes <= o || o + bytes <= in,
           "apply_token_bitmask_row: logits and out must be the same row or not overlap");
  return 0;
}

int apply_token_bitmask_row(const void* logits, const int32_t* bitmask, void* out, int V, cudaStream_t stream) {
  if (int rc = apply_token_bitmask_row_check(logits, bitmask, out, V)) return rc;
  const bool vec = ((reinterpret_cast<uintptr_t>(logits) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
  VB_CUDA(launch_pdl(token_bitmask_row_kernel, dim3((V + kMaskChunk - 1) / kMaskChunk), dim3(kMaskThreads), 0, stream,
                     static_cast<const unsigned short*>(logits), bitmask, static_cast<unsigned short*>(out), V, vec));
  return 0;
}

}  // namespace vb
