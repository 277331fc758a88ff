// Block digests of a bf16 prompt for prefix caching in the continuous-batching engine (vila_b200/serving.py,
// prefix_cache=True): vila_prefix_block_hash.
//
// The rule (stated in numpy by vila_b200/prefix_cache.py, which the tests use), for each full block b of 128 rows
// of a [rows, cols] bf16 matrix with row stride ld (elements) and two 64-bit keys:
//   w_j      the j-th 8-byte little-endian word of the block's 128 rows, read row-major over the cols logical
//            columns (cols / 4 words per row; the ld padding is not read)
//   fmix64   the murmur3 64-bit finalizer
//   d_L      sum over j of fmix64(fmix64(w_j ^ key_L) + j * 0x9E3779B97F4A7C15) mod 2^64, L = 0, 1
// The sums are mod 2^64, so the digest does not depend on the order of the reduction.  Not cryptographic: the keys
// are drawn at random per engine so that colliding blocks cannot be prepared in advance.
//
// One CTA of 1024 threads per block: the CTA reads the block's 128 * cols * 2 bytes once (8-byte loads, four in
// flight per thread), each thread keeps two running sums, and a warp-shuffle plus shared-memory reduction writes
// out[b] = (d_0, d_1).  A 16,470 x 3584 prompt is 128 CTAs, one wave on the H100's 132 SMs.
#include "common.cuh"
#include "kernels.h"

namespace vb {
namespace {

constexpr int kHashThreads = 1024;
constexpr int kHashWarps = kHashThreads / 32;
constexpr int kHashRows = 128;
constexpr int kHashUnroll = 4;
constexpr unsigned long long kGolden = 0x9E3779B97F4A7C15ull;

__device__ __forceinline__ unsigned long long fmix64(unsigned long long k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return k;
}

struct HashArgs {
  const unsigned long long* x;  // row r starts at x + r * ldw
  int64_t ldw;                  // row stride in 8-byte words
  int W;                        // words per row (cols / 4)
  unsigned long long key0, key1;
  unsigned long long* out;      // [blocks][2]
};

__global__ void __launch_bounds__(kHashThreads) prefix_block_hash_kernel(HashArgs a) {
  griddep_launch_dependents();
  griddep_wait();
  __shared__ unsigned long long part[kHashWarps][2];
  const unsigned long long* base = a.x + static_cast<int64_t>(blockIdx.x) * kHashRows * a.ldw;
  const int W = a.W;
  const int64_t total = static_cast<int64_t>(kHashRows) * W;
  // word j sits at row r = j / W, column word c = j % W; advancing j by the CTA width moves (r, c) by (qs, rs)
  const int qs = kHashThreads / W, rs = kHashThreads % W;
  int64_t j = threadIdx.x;
  int r = static_cast<int>(j / W), c = static_cast<int>(j % W);
  unsigned long long s0 = 0, s1 = 0;
  for (; j + (kHashUnroll - 1) * kHashThreads < total; j += kHashUnroll * kHashThreads) {
    unsigned long long w[kHashUnroll];
#pragma unroll
    for (int u = 0; u < kHashUnroll; ++u) {
      w[u] = __ldcs(base + r * a.ldw + c);
      r += qs;
      c += rs;
      if (c >= W) c -= W, ++r;
    }
#pragma unroll
    for (int u = 0; u < kHashUnroll; ++u) {
      const unsigned long long salt = static_cast<unsigned long long>(j + u * kHashThreads) * kGolden;
      s0 += fmix64(fmix64(w[u] ^ a.key0) + salt);
      s1 += fmix64(fmix64(w[u] ^ a.key1) + salt);
    }
  }
  for (; j < total; j += kHashThreads) {
    const unsigned long long w = __ldcs(base + r * a.ldw + c);
    r += qs;
    c += rs;
    if (c >= W) c -= W, ++r;
    const unsigned long long salt = static_cast<unsigned long long>(j) * kGolden;
    s0 += fmix64(fmix64(w ^ a.key0) + salt);
    s1 += fmix64(fmix64(w ^ a.key1) + salt);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s0 += __shfl_down_sync(0xffffffffu, s0, o);
    s1 += __shfl_down_sync(0xffffffffu, s1, o);
  }
  const int warp = threadIdx.x >> 5;
  if (lane_id() == 0) {
    part[warp][0] = s0;
    part[warp][1] = s1;
  }
  __syncthreads();
  if (warp == 0) {
    s0 = part[lane_id()][0];
    s1 = part[lane_id()][1];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s0 += __shfl_down_sync(0xffffffffu, s0, o);
      s1 += __shfl_down_sync(0xffffffffu, s1, o);
    }
    if (lane_id() == 0) {
      a.out[2 * blockIdx.x] = s0;
      a.out[2 * blockIdx.x + 1] = s1;
    }
  }
}

}  // namespace

int prefix_block_hash_check(const void* x, int64_t ld, int64_t rows, int64_t cols, const uint64_t* out) {
  VB_CHECK(rows >= 0 && cols > 0 && cols % 4 == 0,
           "vila_prefix_block_hash: cols must be a positive multiple of 4 (rows=%lld, cols=%lld)", (long long)rows,
           (long long)cols);
  VB_CHECK(ld >= cols && ld % 4 == 0,
           "vila_prefix_block_hash: ld must be a multiple of 4 and >= cols (ld=%lld, cols=%lld)", (long long)ld,
           (long long)cols);
  VB_CHECK(cols / 4 <= 0x7fffffffLL && rows / kHashRows <= 0x7fffffffLL,
           "vila_prefix_block_hash: shape too large (rows=%lld, cols=%lld)", (long long)rows, (long long)cols);
  if (rows < kHashRows) return 0;
  VB_CHECK(x != nullptr && out != nullptr, "vila_prefix_block_hash: x and out are required");
  VB_CHECK((reinterpret_cast<uintptr_t>(x) & 7) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0,
           "vila_prefix_block_hash: x and out must be 8-byte aligned");
  return 0;
}

int prefix_block_hash(const void* x, int64_t ld, int64_t rows, int64_t cols, uint64_t key0, uint64_t key1,
                      uint64_t* out, cudaStream_t stream) {
  const int64_t blocks = rows / kHashRows;
  if (blocks == 0) return 0;
  HashArgs a{static_cast<const unsigned long long*>(x), ld / 4, static_cast<int>(cols / 4), key0, key1,
             reinterpret_cast<unsigned long long*>(out)};
  VB_CUDA(launch_pdl(prefix_block_hash_kernel, dim3(static_cast<unsigned>(blocks)), dim3(kHashThreads), 0, stream,
                     a));
  return 0;
}

}  // namespace vb
