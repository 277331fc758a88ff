// OpenAI presence and frequency penalties on the device: vila_apply_penalties for the continuous-batching engine
// (vila_b200/serving.py, penalties=True) and vila_apply_penalties_row for the single-stream graph decoder (GraphDecoder
// with penalties, vila_b200/model/qwen2.py).  Both run the same kernel, templated on the type of the history and of
// the step counter (int64 per row in the batched engine, int32 in the graph decoder).
//
// The rule (stated in numpy by vila_b200/penalties.py, which the tests use), for a row x of bf16 logits with presence
// p, frequency f and c_j the number of times id j occurs among the ids the request generated before this token:
//   c_j > 0:  y_j = bf16_rn(float(x_j) - (fp32(c_j * f) + p))   (each operation rounded to nearest, no FMA)
//   c_j == 0: y_j = x_j, bit for bit
//
// One CTA per (chunk of kPenChunk entries, row).  The CTA first issues the loads of its chunk of the row, so that they
// are in flight while it counts the history ids that fall in the chunk into a shared-memory histogram with integer
// atomics; then each thread writes its entries once.  Nothing depends on which thread counted first, so the output is
// bit-deterministic and a row's bits depend on that row only.  Bytes: one read and one write of each active row, plus
// the history (read once per chunk, from L2 after the first).
#include "common.cuh"
#include "kernels.h"

namespace vb {
namespace {

constexpr int kPenThreads = 256;
constexpr int kPenVec = 2;                              // 16-byte groups of 8 entries per thread
constexpr int kPenChunk = kPenThreads * kPenVec * 8;    // 4096 entries per CTA: 38 CTAs per row at V = 152,064
constexpr int kPenMaxVocab = 8 * 40960;                 // the samplers' limit: the penalised row goes to them

template <typename Idx>
struct PenaltyArgs {
  const __nv_bfloat16* logits;
  int64_t ld;
  const Idx* history;
  const Idx* step;
  const int32_t* position;  // null: every row is active
  const float* presence;
  const float* frequency;
  __nv_bfloat16* out;
  int V, cols;
};

__device__ __forceinline__ uint32_t bf_bits(const __nv_bfloat16* p) {
  return *reinterpret_cast<const unsigned short*>(p);
}

template <typename Idx>
__global__ void __launch_bounds__(kPenThreads) apply_penalties_kernel(PenaltyArgs<Idx> a) {
  __shared__ __align__(16) int count[kPenChunk];
  griddep_wait();
  griddep_launch_dependents();
  const int row = blockIdx.y;
  if (a.position && a.position[row] < 0) return;  // idle row: its output row is left as it is
  const int base = blockIdx.x * kPenChunk;
  const int n_local = min(kPenChunk, a.V - base);
  const __nv_bfloat16* x = a.logits + static_cast<int64_t>(row) * a.ld + base;
  __nv_bfloat16* y = a.out + static_cast<int64_t>(row) * a.V + base;
  const bool vec = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;

  // the chunk's entries, as packed bf16 pairs: thread t holds entries [(k * kPenThreads + t) * 8, ... + 8)
  uint32_t w[kPenVec][4];
#pragma unroll
  for (int k = 0; k < kPenVec; ++k) {
    const int j = (k * kPenThreads + threadIdx.x) * 8;
    if (vec && j + 8 <= n_local) {
      const uint4 v = *reinterpret_cast<const uint4*>(x + j);
      w[k][0] = v.x; w[k][1] = v.y; w[k][2] = v.z; w[k][3] = v.w;
    } else {
#pragma unroll
      for (int e = 0; e < 8; e += 2) {
        const uint32_t lo = j + e < n_local ? bf_bits(x + j + e) : 0u;
        const uint32_t hi = j + e + 1 < n_local ? bf_bits(x + j + e + 1) : 0u;
        w[k][e / 2] = lo | (hi << 16);
      }
    }
  }

  for (int i = threadIdx.x; i < kPenChunk; i += kPenThreads) count[i] = 0;
  __syncthreads();
  const int64_t n_hist = max(int64_t(0), min(static_cast<int64_t>(a.step[row]), static_cast<int64_t>(a.cols)));
  const Idx* h = a.history + static_cast<int64_t>(row) * a.cols;
  for (int64_t i = threadIdx.x; i < n_hist; i += kPenThreads) {
    const int64_t id = static_cast<int64_t>(h[i]) - base;
    if (id >= 0 && id < n_local) atomicAdd(&count[id], 1);  // ids outside [0, V) fall outside every chunk
  }
  __syncthreads();

  const float p = a.presence[row], f = a.frequency[row];
#pragma unroll
  for (int k = 0; k < kPenVec; ++k) {
    const int j = (k * kPenThreads + threadIdx.x) * 8;
    if (j >= n_local) continue;
    const int4 c0 = *reinterpret_cast<const int4*>(count + j);
    const int4 c1 = *reinterpret_cast<const int4*>(count + j + 4);
    const int c[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      if (c[e] > 0) {
        const uint32_t bits = (w[k][e / 2] >> ((e & 1) * 16)) & 0xffffu;
        const float pen = __fadd_rn(__fmul_rn(static_cast<float>(c[e]), f), p);
        const __nv_bfloat16 r = __float2bfloat16_rn(__fsub_rn(__uint_as_float(bits << 16), pen));
        const uint32_t rb = *reinterpret_cast<const unsigned short*>(&r);
        w[k][e / 2] = (w[k][e / 2] & ~(0xffffu << ((e & 1) * 16))) | (rb << ((e & 1) * 16));
      }
    }
    if (vec && j + 8 <= n_local) {
      *reinterpret_cast<uint4*>(y + j) = make_uint4(w[k][0], w[k][1], w[k][2], w[k][3]);
    } else {
      unsigned short* ys = reinterpret_cast<unsigned short*>(y);
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (j + e < n_local) ys[j + e] = static_cast<unsigned short>(w[k][e / 2] >> ((e & 1) * 16));
    }
  }
}

}  // namespace

int apply_penalties_check(const vila_penalty_params& p) {
  VB_CHECK(p.logits && p.history && p.step && p.position && p.presence && p.frequency && p.out,
           "apply_penalties: logits, history, step, position, presence, frequency and out are required");
  VB_CHECK(p.M >= 1 && p.M <= 65535, "apply_penalties: bad row count M=%d (1..65535)", p.M);
  VB_CHECK(p.V >= 1 && p.V <= kPenMaxVocab, "apply_penalties: bad vocabulary size V=%d (1..%d)", p.V, kPenMaxVocab);
  VB_CHECK(p.ld >= p.V, "apply_penalties: row stride %lld is smaller than V=%d", (long long)p.ld, p.V);
  VB_CHECK(p.cols >= 1, "apply_penalties: cols=%d must be >= 1", p.cols);
  VB_CHECK((reinterpret_cast<uintptr_t>(p.logits) & 1) == 0 && (reinterpret_cast<uintptr_t>(p.out) & 1) == 0 &&
               (reinterpret_cast<uintptr_t>(p.history) & 7) == 0 && (reinterpret_cast<uintptr_t>(p.step) & 7) == 0 &&
               (reinterpret_cast<uintptr_t>(p.position) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.presence) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.frequency) & 3) == 0,
           "apply_penalties: misaligned pointer");
  return 0;
}

int apply_penalties(const vila_penalty_params& p, cudaStream_t stream) {
  if (int rc = apply_penalties_check(p)) return rc;
  PenaltyArgs<int64_t> a{static_cast<const __nv_bfloat16*>(p.logits), p.ld, p.history, p.step, p.position, p.presence,
                         p.frequency, static_cast<__nv_bfloat16*>(p.out), p.V, p.cols};
  VB_CUDA(launch_pdl(apply_penalties_kernel<int64_t>, dim3((p.V + kPenChunk - 1) / kPenChunk, p.M), dim3(kPenThreads),
                     0, stream, a));
  return 0;
}

int apply_penalties_row_check(const vila_penalty_row_params& p) {
  VB_CHECK(p.logits && p.history && p.step && p.presence && p.frequency && p.out,
           "apply_penalties_row: logits, history, step, presence, frequency and out are required");
  VB_CHECK(p.V >= 1 && p.V <= kPenMaxVocab, "apply_penalties_row: bad vocabulary size V=%d (1..%d)", p.V,
           kPenMaxVocab);
  VB_CHECK(p.cols >= 1, "apply_penalties_row: cols=%d must be >= 1", p.cols);
  VB_CHECK((reinterpret_cast<uintptr_t>(p.logits) & 1) == 0 && (reinterpret_cast<uintptr_t>(p.out) & 1) == 0 &&
               (reinterpret_cast<uintptr_t>(p.history) & 3) == 0 && (reinterpret_cast<uintptr_t>(p.step) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.presence) & 3) == 0 &&
               (reinterpret_cast<uintptr_t>(p.frequency) & 3) == 0,
           "apply_penalties_row: misaligned pointer");
  return 0;
}

int apply_penalties_row(const vila_penalty_row_params& p, cudaStream_t stream) {
  if (int rc = apply_penalties_row_check(p)) return rc;
  PenaltyArgs<int32_t> a{static_cast<const __nv_bfloat16*>(p.logits), p.V, p.history, p.step, nullptr, p.presence,
                         p.frequency, static_cast<__nv_bfloat16*>(p.out), p.V, p.cols};
  VB_CUDA(launch_pdl(apply_penalties_kernel<int32_t>, dim3((p.V + kPenChunk - 1) / kPenChunk, 1), dim3(kPenThreads), 0,
                     stream, a));
  return 0;
}

}  // namespace vb
