// Test hooks for the programmatic-dependent-launch (PDL) contract of every kernel (tests/test_pdl_gpu.py).
//
// Every vila_* kernel is launched with launch_pdl and triggers its dependents at or near its top, so the next kernel
// in the stream can become resident while this one still runs.  A consumer is correct only if it reads nothing its
// predecessor produces, and writes nothing its predecessor still reads, before griddep_wait().  A torch kernel never
// triggers early, so a consumer launched after torch ops never exercises that window.  These hooks make it visible:
//
//   pdl_late_kernel   a producer that triggers its dependents first, then spins on %globaltimer for delay_ns, then
//                     copies every "snapshot" range (the consumer's outputs) to a side buffer, then every "late"
//                     range (the consumer's true inputs) from staging into place.  A consumer launched right after it
//                     runs its pre-wait part while the inputs still hold poison and before the snapshot is taken.
//   pdl_probe_kernel  the positive control: seen[0] = *flag before its wait, seen[1] = *flag after.  After a late
//                     producer that flips flag, seen == (old, new) proves that the window exists.
//
// Both copy phases split every range over the grid the same way, so when a snapshot range and a late range cover the
// same bytes (an in-place buffer), each byte is snapshotted by the thread that later overwrites it.
#include "common.cuh"
#include "kernels.h"

namespace vb {
namespace {

constexpr int kLateCtas = 8;  // small, so the consumer has free SMs while the producer spins
constexpr int kLateThreads = 256;
constexpr int kMaxCopies = 64;
constexpr int64_t kMaxDelayNs = 2000000;      // 2 ms
constexpr uint32_t kMaxSpinIters = 1u << 20;  // with the 256 ns sleep: a hard bound on the spin, whatever the timer

__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// [src, src + bytes) -> [dst, ...): 16-byte chunks when both ends allow it, single bytes otherwise.  Chunk c goes to
// global thread c % (grid threads), so the partition depends on (dst, src, bytes) alone.
__device__ void grid_copy(const vila_pdl_copy& c) {
  const int64_t tid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t nthreads = static_cast<int64_t>(gridDim.x) * blockDim.x;
  const uint8_t* src = static_cast<const uint8_t*>(c.src);
  uint8_t* dst = static_cast<uint8_t*>(c.dst);
  const bool vec = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
  int64_t done = 0;
  if (vec) {
    const int64_t n16 = c.bytes >> 4;
    for (int64_t i = tid; i < n16; i += nthreads)
      reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
    done = n16 << 4;
  }
  for (int64_t i = done + tid; i < c.bytes; i += nthreads) dst[i] = src[i];
}

__global__ void __launch_bounds__(kLateThreads) pdl_late_kernel(const vila_pdl_copy* snap, int n_snap,
                                                                 const vila_pdl_copy* late, int n_late,
                                                                 int64_t delay_ns) {
  griddep_launch_dependents();
  griddep_wait();  // the copy lists and staging buffers come from ordinary stream work before this launch
  const uint64_t t0 = globaltimer_ns();
  for (uint32_t it = 0; it < kMaxSpinIters; ++it) {
    if (globaltimer_ns() - t0 >= static_cast<uint64_t>(delay_ns)) break;
    __nanosleep(256);
  }
  for (int i = 0; i < n_snap; ++i) grid_copy(snap[i]);
  for (int i = 0; i < n_late; ++i) grid_copy(late[i]);
}

__global__ void pdl_probe_kernel(const int32_t* flag, int32_t* seen) {
  if (threadIdx.x != 0) return;
  seen[0] = *reinterpret_cast<const volatile int32_t*>(flag);
  griddep_wait();
  seen[1] = *reinterpret_cast<const volatile int32_t*>(flag);
}

}  // namespace

int pdl_late_check(const vila_pdl_copy* snap, int n_snap, const vila_pdl_copy* late, int n_late, int64_t delay_ns) {
  VB_CHECK(delay_ns >= 0 && delay_ns <= kMaxDelayNs, "test_pdl_late: delay_ns=%lld outside [0, %lld]",
           static_cast<long long>(delay_ns), static_cast<long long>(kMaxDelayNs));
  VB_CHECK(n_snap >= 0 && n_snap <= kMaxCopies && n_late >= 0 && n_late <= kMaxCopies,
           "test_pdl_late: n_snap=%d and n_late=%d must be in [0, %d]", n_snap, n_late, kMaxCopies);
  VB_CHECK((n_snap == 0 || snap != nullptr) && (n_late == 0 || late != nullptr),
           "test_pdl_late: a non-empty copy list needs its device array");
  VB_CHECK(((reinterpret_cast<uintptr_t>(snap) | reinterpret_cast<uintptr_t>(late)) & 7) == 0,
           "test_pdl_late: misaligned copy list");
  return 0;
}

int pdl_late(const vila_pdl_copy* snap, int n_snap, const vila_pdl_copy* late, int n_late, int64_t delay_ns,
             cudaStream_t stream) {
  if (int rc = pdl_late_check(snap, n_snap, late, n_late, delay_ns)) return rc;
  VB_CUDA(launch_pdl(pdl_late_kernel, dim3(kLateCtas), dim3(kLateThreads), 0, stream, snap, n_snap, late, n_late,
                     delay_ns));
  return 0;
}

int pdl_probe_check(const int32_t* flag, const int32_t* seen) {
  VB_CHECK((flag == nullptr) == (seen == nullptr), "test_pdl_probe: flag and seen go together");
  VB_CHECK(((reinterpret_cast<uintptr_t>(flag) | reinterpret_cast<uintptr_t>(seen)) & 3) == 0,
           "test_pdl_probe: misaligned pointer");
  return 0;
}

int pdl_probe(const int32_t* flag, int32_t* seen, cudaStream_t stream) {
  if (int rc = pdl_probe_check(flag, seen)) return rc;
  VB_CUDA(launch_pdl(pdl_probe_kernel, dim3(1), dim3(32), 0, stream, flag, seen));
  return 0;
}

}  // namespace vb
