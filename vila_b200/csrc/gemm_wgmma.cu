// Persistent warp-specialised bf16 GEMM for sm_90a:  C[M,N] = epi(A[M,K] · W[N,K]^T)
//
//   * operands staged global -> shared by TMA (cp.async.bulk.tensor, 128B swizzle, K-major) into a
//     kStages-deep mbarrier ring filled by one producer warp
//   * two consumer warpgroups, 64 rows of the 128-row tile each, issue wgmma.mma_async
//     (m64 x BLOCK_N x k16) straight from shared memory; fp32 accumulators live in registers
//   * the epilogue fuses bias / GELU / SwiGLU / residual (+ broadcast "row modulo" residual for
//     position embeddings) on the accumulator fragments
//   * scheduling: data-parallel over output tiles, or STREAM-K (opt-in): the (tile, k-block)
//     iteration space is cut into equal contiguous ranges, each partial tile is parked in its own
//     fp32 workspace slot and the last-arriving CTA sums the slots in a fixed order (deterministic)
//     and applies the epilogue
//   * CTA pairs (2-CTA clusters): a pair computes a 256 x BLOCK_N tile; each CTA loads half of the W
//     tile and TMA-multicasts it to both, halving the W bytes each SM pulls from L2
//   * split-K pairs: a 2-CTA cluster computes one 128 x BLOCK_N tile, each CTA half of the K range;
//     the fp32 partials are exchanged through distributed shared memory
//   * programmatic dependent launch: barrier init / descriptor prefetch and — for parameter
//     matrices — the first pipeline stages of W overlap the predecessor kernel's tail
//
// Replaces the cuBLAS calls behind nn.Linear on the reference hot path:
//   SigLIP q/k/v/out_proj, fc1/fc2      (modeling_siglip.py:384-387,707-715)
//   mm_projector Linear layers          (base_projector.py:145-162)
//   Qwen2 q/k/v/o, gate/up/down, lm_head (modeling_qwen2.py:164-176,223-226)
//   patch-embed conv as im2col GEMM     (modeling_siglip.py:269-275,322-328)
#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace vb {

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 bytes = one 128B-swizzle row
constexpr int kConsumerThreads = 256;               // warps 0-7: two consumer warpgroups
constexpr int kNumThreads = kConsumerThreads + 32;  // warp 8: TMA producer

enum { kModeSingle = 0, kModePair = 1, kModeSplitK2 = 2 };

template <int BLOCK_N, int kStages, int kMode = kModeSingle>
struct GemmSmem {
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kBarrierBytes = 2 * kStages * 8 + 16;
  static constexpr int kTotal = kStages * kStageBytes + kBarrierBytes + 1024;  // + align slack
  // split-K pair exchange buffer ([BLOCK_N/2 columns][128 rows] fp32) reuses the dead stages
  static_assert(kMode != kModeSplitK2 || BLOCK_M * BLOCK_N * 2 <= kStages * kStageBytes, "");
};

__device__ __forceinline__ float2 ld_cg_v2(const float* p) {
  float2 r;
  asm volatile("ld.global.cg.v2.f32 {%0,%1}, [%2];" : "=f"(r.x), "=f"(r.y) : "l"(p));
  return r;
}

// Tile rasterisation: tiles are numbered so that the CTAs working at the same time share operand
// panels in L2.  Plain M-fastest numbering streams the whole A matrix once per N block, so tiles are
// grouped in bands of kBandM M-blocks; inside a band M runs fastest, then N: the concurrent tiles
// touch kBandM A panels and a sliding window of W panels.  With <= kBandM M-blocks (every prefill
// shape up to 1024 tokens) this IS the M-fastest order.
constexpr int kBandM = 8;
__device__ __forceinline__ void tile_coords(int t, int num_m_blocks, int num_n_blocks, int& m_blk, int& n_blk) {
  const int per_band = kBandM * num_n_blocks;
  const int band = t / per_band;
  const int r = t - band * per_band;
  const int m0 = band * kBandM;
  const int bm = min(kBandM, num_m_blocks - m0);
  n_blk = r / bm;
  m_blk = m0 + (r - n_blk * bm);
}

// Work decomposition shared by the producer and the consumers: a CTA walks a sequence of segments
// (tile, [kb0, kb1)).  Data-parallel: whole tiles blockIdx.x, +gridDim.x, ...  Stream-K: the
// contiguous iteration range [it0, it1) of the (tile, k-block) space.
struct Sched {
  int nkb, num_m_blocks, num_tiles;
  int stream_k;
  long it, it_end;  // stream-K
  int tile;         // data-parallel
  int stride;       // data-parallel: tiles between two visits of this CTA (or CTA pair)
  // tile_m: rows of one scheduling tile (128, or 256 for a CTA pair); worker/n_workers: index and
  // number of the units that walk the tile list (CTAs, or CTA pairs)
  __device__ __forceinline__ Sched(int M, int N, int K, int block_n, int stream_k_, int tile_m,
                                   int worker, int n_workers) {
    nkb = (K + BLOCK_K - 1) / BLOCK_K;
    num_m_blocks = (M + tile_m - 1) / tile_m;
    num_tiles = num_m_blocks * ((N + block_n - 1) / block_n);
    stream_k = stream_k_;
    const long total = static_cast<long>(num_tiles) * nkb;
    it = total * worker / n_workers;
    it_end = total * (worker + 1) / n_workers;
    tile = worker;
    stride = n_workers;
  }
  // returns false when done; otherwise the next segment
  __device__ __forceinline__ bool next(int& t, int& kb0, int& kb1) {
    if (stream_k) {
      if (it >= it_end) return false;
      t = static_cast<int>(it / nkb);
      kb0 = static_cast<int>(it - static_cast<long>(t) * nkb);
      const long rem = it_end - it;
      kb1 = (nkb - kb0) < rem ? nkb : kb0 + static_cast<int>(rem);
      it += kb1 - kb0;
      return true;
    }
    if (tile >= num_tiles) return false;
    t = tile;
    kb0 = 0;
    kb1 = nkb;
    tile += stride;
    return true;
  }
};

// Epilogue on one thread's accumulator fragment.  wgmma m64nN layout: acc[4j + 2h + e] is row
// (row0 + 8h), column 8j + col0 + e.  Only n8 groups j in [j_lo, j_hi) are written.
template <int BLOCK_N>
__device__ __forceinline__ void epilogue_store(const float* acc, const GemmEpilogue& epi, __nv_bfloat16* C,
                                               int ldc, int M, int N, int row0, int n_base, int col0,
                                               int j_lo, int j_hi) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + 8 * h;
    if (row >= M) continue;
    const __nv_bfloat16* res_row = nullptr;
    if (epi.residual != nullptr) {
      const int rr = epi.res_row_mod > 0 ? (row % epi.res_row_mod) : row;
      res_row = epi.residual + static_cast<size_t>(rr) * epi.ld_res;
    }
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      if (j < j_lo || j >= j_hi) continue;
      const int n = n_base + 8 * j + col0;
      if (n >= N) continue;
      float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      if (epi.bias != nullptr) {
        const uint32_t b = *reinterpret_cast<const uint32_t*>(epi.bias + n);
        v0 += bf_lo(b);
        v1 += bf_hi(b);
      }
      if (epi.swiglu) {
        // interleaved (gate, up) column pair -> silu(gate) * up, rounding to bf16 at the points the
        // reference's unfused ops do
        const float g = bf16_round(v0), u = bf16_round(v1);
        C[static_cast<size_t>(row) * ldc + (n >> 1)] = __float2bfloat16_rn(bf16_round(silu_f(g)) * u);
        continue;
      }
      if (epi.act != ACT_NONE) {
        const float x0 = bf16_round(v0), x1 = bf16_round(v1);
        if (epi.act == ACT_GELU_TANH) {
          v0 = gelu_tanh_f(x0);
          v1 = gelu_tanh_f(x1);
        } else if (epi.act == ACT_GELU_ERF) {
          v0 = gelu_erf_f(x0);
          v1 = gelu_erf_f(x1);
        } else {
          v0 = silu_f(x0);
          v1 = silu_f(x1);
        }
      }
      if (res_row != nullptr) {
        const uint32_t r = *reinterpret_cast<const uint32_t*>(res_row + n);
        v0 = bf16_round(v0) + bf_lo(r);
        v1 = bf16_round(v1) + bf_hi(r);
      }
      *reinterpret_cast<uint32_t*>(C + static_cast<size_t>(row) * ldc + n) = pack_bf16(v0, v1);
    }
  }
}

template <int BLOCK_N, int kStages, int kMode>
__global__ void __launch_bounds__(kNumThreads, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a,
                       const __grid_constant__ CUtensorMap tmap_w, __nv_bfloat16* __restrict__ C,
                       int ldc, int M, int N, int K, GemmEpilogue epi) {
  using S = GemmSmem<BLOCK_N, kStages, kMode>;
  constexpr bool kPair = kMode == kModePair;
  constexpr bool kSplit2 = kMode == kModeSplitK2;
  constexpr bool kCluster = kPair || kSplit2;
  constexpr int TILE_M = kPair ? 2 * BLOCK_M : BLOCK_M;
  constexpr int kAcc = BLOCK_N / 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * S::kABytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * S::kStageBytes);
  uint64_t* empty_bar = full_bar + kStages;
  uint32_t* last_flag = reinterpret_cast<uint32_t*>(empty_bar + kStages);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_m_blocks = (M + TILE_M - 1) / TILE_M;
  const int num_n_blocks = (N + BLOCK_N - 1) / BLOCK_N;
  const int stream_k = (!kCluster && epi.split_k > 1) ? 1 : 0;
  const uint32_t rank = kCluster ? cluster_ctarank() : 0u;  // CTA within the pair
  const uint32_t mrank = kPair ? rank : 0u;                 // pair mode: which 128 rows of the tile
  const int worker = kCluster ? static_cast<int>(blockIdx.x >> 1) : static_cast<int>(blockIdx.x);
  const int n_workers = kCluster ? static_cast<int>(gridDim.x >> 1) : static_cast<int>(gridDim.x);
  // split-K pair: this CTA's k-block range of its tile
  const int nkb_all = (K + BLOCK_K - 1) / BLOCK_K;
  const int sk_lo = (kSplit2 && rank == 1) ? (nkb_all + 1) / 2 : 0;
  const int sk_hi = (kSplit2 && rank == 0) ? (nkb_all + 1) / 2 : nkb_all;

  if (threadIdx.x == kConsumerThreads) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_w);
#pragma unroll
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      // one arrival per consumer warpgroup (of both CTAs of a pair: the W stage is shared)
      mbar_init(&empty_bar[i], kPair ? 4 : 2);
    }
    fence_barrier_init();
  }
  if (kCluster) cluster_sync_all();  // the peer's barriers exist before any remote signal
  else __syncthreads();
  griddep_launch_dependents();

  if (warp == kConsumerThreads / 32) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      Sched sch(M, N, K, BLOCK_N, stream_k, TILE_M, worker, n_workers);
      constexpr int kWRows = kPair ? BLOCK_N / 2 : BLOCK_N;  // W rows this CTA fetches
      const int a_row_off = static_cast<int>(mrank) * BLOCK_M;
      const int w_row_off = static_cast<int>(mrank) * kWRows;
      auto load_w = [&](int stage, int kb, int n_blk) {
        uint8_t* dst = smem_b + stage * S::kBBytes + w_row_off * (BLOCK_K * 2);
        if (kPair) tma_load_2d_multicast(dst, &tmap_w, &full_bar[stage], kb * BLOCK_K, n_blk * BLOCK_N + w_row_off, 3);
        else tma_load_2d(dst, &tmap_w, &full_bar[stage], kb * BLOCK_K, n_blk * BLOCK_N);
      };
      int stage = 0;
      uint32_t phase = 0;
      int t, kb0, kb1;
      // W is a parameter: fetch its first stages before the dependency wait (A comes after).  Not
      // in pair mode: the multicast writes into the peer, which must have released the stage.
      int pre = 0;
      int pt = 0, pkb0 = 0, pkb1 = 0;
      Sched peek = sch;
      const bool have_first = peek.next(pt, pkb0, pkb1);
      if (kSplit2) {
        pkb0 = sk_lo;
        pkb1 = sk_hi;
      }
      if (!kPair && epi.static_w && have_first) {
        pre = min(kStages, pkb1 - pkb0);
        int m_blk_unused, n_blk;
        tile_coords(pt, num_m_blocks, num_n_blocks, m_blk_unused, n_blk);
        for (int i = 0; i < pre; ++i) {
          mbar_arrive_expect_tx(&full_bar[i], S::kStageBytes);
          load_w(i, pkb0 + i, n_blk);
        }
      }
      griddep_wait();
      bool first = true;
      while (sch.next(t, kb0, kb1)) {
        int m_blk, n_blk;
        tile_coords(t, num_m_blocks, num_n_blocks, m_blk, n_blk);
        if (kSplit2) {
          kb0 = sk_lo;
          kb1 = sk_hi;
        }
        for (int kb = kb0; kb < kb1; ++kb) {
          if (first && (kb - kb0) < pre) {
            // W already in flight for this stage: only A is missing
            tma_load_2d(smem_a + stage * S::kABytes, &tmap_a, &full_bar[stage], kb * BLOCK_K,
                        m_blk * TILE_M + a_row_off);
          } else {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full_bar[stage], S::kStageBytes);
            tma_load_2d(smem_a + stage * S::kABytes, &tmap_a, &full_bar[stage], kb * BLOCK_K,
                        m_blk * TILE_M + a_row_off);
            load_w(stage, kb, n_blk);
          }
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
        first = false;
      }
    }
  } else {
    // ===================== consumer warpgroups: wgmma main loop + epilogue =====================
    const int wg = warp >> 2;                        // 64-row half of the 128-row CTA tile
    const int ctid = threadIdx.x;                    // 0..255
    const int frag_row = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // first of this thread's two rows
    const int col0 = (lane & 3) * 2;
    Sched sch(M, N, K, BLOCK_N, stream_k, TILE_M, worker, n_workers);
    int stage = 0;
    uint32_t phase = 0;
    int t, kb0, kb1;
    float acc[kAcc];
    griddep_wait();  // C / residual / workspace may still be in use by the predecessor
    while (sch.next(t, kb0, kb1)) {
      int m_blk, n_blk;
      tile_coords(t, num_m_blocks, num_n_blocks, m_blk, n_blk);
      if (kSplit2) {
        kb0 = sk_lo;
        kb1 = sk_hi;
      }
      // release the previous k-block's stage once the wgmma reading it has retired (one group kept
      // in flight)
      auto release = [&](int s) {
        __syncwarp();
        if ((warp & 3) == 0 && lane == 0) {
          if (kPair) {
            mbar_arrive_cluster(mapa_u32(smem_u32(&empty_bar[s]), 0));
            mbar_arrive_cluster(mapa_u32(smem_u32(&empty_bar[s]), 1));
          } else {
            mbar_arrive(&empty_bar[s]);
          }
        }
      };
      int prev_stage = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        wgmma_fence_operand<kAcc>(acc);
        wgmma_fence();
        const uint32_t a_base = smem_u32(smem_a + stage * S::kABytes) + wg * (64 * BLOCK_K * 2);
        const uint32_t b_base = smem_u32(smem_b + stage * S::kBBytes);
#pragma unroll
        for (int k = 0; k < BLOCK_K / 16; ++k) {
          // advance 32 bytes (16 bf16) along K inside the 128B swizzle row
          const uint64_t ad = make_wgmma_desc(a_base + k * 32, 16, 1024, kWgmmaSW128);
          const uint64_t bd = make_wgmma_desc(b_base + k * 32, 16, 1024, kWgmmaSW128);
          Wgmma<BLOCK_N>::ss(acc, ad, bd, (kb != kb0 || k != 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        wgmma_fence_operand<kAcc>(acc);
        if (prev_stage >= 0) release(prev_stage);
        prev_stage = stage;
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_operand<kAcc>(acc);
      if (prev_stage >= 0) release(prev_stage);

      const int row0 = m_blk * TILE_M + static_cast<int>(mrank) * BLOCK_M + frag_row;
      const int n_base = n_blk * BLOCK_N;
      int j_lo = 0, j_hi = BLOCK_N / 8;
      if (kSplit2) {
        // park the column half the PEER finalises ([element][thread] -> conflict-free for the writer
        // here and for the peer's DSMEM reads), then meet the peer at the cluster barrier
        named_bar_sync(1, kConsumerThreads);  // both warpgroups are done reading the stages
        // (loops over all n8 groups with compile-time indices keep acc in registers)
        float2* xchg = reinterpret_cast<float2*>(smem_a);
        constexpr int kHalfJ = BLOCK_N / 16;
        const bool mine_low = rank == 0;  // rank 0 finalises columns [0, BLOCK_N/2)
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          if ((j < kHalfJ) == mine_low) continue;
#pragma unroll
          for (int h = 0; h < 2; ++h)
            xchg[((j % kHalfJ) * 2 + h) * kConsumerThreads + ctid] =
                make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
        cluster_sync_all();  // (the producer warp executes the matching barrier after its loop)
        const uint32_t xchg_peer = mapa_u32(smem_u32(xchg), 1u - rank);
        j_lo = static_cast<int>(rank) * kHalfJ;
        j_hi = j_lo + kHalfJ;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          if ((j < kHalfJ) != mine_low) continue;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            // + the peer's partial of the same columns (two operands: order-independent)
            const float2 q =
                ld_dsmem_v2f(xchg_peer + static_cast<uint32_t>(((j % kHalfJ) * 2 + h) * kConsumerThreads + ctid) * 8u);
            acc[4 * j + 2 * h] += q.x;
            acc[4 * j + 2 * h + 1] += q.y;
          }
        }
      }
      const bool partial = stream_k && ((kb0 != 0) || (kb1 != sch.nkb));
      bool finalize = true;
      if (partial) {
        // ---- stream-K partial tile: park the fp32 partial in this segment's own workspace slot
        // (slots are summed later in a fixed order -> deterministic, no atomics on data) ----
        const long total = static_cast<long>(sch.num_tiles) * sch.nkb;
        const long i0 = static_cast<long>(t) * sch.nkb;
        auto cta_of = [&](long i) {
          long g = i * gridDim.x / total;
          while (g + 1 < static_cast<long>(gridDim.x) && total * (g + 1) / gridDim.x <= i) ++g;
          return static_cast<int>(g);
        };
        const int c_first = cta_of(i0);
        const int n_slots = cta_of(i0 + sch.nkb - 1) - c_first + 1;
        const int my_slot = static_cast<int>(blockIdx.x) - c_first;
        const size_t tile_base = static_cast<size_t>(t) * epi.split_k * (BLOCK_M * BLOCK_N);
        float* slot0 = epi.splitk_ws + tile_base;
        float* mine = slot0 + static_cast<size_t>(my_slot) * (BLOCK_M * BLOCK_N);
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h)
            if (row0 + 8 * h < M)  // rows past M are never stored: do not park them either
              *reinterpret_cast<float2*>(mine + (frag_row + 8 * h) * BLOCK_N + 8 * j + col0) =
                  make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        __threadfence();
        named_bar_sync(1, kConsumerThreads);
        if (ctid == 0) {
          const int add = kb1 - kb0;
          const int prev = atomicAdd(&epi.splitk_counters[t], add);
          const int last = (prev + add == sch.nkb) ? 1 : 0;
          if (last) epi.splitk_counters[t] = 0;  // self-cleaning
          *last_flag = last;
        }
        named_bar_sync(1, kConsumerThreads);
        finalize = (*last_flag != 0);
        named_bar_sync(1, kConsumerThreads);  // everyone has read last_flag
        if (finalize) {
          __threadfence();
#pragma unroll
          for (int i = 0; i < kAcc; ++i) acc[i] = 0.f;
          for (int s = 0; s < n_slots; ++s) {  // fixed order: slot 0 (lowest k) first
            const float* wsp = slot0 + static_cast<size_t>(s) * (BLOCK_M * BLOCK_N);
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                if (row0 + 8 * h >= M) continue;
                const float2 q = ld_cg_v2(wsp + (frag_row + 8 * h) * BLOCK_N + 8 * j + col0);
                acc[4 * j + 2 * h] += q.x;
                acc[4 * j + 2 * h + 1] += q.y;
              }
          }
        }
      }
      if (finalize) epilogue_store<BLOCK_N>(acc, epi, C, ldc, M, N, row0, n_base, col0, j_lo, j_hi);
    }
  }

  // split-K pair: matches the consumers' exchange barrier; then the peer may still read this CTA's
  // parked partial.  Pair: the peer's multicasts and barrier arrivals target this CTA until the end.
  if (kSplit2 && warp == kConsumerThreads / 32) cluster_sync_all();
  if (kCluster) cluster_sync_all();
}

// caller-registered scratch for stream-K partial sums (vila_set_workspace)
struct Workspace {
  void* ptr = nullptr;
  size_t bytes = 0;
};
// one registration per DEVICE (a process may drive several GPUs; the scratch is device memory)
Workspace g_ws_dev[64];
inline Workspace& cur_ws() {
  int d = 0;
  cudaGetDevice(&d);
  return g_ws_dev[(d < 0 || d >= 64) ? 0 : d];
}
#define g_ws cur_ws()
constexpr size_t kCounterBytes = 64 * 1024;  // 16384 tile counters

template <int BLOCK_N, int kStages, int kMode = kModeSingle>
int launch_gemm(const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int ldw, __nv_bfloat16* C,
                int ldc, int M, int N, int K, GemmEpilogue epi, int force_stream_k,
                cudaStream_t stream) {
  using S = GemmSmem<BLOCK_N, kStages, kMode>;
  constexpr bool kPair = kMode == kModePair;
  constexpr int TILE_M = kPair ? 2 * BLOCK_M : BLOCK_M;
  CUtensorMap ta, tw;
  if (make_tmap_2d_bf16(&ta, A, M, K, lda, BLOCK_M, BLOCK_K, 128)) return 1;
  if (make_tmap_2d_bf16(&tw, W, N, K, ldw, kPair ? BLOCK_N / 2 : BLOCK_N, BLOCK_K, 128)) return 1;
  auto kern = gemm_bf16_wgmma_kernel<BLOCK_N, kStages, kMode>;
  static PerDeviceOnce attr_once;
  if (attr_once.first()) {
    VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal));
  }
  const int sms = num_sms();
  const int tiles = ((M + TILE_M - 1) / TILE_M) * ((N + BLOCK_N - 1) / BLOCK_N);
  if (kMode == kModeSplitK2) {
    // one 128 x BLOCK_N tile per CTA pair, half of K each; pairs beyond #SMs / 2 run in a later wave
    // (gemm_bf16 only picks this mode when one wave holds every tile)
    if ((K + BLOCK_K - 1) / BLOCK_K < 2) {
      set_last_error("gemm: split-K pairs need >= 2 k-blocks (K=%d)", K);
      return 1;
    }
    epi.split_k = 1;
    VB_CUDA(launch_pdl_cluster(kern, dim3(2 * tiles), dim3(kNumThreads), S::kTotal, stream,
                               dim3(2, 1, 1), ta, tw, C, ldc, M, N, K, epi));
    return 0;
  }
  if (kPair) {
    // data-parallel over 256 x BLOCK_N tiles, one tile at a time per CTA pair
    const int pairs = tiles < sms / 2 ? tiles : sms / 2;
    epi.split_k = 1;
    VB_CUDA(launch_pdl_cluster(kern, dim3(2 * pairs), dim3(kNumThreads), S::kTotal, stream,
                               dim3(2, 1, 1), ta, tw, C, ldc, M, N, K, epi));
    return 0;
  }
  const int nkb = (K + BLOCK_K - 1) / BLOCK_K;
  // stream-K (force_stream_k 1 / 0: on / off, 2: on if the workspace fits, -1: off): fixes SM
  // under-fill at the price of a partial-tile  // fix-up through the workspace
  bool sk = false;
  const long total_it = static_cast<long>(tiles) * nkb;
  const int sk_grid = total_it < sms ? static_cast<int>(total_it) : sms;
  const long ipc = total_it / sk_grid;  // k-iterations per CTA (floor)
  const int max_slots = static_cast<int>((nkb + ipc - 1) / ipc) + 1;
  const size_t need = kCounterBytes + static_cast<size_t>(tiles) * max_slots * BLOCK_M * BLOCK_N * 4;
  const bool ws_ok = g_ws.ptr != nullptr && g_ws.bytes >= need && tiles <= 16384;
  if (force_stream_k == 2) {
    sk = ws_ok;  // the dispatcher's choice: stream-K when the registered workspace holds the partials
  } else if (force_stream_k >= 0) {
    sk = force_stream_k != 0;
  }
  if (sk && !ws_ok) {
    set_last_error("gemm: stream-K needs a registered workspace of >= %zu bytes (vila_set_workspace)",
                   need);
    return 1;
  }
  int grid = tiles < sms ? tiles : sms;
  epi.split_k = 1;
  if (sk) {
    grid = sk_grid;
    epi.split_k = max_slots;  // > 1 selects the stream-K schedule; = workspace slots per tile
    epi.splitk_counters = static_cast<int*>(g_ws.ptr);
    epi.splitk_ws = reinterpret_cast<float*>(static_cast<char*>(g_ws.ptr) + kCounterBytes);
  }
  VB_CUDA(launch_pdl(kern, dim3(grid), dim3(kNumThreads), S::kTotal, stream, ta, tw, C, ldc, M, N,
                     K, epi));
  return 0;
}

int check_args(const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int ldw, __nv_bfloat16* C,
               int ldc, int M, int N, int K, const GemmEpilogue& epi) {
  VB_CHECK(M > 0 && N > 0 && K > 0, "gemm: empty problem M=%d N=%d K=%d", M, N, K);
  VB_CHECK(K % 8 == 0 && lda % 8 == 0 && ldw % 8 == 0,
           "gemm: K, lda, ldw must be multiples of 8 (TMA 16-byte strides): K=%d lda=%d ldw=%d", K,
           lda, ldw);
  VB_CHECK(N % 8 == 0 && ldc % 8 == 0, "gemm: N and ldc must be multiples of 8: N=%d ldc=%d", N,
           ldc);
  VB_CHECK((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0 &&
               (reinterpret_cast<uintptr_t>(C) & 15) == 0,
           "gemm: pointers must be 16-byte aligned");
  if (epi.swiglu) VB_CHECK(N % 32 == 0, "gemm: swiglu epilogue needs N %% 32 == 0 (N=%d)", N);
  return 0;
}

// Few tokens (short-prompt prefill, projector, M <= 384): 128 x 128 tiles, the fastest flavour at
// the q/k/v and o projections of a 279-token prefill on H100; `pair` shares each W tile between the
// two CTAs of a cluster (multicast) instead.
int gemm_skinny(const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int ldw, __nv_bfloat16* C,
                int ldc, int M, int N, int K, const GemmEpilogue& epi, int pair, cudaStream_t stream) {
  if (pair) return launch_gemm<128, 6, kModePair>(A, lda, W, ldw, C, ldc, M, N, K, epi, -1, stream);
  return launch_gemm<128, 6>(A, lda, W, ldw, C, ldc, M, N, K, epi, -1, stream);
}

}  // namespace

// q/k/v projection followed by RoPE + KV-cache append (M <= 384, head_dim 128): the skinny GEMM
// writes q/k/v to C, then rope_kv_append_table rotates q/k in place and scatters k/v into the pools.
// Returns -1 when the shape is not covered (caller: plain GEMM + rope_kv_append).
int gemm_qkv_rope_bf16(const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int ldw, __nv_bfloat16* C,
                       int ldc, int M, int N, int K, const GemmEpilogue& epi, cudaStream_t stream) {
  if (check_args(A, lda, W, ldw, C, ldc, M, N, K, epi)) return 1;
  if (M > 384) return -1;
  VB_CHECK(ldc == N, "gemm_qkv_rope: the q/k/v output must be dense (ldc %d != N %d)", ldc, N);
  GemmEpilogue plain;
  plain.bias = epi.bias;
  plain.static_w = epi.static_w;
  const int rc = gemm_skinny(A, lda, W, ldw, C, ldc, M, N, K, plain, 0, stream);
  if (rc != 0) return rc;
  return rope_kv_append_table(C, epi.rope_table, M, epi.rope_hq, epi.rope_hkv, 128, epi.k_pool, epi.v_pool,
                              epi.page_table, epi.cache_pos0, stream);
}

void get_workspace(void** ptr, size_t* bytes) {
  *ptr = g_ws.ptr;
  *bytes = g_ws.bytes;
}

int set_workspace(void* ptr, size_t bytes) {
  VB_CHECK(ptr == nullptr || bytes >= kCounterBytes + 1024, "workspace too small (%zu bytes)", bytes);
  VB_CHECK((reinterpret_cast<uintptr_t>(ptr) & 255) == 0, "workspace must be 256-byte aligned");
  g_ws.ptr = ptr;
  g_ws.bytes = ptr ? bytes : 0;
  return 0;
}

int gemm_bf16(const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int ldw, __nv_bfloat16* C,
              int ldc, int M, int N, int K, const GemmEpilogue& epi, cudaStream_t stream) {
  if (check_args(A, lda, W, ldw, C, ldc, M, N, K, epi)) return 1;
  VB_CHECK(epi.rope_table == nullptr, "gemm: the fused RoPE epilogue is only available through gemm_qkv_rope_bf16");
  // Tile-shape heuristic, from tools/bench_gemm_dispatch.py on an H100 SXM (table in DESIGN.md §4):
  // 128x256 tiles once they fill ~70 % of the SMs (gate/up, ViT fc1), 128x128 otherwise (q/k/v, o);
  // long-K GEMMs whose 128x128 grid under-fills the SMs split K (down projection at M = 8..279).
  // For N >= 128, 64-wide tiles and the multicast CTA pairs were slower at every shape timed, so
  // neither is picked; 64-wide tiles remain for outputs narrower than 128.
  const int sms = num_sms();
  const int mb = (M + BLOCK_M - 1) / BLOCK_M;
  // Long-K GEMMs with at most one 128x128 tile per SM pair (ViT fc2: 72 tiles, K = 4304; projector):
  // split K over a CTA pair with a DSMEM exchange -> all SMs stream operands.
  const long tiles128 = static_cast<long>(mb) * ((N + 127) / 128);
  const bool split2 = tiles128 <= sms / 2 && K >= 2048 && M * 10 >= mb * BLOCK_M * 9;
  if (split2) return launch_gemm<128, 6, kModeSplitK2>(A, lda, W, ldw, C, ldc, M, N, K, epi, -1, stream);
  if (K >= 8192 && tiles128 < sms) {
    // decode batches (M <= 64: 28 tiles of the down projection) stream K over every SM; a prefill
    // (M = 279: 84 tiles) splits each tile over a CTA pair
    if (tiles128 * 2 <= sms) return launch_gemm<128, 6>(A, lda, W, ldw, C, ldc, M, N, K, epi, 2, stream);
    return launch_gemm<128, 6, kModeSplitK2>(A, lda, W, ldw, C, ldc, M, N, K, epi, -1, stream);
  }
  const long tiles256 = static_cast<long>(mb) * ((N + 255) / 256);
  if (tiles256 * 10 >= 7L * sms)
    return launch_gemm<256, 4>(A, lda, W, ldw, C, ldc, M, N, K, epi, -1, stream);
  if (N < 128) return launch_gemm<64, 8>(A, lda, W, ldw, C, ldc, M, N, K, epi, -1, stream);
  return launch_gemm<128, 6>(A, lda, W, ldw, C, ldc, M, N, K, epi, -1, stream);
}

// test hook: force a tile configuration (block_n in {64,128,256}; +1000 forces stream-K, +2000 off;
// 3000 / 3001: skinny path, single CTA / CTA pair; 4128 / 4256: CTA-pair 256 x BLOCK_N tiles;
// 5128: split-K CTA pairs on 128 x 128 tiles)
int gemm_bf16_cfg(int block_n, const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int ldw,
                  __nv_bfloat16* C, int ldc, int M, int N, int K, const GemmEpilogue& epi,
                  cudaStream_t stream) {
  if (check_args(A, lda, W, ldw, C, ldc, M, N, K, epi)) return 1;
  if (block_n == 4256) return launch_gemm<256, 4, kModePair>(A, lda, W, ldw, C, ldc, M, N, K, epi, -1, stream);
  if (block_n == 4128) return launch_gemm<128, 6, kModePair>(A, lda, W, ldw, C, ldc, M, N, K, epi, -1, stream);
  if (block_n == 5128) return launch_gemm<128, 6, kModeSplitK2>(A, lda, W, ldw, C, ldc, M, N, K, epi, -1, stream);
  if (block_n == 3000 || block_n == 3001) {
    VB_CHECK(M <= 512, "gemm_bf16_cfg: the skinny path handles M <= 512 (M=%d)", M);
    return gemm_skinny(A, lda, W, ldw, C, ldc, M, N, K, epi, block_n - 3000, stream);
  }
  int fsk = -1;
  if (block_n >= 2000) {
    fsk = 0;
    block_n -= 2000;
  } else if (block_n >= 1000) {
    fsk = 1;
    block_n -= 1000;
  }
  switch (block_n) {
    case 64: return launch_gemm<64, 8>(A, lda, W, ldw, C, ldc, M, N, K, epi, fsk, stream);
    case 128: return launch_gemm<128, 6>(A, lda, W, ldw, C, ldc, M, N, K, epi, fsk, stream);
    case 256: return launch_gemm<256, 4>(A, lda, W, ldw, C, ldc, M, N, K, epi, fsk, stream);
    default: set_last_error("gemm_bf16_cfg: unsupported block_n %d", block_n); return 1;
  }
}

}  // namespace vb
