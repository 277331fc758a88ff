// Persistent decode "mega-kernel" for sm_90a: ALL layers of n_tokens greedy decode steps in ONE launch.
//
// Why: at batch 1 the decode step is pure weight streaming (15.2 GB / token).  As separate kernels
// (5 per layer) every kernel boundary drains the HBM pipe for a few microseconds (tail, launch,
// x staging, first-byte latency).  Here one CTA per SM stays resident; each of its 8 warps owns a
// shared-memory ring that its lane 0 keeps filled with cp.async.bulk (1-D TMA) copies of weight-row
// chunks, and that ring runs AHEAD ACROSS PHASE AND TOKEN BOUNDARIES (weights never depend on
// activations), so while a CTA waits at a grid barrier or stages the next activation vector its next
// ~170 KB of weights are already landing.  Phases of one layer (grid barrier after each):
//     qkv = Wqkv·rmsnorm(x)+b | RoPE + KV append + split-KV attention (first Hkv*splits CTAs)
//     x += Wo·attn (the split partials are combined while staging the vector) |
//     act = SwiGLU(Wgu·rmsnorm(x)) | x += Wdown·act
// then lm_head·rmsnorm(x) with a fused arg-max, and a finalize phase (token history, position++, next
// embedding) — the loop never returns to the host.
//
// Arithmetic and rounding points are those of gemv_tma.cu / decode.cu (same parity tests).
#include <math.h>

#include "common.cuh"
#include "kernels.h"

namespace vb {
namespace {

constexpr int MW = 8;            // consumer warps
constexpr int MT = MW * 32;
constexpr int MSTAGES = 3;       // ring slots per warp
constexpr int SLOT = 7168;       // bytes per slot (one 3584-element bf16 row)
constexpr int MD = 128;          // head dim
constexpr int ACC_FLOATS = 2304;

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
__device__ __forceinline__ uint32_t float_order(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ uint4 ldcg_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ float ldcg_bf16(const __nv_bfloat16* p) {
  unsigned short v;
  asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(v) : "l"(p));
  return __uint_as_float(static_cast<uint32_t>(v) << 16);
}

__device__ __forceinline__ void grid_sync(unsigned int* bar, unsigned int target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(bar, 1u);
    unsigned int v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
    } while (static_cast<int>(v - target) < 0);
    __threadfence();
  }
  __syncthreads();
}

struct GPhase {
  const __nv_bfloat16* w;
  int N, K, ks, rpb, kind;  // kind: 0 qkv, 1 o, 2 gate/up, 3 down, 4 lm_head
};

__device__ __forceinline__ GPhase get_phase(const MegaParams& p, int g /* 0 .. 4L */) {
  GPhase ph;
  const int L = p.num_layers;
  const int grid = gridDim.x;
  if (g == 4 * L) {
    ph.w = p.lm_head_w; ph.N = p.vocab; ph.K = p.hidden; ph.ks = p.ks_hidden; ph.kind = 4;
  } else {
    const MegaLayer& ly = p.layers[g >> 2];
    const int k = g & 3;
    ph.kind = k;
    if (k == 0) { ph.w = ly.qkv_w; ph.N = (p.Hq + 2 * p.Hkv) * MD; ph.K = p.hidden; ph.ks = p.ks_hidden; }
    else if (k == 1) { ph.w = ly.o_w; ph.N = p.hidden; ph.K = p.Hq * MD; ph.ks = p.ks_attn; }
    else if (k == 2) { ph.w = ly.gu_w; ph.N = 2 * p.inter; ph.K = p.hidden; ph.ks = p.ks_hidden; }
    else { ph.w = ly.down_w; ph.N = p.hidden; ph.K = p.inter; ph.ks = p.ks_inter; }
  }
  int rpb = (ph.N + grid - 1) / grid;
  if (ph.kind == 2 && (rpb & 1)) rpb += 1;
  ph.rpb = rpb;
  return ph;
}

template <int G>
__global__ void __launch_bounds__(MT, 1) decode_mega_kernel(MegaParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  // layout: [xs: p.xs_bytes][acc: ACC_FLOATS f32][ring: MW*MSTAGES*SLOT][bars]
  uint4* xs = reinterpret_cast<uint4*>(smem);
  float* acc = reinterpret_cast<float*>(smem + p.xs_bytes);
  uint8_t* ring = smem + p.xs_bytes + ACC_FLOATS * 4;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + MW * MSTAGES * SLOT);
  MegaLayer* layers_s = reinterpret_cast<MegaLayer*>(bars + MW * MSTAGES);  // [num_layers] copy
  __shared__ float red[32];
  __shared__ unsigned long long best_s;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cta = blockIdx.x, grid = gridDim.x;
  const int L = p.num_layers;
  const int gphases_per_token = 4 * L + 1;
  const int total_gphases = gphases_per_token * p.n_tokens;
  uint8_t* my_ring = ring + warp * MSTAGES * SLOT;
  uint64_t* my_bars = bars + warp * MSTAGES;

  if (lane == 0) {
    for (int s = 0; s < MSTAGES; ++s) mbar_init(&my_bars[s], 1);
    fence_barrier_init();
  }
  {  // the per-layer pointer table is read on every chunk issue: keep it in shared memory
    const uint64_t* src = reinterpret_cast<const uint64_t*>(p.layers);
    uint64_t* dst = reinterpret_cast<uint64_t*>(layers_s);
    for (int i = threadIdx.x; i < p.num_layers * static_cast<int>(sizeof(MegaLayer) / 8); i += MT) dst[i] = src[i];
  }
  __syncthreads();
  p.layers = layers_s;

  unsigned int sync_target = *reinterpret_cast<volatile unsigned int*>(p.epoch);
  long long* dbg = p.debug_times;  // optional [n_phases][6] clock64 stamps of CTA `debug_cta`
  int dbg_i = 0;
  auto stamp = [&](int k) {
    if (dbg != nullptr && cta == p.debug_cta && threadIdx.x == 0) dbg[dbg_i * 6 + k] = clock64();
  };

  // ---------------- ring producer (lane 0 of every warp) ----------------
  int issued = 0, consumed = 0;    // chunks of this warp
  int pg = 0, pj = 0;              // producer cursor: global phase, item index within this warp's items
  auto my_items = [&](const GPhase& ph) {
    const int nrows = min(ph.rpb, ph.N - cta * ph.rpb);
    const int items = nrows > 0 ? nrows * ph.ks : 0;
    return items > warp ? (items - warp + MW - 1) / MW : 0;
  };
  // cached description of the producer's current phase (refreshed only when pg changes)
  int pg_in_tok = 0, p_nmy = 0, p_ks = 1, p_ce = 0, p_K = 0;
  const __nv_bfloat16* p_wbase = nullptr;  // first row of this CTA's slab
  auto producer_load_phase = [&]() {
    const GPhase ph = get_phase(p, pg_in_tok);
    p_nmy = my_items(ph);
    p_ks = ph.ks;
    p_K = ph.K;
    p_ce = ph.K / ph.ks;
    p_wbase = ph.w + static_cast<size_t>(cta) * ph.rpb * ph.K;
  };
  producer_load_phase();
  auto producer_advance = [&]() {  // lane 0 only
    while (issued - consumed < MSTAGES && pg < total_gphases) {
      if (pj >= p_nmy) {
        ++pg;
        pj = 0;
        if (++pg_in_tok == gphases_per_token) pg_in_tok = 0;
        if (pg < total_gphases) producer_load_phase();
        continue;
      }
      const int item = warp + pj * MW;
      const int r = item / p_ks, part = item - r * p_ks;
      const __nv_bfloat16* src = p_wbase + static_cast<size_t>(r) * p_K + part * p_ce;
      const int s = issued % MSTAGES;
      mbar_arrive_expect_tx(&my_bars[s], p_ce * 2);
      bulk_g2s(my_ring + s * SLOT, src, p_ce * 2, &my_bars[s]);
      ++issued;
      ++pj;
    }
  };
  if (lane == 0) producer_advance();

  for (int tok = 0; tok < p.n_tokens; ++tok) {
    for (int g = 0; g < gphases_per_token; ++g) {
      const GPhase ph = get_phase(p, g);
      const int layer = g >> 2;
      const int row0 = cta * ph.rpb;
      const int nrows = max(0, min(ph.rpb, ph.N - row0));
      const int nvec = ph.K >> 3;

      stamp(0);
      // ================= attention phase (before the o_proj GEMV of each layer) =================
      if (ph.kind == 1) {
        if (cta < p.Hkv * p.splits) {
          const MegaLayer& ly = p.layers[layer];
          const int hk = cta / p.splits, split = cta - hk * p.splits;
          float* q_s = reinterpret_cast<float*>(smem);                      // [G][128]
          __nv_bfloat16* knew_s = reinterpret_cast<__nv_bfloat16*>(q_s + G * MD);
          __nv_bfloat16* vnew_s = knew_s + MD;
          float* red_m = reinterpret_cast<float*>(vnew_s + MD);              // [MW][G]
          float* red_l = red_m + MW * G;                                     // [MW][G]
          float* red_o = red_l + MW * G;                                     // [MW][G][128]
          const int sub = lane >> 4, dl = lane & 15;
          const int pos = *reinterpret_cast<volatile int*>(p.position);
          const int n_tok = pos + 1;
          constexpr int TB = 4;
          const int per = (n_tok + p.splits - 1) / p.splits;
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
                const size_t o = ((static_cast<size_t>(page) * 128 + (t & 127)) * p.Hkv + hk) * MD + dl * 8;
                kreg[i] = ldcg_v4(ly.k_pool + o);
                vreg[i] = ldcg_v4(ly.v_pool + o);
              }
            }
          };
          load_batch(t0);
          // RoPE on the G query heads and the new key
          for (int idx = threadIdx.x; idx < (G + 1) * (MD / 2); idx += MT) {
            const int hh = idx / (MD / 2), i = idx % (MD / 2);
            const __nv_bfloat16* src = hh < G ? p.qkv + (hk * G + hh) * MD : p.qkv + (p.Hq + hk) * MD;
            const float x0 = ldcg_bf16(src + i), x1 = ldcg_bf16(src + i + MD / 2);
            const float ang = static_cast<float>(pos) * p.inv_freq[i];
            float sn, cs;
            sincosf(ang, &sn, &cs);
            cs = bf16_round(cs);
            sn = bf16_round(sn);
            const float y0 = bf16_round(bf16_round(x0 * cs) + bf16_round(-x1 * sn));
            const float y1 = bf16_round(bf16_round(x1 * cs) + bf16_round(x0 * sn));
            if (hh < G) {
              q_s[hh * MD + i] = y0;
              q_s[hh * MD + i + MD / 2] = y1;
            } else {
              knew_s[i] = __float2bfloat16(y0);
              knew_s[i + MD / 2] = __float2bfloat16(y1);
            }
          }
          for (int i = threadIdx.x; i < MD; i += MT)
            vnew_s[i] = __float2bfloat16(ldcg_bf16(p.qkv + (p.Hq + p.Hkv + hk) * MD + i));
          __syncthreads();
          if (split == 0) {
            const int page = p.page_table[pos >> 7];
            const size_t o = ((static_cast<size_t>(page) * 128 + (pos & 127)) * p.Hkv + hk) * MD;
            for (int i = threadIdx.x; i < MD; i += MT) {
              ly.k_pool[o + i] = knew_s[i];
              ly.v_pool[o + i] = vnew_s[i];
            }
          }
          float qreg[G][8];
#pragma unroll
          for (int gq = 0; gq < G; ++gq)
#pragma unroll
            for (int e = 0; e < 8; ++e) qreg[gq][e] = q_s[gq * MD + dl * 8 + e];
          float m[G], l[G], o_acc[G][8];
#pragma unroll
          for (int gq = 0; gq < G; ++gq) {
            m[gq] = -INFINITY;
            l[gq] = 0.f;
#pragma unroll
            for (int e = 0; e < 8; ++e) o_acc[gq][e] = 0.f;
          }
          const float sl2 = p.scale * 1.4426950408889634f;
          for (int base = t0; base < t1; base += 16 * TB) {
            if (base != t0) load_batch(base);
#pragma unroll
            for (int i = 0; i < TB; ++i) {
              const int t = base + hw + 16 * i;
              const bool valid = t < t1;
              uint4 kv = kreg[i], vv = vreg[i];
              if (valid && t == pos) {
                kv = *reinterpret_cast<const uint4*>(knew_s + dl * 8);
                vv = *reinterpret_cast<const uint4*>(vnew_s + dl * 8);
              }
              const float kf[8] = {bf_lo(kv.x), bf_hi(kv.x), bf_lo(kv.y), bf_hi(kv.y),
                                   bf_lo(kv.z), bf_hi(kv.z), bf_lo(kv.w), bf_hi(kv.w)};
              const float vf[8] = {bf_lo(vv.x), bf_hi(vv.x), bf_lo(vv.y), bf_hi(vv.y),
                                   bf_lo(vv.z), bf_hi(vv.z), bf_lo(vv.w), bf_hi(vv.w)};
#pragma unroll
              for (int gq = 0; gq < G; ++gq) {
                float s = 0.f;
#pragma unroll
                for (int e = 0; e < 8; ++e) s = fmaf(qreg[gq][e], kf[e], s);
#pragma unroll
                for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
                if (valid) {
                  s *= sl2;
                  const float m_new = fmaxf(m[gq], s);
                  const float alpha = exp2f(m[gq] - m_new);
                  const float pexp = exp2f(s - m_new);
                  l[gq] = l[gq] * alpha + pexp;
                  const float pb = bf16_round(pexp);
#pragma unroll
                  for (int e = 0; e < 8; ++e) o_acc[gq][e] = o_acc[gq][e] * alpha + pb * vf[e];
                  m[gq] = m_new;
                }
              }
            }
          }
          // combine the two half-warps (lanes l and l^16 hold the same d-slice), then the 8 warps
#pragma unroll
          for (int gq = 0; gq < G; ++gq) {
            const float mo = __shfl_xor_sync(0xffffffffu, m[gq], 16);
            const float lo = __shfl_xor_sync(0xffffffffu, l[gq], 16);
            const float mm = fmaxf(m[gq], mo);
            const float wa = (m[gq] == -INFINITY) ? 0.f : exp2f(m[gq] - mm);
            const float wb = (mo == -INFINITY) ? 0.f : exp2f(mo - mm);
            l[gq] = l[gq] * wa + lo * wb;
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              const float oo = __shfl_xor_sync(0xffffffffu, o_acc[gq][e], 16);
              o_acc[gq][e] = o_acc[gq][e] * wa + oo * wb;
            }
            m[gq] = mm;
            if (lane == 0) {
              red_m[warp * G + gq] = mm;
              red_l[warp * G + gq] = l[gq];
            }
            if (sub == 0) {
#pragma unroll
              for (int e = 0; e < 8; ++e) red_o[(warp * G + gq) * MD + dl * 8 + e] = o_acc[gq][e];
            }
          }
          __syncthreads();
          float* ws_m = p.attn_ws;
          float* ws_l = ws_m + p.Hkv * p.splits * G;
          float* ws_o = ws_l + p.Hkv * p.splits * G;
          for (int idx = threadIdx.x; idx < G * MD; idx += MT) {
            const int gq = idx / MD, d = idx % MD;
            float mm = -INFINITY;
            for (int s = 0; s < MW; ++s) mm = fmaxf(mm, red_m[s * G + gq]);
            float ll = 0.f, oo = 0.f;
            for (int s = 0; s < MW; ++s) {
              const float w = (red_m[s * G + gq] == -INFINITY) ? 0.f : exp2f(red_m[s * G + gq] - mm);
              ll += red_l[s * G + gq] * w;
              oo += red_o[(s * G + gq) * MD + d] * w;
            }
            const size_t b = (static_cast<size_t>(hk) * p.splits + split) * G + gq;
            if (d == 0) {
              ws_m[b] = mm;
              ws_l[b] = ll;
            }
            ws_o[b * MD + d] = oo;
          }
          // the last-arriving split CTA of this KV head combines all splits and publishes the bf16
          // attention vector (so the o_proj phase stages a plain 2*Hq*128-byte vector)
          __shared__ int is_last_s;
          __threadfence();
          __syncthreads();
          if (threadIdx.x == 0) {
            const int prev = atomicAdd(&p.attn_counters[hk], 1);
            is_last_s = (prev == p.splits - 1);
            if (is_last_s) p.attn_counters[hk] = 0;
          }
          __syncthreads();
          if (is_last_s) {
            __threadfence();
            constexpr int MAXS = 16;
            for (int idx = threadIdx.x; idx < G * MD; idx += MT) {
              const int gq = idx / MD, d = idx % MD;
              float ms[MAXS], ls[MAXS], os[MAXS];
#pragma unroll
              for (int s = 0; s < MAXS; ++s) {
                const bool ok = s < p.splits;
                const size_t b = (static_cast<size_t>(hk) * p.splits + (ok ? s : 0)) * G + gq;
                ms[s] = ok ? __ldcg(ws_m + b) : -INFINITY;
                ls[s] = ok ? __ldcg(ws_l + b) : 0.f;
                os[s] = ok ? __ldcg(ws_o + b * MD + d) : 0.f;
              }
              float mm = -INFINITY;
#pragma unroll
              for (int s = 0; s < MAXS; ++s) mm = fmaxf(mm, ms[s]);
              float ll = 0.f, oo = 0.f;
#pragma unroll
              for (int s = 0; s < MAXS; ++s) {
                const float w = (ms[s] == -INFINITY) ? 0.f : exp2f(ms[s] - mm);
                ll += ls[s] * w;
                oo += os[s] * w;
              }
              p.act[(hk * G + gq) * MD + d] = __float2bfloat16(oo / ll);  // act doubles as the attn vector
            }
          }
        }
        sync_target += grid;
        grid_sync(p.barrier, sync_target);
      }
      stamp(1);

      // ================= stage the activation vector of this GEMV phase =================
      {
        const __nv_bfloat16* xsrc = (ph.kind == 3 || ph.kind == 1) ? p.act : p.x;
        const __nv_bfloat16* nw = nullptr;
        if (ph.kind == 0) nw = p.layers[layer].ln1_w;
        else if (ph.kind == 2) nw = p.layers[layer].ln2_w;
        else if (ph.kind == 4) nw = p.final_norm_w;
        const uint4* xg = reinterpret_cast<const uint4*>(xsrc);
        if (nw != nullptr) {
          float s = 0.f;
          for (int i = threadIdx.x; i < nvec; i += MT) {
            const uint4 v = ldcg_v4(xg + i);
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
          __syncthreads();
          if (lane == 0) red[warp] = s;
          __syncthreads();
          float t = lane < MW ? red[lane] : 0.f;
          t = warp_sum(t);
          const float rstd = rsqrtf(t / ph.K + p.eps);
          const uint4* wv = reinterpret_cast<const uint4*>(nw);
          for (int i = threadIdx.x; i < nvec; i += MT) {
            const uint4 v = xs[i], gg = ldg_v4(wv + i);
            uint4 o;
            o.x = pack_bf16(bf16_round(bf_lo(v.x) * rstd) * bf_lo(gg.x), bf16_round(bf_hi(v.x) * rstd) * bf_hi(gg.x));
            o.y = pack_bf16(bf16_round(bf_lo(v.y) * rstd) * bf_lo(gg.y), bf16_round(bf_hi(v.y) * rstd) * bf_hi(gg.y));
            o.z = pack_bf16(bf16_round(bf_lo(v.z) * rstd) * bf_lo(gg.z), bf16_round(bf_hi(v.z) * rstd) * bf_hi(gg.z));
            o.w = pack_bf16(bf16_round(bf_lo(v.w) * rstd) * bf_lo(gg.w), bf16_round(bf_hi(v.w) * rstd) * bf_hi(gg.w));
            xs[i] = o;
          }
        } else {
          for (int i = threadIdx.x; i < nvec; i += MT) xs[i] = ldcg_v4(xg + i);
        }
      }
      if (threadIdx.x == 0) best_s = 0ull;
      __syncthreads();
      stamp(2);

      // ================= consume this warp's chunks of the phase =================
      {
        const int n_my = my_items(ph);
        const int ce = ph.K / ph.ks;
        const int chunk_vecs = ce >> 3;
        for (int j = 0; j < n_my; ++j) {
          const int s = consumed % MSTAGES;
          const int item = warp + j * MW;
          const int part = item % ph.ks;
          mbar_wait(&my_bars[s], (consumed / MSTAGES) & 1);
          const uint4* wv = reinterpret_cast<const uint4*>(my_ring + s * SLOT);
          const uint4* xv = xs + part * chunk_vecs;
          float s0 = 0.f, s1 = 0.f;
          int v = lane;
          for (; v + 32 < chunk_vecs; v += 64) {
            const uint4 a = wv[v], b = wv[v + 32];
            s0 = dot8(a, xv[v], s0);
            s1 = dot8(b, xv[v + 32], s1);
          }
          if (v < chunk_vecs) s0 = dot8(wv[v], xv[v], s0);
          const float tot = warp_sum(s0 + s1);
          __syncwarp();
          ++consumed;
          if (lane == 0) {
            acc[item] = tot;
            producer_advance();
          }
        }
      }
      __syncthreads();
      stamp(3);
      if (ph.ks > 1) {
        for (int base = 0; base < nrows; base += MT) {
          const int i = base + threadIdx.x;
          float tot = 0.f;
          if (i < nrows)
            for (int q = 0; q < ph.ks; ++q) tot += acc[i * ph.ks + q];
          __syncthreads();
          if (i < nrows) acc[i] = tot;
          __syncthreads();
        }
      }

      // ================= epilogue =================
      if (ph.kind == 2) {
        for (int j = threadIdx.x; j < (nrows >> 1); j += MT) {
          const float gt = bf16_round(acc[2 * j]), up = bf16_round(acc[2 * j + 1]);
          p.act[(row0 >> 1) + j] = __float2bfloat16(bf16_round(silu_f(gt)) * up);
        }
      } else if (ph.kind == 4) {
        unsigned long long best = 0ull;
        for (int r = threadIdx.x; r < nrows; r += MT) {
          const float v = bf16_round(acc[r]);
          const unsigned long long key =
              (static_cast<unsigned long long>(float_order(v)) << 32) |
              static_cast<unsigned long long>(0xffffffffu - static_cast<uint32_t>(row0 + r));
          best = key > best ? key : best;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
          best = other > best ? other : best;
        }
        if (lane == 0) atomicMax(&best_s, best);
        __syncthreads();
        if (threadIdx.x == 0 && nrows > 0) atomicMax(p.key, best_s);
      } else {
        const __nv_bfloat16* bias = (ph.kind == 0) ? p.layers[layer].qkv_b : nullptr;
        __nv_bfloat16* out = (ph.kind == 0) ? p.qkv : p.x;
        const bool residual = (ph.kind == 1 || ph.kind == 3);
        for (int r = threadIdx.x; r < nrows; r += MT) {
          float v = acc[r];
          if (bias) v += __bfloat162float(bias[row0 + r]);
          v = bf16_round(v);
          if (residual) v = bf16_round(v + ldcg_bf16(p.x + row0 + r));
          out[row0 + r] = __float2bfloat16(v);
        }
      }
      stamp(4);
      sync_target += grid;
      grid_sync(p.barrier, sync_target);
      stamp(5);
      ++dbg_i;
    }

    // ================= finalize the token =================
    if (cta == 0) {
      __shared__ int tok_s;
      if (threadIdx.x == 0) {
        const unsigned long long k = *reinterpret_cast<volatile unsigned long long*>(p.key);
        const int t = static_cast<int>(0xffffffffu - static_cast<uint32_t>(k & 0xffffffffull));
        *p.token = t;
        const int st = *reinterpret_cast<volatile int*>(p.step);
        p.hist[st] = t;
        *p.step = st + 1;
        *p.position = *reinterpret_cast<volatile int*>(p.position) + 1;
        *p.key = 0ull;
        tok_s = t;
      }
      __syncthreads();
      const uint4* src = reinterpret_cast<const uint4*>(p.embed + static_cast<size_t>(tok_s) * p.hidden);
      uint4* dst = reinterpret_cast<uint4*>(p.x);
      for (int i = threadIdx.x; i < (p.hidden >> 3); i += MT) dst[i] = src[i];
    }
    sync_target += grid;
    grid_sync(p.barrier, sync_target);
  }
  if (cta == 0 && threadIdx.x == 0) *p.epoch = sync_target;
}

}  // namespace

int decode_mega(const MegaParams& pin, cudaStream_t stream) {
  MegaParams p = pin;
  VB_CHECK(p.n_tokens >= 1 && p.num_layers >= 1, "decode_mega: bad n_tokens / num_layers");
  VB_CHECK(p.Hq % p.Hkv == 0, "decode_mega: Hq %% Hkv != 0");
  VB_CHECK(p.hidden % 8 == 0 && p.inter % 8 == 0, "decode_mega: hidden / inter must be multiples of 8");
  auto pick_ks = [](int K) {
    for (int ks = 1; ks <= 64; ++ks)
      if (K % ks == 0 && (K / ks) % 8 == 0 && (K / ks) * 2 <= SLOT) return ks;
    return -1;
  };
  p.ks_hidden = pick_ks(p.hidden);
  p.ks_inter = pick_ks(p.inter);
  p.ks_attn = pick_ks(p.Hq * MD);
  VB_CHECK(p.ks_hidden > 0 && p.ks_inter > 0 && p.ks_attn > 0, "decode_mega: K not chunkable");
  const int G = p.Hq / p.Hkv;
  const int sms = num_sms();
  const int grid = sms;
  VB_CHECK(p.Hkv * p.splits <= grid && p.splits <= 16, "decode_mega: Hkv*splits exceeds the grid / splits > 16");
  VB_CHECK(p.inter >= p.Hq * MD, "decode_mega: act buffer (inter) must hold the attention vector");
  const int kmax = p.hidden > p.inter ? p.hidden : p.inter;
  const int attn_bytes = (G * MD * 4) + 2 * MD * 2 + 2 * MW * G * 4 + MW * G * MD * 4;
  int xs_bytes = kmax * 2;
  if (p.Hq * MD * 2 > xs_bytes) xs_bytes = p.Hq * MD * 2;
  if (attn_bytes > xs_bytes) xs_bytes = attn_bytes;
  xs_bytes = (xs_bytes + 127) / 128 * 128;
  p.xs_bytes = xs_bytes;
  // acc slots: rows_per_block * ks of the largest phase
  auto rows = [&](int N, int ks, bool even) {
    int rpb = (N + grid - 1) / grid;
    if (even && (rpb & 1)) ++rpb;
    return rpb * ks;
  };
  int need_acc = rows(p.vocab, p.ks_hidden, false);
  need_acc = max(need_acc, rows(2 * p.inter, p.ks_hidden, true));
  need_acc = max(need_acc, rows(p.hidden, p.ks_inter, false));
  need_acc = max(need_acc, rows(p.hidden, p.ks_attn, false));
  need_acc = max(need_acc, rows((p.Hq + 2 * p.Hkv) * MD, p.ks_hidden, false));
  VB_CHECK(need_acc <= ACC_FLOATS, "decode_mega: %d accumulator slots needed (max %d)", need_acc, ACC_FLOATS);
  VB_CHECK(p.num_layers <= 64, "decode_mega: at most 64 layers");
  const size_t smem = static_cast<size_t>(xs_bytes) + ACC_FLOATS * 4 + MW * MSTAGES * SLOT + MW * MSTAGES * 8 +
                      static_cast<size_t>(p.num_layers) * sizeof(MegaLayer) + 128;
  VB_CHECK(smem <= 225 * 1024, "decode_mega: needs %zu bytes of shared memory", smem);
#define VB_MEGA_CASE(GG)                                                                         \
  case GG: {                                                                                     \
    auto kern = decode_mega_kernel<GG>;                                                          \
    static PerDeviceOnce attr_once;                                                              \
    if (attr_once.first()) {                                                                     \
      VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 225 * 1024)); \
    }                                                                                            \
    int occ = 0;                                                                                 \
    VB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, MT, smem));                \
    VB_CHECK(occ >= 1, "decode_mega: kernel does not fit on an SM");                             \
    kern<<<grid, MT, smem, stream>>>(p);                                                         \
    break;                                                                                       \
  }
  switch (G) {
    VB_MEGA_CASE(1)
    VB_MEGA_CASE(2)
    VB_MEGA_CASE(4)
    VB_MEGA_CASE(7)
    VB_MEGA_CASE(8)
    default:
      set_last_error("decode_mega: unsupported GQA group size %d", G);
      return 1;
  }
#undef VB_MEGA_CASE
  VB_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace vb
