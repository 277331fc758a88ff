// extern "C" surface declared in include/vila_b200.h: thin argument marshalling onto vb::*.
#include "../../include/vila_b200.h"

#include <cstdio>
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"

using bf = __nv_bfloat16;
static inline const bf* cb(const void* p) { return static_cast<const bf*>(p); }
static inline bf* mb(void* p) { return static_cast<bf*>(p); }
static inline cudaStream_t st(void* s) { return static_cast<cudaStream_t>(s); }

static int require_sm90() {
  static int ok = -1;
  if (ok < 0) {
    int dev = 0, major = 0, minor = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) {
      vb::set_last_error("vila_b200: no CUDA device available (this library has no CPU fallback)");
      cudaGetLastError();
      return 1;
    }
    ok = (major == 9 && minor == 0) ? 1 : 0;
    if (!ok) {
      vb::set_last_error("vila_b200: built for sm_90a only, device is sm_%d%d", major, minor);
    }
  }
  if (ok != 1) {
    if (ok == 0) vb::set_last_error("vila_b200: built for sm_90a only (no fallback path)");
    return 1;
  }
  return 0;
}
#define VB_REQUIRE_DEVICE() \
  do {                      \
    if (require_sm90()) return 3; \
  } while (0)

extern "C" {

const char* vila_last_error(void) { return vb::last_error(); }
int vila_abi_version(void) { return 3; }

int vila_set_workspace(void* ptr, uint64_t bytes) { return vb::set_workspace(ptr, (size_t)bytes); }

int vila_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  VB_CUDA(cudaGetDevice(&dev));
  VB_CUDA(cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, dev));
  VB_CUDA(cudaDeviceGetAttribute(cc_major, cudaDevAttrComputeCapabilityMajor, dev));
  VB_CUDA(cudaDeviceGetAttribute(cc_minor, cudaDevAttrComputeCapabilityMinor, dev));
  return 0;
}

static vb::GemmEpilogue make_epi(const void* bias, const void* residual, int64_t ld_res,
                                 int res_row_mod, int act, int flags) {
  vb::GemmEpilogue e;
  e.bias = cb(bias);
  e.residual = cb(residual);
  e.ld_res = static_cast<int>(ld_res);
  e.res_row_mod = res_row_mod;
  e.act = act;
  e.swiglu = (flags & VILA_FLAG_SWIGLU) ? 1 : 0;
  e.static_w = (flags & VILA_FLAG_STATIC_W) ? 1 : 0;
  return e;
}

int vila_linear(const void* x, int64_t ldx, const void* w, int64_t ldw, const void* bias,
                const void* residual, int64_t ld_res, int res_row_mod, void* out, int64_t ldo,
                int M, int N, int K, int act, int swiglu, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::gemm_bf16(cb(x), (int)ldx, cb(w), (int)ldw, mb(out), (int)ldo, M, N, K,
                       make_epi(bias, residual, ld_res, res_row_mod, act, swiglu), st(stream));
}

int vila_linear_cfg(int block_n, const void* x, int64_t ldx, const void* w, int64_t ldw,
                    const void* bias, const void* residual, int64_t ld_res, int res_row_mod,
                    void* out, int64_t ldo, int M, int N, int K, int act, int swiglu, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::gemm_bf16_cfg(block_n, cb(x), (int)ldx, cb(w), (int)ldw, mb(out), (int)ldo, M, N, K,
                           make_epi(bias, residual, ld_res, res_row_mod, act, swiglu), st(stream));
}

int vila_layernorm(const void* x, const void* weight, const void* bias, void* out, int rows,
                   int cols, float eps, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::layernorm_bf16(cb(x), cb(weight), cb(bias), mb(out), rows, cols, eps, st(stream));
}

int vila_rmsnorm(void* x_inout, const void* residual_add, const void* weight, void* out, int rows,
                 int cols, float eps, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::rmsnorm_bf16(mb(x_inout), cb(residual_add), cb(weight), mb(out), rows, cols, eps,
                          st(stream));
}

int vila_fmha(const vila_fmha_params* p, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::fmha_prefill(*p, st(stream));
}

int vila_fmha_cfg(int variant, const vila_fmha_params* p, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::fmha_prefill_cfg(variant, *p, st(stream));
}

int vila_patch_im2col(const void* pixels, void* out, int B, int C, int H, int W, int patch,
                      int k_pad, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::im2col_patch14(cb(pixels), mb(out), B, C, H, W, patch, k_pad, st(stream));
}

int vila_resize_bicubic_tiles(const uint8_t* src, int H, int W, int out_w, int out_h,
                              const int32_t* coef_x, const int32_t* bounds_x, int ksize_x,
                              const int32_t* coef_y, const int32_t* bounds_y, int ksize_y, uint8_t* tmp,
                              void* out_tiles, int tile, int tile_index0, float mean, float stdv,
                              void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::resize_bicubic_tiles(src, H, W, out_w, out_h, coef_x, bounds_x, ksize_x, coef_y, bounds_y,
                                  ksize_y, tmp, mb(out_tiles), tile, tile_index0, mean, stdv, st(stream));
}

int vila_space_to_depth(const void* x, void* out, int B, int h, int w, int C, int r, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::space_to_depth(cb(x), mb(out), B, h, w, C, r, st(stream));
}

int vila_s2_merge(const void* tiles, void* out, int side, int C, int n_scales, const int* splits_h,
                  const int* splits_w, int out_bh, int out_bw, int share_tile, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::s2_merge(cb(tiles), mb(out), side, C, n_scales, splits_h, splits_w, out_bh, out_bw,
                      share_tile, st(stream));
}

int vila_chessboard_merge(const void* tiles, void* out, int bh, int bw, int s, int C, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::chessboard_merge(cb(tiles), mb(out), bh, bw, s, C, st(stream));
}

int vila_tsp_pool(const void* x, void* out, int T, int h, int w, int C, int pt, int ph, int pw,
                  void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::tsp_pool(cb(x), mb(out), T, h, w, C, pt, ph, pw, st(stream));
}

int vila_embed_splice(const void* table, const void* media, const int32_t* src, void* out, int rows,
                      int cols, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::embed_splice(cb(table), cb(media), src, mb(out), rows, cols, st(stream));
}

int vila_rope_kv_append(void* qkv, const int32_t* positions, int S, int Hq, int Hkv, int D,
                        const float* inv_freq, void* k_pool, void* v_pool,
                        const int32_t* page_table, int cache_pos0, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::rope_kv_append(mb(qkv), positions, S, Hq, Hkv, D, inv_freq, mb(k_pool), mb(v_pool),
                            page_table, cache_pos0, st(stream));
}

int vila_rope_kv_append_table(void* qkv, const void* rope_table, int S, int Hq, int Hkv, int D,
                              void* k_pool, void* v_pool, const int32_t* page_table, int cache_pos0,
                              void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::rope_kv_append_table(mb(qkv), cb(rope_table), S, Hq, Hkv, D, mb(k_pool), mb(v_pool),
                                  page_table, cache_pos0, st(stream));
}

int vila_linear_qkv_rope(const void* x, int64_t ldx, const void* w, int64_t ldw, const void* bias,
                         void* qkv_out, int64_t ldo, int M, int K, int Hq, int Hkv, int D,
                         const void* rope_table, void* k_pool, void* v_pool,
                         const int32_t* page_table, int cache_pos0, int flags, void* stream) {
  VB_REQUIRE_DEVICE();
  if (D != 128 || M > 384 || rope_table == nullptr) {
    vb::set_last_error("vila_linear_qkv_rope: needs head_dim 128 and M <= 384 (D=%d, M=%d)", D, M);
    return 3;
  }
  vb::GemmEpilogue e;
  e.bias = cb(bias);
  e.static_w = (flags & VILA_FLAG_STATIC_W) ? 1 : 0;
  e.rope_table = cb(rope_table);
  e.k_pool = mb(k_pool);
  e.v_pool = mb(v_pool);
  e.page_table = page_table;
  e.cache_pos0 = cache_pos0;
  e.rope_hq = Hq;
  e.rope_hkv = Hkv;
  const int rc = vb::gemm_qkv_rope_bf16(cb(x), (int)ldx, cb(w), (int)ldw, mb(qkv_out), (int)ldo, M,
                                        (Hq + 2 * Hkv) * D, K, e, st(stream));
  if (rc < 0) {
    vb::set_last_error("vila_linear_qkv_rope: shape not covered (M=%d)", M);
    return 3;
  }
  return rc;
}

int vila_rope_table(const int32_t* positions, int S, int D, const float* inv_freq, void* table,
                    void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::rope_table(positions, S, D, inv_freq, mb(table), st(stream));
}

static vb::GemvParams to_gemv(const vila_gemv_params* p) {
  vb::GemvParams g;
  g.x = cb(p->x);
  g.w = cb(p->w);
  g.bias = cb(p->bias);
  g.norm_w = cb(p->norm_w);
  g.norm_eps = p->norm_eps;
  g.residual = cb(p->residual);
  g.y = mb(p->y);
  g.N = p->N;
  g.K = p->K;
  g.flags = p->flags;
  g.argmax_key = p->argmax_key;
  g.w_scale = nullptr;
  return g;
}

int vila_gemv(const vila_gemv_params* p, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::gemv_bf16(to_gemv(p), st(stream));
}

int vila_gemv_fp8(const vila_gemv_params* p, const float* w_scale, void* stream) {
  VB_REQUIRE_DEVICE();
  vb::GemvParams g = to_gemv(p);
  g.w_scale = w_scale;
  return vb::gemv_tma_fp8(g, st(stream));
}

int vila_gemv_w4a16(const vila_gemv_params* p, const void* w_scale, const uint8_t* w_zero, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::gemv_tma_w4a16(to_gemv(p), cb(w_scale), w_zero, st(stream));
}

// the Linear layers of a batched decode step (modeling_qwen2.py:81-95,164-176,223-226) on e4m3 weights
int vila_gemv_batch_fp8(const vila_gemv_batch_params* p, const float* w_scale, void* stream) {
  VB_REQUIRE_DEVICE();
  VB_CHECK(p != nullptr, "vila_gemv_batch_fp8: params are required");
  return vb::gemv_batch_fp8(*p, w_scale, st(stream));
}

// the TinyChat W4A16 GEMM of the reference's 4-bit deployment (README "Quantization and Deployment")
int vila_gemv_batch_w4a16(const vila_gemv_batch_params* p, const void* w_scale, const uint8_t* w_zero,
                          void* stream) {
  VB_REQUIRE_DEVICE();
  VB_CHECK(p != nullptr, "vila_gemv_batch_w4a16: params are required");
  return vb::gemv_batch_w4a16(*p, cb(w_scale), w_zero, st(stream));
}

int vila_gemv_batch_partition(int N, int K, int fp8, int32_t* out) {
  VB_REQUIRE_DEVICE();
  return vb::gemv_batch_partition(N, K, fp8, out);
}

int vila_argmax_finalize(unsigned long long* key, int32_t* token_out, int32_t* token_hist,
                         int32_t* step_counter, int32_t* position, const void* embed_table,
                         void* x_next, int hidden, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::argmax_finalize(key, token_out, token_hist, step_counter, position, cb(embed_table),
                             mb(x_next), hidden, st(stream));
}

int vila_decode_attention(const vila_decode_attn_params* p, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::decode_attention(*p, st(stream));
}

int vila_decode_attention_batch(const vila_decode_attn_params* p, int batch, int qkv_stride,
                                int out_stride, int pt_stride, int max_pages, void* stream) {
  VB_REQUIRE_DEVICE();
  vila_decode_attn_params d = *p;  // the batched kernel has no split: ws, counters and num_splits are ignored
  d.ws = nullptr;
  d.counters = nullptr;
  d.num_splits = 0;
  return vb::decode_attention_batch(d, batch, qkv_stride, out_stride, pt_stride, max_pages, st(stream));
}

int vila_decode_attention_split(const vila_decode_attn_split_params* p, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::decode_attention_split(*p, st(stream));
}

int vila_decode_attention_split_batch(const vila_decode_attn_split_params* p, int batch, int qkv_stride,
                                      int out_stride, int pt_stride, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::decode_attention_split_batch(*p, batch, qkv_stride, out_stride, pt_stride, st(stream));
}

// DynamicCache.update + flash-attn decode (modeling_qwen2.py:99-160,262-310) over an e4m3 KV pool
int vila_kv_quantize_fp8(const void* src, int64_t src_tokens, void* dst, float* dst_scale, int64_t dst_pages,
                         const int32_t* page_table, int pt_len, int L, int Hkv, int D, int S, void* stream) {
  VB_REQUIRE_DEVICE();
  return vb::kv_quantize_fp8(cb(src), src_tokens, static_cast<uint8_t*>(dst), dst_scale, dst_pages, page_table,
                             pt_len, L, Hkv, D, S, st(stream));
}

int vila_decode_attention_fp8_batch(const vila_decode_attn_fp8_params* p, void* stream) {
  VB_REQUIRE_DEVICE();
  VB_CHECK(p != nullptr, "vila_decode_attention_fp8_batch: params are required");
  return vb::decode_attention_fp8_batch(*p, st(stream));
}

// HF Temperature / TopK / TopP LogitsWarper + torch.multinomial (GenerationMixin._sample)
int vila_sample_batch(const vila_sample_params* p, void* stream) {
  VB_REQUIRE_DEVICE();
  VB_CHECK(p != nullptr, "vila_sample_batch: params are required");
  return vb::sample_batch(*p, st(stream));
}

// GenerationMixin._sample's warpers + torch.multinomial for the single-stream graph decoder
int vila_sample_finalize(const vila_sample_finalize_params* p, void* stream) {
  VB_CHECK(p != nullptr, "vila_sample_finalize: params are required");
  if (int rc = vb::sample_finalize_check(*p)) return rc;
  VB_REQUIRE_DEVICE();
  return vb::sample_finalize(*p, st(stream));
}

// HF generate(output_scores=True) + torch.log_softmax / OpenAI logprobs for the batched engine
int vila_token_logprobs(const vila_logprobs_params* p, void* stream) {
  VB_CHECK(p != nullptr, "vila_token_logprobs: params are required");
  if (int rc = vb::token_logprobs_check(*p)) return rc;
  VB_REQUIRE_DEVICE();
  return vb::token_logprobs(*p, st(stream));
}

// the same for the single-stream graph decoder's one row
int vila_token_logprobs_row(const vila_logprobs_row_params* p, void* stream) {
  VB_CHECK(p != nullptr, "vila_token_logprobs_row: params are required");
  if (int rc = vb::token_logprobs_row_check(*p)) return rc;
  VB_REQUIRE_DEVICE();
  return vb::token_logprobs_row(*p, st(stream));
}

// OpenAI presence_penalty / frequency_penalty for the batched engine (the reference serves neither)
int vila_apply_penalties(const vila_penalty_params* p, void* stream) {
  VB_CHECK(p != nullptr, "vila_apply_penalties: params are required");
  if (int rc = vb::apply_penalties_check(*p)) return rc;
  VB_REQUIRE_DEVICE();
  return vb::apply_penalties(*p, st(stream));
}

// the same for the single-stream graph decoder's one row
int vila_apply_penalties_row(const vila_penalty_row_params* p, void* stream) {
  VB_CHECK(p != nullptr, "vila_apply_penalties_row: params are required");
  if (int rc = vb::apply_penalties_row_check(*p)) return rc;
  VB_REQUIRE_DEVICE();
  return vb::apply_penalties_row(*p, st(stream));
}

// xgrammar's HF LogitsProcessor (llava_arch.py:802-821) for the single-stream graph decoder's one row
int vila_apply_token_bitmask_row(const void* logits, const int32_t* bitmask, void* out, int32_t V, void* stream) {
  if (int rc = vb::apply_token_bitmask_row_check(logits, bitmask, out, V)) return rc;
  VB_REQUIRE_DEVICE();
  return vb::apply_token_bitmask_row(logits, bitmask, out, V, st(stream));
}

// the reference prefills every request in full (serving/server.py:65-73, llava_arch.py:823-833): no seam
int vila_prefix_block_hash(const void* x, int64_t ld, int64_t rows, int64_t cols, uint64_t key0, uint64_t key1,
                           uint64_t* out, void* stream) {
  if (int rc = vb::prefix_block_hash_check(x, ld, rows, cols, out)) return rc;
  if (rows < 128) return 0;
  VB_REQUIRE_DEVICE();
  return vb::prefix_block_hash(x, ld, rows, cols, key0, key1, out, st(stream));
}

// test hooks: no reference seam (the reference launches without programmatic dependent launch)
int vila_test_pdl_late(const vila_pdl_copy* snap, int n_snap, const vila_pdl_copy* late, int n_late, int64_t delay_ns,
                       void* stream) {
  if (int rc = vb::pdl_late_check(snap, n_snap, late, n_late, delay_ns)) return rc;
  VB_REQUIRE_DEVICE();
  return vb::pdl_late(snap, n_snap, late, n_late, delay_ns, st(stream));
}

int vila_test_pdl_probe(const int32_t* flag, int32_t* seen, int* pdl_enabled, void* stream) {
  if (int rc = vb::pdl_probe_check(flag, seen)) return rc;
  if (pdl_enabled != nullptr) *pdl_enabled = vb::pdl_enabled() ? 1 : 0;
  if (flag == nullptr) return 0;
  VB_REQUIRE_DEVICE();
  return vb::pdl_probe(flag, seen, st(stream));
}

}  // extern "C"
