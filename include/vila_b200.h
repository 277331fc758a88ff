/*
 * vila_b200 — C-ABI of the H100-native (sm_90a) VILA multimodal forward hot path.
 *
 * The reference (NVlabs/VILA) has no FFI on this path: every GPU op is a library call made from
 * Python (flash_attn, cuBLAS through nn.Linear, cuDNN through nn.Conv2d, ATen elementwise).  This
 * header is the boundary a maintainer would bind instead of those calls; each entry point names the
 * reference call site (paths relative to the VILA repo root) it replaces.  The only native-extension
 * precedent in the tree (llava/model/coat/optimizer/kernels/bindings.cpp:6-10) takes tensors,
 * mutates in place, returns void and runs on the current stream; we keep "caller owns all memory,
 * in-place/out-param, stream-ordered", but with plain pointers so any host language can bind it.
 *
 * Conventions
 *   - all tensor pointers are DEVICE pointers to bf16 (uint16 storage) unless stated otherwise,
 *     row-major, 16-byte aligned; leading dimensions are in ELEMENTS;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - every function returns 0 on success; non-zero on error, message via vila_last_error()
 *     (thread-local). Nothing falls back to the CPU: without an sm_90a device calls fail.
 *   - no hidden state beyond (a) the per-device stream-K scratch registered with vila_set_workspace and
 *     (b) per-device "function attributes set" flags: KV pool, page tables, workspaces and counters
 *     are caller-allocated.
 */
#ifndef VILA_B200_H_
#define VILA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VILA_ACT_NONE 0
#define VILA_ACT_GELU_TANH 1 /* SigLIP "gelu_pytorch_tanh"  (modeling_siglip.py:707-715) */
#define VILA_ACT_GELU_ERF 2  /* nn.GELU() in mm_projector   (base_projector.py:145-162)  */
#define VILA_ACT_SILU 3

/* `flags` of vila_linear / vila_gemv:
 *   VILA_FLAG_SWIGLU    weight rows are interleaved (gate_0, up_0, gate_1, ...); out is [M, N/2] =
 *                       silu(gate) * up
 *   VILA_FLAG_STATIC_W  the weight matrix is a parameter that no earlier kernel in this stream is
 *                       still writing: the kernel may fetch it BEFORE the programmatic-dependent-launch
 *                       wait (all vila_* kernels are launched with PDL so that prologues and weight
 *                       prefetch overlap the predecessor's tail). Leave it clear for weights produced
 *                       on the fly. */
#define VILA_FLAG_SWIGLU 1
#define VILA_FLAG_STATIC_W 2

const char* vila_last_error(void);
int vila_abi_version(void); /* 3 */
/* Register caller-owned, ZERO-INITIALISED device scratch (256-byte aligned) used by vila_linear's
 * stream-K schedule for fp32 partial sums (64 KiB of counters + M*N*4 bytes per call that uses it;
 * calls that do not fit simply use the data-parallel schedule).  The kernels leave it zeroed again.
 * The registration is per DEVICE (the current device at the time of the call); one workspace serves
 * one stream at a time.  ptr == NULL unregisters. */
int vila_set_workspace(void* ptr, uint64_t bytes);
/* fills SM count and compute capability of the current device */
int vila_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---------------------------------------------------------------------------------------------
 * vila_linear — out[M,N] = epilogue(x[M,K] · w[N,K]^T)        (wgmma / TMA GEMM)
 *   epilogue: (+bias[N]) -> act -> (+residual[row % res_row_mod or row, :])   or SwiGLU:
 *   flags & VILA_FLAG_SWIGLU: w rows are interleaved (gate_0, up_0, gate_1, up_1, ...) and out is
 *   [M, N/2] = silu(gate) * up.
 * Replaces nn.Linear (+ the ATen GELU / SiLU*mul / residual add that follows it):
 *   SigLIP q/k/v/out_proj, fc1/fc2 : llava/model/multimodal_encoder/siglip/modeling_siglip.py:384-387,707-715,752,757
 *   patch-embed Conv2d (as im2col GEMM, residual = position embedding with res_row_mod = #patches): :269-275,322-328
 *   mm_projector Linear layers     : llava/model/multimodal_projector/base_projector.py:145-162
 *   Qwen2 q/k/v/o, gate/up/down, lm_head: transformers Qwen2 (in-tree copy
 *     llava/eval/vision_niah_vila/zigzag_ring_attn/modeling_qwen2.py:164-176,223-226,633-706)
 * ------------------------------------------------------------------------------------------- */
int vila_linear(const void* x, int64_t ldx, const void* w, int64_t ldw, const void* bias,
                const void* residual, int64_t ld_res, int res_row_mod, void* out, int64_t ldo,
                int M, int N, int K, int act, int flags, void* stream);
/* test hook: same, forcing the kernel configuration instead of the size heuristic:
 *   64 / 128 / 256   single-CTA tiles 128 x block_n (+1000: deterministic stream-K, +2000: stream-K off)
 *   4128 / 4256      CTA-pair tiles 256 x {128,256} (2-CTA cluster, W tile multicast to both CTAs)
 *   5128             split-K CTA pairs on 128 x 128 tiles, one tile per pair (K > 64)
 *   3000 / 3001      small-M path (M <= 512): 128 x 128 tiles, single CTAs / CTA pairs (W multicast) */
int vila_linear_cfg(int block_n, const void* x, int64_t ldx, const void* w, int64_t ldw,
                    const void* bias, const void* residual, int64_t ld_res, int res_row_mod,
                    void* out, int64_t ldo, int M, int N, int K, int act, int flags, void* stream);

/* nn.LayerNorm over the last dim (modeling_siglip.py:723,725,746,755; base_projector.py:147) */
int vila_layernorm(const void* x, const void* weight, const void* bias, void* out, int rows,
                   int cols, float eps, void* stream);
/* Qwen2RMSNorm (modeling_qwen2.py:81-95). If residual_add != NULL: x += residual_add first (in place). */
int vila_rmsnorm(void* x_inout, const void* residual_add, const void* weight, void* out, int rows,
                 int cols, float eps, void* stream);

/* ---------------------------------------------------------------------------------------------
 * vila_fmha — flash attention forward, wgmma QK^T / PV with register accumulators.
 *   q/o element (token t, head h, dim d) at  base + t*tok_stride + h*head_stride + d
 *   k/v: if kv_page_stride != 0 the KV cache is paged (128 tokens per page):
 *          element (page p, row r, head h, d) at base + p*kv_page_stride + r*kv_tok_stride + h*kv_head_stride + d
 *          and page_table[b*page_table_stride + j] gives the page of block j (NULL: identity);
 *        else k/v are [B*Sk, Hkv, D] views like q.
 * Replaces flash_attn_func(q,k,v,causal=False) in SiglipFlashAttention2 (modeling_siglip.py:583-585)
 * and HF _flash_attention_forward for Qwen2/Llama (patched at llava/train/sequence_parallel/
 * monkey_patch.py:133-239, llava/model/utils/packing.py:36), causal GQA.
 * ------------------------------------------------------------------------------------------- */
typedef struct vila_fmha_params {
  const void* q;
  int64_t q_tok_stride, q_head_stride;
  const void* k;
  const void* v;
  int64_t kv_page_stride, kv_tok_stride, kv_head_stride, kv_num_pages;
  const int32_t* page_table;
  int32_t page_table_stride;
  void* o;
  int64_t o_tok_stride, o_head_stride;
  int32_t B, Sq, Sk, Hq, Hkv, D, causal;
  float scale;
} vila_fmha_params;
int vila_fmha(const vila_fmha_params* p, void* stream);
/* test hook (like vila_linear_cfg): same, forcing the kernel flavour instead of the default:
 *   0 default; 1 / 2 the wgmma kernel (one 128-row query tile per CTA, two consumer warpgroups);
 *   3 / 4: as 1 with every 4th / every 2nd exponential as an FMA-pipe polynomial */
int vila_fmha_cfg(int variant, const vila_fmha_params* p, void* stream);

/* im2col for Conv2d(3,1152,k=14,s=14) (modeling_siglip.py:269-275): pixels [B,C,H,W] ->
 * out [B*(H/P)*(W/P), k_pad], column = (c, ky, kx); columns >= C*P*P are zero. */
int vila_patch_im2col(const void* pixels, void* out, int B, int C, int H, int W, int patch,
                      int k_pad, void* stream);
/* Image preprocessing on the device (SURVEY §8 f2).  Replaces, per resize grid of
 * mm_utils.process_image (llava/mm_utils.py:442-522; dynamic_preprocess :299-338, dynamic_s2_preprocess
 * :341-405), PIL `image.resize((out_w, out_h))` (bicubic; Pillow Resample.c 8bpc fixed point) + the crop
 * into tile x tile blocks + SiglipImageProcessor.preprocess (rescale 1/255, normalise (x-mean)/std):
 *   src      uint8 [H, W, 3] (device)      tmp  uint8 scratch [H, out_w, 3]
 *   coef_*   int32 [out, ksize] 22-bit filter taps, bounds_* int32 [out, 2] = (first input index, count)
 *            (host: vila_b200.model.media.bicubic_coeffs == Pillow precompute_coeffs/normalize_coeffs_8bpc)
 *   out      bf16 [n_tiles, 3, tile, tile]; pixel (Y, X) of the resized image lands in tile
 *            tile_index0 + (Y / tile) * (out_w / tile) + X / tile.  Bit-identical to the PIL path. */
int vila_resize_bicubic_tiles(const uint8_t* src, int H, int W, int out_w, int out_h,
                              const int32_t* coef_x, const int32_t* bounds_x, int ksize_x,
                              const int32_t* coef_y, const int32_t* bounds_y, int ksize_y, uint8_t* tmp,
                              void* out_tiles, int tile, int tile_index0, float mean, float stdv,
                              void* stream);
/* DownSampleBlock.flat_square / flat_square_2x2 / flat_square_3x3 (base_projector.py:58-123):
 * x [B, h*w, C] -> out [B, ceil(h/r)*ceil(w/r), r*r*C], zero padded. */
int vila_space_to_depth(const void* x, void* out, int B, int h, int w, int C, int r, void* stream);
/* merge_features_for_dynamic_s2 + split_chessboard for one image (llava_arch.py:282-364). */
int vila_s2_merge(const void* tiles, void* out, int side, int C, int n_scales,
                  const int* splits_h, const int* splits_w, int out_bh, int out_bw, int share_tile,
                  void* stream);
/* merge_chessboard + "(h w) c" flatten of projected tiles (llava_arch.py:255-280,384-390). */
int vila_chessboard_merge(const void* tiles, void* out, int bh, int bw, int s, int C, void* stream);
/* TSPVideoEncoder pooling (llava/model/encoders/video/tsp.py:11-12,28-51). */
int vila_tsp_pool(const void* x, void* out, int T, int h, int w, int C, int pt, int ph, int pw,
                  void* stream);
/* text/media embedding splice of LlavaMetaForCausalLM._embed (llava_arch.py:429,457-479):
 * out[i] = src[i] >= 0 ? table[src[i]] : media[-(src[i]+1)].  src is int32 on the device. */
int vila_embed_splice(const void* table, const void* media, const int32_t* src, void* out, int rows,
                      int cols, void* stream);
/* HF apply_rotary_pos_emb (modeling_qwen2.py:99-160) in place on q,k of qkv [S,(Hq+2Hkv)*D] and
 * DynamicCache.update as a scatter into the paged pool (k_pool may be NULL: RoPE only).
 * inv_freq: fp32 [D/2] on the device. positions: int32 [S] on the device. */
int vila_rope_kv_append(void* qkv, const int32_t* positions, int S, int Hq, int Hkv, int D,
                        const float* inv_freq, void* k_pool, void* v_pool,
                        const int32_t* page_table, int cache_pos0, void* stream);
/* (cache_pos0 < 0: the cache slot of row s is positions[s] itself — decode, position on the device) */
/* vila_rope_kv_append with cos / sin taken from vila_rope_table(positions) (computed once per request
 * and shared by all layers and heads; 16-byte accesses): the long-prefill form, bit-identical. */
int vila_rope_kv_append_table(void* qkv, const void* rope_table, int S, int Hq, int Hkv, int D,
                              void* k_pool, void* v_pool, const int32_t* page_table, int cache_pos0,
                              void* stream);
/* q/k/v projection for a short prefill chunk (M <= 384 tokens, head_dim 128):
 * qkv = x @ w^T + bias; RoPE on the q and k heads; q heads -> qkv_out[:, :Hq*128]; k / v heads ->
 * the paged pools (k_pool NULL: they stay in qkv_out).  Runs the GEMM and then the table-driven
 * RoPE + KV-append kernel, bit-identical to vila_linear followed by vila_rope_kv_append
 * (rope_table: vila_rope_table of the chunk's positions).  Replaces Qwen2Attention's q_proj/k_proj/v_proj +
 * apply_rotary_pos_emb + past_key_value.update (modeling_qwen2.py:223-226,99-160,262-266 of the
 * in-tree copy).  Returns 3 (and sets vila_last_error) when the shape is not covered: the caller
 * then issues the two separate calls. */
int vila_linear_qkv_rope(const void* x, int64_t ldx, const void* w, int64_t ldw, const void* bias,
                         void* qkv_out, int64_t ldo, int M, int K, int Hq, int Hkv, int D,
                         const void* rope_table, void* k_pool, void* v_pool,
                         const int32_t* page_table, int cache_pos0, int flags, void* stream);
/* cos / sin table of Qwen2RotaryEmbedding.forward (modeling_qwen2.py:99-143) for one request,
 * computed once and shared by all layers: table [S, D] bf16 = cos(pos*inv_freq[0..D/2)) | sin(...). */
int vila_rope_table(const int32_t* positions, int S, int D, const float* inv_freq, void* table,
                    void* stream);

/* ---------------------------------------------------------------------------------------------
 * decode (one token): weight-streaming GEMV with fused RMSNorm prologue and bias / residual /
 * SwiGLU / greedy-argmax epilogues; split-KV paged GQA attention with fused RoPE + KV append.
 * ------------------------------------------------------------------------------------------- */
typedef struct vila_gemv_params {
  const void* x;
  const void* w;
  const void* bias;
  const void* norm_w;
  float norm_eps;
  const void* residual;
  void* y;
  int32_t N, K;
  int32_t flags; /* VILA_FLAG_SWIGLU: rows interleaved (gate, up), y is [N/2];
                    VILA_FLAG_STATIC_W: see below */
  unsigned long long* argmax_key; /* device u64, zero before the first launch */
} vila_gemv_params;
int vila_gemv(const vila_gemv_params* p, void* stream);

/* vila_gemv with FP8 weights: p->w is [N, K] e4m3 (1 byte per element, 16-byte aligned), w_scale is fp32
 * [N], one scale per output row; x, bias, residual, norm_w and y stay bf16 and the VILA_FLAG_* meanings
 * are unchanged.  acc_n = sum_k float(w[n,k]) * float(x[k]) in fp32, then v = acc_n * w_scale[n] enters
 * vila_gemv's epilogue (bias, residual, SwiGLU, argmax).  Needs K % 16 == 0; there is no register-staged
 * variant, so an unsupported shape is an error, never a launch.  Halves the weight bytes a decode token
 * streams.  Replaces the reference's quantized loading (load_8bit / load_4bit,
 * llava/model/builder.py:42-51) and the weight-only quantized deployment of its README ("Quantization
 * and Deployment"). */
int vila_gemv_fp8(const vila_gemv_params* p, const float* w_scale, void* stream);

/* vila_gemv with 4-bit weights (W4A16): groups of 128 consecutive k of a row share a bf16 scale s and a uint8
 * zero point z, and w = (q - z) * s for the 4-bit code q.  p->w holds the codes as packed by
 * quantize_w4_groups (vila_b200/model/qwen2.py, which owns the byte order: 16-row tiles in mma fragment
 * order, ceil(N / 16) * 16 * K / 2 bytes, 16-byte aligned); w_scale is bf16 [N, K / 128] and w_zero uint8
 * [N, K / 128].  p->K is the logical K.  x, bias, residual, norm_w and y stay bf16 and the VILA_FLAG_*
 * meanings are unchanged; the epilogue is vila_gemv's (bias, residual, SwiGLU, argmax) and the k-parts
 * are added in a fixed order, so results are bit-repeatable.  Needs K % 128 == 0; there is no
 * register-staged variant, so an unsupported shape is an error, never a launch.  A quarter of the bf16
 * weight bytes.  Replaces the reference's 4-bit loading (load_4bit, llava/model/builder.py:44-51) and
 * its TinyChat W4A16 deployment (AWQ, group 128; README "Quantization and Deployment"). */
int vila_gemv_w4a16(const vila_gemv_params* p, const void* w_scale, const uint8_t* w_zero, void* stream);

/* Batched decode step on the quantized weights: y[m, :] = epilogue(W x[m, :]) for M = 1..16 activation
 * rows in one launch, every weight byte read once.  w, w_scale and w_zero are the same copies as for
 * vila_gemv_fp8 / vila_gemv_w4a16.  Row m of x is at x + m * ldx, of residual at residual + m * ld_res and
 * of y at y + m * ldy (element strides, 16-byte multiples; x, w, y and residual 16-byte aligned).
 * Epilogue per (row, m): the e4m3 row scale, bias, residual (may alias y: added in place) or SwiGLU on
 * interleaved (gate, up) rows (y then has N / 2 values per row); no RMSNorm prologue and no argmax.
 * Each output row depends on its own x row only: the partition follows from (N, K) and the device, and
 * every sum runs in a fixed order, so a row's bits do not change with M or with the other rows.
 * Errors, never a launch: M outside 1..16, K % 128 != 0 (w4a16) or K % 16 != 0 (fp8), misaligned
 * pointers or strides, missing scales or zero points, odd N with SwiGLU, flags other than
 * VILA_FLAG_SWIGLU | VILA_FLAG_STATIC_W.
 * vila_gemv_batch_fp8 replaces the Linear layers of a batched decode step (HF nn.Linear at
 * modeling_qwen2.py:81-95,164-176,223-226 over a batch of sequences) on e4m3 weights; vila_gemv_batch_w4a16
 * the TinyChat W4A16 GEMM of the reference's 4-bit deployment (README "Quantization and Deployment"). */
typedef struct vila_gemv_batch_params {
  const void* x;
  int64_t ldx;
  const void* w;
  const void* bias;
  const void* residual;
  int64_t ld_res;
  void* y;
  int64_t ldy;
  int32_t M, N, K;
  int32_t flags;
} vila_gemv_batch_params;
int vila_gemv_batch_fp8(const vila_gemv_batch_params* p, const float* w_scale, void* stream);
int vila_gemv_batch_w4a16(const vila_gemv_batch_params* p, const void* w_scale, const uint8_t* w_zero,
                          void* stream);
/* The partition vila_gemv_batch_* use for (N, K) on the current device (fp8: 1 for e4m3 weights, 0 for
 * w4a16): out[0] cluster size, out[1] CTAs, out[2] 16-row tiles per cluster, out[3] k-parts per slice,
 * out[4] cudaOccupancyMaxActiveClusters at that cluster size, out[5] dynamic shared memory per CTA. */
int vila_gemv_batch_partition(int N, int K, int fp8, int32_t* out);

int vila_argmax_finalize(unsigned long long* key, int32_t* token_out, int32_t* token_hist,
                         int32_t* step_counter, int32_t* position, const void* embed_table,
                         void* x_next, int hidden, void* stream);

typedef struct vila_decode_attn_params {
  void* qkv;
  const int32_t* position;
  void* k_pool;
  void* v_pool;
  const int32_t* page_table;
  void* out;
  float* ws;         /* >= Hkv*num_splits*G*(D+2) floats */
  int32_t* counters; /* Hkv ints, zero-initialised once */
  const float* inv_freq;
  int32_t Hq, Hkv, D, num_splits; /* num_splits 0: one CTA per query head, no split: the cache holds at
                                     most 1024 tokens (page_table has >= 8 entries); 1..8: KV splits as a
                                     thread-block cluster; 9..64: splits combined through ws/counters */
  float scale;
} vila_decode_attn_params;
int vila_decode_attention(const vila_decode_attn_params* p, void* stream);

/* Batched decode attention for continuous batching over ONE shared paged pool: `batch` sequences, sequence
 * b uses qkv + b*qkv_stride, out + b*out_stride, position[b] (< 0: idle slot, skipped) and the page-table
 * row page_table + b*pt_stride (max_pages <= 32 valid entries: contexts up to 4096 tokens; longer ones:
 * vila_decode_attention_split_batch).  ws / counters / num_splits of the struct are ignored.  One CTA per
 * (query head, sequence); RoPE + KV append fused. */
int vila_decode_attention_batch(const vila_decode_attn_params* p, int batch, int qkv_stride,
                                int out_stride, int pt_stride, int max_pages, void* stream);

/* Long-context decode attention (video: 16K-66K cached tokens = 34-135 MB of K/V per layer): RoPE +
 * KV append for the new token, then the wgmma FMHA kernel in split-KV mode (the G query heads of a
 * KV group are the query rows of its 128-row tile; K/V pages stream through TMA on
 * Hkv * num_splits CTAs), then a deterministic combine.  split j covers tokens
 * [j*split_tokens, (j+1)*split_tokens) (multiple of 128; num_splits*split_tokens >= max context).
 * Replaces the same HF calls as vila_decode_attention (apply_rotary_pos_emb + DynamicCache.update +
 * flash-attn decode, modeling_qwen2.py:99-160,262-310). */
typedef struct vila_decode_attn_split_params {
  void* qkv;
  const int32_t* position;
  void* k_pool;
  void* v_pool;
  const int32_t* page_table;
  int64_t kv_num_pages;
  void* out;
  float* o_partial; /* >= num_splits*Hq*D floats */
  float* lse;       /* >= num_splits*Hq floats */
  int32_t* counters; /* Hkv ints, zero before the first launch (self-cleaning): the last split CTA of a KV head
                        merges the partials itself; NULL: a separate combine kernel is launched */
  const float* inv_freq;
  int32_t Hq, Hkv, D, num_splits, split_tokens;
  float scale;
} vila_decode_attn_split_params;
int vila_decode_attention_split(const vila_decode_attn_split_params* p, void* stream);

/* Batched form of vila_decode_attention_split for continuous batching at video contexts, over ONE shared
 * paged pool: sequence b uses qkv + b*qkv_stride, out + b*out_stride, position[b] (< 0: idle slot, skipped
 * entirely) and the page-table row page_table + b*pt_stride.  o_partial / lse / counters grow by `batch`:
 * batch*num_splits*Hq*D floats, batch*num_splits*Hq floats and batch*Hkv ints; counters are required
 * (zero before the first launch, self-cleaning).  Split CTAs past a sequence's length exit at once.
 * Every non-idle sequence's output and appended K/V are bit-identical to vila_decode_attention_split with
 * counters on that sequence alone with the same num_splits / split_tokens. */
int vila_decode_attention_split_batch(const vila_decode_attn_split_params* p, int batch, int qkv_stride,
                                      int out_stride, int pt_stride, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Opt-in FP8 KV cache of the batched engine.  Format: codes e4m3 [L, 2, P, 128, Hkv, 128] (the bf16 pool's
 * layout with 1-byte elements, K after RoPE) and fp32 scales [L, 2, P, 128, Hkv], one per row of 128 values:
 *   amax = max|x|, inv = 448 / amax (fp32), code = e4m3(rn, satfinite)(x * inv), scale = amax / 448;
 *   amax == 0: codes and scale 0.  The dequantised value is float(code) * scale.
 * Both entry points replace DynamicCache.update + flash-attn decode (in-tree copy
 * llava/eval/vision_niah_vila/zigzag_ring_attn/modeling_qwen2.py:99-160,262-310) for this format.
 * ------------------------------------------------------------------------------------------- */
/* Rows [0, S) of every layer's K and V of a bf16 cache src [L, 2, src_tokens, Hkv, 128] (a prefill's staging
 * cache with identity pages) -> dst codes [L, 2, dst_pages, 128, Hkv, 128] and dst_scale [L, 2, dst_pages, 128,
 * Hkv], token t going to page page_table[t / 128] (pt_len entries, device int32).  One launch.  head_dim 128;
 * src / dst 16-byte aligned. */
int vila_kv_quantize_fp8(const void* src, int64_t src_tokens, void* dst, float* dst_scale, int64_t dst_pages,
                         const int32_t* page_table, int pt_len, int L, int Hkv, int D, int S, void* stream);
/* One decode step of `batch` sequences over one shared e4m3 pool (this layer's k_pool / v_pool [P, 128, Hkv, 128],
 * k_scale / v_scale [P, 128, Hkv]).  Sequence b uses qkv + b*qkv_stride (bf16, pre-RoPE, not modified),
 * out + b*out_stride, position[b] (< 0: idle, skipped) and the page-table row page_table + b*pt_stride.  Per
 * sequence: RoPE of q and of the new k, the new k / v row quantised and appended at position[b], attention over
 * [0, position[b]] on the dequantised rows (the new row as later steps will read it).  Grid (num_splits, Hkv,
 * batch): split j covers tokens [j*split_tokens, (j+1)*split_tokens) (split_tokens a multiple of 128, <= 2048;
 * num_splits * split_tokens and pt_stride * 128 must exceed every position), split CTAs past a sequence's length
 * exit at once and the last CTA of a (sequence, KV head) combines the splits that hold tokens in index order.  A
 * sequence's output and appended bytes depend on that sequence only (not on num_splits or the other rows).
 * ws >= batch*Hkv*num_splits*G*(D+2) floats; counters batch*Hkv ints, zero before the first launch
 * (self-cleaning).  head_dim 128, G = Hq / Hkv <= 16. */
typedef struct vila_decode_attn_fp8_params {
  const void* qkv;
  const int32_t* position;
  void* k_pool;
  void* v_pool;
  float* k_scale;
  float* v_scale;
  const int32_t* page_table;
  void* out;
  float* ws;
  int32_t* counters;
  const float* inv_freq;
  int32_t Hq, Hkv, D, batch, qkv_stride, out_stride, pt_stride, num_splits, split_tokens;
  float scale;
} vila_decode_attn_fp8_params;
int vila_decode_attention_fp8_batch(const vila_decode_attn_fp8_params* p, void* stream);

/* ---------------------------------------------------------------------------------------------
 * vila_sample_batch — the next token of M rows of bf16 logits [M, V] (row stride ld), each with its own
 * temperature, top-k, top-p, 64-bit seed and token index, drawn on the device.  Replaces HF
 * TemperatureLogitsWarper / TopKLogitsWarper / TopPLogitsWarper + torch.multinomial in GenerationMixin._sample,
 * reached from llava_arch.py:823-833.  The rule (vila_b200/sampling.py states it in torch / numpy):
 *   greedy   inv_temperature == 0 or top_k == 1: the first index of max float(logit) (torch.argmax)
 *   scaling  s_i = float(logit_i) * inv_temperature (fp32)
 *   top-k    0 < top_k < V: keep s_i >= the k-th largest s (ties kept)
 *   top-p    top_p < 1: p_i = exp(s_i - max s), Z = sum of p over the top-k survivors; keep survivor i iff the mass
 *            of survivors with a strictly larger s is < top_p * Z (the kernel sums floor(p_i * 2^40) in integers)
 *   draw     argmax over the kept set of s_i + g_i, ties to the lowest index; g_i = -log(-log1p(-u_i)),
 *            u_i = (x_i + 0.5) * 2^-32, x_i word i % 4 of Philox-4x32-10, key (seed lo, seed hi), counter
 *            (i / 4, step lo, step hi, 0)
 * A row with position < 0 is idle: tokens[row] (and n_kept[row]) are left untouched.  n_kept (may be NULL) gets
 * the size of each row's kept set (1 for greedy rows).  A row's token depends only on its logits, parameters, seed
 * and step: not on M, on the row index or on the other rows.  Deterministic bits; no float atomics.
 * 1 <= V <= 327,680, M <= 65535.  One cluster of 8 CTAs per row.
 * ------------------------------------------------------------------------------------------- */
typedef struct vila_sample_params {
  const void* logits;
  int64_t ld;
  const float* inv_temperature;
  const int32_t* top_k;
  const float* top_p;
  const int64_t* seed;
  const int64_t* step;
  const int32_t* position;
  int64_t* tokens;
  int32_t* n_kept;
  int32_t M, V;
} vila_sample_params;
int vila_sample_batch(const vila_sample_params* p, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VILA_B200_H_ */
