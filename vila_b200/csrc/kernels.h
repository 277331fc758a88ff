// Internal (C++) launcher declarations shared between the .cu translation units.
// The public surface is the C-ABI in include/vila_b200.h (implemented in api.cu).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace vb {

enum Act : int { ACT_NONE = 0, ACT_GELU_TANH = 1, ACT_GELU_ERF = 2, ACT_SILU = 3 };

struct GemmEpilogue {
  const __nv_bfloat16* bias = nullptr;      // [N]
  const __nv_bfloat16* residual = nullptr;  // [rows, ld_res]; row = m % res_row_mod (if > 0) else m
  int ld_res = 0;
  int res_row_mod = 0;
  int act = ACT_NONE;
  int swiglu = 0;  // interleaved (gate, up) columns -> N/2 outputs of silu(gate) * up
  int static_w = 0;  // W is a parameter: its first pipeline stages may be fetched before the PDL wait
  // split-K (set by the launcher): fp32 partial-sum workspace [M, N] (zeroed, self-cleaning) and
  // per-tile arrival counters (zeroed, self-cleaning)
  float* splitk_ws = nullptr;
  int* splitk_counters = nullptr;
  int split_k = 1;
  // q/k/v projection + RoPE (gemm_qkv_rope_bf16 only, head_dim == 128): RoPE on the q and k heads
  // and the KV-cache append after the GEMM.  N = (rope_hq + 2 rope_hkv) * 128; q heads stay in C,
  // k/v heads go to the pools (or stay in C when the pools are null).
  const __nv_bfloat16* rope_table = nullptr;  // [M, 128]: cos[0..64) | sin[0..64) per token (rope_table())
  __nv_bfloat16* k_pool = nullptr;         // paged pools [pages, 128, Hkv, 128] (nullptr: k/v stay in C)
  __nv_bfloat16* v_pool = nullptr;
  const int32_t* page_table = nullptr;
  int cache_pos0 = 0;
  int rope_hq = 0, rope_hkv = 0;
};

int set_workspace(void* ptr, size_t bytes);
void get_workspace(void** ptr, size_t* bytes);
int gemm_bf16(const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int ldw, __nv_bfloat16* C,
              int ldc, int M, int N, int K, const GemmEpilogue& epi, cudaStream_t stream);
int gemm_qkv_rope_bf16(const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int ldw, __nv_bfloat16* C,
                       int ldc, int M, int N, int K, const GemmEpilogue& epi, cudaStream_t stream);  // -1: not covered
int gemm_bf16_cfg(int block_n, const __nv_bfloat16* A, int lda, const __nv_bfloat16* W, int ldw,
                  __nv_bfloat16* C, int ldc, int M, int N, int K, const GemmEpilogue& epi,
                  cudaStream_t stream);

// ---- attention (prefill / ViT) -----------------------------------------------------------------
struct FmhaParams {
  const __nv_bfloat16* q;  // [B*Sq, Hq, D] view: element (t, h, d) at q + t*q_tok_stride + h*q_head_stride + d
  int64_t q_tok_stride, q_head_stride;
  // K/V are addressed as pages of 128 tokens: page p, token r, head h at
  //   k + p*kv_page_stride + r*kv_tok_stride + h*kv_head_stride
  const __nv_bfloat16* k;
  const __nv_bfloat16* v;
  int64_t kv_page_stride, kv_tok_stride, kv_head_stride;
  int64_t kv_num_pages;        // extent of the page dimension (TMA bound)
  const int32_t* page_table;   // [B, max_pages_per_seq] or nullptr (then page = b*pages_per_seq + j)
  int page_table_stride;
  __nv_bfloat16* o;            // [B*Sq, Hq, D] same addressing scheme as q (o_tok_stride, o_head_stride)
  int64_t o_tok_stride, o_head_stride;
  int B, Sq, Sk, Hq, Hkv;
  int D;            // real head dim (72 or 128); padded internally by TMA zero fill
  int causal;       // 1: kv <= q + (Sk - Sq)
  float scale;      // softmax scale (1/sqrt(D))
};
int fmha_prefill(const FmhaParams& p, cudaStream_t stream);
// variant: 0 default, 1 / 2 the wgmma kernel, 3 / 4 with every 4th / 2nd exp2 on the FMA pipe
int fmha_prefill_cfg(int variant, const FmhaParams& p, cudaStream_t stream);
// split-KV mode of the attention kernel for decode at long context (see fmha_wgmma.cu)
// counters != nullptr ([Hq] ints, zero-initialised once): the last split CTA of a head combines into p.o
// batch > 0: that many sequences in one launch (per-sequence lengths, page-table rows, work buffers)
int fmha_decode_split(const FmhaParams& p, const int32_t* n_tok_minus_1, int split_tokens,
                      float* o_partial, float* lse, int* counters, cudaStream_t stream,
                      int batch = 0, int64_t q_seq_stride = 0, int64_t o_seq_stride = 0);

// ---- norms ---------------------------------------------------------------------------------------
int layernorm_bf16(const __nv_bfloat16* x, const __nv_bfloat16* w, const __nv_bfloat16* b,
                   __nv_bfloat16* out, int rows, int cols, float eps, cudaStream_t stream);
// out = w * bf16(x * rsqrt(mean(x^2) + eps));  if residual_add != nullptr: x += residual_add first
// (the sum is written back to x_inout so it becomes the new residual stream).
int rmsnorm_bf16(__nv_bfloat16* x_inout, const __nv_bfloat16* residual_add,
                 const __nv_bfloat16* w, __nv_bfloat16* out, int rows, int cols, float eps,
                 cudaStream_t stream);

// ---- vision-side data movement ------------------------------------------------------------------
int im2col_patch14(const __nv_bfloat16* pixels, __nv_bfloat16* out, int B, int C, int H, int W,
                   int patch, int k_pad, cudaStream_t stream);
int space_to_depth(const __nv_bfloat16* x, __nv_bfloat16* out, int B, int h, int w, int C, int r,
                   cudaStream_t stream);
// dynamic-S2: tiles [n_tiles, side*side, C] of one image (scales[0..ns), last scale bh x bw tiles)
// -> out [bh_o*bw_o, side*side, ns*C] (merge_chessboard + area resize + channel concat + split)
int s2_merge(const __nv_bfloat16* tiles, __nv_bfloat16* out, int side, int C, int n_scales,
             const int* scale_splits_h, const int* scale_splits_w, int out_bh, int out_bw,
             int share_tile /* block_size None: every scale reads tile 0 */, cudaStream_t stream);
// merge_chessboard of projected tiles: [bh*bw, s*s, C] -> [(bh*s)*(bw*s), C]
int chessboard_merge(const __nv_bfloat16* tiles, __nv_bfloat16* out, int bh, int bw, int s, int C,
                     cudaStream_t stream);
// TSP pooling: [T, h, w, C] mean over (pt, ph, pw) groups -> [T/pt, h/ph, w/pw, C]
int tsp_pool(const __nv_bfloat16* x, __nv_bfloat16* out, int T, int h, int w, int C, int pt, int ph,
             int pw, cudaStream_t stream);

// PIL-exact bicubic resize (+ 1/255 rescale, (x-mean)/std, tiling) of a uint8 HWC image into bf16
// tiles [n, 3, tile, tile]; integer filter taps (Pillow's 22-bit fixed point) come from the host.
int resize_bicubic_tiles(const uint8_t* src, int H, int W, int out_w, int out_h, const int32_t* coef_x,
                         const int32_t* bounds_x, int ksize_x, const int32_t* coef_y,
                         const int32_t* bounds_y, int ksize_y, uint8_t* tmp, __nv_bfloat16* out_tiles,
                         int tile, int tile_index0, float mean, float stdv, cudaStream_t stream);

// ---- LLM-side data movement ---------------------------------------------------------------------
// out[i,:] = src[i] >= 0 ? table[src[i],:] : media[-(src[i]+1),:]
int embed_splice(const __nv_bfloat16* table, const __nv_bfloat16* media, const int32_t* src,
                 __nv_bfloat16* out, int rows, int cols, cudaStream_t stream);
// In-place rotate-half RoPE on q and k heads of a fused qkv buffer [S, (Hq+2Hkv)*D], then scatter
// k and v rows into the paged KV pool.
int rope_table(const int32_t* positions, int S, int D, const float* inv_freq, __nv_bfloat16* table,
               cudaStream_t stream);
int rope_kv_append(__nv_bfloat16* qkv, const int32_t* positions, int S, int Hq, int Hkv, int D,
                   const float* inv_freq, __nv_bfloat16* k_pool, __nv_bfloat16* v_pool,
                   const int32_t* page_table, int cache_pos0, cudaStream_t stream);
// decode step of `batch` sequences: row b of qkv at qkv + b*qkv_stride, position positions[b] (< 0: idle
// row, untouched), page-table row page_table + b*pt_stride; the k / v rows go to slot = position
int rope_kv_append_decode_batch(__nv_bfloat16* qkv, long qkv_stride, const int32_t* positions, int batch,
                                int Hq, int Hkv, int D, const float* inv_freq, __nv_bfloat16* k_pool,
                                __nv_bfloat16* v_pool, const int32_t* page_table, int pt_stride,
                                cudaStream_t stream);

// same with cos / sin read from rope_table(positions) (long prefills; bit-identical)
int rope_kv_append_table(__nv_bfloat16* qkv, const __nv_bfloat16* table, int S, int Hq, int Hkv, int D,
                         __nv_bfloat16* k_pool, __nv_bfloat16* v_pool, const int32_t* page_table,
                         int cache_pos0, cudaStream_t stream);

// ---- decode (M == 1) ----------------------------------------------------------------------------
struct GemvParams {
  const __nv_bfloat16* x;       // [K]
  const __nv_bfloat16* w;       // [N, K] (gemv_tma_fp8: e4m3 bytes; gemv_tma_w4a16: packed 4-bit codes)
  const __nv_bfloat16* bias;    // [N] or null
  const __nv_bfloat16* norm_w;  // [K] or null: fused RMSNorm prologue on x
  float norm_eps;
  const __nv_bfloat16* residual;  // [N] or null (added after bias)
  __nv_bfloat16* y;               // [N] (or [N/2] with swiglu)
  int N, K;
  int flags;   // bit0: SwiGLU (rows interleaved gate, up); bit1: weights are static (stream before the PDL wait); bit2: force the register-staged kernel
  // optional fused greedy argmax over y (lm_head): 64-bit packed (value, ~index) max-reduction
  unsigned long long* argmax_key;
  const float* w_scale;  // [N] per-row scale of e4m3 weights (gemv_tma_fp8 only)
};
int gemv_bf16(const GemvParams& p, cudaStream_t stream);
int gemv_tma_bf16(const GemvParams& p, cudaStream_t stream);  // -1: shape not supported
int gemv_tma_fp8(const GemvParams& p, cudaStream_t stream);   // e4m3 weights, K % 16 == 0
// 4-bit weights packed by quantize_w4_groups (vila_b200/model/qwen2.py), bf16 scales and uint8 zero
// points [N, K / 128]; K % 128 == 0
int gemv_tma_w4a16(const GemvParams& p, const __nv_bfloat16* w_gscale, const uint8_t* w_zero, cudaStream_t stream);
// M <= 16 activation rows against the same quantized copies (gemv_batch_kernel): y[m] = epilogue(W x[m])
struct GemvBatchArgs {
  const __nv_bfloat16* x;         // [M, ldx]
  int64_t ldx;
  const void* w;                  // e4m3 [N, K], or the packed 4-bit codes
  const __nv_bfloat16* bias;      // [N] or null
  const __nv_bfloat16* residual;  // [M, ld_res] or null; may alias y
  int64_t ld_res;
  __nv_bfloat16* y;               // [M, ldy]: N (or N/2 with SwiGLU) values per row
  int64_t ldy;
  int M, N, K, flags;             // flags: bit0 SwiGLU, bit1 static weights
};
int gemv_batch_fp8(const GemvBatchArgs& p, const float* w_scale, cudaStream_t stream);
int gemv_batch_w4a16(const GemvBatchArgs& p, const __nv_bfloat16* w_gscale, const uint8_t* w_zero,
                     cudaStream_t stream);
// out: {cluster size, CTAs, tiles per cluster, k-parts per slice, max active clusters, dynamic smem bytes}
int gemv_batch_partition(int N, int K, int fp8, int32_t* out);
// token = argmax key; token_hist[step++] = token; position++; key = 0; x_next = embed_table[token]
int argmax_finalize(unsigned long long* key, int32_t* token_out, int32_t* token_hist,
                    int32_t* step_counter, int32_t* position, const __nv_bfloat16* embed_table,
                    __nv_bfloat16* x_next, int hidden, cudaStream_t stream);

struct DecodeAttnParams {
  __nv_bfloat16* qkv;          // [ (Hq+2Hkv)*D ] pre-RoPE, current token
  const int32_t* position;     // device scalar: position id of the current token (== cache length)
  __nv_bfloat16* k_pool;       // this layer's K pages [P,128,Hkv,D]
  __nv_bfloat16* v_pool;
  const int32_t* page_table;   // [max_pages]
  __nv_bfloat16* out;          // [Hq*D]
  float* ws;                   // split-KV workspace
  int32_t* counters;           // [Hkv] zero-initialised arrival counters
  const float* inv_freq;       // [D/2] fp32 (HF rotary inv_freq, computed on the host like HF does)
  int Hq, Hkv, D, num_splits;
  float scale;
};
int decode_attention(const DecodeAttnParams& p, cudaStream_t stream);
// batch of sequences over ONE shared paged pool (continuous batching): sequence b uses qkv + b*qkv_stride,
// out + b*out_stride, position[b] (< 0: idle slot) and page_table + b*pt_stride (max_pages valid entries,
// <= 32 = 4096 tokens); one CTA per (query head, sequence)
int decode_attention_batch(const DecodeAttnParams& p, int batch, int qkv_stride, int out_stride,
                           int pt_stride, int max_pages, cudaStream_t stream);
struct DecodeAttnSplitParams {
  __nv_bfloat16* qkv;          // [(Hq+2Hkv)*D] pre-RoPE, current token (q / k rotated in place)
  const int32_t* position;     // device scalar: position id of the current token == tokens cached so far
  __nv_bfloat16* k_pool;       // this layer's K pages [P,128,Hkv,D]
  __nv_bfloat16* v_pool;
  const int32_t* page_table;
  int64_t kv_num_pages;
  __nv_bfloat16* out;          // [Hq*D]
  float* o_partial;            // [num_splits, Hq, D] fp32
  float* lse;                  // [num_splits, Hq]
  int32_t* counters;           // [Hkv] zero-initialised once (self-cleaning), or null: separate combine launch
  const float* inv_freq;
  int Hq, Hkv, D, num_splits, split_tokens;
  float scale;
};
int decode_attention_split(const DecodeAttnSplitParams& p, cudaStream_t stream);
// batch of sequences over ONE shared paged pool, long contexts: sequence b uses qkv + b*qkv_stride,
// out + b*out_stride, position[b] (< 0: idle) and page_table + b*pt_stride; o_partial / lse / counters
// hold `batch` blocks of the single-sequence sizes; counters are required (fused combine)
int decode_attention_split_batch(const DecodeAttnSplitParams& p, int batch, int qkv_stride, int out_stride,
                                 int pt_stride, cudaStream_t stream);

// ---- opt-in e4m3 KV cache of the batched engine (kv_fp8.cu) -------------------------------------
// rows [0, S) of every layer's K and V of a bf16 staging cache [L, 2, src_tokens, Hkv, 128] -> e4m3 codes
// [L, 2, dst_pages, 128, Hkv, 128] and fp32 scales [L, 2, dst_pages, 128, Hkv] through one page-table row
int kv_quantize_fp8(const __nv_bfloat16* src, int64_t src_tokens, uint8_t* dst, float* dst_scale, int64_t dst_pages,
                    const int32_t* page_table, int pt_len, int L, int Hkv, int D, int S, cudaStream_t stream);
struct DecodeAttnFp8Params {
  const __nv_bfloat16* qkv;    // [batch, qkv_stride] pre-RoPE, current token (not modified)
  const int32_t* position;     // [batch] position of the new token == tokens cached (< 0: idle slot)
  uint8_t* k_pool;             // this layer's e4m3 K pages [P, 128, Hkv, 128]
  uint8_t* v_pool;
  float* k_scale;              // [P, 128, Hkv]
  float* v_scale;
  const int32_t* page_table;   // [batch, pt_stride]
  __nv_bfloat16* out;          // [batch, out_stride]
  float* ws;                   // >= batch * Hkv * num_splits * G * (D + 2) floats
  int32_t* counters;           // [batch * Hkv], zero before the first launch (self-cleaning)
  const float* inv_freq;       // [D/2]
  int Hq, Hkv, D, batch, qkv_stride, out_stride, pt_stride, num_splits, split_tokens;
  float scale;
};
int decode_attention_fp8_batch(const DecodeAttnFp8Params& p, cudaStream_t stream);

// ---- temperature / top-k / top-p sampling of the batched engine (sample.cu) ----------------------
struct SampleParams {
  const __nv_bfloat16* logits;   // [M, ld]
  int64_t ld;                    // row stride (elements), >= V
  const float* inv_temperature;  // [M] 1/T (0: greedy)
  const int32_t* top_k;          // [M] 0 or >= V: off
  const float* top_p;            // [M] 1: off
  const int64_t* seed;           // [M]
  const int64_t* step;           // [M] index t of the token being drawn
  const int32_t* position;       // [M] < 0: idle row, tokens[row] untouched
  int64_t* tokens;               // [M] out
  int32_t* n_kept;               // [M] out (size of the kept set) or null
  int M, V;
};
int sample_batch(const SampleParams& p, cudaStream_t stream);

}  // namespace vb
