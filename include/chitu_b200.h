/*
 * chitu_b200.h — C ABI of the H100-native (sm_90a) decode operator library (libchitu_b200.so).
 *
 * This is the drop-in boundary for Chitu's decode hot path (SURVEY.md §8b). Every entry
 * point replaces one reference operator; the reference interface it replaces is cited as
 * file:line relative to the thu-pacman/chitu tree.  The reference binds native code through
 * a pybind11 module (csrc/binding.cpp:11-19) and Triton JIT launches; here the binding is a
 * plain C ABI (ctypes from Python, see INTEGRATION.md).
 *
 * Conventions (all entry points)
 *   - Plain pointers + sizes only.  Pointers are DEVICE pointers unless stated otherwise.
 *   - The library never allocates, frees or synchronises: callers own outputs/workspaces.
 *   - Every function takes the CUDA stream to launch on (`void* stream` == cudaStream_t);
 *     no default-stream use, no host sync  => CUDA-graph capturable
 *     (reference requirement: chitu/models/model.py:572-611).
 *   - Return value: 0 = ok, <0 = bad argument, >0 = cudaError_t.  Message via
 *     chitu_b200_last_error() (thread local).  Never exit()/abort() (the reference does:
 *     csrc/common.h:20-41).
 *   - dtype codes: see CB_* below.
 */
#ifndef CHITU_B200_H_
#define CHITU_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
  CB_BF16 = 0,
  CB_F16 = 1,
  CB_F32 = 2,
  CB_FP8_E4M3 = 3,
  CB_I8 = 4,
  CB_U8 = 5,
  CB_I16 = 6,
  CB_I32 = 7,
  CB_I64 = 8
};

/* ---- library / error plumbing ------------------------------------------------------- */
const char* chitu_b200_last_error(void);
int chitu_b200_version(void);
/* Number of kernels this library has launched in this process (bench.py "gpu_launches"). */
int64_t chitu_b200_launch_count(void);

/* ---- KV paging ---------------------------------------------------------------------- */
/* Replaces chitu/ops.py:50-91 append_to_paged_kv_cache + triton_kernels.py:18-48.
 * kv_cache[page_table[b, old_len[b] / index_div], old_len[b] % index_div, :] = this_kv[b, :]
 * The reference hard-codes index_div = 64 (triton_kernels.py:38,42) while the row address
 * uses the true page_size; both are parameters here so the quirk is reproducible bit-exactly.
 * row_bytes = bytes of one token's entry (all trailing dims). */
int chitu_b200_append_paged_kv(void* kv_cache, const int32_t* page_table, const void* this_kv,
                               const int32_t* old_seq_lens, int batch, int pages_per_sample,
                               int page_size, int index_div, int64_t row_bytes, void* stream);

/* ---- MoE routing / permutation -------------------------------------------------------- */
/* Replaces csrc/moe_align_kernel.cu:27-122 (pybind csrc/binding.cpp:11,
 * chitu_backend.cuda_moe_align_block_size) and the Triton fallback fused_moe.py:314-442.
 * Same in-place contract: sorted_ids pre-filled with numel, expert_ids zero-filled by caller
 * (fused_moe.py:491-505).  Order inside an expert segment is ascending token index (the
 * Triton fallback's order; the reference CUDA kernel's atomics make it non-deterministic). */
int chitu_b200_moe_align_block_size(const void* topk_ids, int ids_dtype, int64_t numel,
                                    int num_experts, int block_size, int32_t* sorted_ids,
                                    int32_t* expert_ids, int32_t* num_tokens_post_pad,
                                    int32_t* cumsum, void* stream);

/* Replaces GateDeepSeekV3.forward (model_deepseek_v3.py:810-842): gate GEMV + sigmoid|softmax
 * + bias + group-limited top-k + renormalise + route_scale, one kernel.
 * x[T,dim] (bf16), w[E,dim] (bf16), bias[E] (f32 or bf16, may be NULL).
 * out_weights[T,topk] (bf16), out_indices[T,topk] (int64 as torch.topk returns).
 * workspace (zero-filled once, chitu_b200_moe_gate_workspace_bytes): gate logits + the GEMM's
 * split-K scratch; NULL selects a slow in-kernel GEMV. */
int64_t chitu_b200_moe_gate_workspace_bytes(int T, int E);
int chitu_b200_moe_gate(const void* x, const void* w, const void* bias, int bias_dtype, int T,
                        int dim, int E, int n_groups, int topk_groups, int topk, int score_sigmoid /* 0 softmax, 1 sigmoid (DeepSeek), 2 softmax + top-k renormalisation (Mixtral, model_hf_mixtral.py:57-64) */,
                        float route_scale, void* out_weights, int64_t* out_indices,
                        int out_stride /* elements per token row of both outputs, >= topk */, void* workspace,
                        int64_t workspace_bytes, void* stream);
/* The same gate, whose LAST CTA also writes the expert plan (sort by expert, row chunks, tile lists — the work of
 * moe_align_block_size, fused_moe.py:599-610, inside fused_experts_impl fused_moe.py:1130-1307) of the fused_experts call
 * that follows, into that call's workspace: the pairs are the [T, out_stride] rows of out_indices / out_weights (engines pre-fill column `topk` with the shared
 * expert).  Follow with chitu_b200_fused_experts_planned(T, topk = out_stride, E_total, N1, K1, moe_workspace).
 * One dependent launch fewer per MoE layer; the in-kernel hand-off is serial work on the critical path, so the
 * engines keep it off by default. */
int chitu_b200_moe_gate_plan(const void* x, const void* w, const void* bias, int bias_dtype, int T, int dim, int E,
                             int n_groups, int topk_groups, int topk, int score_sigmoid, float route_scale,
                             void* out_weights, int64_t* out_indices, int out_stride, void* workspace,
                             int64_t workspace_bytes, int E_total, int N1, int K1, void* moe_workspace,
                             int64_t moe_workspace_bytes, void* stream);

/* ---- rotary --------------------------------------------------------------------------- */
/* Replaces triton_kernels.py:101-190 (rotary_type="llama", interleaved pairs; cos/sin f32
 * [bs, rot/2]) — ops.py:178-237.  q:[bs,hq,rot] k:[bs,hk,rot], strides in elements. */
int chitu_b200_rotary_interleaved(const void* q, const void* k, void* out_q, void* out_k,
                                  const float* cos, const float* sin, int bs, int hq, int hk,
                                  int rot_dim, int64_t q_sb, int64_t q_sh, int64_t k_sb, int64_t k_sh,
                                  int dtype, void* stream);
/* Same, with explicit output batch strides (elements) so the rotated k_pe can be written
 * straight into the [kv_norm(kv) | k_pe] row that is appended to the MLA cache
 * (model_deepseek_v3.py:684-686 builds it with torch.cat). */
int chitu_b200_rotary_interleaved_strided(const void* q, const void* k, void* out_q, void* out_k,
                                          const float* cos, const float* sin, int bs, int hq, int hk,
                                          int rot_dim, int64_t q_sb, int64_t q_sh, int64_t k_sb,
                                          int64_t k_sh, int64_t oq_sb, int64_t ok_sb, int dtype,
                                          void* stream);
/* Replaces triton_kernels.py:51-98 (rotary_type="hf-llama", half-split); cos/sin in the
 * tensor dtype [bs, head_dim/2] (ops.py:124-176).  x:[bs,h,head_dim] contiguous. */
int chitu_b200_rotary_half(const void* x, void* out, const void* cos, const void* sin, int bs,
                           int heads, int head_dim, int dtype, void* stream);
/* Same with a batch stride (elements) on the input rows: x is a q / k view of a merged qkv GEMM output. */
int chitu_b200_rotary_half_strided(const void* x, int64_t x_sb, void* out, const void* cos, const void* sin, int bs,
                                   int heads, int head_dim, int dtype, void* stream);

/* ---- norms / activation / quantisers -------------------------------------------------- */
/* RMSNorm.forward (models/model.py:50-78): y = x * rsqrt(mean(x^2)+eps) * w, fp32 math,
 * one rounding to the io dtype.  Optional fused residual: if residual != NULL,
 * x <- x + residual is written to residual_out first (used by the decode engine). */
int chitu_b200_rmsnorm(const void* x, const void* w, void* y, int rows, int dim, float eps,
                       int dtype, void* stream);
/* Same with row strides in elements (q_norm / kv_norm act on column slices of the fused
 * wqkv_a output, model_deepseek_v3.py:480-488, 684). */
int chitu_b200_rmsnorm_strided(const void* x, const void* w, void* y, int rows, int dim, int64_t x_stride,
                               int64_t y_stride, float eps, int dtype, void* stream);
/* Fused RMSNorm + act_quant_deepseek_v3 (the `norm -> linear_deepseek_v3` pairs of the DeepSeek layer,
 * model_deepseek_v3.py:488,1108,1113 + :53-106): reads the row once; writes y (bf16, may be NULL) and / or
 * the fp8 payload q [rows, dim] + scales [rows, dim/128] (both NULL to skip).  bf16, dim % 128 == 0. */
int chitu_b200_rmsnorm_quant_fp8(const void* x, const void* w, void* y, void* q, float* q_scales, int rows,
                                 int dim, int64_t x_stride, int64_t y_stride, float eps, void* stream);
/* Fused SiluAndMul + act_quant_deepseek_v3: x [rows, 2F] bf16 -> q fp8 [rows, F], scales [rows, F/128]. */
int chitu_b200_silu_mul_quant_fp8(const void* x, void* q, float* q_scales, int64_t rows, int F, void* stream);
/* SiluAndMul (fused_moe.py:24-39): out[r, :d] = silu(x[r, :d]) * x[r, d:2d]. */
int chitu_b200_silu_and_mul(const void* x, void* out, int64_t rows, int d, int dtype, void* stream);
/* act_quant_deepseek_v3 (ops.py:329-353, kernel triton_kernels.py:193-214): per (row, 128-group)
 * s = max|x|/448 (no eps, no clamp), y = fp8_e4m3(x/s).  mode 1 = per_token_group_quant_fp8
 * (fused_moe.py:667-710): s = max(max|x|, eps)/448, y = fp8(clamp(x/s, +-448)). */
int chitu_b200_act_quant_fp8(const void* x, void* y, float* s, int64_t rows, int K, int group,
                             int mode, float eps, int dtype, void* stream);
/* quant_act (quantize/w8a8.py:18-26): per-row scale = clamp(max|x|,1e-5)/127 (fp32),
 * q = int8(round_half_even(x/scale)). x is fp16 or bf16. */
int chitu_b200_quant_act_int8(const void* x, int8_t* q, float* scales, int64_t rows, int K,
                              int dtype, void* stream);
/* weight_dequant_deepseek_v3 / weight_dequant_soft_fp8_deepseek_v3 (ops.py:356-449):
 * y[b,m,n] = fp8(x[b,m,n]) * s[b, m/128, n/128]  -> bf16.  soft != 0 reproduces the
 * bit-trick path ((x&0x80)<<24 | (x&0x7f)<<20) * (s * 2^120). */
int chitu_b200_weight_dequant_fp8(const void* x, const float* s, void* y, int B, int M, int N,
                                  int block, int soft, void* stream);

/* ---- linears (weight-streaming skinny GEMMs; weights are [N,K] row-major = nn.Linear) --- */
/* Workspace for split-K partials + ticket counters: chitu_b200_linear_workspace_bytes(M_max, N_max).
 * It must be zero-filled ONCE before its first use; every call leaves the counters at zero again. */
int64_t chitu_b200_linear_workspace_bytes(int M, int N);
/* impl: 0 = auto, 1 = SIMT weight-streaming GEMV, 2 = wgmma/TMA swap-AB GEMM. */
/* F.linear for bf16/fp16 weights (linear_deepseek_v3 element_size()>1 branch,
 * model_deepseek_v3.py:84-85; tensor_parallel.py linear_op default). y = x W^T (+bias) (+residual). */
int chitu_b200_linear_bf16(const void* x, const void* w, const void* bias, const void* residual,
                           void* y, int M, int N, int K, int dtype, void* workspace,
                           int64_t workspace_bytes, int impl, void* stream);
/* FeedForward gate_up linear + SiluAndMul in one launch (models/model_llama.py:139-149 + fused_moe.py:24-39):
 * w_pairs = the merged [w1 ; w3] weight [N, K] with rows interleaved at load time (row 2i = gate_i, row 2i+1 = up_i);
 * y [M, N/2] bf16 with the roundings of the two separate reference ops.  bf16, wgmma path only. */
int chitu_b200_linear_bf16_silu_pairs(const void* x, const void* w_pairs, void* y, int M, int N, int K, void* workspace,
                                      int64_t workspace_bytes, void* stream);
/* fp8_gemm_deepseek_v3 (ops.py:452-483; kernel triton_kernels.py:303-365):
 * c[m,n] = sum_kb (a[m,kb]·b[n,kb]) * a_s[m,kb] * b_s[n/128,kb], fp32 acc, bf16 out. */
int chitu_b200_fp8_gemm(const void* a, const float* a_s, const void* b, const float* b_s, void* c,
                        int M, int N, int K, const void* residual /* [M,N] bf16 added after rounding, or NULL */,
                        void* workspace, int64_t workspace_bytes, int impl, void* stream);
/* soft_fp8_gemm_deepseek_v3 (ops.py:486-511; kernel triton_kernels.py:388-508): W8A16,
 * weight -> bf16(bits(w) * (b_s*2^120)) then bf16 x bf16 -> fp32 acc -> bf16 out. */
int chitu_b200_soft_fp8_gemm(const void* a, const void* b, const float* b_s, void* c, int M, int N,
                             int K, int out_dtype, void* workspace, int64_t workspace_bytes,
                             int impl, void* stream);
/* w8a8gemm.mm(out, a, b, a_scales, b_scales, bias) and w8a8gemv.mv(a, b, scale_tok, scale_ch)
 * (closed-source; call sites quantize/w8a8.py:105,120,125; pinned by test/pytest/test_w8a8.py):
 * out[m,n] = fp16( (sum_k a[m,k]*b[n,k]) * a_scales[m] * b_scales[n] ) (+ bias[n]). */
int chitu_b200_w8a8_gemm(void* out, const int8_t* a, const int8_t* b, const float* a_scales,
                         const float* b_scales, const void* bias, int M, int N, int K,
                         void* workspace, int64_t workspace_bytes, int impl, void* stream);

/* ---- decode attention -------------------------------------------------------------------- */
/* Workspace sizing for split-KV partials. */
int64_t chitu_b200_attn_workspace_bytes(int batch, int heads, int head_dim_v, int max_splits);

/* AttnBackend.attn_with_kvcache with block_table (attn_backend.py:92-164, FlashAttn impl
 * :208-243; callers models/model.py:167-198): GQA decode, new k/v appended in place at
 * position cache_seqlens[b] (true page_size indexing, as flash_attn does), attention over
 * cache_seqlens[b]+1 keys.  q:[B,Hq,D]  k_cache/v_cache:[num_blocks,page,Hkv,D]
 * k_new/v_new:[B,Hkv,D] with batch strides k_new_sb / v_new_sb in elements (so a fused-qkv GEMM
 * output can be passed without a copy; may be NULL: no append, attend over cache_seqlens[b] keys).
 * out:[B,Hq,D].  dtype bf16|fp16. */
int chitu_b200_gqa_paged_decode(const void* q, void* k_cache, void* v_cache, const void* k_new,
                                const void* v_new, int64_t k_new_sb, int64_t v_new_sb,
                                const int32_t* cache_seqlens,
                                const int32_t* block_table, int bt_stride, int B, int Hq, int Hkv,
                                int D, int page_size, int max_seqlen_hint, float softmax_scale,
                                void* out, void* workspace, int64_t workspace_bytes, int dtype,
                                void* stream);
/* Same kernel with the rotary embedding that precedes it in Attention.decode_forward_paged fused in
 * (models/model.py:167-198: apply_rotary_pos_emb "llama" on q and the new k, then attn_with_kvcache): q / k_new are
 * the UN-rotated views of the fused qkv GEMM output (q batch stride q_sb elements), rope_cos / rope_sin fp32
 * [B, D/2] (ops.py:311-326).  rope_cos == NULL: no rotation (== chitu_b200_gqa_paged_decode with a strided q).
 * Needs D == 128 and a power-of-two page (the tensor-core kernel). */
int chitu_b200_gqa_paged_decode_rope(const void* q, int64_t q_sb, void* k_cache, void* v_cache, const void* k_new,
                                     const void* v_new, int64_t k_new_sb, int64_t v_new_sb, const float* rope_cos,
                                     const float* rope_sin, const int32_t* cache_seqlens, const int32_t* block_table,
                                     int bt_stride, int B, int Hq, int Hkv, int D, int page_size, int max_seqlen_hint,
                                     float softmax_scale, void* out, void* workspace, int64_t workspace_bytes,
                                     int dtype, void* stream);


/* *.mla_attn_with_kvcache (attn_backend.py:536-572 / 660-684 / 707-774) = append
 * (ops.py:50-91) + mla_decode (triton_decode_attention.py:259-290) in one call.
 * q_nope:[B,H,C] q_pe:[B,H,R] kv_cache:[num_blocks,page,C+R] new_kv:[B,C+R] (may be NULL)
 * seqlens_excl:[B] (length before this token) ; attention runs over seqlens_excl+1 keys when
 * new_kv != NULL else over seqlens_excl keys.  out:[B,H,C] (latent space). bf16.
 * num_blocks = kv_cache.shape[0] (bounds the TMA tensor map that stages whole 64-key pages).
 * out == NULL (wgmma kernel only: page 64): the split merge is deferred to chitu_b200_mla_absorb_o_merge_quant. */
int chitu_b200_mla_decode(const void* q_nope, const void* q_pe, void* kv_cache, const void* new_kv,
                          const int32_t* seqlens_excl, const int32_t* block_table, int bt_stride,
                          int B, int H, int C, int R, int page_size, int num_blocks, int max_seqlen_hint,
                          float softmax_scale, void* out, void* workspace, int64_t workspace_bytes,
                          void* stream);

/* invoke_fused_moe_kernel (fused_moe.py:796-891; Triton kernel :62-307) as ONE grouped wgmma GEMM:
 * A bf16 [numel/top_k (GEMM1) or numel (top_k = 1), K]; B stacked expert weights [E, N, K] (bf16 for wmode 0, fp8 +
 * B_scale [E, N/128, K/128] for wmode 1 = fp8_w8a8 — A is quantised per_token_group_quant_fp8 inside, as the reference
 * does at :826 — and wmode 2 = soft_fp8); C bf16 = C.view(-1, N) with `numel` rows; sorted_token_ids int32 [EM],
 * expert_ids int32 [EM / block_m], num_tokens_post_padded int32 [1] = the outputs of moe_align_block_size with
 * block_size = block_m (16 / 32 / 64 / 128); topk_weights flat [numel] (bf16 or fp32), applied when mul_routed_weight. */
int64_t chitu_b200_moe_grouped_gemm_workspace_bytes(int EM, int N, int K);
int chitu_b200_moe_grouped_gemm(const void* A, const void* B, void* C, const float* B_scale, const void* topk_weights,
                                int topk_w_dtype, const int32_t* sorted_token_ids, const int32_t* expert_ids,
                                const int32_t* num_tokens_post_padded, int EM, int numel, int mul_routed_weight, int top_k,
                                int block_m, int E, int N, int K, int wmode, void* workspace, int64_t workspace_bytes,
                                void* stream);

/* Sampling of the decode step (executor.py:104-110 + utils.py:62-81): softmax(logits / temperature), keep the entries
 * whose exclusive cumulative mass (descending order) is <= top_p and whose rank is < top_k, draw from the renormalised
 * kept set.  No sort: the kept set's probability threshold is found by a radix histogram; the draw is the inverse CDF
 * in vocabulary order at the caller's uniform u in [0,1) (same distribution as torch.multinomial; its RNG stream cannot
 * be reproduced).  logits [B, V] bf16 / fp16 / fp32 with row stride; top_ks int32 (<= 0 = off); out_kept / out_mass may
 * be NULL (size and mass of the kept set, diagnostics). */
int chitu_b200_sample_top_k_top_p(const void* logits, int64_t row_stride, int B, int V, int dtype,
                                  const float* temperatures, const int32_t* top_ks, const float* top_ps,
                                  const float* uniforms, int64_t* out_tokens, int32_t* out_kept, float* out_mass,
                                  void* stream);

/* ---- dev tool: in-graph kernel timeline (see csrc/common.cuh) ------------------------------------------------ */
int chitu_b200_debug_timeline(void* buf /* uint64 [2 + capacity] on the device, or NULL to disarm */);
const char* chitu_b200_debug_timeline_names(void);

/* ---- device-side decode-step preparation (SURVEY §8f n2 / §8a a1) ------------------------------------------
 * chitu_b200_decode_prepare = PagedKVCacheManager.prepare_cache_decode + prepare_block_table_for_decode
 * (cache_manager.py:148-158, 196-209) [+ finalize_cache_single_decode :211-215 of the previous step when advance != 0]
 * on device state: seq_lens_excl int32[B] (updated in place when advance), seq_lens_incl int32[B] (may be NULL),
 * block_table int32[B, bt_stride], free_pages int32[..] + free_count int32[1] (a stack of free page ids),
 * status int32[1] (0 ok, 1 = out of free pages — the reference raises "No more free blocks." —, 2 = row full). */
int chitu_b200_decode_prepare(int32_t* seq_lens_excl, int32_t* seq_lens_incl, int32_t* block_table, int bt_stride,
                              int32_t* free_pages, int32_t* free_count, int32_t* status, int B, int page_size,
                              int advance, void* stream);
/* AttnBackend.prepare_metadata_for_decode (attn_backend.py:515-534, FlashMLA get_mla_metadata): length-aware
 * split-KV plan for this step's batch, written into the last 256 bytes of the attention workspace and consumed by
 * chitu_b200_mla_decode when the same workspace / workspace_bytes are passed.  No host synchronisation. */
int chitu_b200_attn_plan(const int32_t* seqlens_incl, int B, int heads, int page_size, int max_seqlen_hint,
                         void* workspace, int64_t workspace_bytes, void* stream);
/* grid.x (upper bound of KV splits per request) the wgmma MLA kernel uses for these arguments */
int chitu_b200_mla_num_splits(int B, int H, int max_seqlen_hint, int64_t workspace_bytes);

/* MLA weight absorption = the two torch.einsum around the attention call
 * (AttentionDeepSeekV3._run_linear model_deepseek_v3.py:529-531 "shd,hdc->shc" and
 * decode_forward_paged :697 "bshc,hdc->bshd").  wkv_b: bf16 [H, dn+dv, C] (dequantised,
 * ops.py:356-392); q_nope: [B,H,dn] with element strides q_sb / q_sh (a view of q[B,H,dn+R]). */
int chitu_b200_mla_absorb_q(const void* q_nope, int64_t q_sb, int64_t q_sh, const void* wkv_b, void* out,
                            int B, int H, int dn, int dv, int C, void* stream);
int chitu_b200_mla_absorb_o(const void* x, const void* wkv_b, void* out, int B, int H, int dn, int dv, int C,
                            void* stream);
/* absorb_o + act_quant_deepseek_v3 of the result (the input of the `wo` linear): out (bf16, may be NULL),
 * q_out fp8 [B, H*dv], q_scales [B, H*dv/128]. dv must be 128 (one quantisation group per head). */
int chitu_b200_mla_absorb_o_quant(const void* x, const void* wkv_b, void* out, void* q_out, float* q_scales,
                                  int B, int H, int dn, int dv, int C, void* stream);
/* Same, but the latent input is the split-KV partials that chitu_b200_mla_decode(out = NULL) left in `workspace`
 * (the LSE merge of triton_decode_attention.py:185-232 happens while staging: one launch instead of merge +
 * absorb).  B, H, max_seqlen_hint, workspace(_bytes) must be those passed to chitu_b200_mla_decode.
 * x_out (may be NULL): the merged latent attention output [B,H,C] bf16. */
int chitu_b200_mla_absorb_o_merge_quant(const void* workspace, int64_t workspace_bytes, int max_seqlen_hint,
                                        const void* wkv_b, void* x_out, void* out, void* q_out, float* q_scales,
                                        int B, int H, int dn, int dv, int C, void* stream);

/* Everything between the wq_b GEMM and the attention call of AttentionDeepSeekV3.decode_forward_paged in one
 * launch: rotary (ops.py:311-326) on q_pe / k_pe, kv_norm (models/model.py:50-78), the cat that builds the
 * appended row (model_deepseek_v3.py:684-686) and the W_UK absorption (:529-531).
 * q:[B,H,dn+R]; kv_in: rows [C kv | R k_pe] with row stride kv_sb (a view of the wqkv_a output);
 * outputs q_abs [B,H,C], q_pe [B,H,R], new_kv [B,C+R]. bf16. */
int chitu_b200_mla_prep(const void* q, const void* kv_in, int64_t kv_sb, const void* kv_norm_w,
                        const float* cos, const float* sin, const void* wkv_b, void* q_abs, void* q_pe,
                        void* new_kv, int B, int H, int dn, int dv, int C, int R, float eps, void* stream);

/* ---- fused MoE experts --------------------------------------------------------------------- */
int64_t chitu_b200_moe_workspace_bytes(int T, int topk, int E, int N1, int K1);
/* fused_experts (fused_moe.py:1060-1307; caller model_deepseek_v3.py:995-1009):
 * out[t,:] = sum_j topk_w[t,j] * W2[e_tj] · silu_mul(W1[e_tj] · x[t,:]).
 * wmode: 0 = bf16 weights, 1 = fp8 block-scaled w8a8 (per_token_group_quant_fp8 on both GEMM
 * inputs, fused_moe.py:277-281), 2 = soft-fp8 (fp8 weights -> bf16, bf16 activations).
 * x:[T,K1] bf16;  w1:[E,N1,K1];  w2:[E,K1,N1/2];  w1_s:[E,N1/128,K1/128]; w2_s:[E,K1/128,N1/2/128]
 * topk_w:[T,topk] bf16|f32, topk_ids:[T,topk] int32|int64. out:[T,K1] bf16 (may alias x). */
int chitu_b200_fused_experts(const void* x, const void* w1, const void* w2, const float* w1_s,
                             const float* w2_s, const void* topk_w, int topk_w_dtype,
                             const void* topk_ids, int ids_dtype, int T, int topk, int E, int N1,
                             int K1, int wmode, void* out,
                             const void* residual /* [T,K1] bf16 added to the rounded result, or NULL */,
                             void* workspace, int64_t workspace_bytes, void* stream);
/* fused_experts whose plan chitu_b200_moe_gate_plan already wrote into `workspace` (same T, topk, E, N1, K1). */
int chitu_b200_fused_experts_planned(const void* x, const void* w1, const void* w2, const float* w1_s,
                             const float* w2_s, const void* topk_w, int topk_w_dtype,
                             const void* topk_ids, int ids_dtype, int T, int topk, int E, int N1,
                             int K1, int wmode, void* out,
                             const void* residual /* [T,K1] bf16 added to the rounded result, or NULL */,
                             void* workspace, int64_t workspace_bytes, void* stream);

/* ---- tensor-parallel collective fused with what follows it ------------------------------------------ */
/* Replaces `all_reduce` of RowParallelLinear.forward (tensor_parallel.py:157-169) / MoEDeepSeekV3
 * (model_deepseek_v3.py:1011) + the residual add + the next RMSNorm (+ act_quant) by ONE kernel that pulls the
 * partial rows of all ranks over NVLink peer memory (one-shot all-reduce, fixed rank order => deterministic).
 * Setup (host pointers here): comm_create allocates this rank's symmetric buffer (2 slots of slot_bytes) and
 * returns 128 bytes of CUDA IPC handles; exchange them between the ranks (torch.distributed all_gather), then
 * comm_connect maps the peers.  One process per GPU, single node, world <= 8. */
int chitu_b200_comm_create(int rank, int world, int64_t slot_bytes, void** handle_out, uint8_t* ipc_out);
int chitu_b200_comm_connect(void* handle, const uint8_t* all_ipc /* world x 128 bytes, rank order */);
int chitu_b200_comm_destroy(void* handle);
/* 0 = healthy, 1 + r = the wait for peer r exceeded CHITU_B200_COMM_TIMEOUT_S (default 600, 0 = never) */
int chitu_b200_comm_status(void* handle);

/* ---- all-reduce started from the producing kernel's epilogue ("push" mode; SURVEY §5.8) -----------------------------
 * The row-parallel linear (RowParallelLinear.forward, tensor_parallel.py:157-169) / the MoE block (model_deepseek_v3.py:
 * 1011) of a tensor-parallel layer does not write its partial result locally: the epilogue stores every bf16 output tile
 * into the push area of EVERY rank over NVLink as 8-byte words {2 x bf16, epoch} — the word is its own arrival flag
 * (aligned 8-byte stores land whole), so the producer needs no fence and no counter.  chitu_b200_allreduce_consume polls the
 * words of its rows until every source's epoch matches and then reduces from LOCAL memory (rank order, fp32,
 * deterministic), adds the residual, and applies RMSNorm (+ act_quant) — the same outputs as
 * chitu_b200_allreduce_residual_rmsnorm.  N (K1 for the experts) must be even; M * N * 2 <= the slot_bytes of comm_create. */
int chitu_b200_fp8_gemm_ar(const void* a, const float* a_s, const void* b, const float* b_s, int M, int N, int K, void* comm,
                           void* workspace, int64_t workspace_bytes, void* stream);
int chitu_b200_linear_bf16_ar(const void* x, const void* w, int M, int N, int K, void* comm, void* workspace,
                              int64_t workspace_bytes, void* stream);
int chitu_b200_fused_experts_ar(const void* x, const void* w1, const void* w2, const float* w1_s, const float* w2_s,
                                const void* topk_w, int topk_w_dtype, const void* topk_ids, int ids_dtype, int T, int topk,
                                int E, int N1, int K1, int wmode, void* comm, void* workspace, int64_t workspace_bytes,
                                int planned /* 1: plan written by chitu_b200_moe_gate_plan */, void* stream);
int chitu_b200_allreduce_consume(void* comm, const void* residual, void* h_out, const void* norm_w, void* y,
                                 void* q, float* q_scales, int rows, int dim, float eps, void* stream);
/* h = bf16(sum_r partial_r) (+ residual);  optional outputs of RMSNorm(h)*norm_w: y (bf16) and / or q (fp8,
 * 128-group scales).  partial/residual/h_out: [rows, dim] bf16 (h_out may alias partial); rows <= 256. */
int chitu_b200_allreduce_residual_rmsnorm(void* handle, const void* partial, const void* residual,
                                          void* h_out, const void* norm_w, void* y, void* q, float* q_scales,
                                          int rows, int dim, float eps, void* stream);

/* ---- small decode-engine helpers (adjacent rows §8f; used by bench/engine) -------------------- */
/* out[t,:] = table[ids[t],:]  (VocabParallelEmbedding local lookup, tensor_parallel.py:199-208;
 * rows outside [vocab_start, vocab_start+rows) produce zeros). */
int chitu_b200_embedding(const int64_t* ids, const void* table, void* out, int T, int dim,
                         int64_t vocab_start, int64_t rows, int dtype, void* stream);
/* y = a + b (residual add), bf16/fp16. */
int chitu_b200_add(const void* a, const void* b, void* y, int64_t n, int dtype, void* stream);
/* argmax over the last dim of f32|bf16 logits [T, V] -> int64 ids (greedy sampling,
 * executor.py:82-112 argmax branch). */
int chitu_b200_argmax(const void* logits, int64_t* out, int T, int64_t V, int dtype, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CHITU_B200_H_ */
