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
/* The same append into an fp8 (e4m3fn) paged cache of 64-token pages: this_kv [batch, n] in the io dtype (bf16 | fp16),
 * each element stored as e4m3(clamp(x, -448, 448)), nearest even, NaN kept (the store rule of
 * chitu_b200_gqa_paged_attn_fp8kv and chitu_b200_mla_attn_fp8kv).  n % 8 == 0, this_kv 16-byte aligned. */
int chitu_b200_append_paged_kv_e4m3(void* kv_cache, const int32_t* page_table, const void* this_kv,
                                    const int32_t* old_seq_lens, int batch, int pages_per_sample, int n, int dtype,
                                    void* stream);
/* The prompt's k / v (GQA: cache0 = k, cache1 = v) or latent rows (MLA: cache1 = src1 = NULL) into the KV cache after
 * the prefill attention: the page scatter of PagedKVCacheManager.finalize_cache_bylayer_prefill
 * (cache_manager.py:93-142) and the prompt write of KVCacheManager, for every request of a batch in one launch.
 * src0 / src1: [total_rows, n] in src_dtype (bf16 | fp16), row strides src0_st / src1_st in elements.
 * cu_seqlens: int32 [B + 1] on the device, nondecreasing; cache_seqlens: int32 [B] (tokens already cached) or NULL (0).
 * Row t < cu_seqlens[b + 1] - cu_seqlens[b] of request b, source row cu_seqlens[b] + t, goes to position
 * p = cache_seqlens[b] + t of request b:
 *  - paged (block_table != NULL, int32 [B, bt_stride]): page block_table[b, p / page_size], slot p % page_size (true page
 *    indexing, any page_size >= 1); only block_table[b, 0 .. ceil((cache_seqlens[b] + len_b) / page_size) - 1] is read;
 *  - contiguous (block_table == NULL): element b * cache_sb + p * n, with cache_sb a multiple of n and at least
 *    cache_rows * n; rows with p >= cache_rows are not written (the capacity rule of chitu_b200_gqa_contiguous_attn).
 * Source rows outside [cu_seqlens[0], cu_seqlens[B]) and from total_rows on are not read; nothing outside the written
 * slots is touched.  Store: cache_dtype == src_dtype copies the bits (16-byte copies when every address and stride
 * allows them); cache_dtype CB_FP8_E4M3 (paged only) stores e4m3(clamp(x, -448, 448)), nearest even, NaN kept, the
 * rule of the e4m3 attention entries, and needs n % 8 == 0, 16-byte aligned sources, strides that are multiples of 8
 * and 8-byte aligned caches.  One launch whose grid depends on total_rows alone (no host synchronisation, capturable in
 * a CUDA graph that replays new lengths and positions), deterministic.  Anything else returns a negative status before
 * any launch; B == 0 or total_rows == 0 launches nothing. */
int chitu_b200_scatter_kv(void* cache0, void* cache1, const void* src0, int64_t src0_st, const void* src1,
                          int64_t src1_st, const int32_t* cu_seqlens, const int32_t* cache_seqlens,
                          const int32_t* block_table, int bt_stride, int page_size, int64_t cache_sb, int cache_rows,
                          int B, int total_rows, int n, int src_dtype, int cache_dtype, void* stream);

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

/* ---- rotary --------------------------------------------------------------------------- */
/* Replaces triton_kernels.py:101-190 (rotary_type="llama", interleaved pairs; cos/sin f32
 * [bs, rot/2]) — ops.py:178-237.  q:[bs,hq,rot] k:[bs,hk,rot], strides in elements. */
int chitu_b200_rotary_interleaved(const void* q, const void* k, void* out_q, void* out_k,
                                  const float* cos, const float* sin, int bs, int hq, int hk,
                                  int rot_dim, int64_t q_sb, int64_t q_sh, int64_t k_sb, int64_t k_sh,
                                  int dtype, void* stream);
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
 * the fp8 payload q [rows, dim] + scales [rows, dim/128] (both NULL to skip).  bf16, dim % 128 == 0; x / w / y 8-byte
 * aligned, q 4-byte aligned. */
int chitu_b200_rmsnorm_quant_fp8(const void* x, const void* w, void* y, void* q, float* q_scales, int rows,
                                 int dim, int64_t x_stride, int64_t y_stride, float eps, void* stream);
/* Fused SiluAndMul + act_quant_deepseek_v3: x [rows, 2F] bf16 -> q fp8 [rows, F], scales [rows, F/128].  x 8-byte
 * aligned, q 4-byte aligned. */
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
/* Per-token e4m3 quantisation of bf16 rows, the rule of vLLM's QuantFP8(GroupShape.PER_TOKEN).forward_native:
 * dynamic (scale == NULL): s[r] = max(min(max_k |x[r,k]|, *scale_ub) / 448, 1 / (448*512)) in fp32, the upper bound
 * only when scale_ub != NULL; static: s[r] = *scale for every row.  q = e4m3_rn(clamp(fp32(x) * rcp_rn(s[r]), +-448)).
 * x [rows, K] bf16, q [rows, K] e4m3, q_scales [rows] fp32; scale and scale_ub are fp32 device scalars.  K % 16 == 0,
 * x and q 16-byte aligned; a static scale with an upper bound is refused. */
int chitu_b200_quant_fp8_rowwise(const void* x, void* q, float* q_scales, int64_t rows, int K, const float* scale,
                                 const float* scale_ub, void* stream);
/* RMSNorm followed by the dynamic per-token quantisation above, in one launch and bit for bit chitu_b200_rmsnorm and
 * chitu_b200_quant_fp8_rowwise in sequence: q [rows, dim] e4m3 and q_scales [rows] from the bf16-rounded norm output,
 * which is also written to y unless y is NULL.  bf16, dim <= 8192. */
int chitu_b200_rmsnorm_quant_fp8_rowwise(const void* x, const void* w, void* y, void* q, float* q_scales, int rows,
                                         int dim, float eps, void* stream);
/* weight_dequant_deepseek_v3 / weight_dequant_soft_fp8_deepseek_v3 (ops.py:356-449):
 * y[b,m,n] = fp8(x[b,m,n]) * s[b, m/128, n/128]  -> bf16.  soft != 0 reproduces the
 * bit-trick path ((x&0x80)<<24 | (x&0x7f)<<20) * (s * 2^120).  The kernel does not let the next kernel of the stream
 * start before it has finished, so a linear launched right after it may read y as its weight. */
int chitu_b200_weight_dequant_fp8(const void* x, const float* s, void* y, int B, int M, int N,
                                  int block, int soft, void* stream);

/* ---- linears (weight-streaming skinny GEMMs; weights are [N,K] row-major = nn.Linear) --- */
/* Workspace for split-K partials + ticket counters: chitu_b200_linear_workspace_bytes(M_max, N_max).
 * It must be zero-filled ONCE before its first use; every call leaves the counters at zero again. */
int64_t chitu_b200_linear_workspace_bytes(int M, int N);
/* impl: 0 = auto, 1 = SIMT weight-streaming GEMV, 2 = wgmma/TMA swap-AB GEMM.
 * Weight contract: the wgmma GEMM starts streaming its weights while the previous kernel of the stream is still running
 * (before griddepcontrol.wait).  A weight must therefore be written by host copies, torch kernels or
 * chitu_b200_weight_dequant_fp8, never by a kernel that triggers its dependents early (griddepcontrol.launch_dependents)
 * directly before the linear.
 * KV contract: the cache writers (chitu_b200_scatter_kv, chitu_b200_append_paged_kv[_e4m3], the seqlen_q > 1 attention
 * entries and the in-place append of the decode entries) trigger their dependents early and write after their own
 * wait, so the attention kernels load no KV cache row before griddepcontrol.wait; any writer may directly precede any
 * reader of the same cache.  The decode kernels do read cache_seqlens / seqlens_excl, the block table and the MLA split
 * plan before that wait: those must come from host copies, torch kernels, chitu_b200_decode_prepare or
 * chitu_b200_attn_plan, none of which triggers its dependents early. */
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

/* W4A16 with groups of 128 along K (GPTQ / AWQ checkpoints after chitu_b200.quantize.W4A16Linear's repack), for the
 * weight W[N, K], K % 128 == 0:
 *   qweight uint8 [N, K/2] row-major: element k of row n in byte k/2, low nibble for even k, high nibble for odd k;
 *   scales  [N, K/128] in the io dtype;  zeros uint8 [N, K/128], 0..15 (a symmetric checkpoint has zeros = 8).
 * w[n,k] = io((q[n,k] - zeros[n,k/128]) * scales[n,k/128]) with one rounding (q - z is exact), and y = x w^T with fp32
 * accumulation, io out; residual [M,N] (or NULL) is added after that rounding, as chitu_b200_linear_bf16 does.
 * dtype CB_BF16 | CB_F16 for x, scales, residual and y.  wgmma path only: where it cannot run (shape or workspace) the
 * entries return -2 and launch nothing.  Refused before any launch, under the entry's name: a NULL operand, a base
 * (residual included) that is not 16-byte aligned, K % 128 != 0, another dtype, an odd N for the pairs entry.  M == 0
 * launches nothing.  qweight, scales and zeros are weights under the weight contract above. */
int chitu_b200_w4a16_gemm(const void* x, const void* qweight, const void* scales, const uint8_t* zeros,
                          const void* residual, void* y, int M, int N, int K, int dtype, void* workspace,
                          int64_t workspace_bytes, void* stream);
/* The gate_up linear + SiluAndMul of chitu_b200_linear_bf16_silu_pairs on W4A16 weights: rows 2i / 2i+1 of the [N, K]
 * weight (with their scales and zeros) are gate_i / up_i; y [M, N/2] in the io dtype with the roundings of the two
 * separate ops (g, u -> io, silu(g) -> io, product -> io). */
int chitu_b200_w4a16_gemm_silu_pairs(const void* x, const void* qweight, const void* scales, const uint8_t* zeros,
                                     void* y, int M, int N, int K, int dtype, void* workspace, int64_t workspace_bytes,
                                     void* stream);

/* FP8 W8A8 with rowwise scales (vLLM Fp8LinearMethod for compressed-tensors FP8 / FP8_DYNAMIC and fbgemm rowwise
 * checkpoints; torch._scaled_mm(a, b.T, scale_a [M,1], scale_b [1,N], bias, out_dtype=bf16)):
 *   y[m,n] = bf16((sum_k a[m,k] b[n,k]) * a_s[m] * b_s[n] (+ bias[n])), residual [M,N] (or NULL) added after that
 *   rounding; a [M,K] and b [N,K] e4m3, a_s [M] and b_s [N] fp32, bias [N] bf16 or NULL.
 * Every 128 K-elements are summed by the tensor cores and then added into an fp32 accumulator; the scales are applied
 * once, (acc * a_s) * b_s.  wgmma path only, sharing chitu_b200_linear_workspace_bytes: where it cannot run (shape or
 * workspace) the entries return -2 and launch nothing.  Refused before any launch, under the entry's name: a NULL
 * operand, a base that is not 16-byte aligned, K % 16 != 0, an odd N for the pairs entry.  M == 0 launches nothing.
 * b and b_s are weights under the weight contract above; a_s is read after griddepcontrol.wait, so the quantiser that
 * writes a and a_s may directly precede the GEMM. */
int chitu_b200_fp8_rowwise_gemm(const void* a, const float* a_s, const void* b, const float* b_s, const void* bias,
                                const void* residual, void* y, int M, int N, int K, void* workspace,
                                int64_t workspace_bytes, void* stream);
/* The gate_up linear + SiluAndMul of chitu_b200_linear_bf16_silu_pairs on rowwise fp8 weights: rows 2i / 2i+1 of b
 * (each with its own b_s) are gate_i / up_i; y [M, N/2] bf16 with the roundings of the two separate ops. */
int chitu_b200_fp8_rowwise_gemm_silu_pairs(const void* a, const float* a_s, const void* b, const float* b_s, void* y,
                                           int M, int N, int K, void* workspace, int64_t workspace_bytes, void* stream);

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
/* AttnBackend.attn_with_kvcache with block_table and seqlen_q = sq >= 1 (attn_backend.py:92-164, FlashAttn impl
 * :208-243, flash_attn_with_kvcache semantics): chunked prefill, prefill on a cached prefix, speculative verification.
 * q [B, sq, Hq, D] contiguous; k_cache / v_cache [num_blocks, page_size, Hkv, D] contiguous; k_new / v_new
 * [B, sq, Hkv, D] with dense heads and batch / token strides *_sb / *_st in elements (views into a fused-qkv GEMM
 * output), or both NULL.  With k_new: token i of request b is written to position cache_seqlens[b] + i (true page
 * indexing) before the attention, which then runs over Lk = cache_seqlens[b] + sq keys; without, Lk = cache_seqlens[b].
 * cache_seqlens is not modified.  causal != 0: query i sees key j iff j <= i + Lk - sq; a row that sees no key is 0.
 * fp32 scores and softmax, P rounded to the io dtype before P.V.  out [B, sq, Hq, D] contiguous.
 * Only block_table[b, 0 .. ceil(Lk / page_size) - 1] is read; cache slots past Lk may hold anything (NaN included).
 * Splits over keys when the GPU would otherwise be idle (count from B, Hkv, sq and max_seqlen_hint, shrunk to the
 * workspace; NULL workspace: no split) -> no host synchronisation, capturable in a CUDA graph, deterministic.
 * Built for D == 128, page_size % 64 == 0, Hq / Hkv in {1, 2, 4, 8}, bf16 | fp16; 16-byte aligned bases and strides
 * that are multiples of 8 elements.  Anything else returns a negative status. */
int chitu_b200_gqa_paged_prefill(const void* q, void* k_cache, void* v_cache, const void* k_new, const void* v_new,
                                 int64_t k_new_sb, int64_t k_new_st, int64_t v_new_sb, int64_t v_new_st,
                                 const int32_t* cache_seqlens, const int32_t* block_table, int bt_stride, int B, int sq,
                                 int Hq, int Hkv, int D, int page_size, int num_blocks, int max_seqlen_hint, int causal,
                                 float softmax_scale, void* out, void* workspace, int64_t workspace_bytes, int dtype,
                                 void* stream);
/* AttnBackend.attn_with_kvcache WITHOUT block_table (attn_backend.py:92-164; FlashAttn impl :208-243 passes no block
 * table, RefAttnBackend :458-501 implements only this form), seqlen_q = sq >= 1: GQA attention over the non-paged
 * per-request cache of KVCacheManager (cache_manager.py:228-370).  k_cache / v_cache [Bc, cache_rows, Hkv, D] with
 * Bc >= B, the same shape and strides, dense last two dims and a batch stride cache_sb in elements (a multiple of
 * Hkv * D and of 8, at least cache_rows * Hkv * D: a [:B, :S] view of a larger buffer is accepted); request b uses
 * cache row b.  q [B, sq, Hq, D] contiguous; k_new / v_new [B, sq, Hkv, D] with dense heads and batch / token strides
 * *_sb / *_st in elements, or both NULL.  With k_new: token i of request b is written to position cache_seqlens[b] + i
 * before the attention, which then runs over Lk = cache_seqlens[b] + sq keys; without, Lk = cache_seqlens[b].
 * cache_seqlens is not modified.  causal != 0: query i sees key j iff j <= i + Lk - sq; a row that sees no key is 0.
 * fp32 scores and softmax, P rounded to the io dtype before P.V.  out [B, sq, Hq, D] contiguous.
 * Capacity: a new row at a position >= cache_rows is not written and no key >= cache_rows is read (the output of such
 * a request is unspecified); nothing outside the request's rows of the caches is touched.
 * sq == 1 runs the decode kernels (tensor cores for D == 128), sq > 1 the multi-token kernel; splits over keys as in
 * the paged entries, from B, Hkv, sq and max_seqlen_hint (<= 0: cache_rows), shrunk to the workspace (NULL: no split)
 * -> no host synchronisation, capturable in a CUDA graph, deterministic.
 * Built for Hq / Hkv in {1, 2, 4, 8}, bf16 | fp16, D in {64, 128} for sq == 1 and D == 128 for sq > 1, any
 * cache_rows >= 1; 16-byte aligned bases; k / v strides multiples of 4 elements (sq == 1) or 8 (sq > 1).  Anything
 * else returns a negative status.  B == 0 launches nothing. */
int chitu_b200_gqa_contiguous_attn(const void* q, void* k_cache, void* v_cache, int64_t cache_sb, int cache_rows,
                                   const void* k_new, const void* v_new, int64_t k_new_sb, int64_t k_new_st,
                                   int64_t v_new_sb, int64_t v_new_st, const int32_t* cache_seqlens, int B, int sq,
                                   int Hq, int Hkv, int D, int max_seqlen_hint, int causal, float softmax_scale,
                                   void* out, void* workspace, int64_t workspace_bytes, int dtype, void* stream);

/* AttnBackend.attn_with_kvcache with block_table over an fp8 (e4m3fn) paged cache, seqlen_q = sq >= 1: the
 * arguments and semantics of chitu_b200_gqa_paged_prefill with k_cache / v_cache [num_blocks, page_size, Hkv, D] of
 * e4m3 bytes and q / k_new / v_new / out in the io dtype (bf16 | fp16), with these differences:
 *  - Store: a new k / v element x is written as e4m3(clamp(x, -448, 448)), rounded to nearest even; NaN stays NaN
 *    (torch: x.float().clamp(-448, 448).to(float8_e4m3fn)).  No scale (a per-tensor scale of 1).
 *  - Read: a cache element is decoded to the io dtype exactly; the arithmetic is then the io-dtype cache's (fp32 scores
 *    and softmax, P rounded to the io dtype before P.V, bottom-right causal mask, 0 for a row that sees no key).  The
 *    rows appended by the call are attended in their stored form, so sq = n agrees with n successive decodes.
 *  - q [B, sq, Hq, D] with batch stride q_sb elements: any multiple of 8 >= Hq * D for sq == 1 (a view of a fused qkv
 *    GEMM output), sq * Hq * D for sq > 1.
 *  - rope_cos / rope_sin (fp32 [B, D / 2], both or neither, sq == 1 only): the rotary of
 *    chitu_b200_gqa_paged_decode_rope on q and the new k, which is rotated and rounded to the io dtype before it is
 *    stored as above.
 *  - k / v strides: multiples of 8 elements (the token strides are unused for sq == 1).
 * sq == 1 runs the tensor-core decode kernel, sq > 1 the multi-token kernel after an append; the splits and the
 * workspace are those of the io-dtype entries -> no host synchronisation, capturable in a CUDA graph, deterministic.
 * Built for D == 128, Hq / Hkv in {1, 2, 4, 8}, page_size a power of two and a multiple of 64, bf16 | fp16 io,
 * 16-byte aligned bases.  Anything else returns a negative status before any launch.  B == 0 launches nothing. */
int chitu_b200_gqa_paged_attn_fp8kv(const void* q, int64_t q_sb, void* k_cache, void* v_cache, const void* k_new,
                                    const void* v_new, int64_t k_new_sb, int64_t k_new_st, int64_t v_new_sb,
                                    int64_t v_new_st, const float* rope_cos, const float* rope_sin,
                                    const int32_t* cache_seqlens, const int32_t* block_table, int bt_stride, int B,
                                    int sq, int Hq, int Hkv, int D, int page_size, int num_blocks, int max_seqlen_hint,
                                    int causal, float softmax_scale, void* out, void* workspace,
                                    int64_t workspace_bytes, int dtype, void* stream);

/* *.mla_attn_with_kvcache (attn_backend.py:536-572 / 660-684 / 707-774) = append
 * (ops.py:50-91) + mla_decode (triton_decode_attention.py:259-290) in one call.
 * q_nope:[B,H,C] q_pe:[B,H,R] kv_cache:[num_blocks,64,C+R] new_kv:[B,C+R] (may be NULL)
 * seqlens_excl:[B] (length before this token) ; attention runs over seqlens_excl+1 keys when
 * new_kv != NULL else over seqlens_excl keys.  out:[B,H,C] (latent space). bf16.
 * page_size must be 64; num_blocks = kv_cache.shape[0] (bounds the TMA tensor map that stages whole pages).
 * out == NULL: the split merge is deferred to chitu_b200_mla_absorb_o_merge_quant, and the workspace must hold the
 * partials of one split (chitu_b200_attn_workspace_bytes(B, H, C, 1)).  A workspace holds at least the 256-byte plan. */
int chitu_b200_mla_decode(const void* q_nope, const void* q_pe, void* kv_cache, const void* new_kv,
                          const int32_t* seqlens_excl, const int32_t* block_table, int bt_stride,
                          int B, int H, int C, int R, int page_size, int num_blocks, int max_seqlen_hint,
                          float softmax_scale, void* out, void* workspace, int64_t workspace_bytes,
                          void* stream);

/* FlashAttnBackend.attn_varlen_func (attn_backend.py:193-206) for the absorbed-MLA prefill of DeepSeek
 * (model_deepseek_v3.py:588-602), with flash_attn_varlen_func semantics: q [total_q, H, 576] contiguous,
 * k [total_k, 576] (row stride k_sb elements), v [total_k, 512] (row stride v_sb), one KV head shared by the H query
 * heads; out [total_q, H, 512] contiguous.  bf16; fp32 scores and softmax, P rounded to bf16 before P.V.
 * cu_seqlens_q / cu_seqlens_k: int32 [B + 1] on the device (zero-length sequences allowed); max_seqlen_q (host) sizes
 * the grid.  causal != 0: bottom-right aligned mask (query i sees keys j <= i + Lk - Lq); a row that sees no key is 0.
 * No host synchronisation, no workspace (capturable in a CUDA graph); deterministic (no split over keys).
 * Bases 16-byte aligned, k_sb / v_sb multiples of 8; total_q * H must fit int32. */
int chitu_b200_mla_prefill(const void* q, const void* k, int64_t k_sb, const void* v, int64_t v_sb,
                           const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k, int B, int H,
                           int total_q, int total_k, int max_seqlen_q, int causal, float softmax_scale,
                           void* out, void* stream);

/* *.mla_attn_with_kvcache with sq >= 1 query tokens per request (FlashMLA's s_q > 1): multi-token-prediction
 * verification and chunked prefill on the paged latent cache of absorbed MLA.
 * q_nope [B, sq, H, C] and q_pe [B, sq, H, R] contiguous; kv_cache [num_blocks, 64, C + R] contiguous; new_kv
 * [B, sq, C + R] contiguous, or NULL.  With new_kv: token i of request b is written to position seqlens_excl[b] + i
 * (pages indexed with a literal 64, as the decode append) before the attention, which then runs over
 * Lk = seqlens_excl[b] + sq keys; without, Lk = seqlens_excl[b].  seqlens_excl is not modified.
 * causal != 0: query i sees key j iff j <= i + Lk - sq; a row that sees no key is 0.  The decode arithmetic:
 * scale * (q_nope.k_c + q_pe.k_pe) in fp32, softmax in fp32, P rounded to bf16 before P.V, V = the first C columns of the
 * same cache rows.  out [B, sq, H, C] bf16 contiguous, never NULL (no deferred merge).
 * Only block_table[b, 0 .. ceil(Lk / 64) - 1] is read; cache slots past Lk may hold anything (NaN included).
 * Splits over keys when B x ceil(sq * H / 64) CTAs cannot fill the GPU (count from max_seqlen_hint, shrunk to the
 * workspace; NULL workspace: no split) -> no host synchronisation, capturable in a CUDA graph, deterministic.
 * Built for C = 512, R = 64, page_size = 64; bases 16-byte aligned; B * sq * H and num_blocks * 64 must fit int32.
 * Anything else returns a negative status. */
int chitu_b200_mla_paged_prefill(const void* q_nope, const void* q_pe, void* kv_cache, const void* new_kv,
                                 const int32_t* seqlens_excl, const int32_t* block_table, int bt_stride, int B, int sq,
                                 int H, int C, int R, int page_size, int num_blocks, int max_seqlen_hint, int causal,
                                 float softmax_scale, void* out, void* workspace, int64_t workspace_bytes,
                                 void* stream);

/* *.mla_attn_with_kvcache over an fp8 (e4m3fn) paged latent cache, seqlen_q = sq >= 1: the arguments and semantics
 * of chitu_b200_mla_paged_prefill with kv_cache [num_blocks, 64, C + R] of e4m3 bytes (q_nope, q_pe, new_kv and out
 * stay bf16), with these differences:
 *  - Store: every element x of a new row (latent and rope) is written as e4m3(clamp(x, -448, 448)), rounded to
 *    nearest even; NaN stays NaN (torch: x.float().clamp(-448, 448).to(float8_e4m3fn)).  No scale (a per-tensor scale
 *    of 1).
 *  - Read: a cache element is decoded to bf16 exactly; the arithmetic is then the bf16 cache's (scale * (q_nope.k_c +
 *    q_pe.k_pe) in fp32, softmax in fp32, P rounded to bf16 before P.V with V = the first C columns of the same rows,
 *    bottom-right causal mask, 0 for a row that sees no key).  The rows appended by the call are attended in their
 *    stored form, so sq = n agrees with n successive decodes.
 *  - sq == 1 is the decode of chitu_b200_mla_decode: q_nope [B, 1, H, C] = [B, H, C], new_kv [B, C + R] appended in
 *    the same launch, the device split plan of chitu_b200_attn_plan honoured, `causal` ignored (the one query row sees
 *    every key), and out == NULL defers the merge to chitu_b200_mla_absorb_o_merge_quant (the workspace must then hold
 *    the partials of one split).  sq > 1 appends the new rows first, then runs the multi-token kernel; out != NULL.
 * Splits and workspace as in the bf16 entries -> no host synchronisation, capturable in a CUDA graph, deterministic.
 * Built for C = 512, R = 64, page_size = 64; bases 16-byte aligned.  Anything else returns a negative status before any
 * launch.  B == 0 launches nothing. */
int chitu_b200_mla_attn_fp8kv(const void* q_nope, const void* q_pe, void* kv_cache, const void* new_kv,
                              const int32_t* seqlens_excl, const int32_t* block_table, int bt_stride, int B, int sq,
                              int H, int C, int R, int page_size, int num_blocks, int max_seqlen_hint, int causal,
                              float softmax_scale, void* out, void* workspace, int64_t workspace_bytes, void* stream);

/* invoke_fused_moe_kernel (fused_moe.py:796-891; Triton kernel :62-307) as ONE grouped wgmma GEMM:
 * A bf16 [numel/top_k (GEMM1) or numel (top_k = 1), K]; B stacked expert weights [E, N, K] (bf16 for wmode 0, fp8 +
 * B_scale [E, N/128, K/128] for wmode 1 = fp8_w8a8 — A is quantised per_token_group_quant_fp8 inside, as the reference
 * does at :826 — and wmode 2 = soft_fp8); C bf16 = C.view(-1, N) with `numel` rows; sorted_token_ids int32 [EM],
 * expert_ids int32 [EM / block_m], num_tokens_post_padded int32 [1] = the outputs of moe_align_block_size with
 * block_size = block_m (16 / 32 / 64 / 128); topk_weights flat [numel] (bf16 or fp32), applied when mul_routed_weight.
 * N and K are multiples of 128 for every wmode. */
int64_t chitu_b200_moe_grouped_gemm_workspace_bytes(int EM, int N, int K);
int chitu_b200_moe_grouped_gemm(const void* A, const void* B, void* C, const float* B_scale, const void* topk_weights,
                                int topk_w_dtype, const int32_t* sorted_token_ids, const int32_t* expert_ids,
                                const int32_t* num_tokens_post_padded, int EM, int numel, int mul_routed_weight, int top_k,
                                int block_m, int E, int N, int K, int wmode, void* workspace, int64_t workspace_bytes,
                                void* stream);

/* Sampling of the decode step (executor.py:104-110 + utils.py:62-81): softmax(logits / temperature), keep the entries
 * whose exclusive cumulative mass (descending order) is <= top_p and whose rank is < top_k, draw from the renormalised
 * kept set (an entry of probability 0 is never kept).  No sort: the kept set's probability threshold is found by a radix histogram; the draw is the inverse CDF
 * in vocabulary order at the caller's uniform u in [0,1) (same distribution as torch.multinomial; its RNG stream cannot
 * be reproduced).  logits [B, V] bf16 / fp16 / fp32 with row stride; top_ks int32 (<= 0 = off); out_kept / out_mass may
 * be NULL (size and mass of the kept set, diagnostics). */
int chitu_b200_sample_top_k_top_p(const void* logits, int64_t row_stride, int B, int V, int dtype,
                                  const float* temperatures, const int32_t* top_ks, const float* top_ps,
                                  const float* uniforms, int64_t* out_tokens, int32_t* out_kept, float* out_mass,
                                  void* stream);
/* Greedy acceptance of speculative drafts after a verify step over k + 1 positions per request.  target int64
 * [B, k + 1]: the argmax at each verified position; drafts int64 [B, k]; n_draft int32 [B]: each request's draft length
 * (clamped to 0..k); seq_lens int32 [B], updated in place.  a_b = the number of leading i < n_draft[b] with
 * drafts[b, i] == target[b, i]; request b emits target[b, 0..a_b] into out_tokens int64 [B, k + 1] (the rest of the row
 * is -1), accepted int32 [B] = a_b, next_tokens int64 [B] = target[b, a_b], seq_lens[b] += a_b + 1.
 * One launch, no host synchronisation, capturable.  It writes seq_lens, which the decode kernels read before their
 * griddepcontrol.wait, so it waits for its predecessor and never triggers its dependents early.  Null pointers, B < 0
 * or k < 1 return a negative status before any launch; B == 0 launches nothing. */
int chitu_b200_spec_accept_greedy(const int64_t* target, const int64_t* drafts, const int32_t* n_draft,
                                  int32_t* seq_lens, int64_t* out_tokens, int32_t* accepted, int64_t* next_tokens,
                                  int B, int k, void* stream);
/* Speculative sampling (rejection sampling) of k draft tokens per request after a verify step: the emitted tokens have
 * the distribution of sampling the target one token at a time.  logits [B * (k + 1), V] (row stride in elements; row
 * b * (k + 1) + i is request b's position i), bf16 / fp16 / fp32.  p_i: softmax(l / T) over the kept set of
 * chitu_b200_sample_top_k_top_p with the request's temperatures / top_ks / top_ps [B] (T <= 0: greedy, the rule of
 * chitu_b200_spec_accept_greedy on the first maximal index; top_k <= 0: no top-k).  q_i: fp32 row draft_probs
 * + (b * k + i) * draft_probs_stride, or one-hot at drafts[b, i] when draft_probs is NULL.  Draft i is accepted iff
 * u_accept[b, i] * q_i(d_i) < p_i(d_i) (never outside the kept set); a_b = the leading accepted count (<= n_draft[b],
 * clamped to 0..k).  The drawn token comes from max(p_a - q_a, 0) when a_b < n_draft[b] (from p_a when that has no mass),
 * from p_n otherwise: inverse CDF in vocabulary order at u_draw[b] times the mass.  Outputs as the greedy entry:
 * out_tokens int64 [B, k + 1] (drafts 0..a_b - 1, the drawn token, then -1), accepted int32 [B] = a_b, next_tokens
 * int64 [B] = the drawn token, seq_lens int32 [B] += a_b + 1.  workspace: at least
 * chitu_b200_spec_accept_sampled_workspace_bytes(B, k) bytes.  Two launches, no host synchronisation. */
int64_t chitu_b200_spec_accept_sampled_workspace_bytes(int B, int k);
int chitu_b200_spec_accept_sampled(const void* logits, int64_t row_stride, int V, int dtype, const float* temperatures,
                                   const int32_t* top_ks, const float* top_ps, const int64_t* drafts,
                                   const int32_t* n_draft, const float* draft_probs, int64_t draft_probs_stride,
                                   const float* u_accept, const float* u_draw, int32_t* seq_lens, int64_t* out_tokens,
                                   int32_t* accepted, int64_t* next_tokens, int B, int k, void* workspace,
                                   int64_t workspace_bytes, void* stream);

/* ---- dev tool: in-graph kernel timeline (see csrc/common.cuh) ------------------------------------------------ */
int chitu_b200_debug_timeline(void* buf /* uint64 [2 + capacity] on the device, or NULL to disarm */);
const char* chitu_b200_debug_timeline_names(void);
/* Read-only view of a communicator's push-mode state, for tests that write or inspect the words themselves.
 * *area: this rank's push area on the device, [2 slots][world sources][*source_bytes], *source_bytes = 2 * slot_bytes.
 * Word k of a source's [rows, dim] bf16 partial sits at byte k * 8 and holds
 *   { uint32 (bf16 x[2k] | bf16 x[2k+1] << 16), uint32 epoch }.
 * *calls: the device uint32 counting the reduces this rank has consumed; the next reduce reads slot *calls & 1 and
 * waits for epoch *calls + 1. */
int chitu_b200_debug_comm_push_area(void* handle, void** area, int64_t* source_bytes, uint32_t** calls);

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

/* MLA output absorption = the torch.einsum after the attention call (AttentionDeepSeekV3.decode_forward_paged
 * model_deepseek_v3.py:697 "bshc,hdc->bshd"; the q side, :529-531, is part of chitu_b200_mla_prep).  wkv_b: bf16
 * [H, dn+dv, C] (dequantised, ops.py:356-392); x: [B,H,C] bf16.  absorb_o + act_quant_deepseek_v3 of the result (the
 * input of the `wo` linear): out (bf16, may be NULL), q_out fp8 [B, H*dv], q_scales [B, H*dv/128]. dv must be 128
 * (one quantisation group per head).  x / wkv_b 16-byte aligned, out 8-byte, q_out 4-byte. */
int chitu_b200_mla_absorb_o_quant(const void* x, const void* wkv_b, void* out, void* q_out, float* q_scales,
                                  int B, int H, int dn, int dv, int C, void* stream);
/* Same, but the latent input is the split-KV partials that chitu_b200_mla_decode(out = NULL) left in `workspace`
 * (the LSE merge of triton_decode_attention.py:185-232 happens while staging: one launch instead of merge +
 * absorb).  B, H, max_seqlen_hint, workspace(_bytes) must be those passed to chitu_b200_mla_decode; a workspace too
 * small for the partials of the recomputed split count is refused.
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
/* fused_experts over 4-bit weights (W4A16, groups of 128 along K; vLLM's use_int4_w4a16 with block_shape [0, 128]):
 * w1 uint8 [E, N1, K1/2], w2 uint8 [E, K1, N1/4]: element k of a weight row in byte k/2, low nibble for even k
 * (quantize/w4a16.py); w*_scales bf16 [E, N, K/128]; w*_zeros uint8 [E, N, K/128], 0..15, or NULL: every zero is 8.
 * The weight element is bf16((q - z) * s); x, topk_w, topk_ids, out, residual and the workspace
 * (chitu_b200_moe_workspace_bytes) as in chitu_b200_fused_experts with wmode 0.  Runs on the grouped wgmma path only:
 * N1 % 256 == 0, K1 % 128 == 0, (N1/2) % 128 == 0, T * topk <= 8192 and E <= 1024, otherwise -2 before any launch. */
int chitu_b200_fused_experts_w4a16(const void* x, const void* w1, const void* w1_scales, const uint8_t* w1_zeros,
                                   const void* w2, const void* w2_scales, const uint8_t* w2_zeros, const void* topk_w,
                                   int topk_w_dtype, const void* topk_ids, int ids_dtype, int T, int topk, int E, int N1,
                                   int K1, void* out, const void* residual, void* workspace, int64_t workspace_bytes,
                                   void* stream);

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
                                void* stream);
int chitu_b200_allreduce_consume(void* comm, const void* residual, void* h_out, const void* norm_w, void* y,
                                 void* q, float* q_scales, int rows, int dim, float eps, void* stream);
/* h = bf16(sum_r partial_r) (+ residual);  optional outputs of RMSNorm(h)*norm_w: y (bf16) and / or q (fp8,
 * 128-group scales).  partial/residual/h_out: [rows, dim] bf16 (h_out may alias partial); rows <= 256. */
int chitu_b200_allreduce_residual_rmsnorm(void* handle, const void* partial, const void* residual,
                                          void* h_out, const void* norm_w, void* y, void* q, float* q_scales,
                                          int rows, int dim, float eps, void* stream);

/* ---- small decode-engine helpers (adjacent rows §8f; used by bench/engine) -------------------- */
/* out[t,:] = table[ids[t],:]  (VocabParallelEmbedding local lookup, tensor_parallel.py:199-208;
 * rows outside [vocab_start, vocab_start+rows) produce zeros).  table / out 16-byte aligned. */
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
