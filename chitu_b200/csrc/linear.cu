// C-ABI entry points of the decode linears: each runs the persistent stream-K wgmma + TMA kernel (gemm_tc.cu) wherever
// it can (bs=16 needs tensor cores outright: 16 tokens x 2 flop per weight byte exceed the FMA pipes) or the SIMT
// weight-streaming kernels (gemv.cu), as linear_path() picks.
#include "common.cuh"
#include "gemm.cuh"

using namespace cb;

// The path of a linear entry: impl = 1 SIMT, impl = 2 wgmma or the -2 refusal, any other impl wgmma where it can run (a
// shape TMA can address, bf16 activations for soft fp8, a workspace of tc_workspace_bytes) and SIMT elsewhere.
enum { kSimt = 0, kWgmma = 1 };
static int linear_path(const char* entry, int kind, int impl, int dtype, int M, int N, int K, void* ws, int64_t ws_bytes) {
  if (impl == 1) return kSimt;
  if ((kind != KIND_SOFT || dtype == CB_BF16) && tc_supported(kind, M, N, K) && ws && ws_bytes >= tc_workspace_bytes(M, N))
    return kWgmma;
  if (impl != 2) return kSimt;
  return fail(-2, "%s: wgmma path unavailable for M=%d N=%d K=%d (shape, dtype or workspace)", entry, M, N, K);
}

extern "C" int64_t chitu_b200_linear_workspace_bytes(int M, int N) { return tc_workspace_bytes(M, N); }

extern "C" int chitu_b200_linear_bf16(const void* x, const void* w, const void* bias, const void* residual,
                                      void* y, int M, int N, int K, int dtype, void* workspace,
                                      int64_t workspace_bytes, int impl, void* stream) {
  CB_ARG(x && w && y && M >= 0 && N > 0 && K > 0);
  CB_ARG(dtype == CB_BF16 || dtype == CB_F16);
  if (M == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int path = linear_path(__func__, KIND_16, impl, dtype, M, N, K, workspace, workspace_bytes);
  if (path == kWgmma) return tc_linear16(x, w, bias, residual, y, M, N, K, dtype, workspace, workspace_bytes, st);
  return path == kSimt ? simt_linear16(x, w, bias, residual, y, M, N, K, dtype, st) : path;
}

// FeedForward's gate_up linear + SiluAndMul (models/model_llama.py:139-149, fused_moe.py:24-39) in one launch:
// w_pairs = the merged [w1 ; w3] weight with its rows interleaved (row 2i = gate_i, row 2i+1 = up_i) at load time;
// y[M, N/2] = bf16(bf16(silu(bf16 g)) * bf16(u)) — the roundings of the two separate reference ops.  bf16, wgmma only.
extern "C" int chitu_b200_linear_bf16_silu_pairs(const void* x, const void* w_pairs, void* y, int M, int N, int K,
                                                 void* workspace, int64_t workspace_bytes, void* stream) {
  CB_ARG(x && w_pairs && y && M >= 0 && N > 0 && N % 2 == 0 && K > 0);
  if (M == 0) return 0;
  const int path = linear_path(__func__, KIND_16, 2, CB_BF16, M, N, K, workspace, workspace_bytes);
  if (path != kWgmma) return path;
  return tc_linear16_silu_pairs(x, w_pairs, y, M, N, K, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int chitu_b200_fp8_gemm(const void* a, const float* a_s, const void* b, const float* b_s,
                                   void* c, int M, int N, int K, const void* residual, void* workspace,
                                   int64_t workspace_bytes, int impl, void* stream) {
  CB_ARG(a && a_s && b && b_s && c && M >= 0 && N > 0 && K > 0);
  if (M == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int path = linear_path(__func__, KIND_FP8, impl, CB_BF16, M, N, K, workspace, workspace_bytes);
  if (path == kWgmma) return tc_fp8_gemm(a, a_s, b, b_s, c, M, N, K, residual, workspace, workspace_bytes, st);
  if (path != kSimt) return path;
  int rc = simt_fp8_gemm(a, a_s, b, b_s, c, M, N, K, st);
  if (rc || !residual) return rc;
  return chitu_b200_add(c, residual, c, (int64_t)M * N, CB_BF16, stream);
}

// Row-parallel linears of a tensor-parallel layer with the all-reduce started from the GEMM EPILOGUE (SURVEY §5.8,
// tensor_parallel.py:157-169, model_deepseek_v3.py:1011): instead of writing `y` and launching a collective, the epilogue
// stores each bf16 output tile straight into every rank's push area over NVLink as epoch-tagged 8-byte words; the reduce
// itself is chitu_b200_allreduce_consume(comm, ...) fused with the residual add / RMSNorm / fp8 quant.
extern "C" int chitu_b200_fp8_gemm_ar(const void* a, const float* a_s, const void* b, const float* b_s, int M, int N, int K,
                                      void* comm, void* workspace, int64_t workspace_bytes, void* stream) {
  CB_ARG(a && a_s && b && b_s && comm && M > 0 && N > 0 && N % 2 == 0 && K > 0);
  CB_ARG((int64_t)M * N * 2 <= comm_slot_bytes(comm));
  const int path = linear_path(__func__, KIND_FP8, 2, CB_BF16, M, N, K, workspace, workspace_bytes);
  if (path != kWgmma) return path;
  return tc_fp8_gemm(a, a_s, b, b_s, nullptr, M, N, K, nullptr, workspace, workspace_bytes, (cudaStream_t)stream, comm);
}

extern "C" int chitu_b200_linear_bf16_ar(const void* x, const void* w, int M, int N, int K, void* comm, void* workspace,
                                         int64_t workspace_bytes, void* stream) {
  CB_ARG(x && w && comm && M > 0 && N > 0 && N % 2 == 0 && K > 0);
  CB_ARG((int64_t)M * N * 2 <= comm_slot_bytes(comm));
  const int path = linear_path(__func__, KIND_16, 2, CB_BF16, M, N, K, workspace, workspace_bytes);
  if (path != kWgmma) return path;
  return tc_linear16(x, w, nullptr, nullptr, nullptr, M, N, K, CB_BF16, workspace, workspace_bytes, (cudaStream_t)stream, comm);
}

// wgmma path: the fp8 weight tile is converted to bf16 in shared memory between the TMA landing and the bf16 MMA
extern "C" int chitu_b200_soft_fp8_gemm(const void* a, const void* b, const float* b_s, void* c, int M,
                                        int N, int K, int out_dtype, void* workspace,
                                        int64_t workspace_bytes, int impl, void* stream) {
  CB_ARG(a && b && b_s && c && M >= 0 && N > 0 && K > 0);
  if (M == 0) return 0;
  const int path = linear_path(__func__, KIND_SOFT, impl, out_dtype, M, N, K, workspace, workspace_bytes);
  if (path == kWgmma) return tc_soft_fp8_gemm(a, b, b_s, c, M, N, K, workspace, workspace_bytes, (cudaStream_t)stream);
  return path == kSimt ? simt_soft_fp8_gemm(a, b, b_s, c, M, N, K, out_dtype, (cudaStream_t)stream) : path;
}

extern "C" int chitu_b200_w8a8_gemm(void* out, const int8_t* a, const int8_t* b, const float* a_scales,
                                    const float* b_scales, const void* bias, int M, int N, int K,
                                    void* workspace, int64_t workspace_bytes, int impl, void* stream) {
  CB_ARG(out && a && b && a_scales && b_scales && M >= 0 && N > 0 && K > 0);
  if (M == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int path = linear_path(__func__, KIND_I8, impl, CB_F16, M, N, K, workspace, workspace_bytes);
  if (path == kWgmma) return tc_w8a8_gemm(out, a, b, a_scales, b_scales, bias, M, N, K, workspace, workspace_bytes, st);
  return path == kSimt ? simt_w8a8_gemm(out, a, b, a_scales, b_scales, bias, M, N, K, st) : path;
}

// W4A16, group 128 (GPTQ / AWQ after quantize/w4a16.py's repack): the 4-bit weight tile is turned into bf16 / fp16 in
// shared memory between the TMA landing and the 16-bit MMA.  wgmma only; refusals name the entry and launch nothing.
static int w4a16(const char* entry, const void* x, const void* qweight, const void* scales, const uint8_t* zeros,
                 const void* residual, void* y, int M, int N, int K, int dtype, bool pairs, void* workspace,
                 int64_t workspace_bytes, void* stream) {
  CB_ARG_AS(entry, x && qweight && scales && zeros && y && M >= 0 && N > 0 && K > 0);
  CB_ARG_AS(entry, ((uintptr_t)x | (uintptr_t)qweight | (uintptr_t)scales | (uintptr_t)zeros | (uintptr_t)residual |
                    (uintptr_t)y) % 16 == 0);
  CB_ARG_AS(entry, K % 128 == 0);
  CB_ARG_AS(entry, dtype == CB_BF16 || dtype == CB_F16);
  CB_ARG_AS(entry, !pairs || N % 2 == 0);
  if (M == 0) return 0;
  const int path = linear_path(entry, KIND_W4, 2, dtype, M, N, K, workspace, workspace_bytes);
  if (path != kWgmma) return path;
  return tc_w4a16(x, qweight, scales, zeros, residual, y, M, N, K, dtype, pairs, workspace, workspace_bytes,
                  (cudaStream_t)stream);
}

extern "C" int chitu_b200_w4a16_gemm(const void* x, const void* qweight, const void* scales, const uint8_t* zeros,
                                     const void* residual, void* y, int M, int N, int K, int dtype, void* workspace,
                                     int64_t workspace_bytes, void* stream) {
  return w4a16(__func__, x, qweight, scales, zeros, residual, y, M, N, K, dtype, false, workspace, workspace_bytes,
               stream);
}

extern "C" int chitu_b200_w4a16_gemm_silu_pairs(const void* x, const void* qweight, const void* scales,
                                                const uint8_t* zeros, void* y, int M, int N, int K, int dtype,
                                                void* workspace, int64_t workspace_bytes, void* stream) {
  return w4a16(__func__, x, qweight, scales, zeros, nullptr, y, M, N, K, dtype, true, workspace, workspace_bytes,
               stream);
}

// FP8 W8A8 with rowwise scales, the Fp8LinearMethod / torch._scaled_mm(a, b.T, scale_a [M, 1], scale_b [1, N],
// bias, out_dtype=bf16) interface of vLLM's per-channel FP8 checkpoints: e4m3 x e4m3 on the tensor cores, every 128-K
// stage promoted into fp32, the two scales applied in the epilogue.  wgmma only; refusals name the entry and launch
// nothing.
static int fp8_rowwise(const char* entry, const void* a, const float* a_s, const void* b, const float* b_s,
                       const void* bias, const void* residual, void* y, int M, int N, int K, bool pairs, void* workspace,
                       int64_t workspace_bytes, void* stream) {
  CB_ARG_AS(entry, a && a_s && b && b_s && y && M >= 0 && N > 0 && K > 0);
  CB_ARG_AS(entry, ((uintptr_t)a | (uintptr_t)a_s | (uintptr_t)b | (uintptr_t)b_s | (uintptr_t)bias |
                    (uintptr_t)residual | (uintptr_t)y) % 16 == 0);
  CB_ARG_AS(entry, K % 16 == 0);
  CB_ARG_AS(entry, !pairs || N % 2 == 0);
  if (M == 0) return 0;
  const int path = linear_path(entry, KIND_FP8R, 2, CB_BF16, M, N, K, workspace, workspace_bytes);
  if (path != kWgmma) return path;
  return tc_fp8_rowwise_gemm(a, a_s, b, b_s, bias, residual, y, M, N, K, pairs, workspace, workspace_bytes,
                             (cudaStream_t)stream);
}

extern "C" int chitu_b200_fp8_rowwise_gemm(const void* a, const float* a_s, const void* b, const float* b_s,
                                           const void* bias, const void* residual, void* y, int M, int N, int K,
                                           void* workspace, int64_t workspace_bytes, void* stream) {
  return fp8_rowwise(__func__, a, a_s, b, b_s, bias, residual, y, M, N, K, false, workspace, workspace_bytes, stream);
}

extern "C" int chitu_b200_fp8_rowwise_gemm_silu_pairs(const void* a, const float* a_s, const void* b, const float* b_s,
                                                      void* y, int M, int N, int K, void* workspace,
                                                      int64_t workspace_bytes, void* stream) {
  return fp8_rowwise(__func__, a, a_s, b, b_s, nullptr, nullptr, y, M, N, K, true, workspace, workspace_bytes, stream);
}

CB_DEFINE_TL_SETTER(linear)
