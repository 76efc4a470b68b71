// C-ABI entry points of the decode linears; dispatch between the SIMT weight-streaming path
// (gemv.cu) and the wgmma + TMA swap-AB path (gemm_tc.cu).
#include "common.cuh"

namespace cb {
// gemv.cu
int simt_linear16(const void* x, const void* w, const void* bias, const void* residual, void* y, int M,
                  int N, int K, int dtype, cudaStream_t st);
int simt_fp8_gemm(const void* a, const float* a_s, const void* b, const float* b_s, void* c, int M, int N,
                  int K, cudaStream_t st);
int simt_soft_fp8_gemm(const void* a, const void* b, const float* b_s, void* c, int M, int N, int K,
                       int out_dtype, cudaStream_t st);
int simt_w8a8_gemm(void* out, const int8_t* a, const int8_t* b, const float* a_scales,
                   const float* b_scales, const void* bias, int M, int N, int K, cudaStream_t st);
// gemm_tc.cu
bool tc_supported(int kind, int M, int N, int K);
int tc_linear16(const void* x, const void* w, const void* bias, const void* residual, void* y, int M, int N,
                int K, int dtype, void* ws, int64_t ws_bytes, cudaStream_t st, void* comm = nullptr);
int tc_fp8_gemm(const void* a, const float* a_s, const void* b, const float* b_s, void* c, int M, int N,
                int K, const void* residual, void* ws, int64_t ws_bytes, cudaStream_t st, void* comm = nullptr);
int64_t comm_slot_bytes(void* handle);
int tc_w8a8_gemm(void* out, const int8_t* a, const int8_t* b, const float* a_scales, const float* b_scales,
                 const void* bias, int M, int N, int K, void* ws, int64_t ws_bytes, cudaStream_t st);
int tc_soft_fp8_gemm(const void* a, const void* b, const float* b_s, void* c, int M, int N, int K, void* ws,
                     int64_t ws_bytes, cudaStream_t st);
int tc_linear16_silu_pairs(const void* x, const void* w, void* y, int M, int N, int K, void* ws, int64_t ws_bytes,
                           cudaStream_t st);
int64_t tc_workspace_bytes(int M, int N);
}  // namespace cb

using namespace cb;

enum { KIND_16 = 0, KIND_FP8 = 1, KIND_I8 = 2, KIND_SOFT = 3 };

// auto policy: the persistent stream-K wgmma kernel (bs=16 needs tensor cores outright: 16 tokens x 2 flop per weight
// byte exceeds the FMA pipes); the SIMT path remains for
// shapes TMA cannot address (row pitch not a multiple of 16 B, fp8 K % 128 != 0) and as impl=1.
static bool use_tc(int impl, int kind, int M, int N, int K, void* ws, int64_t ws_bytes) {
  if (impl == 1) return false;
  bool ok = tc_supported(kind, M, N, K) && ws && ws_bytes >= tc_workspace_bytes(M, N);
  if (impl == 2) return ok;
  return ok;
}

extern "C" int64_t chitu_b200_linear_workspace_bytes(int M, int N) { return tc_workspace_bytes(M, N); }

extern "C" int chitu_b200_linear_bf16(const void* x, const void* w, const void* bias, const void* residual,
                                      void* y, int M, int N, int K, int dtype, void* workspace,
                                      int64_t workspace_bytes, int impl, void* stream) {
  CB_ARG(x && w && y && M >= 0 && N > 0 && K > 0);
  CB_ARG(dtype == CB_BF16 || dtype == CB_F16);
  if (M == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (use_tc(impl, KIND_16, M, N, K, workspace, workspace_bytes))
    return tc_linear16(x, w, bias, residual, y, M, N, K, dtype, workspace, workspace_bytes, st);
  if (impl == 2) return fail(-2, "linear_bf16: wgmma path unavailable for M=%d N=%d K=%d (or workspace too small)", M, N, K);
  return simt_linear16(x, w, bias, residual, y, M, N, K, dtype, st);
}

// FeedForward's gate_up linear + SiluAndMul (models/model_llama.py:139-149, fused_moe.py:24-39) in one launch:
// w_pairs = the merged [w1 ; w3] weight with its rows interleaved (row 2i = gate_i, row 2i+1 = up_i) at load time;
// y[M, N/2] = bf16(bf16(silu(bf16 g)) * bf16(u)) — the roundings of the two separate reference ops.  bf16, wgmma only.
extern "C" int chitu_b200_linear_bf16_silu_pairs(const void* x, const void* w_pairs, void* y, int M, int N, int K,
                                                 void* workspace, int64_t workspace_bytes, void* stream) {
  CB_ARG(x && w_pairs && y && M >= 0 && N > 0 && N % 2 == 0 && K > 0);
  if (M == 0) return 0;
  if (!use_tc(2, KIND_16, M, N, K, workspace, workspace_bytes))
    return fail(-2, "linear_bf16_silu_pairs: wgmma path unavailable for M=%d N=%d K=%d (or workspace too small)", M, N, K);
  return tc_linear16_silu_pairs(x, w_pairs, y, M, N, K, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int chitu_b200_fp8_gemm(const void* a, const float* a_s, const void* b, const float* b_s,
                                   void* c, int M, int N, int K, const void* residual, void* workspace,
                                   int64_t workspace_bytes, int impl, void* stream) {
  CB_ARG(a && a_s && b && b_s && c && M >= 0 && N > 0 && K > 0);
  if (M == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (use_tc(impl, KIND_FP8, M, N, K, workspace, workspace_bytes))
    return tc_fp8_gemm(a, a_s, b, b_s, c, M, N, K, residual, workspace, workspace_bytes, st);
  if (impl == 2) return fail(-2, "fp8_gemm: wgmma path unavailable for M=%d N=%d K=%d (or workspace too small)", M, N, K);
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
  if (!use_tc(2, KIND_FP8, M, N, K, workspace, workspace_bytes))
    return fail(-2, "fp8_gemm_ar: wgmma path unavailable for M=%d N=%d K=%d (or workspace too small)", M, N, K);
  return tc_fp8_gemm(a, a_s, b, b_s, nullptr, M, N, K, nullptr, workspace, workspace_bytes, (cudaStream_t)stream, comm);
}

extern "C" int chitu_b200_linear_bf16_ar(const void* x, const void* w, int M, int N, int K, void* comm, void* workspace,
                                         int64_t workspace_bytes, void* stream) {
  CB_ARG(x && w && comm && M > 0 && N > 0 && N % 2 == 0 && K > 0);
  CB_ARG((int64_t)M * N * 2 <= comm_slot_bytes(comm));
  if (!use_tc(2, KIND_16, M, N, K, workspace, workspace_bytes))
    return fail(-2, "linear_bf16_ar: wgmma path unavailable for M=%d N=%d K=%d (or workspace too small)", M, N, K);
  return tc_linear16(x, w, nullptr, nullptr, nullptr, M, N, K, CB_BF16, workspace, workspace_bytes, (cudaStream_t)stream, comm);
}

extern "C" int chitu_b200_soft_fp8_gemm(const void* a, const void* b, const float* b_s, void* c, int M,
                                        int N, int K, int out_dtype, void* workspace,
                                        int64_t workspace_bytes, int impl, void* stream) {
  CB_ARG(a && b && b_s && c && M >= 0 && N > 0 && K > 0);
  if (M == 0) return 0;
  // wgmma path: the fp8 weight tile is converted to bf16 in shared memory between the TMA landing and the bf16 MMA
  if (out_dtype == CB_BF16 && use_tc(impl, KIND_SOFT, M, N, K, workspace, workspace_bytes))
    return tc_soft_fp8_gemm(a, b, b_s, c, M, N, K, workspace, workspace_bytes, (cudaStream_t)stream);
  if (impl == 2) return fail(-2, "soft_fp8_gemm: wgmma path unavailable for M=%d N=%d K=%d (bf16 only, K %% 128 == 0)", M, N, K);
  return simt_soft_fp8_gemm(a, b, b_s, c, M, N, K, out_dtype, (cudaStream_t)stream);
}

extern "C" int chitu_b200_w8a8_gemm(void* out, const int8_t* a, const int8_t* b, const float* a_scales,
                                    const float* b_scales, const void* bias, int M, int N, int K,
                                    void* workspace, int64_t workspace_bytes, int impl, void* stream) {
  CB_ARG(out && a && b && a_scales && b_scales && M >= 0 && N > 0 && K > 0);
  if (M == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (use_tc(impl, KIND_I8, M, N, K, workspace, workspace_bytes))
    return tc_w8a8_gemm(out, a, b, a_scales, b_scales, bias, M, N, K, workspace, workspace_bytes, st);
  if (impl == 2) return fail(-2, "w8a8_gemm: wgmma path unavailable for M=%d N=%d K=%d (or workspace too small)", M, N, K);
  return simt_w8a8_gemm(out, a, b, a_scales, b_scales, bias, M, N, K, st);
}

CB_DEFINE_TL_SETTER(linear)
