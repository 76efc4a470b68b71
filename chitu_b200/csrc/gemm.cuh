// The decode GEMMs behind the C entries of linear.cu and moe.cu: the wgmma + TMA kernel (gemm_tc.cu) and the SIMT
// weight-streaming kernels (gemv.cu).
#pragma once
#include "common.cuh"

namespace cb {

// the KIND of the wgmma GEMM kernel; SOFT: fp8 weights -> bf16 in shared memory, bf16 MMA; W4: 4-bit weights with a
// scale and a zero per group of 128 -> bf16 / fp16 in shared memory, 16-bit MMA; FP8R: e4m3 activations and weights
// with a per-token and a per-output-channel scale, e4m3 MMA
enum { KIND_16 = 0, KIND_FP8 = 1, KIND_I8 = 2, KIND_SOFT = 3, KIND_W4 = 4, KIND_FP8R = 5 };

// ---- gemm_tc.cu ----
bool tc_supported(int kind, int M, int N, int K);
int64_t tc_workspace_bytes(int M, int N);
int64_t tc_max_tiles();
// comm != null (a comm.cu communicator): the bf16 result goes to every rank's push area instead of y / c
int tc_linear16(const void* x, const void* w, const void* bias, const void* residual, void* y, int M, int N, int K,
                int dtype, void* ws, int64_t ws_bytes, cudaStream_t st, void* comm = nullptr);
int tc_linear16_silu_pairs(const void* x, const void* w, void* y, int M, int N, int K, void* ws, int64_t ws_bytes,
                           cudaStream_t st);
int tc_fp8_gemm(const void* a, const float* a_s, const void* b, const float* b_s, void* c, int M, int N, int K,
                const void* residual, void* ws, int64_t ws_bytes, cudaStream_t st, void* comm = nullptr);
int tc_soft_fp8_gemm(const void* a, const void* b, const float* b_s, void* c, int M, int N, int K, void* ws,
                     int64_t ws_bytes, cudaStream_t st);
int tc_w4a16(const void* x, const void* qweight, const void* scales, const uint8_t* zeros, const void* residual, void* y,
             int M, int N, int K, int dtype, bool pairs, void* ws, int64_t ws_bytes, cudaStream_t st);
int tc_fp8_rowwise_gemm(const void* a, const float* a_s, const void* b, const float* b_s, const void* bias,
                        const void* residual, void* y, int M, int N, int K, bool pairs, void* ws, int64_t ws_bytes,
                        cudaStream_t st);
int tc_w8a8_gemm(void* out, const int8_t* a, const int8_t* b, const float* a_scales, const float* b_scales,
                 const void* bias, int M, int N, int K, void* ws, int64_t ws_bytes, cudaStream_t st);
int tc_grouped_gemm(int kind, const void* xs, const float* a_s, const void* w, const float* b_s, const void* w4_s,
                    const uint8_t* w4_z, void* out, int rows, int E, int Ng, int K, int max_tokens_per_expert,
                    const int* g_num_tiles, const int* g_tile_wrow, const int* g_tile_xrow, const int* g_tile_cnt,
                    const float* row_scale, const int* out_rows, void* ws, int64_t ws_bytes, cudaStream_t st);

// ---- gemv.cu ----
int simt_linear16(const void* x, const void* w, const void* bias, const void* residual, void* y, int M, int N, int K,
                  int dtype, cudaStream_t st);
int simt_fp8_gemm(const void* a, const float* a_s, const void* b, const float* b_s, void* c, int M, int N, int K,
                  cudaStream_t st);
int simt_soft_fp8_gemm(const void* a, const void* b, const float* b_s, void* c, int M, int N, int K, int out_dtype,
                       cudaStream_t st);
int simt_w8a8_gemm(void* out, const int8_t* a, const int8_t* b, const float* a_scales, const float* b_scales,
                   const void* bias, int M, int N, int K, cudaStream_t st);

// ---- comm.cu ----
int64_t comm_slot_bytes(void* handle);   // the largest bf16 result, in bytes, one reduce carries (0 without a handle)

}  // namespace cb
