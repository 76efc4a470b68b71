// SIMT weight-streaming skinny GEMM ("GEMV" path): y[M,N] = x[M,K] · W[N,K]^T for M <= 16.
//
// Decode linears are HBM-bound weight streams (SURVEY §7.3-1): each warp owns two weight rows,
// the 32 lanes stride K with 128-bit `ld.global.nc.L1::no_allocate` loads (each weight byte is
// read exactly once from HBM), activations are re-read through L1 (they are tiny), fp32
// accumulation, butterfly reduce.  This path is the small-M / any-shape implementation; the
// wgmma + TMA swap-AB kernel in gemm_tc.cu is the tensor-core implementation of the same
// entry points (impl = 2) and the default for M > 2.
#include "common.cuh"

using namespace cb;

namespace {

constexpr int kWarps = 8;
constexpr int kRowsPerWarp = 2;

template <typename T>
__device__ __forceinline__ float dot8(const uint4& w, const uint4& x) {
  const T* tag = nullptr;
  float2 w0 = unpack2(w.x, tag), w1 = unpack2(w.y, tag), w2 = unpack2(w.z, tag), w3 = unpack2(w.w, tag);
  float2 x0 = unpack2(x.x, tag), x1 = unpack2(x.y, tag), x2 = unpack2(x.z, tag), x3 = unpack2(x.w, tag);
  float s = w0.x * x0.x;
  s = fmaf(w0.y, x0.y, s);
  s = fmaf(w1.x, x1.x, s);
  s = fmaf(w1.y, x1.y, s);
  s = fmaf(w2.x, x2.x, s);
  s = fmaf(w2.y, x2.y, s);
  s = fmaf(w3.x, x3.x, s);
  s = fmaf(w3.y, x3.y, s);
  return s;
}

// -------------------------------------------------------------------------------------------
// 16-bit weights (bf16 / fp16): F.linear
// -------------------------------------------------------------------------------------------
template <typename T, int MT>
__global__ void __launch_bounds__(kWarps * 32) gemv16_kernel(const T* __restrict__ x,
                                                            const T* __restrict__ w,
                                                            const T* __restrict__ bias,
                                                            const T* __restrict__ residual,
                                                            T* __restrict__ y, int M, int N, int K) {
  cb::pdl_prologue();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n0 = (blockIdx.x * kWarps + warp) * kRowsPerWarp;
  if (n0 >= N) return;
  const int n1 = min(n0 + 1, N - 1);
  const T* w0p = w + (int64_t)n0 * K;
  const T* w1p = w + (int64_t)n1 * K;
  float acc0[MT], acc1[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) acc0[m] = acc1[m] = 0.f;

#pragma unroll 2
  for (int k = lane * 8; k < K; k += 256) {
    uint4 wa = ld_stream(w0p + k);
    uint4 wb = ld_stream(w1p + k);
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      const int mm = m < M ? m : M - 1;
      uint4 xv = *reinterpret_cast<const uint4*>(x + (int64_t)mm * K + k);
      acc0[m] += dot8<T>(wa, xv);
      acc1[m] += dot8<T>(wb, xv);
    }
  }
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    acc0[m] = warp_sum(acc0[m]);
    acc1[m] = warp_sum(acc1[m]);
  }
  if (lane == 0) {
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      if (m < M) {
        float v0 = acc0[m], v1 = acc1[m];
        if (bias) {  // F.linear: bias joins the fp32 accumulator, one rounding
          v0 += io<T>::to_f(bias[n0]);
          v1 += io<T>::to_f(bias[n1]);
        }
        if (residual) {
          v0 = io<T>::to_f(io<T>::from_f(v0)) + io<T>::to_f(residual[(int64_t)m * N + n0]);
          v1 = io<T>::to_f(io<T>::from_f(v1)) + io<T>::to_f(residual[(int64_t)m * N + n1]);
        }
        y[(int64_t)m * N + n0] = io<T>::from_f(v0);
        if (n0 + 1 < N) y[(int64_t)m * N + n1] = io<T>::from_f(v1);
      }
    }
  }
}

// -------------------------------------------------------------------------------------------
// fp8 x fp8 block-scaled (fp8_gemm_deepseek_v3, triton_kernels.py:303-365)
// lane covers 16 consecutive k (one 16-byte load) -> always inside one 128-wide scale block.
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ float dot16_fp8(const uint4& w, const uint4& a) {
  const uint32_t wv[4] = {w.x, w.y, w.z, w.w};
  const uint32_t av[4] = {a.x, a.y, a.z, a.w};
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 w0 = fp8x2_to_float2((uint16_t)(wv[i] & 0xffff)), w1 = fp8x2_to_float2((uint16_t)(wv[i] >> 16));
    float2 a0 = fp8x2_to_float2((uint16_t)(av[i] & 0xffff)), a1 = fp8x2_to_float2((uint16_t)(av[i] >> 16));
    s = fmaf(w0.x, a0.x, s);
    s = fmaf(w0.y, a0.y, s);
    s = fmaf(w1.x, a1.x, s);
    s = fmaf(w1.y, a1.y, s);
  }
  return s;
}

template <int MT>
__global__ void __launch_bounds__(kWarps * 32) gemv_fp8_kernel(const uint8_t* __restrict__ a,
                                                              const float* __restrict__ a_s,
                                                              const uint8_t* __restrict__ b,
                                                              const float* __restrict__ b_s,
                                                              __nv_bfloat16* __restrict__ c, int M, int N,
                                                              int K) {
  cb::pdl_prologue();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n0 = (blockIdx.x * kWarps + warp) * kRowsPerWarp;
  if (n0 >= N) return;
  const int n1 = min(n0 + 1, N - 1);
  const int kblocks = (K + 127) / 128;
  const uint8_t* w0p = b + (int64_t)n0 * K;
  const uint8_t* w1p = b + (int64_t)n1 * K;
  const float* bs0 = b_s + (int64_t)(n0 / 128) * kblocks;
  const float* bs1 = b_s + (int64_t)(n1 / 128) * kblocks;
  float acc0[MT], acc1[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) acc0[m] = acc1[m] = 0.f;

#pragma unroll 2
  for (int k = lane * 16; k < K; k += 512) {
    uint4 wa = ld_stream(w0p + k);
    uint4 wb = ld_stream(w1p + k);
    const int kb = k >> 7;
    const float s0 = bs0[kb], s1 = bs1[kb];
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      const int mm = m < M ? m : M - 1;
      uint4 av = *reinterpret_cast<const uint4*>(a + (int64_t)mm * K + k);
      const float as = a_s[(int64_t)mm * kblocks + kb];
      acc0[m] = fmaf(dot16_fp8(wa, av) * as, s0, acc0[m]);
      acc1[m] = fmaf(dot16_fp8(wb, av) * as, s1, acc1[m]);
    }
  }
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    acc0[m] = warp_sum(acc0[m]);
    acc1[m] = warp_sum(acc1[m]);
  }
  if (lane == 0) {
#pragma unroll
    for (int m = 0; m < MT; ++m)
      if (m < M) {
        c[(int64_t)m * N + n0] = __float2bfloat16_rn(acc0[m]);
        if (n0 + 1 < N) c[(int64_t)m * N + n1] = __float2bfloat16_rn(acc1[m]);
      }
  }
}

// -------------------------------------------------------------------------------------------
// soft fp8 (W8A16): w_bf16 = bf16(bits(w) * (b_s * 2^120)); bf16 x bf16 -> fp32 acc
// (soft_fp8_gemm_deepseek_v3_kernel, triton_kernels.py:388-508)
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ float softfp8_to_bf16f(uint32_t byte, float scale2) {
  float f = __uint_as_float(((byte & 0x80u) << 24) | ((byte & 0x7fu) << 20));
  return __bfloat162float(__float2bfloat16_rn(f * scale2));
}

template <typename T, int MT>
__global__ void __launch_bounds__(kWarps * 32) gemv_softfp8_kernel(const T* __restrict__ a,
                                                                  const uint8_t* __restrict__ b,
                                                                  const float* __restrict__ b_s,
                                                                  T* __restrict__ c, int M, int N, int K) {
  cb::pdl_prologue();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n0 = (blockIdx.x * kWarps + warp) * kRowsPerWarp;
  if (n0 >= N) return;
  const int n1 = min(n0 + 1, N - 1);
  const int kblocks = (K + 127) / 128;
  const uint8_t* w0p = b + (int64_t)n0 * K;
  const uint8_t* w1p = b + (int64_t)n1 * K;
  const float* bs0 = b_s + (int64_t)(n0 / 128) * kblocks;
  const float* bs1 = b_s + (int64_t)(n1 / 128) * kblocks;
  const float two120 = __uint_as_float(0x7B800000u);
  float acc0[MT], acc1[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) acc0[m] = acc1[m] = 0.f;

  for (int k = lane * 16; k < K; k += 512) {
    uint4 wa = ld_stream(w0p + k);
    uint4 wb = ld_stream(w1p + k);
    const int kb = k >> 7;
    const float s0 = bs0[kb] * two120, s1 = bs1[kb] * two120;
    const uint32_t wav[4] = {wa.x, wa.y, wa.z, wa.w};
    const uint32_t wbv[4] = {wb.x, wb.y, wb.z, wb.w};
    float f0[16], f1[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      f0[i] = softfp8_to_bf16f((wav[i >> 2] >> ((i & 3) * 8)) & 0xffu, s0);
      f1[i] = softfp8_to_bf16f((wbv[i >> 2] >> ((i & 3) * 8)) & 0xffu, s1);
    }
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      const int mm = m < M ? m : M - 1;
      const uint4* ap = reinterpret_cast<const uint4*>(a + (int64_t)mm * K + k);
      uint4 a0 = ap[0], a1 = ap[1];
      const uint32_t av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const T* tag = nullptr;
      float s_0 = 0.f, s_1 = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float2 xv = unpack2(av[i], tag);
        s_0 = fmaf(f0[2 * i], xv.x, s_0);
        s_0 = fmaf(f0[2 * i + 1], xv.y, s_0);
        s_1 = fmaf(f1[2 * i], xv.x, s_1);
        s_1 = fmaf(f1[2 * i + 1], xv.y, s_1);
      }
      acc0[m] += s_0;
      acc1[m] += s_1;
    }
  }
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    acc0[m] = warp_sum(acc0[m]);
    acc1[m] = warp_sum(acc1[m]);
  }
  if (lane == 0) {
#pragma unroll
    for (int m = 0; m < MT; ++m)
      if (m < M) {
        c[(int64_t)m * N + n0] = io<T>::from_f(acc0[m]);
        if (n0 + 1 < N) c[(int64_t)m * N + n1] = io<T>::from_f(acc1[m]);
      }
  }
}

// -------------------------------------------------------------------------------------------
// int8 x int8 (w8a8gemm.mm / w8a8gemv.mv): exact int32 dot via dp4a, fp16 out.
// -------------------------------------------------------------------------------------------
template <int MT>
__global__ void __launch_bounds__(kWarps * 32) gemv_i8_kernel(__half* __restrict__ out,
                                                             const int8_t* __restrict__ a,
                                                             const int8_t* __restrict__ b,
                                                             const float* __restrict__ a_scales,
                                                             const float* __restrict__ b_scales,
                                                             const __half* __restrict__ bias, int M, int N,
                                                             int K) {
  cb::pdl_prologue();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n0 = (blockIdx.x * kWarps + warp) * kRowsPerWarp;
  if (n0 >= N) return;
  const int n1 = min(n0 + 1, N - 1);
  const int8_t* w0p = b + (int64_t)n0 * K;
  const int8_t* w1p = b + (int64_t)n1 * K;
  int acc0[MT], acc1[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) acc0[m] = acc1[m] = 0;

#pragma unroll 2
  for (int k = lane * 16; k < K; k += 512) {
    uint4 wa = ld_stream(w0p + k);
    uint4 wb = ld_stream(w1p + k);
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      const int mm = m < M ? m : M - 1;
      uint4 av = *reinterpret_cast<const uint4*>(a + (int64_t)mm * K + k);
      acc0[m] = __dp4a((int)wa.x, (int)av.x, acc0[m]);
      acc0[m] = __dp4a((int)wa.y, (int)av.y, acc0[m]);
      acc0[m] = __dp4a((int)wa.z, (int)av.z, acc0[m]);
      acc0[m] = __dp4a((int)wa.w, (int)av.w, acc0[m]);
      acc1[m] = __dp4a((int)wb.x, (int)av.x, acc1[m]);
      acc1[m] = __dp4a((int)wb.y, (int)av.y, acc1[m]);
      acc1[m] = __dp4a((int)wb.z, (int)av.z, acc1[m]);
      acc1[m] = __dp4a((int)wb.w, (int)av.w, acc1[m]);
    }
  }
#pragma unroll
  for (int m = 0; m < MT; ++m) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      acc0[m] += __shfl_xor_sync(0xffffffffu, acc0[m], o);
      acc1[m] += __shfl_xor_sync(0xffffffffu, acc1[m], o);
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int m = 0; m < MT; ++m)
      if (m < M) {
        float v0 = (float)acc0[m] * a_scales[m] * b_scales[n0];
        float v1 = (float)acc1[m] * a_scales[m] * b_scales[n1];
        __half h0 = __float2half_rn(v0), h1 = __float2half_rn(v1);
        if (bias) {
          h0 = __hadd(h0, bias[n0]);
          h1 = __hadd(h1, bias[n1]);
        }
        out[(int64_t)m * N + n0] = h0;
        if (n0 + 1 < N) out[(int64_t)m * N + n1] = h1;
      }
  }
}

inline int grid_for(int N) { return cdiv(N, kWarps * kRowsPerWarp); }

}  // namespace

// The SIMT entry points process M in chunks of <= 16 tokens.
#define DISPATCH_MT(Mc, CALL)          \
  if (Mc <= 1) { CALL(1); }            \
  else if (Mc <= 2) { CALL(2); }       \
  else if (Mc <= 4) { CALL(4); }       \
  else if (Mc <= 8) { CALL(8); }       \
  else { CALL(16); }

namespace cb {

int simt_linear16(const void* x, const void* w, const void* bias, const void* residual, void* y, int M,
                  int N, int K, int dtype, cudaStream_t st) {
  CB_ARG(K % 8 == 0);
  int launches = 0;
  for (int m0 = 0; m0 < M; m0 += 16) {
    int Mc = M - m0 < 16 ? M - m0 : 16;
    if (dtype == CB_BF16) {
      using T = __nv_bfloat16;
#define CALL(MT)                                                                                   \
  cb::launch_k(gemv16_kernel<T, MT>, dim3(grid_for(N)), dim3(kWarps * 32), 0, st,                                        \
      (const T*)x + (int64_t)m0 * K, (const T*)w, (const T*)bias,                                  \
      residual ? (const T*)residual + (int64_t)m0 * N : nullptr, (T*)y + (int64_t)m0 * N, Mc, N, K)
      DISPATCH_MT(Mc, CALL)
#undef CALL
    } else if (dtype == CB_F16) {
      using T = __half;
#define CALL(MT)                                                                                   \
  cb::launch_k(gemv16_kernel<T, MT>, dim3(grid_for(N)), dim3(kWarps * 32), 0, st,                                        \
      (const T*)x + (int64_t)m0 * K, (const T*)w, (const T*)bias,                                  \
      residual ? (const T*)residual + (int64_t)m0 * N : nullptr, (T*)y + (int64_t)m0 * N, Mc, N, K)
      DISPATCH_MT(Mc, CALL)
#undef CALL
    } else {
      return fail(-1, "linear_bf16: unsupported dtype %d", dtype);
    }
    ++launches;
  }
  CB_LAUNCHED(launches);
  return 0;
}

int simt_fp8_gemm(const void* a, const float* a_s, const void* b, const float* b_s, void* c, int M, int N,
                  int K, cudaStream_t st) {
  CB_ARG(K % 16 == 0);
  const int kblocks = (K + 127) / 128;
  int launches = 0;
  for (int m0 = 0; m0 < M; m0 += 16) {
    int Mc = M - m0 < 16 ? M - m0 : 16;
#define CALL(MT)                                                                                      \
  cb::launch_k(gemv_fp8_kernel<MT>, dim3(grid_for(N)), dim3(kWarps * 32), 0, st,                                            \
      (const uint8_t*)a + (int64_t)m0 * K, a_s + (int64_t)m0 * kblocks, (const uint8_t*)b, b_s,       \
      (__nv_bfloat16*)c + (int64_t)m0 * N, Mc, N, K)
    DISPATCH_MT(Mc, CALL)
#undef CALL
    ++launches;
  }
  CB_LAUNCHED(launches);
  return 0;
}

int simt_soft_fp8_gemm(const void* a, const void* b, const float* b_s, void* c, int M, int N, int K,
                       int out_dtype, cudaStream_t st) {
  CB_ARG(K % 16 == 0);
  int launches = 0;
  for (int m0 = 0; m0 < M; m0 += 8) {
    int Mc = M - m0 < 8 ? M - m0 : 8;
    if (out_dtype == CB_BF16) {
      using T = __nv_bfloat16;
#define CALL(MT)                                                                              \
  cb::launch_k(gemv_softfp8_kernel<T, MT>, dim3(grid_for(N)), dim3(kWarps * 32), 0, st,                             \
      (const T*)a + (int64_t)m0 * K, (const uint8_t*)b, b_s, (T*)c + (int64_t)m0 * N, Mc, N, K)
      if (Mc <= 1) { CALL(1); } else if (Mc <= 2) { CALL(2); } else if (Mc <= 4) { CALL(4); } else { CALL(8); }
#undef CALL
    } else if (out_dtype == CB_F16) {
      using T = __half;
#define CALL(MT)                                                                              \
  cb::launch_k(gemv_softfp8_kernel<T, MT>, dim3(grid_for(N)), dim3(kWarps * 32), 0, st,                             \
      (const T*)a + (int64_t)m0 * K, (const uint8_t*)b, b_s, (T*)c + (int64_t)m0 * N, Mc, N, K)
      if (Mc <= 1) { CALL(1); } else if (Mc <= 2) { CALL(2); } else if (Mc <= 4) { CALL(4); } else { CALL(8); }
#undef CALL
    } else {
      return fail(-1, "soft_fp8_gemm: unsupported dtype %d", out_dtype);
    }
    ++launches;
  }
  CB_LAUNCHED(launches);
  return 0;
}

int simt_w8a8_gemm(void* out, const int8_t* a, const int8_t* b, const float* a_scales,
                   const float* b_scales, const void* bias, int M, int N, int K, cudaStream_t st) {
  CB_ARG(K % 16 == 0);
  int launches = 0;
  for (int m0 = 0; m0 < M; m0 += 16) {
    int Mc = M - m0 < 16 ? M - m0 : 16;
#define CALL(MT)                                                                                   \
  cb::launch_k(gemv_i8_kernel<MT>, dim3(grid_for(N)), dim3(kWarps * 32), 0, st, (__half*)out + (int64_t)m0 * N,          \
                                                          a + (int64_t)m0 * K, b, a_scales + m0,   \
                                                          b_scales, (const __half*)bias, Mc, N, K)
    DISPATCH_MT(Mc, CALL)
#undef CALL
    ++launches;
  }
  CB_LAUNCHED(launches);
  return 0;
}

}  // namespace cb

CB_DEFINE_TL_SETTER(gemv)
