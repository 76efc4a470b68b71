// Small HBM/latency-bound operators of the decode step: rotary, RMSNorm, SiLU*mul,
// activation quantisers (fp8 group / int8 per token), fp8 weight dequant, embedding, add, argmax.
#include "common.cuh"

using namespace cb;

// ============================================================================================
// rotary, interleaved pairs ("llama"): triton_kernels.py:101-190, host ops.py:178-237
//   o[2i]   = x[2i]*cos[i] - x[2i+1]*sin[i]
//   o[2i+1] = x[2i+1]*cos[i] + x[2i]*sin[i]        (fp32 math: bf16 * fp32 -> fp32, one rounding)
// ============================================================================================
template <typename T>
__global__ void rotary_interleaved_kernel(const T* __restrict__ q, const T* __restrict__ k,
                                          T* __restrict__ oq, T* __restrict__ ok,
                                          const float* __restrict__ cosp, const float* __restrict__ sinp,
                                          int hq, int hk, int rot, int64_t q_sb, int64_t q_sh,
                                          int64_t k_sb, int64_t k_sh, int64_t oq_sb, int64_t ok_sb) {
  cb::pdl_prologue();
  const int b = blockIdx.x;
  const int half = rot >> 1;
  const int total = (hq + hk) * half;
  for (int idx = threadIdx.x; idx < total; idx += blockDim.x) {
    int h = idx / half, i = idx - h * half;
    const T* src;
    T* dst;
    if (h < hq) {
      src = q + b * q_sb + h * q_sh;
      dst = oq + (int64_t)b * oq_sb + (int64_t)h * rot;
    } else {
      int hh = h - hq;
      src = k + b * k_sb + hh * k_sh;
      dst = ok + (int64_t)b * ok_sb + (int64_t)hh * rot;
    }
    float c = cosp[(int64_t)b * half + i], s = sinp[(int64_t)b * half + i];
    float x0 = io<T>::to_f(src[2 * i]), x1 = io<T>::to_f(src[2 * i + 1]);
    dst[2 * i] = io<T>::from_f(x0 * c - x1 * s);
    dst[2 * i + 1] = io<T>::from_f(x1 * c + x0 * s);
  }
}

// 16-byte variant for 2-byte dtypes: one thread rotates 4 adjacent pairs of one head (the scalar kernel above
// spent 8.7 us on [16, 40, 128] — ten serial 2-byte round trips per thread and an integer division each).
// Same arithmetic, same contraction: o0 = fma(x0, c, -(x1*s)), o1 = fma(x1, c, x0*s).
template <typename T>
__global__ void __launch_bounds__(128) rotary_interleaved_vec_kernel(
    const T* __restrict__ q, const T* __restrict__ k, T* __restrict__ oq, T* __restrict__ ok,
    const float* __restrict__ cosp, const float* __restrict__ sinp, int bs, int hq, int hk, int rot, int64_t q_sb,
    int64_t q_sh, int64_t k_sb, int64_t k_sh, int64_t oq_sb, int64_t ok_sb) {
  cb::pdl_prologue();
  const int vec_per_head = rot >> 3;
  const int per_tok = (hq + hk) * vec_per_head;
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= (int64_t)bs * per_tok) return;
  const int b = (int)(gid / per_tok);
  const int r = (int)(gid - (int64_t)b * per_tok);
  const int h = r / vec_per_head, j = r - h * vec_per_head;
  const T* src;
  T* dst;
  if (h < hq) {
    src = q + b * q_sb + h * q_sh;
    dst = oq + (int64_t)b * oq_sb + (int64_t)h * rot;
  } else {
    const int hh = h - hq;
    src = k + b * k_sb + hh * k_sh;
    dst = ok + (int64_t)b * ok_sb + (int64_t)hh * rot;
  }
  const int half = rot >> 1;
  const uint4 xv = *reinterpret_cast<const uint4*>(src + 8 * j);
  const float4 c4 = *reinterpret_cast<const float4*>(cosp + (int64_t)b * half + 4 * j);
  const float4 s4 = *reinterpret_cast<const float4*>(sinp + (int64_t)b * half + 4 * j);
  const uint32_t xw[4] = {xv.x, xv.y, xv.z, xv.w};
  const float cc[4] = {c4.x, c4.y, c4.z, c4.w}, ss[4] = {s4.x, s4.y, s4.z, s4.w};
  uint32_t ow[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const T* pr = reinterpret_cast<const T*>(&xw[i]);
    const float x0 = io<T>::to_f(pr[0]), x1 = io<T>::to_f(pr[1]);
    const float o0 = __fmaf_rn(x0, cc[i], -__fmul_rn(x1, ss[i]));
    const float o1 = __fmaf_rn(x1, cc[i], __fmul_rn(x0, ss[i]));
    T po[2] = {io<T>::from_f(o0), io<T>::from_f(o1)};
    ow[i] = *reinterpret_cast<const uint32_t*>(po);
  }
  *reinterpret_cast<uint4*>(dst + 8 * j) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int chitu_b200_rotary_interleaved(const void* q, const void* k, void* out_q, void* out_k,
                                             const float* cos, const float* sin, int bs, int hq,
                                             int hk, int rot_dim, int64_t q_sb, int64_t q_sh,
                                             int64_t k_sb, int64_t k_sh, int dtype, void* stream) {
  return chitu_b200_rotary_interleaved_strided(q, k, out_q, out_k, cos, sin, bs, hq, hk, rot_dim, q_sb, q_sh, k_sb,
                                               k_sh, (int64_t)hq * rot_dim, (int64_t)hk * rot_dim, dtype, stream);
}

extern "C" int chitu_b200_rotary_interleaved_strided(const void* q, const void* k, void* out_q, void* out_k,
                                                     const float* cos, const float* sin, int bs, int hq, int hk,
                                                     int rot_dim, int64_t q_sb, int64_t q_sh, int64_t k_sb,
                                                     int64_t k_sh, int64_t oq_sb, int64_t ok_sb, int dtype,
                                                     void* stream) {
  CB_ARG(q && k && out_q && out_k && cos && sin);
  CB_ARG(bs >= 0 && hq >= 0 && hk >= 0 && rot_dim > 0 && rot_dim % 2 == 0);
  if (bs == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  int total = (hq + hk) * rot_dim / 2;
  // 16-byte path: a thread rotates 4 pairs (one uint4 of 2-byte elements); needs 16 B aligned rows
  static const bool force_scalar = getenv("CHITU_B200_ROTARY_SCALAR") != nullptr;
  const bool vec_ok = !force_scalar && (dtype == CB_BF16 || dtype == CB_F16) && rot_dim % 8 == 0 &&
                      q_sb % 8 == 0 && q_sh % 8 == 0 && k_sb % 8 == 0 && k_sh % 8 == 0 && oq_sb % 8 == 0 &&
                      ok_sb % 8 == 0 && aligned16(q) && aligned16(k) && aligned16(out_q) && aligned16(out_k) &&
                      aligned16(cos) && aligned16(sin);
  if (vec_ok) {
    const int64_t nthreads = (int64_t)bs * (hq + hk) * (rot_dim / 8);
    const int blocks = (int)((nthreads + 127) / 128);
    if (dtype == CB_BF16)
      cb::launch_k(rotary_interleaved_vec_kernel<__nv_bfloat16>, dim3(blocks), dim3(128), 0, st,
                   (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (__nv_bfloat16*)out_q, (__nv_bfloat16*)out_k, cos, sin,
                   bs, hq, hk, rot_dim, q_sb, q_sh, k_sb, k_sh, oq_sb, ok_sb);
    else
      cb::launch_k(rotary_interleaved_vec_kernel<__half>, dim3(blocks), dim3(128), 0, st, (const __half*)q,
                   (const __half*)k, (__half*)out_q, (__half*)out_k, cos, sin, bs, hq, hk, rot_dim, q_sb, q_sh, k_sb,
                   k_sh, oq_sb, ok_sb);
    CB_LAUNCHED(1);
    return 0;
  }
  int threads = total >= 256 ? 256 : (total >= 128 ? 128 : 64);
  if (dtype == CB_BF16)
    cb::launch_k(rotary_interleaved_kernel<__nv_bfloat16>, dim3(bs), dim3(threads), 0, st, 
        (const __nv_bfloat16*)q, (const __nv_bfloat16*)k, (__nv_bfloat16*)out_q, (__nv_bfloat16*)out_k,
        cos, sin, hq, hk, rot_dim, q_sb, q_sh, k_sb, k_sh, oq_sb, ok_sb);
  else if (dtype == CB_F16)
    cb::launch_k(rotary_interleaved_kernel<__half>, dim3(bs), dim3(threads), 0, st, (const __half*)q, (const __half*)k,
                                                              (__half*)out_q, (__half*)out_k, cos, sin,
                                                              hq, hk, rot_dim, q_sb, q_sh, k_sb, k_sh, oq_sb, ok_sb);
  else if (dtype == CB_F32)
    cb::launch_k(rotary_interleaved_kernel<float>, dim3(bs), dim3(threads), 0, st, (const float*)q, (const float*)k,
                                                             (float*)out_q, (float*)out_k, cos, sin, hq,
                                                             hk, rot_dim, q_sb, q_sh, k_sb, k_sh, oq_sb, ok_sb);
  else
    return fail(-1, "rotary_interleaved: unsupported dtype %d", dtype);
  CB_LAUNCHED(1);
  return 0;
}

// rotary, half split ("hf-llama"): triton_kernels.py:51-98. Math is done in the io dtype's
// fp32 image and rounded once (Triton computes q0*cos0 - q1*sin0 in the tensor dtype; for
// bf16 inputs Triton promotes products to fp32 only for fp32 cos/sin, so parity here is
// tolerance-based, see tests).
template <typename T>
__global__ void rotary_half_kernel(const T* __restrict__ x, T* __restrict__ out,
                                   const T* __restrict__ cosp, const T* __restrict__ sinp, int heads,
                                   int head_dim, int64_t x_sb) {
  cb::pdl_prologue();
  const int b = blockIdx.x;
  const int half = head_dim >> 1;
  const int total = heads * half;
  for (int idx = threadIdx.x; idx < total; idx += blockDim.x) {
    int h = idx / half, i = idx - h * half;
    const T* src = x + (int64_t)b * x_sb + (int64_t)h * head_dim;
    T* dst = out + ((int64_t)b * heads + h) * head_dim;
    float c = io<T>::to_f(cosp[(int64_t)b * half + i]), s = io<T>::to_f(sinp[(int64_t)b * half + i]);
    float x0 = io<T>::to_f(src[i]), x1 = io<T>::to_f(src[i + half]);
    // emulate the reference's dtype-level rounding of each product before the add
    float p0 = io<T>::to_f(io<T>::from_f(x0 * c)), p1 = io<T>::to_f(io<T>::from_f(x1 * s));
    float p2 = io<T>::to_f(io<T>::from_f(x1 * c)), p3 = io<T>::to_f(io<T>::from_f(x0 * s));
    dst[i] = io<T>::from_f(p0 - p1);
    dst[i + half] = io<T>::from_f(p2 + p3);
  }
}

extern "C" int chitu_b200_rotary_half(const void* x, void* out, const void* cos, const void* sin,
                                      int bs, int heads, int head_dim, int dtype, void* stream) {
  return chitu_b200_rotary_half_strided(x, (int64_t)heads * head_dim, out, cos, sin, bs, heads, head_dim, dtype, stream);
}

// x rows [heads * head_dim] with batch stride x_sb elements (a q / k view of a merged qkv GEMM output); out dense.
extern "C" int chitu_b200_rotary_half_strided(const void* x, int64_t x_sb, void* out, const void* cos, const void* sin,
                                              int bs, int heads, int head_dim, int dtype, void* stream) {
  CB_ARG(x && out && cos && sin);
  CB_ARG(bs >= 0 && heads > 0 && head_dim > 0 && head_dim % 2 == 0 && x_sb >= (int64_t)heads * head_dim);
  if (bs == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  int threads = 256;
  if (dtype == CB_BF16)
    cb::launch_k(rotary_half_kernel<__nv_bfloat16>, dim3(bs), dim3(threads), 0, st, (const __nv_bfloat16*)x, (__nv_bfloat16*)out,
                 (const __nv_bfloat16*)cos, (const __nv_bfloat16*)sin, heads, head_dim, x_sb);
  else if (dtype == CB_F16)
    cb::launch_k(rotary_half_kernel<__half>, dim3(bs), dim3(threads), 0, st, (const __half*)x, (__half*)out, (const __half*)cos,
                 (const __half*)sin, heads, head_dim, x_sb);
  else if (dtype == CB_F32)
    cb::launch_k(rotary_half_kernel<float>, dim3(bs), dim3(threads), 0, st, (const float*)x, (float*)out, (const float*)cos,
                 (const float*)sin, heads, head_dim, x_sb);
  else
    return fail(-1, "rotary_half: unsupported dtype %d", dtype);
  CB_LAUNCHED(1);
  return 0;
}

// ============================================================================================
// RMSNorm (models/model.py:50-78): one CTA per row, fp32 math, single rounding.
// ============================================================================================
template <typename T>
__global__ void __launch_bounds__(256) rmsnorm_kernel(const T* __restrict__ x, const T* __restrict__ w,
                                                      T* __restrict__ y, int dim, float eps, int64_t x_stride,
                                                      int64_t y_stride) {
  cb::pdl_prologue();
  const int64_t row = blockIdx.x;
  const T* xr = x + row * x_stride;
  T* yr = y + row * y_stride;
  float ss = 0.f;
  for (int i = threadIdx.x; i < dim; i += 256) {
    float v = io<T>::to_f(xr[i]);
    ss += v * v;
  }
  __shared__ float red[8];
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += red[i];
  const float r = rsqrtf(tot / (float)dim + eps);
  for (int i = threadIdx.x; i < dim; i += 256)
    yr[i] = io<T>::from_f(io<T>::to_f(xr[i]) * r * io<T>::to_f(w[i]));
}

extern "C" int chitu_b200_rmsnorm(const void* x, const void* w, void* y, int rows, int dim, float eps,
                                  int dtype, void* stream) {
  return chitu_b200_rmsnorm_strided(x, w, y, rows, dim, dim, dim, eps, dtype, stream);
}

extern "C" int chitu_b200_rmsnorm_strided(const void* x, const void* w, void* y, int rows, int dim,
                                          int64_t x_stride, int64_t y_stride, float eps, int dtype,
                                          void* stream) {
  CB_ARG(x && w && y && rows >= 0 && dim > 0 && x_stride >= dim && y_stride >= dim);
  if (rows == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == CB_BF16)
    cb::launch_k(rmsnorm_kernel<__nv_bfloat16>, dim3(rows), dim3(256), 0, st, (const __nv_bfloat16*)x, (const __nv_bfloat16*)w,
                                                        (__nv_bfloat16*)y, dim, eps, x_stride, y_stride);
  else if (dtype == CB_F16)
    cb::launch_k(rmsnorm_kernel<__half>, dim3(rows), dim3(256), 0, st, (const __half*)x, (const __half*)w, (__half*)y, dim, eps, x_stride, y_stride);
  else if (dtype == CB_F32)
    cb::launch_k(rmsnorm_kernel<float>, dim3(rows), dim3(256), 0, st, (const float*)x, (const float*)w, (float*)y, dim, eps, x_stride, y_stride);
  else
    return fail(-1, "rmsnorm: unsupported dtype %d", dtype);
  CB_LAUNCHED(1);
  return 0;
}

// ============================================================================================
// Fused RMSNorm (+ act_quant_deepseek_v3): one CTA per row, the row is read ONCE with 8-byte loads and
// kept in registers; y (bf16, optional) and / or the fp8 payload + per-128 scales are produced from the
// bf16-rounded normalised values, i.e. exactly rmsnorm -> act_quant (ops.py:329-353) without the round
// trip through HBM and without the second launch.  dim % 128 == 0, dim <= 8192.
// ============================================================================================
__global__ void __launch_bounds__(256) rmsnorm_quant_kernel(const __nv_bfloat16* __restrict__ x,
                                                            const __nv_bfloat16* __restrict__ w,
                                                            __nv_bfloat16* __restrict__ y, uint8_t* __restrict__ q,
                                                            float* __restrict__ qs, int dim, float eps,
                                                            int64_t x_stride, int64_t y_stride) {
  cb::pdl_prologue();
  constexpr int kMaxIt = 8;                        // 8 x (256 threads x 4 elems) = 8192
  const int64_t row = blockIdx.x;
  const __nv_bfloat16* xr = x + row * x_stride;
  const int lane = threadIdx.x & 31;
  const int nit = (dim + 1023) / 1024;
  float v[kMaxIt][4];
  uint2 wreg[kMaxIt];
  float ss = 0.f;
#pragma unroll
  for (int it = 0; it < kMaxIt; ++it) {
    const int e = it * 1024 + threadIdx.x * 4;
    wreg[it] = make_uint2(0, 0);
    if (it < nit && e < dim) {
      wreg[it] = *reinterpret_cast<const uint2*>(w + e);        // issued together with the x loads
      const uint2 raw = *reinterpret_cast<const uint2*>(xr + e);
      v[it][0] = bf16lo(raw.x); v[it][1] = bf16hi(raw.x); v[it][2] = bf16lo(raw.y); v[it][3] = bf16hi(raw.y);
      ss += v[it][0] * v[it][0] + v[it][1] * v[it][1] + v[it][2] * v[it][2] + v[it][3] * v[it][3];
    } else {
      v[it][0] = v[it][1] = v[it][2] = v[it][3] = 0.f;
    }
  }
  __shared__ float red[8];
  ss = warp_sum(ss);
  if (lane == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += red[i];
  const float r = rsqrtf(tot / (float)dim + eps);
#pragma unroll
  for (int it = 0; it < kMaxIt; ++it) {
    const int e = it * 1024 + threadIdx.x * 4;
    if (it < nit && e < dim) {                      // warp-uniform: dim % 128 == 0
      const uint2 wr = wreg[it];
      float o[4];
      o[0] = __bfloat162float(__float2bfloat16_rn(v[it][0] * r * bf16lo(wr.x)));
      o[1] = __bfloat162float(__float2bfloat16_rn(v[it][1] * r * bf16hi(wr.x)));
      o[2] = __bfloat162float(__float2bfloat16_rn(v[it][2] * r * bf16lo(wr.y)));
      o[3] = __bfloat162float(__float2bfloat16_rn(v[it][3] * r * bf16hi(wr.y)));
      if (y) {
        const __nv_bfloat16* tag = nullptr;
        *reinterpret_cast<uint2*>(y + row * y_stride + e) = make_uint2(pack2(o[0], o[1], tag), pack2(o[2], o[3], tag));
      }
      if (q) {                                      // a warp covers exactly one 128-element group
        float amax = fmaxf(fmaxf(fabsf(o[0]), fabsf(o[1])), fmaxf(fabsf(o[2]), fabsf(o[3])));
        amax = warp_max(amax);
        const float sc = __fdiv_rn(amax, 448.0f);
        uint32_t packed = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) packed |= (uint32_t)float_to_fp8(__fdiv_rn(o[i], sc)) << (8 * i);
        *reinterpret_cast<uint32_t*>(q + row * dim + e) = packed;
        if (lane == 0) qs[row * (dim / 128) + (e >> 7)] = sc;
      }
    }
  }
}

extern "C" int chitu_b200_rmsnorm_quant_fp8(const void* x, const void* w, void* y, void* q, float* q_scales,
                                            int rows, int dim, int64_t x_stride, int64_t y_stride, float eps,
                                            void* stream) {
  CB_ARG(x && w && (y || q) && rows >= 0 && dim > 0 && dim % 128 == 0 && dim <= 8192);
  CB_ARG((q == nullptr) == (q_scales == nullptr));
  CB_ARG(x_stride >= dim && x_stride % 4 == 0 && (y == nullptr || (y_stride >= dim && y_stride % 4 == 0)));
  if (rows == 0) return 0;
  cb::launch_k(rmsnorm_quant_kernel, dim3(rows), dim3(256), 0, (cudaStream_t)stream, (const __nv_bfloat16*)x,
               (const __nv_bfloat16*)w, (__nv_bfloat16*)y, (uint8_t*)q, q_scales, dim, eps, x_stride, y_stride);
  CB_LAUNCHED(1);
  return 0;
}

// ============================================================================================
// Fused SiluAndMul + act_quant (dense FFN: linear_deepseek_v3 of w2 quantises silu(w1 x)*w3 x,
// model_deepseek_v3.py:755-771): x [rows, 2F] bf16 -> fp8 [rows, F] + scales [rows, F/128] (mode 0: no eps)
// ============================================================================================
__global__ void silu_mul_quant_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q,
                                      float* __restrict__ qs, int64_t rows, int F) {
  cb::pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int groups = F / 128;
  const int64_t gidx = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (gidx >= rows * groups) return;
  const int64_t r = gidx / groups;
  const int gk = (int)(gidx - r * groups);
  const __nv_bfloat16* row = x + r * 2 * F;
  const uint2 gr = *reinterpret_cast<const uint2*>(row + gk * 128 + lane * 4);
  const uint2 ur = *reinterpret_cast<const uint2*>(row + F + gk * 128 + lane * 4);
  const float gv[4] = {bf16lo(gr.x), bf16hi(gr.x), bf16lo(gr.y), bf16hi(gr.y)};
  const float uv[4] = {bf16lo(ur.x), bf16hi(ur.x), bf16lo(ur.y), bf16hi(ur.y)};
  float v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float sl = __bfloat162float(__float2bfloat16_rn(gv[i] / (1.f + expf(-gv[i]))));
    v[i] = __bfloat162float(__float2bfloat16_rn(sl * uv[i]));
  }
  float amax = fmaxf(fmaxf(fabsf(v[0]), fabsf(v[1])), fmaxf(fabsf(v[2]), fabsf(v[3])));
  amax = warp_max(amax);
  const float sc = __fdiv_rn(amax, 448.0f);
  uint32_t packed = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) packed |= (uint32_t)float_to_fp8(__fdiv_rn(v[i], sc)) << (8 * i);
  *reinterpret_cast<uint32_t*>(q + r * F + gk * 128 + lane * 4) = packed;
  if (lane == 0) qs[r * groups + gk] = sc;
}

extern "C" int chitu_b200_silu_mul_quant_fp8(const void* x, void* q, float* q_scales, int64_t rows, int F,
                                             void* stream) {
  CB_ARG(x && q && q_scales && rows >= 0 && F > 0 && F % 128 == 0);
  if (rows == 0) return 0;
  const int64_t ng = rows * (F / 128);
  cb::launch_k(silu_mul_quant_kernel, dim3((unsigned)((ng + 7) / 8)), dim3(256), 0, (cudaStream_t)stream,
               (const __nv_bfloat16*)x, (uint8_t*)q, q_scales, rows, F);
  CB_LAUNCHED(1);
  return 0;
}

// ============================================================================================
// SiluAndMul (fused_moe.py:24-39): F.silu(x[:, :d]) * x[:, d:].  F.silu on bf16 rounds its
// result to bf16 before the multiply; reproduced.
// ============================================================================================
template <typename T>
__global__ void silu_and_mul_kernel(const T* __restrict__ x, T* __restrict__ out, int64_t rows, int d) {
  cb::pdl_prologue();
  int64_t n = rows * d;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i / d;
    int c = (int)(i - r * d);
    float g = io<T>::to_f(x[r * 2 * d + c]);
    float u = io<T>::to_f(x[r * 2 * d + d + c]);
    float s = io<T>::to_f(io<T>::from_f(g / (1.f + expf(-g))));
    out[i] = io<T>::from_f(s * u);
  }
}

extern "C" int chitu_b200_silu_and_mul(const void* x, void* out, int64_t rows, int d, int dtype,
                                       void* stream) {
  CB_ARG(x && out && rows >= 0 && d > 0);
  if (rows == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  int64_t n = rows * d;
  int blocks = (int)((n + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  if (dtype == CB_BF16)
    cb::launch_k(silu_and_mul_kernel<__nv_bfloat16>, dim3(blocks), dim3(256), 0, st, (const __nv_bfloat16*)x, (__nv_bfloat16*)out, rows, d);
  else if (dtype == CB_F16)
    cb::launch_k(silu_and_mul_kernel<__half>, dim3(blocks), dim3(256), 0, st, (const __half*)x, (__half*)out, rows, d);
  else if (dtype == CB_F32)
    cb::launch_k(silu_and_mul_kernel<float>, dim3(blocks), dim3(256), 0, st, (const float*)x, (float*)out, rows, d);
  else
    return fail(-1, "silu_and_mul: unsupported dtype %d", dtype);
  CB_LAUNCHED(1);
  return 0;
}

// ============================================================================================
// fp8 group quantisers.  One warp per (row, group); group == 128 -> 4 elements per lane.
//   mode 0: act_quant_deepseek_v3  (triton_kernels.py:193-214)  s = max|x| / 448 ; y = fp8(x / s)
//   mode 1: per_token_group_quant_fp8 (fused_moe.py:667-710)    s = max(max|x|, eps) / 448 ;
//                                                               y = fp8(clamp(x / s, -448, 448))
// The division x / s is an IEEE fp32 division in both (Triton `/` on fp32 is div.full? no:
// Triton lowers fp32 `/` to div.full.f32 — ~2 ulp — unless IEEE rounding is requested; the CPU
// interpreter and this kernel use correctly-rounded division).
// ============================================================================================
template <typename T>
__global__ void act_quant_fp8_kernel(const T* __restrict__ x, uint8_t* __restrict__ y,
                                     float* __restrict__ s, int64_t n_groups, int group, int mode,
                                     float eps) {
  cb::pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int64_t g = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (g >= n_groups) return;
  const T* xg = x + g * group;
  uint8_t* yg = y + g * group;
  float amax = 0.f;
  for (int i = lane; i < group; i += 32) amax = fmaxf(amax, fabsf(io<T>::to_f(xg[i])));
  amax = warp_max(amax);
  if (mode == 1) amax = fmaxf(amax, eps);
  const float sc = __fdiv_rn(amax, 448.0f);
  for (int i = lane; i < group; i += 32) {
    float v = __fdiv_rn(io<T>::to_f(xg[i]), sc);
    if (mode == 1) v = fminf(fmaxf(v, -448.f), 448.f);
    yg[i] = float_to_fp8(v);
  }
  if (lane == 0) s[g] = sc;
}

extern "C" int chitu_b200_act_quant_fp8(const void* x, void* y, float* s, int64_t rows, int K,
                                        int group, int mode, float eps, int dtype, void* stream) {
  CB_ARG(x && y && s && rows >= 0 && K > 0 && group > 0 && K % group == 0);
  CB_ARG(mode == 0 || mode == 1);
  if (rows == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  int64_t n_groups = rows * (K / group);
  int blocks = (int)((n_groups + 7) / 8);
  if (dtype == CB_BF16)
    cb::launch_k(act_quant_fp8_kernel<__nv_bfloat16>, dim3(blocks), dim3(256), 0, st, (const __nv_bfloat16*)x, (uint8_t*)y, s, n_groups, group, mode, eps);
  else if (dtype == CB_F16)
    cb::launch_k(act_quant_fp8_kernel<__half>, dim3(blocks), dim3(256), 0, st, (const __half*)x, (uint8_t*)y, s, n_groups, group, mode, eps);
  else if (dtype == CB_F32)
    cb::launch_k(act_quant_fp8_kernel<float>, dim3(blocks), dim3(256), 0, st, (const float*)x, (uint8_t*)y, s, n_groups, group, mode, eps);
  else
    return fail(-1, "act_quant_fp8: unsupported dtype %d", dtype);
  CB_LAUNCHED(1);
  return 0;
}

// ============================================================================================
// quant_act (quantize/w8a8.py:18-26): scales = clamp(max|x| as fp32, 1e-5) / 127 ;
// q = int8(round_half_even(x / scale)).  `act.div(scales)` on an fp16 tensor with an fp32
// scale promotes to fp32 (torch type promotion: both are dim>=1 tensors) -> fp32 division.
// ============================================================================================
template <typename T>
__global__ void __launch_bounds__(256) quant_act_int8_kernel(const T* __restrict__ x,
                                                             int8_t* __restrict__ q,
                                                             float* __restrict__ scales, int K) {
  cb::pdl_prologue();
  const int64_t row = blockIdx.x;
  const T* xr = x + row * K;
  float amax = 0.f;
  for (int i = threadIdx.x; i < K; i += 256) amax = fmaxf(amax, fabsf(io<T>::to_f(xr[i])));
  __shared__ float red[8];
  amax = warp_max(amax);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
  __syncthreads();
  float m = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) m = fmaxf(m, red[i]);
  const float sc = __fdiv_rn(fmaxf(m, 1e-5f), 127.0f);
  for (int i = threadIdx.x; i < K; i += 256) {
    float v = rintf(__fdiv_rn(io<T>::to_f(xr[i]), sc));
    q[row * K + i] = (int8_t)(int)v;
  }
  if (threadIdx.x == 0) scales[row] = sc;
}

extern "C" int chitu_b200_quant_act_int8(const void* x, int8_t* q, float* scales, int64_t rows, int K,
                                         int dtype, void* stream) {
  CB_ARG(x && q && scales && rows >= 0 && K > 0);
  if (rows == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == CB_F16)
    cb::launch_k(quant_act_int8_kernel<__half>, dim3((unsigned)rows), dim3(256), 0, st, (const __half*)x, q, scales, K);
  else if (dtype == CB_BF16)
    cb::launch_k(quant_act_int8_kernel<__nv_bfloat16>, dim3((unsigned)rows), dim3(256), 0, st, (const __nv_bfloat16*)x, q, scales, K);
  else if (dtype == CB_F32)
    cb::launch_k(quant_act_int8_kernel<float>, dim3((unsigned)rows), dim3(256), 0, st, (const float*)x, q, scales, K);
  else
    return fail(-1, "quant_act_int8: unsupported dtype %d", dtype);
  CB_LAUNCHED(1);
  return 0;
}

// ============================================================================================
// fp8 weight dequant (ops.py:356-449, triton_kernels.py:217-287) -> bf16
// ============================================================================================
__global__ void weight_dequant_fp8_kernel(const uint8_t* __restrict__ x, const float* __restrict__ s,
                                          __nv_bfloat16* __restrict__ y, int M, int N, int block,
                                          int soft) {
  cb::pdl_prologue();
  const int b = blockIdx.z;
  const int m = blockIdx.y;
  const int sn = (N + block - 1) / block, sm = (M + block - 1) / block;
  const uint8_t* xr = x + ((int64_t)b * M + m) * N;
  __nv_bfloat16* yr = y + ((int64_t)b * M + m) * N;
  const float* sr = s + ((int64_t)b * sm + m / block) * sn;
  for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < N; n += gridDim.x * blockDim.x) {
    float sc = sr[n / block];
    float v;
    if (soft) {
      uint32_t u = xr[n];
      float f = __uint_as_float(((u & 0x80u) << 24) | ((u & 0x7fu) << 20));
      v = f * (sc * __uint_as_float(0x7B800000u));
    } else {
      v = fp8_to_float(xr[n]) * sc;
    }
    yr[n] = __float2bfloat16_rn(v);
  }
}

extern "C" int chitu_b200_weight_dequant_fp8(const void* x, const float* s, void* y, int B, int M, int N,
                                             int block, int soft, void* stream) {
  CB_ARG(x && s && y && B > 0 && M > 0 && N > 0 && block > 0);
  CB_ARG(M <= 65535 && B <= 65535);
  dim3 grid(cdiv(N, 256) > 64 ? 64 : cdiv(N, 256), M, B);
  cb::launch_k(weight_dequant_fp8_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, (const uint8_t*)x, s, (__nv_bfloat16*)y, M, N, block, soft);
  CB_LAUNCHED(1);
  return 0;
}

// ============================================================================================
// embedding / add / argmax  (decode-engine helpers, SURVEY §8f n3)
// ============================================================================================
template <typename T>
__global__ void embedding_kernel(const int64_t* __restrict__ ids, const T* __restrict__ table,
                                 T* __restrict__ out, int dim, int64_t vocab_start, int64_t rows) {
  cb::pdl_prologue();
  const int t = blockIdx.x;
  int64_t id = ids[t] - vocab_start;
  bool ok = id >= 0 && id < rows;
  const uint4* src = reinterpret_cast<const uint4*>(table + (ok ? id : 0) * dim);
  uint4* dst = reinterpret_cast<uint4*>(out + (int64_t)t * dim);
  const int n16 = dim * (int)sizeof(T) / 16;
  for (int i = threadIdx.x; i < n16; i += blockDim.x) dst[i] = ok ? src[i] : make_uint4(0, 0, 0, 0);
}

extern "C" int chitu_b200_embedding(const int64_t* ids, const void* table, void* out, int T, int dim,
                                    int64_t vocab_start, int64_t rows, int dtype, void* stream) {
  CB_ARG(ids && table && out && T >= 0 && dim > 0 && rows > 0);
  CB_ARG(dtype == CB_BF16 || dtype == CB_F16);
  CB_ARG((dim * 2) % 16 == 0);
  if (T == 0) return 0;
  cb::launch_k(embedding_kernel<uint16_t>, dim3(T), dim3(128), 0, (cudaStream_t)stream, ids, (const uint16_t*)table, (uint16_t*)out, dim, vocab_start, rows);
  CB_LAUNCHED(1);
  return 0;
}

template <typename T>
__global__ void add_kernel(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ y, int64_t n) {
  cb::pdl_prologue();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = io<T>::from_f(io<T>::to_f(a[i]) + io<T>::to_f(b[i]));
}

extern "C" int chitu_b200_add(const void* a, const void* b, void* y, int64_t n, int dtype, void* stream) {
  CB_ARG(a && b && y && n >= 0);
  if (n == 0) return 0;
  int blocks = (int)((n + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == CB_BF16)
    cb::launch_k(add_kernel<__nv_bfloat16>, dim3(blocks), dim3(256), 0, st, (const __nv_bfloat16*)a, (const __nv_bfloat16*)b, (__nv_bfloat16*)y, n);
  else if (dtype == CB_F16)
    cb::launch_k(add_kernel<__half>, dim3(blocks), dim3(256), 0, st, (const __half*)a, (const __half*)b, (__half*)y, n);
  else
    return fail(-1, "add: unsupported dtype %d", dtype);
  CB_LAUNCHED(1);
  return 0;
}

template <typename T>
__global__ void __launch_bounds__(1024) argmax_kernel(const T* __restrict__ logits, int64_t* __restrict__ out, int64_t V) {
  cb::pdl_prologue();
  const T* row = logits + (int64_t)blockIdx.x * V;
  float best = -INFINITY;
  int64_t bi = 0;
  for (int64_t i = threadIdx.x; i < V; i += 1024) {
    float v = io<T>::to_f(row[i]);
    if (v > best) { best = v; bi = i; }   // ascending i per thread -> first max wins
  }
  __shared__ float sv[1024];
  __shared__ int64_t si[1024];
  sv[threadIdx.x] = best;
  si[threadIdx.x] = bi;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      float v2 = sv[threadIdx.x + o];
      int64_t i2 = si[threadIdx.x + o];
      if (v2 > sv[threadIdx.x] || (v2 == sv[threadIdx.x] && i2 < si[threadIdx.x])) {
        sv[threadIdx.x] = v2;
        si[threadIdx.x] = i2;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) out[blockIdx.x] = si[0];
}

extern "C" int chitu_b200_argmax(const void* logits, int64_t* out, int T, int64_t V, int dtype, void* stream) {
  CB_ARG(logits && out && T >= 0 && V > 0);
  if (T == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == CB_F32)
    cb::launch_k(argmax_kernel<float>, dim3(T), dim3(1024), 0, st, (const float*)logits, out, V);
  else if (dtype == CB_BF16)
    cb::launch_k(argmax_kernel<__nv_bfloat16>, dim3(T), dim3(1024), 0, st, (const __nv_bfloat16*)logits, out, V);
  else
    return fail(-1, "argmax: unsupported dtype %d", dtype);
  CB_LAUNCHED(1);
  return 0;
}

CB_DEFINE_TL_SETTER(elementwise)
