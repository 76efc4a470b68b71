// Shared helpers for libchitu_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>
#include <utility>

#include "../../include/chitu_b200.h"

namespace cb {

int fail(int code, const char* fmt, ...);
void count_launch(int n = 1);

#define CB_ARG(cond)                                                                  \
  do {                                                                                \
    if (!(cond)) return cb::fail(-1, "%s: argument check failed: %s", __func__, #cond); \
  } while (0)

#define CB_LAUNCHED(n)                                                                        \
  do {                                                                                        \
    cudaError_t e__ = cudaGetLastError();                                                     \
    if (e__ != cudaSuccess)                                                                   \
      return cb::fail((int)e__, "%s: launch failed: %s", __func__, cudaGetErrorString(e__)); \
    cb::count_launch(n);                                                                      \
    if (cb::tl_enabled()) cb::tl_log_launch(__func__, n);                                     \
  } while (0)

#define CB_CUDA(call)                                                                       \
  do {                                                                                      \
    cudaError_t e__ = (call);                                                               \
    if (e__ != cudaSuccess)                                                                 \
      return cb::fail((int)e__, "%s: %s failed: %s", __func__, #call, cudaGetErrorString(e__)); \
  } while (0)

static inline int cdiv(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// ---- programmatic dependent launch (PDL) ----------------------------------------------------
// Every kernel of this library is launched with cudaLaunchAttributeProgrammaticStreamSerialization
// and starts with pdl_prologue(): `griddepcontrol.launch_dependents` lets the NEXT kernel of the
// stream be scheduled as soon as SM resources free up (its launch latency, barrier init,
// tensormap prefetch overlap this kernel's tail), `griddepcontrol.wait` blocks until
// the PREVIOUS kernel has completed and flushed — so no kernel touches global memory before its
// predecessor is done.  Inside CUDA graphs this becomes a programmatic dependency edge.
bool pdl_enabled();

// ---- in-graph timeline (dev tool, off by default) --------------------------------------------------------------
// chitu_b200_debug_timeline(buf, capacity) arms a device buffer; every kernel then records %globaltimer when the LAST
// thread of its first CTA has passed its dependency wait (tl_stamp(), called from pdl_prologue() and after the role-
// specific waits of the warp-specialised kernels).  The differences between successive stamps of one CUDA-graph replay
// are the per-kernel critical-path times INSIDE the graph (ncu serialises and times kernels cold).  Host side: the C
// entry name of every launch is logged in order (CB_LAUNCHED), so stamp i <-> entry i.  One pointer per translation
// unit (no -rdc): CB_DEFINE_TL_SETTER(name) in each .cu, chitu_b200_debug_timeline calls them all.
void tl_log_launch(const char* entry, int n);
bool tl_enabled();

#ifdef __CUDACC__
static __device__ unsigned long long* d_tl_buf = nullptr;    // [0] = count, [1] = capacity, [2..] = stamps
#define CB_DEFINE_TL_SETTER(NAME)                                                     \
  extern "C" int chitu_b200_tl_set_##NAME(unsigned long long* p) {                    \
    return (int)cudaMemcpyToSymbol(cb::d_tl_buf, &p, sizeof(p));                       \
  }
// Compiled in only with -DCB_TIMELINE (make TIMELINE=1 -> libchitu_b200_tl.so): the product library pays nothing.
__device__ __forceinline__ void tl_stamp() {
#ifdef CB_TIMELINE
  unsigned long long* b = d_tl_buf;
  if (b != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 &&
      threadIdx.x == blockDim.x - 1 && threadIdx.y == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    const unsigned long long i = atomicAdd(b, 1ull);
    if (i < b[1]) b[2 + i] = t;
  }
#endif
}
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_prologue() {
  pdl_launch_dependents();
  pdl_wait();
  tl_stamp();
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                            Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
#endif

// ---- push-mode all-reduce: descriptor handed to the producing kernels (comm.cu fills it) -------------------------
// A producer (row-parallel GEMM epilogue, expert combine) stores its bf16 partial [rows, ld] into EVERY rank's push area
// as 8-byte words {bf16 x[2k], bf16 x[2k+1], uint32 epoch} (k = (row * ld + col) / 2):
//   base[r] + (slot * world + rank) * ll_bytes + k * 8          epoch = *calls + 1,  slot = *calls & 1
// The word is its own arrival flag (an aligned 8-byte store lands whole): no fence, no counter, see comm.cu.
constexpr int kPushMaxWorld = 8;
struct PushDev {
  uint8_t* base[kPushMaxWorld];
  const uint32_t* calls;              // local: reduces completed so far
  int world, rank;
  int64_t ll_bytes;                   // bytes of one source's rows in word format (= 2 x the bf16 bytes)
};
int comm_push_desc(void* handle, void* out_desc);

#ifdef __CUDACC__
// byte offset of this rank's area inside every push buffer, for the reduce that is being produced
__device__ __forceinline__ int64_t push_area(const PushDev& d, uint32_t calls) {
  return ((int64_t)(calls & 1u) * d.world + d.rank) * d.ll_bytes;
}
// one word to every rank: word_off = byte offset inside the area (k * 8)
__device__ __forceinline__ void push_word(const PushDev& d, int64_t off, uint32_t two_bf16, uint32_t epoch) {
#pragma unroll 1
  for (int r = 0; r < d.world; ++r)
    asm volatile("st.volatile.global.v2.u32 [%0], {%1, %2};" ::"l"(d.base[r] + off), "r"(two_bf16), "r"(epoch) : "memory");
}
#endif

// ---- dtype helpers -----------------------------------------------------------------------
template <typename T> struct io;
template <> struct io<__nv_bfloat16> {
  static __device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  static __device__ __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};
template <> struct io<__half> {
  static __device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
  static __device__ __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
};
template <> struct io<float> {
  static __device__ __forceinline__ float to_f(float v) { return v; }
  static __device__ __forceinline__ float from_f(float v) { return v; }
};

// bf16x2 packed in a 32-bit word -> two floats (exact: bf16 is the top half of fp32).
__device__ __forceinline__ float bf16lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
__device__ __forceinline__ float2 unpack2(uint32_t u, const __nv_bfloat16*) {
  return make_float2(bf16lo(u), bf16hi(u));
}
__device__ __forceinline__ float2 unpack2(uint32_t u, const __half*) {
  return __half22float2(*reinterpret_cast<const __half2*>(&u));
}
__device__ __forceinline__ uint32_t pack2(float a, float b, const __nv_bfloat16*) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ uint32_t pack2(float a, float b, const __half*) {
  __half2 v = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

// fp8 e4m3 (two packed in 16 bits) -> float2, exact.
__device__ __forceinline__ float2 fp8x2_to_float2(uint16_t v) {
  __half2_raw h = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)v, __NV_E4M3);
  return __half22float2(*reinterpret_cast<__half2*>(&h));
}
__device__ __forceinline__ float fp8_to_float(uint8_t v) {
  __half_raw h = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)v, __NV_E4M3);
  return __half2float(*reinterpret_cast<__half*>(&h));
}
// float -> fp8 e4m3fn, round-to-nearest-even, saturate-to-finite (== Triton's cvt on GPU).
__device__ __forceinline__ uint8_t float_to_fp8(float v) {
  return (uint8_t)__nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E4M3);
}

// 128-bit streaming load that does not pollute L1 (weights / KV are read exactly once).
__device__ __forceinline__ uint4 ld_stream(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ uint2 ld_stream8(const void* p) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace cb
