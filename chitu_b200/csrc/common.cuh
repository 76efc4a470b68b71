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
#include <type_traits>
#include <utility>

#include "../../include/chitu_b200.h"

namespace cb {

int fail(int code, const char* fmt, ...);
void count_launch(int n = 1);

// The _AS forms report under `name` (a helper shared by several C entries passes the name of the entry it serves).
#define CB_ARG_AS(name, cond)                                                                \
  do {                                                                                       \
    if (!(cond)) return cb::fail(-1, "%s: argument check failed: %s", (name), #cond);        \
  } while (0)
#define CB_ARG(cond) CB_ARG_AS(__func__, cond)

#define CB_LAUNCHED_AS(name, n)                                                               \
  do {                                                                                        \
    cudaError_t e__ = cudaGetLastError();                                                     \
    if (e__ != cudaSuccess)                                                                   \
      return cb::fail((int)e__, "%s: launch failed: %s", (name), cudaGetErrorString(e__));   \
    cb::count_launch(n);                                                                      \
    if (cb::tl_enabled()) cb::tl_log_launch((name), n);                                       \
  } while (0)
#define CB_LAUNCHED(n) CB_LAUNCHED_AS(__func__, n)

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
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// launch_k of kernel K with `smem` bytes of dynamic shared memory, after raising K's limit once: with Bound = 0 to
// `smem` on K's first launch (every launch of K asks the same), else to Bound, an upper bound of every launch of K, on
// the first launch above the 48 KB default (raising it up front measured slower on the DeepSeek-R1 MoE step).
// The flag is keyed on K itself (two instances with one signature get one each), set by a thread-safe static
// initializer, and keeps the outcome: a failed limit, and a launch above Bound, are reported under `name` by every call.
// Launch errors are left to CB_LAUNCHED.
template <auto K, int Bound = 0, typename... Args>
inline int launch_smem(const char* name, dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  if (Bound == 0 || smem > 48 * 1024) {
    static const cudaError_t limit =
        cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, Bound ? Bound : (int)smem);
    if (limit != cudaSuccess)
      return fail((int)limit, "%s: cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed: %s", name,
                  cudaGetErrorString(limit));
    if (Bound && smem > (size_t)Bound)
      return fail((int)cudaErrorInvalidValue, "%s: %zu bytes of dynamic shared memory exceed %d", name, smem, Bound);
  }
  launch_k(K, grid, block, smem, st, std::forward<Args>(args)...);
  return 0;
}

// The element type of each dtype code a kernel is built for.
template <int Code> struct dtype_of;
template <> struct dtype_of<CB_BF16> { using type = __nv_bfloat16; };
template <> struct dtype_of<CB_F16> { using type = __half; };
template <> struct dtype_of<CB_F32> { using type = float; };

// f(T{}) for the element type T of `dtype` when it is one of Codes, returning f's status; any other code is refused
// under `entry` before f runs.
template <int... Codes, typename F>
inline int dispatch_dtype(const char* entry, int dtype, F&& f) {
  int rc = 0;
  if (((dtype == Codes && (rc = f(typename dtype_of<Codes>::type{}), true)) || ...)) return rc;
  return fail(-1, "%s: unsupported dtype %d", entry, dtype);
}

// f(T{}) for the io type T of `dtype` (CB_BF16, else fp16); returns f's result.
template <typename F>
inline auto dispatch_io(int dtype, F&& f) {
  return dtype == CB_BF16 ? f(dtype_of<CB_BF16>::type{}) : f(dtype_of<CB_F16>::type{});
}
// f(T{}, std::integral_constant<int, G>{}) for the io type of `dtype` and G = 1, 2, 4, else 8; returns f's status.
template <typename F>
inline int dispatch_io_g(int dtype, int G, F&& f) {
  return dispatch_io(dtype, [&](auto t) {
    switch (G) {
      case 1: return f(t, std::integral_constant<int, 1>{});
      case 2: return f(t, std::integral_constant<int, 2>{});
      case 4: return f(t, std::integral_constant<int, 4>{});
      default: return f(t, std::integral_constant<int, 8>{});
    }
  });
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

// ---- paged append (core.cu): new rows into one or two paged caches, for the append, scatter and paged prefill entries
// Fixed length (cu_seqlens == NULL, rows = sq): row i of request b (i < sq, b < B) comes from src + b * src_sb +
// i * src_st (bytes).  Ragged (rows = total_rows): row i of request b (i < cu_seqlens[b + 1] - cu_seqlens[b]) comes
// from src + (cu_seqlens[b] + i) * src_st; src_sb is unused.  Either goes to position p = seqlens[b] + i (seqlens ==
// NULL: p = i): cache row block_table[b, p / index_div] * page_size + p % index_div.  index_div is page_size for true
// page indexing and 64 for the reference's append (triton_kernels.py:38,42).  c1.cache == NULL: one cache only.
// One PDL launch; the caller counts it.
struct PagedAppend {
  void* cache;
  const void* src;
  int64_t src_sb, src_st;
};
void launch_paged_append(PagedAppend c0, PagedAppend c1, int64_t row_bytes, const int32_t* seqlens,
                         const int32_t* cu_seqlens, const int32_t* block_table, int bt_stride, int B, int rows,
                         int page_size, int index_div, cudaStream_t st);
// The same copy into contiguous caches: position p of request b is cache row b * rows_sb + p, and rows with
// p >= cache_rows are skipped.
void launch_contiguous_append(PagedAppend c0, PagedAppend c1, int64_t row_bytes, const int32_t* seqlens,
                              const int32_t* cu_seqlens, int64_t rows_sb, int cache_rows, int B, int rows,
                              cudaStream_t st);
// The paged append (true page indexing) into one or two e4m3 caches (c1.cache == NULL: one): rows of n io elements
// (dtype CB_BF16 | CB_F16, n % 8 == 0, 16-byte aligned sources and strides) stored as e4m3 with io2_to_e4m3x2's
// rounding.
void launch_paged_append_e4m3(PagedAppend c0, PagedAppend c1, int n, int dtype, const int32_t* seqlens,
                              const int32_t* cu_seqlens, const int32_t* block_table, int bt_stride, int B, int rows,
                              int page_size, cudaStream_t st);

// ---- absorbed MLA over the paged latent cache (mla_tc.cu, mla_prefill.cu) ---------------------------------------------
// The arguments of chitu_b200_mla_decode / chitu_b200_mla_paged_prefill over a bf16 cache, or (e4m3) over a cache of
// e4m3 bytes with the store and read rules of chitu_b200_mla_attn_fp8kv.  Argument checks and launches report under
// `entry`, the other refusals under `tag`.
int mla_decode(const char* entry, const char* tag, bool e4m3, const void* q_nope, const void* q_pe, void* kv_cache,
               const void* new_kv, const int32_t* seqlens_excl, const int32_t* block_table, int bt_stride, int B, int H,
               int C, int R, int page_size, int num_blocks, int max_seqlen_hint, float softmax_scale, void* out,
               void* workspace, int64_t workspace_bytes, cudaStream_t st);
int mla_paged_prefill(const char* entry, const char* tag, bool e4m3, const void* q_nope, const void* q_pe,
                      void* kv_cache, const void* new_kv, const int32_t* seqlens_excl, const int32_t* block_table,
                      int bt_stride, int B, int sq, int H, int C, int R, int page_size, int num_blocks,
                      int max_seqlen_hint, int causal, float softmax_scale, void* out, void* workspace,
                      int64_t workspace_bytes, cudaStream_t st);

// ---- GQA attention over the KV cache (attention.cu, gqa_prefill.cu) -------------------------------------------------
// The cache layouts of the GQA entries: paged in the io dtype, contiguous [Bc, cache_rows, Hkv, D] (request b from row
// b * rows_sb, in rows of Hkv * D), paged in e4m3.
enum class KvLayout { kPaged, kContiguous, kPagedE4m3 };

// The argument checks every GQA entry shares, reported under `entry`: the operands, k_new and v_new given together,
// bf16 / fp16, 16-byte aligned bases and 8-element k / v batch strides (token strides too with `token_strides`), as
// the kernels stage q and the new rows 16 bytes at a time.
inline int check_gqa_operands(const char* entry, const void* q, const void* k_cache, const void* v_cache,
                              const int32_t* cache_seqlens, const void* out, const void* k_new, const void* v_new,
                              int64_t k_new_sb, int64_t k_new_st, int64_t v_new_sb, int64_t v_new_st,
                              bool token_strides, int dtype) {
  CB_ARG_AS(entry, q && k_cache && v_cache && cache_seqlens && out);
  CB_ARG_AS(entry, (k_new == nullptr) == (v_new == nullptr));
  CB_ARG_AS(entry, dtype == CB_BF16 || dtype == CB_F16);
  CB_ARG_AS(entry, ((uintptr_t)q | (uintptr_t)k_cache | (uintptr_t)v_cache | (uintptr_t)out | (uintptr_t)k_new |
                    (uintptr_t)v_new) % 16 == 0);
  CB_ARG_AS(entry, k_new == nullptr || (k_new_sb % 8 == 0 && v_new_sb % 8 == 0 &&
                                        (!token_strides || (k_new_st % 8 == 0 && v_new_st % 8 == 0))));
  return 0;
}

// The multi-token kernel of gqa_prefill.cu over any layout, for arguments the calling entry has checked (B > 0):
// launches the append (with k_new), the attention and, with a split, the merge, and logs them as `name`; refusals
// name `entry`.  block_table, bt_stride, page_size and num_blocks describe a paged cache, rows_sb and cache_rows a
// contiguous one.
int gqa_prefill(const char* entry, const char* name, KvLayout layout, const void* q, void* k_cache, void* v_cache,
                const void* k_new, const void* v_new, int64_t k_new_sb, int64_t k_new_st, int64_t v_new_sb,
                int64_t v_new_st, const int32_t* cache_seqlens, const int32_t* block_table, int bt_stride,
                int page_size, int num_blocks, int64_t rows_sb, int cache_rows, int B, int sq, int Hq, int Hkv,
                int max_len, int causal, float softmax_scale, void* out, void* workspace, int64_t workspace_bytes,
                int dtype, cudaStream_t st);

#ifdef __CUDACC__
// byte offset of source `src`'s words inside a push buffer of `world` sources, for the reduce after `calls`
__device__ __forceinline__ int64_t push_area(uint32_t calls, int world, int src, int64_t ll_bytes) {
  return ((int64_t)(calls & 1u) * world + src) * ll_bytes;
}
// byte offset of this rank's area inside every push buffer, for the reduce that is being produced
__device__ __forceinline__ int64_t push_area(const PushDev& d, uint32_t calls) {
  return push_area(calls, d.world, d.rank, d.ll_bytes);
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

// ---- e4m3 KV cache (chitu_b200_gqa_paged_attn_fp8kv) -------------------------------------------------------------
// Store: an io pair (element 0 in the low half) -> two e4m3 bytes (element 0 in the low byte), cvt.rn.satfinite:
// nearest even, clamped to +-448, NaN stays NaN (torch: x.float().clamp(-448, 448).to(float8_e4m3fn)).
template <typename T>
__device__ __forceinline__ uint32_t io2_to_e4m3x2(uint32_t u) {
  return (uint32_t)__nv_cvt_float2_to_fp8x2(unpack2(u, (const T*)nullptr), __NV_SATFINITE, __NV_E4M3);
}
// Read: four e4m3 bytes (element k in byte k) -> io pairs lo = (0, 1), hi = (2, 3), exact (every e4m3 value is a
// bf16 and an fp16 value).  fp16: the hardware conversion.  bf16: the byte's exponent and mantissa placed in a bf16
// whose exponent is 127 lower than e4m3's bias wants, times 2^120 (exact, subnormals included), then e4m3's NaN
// (S.1111.111, which the scaling maps to 480) restored.
template <typename T> struct E4m3;
template <> struct E4m3<__half> {
  static __device__ __forceinline__ void to_io(uint32_t w, uint32_t& lo, uint32_t& hi) {
    const __half2_raw a = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w & 0xffffu), __NV_E4M3);
    const __half2_raw b = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w >> 16), __NV_E4M3);
    lo = *reinterpret_cast<const uint32_t*>(&a);
    hi = *reinterpret_cast<const uint32_t*>(&b);
  }
};
template <> struct E4m3<__nv_bfloat16> {
  static __device__ __forceinline__ uint32_t pair(uint32_t x) {     // x: the two bytes in bits 8-15 and 24-31
    const uint32_t em = x & 0x7f007f00u;
    uint32_t r;
    asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(r) : "r"((em >> 4) | (x & 0x80008000u)), "r"(0x7b807b80u));
    return r | (__vcmpeq2(em, 0x7f007f00u) & 0x7fc07fc0u);
  }
  static __device__ __forceinline__ void to_io(uint32_t w, uint32_t& lo, uint32_t& hi) {
    lo = pair(__byte_perm(w, 0u, 0x1404));
    hi = pair(__byte_perm(w, 0u, 0x3424));
  }
};

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

// The first maximal index of row[0 .. V) (NaN never wins; index 0 when nothing beats -inf), by a block of 1024
// threads; sv / si: 1024 entries of shared memory each.  Every thread gets the result.
template <typename T>
__device__ __forceinline__ int64_t block_argmax_1024(const T* row, int64_t V, float* sv, int64_t* si) {
  float best = -INFINITY;
  int64_t bi = 0;
  for (int64_t i = threadIdx.x; i < V; i += 1024) {
    float v = io<T>::to_f(row[i]);
    if (v > best) { best = v; bi = i; }   // ascending i per thread -> first max wins
  }
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
  return si[0];
}

// ---- e4m3 group quantisation: 128-element groups over 128 / N aligned lanes, N = 4 (a warp) or 8 consecutive elements
// per lane.  scale = amax / 448 and q = v / scale, both divided as torch divides (__fdiv_rn), bit-exact with one of two
// references: kActQuant (act_quant_deepseek_v3) takes amax as is and leaves q unclamped; kPerTokenGroup
// (per_token_group_quant_fp8) floors amax at 1e-10 and clamps q to +-448, which also turns a NaN q (kept as NaN by
// float_to_fp8) into -448.
enum class E4m3Group { kActQuant, kPerTokenGroup };
// the lane's element i in byte i % 4 of bits[i / 4]; the group's scale, on every lane
template <int N>
struct E4m3Word { uint32_t bits[N / 4]; float scale; };
// max |v[I .. I + N)| as the pairwise tree fmaxf(max of the first half, max of the second half)
template <int I, int N>
__device__ __forceinline__ float abs_max(const float* v) {
  if constexpr (N == 1) return fabsf(v[I]);
  else return fmaxf(abs_max<I, N / 2>(v), abs_max<I + N / 2, N / 2>(v));
}
template <E4m3Group kRule, int N>
__device__ __forceinline__ E4m3Word<N> e4m3_group_quant(const float (&v)[N]) {
  static_assert(N == 4 || N == 8, "a lane holds 4 or 8 elements of its group");
  float amax = abs_max<0, N>(v);
#pragma unroll
  for (int o = 64 / N; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if constexpr (kRule == E4m3Group::kPerTokenGroup) amax = fmaxf(amax, 1e-10f);
  const float sc = __fdiv_rn(amax, 448.0f);
  E4m3Word<N> w;
#pragma unroll
  for (int k = 0; k < N / 4; ++k) {
    uint32_t bits = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float q = __fdiv_rn(v[4 * k + i], sc);
      if constexpr (kRule == E4m3Group::kPerTokenGroup) q = fminf(fmaxf(q, -448.f), 448.f);
      bits |= (uint32_t)float_to_fp8(q) << (8 * i);
    }
    w.bits[k] = bits;
  }
  w.scale = sc;
  return w;
}

}  // namespace cb
