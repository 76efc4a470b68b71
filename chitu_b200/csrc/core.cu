// Error plumbing + the integer / bit-exact operators: paged-KV append, MoE align.
#include <string.h>

#include "common.cuh"
#include "splitkv.cuh"

namespace cb {

static thread_local char g_err[1024] = "";
static std::atomic<int64_t> g_launches{0};

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  if (code > 0) (void)cudaGetLastError();   // do not leak a stale error into the next entry point
  return code;
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

// ---- timeline (dev tool): host-side log of the C entry behind every launch, in launch order ----
static bool g_tl_on = false;
static char g_tl_names[1 << 16];
static size_t g_tl_len = 0;
bool tl_enabled() { return g_tl_on; }
void tl_log_launch(const char* entry, int n) {
  for (int i = 0; i < n; ++i) {
    const size_t l = strlen(entry);
    if (g_tl_len + l + 2 >= sizeof(g_tl_names)) return;
    memcpy(g_tl_names + g_tl_len, entry, l);
    g_tl_len += l;
    g_tl_names[g_tl_len++] = '\n';
    g_tl_names[g_tl_len] = 0;
  }
}

}  // namespace cb

extern "C" const char* chitu_b200_last_error(void) { return cb::g_err; }
extern "C" int chitu_b200_version(void) { return 100; }
extern "C" int64_t chitu_b200_launch_count(void) { return cb::g_launches.load(); }

extern "C" {
int chitu_b200_tl_set_core(unsigned long long*);
int chitu_b200_tl_set_elementwise(unsigned long long*);
int chitu_b200_tl_set_gemv(unsigned long long*);
int chitu_b200_tl_set_gemm_tc(unsigned long long*);
int chitu_b200_tl_set_linear(unsigned long long*);
int chitu_b200_tl_set_attention(unsigned long long*);
int chitu_b200_tl_set_mla_tc(unsigned long long*);
int chitu_b200_tl_set_mla_prefill(unsigned long long*);
int chitu_b200_tl_set_gqa_prefill(unsigned long long*);
int chitu_b200_tl_set_moe(unsigned long long*);
int chitu_b200_tl_set_comm(unsigned long long*);
int chitu_b200_tl_set_sampling(unsigned long long*);
}
// Dev tool: arm (buf != NULL: uint64 [2 + capacity], buf[0] = 0, buf[1] = capacity set by the caller) or disarm the
// in-graph timeline; while armed the entry name of every launch is appended to the log chitu_b200_debug_timeline_names returns.
extern "C" int chitu_b200_debug_timeline(void* buf) {
  unsigned long long* p = (unsigned long long*)buf;
  int rc = chitu_b200_tl_set_core(p) | chitu_b200_tl_set_elementwise(p) | chitu_b200_tl_set_gemv(p) |
           chitu_b200_tl_set_gemm_tc(p) | chitu_b200_tl_set_linear(p) | chitu_b200_tl_set_attention(p) |
           chitu_b200_tl_set_mla_tc(p) | chitu_b200_tl_set_mla_prefill(p) | chitu_b200_tl_set_gqa_prefill(p) |
           chitu_b200_tl_set_moe(p) | chitu_b200_tl_set_comm(p) | chitu_b200_tl_set_sampling(p);
  cb::g_tl_on = p != nullptr;
  cb::g_tl_len = 0;
  cb::g_tl_names[0] = 0;
  return rc;
}
extern "C" const char* chitu_b200_debug_timeline_names(void) { return cb::g_tl_names; }

// ============================================================================================
// Paged append: row i of request b is written to position p = seqlens[b] + i, i.e. to cache row
// block_table[b, p / index_div] * page_size + p % index_div, of one or two caches (contiguous
// caches: row b * rows_sb + p, p < cache_rows).  One CTA per row; 16-byte copies when every
// address and stride allows them, byte copies otherwise.
// ============================================================================================
// The rows of one append launch, as f(b, i, sb, si): row i of request b, read from src + sb * src_sb + si * src_st.
// Fixed length (cu_seqlens == NULL), grid (sq, min(B, 65535)): row blockIdx.x of requests blockIdx.y, blockIdx.y +
// gridDim.y, ...; sb = b, si = i.  Ragged, grid (total_rows): source row r = blockIdx.x belongs to the request b with
// cu_seqlens[b] <= r < cu_seqlens[b + 1] (binary search; rows outside [cu[0], cu[B]) belong to none); sb = 0, si = r.
template <typename F>
__device__ __forceinline__ void for_each_append_row(const int32_t* __restrict__ cu_seqlens, int B, F&& f) {
  const int r = blockIdx.x;
  if (cu_seqlens == nullptr) {
    for (int b = blockIdx.y; b < B; b += gridDim.y) f(b, r, b, r);     // more than 65535 requests: a CTA takes several
    return;
  }
  if (r < cu_seqlens[0] || r >= cu_seqlens[B]) return;
  int lo = 0, hi = B;                                 // cu_seqlens[lo] <= r < cu_seqlens[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (cu_seqlens[mid] <= r) lo = mid;
    else hi = mid;
  }
  f(lo, r - cu_seqlens[lo], 0, r);
}

// Row i of request b (n units of V) into both caches; bt is the request's block-table row.  A thread issues its source
// loads for two passes over both caches before the page lookup and the stores, so the copy's memory round trip
// overlaps the lookup's.  The compiler would not order them so itself: it cannot tell that sources and caches never
// overlap, and with bt __restrict__ it hoists the lookup above the loads.
// CONTIG: the destination is row b * rows_sb + p of contiguous caches; bt, page_size and index_div are unused.
template <typename V, bool CONTIG>
__device__ __forceinline__ void copy_row(const cb::PagedAppend& c0, const cb::PagedAppend& c1, int p,
                                         const int32_t* bt, int page_size, int index_div, int64_t rows_sb, int b,
                                         int sb, int si, int64_t n) {
  const V* s0 = reinterpret_cast<const V*>((const uint8_t*)c0.src + sb * c0.src_sb + si * c0.src_st);
  const V* s1 = reinterpret_cast<const V*>((const uint8_t*)c1.src + sb * c1.src_sb + si * c1.src_st);
  const bool two = c1.cache != nullptr;
#pragma unroll 1
  for (int64_t u = threadIdx.x; u < n; u += 2 * blockDim.x) {
    const int64_t w = u + blockDim.x;
    V x0 = s0[u], x1, y0, y1;
    if (w < n) y0 = s0[w];
    if (two) x1 = s1[u];
    if (two && w < n) y1 = s1[w];
    const int64_t row = CONTIG ? (int64_t)b * rows_sb + p : (int64_t)bt[p / index_div] * page_size + p % index_div;
    V* d0 = reinterpret_cast<V*>(c0.cache) + row * n;
    V* d1 = reinterpret_cast<V*>(c1.cache) + row * n;
    d0[u] = x0;
    if (w < n) d0[w] = y0;
    if (two) d1[u] = x1;
    if (two && w < n) d1[w] = y1;
  }
}

// seqlens == NULL: every request starts at position 0
template <bool CONTIG>
__device__ __forceinline__ void append_rows(const cb::PagedAppend& c0, const cb::PagedAppend& c1, int64_t row_bytes,
                                            const int32_t* __restrict__ seqlens, const int32_t* cu_seqlens,
                                            const int32_t* block_table, int bt_stride, int B, int page_size,
                                            int index_div, int64_t rows_sb, int cache_rows, int vec) {
  cb::pdl_prologue();
  for_each_append_row(cu_seqlens, B, [&](int b, int i, int sb, int si) {
    const int p = (seqlens ? seqlens[b] : 0) + i;
    if (CONTIG && p >= cache_rows) return;             // past the contiguous cache's capacity: not written
    const int32_t* bt = block_table + (int64_t)b * bt_stride;
    if (vec) copy_row<uint4, CONTIG>(c0, c1, p, bt, page_size, index_div, rows_sb, b, sb, si, row_bytes >> 4);
    else copy_row<uint8_t, CONTIG>(c0, c1, p, bt, page_size, index_div, rows_sb, b, sb, si, row_bytes);
  });
}

__global__ void __launch_bounds__(128) paged_append_kernel(cb::PagedAppend c0, cb::PagedAppend c1, int64_t row_bytes,
                                                           const int32_t* __restrict__ seqlens,
                                                           const int32_t* cu_seqlens, const int32_t* block_table,
                                                           int bt_stride, int B, int page_size, int index_div,
                                                           int vec) {
  append_rows<false>(c0, c1, row_bytes, seqlens, cu_seqlens, block_table, bt_stride, B, page_size, index_div, 0, 0,
                     vec);
}

__global__ void __launch_bounds__(128) contiguous_append_kernel(cb::PagedAppend c0, cb::PagedAppend c1,
                                                                int64_t row_bytes, const int32_t* __restrict__ seqlens,
                                                                const int32_t* cu_seqlens, int64_t rows_sb,
                                                                int cache_rows, int B, int vec) {
  append_rows<true>(c0, c1, row_bytes, seqlens, cu_seqlens, nullptr, 0, B, 1, 1, rows_sb, cache_rows, vec);
}

// Rows of n io elements into one or two e4m3 caches, 8 elements (16 bytes in, 8 out) per thread and step.
template <typename T>
__global__ void __launch_bounds__(128) paged_append_e4m3_kernel(cb::PagedAppend c0, cb::PagedAppend c1, int n,
                                                                const int32_t* __restrict__ seqlens,
                                                                const int32_t* __restrict__ cu_seqlens,
                                                                const int32_t* __restrict__ block_table, int bt_stride,
                                                                int B, int page_size) {
  cb::pdl_prologue();
  for_each_append_row(cu_seqlens, B, [&](int b, int i, int sb, int si) {
    const int p = (seqlens ? seqlens[b] : 0) + i;
    const int64_t row = (int64_t)block_table[(int64_t)b * bt_stride + p / page_size] * page_size + p % page_size;
    for (int u = threadIdx.x; u < (c1.cache ? 2 : 1) * (n / 8); u += blockDim.x) {
      const cb::PagedAppend& c = u < n / 8 ? c0 : c1;
      const int e = (u < n / 8 ? u : u - n / 8) * 8;
      const uint4 x = *reinterpret_cast<const uint4*>((const uint8_t*)c.src + sb * c.src_sb + si * c.src_st + e * 2);
      const uint2 y = make_uint2(cb::io2_to_e4m3x2<T>(x.x) | cb::io2_to_e4m3x2<T>(x.y) << 16,
                                 cb::io2_to_e4m3x2<T>(x.z) | cb::io2_to_e4m3x2<T>(x.w) << 16);
      *reinterpret_cast<uint2*>((uint8_t*)c.cache + row * n + e) = y;
    }
  });
}

namespace cb {
// for_each_append_row's grids: `rows` is sq (fixed length) or total_rows (with cu_seqlens)
static dim3 append_grid(const int32_t* cu_seqlens, int B, int rows) {
  return cu_seqlens ? dim3(rows) : dim3(rows, B < 65535 ? B : 65535);
}

void launch_paged_append_e4m3(PagedAppend c0, PagedAppend c1, int n, int dtype, const int32_t* seqlens,
                              const int32_t* cu_seqlens, const int32_t* block_table, int bt_stride, int B, int rows,
                              int page_size, cudaStream_t st) {
  const dim3 grid = append_grid(cu_seqlens, B, rows);
  const int threads = n / 4 < 128 ? 64 : 128;
  dispatch_io(dtype, [&](auto t) {
    launch_k(paged_append_e4m3_kernel<decltype(t)>, grid, dim3(threads), 0, st, c0, c1, n, seqlens, cu_seqlens,
             block_table, bt_stride, B, page_size);
  });
}

// 16-byte copies when every address and stride allows them; 64 threads for rows of fewer than 128 copy units
static int append_vec(const PagedAppend& c0, const PagedAppend& c1, int64_t row_bytes) {
  uintptr_t bits = (uintptr_t)row_bytes;
  for (const PagedAppend& c : {c0, c1})
    if (c.cache) bits |= (uintptr_t)c.cache | (uintptr_t)c.src | (uintptr_t)c.src_sb | (uintptr_t)c.src_st;
  return bits % 16 == 0;
}
static int append_threads(int64_t row_bytes, int vec) { return row_bytes / (vec ? 16 : 1) < 128 ? 64 : 128; }

void launch_paged_append(PagedAppend c0, PagedAppend c1, int64_t row_bytes, const int32_t* seqlens,
                         const int32_t* cu_seqlens, const int32_t* block_table, int bt_stride, int B, int rows,
                         int page_size, int index_div, cudaStream_t st) {
  const int vec = append_vec(c0, c1, row_bytes);
  launch_k(paged_append_kernel, append_grid(cu_seqlens, B, rows), dim3(append_threads(row_bytes, vec)), 0, st, c0, c1,
           row_bytes, seqlens, cu_seqlens, block_table, bt_stride, B, page_size, index_div, vec);
}

void launch_contiguous_append(PagedAppend c0, PagedAppend c1, int64_t row_bytes, const int32_t* seqlens,
                              const int32_t* cu_seqlens, int64_t rows_sb, int cache_rows, int B, int rows,
                              cudaStream_t st) {
  const int vec = append_vec(c0, c1, row_bytes);
  launch_k(contiguous_append_kernel, append_grid(cu_seqlens, B, rows), dim3(append_threads(row_bytes, vec)), 0, st, c0,
           c1, row_bytes, seqlens, cu_seqlens, rows_sb, cache_rows, B, vec);
}
}  // namespace cb

// append_to_paged_kv_cache (reference: chitu/ops.py:50-91, triton_kernels.py:18-48).  Reference quirk kept on purpose:
// page index and in-page offset use `index_div` (literal 64 in triton_kernels.py:38,42) while the row address uses
// the real page_size.
extern "C" int chitu_b200_append_paged_kv(void* kv_cache, const int32_t* page_table,
                                          const void* this_kv, const int32_t* old_seq_lens,
                                          int batch, int pages_per_sample, int page_size,
                                          int index_div, int64_t row_bytes, void* stream) {
  CB_ARG(kv_cache && page_table && this_kv && old_seq_lens);
  CB_ARG(batch >= 0 && pages_per_sample > 0 && page_size > 0 && index_div > 0 && row_bytes > 0);
  if (batch == 0) return 0;
  cb::launch_paged_append({kv_cache, this_kv, row_bytes, row_bytes}, {}, row_bytes, old_seq_lens, nullptr, page_table,
                          pages_per_sample, batch, 1, page_size, index_div, (cudaStream_t)stream);
  CB_LAUNCHED(1);
  return 0;
}

extern "C" int chitu_b200_append_paged_kv_e4m3(void* kv_cache, const int32_t* page_table, const void* this_kv,
                                               const int32_t* old_seq_lens, int batch, int pages_per_sample, int n,
                                               int dtype, void* stream) {
  CB_ARG(kv_cache && page_table && this_kv && old_seq_lens);
  CB_ARG(batch >= 0 && pages_per_sample > 0 && n > 0 && n % 8 == 0 && (dtype == CB_BF16 || dtype == CB_F16));
  CB_ARG((uintptr_t)this_kv % 16 == 0);
  if (batch == 0) return 0;
  const int64_t row_bytes = (int64_t)n * 2;
  cb::launch_paged_append_e4m3({kv_cache, this_kv, row_bytes, row_bytes}, {}, n, dtype, old_seq_lens, nullptr,
                               page_table, pages_per_sample, batch, 1, 64, (cudaStream_t)stream);
  CB_LAUNCHED(1);
  return 0;
}

// The prompt's k / v (or latent) rows into the cache after the prefill attention (include/chitu_b200.h): the appends
// above with ragged lengths, one CTA per source row.
extern "C" int chitu_b200_scatter_kv(void* cache0, void* cache1, const void* src0, int64_t src0_st, const void* src1,
                                     int64_t src1_st, const int32_t* cu_seqlens, const int32_t* cache_seqlens,
                                     const int32_t* block_table, int bt_stride, int page_size, int64_t cache_sb,
                                     int cache_rows, int B, int total_rows, int n, int src_dtype, int cache_dtype,
                                     void* stream) {
  CB_ARG(cache0 && src0 && cu_seqlens && (cache1 == nullptr) == (src1 == nullptr));
  CB_ARG(B >= 0 && total_rows >= 0 && n > 0);
  CB_ARG(src_dtype == CB_BF16 || src_dtype == CB_F16);
  const bool e4m3 = cache_dtype == CB_FP8_E4M3;
  CB_ARG(cache_dtype == src_dtype || (e4m3 && block_table));          // e4m3: paged caches only
  if (block_table) CB_ARG(bt_stride > 0 && page_size > 0);
  else CB_ARG(cache_rows >= 0 && cache_sb % n == 0 && cache_sb >= (int64_t)cache_rows * n);
  if (e4m3)     // 16-byte loads of 8 elements, 8-byte stores
    CB_ARG(n % 8 == 0 && ((uintptr_t)src0 | (uintptr_t)src1) % 16 == 0 && src0_st % 8 == 0 &&
           (!src1 || src1_st % 8 == 0) && ((uintptr_t)cache0 | (uintptr_t)cache1) % 8 == 0);
  if (B == 0 || total_rows == 0) return 0;
  const cb::PagedAppend c0{cache0, src0, 0, src0_st * 2}, c1{cache1, src1, 0, src1_st * 2};
  const cudaStream_t st = (cudaStream_t)stream;
  if (e4m3)
    cb::launch_paged_append_e4m3(c0, c1, n, src_dtype, cache_seqlens, cu_seqlens, block_table, bt_stride, B,
                                 total_rows, page_size, st);
  else if (block_table)
    cb::launch_paged_append(c0, c1, (int64_t)n * 2, cache_seqlens, cu_seqlens, block_table, bt_stride, B, total_rows,
                            page_size, page_size, st);
  else
    cb::launch_contiguous_append(c0, c1, (int64_t)n * 2, cache_seqlens, cu_seqlens, cache_sb / n, cache_rows, B,
                                 total_rows, st);
  CB_LAUNCHED(1);
  return 0;
}

// ============================================================================================
// moe_align_block_size (reference: csrc/moe_align_kernel.cu:27-122, fused_moe.py:314-442)
//
// Grid = one CTA per expert, no inter-CTA communication, fully deterministic:
//   1. every CTA histograms all topk ids in shared memory (ids are tiny and L2 resident),
//   2. block-wide exclusive scan of the block-padded counts -> cumsum (CTA 0 publishes it),
//   3. CTA e writes expert_ids for its blocks and compacts "ids == e" in ascending token
//      order (ballot + popc) into sorted_ids[cumsum[e] ...].
// No serial thread-0 loop, no atomics on the output order (the reference's `atomicAdd`
// scatter, moe_align_kernel.cu:90-95, is order non-deterministic), any num_experts.
// ============================================================================================
template <typename T>
__global__ void __launch_bounds__(256) moe_align_kernel(const T* __restrict__ topk_ids,
                                                        int32_t* __restrict__ sorted_ids,
                                                        int32_t* __restrict__ expert_ids,
                                                        int32_t* __restrict__ total_post_pad,
                                                        int32_t* __restrict__ cumsum, int num_experts,
                                                        int block_size, int64_t numel) {
  cb::pdl_prologue();
  extern __shared__ int32_t smem[];
  int32_t* counts = smem;                     // [num_experts]  (becomes padded exclusive prefix)
  __shared__ int32_t warp_tot[8];
  __shared__ int32_t s_carry;
  const int e = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  for (int i = tid; i < num_experts; i += 256) counts[i] = 0;
  __syncthreads();
  for (int64_t i = tid; i < numel; i += 256) {
    int id = (int)topk_ids[i];
    if (id >= 0 && id < num_experts) atomicAdd(&counts[id], 1);
  }
  __syncthreads();

  // exclusive scan over experts of ceil(count/block)*block, processed in chunks of 256 experts
  if (tid == 0) s_carry = 0;
  __syncthreads();
  int32_t my_start = 0, my_end = 0;
  for (int base = 0; base < num_experts; base += 256) {
    int idx = base + tid;
    int32_t c = (idx < num_experts) ? counts[idx] : 0;
    int32_t padded = (c + block_size - 1) / block_size * block_size;
    int32_t incl = padded;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int32_t n = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += n;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    int32_t woff = 0;
    for (int w = 0; w < warp; ++w) woff += warp_tot[w];
    int32_t carry = s_carry;
    int32_t excl = carry + woff + incl - padded;
    if (idx < num_experts) {
      if (e == 0) cumsum[idx + 1] = excl + padded;
      if (idx == e) { my_start = excl; my_end = excl + padded; }
    }
    __syncthreads();
    if (tid == 255) s_carry = carry + woff + incl;
    __syncthreads();
  }
  if (e == 0 && tid == 0) {
    cumsum[0] = 0;
    *total_post_pad = s_carry;
  }
  // broadcast my_start/my_end from the owning thread
  __shared__ int32_t s_se[2];
  if (tid == (e & 255)) { s_se[0] = my_start; s_se[1] = my_end; }
  __syncthreads();
  my_start = s_se[0];
  my_end = s_se[1];

  for (int i = my_start + tid * block_size; i < my_end; i += 256 * block_size)
    expert_ids[i / block_size] = e;

  // stable compaction of token indices routed to expert e
  int32_t base_out = my_start;
  for (int64_t t0 = 0; t0 < numel; t0 += 256) {
    int64_t i = t0 + tid;
    bool hit = (i < numel) && ((int)topk_ids[i] == e);
    unsigned bal = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) warp_tot[warp] = __popc(bal);
    __syncthreads();
    int32_t woff = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      int32_t c = warp_tot[w];
      if (w < warp) woff += c;
      tot += c;
    }
    if (hit) sorted_ids[base_out + woff + __popc(bal & ((1u << lane) - 1u))] = (int32_t)i;
    base_out += tot;
    __syncthreads();
  }
}

extern "C" int chitu_b200_moe_align_block_size(const void* topk_ids, int ids_dtype, int64_t numel,
                                               int num_experts, int block_size,
                                               int32_t* sorted_ids, int32_t* expert_ids,
                                               int32_t* num_tokens_post_pad, int32_t* cumsum,
                                               void* stream) {
  CB_ARG(sorted_ids && expert_ids && num_tokens_post_pad && cumsum);
  CB_ARG(numel >= 0 && (numel == 0 || topk_ids));
  CB_ARG(num_experts > 0 && num_experts <= 16384 && block_size > 0);
  size_t smem = (size_t)num_experts * sizeof(int32_t);
  cudaStream_t st = (cudaStream_t)stream;
#define LAUNCH_ALIGN(T)                                                                          \
  cb::launch_k(moe_align_kernel<T>, dim3(num_experts), dim3(256), smem, st, (const T*)topk_ids, sorted_ids, expert_ids, \
                                                      num_tokens_post_pad, cumsum, num_experts,  \
                                                      block_size, numel)
  switch (ids_dtype) {
    case CB_U8: LAUNCH_ALIGN(uint8_t); break;
    case CB_I8: LAUNCH_ALIGN(int8_t); break;
    case CB_I16: LAUNCH_ALIGN(int16_t); break;
    case CB_I32: LAUNCH_ALIGN(int32_t); break;
    case CB_I64: LAUNCH_ALIGN(int64_t); break;
    default: return cb::fail(-1, "moe_align_block_size: topk_ids must be an integral dtype (got code %d)", ids_dtype);
  }
#undef LAUNCH_ALIGN
  CB_LAUNCHED(1);
  return 0;
}

// ============================================================================================
// Device-side decode-step preparation (SURVEY §8f n2, §8a a1).
//
//  * decode_prepare : PagedKVCacheManager.prepare_cache_decode + prepare_block_table_for_decode
//    (cache_manager.py:148-158, 196-209) without the per-request Python loops and H2D copies: the sequence lengths, the
//    block table and the free-page stack live on the device; a request whose length sits on a page boundary pops a page
//    and appends it to its block-table row; seq_lens_excl / seq_lens_incl are refreshed.  `advance` != 0 first applies
//    finalize_cache_single_decode (:211-215, seq_len += 1) of the previous step, so one launch per decode step suffices.
//  * attn_plan      : AttnBackend.prepare_metadata_for_decode (attn_backend.py:515-534; FlashMLA get_mla_metadata,
//    third_party/FlashMLA/csrc/flash_fwd_mla_metadata.cu:5-75): a length-aware split-KV plan — the number of keys per
//    split (whole pages) such that the batch's splits fill one wave of CTAs; written to the plan tail of the attention
//    workspace (splitkv.cuh), where the MLA decode kernel finds it.
//
// Neither kernel triggers its dependents early (no griddepcontrol.launch_dependents): everything launched after them
// sees their writes, even kernels that prefetch before their own griddepcontrol.wait.
// ============================================================================================
__global__ void decode_prepare_kernel(int32_t* __restrict__ seq_lens, int32_t* __restrict__ seq_lens_incl,
                                      int32_t* __restrict__ block_table, int bt_stride, int32_t* __restrict__ free_pages,
                                      int32_t* __restrict__ free_count, int32_t* __restrict__ status, int B,
                                      int page_size, int advance) {
  cb::pdl_wait();
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x) {
    int L = seq_lens[b];
    if (advance) { L += 1; seq_lens[b] = L; }
    if (seq_lens_incl) seq_lens_incl[b] = L + 1;
    if (L % page_size == 0) {                         // the token of this decode opens a new page
      const int slot = L / page_size;
      if (slot >= bt_stride) { atomicExch(status, 2); continue; }     // block-table row is full (max_seq_len reached)
      const int idx = atomicSub(free_count, 1) - 1;   // pop
      if (idx < 0) { atomicAdd(free_count, 1); atomicExch(status, 1); continue; }   // "No more free blocks."
      block_table[(int64_t)b * bt_stride + slot] = free_pages[idx];
    }
  }
}

extern "C" int chitu_b200_decode_prepare(int32_t* seq_lens_excl, int32_t* seq_lens_incl, int32_t* block_table,
                                         int bt_stride, int32_t* free_pages, int32_t* free_count, int32_t* status,
                                         int B, int page_size, int advance, void* stream) {
  CB_ARG(seq_lens_excl && block_table && free_pages && free_count && status && B >= 0 && page_size > 0 && bt_stride > 0);
  if (B == 0) return 0;
  cb::launch_k(decode_prepare_kernel, dim3(cb::cdiv(B, 128)), dim3(128), 0, (cudaStream_t)stream, seq_lens_excl,
               seq_lens_incl, block_table, bt_stride, free_pages, free_count, status, B, page_size, advance);
  CB_LAUNCHED(1);
  return 0;
}

__global__ void attn_plan_kernel(const int32_t* __restrict__ seqlens_incl, int B, int page_size, int slots,
                                 int max_splits, int min_pages, int heads, int32_t* __restrict__ plan) {
  cb::pdl_wait();
  const int lane = threadIdx.x;
  int total_pages = 0, max_pages = 0;
  for (int b = lane; b < B; b += 32) {
    const int pg = (seqlens_incl[b] + page_size - 1) / page_size;
    total_pages += pg;
    max_pages = max(max_pages, pg);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    total_pages += __shfl_xor_sync(0xffffffffu, total_pages, o);
    max_pages = max(max_pages, __shfl_xor_sync(0xffffffffu, max_pages, o));
  }
  // smallest number of pages per split (>= min_pages, and large enough that the longest request fits max_splits)
  // whose splits fit one wave of `slots` CTAs
  int pps = max(max(min_pages, (total_pages + slots - 1) / max(slots, 1)), (max_pages + max_splits - 1) / max_splits);
  pps = max(pps, 1);
  int total = 0, mx = 0;
  for (int iter = 0; iter < 64; ++iter) {
    total = 0;
    mx = 0;
    for (int b = lane; b < B; b += 32) {
      const int pg = (seqlens_incl[b] + page_size - 1) / page_size;
      const int s = (pg + pps - 1) / pps;
      total += s;
      mx = max(mx, s);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      total += __shfl_xor_sync(0xffffffffu, total, o);
      mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    if (total <= slots || pps >= max_pages) break;
    ++pps;
  }
  if (lane == 0) {
    plan[cb::kPlanWordKeysPerSplit] = pps * page_size;
    plan[cb::kPlanWordMaxSplits] = mx;
    plan[cb::kPlanWordTotalSplits] = total;
    plan[cb::kPlanWordBatch] = B;
    plan[cb::kPlanWordPageSize] = page_size;
    plan[cb::kPlanWordHeads] = heads;
    __threadfence();
    plan[cb::kPlanWordMagic] = cb::kPlanMagic;
  }
}

extern "C" int chitu_b200_attn_plan(const int32_t* seqlens_incl, int B, int heads, int page_size, int max_seqlen_hint,
                                    void* workspace, int64_t workspace_bytes, void* stream) {
  CB_ARG(seqlens_incl && workspace && workspace_bytes >= 512 && B >= 0 && heads > 0 && page_size > 0 && max_seqlen_hint > 0);
  if (B == 0) return 0;
  const int hgroups = cb::cdiv(heads, 16);
  int slots = 132 / hgroups;                                  // one CTA per H100 SM
  if (slots < 1) slots = 1;
  // the grid the decode kernel will be launched with for this (B, heads, hint): upper bound of a request's splits
  const int max_splits = cb::mla_num_splits(B, heads, max_seqlen_hint, workspace_bytes);
  cb::launch_k(attn_plan_kernel, dim3(1), dim3(32), 0, (cudaStream_t)stream, seqlens_incl, B, page_size, slots, max_splits,
               2, heads, cb::split_kv_plan(workspace, workspace_bytes));
  CB_LAUNCHED(1);
  return 0;
}

CB_DEFINE_TL_SETTER(core)
