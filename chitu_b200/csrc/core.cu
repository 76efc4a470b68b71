// Error plumbing + the integer / bit-exact operators: paged-KV append, MoE align.
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

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
bool pdl_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("CHITU_B200_PDL");
    on = (e && e[0] == '0') ? 0 : 1;
  }
  return on != 0;
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
           chitu_b200_tl_set_mla_tc(p) | chitu_b200_tl_set_moe(p) | chitu_b200_tl_set_comm(p) | chitu_b200_tl_set_sampling(p);
  cb::g_tl_on = p != nullptr;
  cb::g_tl_len = 0;
  cb::g_tl_names[0] = 0;
  return rc;
}
extern "C" const char* chitu_b200_debug_timeline_names(void) { return cb::g_tl_names; }

// ============================================================================================
// append_to_paged_kv_cache   (reference: chitu/ops.py:50-91, triton_kernels.py:18-48)
// One CTA per request; the token's row (row_bytes) is copied with 16-byte vectors when aligned.
// ============================================================================================
__global__ void append_paged_kv_kernel(uint8_t* __restrict__ kv_cache,
                                       const int32_t* __restrict__ page_table,
                                       const uint8_t* __restrict__ this_kv,
                                       const int32_t* __restrict__ old_seq_lens,
                                       int pages_per_sample, int page_size, int index_div,
                                       int64_t row_bytes, int vec_ok) {
  cb::pdl_prologue();
  const int b = blockIdx.x;
  const int seqlen = old_seq_lens[b];
  // Reference quirk kept on purpose: page index and in-page offset use `index_div` (literal 64
  // in triton_kernels.py:38,42) while the row address uses the real PAGE_SIZE.
  const int page_id = page_table[(int64_t)b * pages_per_sample + seqlen / index_div];
  const int64_t row = (int64_t)page_id * page_size + seqlen % index_div;
  uint8_t* dst = kv_cache + row * row_bytes;
  const uint8_t* src = this_kv + (int64_t)b * row_bytes;
  if (vec_ok) {
    const int64_t n16 = row_bytes >> 4;
    for (int64_t i = threadIdx.x; i < n16; i += blockDim.x)
      reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
  } else {
    for (int64_t i = threadIdx.x; i < row_bytes; i += blockDim.x) dst[i] = src[i];
  }
}

extern "C" int chitu_b200_append_paged_kv(void* kv_cache, const int32_t* page_table,
                                          const void* this_kv, const int32_t* old_seq_lens,
                                          int batch, int pages_per_sample, int page_size,
                                          int index_div, int64_t row_bytes, void* stream) {
  CB_ARG(kv_cache && page_table && this_kv && old_seq_lens);
  CB_ARG(batch >= 0 && pages_per_sample > 0 && page_size > 0 && index_div > 0 && row_bytes > 0);
  if (batch == 0) return 0;
  int vec_ok = (row_bytes % 16 == 0) && ((uintptr_t)kv_cache % 16 == 0) && ((uintptr_t)this_kv % 16 == 0);
  int threads = (int)((row_bytes / (vec_ok ? 16 : 1)) < 128 ? 64 : 128);
  cb::launch_k(append_paged_kv_kernel, dim3(batch), dim3(threads), 0, (cudaStream_t)stream, 
      (uint8_t*)kv_cache, page_table, (const uint8_t*)this_kv, old_seq_lens, pages_per_sample,
      page_size, index_div, row_bytes, vec_ok);
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
//    split (whole pages) such that the batch's splits fill one wave of CTAs; written to the last 256 bytes of the
//    attention workspace, where the decode kernels find it.
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

// plan words (int32) at workspace + workspace_bytes - 256:
//   [0] magic 0x504c414e ("PLAN")  [1] keys per split (multiple of the page size)  [2] max splits of a request
//   [3] total splits of the batch  [4] B  [5] page size  [6] heads the plan was made for
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
    plan[1] = pps * page_size;
    plan[2] = mx;
    plan[3] = total;
    plan[4] = B;
    plan[5] = page_size;
    plan[6] = heads;
    __threadfence();
    plan[0] = 0x504c414e;
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
  const int max_splits = chitu_b200_mla_num_splits(B, heads, max_seqlen_hint, workspace_bytes);
  int32_t* plan = (int32_t*)((uint8_t*)workspace + workspace_bytes - 256);
  cb::launch_k(attn_plan_kernel, dim3(1), dim3(32), 0, (cudaStream_t)stream, seqlens_incl, B, page_size, slots, max_splits,
               2, heads, plan);
  CB_LAUNCHED(1);
  return 0;
}

CB_DEFINE_TL_SETTER(core)
