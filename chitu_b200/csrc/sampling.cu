// Temperature / top-k / top-p sampling of the decode step (SURVEY §8f n3).
//
// Reference: NormalExecutor.update_response (executor.py:104-110): probs = softmax(logits / temperature), then
// top_k_top_p_min_p_sampling_from_probs_torch (utils.py:62-81): sort descending, zero every entry whose EXCLUSIVE
// cumulative mass exceeds top_p, zero every entry of rank >= top_k, renormalise, torch.multinomial.  That is a full
// [B, V] sort (V = 129 280) + cumsum + scatter per step.  Here: one CTA per request, no sort —
//   1. max and sum-exp of the row (fp32) -> p_i;
//   2. the kept set {i : mass of strictly larger entries <= top_p  and  number of strictly larger entries < top_k} is a
//      threshold on p_i; the threshold's 32-bit ordered key is found by a 3-level radix histogram (11 + 11 + 10 bits) of
//      (count, mass) per bin — exactly the reference's rule on tie-free rows (ties: all equal entries are kept together);
//   3. inverse-CDF draw over the kept entries in vocabulary order with the caller's uniform u in [0, 1)
//      (torch.multinomial's Philox stream cannot be reproduced from outside; the DISTRIBUTION is the reference's).
// Logits are re-read from L2 for every pass (258 KB per row in bf16): six passes, no [B, V] temporaries.
#include "common.cuh"

using namespace cb;

namespace {

constexpr int kThreads = 1024;

__device__ __forceinline__ uint32_t okey(float v) {            // monotone float -> uint32 (p >= 0 here)
  const uint32_t u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

template <typename T>
__device__ __forceinline__ float ldv(const T* p, int64_t i) { return io<T>::to_f(p[i]); }

__device__ __forceinline__ float block_reduce(float v, bool is_max, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = is_max ? warp_max(v) : warp_sum(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = red[0];
  for (int i = 1; i < kThreads / 32; ++i) r = is_max ? fmaxf(r, red[i]) : r + red[i];
  return r;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) sample_kernel(const T* __restrict__ logits, int64_t row_stride, int V,
                                                          const float* __restrict__ temperatures,
                                                          const int32_t* __restrict__ top_ks, const float* __restrict__ top_ps,
                                                          const float* __restrict__ uniforms, int64_t* __restrict__ out_tokens,
                                                          int32_t* __restrict__ out_kept, float* __restrict__ out_mass) {
  cb::pdl_prologue();
  __shared__ float red[kThreads / 32];
  __shared__ float h_sum[2048];
  __shared__ int h_cnt[2048];
  __shared__ uint32_t s_prefix;
  __shared__ float s_above_mass;
  __shared__ int s_above_cnt;
  __shared__ float s_scan[kThreads];
  __shared__ int s_pick;
  __shared__ bool s_tail;
  const int b = blockIdx.x, tid = threadIdx.x;
  const T* row = logits + (int64_t)b * row_stride;
  const float inv_t = 1.f / temperatures[b];
  const float top_p = top_ps[b];
  const int top_k = top_ks[b] > 0 ? top_ks[b] : V;

  float mx = -INFINITY;
  for (int i = tid; i < V; i += kThreads) mx = fmaxf(mx, ldv(row, i) * inv_t);
  mx = block_reduce(mx, true, red);
  float sm = 0.f;
  for (int i = tid; i < V; i += kThreads) sm += __expf(ldv(row, i) * inv_t - mx);
  sm = block_reduce(sm, false, red);
  const float inv_sum = 1.f / sm;
  auto prob = [&](int i) { return __expf(ldv(row, i) * inv_t - mx) * inv_sum; };

  // ---- radix search of the threshold key: levels of 11, 11, 10 bits ----
  if (tid == 0) { s_prefix = 0u; s_above_mass = 0.f; s_above_cnt = 0; }
  __syncthreads();
  const int shifts[3] = {21, 10, 0}, bits[3] = {11, 11, 10};
  for (int lv = 0; lv < 3; ++lv) {
    const int shift = shifts[lv], nb = 1 << bits[lv];
    for (int i = tid; i < nb; i += kThreads) { h_sum[i] = 0.f; h_cnt[i] = 0; }
    __syncthreads();
    const uint32_t prefix = s_prefix;
    const uint32_t hi_mask = lv == 0 ? 0u : (0xffffffffu << (shift + bits[lv]));
    for (int i = tid; i < V; i += kThreads) {
      const float p = prob(i);
      const uint32_t k = okey(p);
      if ((k & hi_mask) == (prefix & hi_mask)) {
        const int bin = (k >> shift) & (nb - 1);
        atomicAdd(&h_sum[bin], p);
        atomicAdd(&h_cnt[bin], 1);
      }
    }
    __syncthreads();
    if (tid == 0) {
      // walk the bins from the largest values down: the boundary bin is the LAST bin whose largest element is still kept
      float mass = s_above_mass;
      int cnt = s_above_cnt, pick = -1;
      float pm = mass;
      int pc = cnt;
      for (int bin = nb - 1; bin >= 0; --bin) {
        if (h_cnt[bin] == 0) continue;
        if (mass <= top_p && cnt < top_k) { pick = bin; pm = mass; pc = cnt; }
        else break;
        mass += h_sum[bin];
        cnt += h_cnt[bin];
      }
      if (pick < 0) {                      // cannot happen on a non-empty row (the maximum is always kept)
        pick = nb - 1;
      }
      s_prefix = prefix | ((uint32_t)pick << shift);
      s_above_mass = pm;
      s_above_cnt = pc;
    }
    __syncthreads();
  }
  const uint32_t thr = s_prefix;               // entries with key >= thr are kept
  // ... except p == 0: the walk ends on the bin of p = 0 when the fp32 mass of the positive entries is <= top_p
  auto kept_p = [&](float p) { return p > 0.f && okey(p) >= thr; };

  // ---- kept mass / count, then the inverse-CDF draw in vocabulary order ----
  const int per = (V + kThreads - 1) / kThreads;
  const int i0 = tid * per, i1 = min(i0 + per, V);
  float part = 0.f;
  int kept = 0;
  for (int i = i0; i < i1; ++i) {
    const float p = prob(i);
    if (kept_p(p)) { part += p; ++kept; }
  }
  s_scan[tid] = part;
  const float z = block_reduce(part, false, red);
  const int nkept = (int)block_reduce((float)kept, false, red);
  __syncthreads();
  if (tid == 0) {
    const float target = uniforms[b] * z;
    float run = 0.f;
    int pick = -1;
    for (int t = 0; t < kThreads; ++t) {
      if (run + s_scan[t] > target) { pick = t; break; }
      run += s_scan[t];
    }
    // rounding pushed the target past the end of the scan: the draw is the last kept entry (of the last thread with any)
    s_tail = pick < 0;
    if (pick < 0) {
      pick = kThreads - 1;
      while (pick > 0 && s_scan[pick] == 0.f) --pick;
    }
    s_pick = pick;
    s_above_mass = run;
    if (out_kept) out_kept[b] = nkept;
    if (out_mass) out_mass[b] = z;
  }
  __syncthreads();
  if (tid == s_pick) {
    const float target = uniforms[b] * z;
    float run = s_above_mass;
    int tok = -1, last = -1;
    for (int i = i0; i < i1; ++i) {
      const float p = prob(i);
      if (kept_p(p)) {
        last = i;
        run += p;
        if (!s_tail && run > target) { tok = i; break; }
      }
    }
    out_tokens[b] = tok >= 0 ? tok : last;
  }
}

// Greedy acceptance of k draft tokens per request, one thread per request.  It writes seq_lens, which the decode kernels
// read before their griddepcontrol.wait, so it waits for its predecessor and never lets its dependents start early
// (the rule of decode_prepare_kernel).
__global__ void spec_accept_greedy_kernel(const int64_t* __restrict__ target, const int64_t* __restrict__ drafts,
                                          const int32_t* __restrict__ n_draft, int32_t* __restrict__ seq_lens,
                                          int64_t* __restrict__ out_tokens, int32_t* __restrict__ accepted,
                                          int64_t* __restrict__ next_tokens, int B, int k) {
  cb::pdl_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int64_t* t = target + (int64_t)b * (k + 1);
  const int64_t* d = drafts + (int64_t)b * k;
  const int n = min(max(n_draft[b], 0), k);
  int a = 0;
  while (a < n && d[a] == t[a]) ++a;
  int64_t* o = out_tokens + (int64_t)b * (k + 1);
  for (int i = 0; i <= k; ++i) o[i] = i <= a ? t[i] : -1;
  accepted[b] = a;
  next_tokens[b] = t[a];
  seq_lens[b] += a + 1;
}

}  // namespace

// target int64 [B, k + 1], drafts int64 [B, k], n_draft int32 [B] (clamped to 0..k), seq_lens int32 [B] (in place);
// out_tokens int64 [B, k + 1], accepted int32 [B], next_tokens int64 [B].
extern "C" int chitu_b200_spec_accept_greedy(const int64_t* target, const int64_t* drafts, const int32_t* n_draft,
                                             int32_t* seq_lens, int64_t* out_tokens, int32_t* accepted,
                                             int64_t* next_tokens, int B, int k, void* stream) {
  CB_ARG(target && drafts && n_draft && seq_lens && out_tokens && accepted && next_tokens && B >= 0 && k >= 1);
  if (B == 0) return 0;
  cb::launch_k(spec_accept_greedy_kernel, dim3(cb::cdiv(B, 128)), dim3(128), 0, (cudaStream_t)stream, target, drafts,
               n_draft, seq_lens, out_tokens, accepted, next_tokens, B, k);
  CB_LAUNCHED(1);
  return 0;
}

// logits [B, V] (row stride in elements), bf16 / fp16 / fp32; temperatures, top_ps, uniforms fp32 [B]; top_ks int32 [B]
// (<= 0: no top-k); out_tokens int64 [B]; out_kept / out_mass (optional, diagnostics): size and mass of the kept set.
extern "C" int chitu_b200_sample_top_k_top_p(const void* logits, int64_t row_stride, int B, int V, int dtype,
                                             const float* temperatures, const int32_t* top_ks, const float* top_ps,
                                             const float* uniforms, int64_t* out_tokens, int32_t* out_kept,
                                             float* out_mass, void* stream) {
  CB_ARG(logits && temperatures && top_ks && top_ps && uniforms && out_tokens && B >= 0 && V > 0 && row_stride >= V);
  if (B == 0) return 0;
  const int rc = cb::dispatch_dtype<CB_BF16, CB_F16, CB_F32>(__func__, dtype, [&](auto t) {
    using T = decltype(t);
    cb::launch_k(sample_kernel<T>, dim3(B), dim3(kThreads), 0, (cudaStream_t)stream, (const T*)logits, row_stride, V,
                 temperatures, top_ks, top_ps, uniforms, out_tokens, out_kept, out_mass);
    return 0;
  });
  if (rc) return rc;
  CB_LAUNCHED(1);
  return 0;
}

CB_DEFINE_TL_SETTER(sampling)
