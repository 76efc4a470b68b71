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

// ---- the kept-set rule as block-wide device helpers (kThreads threads), shared by the sampler and the sampled
// acceptance of speculative drafts ----

// softmax(l / T) of one row: p_i = exp(l_i * inv_t - mx) * inv_sum
struct RowSoftmax {
  float inv_t, mx, inv_sum;
};

template <typename T>
__device__ __forceinline__ float row_prob(const T* row, const RowSoftmax& s, int i) {
  return __expf(ldv(row, i) * s.inv_t - s.mx) * s.inv_sum;
}

template <typename T>
__device__ __forceinline__ RowSoftmax row_softmax(const T* row, int V, float inv_t, float* red) {
  const int tid = threadIdx.x;
  float mx = -INFINITY;
  for (int i = tid; i < V; i += kThreads) mx = fmaxf(mx, ldv(row, i) * inv_t);
  mx = block_reduce(mx, true, red);
  float sm = 0.f;
  for (int i = tid; i < V; i += kThreads) sm += __expf(ldv(row, i) * inv_t - mx);
  sm = block_reduce(sm, false, red);
  return {inv_t, mx, 1.f / sm};
}

struct KeptSmem {
  float h_sum[2048];
  int h_cnt[2048];
  uint32_t prefix;
  float above_mass;
  int above_cnt;
};

// The threshold key of the kept set: entries with okey(p) >= the result (and p > 0) are kept.  A radix search of the
// key over levels of 11, 11 and 10 bits, each a histogram of (count, mass) per bin.
template <class Prob>
__device__ __forceinline__ uint32_t kept_threshold(Prob prob, int V, int top_k, float top_p, KeptSmem& sm) {
  const int tid = threadIdx.x;
  if (tid == 0) { sm.prefix = 0u; sm.above_mass = 0.f; sm.above_cnt = 0; }
  __syncthreads();
  const int shifts[3] = {21, 10, 0}, bits[3] = {11, 11, 10};
  for (int lv = 0; lv < 3; ++lv) {
    const int shift = shifts[lv], nb = 1 << bits[lv];
    for (int i = tid; i < nb; i += kThreads) { sm.h_sum[i] = 0.f; sm.h_cnt[i] = 0; }
    __syncthreads();
    const uint32_t prefix = sm.prefix;
    const uint32_t hi_mask = lv == 0 ? 0u : (0xffffffffu << (shift + bits[lv]));
    for (int i = tid; i < V; i += kThreads) {
      const float p = prob(i);
      const uint32_t k = okey(p);
      if ((k & hi_mask) == (prefix & hi_mask)) {
        const int bin = (k >> shift) & (nb - 1);
        atomicAdd(&sm.h_sum[bin], p);
        atomicAdd(&sm.h_cnt[bin], 1);
      }
    }
    __syncthreads();
    if (tid == 0) {
      // walk the bins from the largest values down: the boundary bin is the LAST bin whose largest element is still kept
      float mass = sm.above_mass;
      int cnt = sm.above_cnt, pick = -1;
      float pm = mass;
      int pc = cnt;
      for (int bin = nb - 1; bin >= 0; --bin) {
        if (sm.h_cnt[bin] == 0) continue;
        if (mass <= top_p && cnt < top_k) { pick = bin; pm = mass; pc = cnt; }
        else break;
        mass += sm.h_sum[bin];
        cnt += sm.h_cnt[bin];
      }
      if (pick < 0) {                      // cannot happen on a non-empty row (the maximum is always kept)
        pick = nb - 1;
      }
      sm.prefix = prefix | ((uint32_t)pick << shift);
      sm.above_mass = pm;
      sm.above_cnt = pc;
    }
    __syncthreads();
  }
  return sm.prefix;
}

// kept: p > 0 and at or above the threshold key (the walk ends on the bin of p = 0 when the fp32 mass of the positive
// entries is <= top_p)
__device__ __forceinline__ bool kept_p(float p, uint32_t thr) { return p > 0.f && okey(p) >= thr; }

// Thread t's share of the weights w(i) over its contiguous range of the vocabulary (the order of the draw), and the
// number of positive ones.
template <class W>
__device__ __forceinline__ float range_sum(W w, int V, int& cnt) {
  const int per = (V + kThreads - 1) / kThreads;
  const int i0 = threadIdx.x * per, i1 = min(i0 + per, V);
  float part = 0.f;
  cnt = 0;
  for (int i = i0; i < i1; ++i) {
    const float x = w(i);
    if (x > 0.f) { part += x; ++cnt; }
  }
  return part;
}

struct DrawSmem {
  float scan[kThreads];
  float run;
  int pick;
  bool tail;
  int tok;
};

// Inverse-CDF draw in vocabulary order over the weights w(i) (only w > 0 is drawable) at u * z, z their sum.  Thread 0
// scans the per-thread sums, the picked thread walks its range.  If rounding pushes the target past the end, the draw
// is the last positive entry.  Returns the token (-1 when no weight is positive) and z, and the positive count in
// *n_pos, to every thread.
template <class W>
__device__ __forceinline__ int draw_inverse_cdf(W w, int V, float u, float* red, DrawSmem& sm, float& z, int& n_pos) {
  const int tid = threadIdx.x;
  const int per = (V + kThreads - 1) / kThreads;
  const int i0 = tid * per, i1 = min(i0 + per, V);
  int cnt;
  const float part = range_sum(w, V, cnt);
  sm.scan[tid] = part;
  z = block_reduce(part, false, red);
  n_pos = (int)block_reduce((float)cnt, false, red);
  __syncthreads();
  if (tid == 0) {
    const float target = u * z;
    float run = 0.f;
    int pick = -1;
    for (int t = 0; t < kThreads; ++t) {
      if (run + sm.scan[t] > target) { pick = t; break; }
      run += sm.scan[t];
    }
    // rounding pushed the target past the end of the scan: the draw is the last positive entry (of the last thread
    // with any)
    sm.tail = pick < 0;
    if (pick < 0) {
      pick = kThreads - 1;
      while (pick > 0 && sm.scan[pick] == 0.f) --pick;
    }
    sm.pick = pick;
    sm.run = run;
  }
  __syncthreads();
  if (tid == sm.pick) {
    const float target = u * z;
    float run = sm.run;
    int tok = -1, last = -1;
    for (int i = i0; i < i1; ++i) {
      const float x = w(i);
      if (x > 0.f) {
        last = i;
        run += x;
        if (!sm.tail && run > target) { tok = i; break; }
      }
    }
    sm.tok = tok >= 0 ? tok : last;
  }
  __syncthreads();
  return sm.tok;
}

// Temperature / top-k / top-p sampling, one CTA per row.
template <typename T>
__global__ void __launch_bounds__(kThreads) sample_kernel(const T* __restrict__ logits, int64_t row_stride, int V,
                                                          const float* __restrict__ temperatures,
                                                          const int32_t* __restrict__ top_ks, const float* __restrict__ top_ps,
                                                          const float* __restrict__ uniforms, int64_t* __restrict__ out_tokens,
                                                          int32_t* __restrict__ out_kept, float* __restrict__ out_mass) {
  cb::pdl_prologue();
  __shared__ float red[kThreads / 32];
  __shared__ KeptSmem ks;
  __shared__ DrawSmem ds;
  const int b = blockIdx.x;
  const T* row = logits + (int64_t)b * row_stride;
  const float top_p = top_ps[b];
  const int top_k = top_ks[b] > 0 ? top_ks[b] : V;
  const RowSoftmax sm = row_softmax(row, V, 1.f / temperatures[b], red);
  auto prob = [&](int i) { return row_prob(row, sm, i); };
  const uint32_t thr = kept_threshold(prob, V, top_k, top_p, ks);
  float z;
  int nkept;
  const int tok = draw_inverse_cdf([&](int i) { const float p = prob(i); return kept_p(p, thr) ? p : 0.f; }, V,
                                   uniforms[b], red, ds, z, nkept);
  if (threadIdx.x == 0) {
    out_tokens[b] = tok;
    if (out_kept) out_kept[b] = nkept;
    if (out_mass) out_mass[b] = z;
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

// ---- sampled acceptance of k draft tokens per request (speculative sampling) ----
// Row statistics the row kernel leaves for the acceptance kernel, one per verified row b * (k + 1) + i.
struct SpecRow {
  float mx, inv_sum;      // the row's softmax (sampled requests)
  float inv_z;            // 1 / the kept mass: p_i(x) = prob(x) * inv_z on the kept set
  uint32_t thr;           // the kept set's threshold key
  float p_draft;          // p_i(d_i) (rows i < n_draft[b] of sampled requests; 0 outside the kept set)
  int32_t argmax;         // the first maximal index (greedy requests)
};

// One CTA per verified row; rows past n_draft[b] exit at once.  Greedy requests (T <= 0) take the row's argmax, the
// others its softmax, kept set, kept mass and the target probability of the row's draft.
template <typename T>
__global__ void __launch_bounds__(kThreads, 1) spec_rows_kernel(const T* __restrict__ logits, int64_t row_stride, int V,
                                                             const float* __restrict__ temperatures,
                                                             const int32_t* __restrict__ top_ks,
                                                             const float* __restrict__ top_ps,
                                                             const int64_t* __restrict__ drafts,
                                                             const int32_t* __restrict__ n_draft, int k,
                                                             SpecRow* __restrict__ ws) {
  cb::pdl_prologue();
  __shared__ float red[kThreads / 32];
  __shared__ KeptSmem ks;
  __shared__ float sv[kThreads];
  __shared__ int64_t si[kThreads];
  const int r = blockIdx.x, b = r / (k + 1), i = r % (k + 1);
  const int n = min(max(n_draft[b], 0), k);
  if (i > n) return;
  const T* row = logits + (int64_t)r * row_stride;
  const float temp = temperatures[b];
  if (!(temp > 0.f)) {
    const int64_t best = block_argmax_1024(row, (int64_t)V, sv, si);
    if (threadIdx.x == 0) ws[r].argmax = (int32_t)best;
    return;
  }
  const float top_p = top_ps[b];
  const int top_k = top_ks[b] > 0 ? top_ks[b] : V;
  const RowSoftmax sm = row_softmax(row, V, 1.f / temp, red);
  auto prob = [&](int x) { return row_prob(row, sm, x); };
  const uint32_t thr = kept_threshold(prob, V, top_k, top_p, ks);
  int cnt;
  const float z = block_reduce(range_sum([&](int x) { const float p = prob(x); return kept_p(p, thr) ? p : 0.f; }, V,
                                         cnt), false, red);
  if (threadIdx.x == 0) {
    const float inv_z = 1.f / z;
    float pd = 0.f;
    if (i < n) {
      const int64_t d = drafts[(int64_t)b * k + i];
      if (d >= 0 && d < V) {
        const float p = prob((int)d);
        pd = kept_p(p, thr) ? p * inv_z : 0.f;
      }
    }
    ws[r] = SpecRow{sm.mx, sm.inv_sum, inv_z, thr, pd, -1};
  }
}

// One CTA per request.  It writes seq_lens, which the decode kernels read before their griddepcontrol.wait, so it
// waits for its predecessor and never lets its dependents start early (the rule of decode_prepare_kernel).
template <typename T>
__global__ void __launch_bounds__(kThreads) spec_accept_sampled_kernel(
    const T* __restrict__ logits, int64_t row_stride, int V, const float* __restrict__ temperatures,
    const int64_t* __restrict__ drafts, const int32_t* __restrict__ n_draft, const float* __restrict__ draft_probs,
    int64_t q_stride, const float* __restrict__ u_accept, const float* __restrict__ u_draw,
    const SpecRow* __restrict__ ws, int32_t* __restrict__ seq_lens, int64_t* __restrict__ out_tokens,
    int32_t* __restrict__ accepted, int64_t* __restrict__ next_tokens, int k) {
  cb::pdl_wait();
  __shared__ float red[kThreads / 32];
  __shared__ DrawSmem ds;
  __shared__ int s_a;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int n = min(max(n_draft[b], 0), k);
  const SpecRow* st = ws + (int64_t)b * (k + 1);
  const int64_t* d = drafts + (int64_t)b * k;
  const float temp = temperatures[b];
  const bool greedy = !(temp > 0.f);
  // q_i(x): the caller's row in draft-model mode, one-hot at d_i in token-only mode
  auto q_row = [&](int i) { return draft_probs ? draft_probs + ((int64_t)b * k + i) * q_stride : nullptr; };
  if (tid == 0) {
    int a = 0;
    if (greedy) {
      while (a < n && d[a] == st[a].argmax) ++a;
    } else {
      for (; a < n; ++a) {
        const float* q = q_row(a);
        const float qd = q == nullptr ? 1.f : (d[a] >= 0 && d[a] < V ? q[d[a]] : 0.f);
        const float pd = st[a].p_draft;
        if (!(pd > 0.f && u_accept[(int64_t)b * k + a] * qd < pd)) break;
      }
    }
    s_a = a;
  }
  __syncthreads();
  const int a = s_a;
  int64_t tok;
  if (greedy) {
    tok = st[a].argmax;
  } else {
    const SpecRow sa = st[a];
    const T* row = logits + ((int64_t)b * (k + 1) + a) * row_stride;
    const RowSoftmax sm{1.f / temp, sa.mx, sa.inv_sum};
    auto p_w = [&](int x) { const float p = row_prob(row, sm, x); return kept_p(p, sa.thr) ? p : 0.f; };
    const float u = u_draw[b];
    float z;
    int cnt;
    int t = -1;
    if (a < n) {                         // the residual max(p_a - q_a, 0)
      const float* q = q_row(a);
      const int64_t da = d[a];
      t = draw_inverse_cdf([&](int x) {
        const float qx = q == nullptr ? (x == da ? 1.f : 0.f) : q[x];
        return fmaxf(p_w(x) * sa.inv_z - qx, 0.f);
      }, V, u, red, ds, z, cnt);
    } else {
      z = 0.f;
    }
    if (!(z > 0.f)) t = draw_inverse_cdf(p_w, V, u, red, ds, z, cnt);   // all drafts accepted, or a residual of mass 0
    tok = t;
  }
  if (tid == 0) {
    int64_t* o = out_tokens + (int64_t)b * (k + 1);
    for (int i = 0; i <= k; ++i) o[i] = i < a ? d[i] : (i == a ? tok : -1);
    accepted[b] = a;
    next_tokens[b] = tok;
    seq_lens[b] += a + 1;
  }
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

extern "C" int64_t chitu_b200_spec_accept_sampled_workspace_bytes(int B, int k) {
  return B < 0 || k < 0 ? 0 : (int64_t)B * (k + 1) * (int64_t)sizeof(SpecRow);
}

// logits [B * (k + 1), V] (row stride in elements), bf16 / fp16 / fp32; temperatures, top_ps fp32 [B] (T <= 0: greedy);
// top_ks int32 [B] (<= 0: no top-k); drafts int64 [B, k]; n_draft int32 [B] (clamped to 0..k); draft_probs fp32, row
// [b, i] at (b * k + i) * draft_probs_stride, or NULL (token-only drafts); u_accept fp32 [B, k], u_draw fp32 [B] in
// [0, 1); seq_lens int32 [B] (in place); out_tokens int64 [B, k + 1], accepted int32 [B], next_tokens int64 [B].
extern "C" int chitu_b200_spec_accept_sampled(const void* logits, int64_t row_stride, int V, int dtype,
                                              const float* temperatures, const int32_t* top_ks, const float* top_ps,
                                              const int64_t* drafts, const int32_t* n_draft, const float* draft_probs,
                                              int64_t draft_probs_stride, const float* u_accept, const float* u_draw,
                                              int32_t* seq_lens, int64_t* out_tokens, int32_t* accepted,
                                              int64_t* next_tokens, int B, int k, void* workspace,
                                              int64_t workspace_bytes, void* stream) {
  CB_ARG(logits && temperatures && top_ks && top_ps && drafts && n_draft && u_accept && u_draw && seq_lens &&
         out_tokens && accepted && next_tokens && workspace && B >= 0 && k >= 1 && V > 0 && row_stride >= V);
  CB_ARG(draft_probs == nullptr || draft_probs_stride >= V);
  CB_ARG(workspace_bytes >= chitu_b200_spec_accept_sampled_workspace_bytes(B, k));
  if (B == 0) return 0;
  const int rc = cb::dispatch_dtype<CB_BF16, CB_F16, CB_F32>(__func__, dtype, [&](auto t) {
    using T = decltype(t);
    const cudaStream_t st = (cudaStream_t)stream;
    SpecRow* ws = (SpecRow*)workspace;
    cb::launch_k(spec_rows_kernel<T>, dim3(B * (k + 1)), dim3(kThreads), 0, st, (const T*)logits, row_stride, V,
                 temperatures, top_ks, top_ps, drafts, n_draft, k, ws);
    cb::launch_k(spec_accept_sampled_kernel<T>, dim3(B), dim3(kThreads), 0, st, (const T*)logits, row_stride, V,
                 temperatures, drafts, n_draft, draft_probs, draft_probs_stride, u_accept, u_draw,
                 (const SpecRow*)ws, seq_lens, out_tokens, accepted, next_tokens, k);
    return 0;
  });
  if (rc) return rc;
  CB_LAUNCHED(2);
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
