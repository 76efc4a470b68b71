// MoE: DeepSeek gate (routing) and fused experts.
//
//  * moe_gate       : GateDeepSeekV3.forward (model_deepseek_v3.py:810-842) as ONE kernel
//                     (the reference issues ~12 torch kernels: linear, sigmoid, +bias, view,
//                     topk(2).sum, topk groups, scatter mask, mul, topk, gather, normalise, scale).
//  * fused_experts  : fused_moe.py:1060-1307 (align -> quant -> GEMM1 -> SiluAndMul -> quant ->
//                     GEMM2 x routed weight -> sum over top-k).  Decode batches give 1-2 tokens
//                     per expert, so each (token, slot) pair streams its expert's weight rows once:
//                     a batched weight-streaming GEMV (the grouped wgmma path lives in
//                     gemm_tc.cu and is selected for larger token counts per expert).
#include <string.h>

#include "common.cuh"
#include "gemm.cuh"
#include "tc_ptx.cuh"

using namespace cb;

namespace {

inline int64_t align256(int64_t v) { return (v + 255) / 256 * 256; }

__device__ __forceinline__ float round_bf16(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

struct MoePlan {
  int* pair_sorted;   // [P]   pair index (t*topk + j) of sorted row r
  int* pos;           // [P]   sorted row of pair p
  int* seg_start;     // [E+1]
  int* num_tiles1;    // [1]   active tiles of GEMM1 (= active experts * N1/128)
  int* tile1_wrow;    // [E*N1/128]
  int* tile1_xrow;
  int* tile1_cnt;
  int* num_tiles2;
  int* tile2_wrow;    // [E*K1/128]
  int* tile2_xrow;
  int* tile2_cnt;
  float* w_sorted;    // [P] routed weight of sorted row r
};

// The plan itself, run by one CTA of kPlanThreads threads.  `sm` needs moe_plan_smem_ints(P, E) ints.  E <= kPlanThreads:
// a thread owns one expert in the block-wide scans.
constexpr int kPlanThreads = 1024;
__host__ __device__ constexpr int64_t moe_plan_smem_ints(int64_t P, int E) { return 3 * (int64_t)E + 2 + 2 * P + 2 * (E + P / 16 + 2); }

template <typename IdT>
__device__ __forceinline__ void moe_plan_large(const IdT* ids, const void* topk_w, int topk_w_f32,
                                               int P, int E, int N1, int K1, int BN, const MoePlan& pl, int* sm) {
  constexpr int NT = kPlanThreads, NW = NT / 32;
  int* cnt = sm;              // [E]
  int* start = sm + E;        // [E+1]
  int* act = start + E + 1;   // [E] first row chunk (of BN sorted rows) of the expert among all chunks
  int* sid = act + E;         // [P] expert id of every pair (read once from global)
  float* swt = reinterpret_cast<float*>(sid + P);   // [P] routed weight of every pair: a global load inside the scatter
                                                    // loop below stalled its warp for an L2 round trip per hit
  __shared__ int s_wsum[32], s_wact[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int e = tid; e < E; e += NT) cnt[e] = 0;
  for (int p = tid; p < P; p += NT) {
    sid[p] = (int)ids[p];
    swt[p] = topk_w_f32 ? reinterpret_cast<const float*>(topk_w)[p]
                        : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(topk_w)[p]);
  }
  __syncthreads();
  for (int p = tid; p < P; p += NT) {
    const int e = sid[p];
    if (e >= 0 && e < E) atomicAdd(&cnt[e], 1);
    else pl.pos[p] = -1;      // expert not on this rank (expert_map == -1)
  }
  __syncthreads();
  // block-wide exclusive scan of cnt[] and of the row-chunk counts (E <= 1024).  An expert with more than BN routed rows
  // (bs > 128, or the shared expert that every token visits) is cut into chunks of BN rows: each chunk is a tile column
  // of the grouped GEMM (its weight tile is re-read per chunk, mostly from L2).
  const int c = tid < E ? cnt[tid] : 0, ch = (c + BN - 1) / BN;
  int ci = c, ai = ch;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int n1 = __shfl_up_sync(0xffffffffu, ci, o), n2 = __shfl_up_sync(0xffffffffu, ai, o);
    if (lane >= o) { ci += n1; ai += n2; }
  }
  if (lane == 31) { s_wsum[warp] = ci; s_wact[warp] = ai; }
  __syncthreads();
  int woff = 0, aoff = 0, na = 0, tot = 0;
  for (int w = 0; w < NW; ++w) {
    if (w < warp) { woff += s_wsum[w]; aoff += s_wact[w]; }
    na += s_wact[w];
    tot += s_wsum[w];
  }
  const int run_c = woff + ci - c, run_a = aoff + ai - ch;    // exclusive prefixes of this thread's expert
  if (tid < E) {
    start[tid] = run_c;
    act[tid] = ch ? run_a : -1;
    pl.seg_start[tid] = run_c;
  }
  if (tid == 0) {
    pl.seg_start[E] = tot;    // pairs with absent experts excluded
    *pl.num_tiles1 = na * (N1 / 128);
    *pl.num_tiles2 = na * (K1 / 128);
  }
  __syncthreads();
  // stable scatter: one warp per active expert, ballot-compaction over the pairs in order
  for (int e = warp; e < E; e += NW) {
    const int n = cnt[e];
    if (n == 0) continue;
    int r = start[e];
    for (int p0 = 0; p0 < P; p0 += 32) {
      const int p = p0 + lane;
      const bool hit = p < P && sid[p] == e;
      const unsigned bal = __ballot_sync(0xffffffffu, hit);
      if (hit) {
        const int rr = r + __popc(bal & ((1u << lane) - 1u));
        pl.pair_sorted[rr] = p;
        pl.pos[p] = rr;
        pl.w_sorted[rr] = swt[p];
      }
      r += __popc(bal);
    }
    const int ar = act[e], nch = (n + BN - 1) / BN;
    for (int cc = 0; cc < nch; ++cc) {
      const int xrow = start[e] + cc * BN, rows = min(BN, n - cc * BN);
      for (int i = lane; i < N1 / 128; i += 32) {
        const int ti = (ar + cc) * (N1 / 128) + i;
        pl.tile1_wrow[ti] = e * N1 + i * 128;
        pl.tile1_xrow[ti] = xrow;
        pl.tile1_cnt[ti] = rows;
      }
      for (int i = lane; i < K1 / 128; i += 32) {
        const int ti = (ar + cc) * (K1 / 128) + i;
        pl.tile2_wrow[ti] = e * K1 + i * 128;
        pl.tile2_xrow[ti] = xrow;
        pl.tile2_cnt[ti] = rows;
      }
    }
  }
}

// Decode-sized plans (P <= 1024 pairs): every phase is parallel over PAIRS or over TILE-LIST ENTRIES instead of one warp
// per expert.  In-graph probes of the per-expert version at bs = 16 (144 pairs, ~100 active experts): 1.0 us staging, 1.9 us
// scan, 4.6 - 7 us scatter + tile lists = 10 us after the dependency wait; the same
// stable order (pairs of an expert keep their pair-index order), so every output array is identical.
template <typename IdT>
__device__ __forceinline__ void moe_plan_small(const IdT* ids, const void* topk_w, int topk_w_f32,
                                               int P, int E, int N1, int K1, int BN, const MoePlan& pl, int* sm) {
  constexpr int NT = kPlanThreads, NW = NT / 32;
  int* cnt = sm;              // [E]
  int* start = sm + E;        // [E+1]
  int* act = start + E + 1;   // [E] first row chunk of the expert among all chunks, -1 = no rows
  int* sid = act + E;         // [P]
  float* swt = reinterpret_cast<float*>(sid + P);          // [P]
  int* chunk_e = reinterpret_cast<int*>(swt + P);          // [<= E + P/16 + 1] expert of every active chunk
  int* chunk_c = chunk_e + (E + P / 16 + 2);               //                    its chunk number inside the expert
  __shared__ int s_wsum[32], s_wact[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int e = tid; e < E; e += NT) cnt[e] = 0;
  for (int p = tid; p < P; p += NT) {
    sid[p] = (int)ids[p];
    swt[p] = topk_w_f32 ? reinterpret_cast<const float*>(topk_w)[p]
                        : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(topk_w)[p]);
  }
  __syncthreads();
  // histogram + the pair's rank among the earlier pairs of the same expert (stable order), one pass over shared memory;
  // thread p owns pair p
  int my_rank = -1;
  if (tid < P) {
    const int e = sid[tid];
    if (e >= 0 && e < E) {
      atomicAdd(&cnt[e], 1);
      int r = 0;
      for (int q = 0; q < tid; ++q) r += (sid[q] == e);
      my_rank = r;
    } else {
      pl.pos[tid] = -1;       // expert not on this rank (expert_map == -1)
    }
  }
  __syncthreads();
  // block-wide exclusive scan of the counts and of the row-chunk counts (E <= 1024)
  const int c = tid < E ? cnt[tid] : 0, ch = (c + BN - 1) / BN;
  int ci = c, ai = ch;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int n1 = __shfl_up_sync(0xffffffffu, ci, o), n2 = __shfl_up_sync(0xffffffffu, ai, o);
    if (lane >= o) { ci += n1; ai += n2; }
  }
  if (lane == 31) { s_wsum[warp] = ci; s_wact[warp] = ai; }
  __syncthreads();
  // every warp scans the NW warp totals with shuffles (no serial loop over shared memory)
  int wt = lane < NW ? s_wsum[lane] : 0, at = lane < NW ? s_wact[lane] : 0;
  int wi = wt, aii = at;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int n1 = __shfl_up_sync(0xffffffffu, wi, o), n2 = __shfl_up_sync(0xffffffffu, aii, o);
    if (lane >= o) { wi += n1; aii += n2; }
  }
  const int tot = __shfl_sync(0xffffffffu, wi, 31), na = __shfl_sync(0xffffffffu, aii, 31);
  const int woff = __shfl_sync(0xffffffffu, wi - wt, warp), aoff = __shfl_sync(0xffffffffu, aii - at, warp);
  const int run_c = woff + ci - c, run_a = aoff + ai - ch;    // exclusive prefixes of this thread's expert
  if (tid < E) {
    start[tid] = run_c;
    act[tid] = ch ? run_a : -1;
    pl.seg_start[tid] = run_c;
#pragma unroll 1
    for (int cc = 0; cc < ch; ++cc) { chunk_e[run_a + cc] = tid; chunk_c[run_a + cc] = cc; }
  }
  if (tid == 0) {
    pl.seg_start[E] = tot;    // pairs with absent experts excluded
    *pl.num_tiles1 = na * (N1 / 128);
    *pl.num_tiles2 = na * (K1 / 128);
  }
  __syncthreads();
  // one thread per pair: its sorted row
  if (my_rank >= 0) {
    const int rr = start[sid[tid]] + my_rank;
    pl.pair_sorted[rr] = tid;
    pl.pos[tid] = rr;
    pl.w_sorted[rr] = swt[tid];
  }
  // one thread per tile-list entry of either GEMM
  const int t1 = N1 / 128, t2 = K1 / 128, per = t1 + t2;
  for (int wk = tid; wk < na * per; wk += NT) {
    const int g = wk / per, i = wk - g * per;
    const int e = chunk_e[g], cc = chunk_c[g];
    const int xrow = start[e] + cc * BN, rows = min(BN, cnt[e] - cc * BN);
    if (i < t1) {
      const int ti = g * t1 + i;
      pl.tile1_wrow[ti] = e * N1 + i * 128;
      pl.tile1_xrow[ti] = xrow;
      pl.tile1_cnt[ti] = rows;
    } else {
      const int i2 = i - t1, ti = g * t2 + i2;
      pl.tile2_wrow[ti] = e * K1 + i2 * 128;
      pl.tile2_xrow[ti] = xrow;
      pl.tile2_cnt[ti] = rows;
    }
  }
}

// --------------------------------------------------------------------------------------------
// gate: one CTA (256 threads) per token.
// dtype pipeline reproduced from the reference (x, W bf16):
//   logits = bf16(F.linear)                       -> sigmoid -> bf16  (original_scores)
//   scores = original + bias  (bf16 if bias is bf16, fp32 if bias is fp32: torch promotion; softmax scores are fp32, so
//                              any bias is an fp32 add there)
//   group score = sum of top-2 (in that dtype), keep top `topk_groups` groups, others * 0
//   indices = top-k of masked scores (ties -> lowest index), weights = original.gather,
//   /= sum (bf16), *= route_scale (bf16).
// softmax variant (score mode 0): scores = softmax(logits, fp32); no normalisation; group score = amax if no bias.
// score mode 2 (SparseMoeBlockHFMixtral, model_hf_mixtral.py:57-64): softmax(fp32), top-k, weights /= sum in fp32, cast.
// --------------------------------------------------------------------------------------------
// monotone map float -> uint32 (larger float <=> larger key, -0 == +0, every finite / infinite value > 0)
__device__ __forceinline__ uint32_t ordered_key(float v) {
  const uint32_t u = __float_as_uint(v + 0.f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Gate logits for a decode batch (T <= 16): logits[t, e] = bf16(sum_k x[t,k] w[e,k]), fp32 accumulation.  One CTA per PAIR of
// experts streams its two weight rows ONCE (prefetched before griddepcontrol.wait: weights are immutable) against all T
// rows of x (L2-resident, 2 T dim bytes).  The tensor-core GEMM would have only E / 128 = 2 weight tiles to share among
// all SMs: a 66-way split-K and a fix-up of 66 partial tiles for 3.7 MB of weights.
constexpr int kGateVecIters = 4;      // 256 threads x 4 x 8 elements: dim <= 8192
template <int TB>
__global__ void __launch_bounds__(256) gate_logits_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                                                         __nv_bfloat16* __restrict__ logits, int T, int dim, int E) {
  cb::pdl_launch_dependents();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int e0 = blockIdx.x * 2;
  const int nvec = dim >> 3;
  uint4 wv[2][kGateVecIters];
#pragma unroll
  for (int it = 0; it < kGateVecIters; ++it) {
    const int v = it * 256 + tid;
#pragma unroll
    for (int ee = 0; ee < 2; ++ee)
      wv[ee][it] = (v < nvec && e0 + ee < E) ? ld_stream(w + (int64_t)(e0 + ee) * dim + v * 8) : make_uint4(0, 0, 0, 0);
  }
  cb::pdl_wait();
  cb::tl_stamp();
  float acc[2][TB];
#pragma unroll
  for (int ee = 0; ee < 2; ++ee)
#pragma unroll
    for (int t = 0; t < TB; ++t) acc[ee][t] = 0.f;
#pragma unroll
  for (int it = 0; it < kGateVecIters; ++it) {
    const int v = it * 256 + tid;
    if (v >= nvec) break;
    const uint32_t w0[4] = {wv[0][it].x, wv[0][it].y, wv[0][it].z, wv[0][it].w};
    const uint32_t w1[4] = {wv[1][it].x, wv[1][it].y, wv[1][it].z, wv[1][it].w};
#pragma unroll
    for (int t0 = 0; t0 < TB; t0 += 4) {
      uint4 xv[4];
#pragma unroll
      for (int tt = 0; tt < 4; ++tt)
        xv[tt] = (t0 + tt < TB && t0 + tt < T) ? *reinterpret_cast<const uint4*>(x + (int64_t)(t0 + tt) * dim + v * 8)
                                                : make_uint4(0, 0, 0, 0);
#pragma unroll
      for (int tt = 0; tt < 4; ++tt) {
        if (t0 + tt >= TB) break;
        const uint32_t xu[4] = {xv[tt].x, xv[tt].y, xv[tt].z, xv[tt].w};
        float a0 = acc[0][t0 + tt], a1 = acc[1][t0 + tt];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float xl = bf16lo(xu[j]), xh = bf16hi(xu[j]);
          a0 = fmaf(xl, bf16lo(w0[j]), a0);
          a0 = fmaf(xh, bf16hi(w0[j]), a0);
          a1 = fmaf(xl, bf16lo(w1[j]), a1);
          a1 = fmaf(xh, bf16hi(w1[j]), a1);
        }
        acc[0][t0 + tt] = a0;
        acc[1][t0 + tt] = a1;
      }
    }
  }
  __shared__ float red[8][2 * TB];
#pragma unroll
  for (int ee = 0; ee < 2; ++ee)
#pragma unroll
    for (int t = 0; t < TB; ++t) {
      const float sum = warp_sum(acc[ee][t]);
      if (lane == 0) red[warp][ee * TB + t] = sum;
    }
  __syncthreads();
  if (tid < 2 * TB) {
    float tot = 0.f;
#pragma unroll
    for (int wi = 0; wi < 8; ++wi) tot += red[wi][tid];
    const int ee = tid / TB, t = tid - ee * TB;
    if (t < T && e0 + ee < E) logits[(int64_t)t * E + e0 + ee] = __float2bfloat16_rn(tot);
  }
}

__global__ void __launch_bounds__(256) moe_gate_kernel(
    const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w, const void* __restrict__ bias,
    int bias_is_f32, int dim, int E, int n_groups, int topk_groups, int topk, int score_sigmoid,
    float route_scale, __nv_bfloat16* __restrict__ out_w, int64_t* __restrict__ out_idx,
    const __nv_bfloat16* __restrict__ logits, int out_stride) {
  cb::pdl_prologue();
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __nv_bfloat16* sx = reinterpret_cast<__nv_bfloat16*>(smem_raw);                 // [dim]
  float* s_orig = reinterpret_cast<float*>(smem_raw + (size_t)dim * 2);           // [E]
  float* s_score = s_orig + E;                                                    // [E]
  float* s_group = s_score + E;                                                   // [n_groups]
  int* s_sel = reinterpret_cast<int*>(s_group + n_groups);                        // [topk]
  const int t = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (logits) {
    // logits = F.linear(x, W) were produced by the wgmma GEMM (bf16, as the reference's are)
    for (int e = tid; e < E; e += 256) s_orig[e] = __bfloat162float(logits[(int64_t)t * E + e]);
  } else {
    for (int i = tid; i < dim / 8; i += 256)
      reinterpret_cast<uint4*>(sx)[i] = reinterpret_cast<const uint4*>(x + (int64_t)t * dim)[i];
    __syncthreads();
    for (int e = warp; e < E; e += 8) {
      const __nv_bfloat16* wr = w + (int64_t)e * dim;
      float acc = 0.f;
      for (int k = lane * 8; k < dim; k += 256) {
        uint4 wv = *reinterpret_cast<const uint4*>(wr + k);
        uint4 xv = *reinterpret_cast<const uint4*>(sx + k);
        const uint32_t ww[4] = {wv.x, wv.y, wv.z, wv.w}, xx[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          acc = fmaf(bf16lo(ww[i]), bf16lo(xx[i]), acc);
          acc = fmaf(bf16hi(ww[i]), bf16hi(xx[i]), acc);
        }
      }
      acc = warp_sum(acc);
      if (lane == 0) s_orig[e] = round_bf16(acc);   // F.linear output is bf16
    }
  }
  __syncthreads();

  if (score_sigmoid == 1) {
    for (int e = tid; e < E; e += 256) {
      float v = s_orig[e];
      s_orig[e] = round_bf16(1.f / (1.f + expf(-v)));
    }
  } else {
    // softmax over E in fp32 (scores.softmax(dim=-1, dtype=torch.float32))
    __shared__ float red[8];
    float mx = -INFINITY;
    for (int e = tid; e < E; e += 256) mx = fmaxf(mx, s_orig[e]);
    mx = warp_max(mx);
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    mx = red[0];
    for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
    __syncthreads();
    float sum = 0.f;
    for (int e = tid; e < E; e += 256) {
      float v = expf(s_orig[e] - mx);
      s_orig[e] = v;
      sum += v;
    }
    sum = warp_sum(sum);
    if (lane == 0) red[warp] = sum;
    __syncthreads();
    sum = 0.f;
    for (int i = 0; i < 8; ++i) sum += red[i];
    for (int e = tid; e < E; e += 256) s_orig[e] = s_orig[e] / sum;
  }
  __syncthreads();
  const bool low_prec = score_sigmoid == 1 && !(bias && bias_is_f32);   // score dtype is bf16
  for (int e = tid; e < E; e += 256) {
    float v = s_orig[e];
    if (bias) {
      // bf16 scores + bf16 bias is a bf16 add; softmax scores are fp32, so a bf16 bias promotes to an fp32 add
      const float b = bias_is_f32 ? reinterpret_cast<const float*>(bias)[e]
                                  : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(bias)[e]);
      v = low_prec ? round_bf16(v + b) : v + b;
    }
    s_score[e] = v;
  }
  __syncthreads();

  if (n_groups > 1) {
    const int gs = E / n_groups;
    for (int g = warp; g < n_groups; g += 8) {
      // top-2 (or max) inside the group by warp argmax passes
      float best1 = -INFINITY; int i1 = -1;
      for (int e = lane; e < gs; e += 32) { float v = s_score[g * gs + e]; if (v > best1) { best1 = v; i1 = e; } }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        float ov = __shfl_xor_sync(0xffffffffu, best1, o); int oi = __shfl_xor_sync(0xffffffffu, i1, o);
        if (ov > best1 || (ov == best1 && oi >= 0 && (i1 < 0 || oi < i1))) { best1 = ov; i1 = oi; }
      }
      float gscore = best1;
      if (bias) {
        float best2 = -INFINITY;
        for (int e = lane; e < gs; e += 32) { float v = s_score[g * gs + e]; if (e != i1 && v > best2) best2 = v; }
        best2 = warp_max(best2);
        gscore = best1 + best2;
        if (low_prec) gscore = round_bf16(gscore);
      }
      if (lane == 0) s_group[g] = gscore;
    }
    __syncthreads();
    if (n_groups <= 32) {
      // choose topk_groups groups (ties -> lowest index): lane g owns group g, one redux.max + redux.min per pick
      if (warp == 0) {
        const bool mine = lane < n_groups;
        const uint32_t gkey = mine ? ordered_key(s_group[lane]) : 0u;
        bool kept = false;
        for (int r = 0; r < topk_groups; ++r) {
          const uint32_t k = (mine && !kept) ? gkey : 0u;
          const uint32_t mx = __reduce_max_sync(0xffffffffu, k);
          const uint32_t win = __reduce_min_sync(0xffffffffu, (mine && !kept && k == mx) ? (uint32_t)lane : 64u);
          if ((uint32_t)lane == win) kept = true;
        }
        if (mine) s_group[lane] = kept ? 1.f : 0.f;
      }
    } else if (tid == 0) {
      // choose topk_groups groups (ties -> lowest index); mark the rest with -1
      unsigned long long keep = 0ull;
      for (int r = 0; r < topk_groups; ++r) {
        float best = -INFINITY; int bi = -1;
        for (int g = 0; g < n_groups; ++g)
          if (!((keep >> g) & 1ull) && (bi < 0 || s_group[g] > best)) { best = s_group[g]; bi = g; }
        keep |= 1ull << bi;
      }
      for (int g = 0; g < n_groups; ++g) s_group[g] = ((keep >> g) & 1ull) ? 1.f : 0.f;
    }
    __syncthreads();
    for (int e = tid; e < E; e += 256) s_score[e] = s_score[e] * s_group[e / gs];   // masked -> (+-)0
    __syncthreads();
  }

  // top-k over the masked scores: warp 0, k argmax passes, ties -> lowest index
  if (warp == 0) {
    if (E <= 256) {
      // scores live in registers (element i*32 + lane); a pick is a local scan + redux.max + redux.min
      uint32_t key[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int e = i * 32 + lane;
        key[i] = e < E ? ordered_key(s_score[e]) : 0u;
      }
      for (int r = 0; r < topk; ++r) {
        uint32_t bk = 0u; int be = 0x7fffffff;
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (key[i] > bk) { bk = key[i]; be = i * 32 + lane; }
        const uint32_t mx = __reduce_max_sync(0xffffffffu, bk);
        const uint32_t win = __reduce_min_sync(0xffffffffu, (bk == mx && bk != 0u) ? (uint32_t)be : 0x7fffffffu);
        if (lane == 0) s_sel[r] = (int)win;
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if ((uint32_t)(i * 32 + lane) == win) key[i] = 0u;
      }
      __syncwarp();
    } else
    for (int r = 0; r < topk; ++r) {
      float best = -INFINITY; int bi = 0x7fffffff;
      for (int e = lane; e < E; e += 32) {
        float v = s_score[e];
        bool taken = false;
        for (int q = 0; q < r; ++q) taken |= (s_sel[q] == e);
        if (!taken && (v > best || (v == best && e < bi))) { best = v; bi = e; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        float ov = __shfl_xor_sync(0xffffffffu, best, o); int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
      }
      if (lane == 0) s_sel[r] = bi;
      __syncwarp();
    }
    // weights
    const float w_mine = lane < topk ? s_orig[s_sel[lane]] : 0.f;
    float wsum = 0.f;
    for (int r = 0; r < topk; ++r) wsum += __shfl_sync(0xffffffffu, w_mine, r);   // r = 0, 1, ... order (fp32 sum)
    if (score_sigmoid == 1) wsum = round_bf16(wsum);
    for (int r = lane; r < topk; r += 32) {
      float wv = s_orig[s_sel[r]];
      if (score_sigmoid == 1) wv = round_bf16(wv / wsum);
      else if (score_sigmoid == 2) wv = wv / wsum;          // Mixtral: fp32 renormalisation, one rounding at the cast
      wv = wv * route_scale;
      if (score_sigmoid == 1) wv = round_bf16(wv);
      out_w[(int64_t)t * out_stride + r] = __float2bfloat16_rn(wv);
      out_idx[(int64_t)t * out_stride + r] = s_sel[r];
    }
  }
}

// --------------------------------------------------------------------------------------------
// batched expert GEMV: blockIdx.y = (token, slot) pair; the pair's expert picks the weight slab.
//   MODE 0: bf16 weights x bf16 activations
//   MODE 1: fp8 weights x fp8 activations, 128x128 / 1x128 block scales (fused_moe.py:277-281)
//   MODE 2: soft fp8 (fp8 weights -> bf16) x bf16 activations (fused_moe.py:234-276)
// a_row = pair / a_div (GEMM1: a_div = top_k, GEMM2: a_div = 1); c row = pair.
// --------------------------------------------------------------------------------------------
template <typename IdT>
__device__ __forceinline__ int load_id(const void* p, int i) { return (int)reinterpret_cast<const IdT*>(p)[i]; }

template <int MODE>
__global__ void __launch_bounds__(256) moe_pair_gemv_kernel(
    const void* __restrict__ a, const float* __restrict__ a_s, const uint8_t* __restrict__ w,
    const float* __restrict__ w_s, const void* __restrict__ topk_ids, int ids_i64,
    const void* __restrict__ topk_w, int topk_w_f32, int mul_routed, int a_div, int E, int N, int K,
    __nv_bfloat16* __restrict__ c) {
  cb::pdl_prologue();
  const int pair = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n0 = (blockIdx.x * 8 + warp) * 2;
  if (n0 >= N) return;
  const int n1 = min(n0 + 1, N - 1);
  const int e = ids_i64 ? load_id<int64_t>(topk_ids, pair) : load_id<int32_t>(topk_ids, pair);
  if (e < 0 || e >= E) {   // expert not on this rank (expert_map == -1): zeros (fused_moe.py:160-176)
    if (lane == 0) {
      c[(int64_t)pair * N + n0] = __float2bfloat16_rn(0.f);
      if (n0 + 1 < N) c[(int64_t)pair * N + n1] = __float2bfloat16_rn(0.f);
    }
    return;
  }
  const int arow = pair / a_div;
  const int kblocks = (K + 127) / 128, nblocks = (N + 127) / 128;
  float acc0 = 0.f, acc1 = 0.f;
  if (MODE == 0) {
    const __nv_bfloat16* wb = reinterpret_cast<const __nv_bfloat16*>(w) + (int64_t)e * N * K;
    const __nv_bfloat16* ar = reinterpret_cast<const __nv_bfloat16*>(a) + (int64_t)arow * K;
#pragma unroll 2
    for (int k = lane * 8; k < K; k += 256) {
      uint4 wa = ld_stream(wb + (int64_t)n0 * K + k), wc = ld_stream(wb + (int64_t)n1 * K + k);
      uint4 xv = *reinterpret_cast<const uint4*>(ar + k);
      const uint32_t w0[4] = {wa.x, wa.y, wa.z, wa.w}, w1[4] = {wc.x, wc.y, wc.z, wc.w}, xx[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        acc0 = fmaf(bf16lo(w0[i]), bf16lo(xx[i]), acc0); acc0 = fmaf(bf16hi(w0[i]), bf16hi(xx[i]), acc0);
        acc1 = fmaf(bf16lo(w1[i]), bf16lo(xx[i]), acc1); acc1 = fmaf(bf16hi(w1[i]), bf16hi(xx[i]), acc1);
      }
    }
  } else {
    const uint8_t* wb = w + (int64_t)e * N * K;
    const float* ws0 = w_s + ((int64_t)e * nblocks + n0 / 128) * kblocks;
    const float* ws1 = w_s + ((int64_t)e * nblocks + n1 / 128) * kblocks;
    if (MODE == 1) {
      const uint8_t* ar = reinterpret_cast<const uint8_t*>(a) + (int64_t)arow * K;
      const float* as = a_s + (int64_t)arow * kblocks;
#pragma unroll 2
      for (int k = lane * 16; k < K; k += 512) {
        uint4 wa = ld_stream(wb + (int64_t)n0 * K + k), wc = ld_stream(wb + (int64_t)n1 * K + k);
        uint4 av = *reinterpret_cast<const uint4*>(ar + k);
        const int kb = k >> 7;
        const uint32_t w0[4] = {wa.x, wa.y, wa.z, wa.w}, w1[4] = {wc.x, wc.y, wc.z, wc.w}, aa[4] = {av.x, av.y, av.z, av.w};
        float p0 = 0.f, p1 = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float2 a0 = fp8x2_to_float2((uint16_t)(aa[i] & 0xffff)), a1 = fp8x2_to_float2((uint16_t)(aa[i] >> 16));
          float2 u0 = fp8x2_to_float2((uint16_t)(w0[i] & 0xffff)), u1 = fp8x2_to_float2((uint16_t)(w0[i] >> 16));
          float2 v0 = fp8x2_to_float2((uint16_t)(w1[i] & 0xffff)), v1 = fp8x2_to_float2((uint16_t)(w1[i] >> 16));
          p0 = fmaf(u0.x, a0.x, p0); p0 = fmaf(u0.y, a0.y, p0); p0 = fmaf(u1.x, a1.x, p0); p0 = fmaf(u1.y, a1.y, p0);
          p1 = fmaf(v0.x, a0.x, p1); p1 = fmaf(v0.y, a0.y, p1); p1 = fmaf(v1.x, a1.x, p1); p1 = fmaf(v1.y, a1.y, p1);
        }
        const float sa = as[kb];
        acc0 = fmaf(p0 * sa, ws0[kb], acc0);
        acc1 = fmaf(p1 * sa, ws1[kb], acc1);
      }
    } else {
      const __nv_bfloat16* ar = reinterpret_cast<const __nv_bfloat16*>(a) + (int64_t)arow * K;
      const float two120 = __uint_as_float(0x7B800000u);
      for (int k = lane * 16; k < K; k += 512) {
        uint4 wa = ld_stream(wb + (int64_t)n0 * K + k), wc = ld_stream(wb + (int64_t)n1 * K + k);
        const uint4* ap = reinterpret_cast<const uint4*>(ar + k);
        uint4 a0 = ap[0], a1 = ap[1];
        const int kb = k >> 7;
        const float s0 = ws0[kb] * two120, s1 = ws1[kb] * two120;
        const uint32_t w0[4] = {wa.x, wa.y, wa.z, wa.w}, w1[4] = {wc.x, wc.y, wc.z, wc.w};
        const uint32_t av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const uint32_t b0 = (w0[i >> 2] >> ((i & 3) * 8)) & 0xffu, b1 = (w1[i >> 2] >> ((i & 3) * 8)) & 0xffu;
          const float f0 = round_bf16(__uint_as_float(((b0 & 0x80u) << 24) | ((b0 & 0x7fu) << 20)) * s0);
          const float f1 = round_bf16(__uint_as_float(((b1 & 0x80u) << 24) | ((b1 & 0x7fu) << 20)) * s1);
          const float xa = (i & 1) ? bf16hi(av[i >> 1]) : bf16lo(av[i >> 1]);
          acc0 = fmaf(f0, xa, acc0);
          acc1 = fmaf(f1, xa, acc1);
        }
      }
    }
  }
  acc0 = warp_sum(acc0);
  acc1 = warp_sum(acc1);
  if (lane == 0) {
    if (mul_routed) {
      const float rw = topk_w_f32 ? reinterpret_cast<const float*>(topk_w)[pair]
                                  : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(topk_w)[pair]);
      acc0 *= rw;
      acc1 *= rw;
    }
    c[(int64_t)pair * N + n0] = __float2bfloat16_rn(acc0);
    if (n0 + 1 < N) c[(int64_t)pair * N + n1] = __float2bfloat16_rn(acc1);
  }
}

// out[t, :] = sum_j c3[t, j, :]  (fp32 accumulate, one rounding: torch.sum(dim=1) on bf16)
__global__ void moe_sum_kernel(const __nv_bfloat16* __restrict__ c3, __nv_bfloat16* __restrict__ out, int T,
                               int topk, int K) {
  cb::pdl_prologue();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (int64_t)T * K;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = i / K;
    const int k = (int)(i - t * K);
    float s = 0.f;
    for (int j = 0; j < topk; ++j) s += __bfloat162float(c3[(t * topk + j) * K + k]);
    out[i] = __float2bfloat16_rn(s);
  }
}

// --------------------------------------------------------------------------------------------
// Grouped-GEMM path of fused_experts (tokens sorted by expert, every distinct expert's weights are
// streamed ONCE by the wgmma stream-K kernel of gemm_tc.cu):
//   moe_plan_kernel        counting sort of the (token, slot) pairs by expert (stable, deterministic)
//                          + the active (expert, n-tile) lists of both GEMMs
//   moe_gather_quant_kernel  xs[r] = quant(x[pair_sorted[r] / topk])   (per_token_group_quant_fp8)
//   moe_silu_quant_kernel    a2[r] = quant(bf16(silu(c1[r,:F]) * c1[r,F:]))
//   moe_combine_kernel       out[t] = sum_j c3[pos[t*topk+j]]  (fp32 sum, one rounding)
// --------------------------------------------------------------------------------------------
template <typename IdT>
__global__ void __launch_bounds__(kPlanThreads) moe_plan_kernel(const IdT* __restrict__ ids, const void* __restrict__ topk_w,
                                                               int topk_w_f32, int P, int E, int N1, int K1, int BN, MoePlan pl) {
  cb::pdl_prologue();
  extern __shared__ int sm[];
  if (P <= kPlanThreads) moe_plan_small<IdT>(ids, topk_w, topk_w_f32, P, E, N1, K1, BN, pl, sm);
  else moe_plan_large<IdT>(ids, topk_w, topk_w_f32, P, E, N1, K1, BN, pl, sm);
}

// one warp per (sorted row, 128-group): gather the token's row, quantise (mode 1) or copy (bf16 mode)
__global__ void moe_gather_quant_kernel(const __nv_bfloat16* __restrict__ x, const int* __restrict__ pair_sorted,
                                        const int* __restrict__ seg_start, int E, int topk, int K, int quant,
                                        uint8_t* __restrict__ xq, float* __restrict__ xs,
                                        __nv_bfloat16* __restrict__ xb) {
  cb::pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int groups = K / 128;
  const int64_t gidx = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int rows = seg_start[E];
  if (gidx >= (int64_t)rows * groups) return;
  const int r = (int)(gidx / groups), gk = (int)(gidx - (int64_t)r * groups);
  const int t = pair_sorted[r] / topk;
  const uint2 raw = *reinterpret_cast<const uint2*>(x + (int64_t)t * K + gk * 128 + lane * 4);
  if (!quant) {
    *reinterpret_cast<uint2*>(xb + (int64_t)r * K + gk * 128 + lane * 4) = raw;
    return;
  }
  const float v[4] = {bf16lo(raw.x), bf16hi(raw.x), bf16lo(raw.y), bf16hi(raw.y)};
  const E4m3Word<4> g = e4m3_group_quant<E4m3Group::kPerTokenGroup>(v);
  *reinterpret_cast<uint32_t*>(xq + (int64_t)r * K + gk * 128 + lane * 4) = g.bits[0];
  if (lane == 0) xs[(int64_t)r * groups + gk] = g.scale;
}

// a2 = SiluAndMul(c1) in sorted space, then per_token_group_quant_fp8 (or bf16 copy)
__global__ void moe_silu_quant_kernel(const __nv_bfloat16* __restrict__ c1, const int* __restrict__ seg_start, int E,
                                      int F, int quant, uint8_t* __restrict__ aq, float* __restrict__ as,
                                      __nv_bfloat16* __restrict__ ab) {
  cb::pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int groups = F / 128;
  const int64_t gidx = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int rows = seg_start[E];
  if (gidx >= (int64_t)rows * groups) return;
  const int r = (int)(gidx / groups), gk = (int)(gidx - (int64_t)r * groups);
  const __nv_bfloat16* row = c1 + (int64_t)r * 2 * F;
  const uint2 gr = *reinterpret_cast<const uint2*>(row + gk * 128 + lane * 4);
  const uint2 ur = *reinterpret_cast<const uint2*>(row + F + gk * 128 + lane * 4);
  const float gv[4] = {bf16lo(gr.x), bf16hi(gr.x), bf16lo(gr.y), bf16hi(gr.y)};
  const float uv[4] = {bf16lo(ur.x), bf16hi(ur.x), bf16lo(ur.y), bf16hi(ur.y)};
  float v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = round_bf16(round_bf16(gv[i] / (1.f + expf(-gv[i]))) * uv[i]);
  if (!quant) {
    const __nv_bfloat16* tag = nullptr;
    uint2 o = make_uint2(pack2(v[0], v[1], tag), pack2(v[2], v[3], tag));
    *reinterpret_cast<uint2*>(ab + (int64_t)r * F + gk * 128 + lane * 4) = o;
    return;
  }
  const E4m3Word<4> g = e4m3_group_quant<E4m3Group::kPerTokenGroup>(v);
  *reinterpret_cast<uint32_t*>(aq + (int64_t)r * F + gk * 128 + lane * 4) = g.bits[0];
  if (lane == 0) as[(int64_t)r * groups + gk] = g.scale;
}

// out[t,:] = sum_j c3[pos[t*topk+j], :]   (torch.sum(dim=1) on bf16: fp32 accumulate, one rounding)
__global__ void moe_combine_kernel(const __nv_bfloat16* __restrict__ c3, const int* __restrict__ pos,
                                   __nv_bfloat16* __restrict__ out, int T, int topk, int K,
                                   const __nv_bfloat16* __restrict__ residual, int has_push, const PushDev push) {
  cb::pdl_prologue();
  const int K2 = K / 2;
  const uint32_t push_calls = has_push ? *push.calls : 0u;
  const int64_t push_off = has_push ? push_area(push, push_calls) : 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (int64_t)T * K2;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = i / K2;
    const int k = (int)(i - t * K2) * 2;
    float s0 = 0.f, s1 = 0.f;
    for (int j = 0; j < topk; ++j) {
      const int r = pos[t * topk + j];
      if (r < 0) continue;
      const uint32_t u = *reinterpret_cast<const uint32_t*>(c3 + (int64_t)r * K + k);
      s0 += bf16lo(u);
      s1 += bf16hi(u);
    }
    if (residual) {      // h = h + y : y is rounded to bf16 first, as the reference's separate add does
      const uint32_t ru = *reinterpret_cast<const uint32_t*>(residual + t * K + k);
      s0 = round_bf16(s0) + bf16lo(ru);
      s1 = round_bf16(s1) + bf16hi(ru);
    }
    const __nv_bfloat162 ov = __floats2bfloat162_rn(s0, s1);
    if (has_push) {      // tensor-parallel partial of the MoE block: straight into every rank's push area as an
                         // epoch-tagged word (model_deepseek_v3.py:1011; comm.cu)
      push_word(push, push_off + (((t * K + k) >> 1) << 3), *reinterpret_cast<const uint32_t*>(&ov), push_calls + 1u);
    } else {
      *reinterpret_cast<__nv_bfloat162*>(out + t * K + k) = ov;
    }
  }
}

// moe_gate_kernel's dynamic shared memory grows with dim and E, so its bound is the device's: the 227 KB a block may
// opt into on sm_90, less the kernel's 32 bytes of static shared memory (`red`).
constexpr int kGateSmemBound = 227 * 1024 - 32;
// The grouped path's plan: E <= kPlanThreads and P <= kPlanMaxPairs keep its shared memory within kPlanSmemBound.
constexpr int kPlanMaxPairs = 8192;
constexpr int kPlanSmemBound = (int)(moe_plan_smem_ints(kPlanMaxPairs, kPlanThreads) * sizeof(int));

// ---- workspace layouts --------------------------------------------------------------------------------------------
// Each layout carves its workspace from `base` in order, or with base == nullptr only measures it; `end` is the size
// the *_workspace_bytes entries are built from.  Every array starts on a 256-byte boundary.
struct Carve {
  uintptr_t base;
  int64_t end = 0;
  template <typename T>
  T* take(int64_t bytes) {
    T* p = reinterpret_cast<T*>(base + end);
    end += align256(bytes);
    return p;
  }
};

// moe_gate: the logits GEMM's scratch (ticket counters first: they must stay zero between calls), then the logits.
struct GateWs : Carve {
  __nv_bfloat16* logits;
  GateWs(void* base, int T, int E) : Carve{(uintptr_t)base} {
    take<void>(cb::tc_workspace_bytes(T, E));
    logits = take<__nv_bfloat16>((int64_t)T * E * 2);
  }
};

// moe_grouped_gemm: the grouped GEMM's scratch, out_rows, row_scale, the tile count, three tile lists of `tiles`
// entries, then the gathered rows (fp8 or bf16) and their scales.
struct BlocksWs : Carve {
  int64_t tiles;
  int *out_rows, *num_tiles, *t_w, *t_x, *t_c;
  float *row_scale, *xs_s;
  uint8_t* xs;
  BlocksWs(void* base, int EM, int N, int K) : Carve{(uintptr_t)base}, tiles(((int64_t)EM / 16 + 1) * (N / 128 + 1)) {
    take<void>(cb::tc_workspace_bytes(128, 128));
    out_rows = take<int>((int64_t)EM * 4);
    row_scale = take<float>((int64_t)EM * 4);
    num_tiles = take<int>(4);
    t_w = take<int>(tiles * 4);
    t_x = take<int>(tiles * 4);
    t_c = take<int>(tiles * 4);
    xs = take<uint8_t>((int64_t)EM * K * 2);
    xs_s = take<float>((int64_t)EM * (K / 128 + 1) * 4);
  }
};

// fused_experts, grouped path: the grouped GEMMs' scratch (tickets + partials, zeroed once), the plan, then in sorted
// row order xs (fp8 or bf16) and its scales, c1, a2 (fp8 or bf16) and its scales, c3.
struct GroupedWs : Carve {
  MoePlan pl;
  uint8_t *xs, *a2;
  float *xs_s, *a2_s;
  __nv_bfloat16 *c1, *c3;
  GroupedWs(void* base, int64_t P, int E, int N1, int K1) : Carve{(uintptr_t)base} {
    const int64_t chunks = E + P / 16 + 1;                  // row chunks of >= 16 sorted rows
    take<void>(cb::tc_workspace_bytes(128, 128));
    int* ip = take<int>((P + P + (E + 1) + 2 + P) * 4);     // pair_sorted, pos, seg_start, counts, w_sorted
    pl.pair_sorted = ip; pl.pos = ip + P; pl.seg_start = ip + 2 * P; pl.num_tiles1 = ip + 2 * P + E + 1;
    pl.num_tiles2 = pl.num_tiles1 + 1; pl.w_sorted = (float*)(ip + 2 * P + E + 3);
    int* t1 = take<int>(chunks * (N1 / 128 + 1) * 3 * 4);
    pl.tile1_wrow = t1; pl.tile1_xrow = t1 + chunks * (N1 / 128); pl.tile1_cnt = t1 + 2 * chunks * (N1 / 128);
    int* t2 = take<int>(chunks * (K1 / 128 + 1) * 3 * 4);
    pl.tile2_wrow = t2; pl.tile2_xrow = t2 + chunks * (K1 / 128); pl.tile2_cnt = t2 + 2 * chunks * (K1 / 128);
    xs = take<uint8_t>(P * K1 * 2);
    xs_s = take<float>(P * (K1 / 128 + 1) * 4);
    c1 = take<__nv_bfloat16>(P * N1 * 2);
    a2 = take<uint8_t>(P * (N1 / 2) * 2);
    a2_s = take<float>(P * (N1 / 2 / 128 + 1) * 4);
    c3 = take<__nv_bfloat16>(P * K1 * 2);
  }
};

// fused_experts, pair-GEMV path: after the grouped GEMMs' scratch (its ticket counters must stay zero), x quantised
// and its scales (mode 1), c1, a2, a2 quantised and its scales (mode 1), c3.
struct PairWs : Carve {
  uint8_t *a1_q, *a2_q;
  float *a1_s, *a2_s;
  __nv_bfloat16 *c1, *a2, *c3;
  PairWs(void* base, int T, int64_t P, int N1, int K1) : Carve{(uintptr_t)base} {
    take<void>(cb::tc_workspace_bytes(128, 128));
    a1_q = take<uint8_t>((int64_t)T * K1);
    a1_s = take<float>((int64_t)T * (K1 / 128 + 1) * 4);
    c1 = take<__nv_bfloat16>(P * N1 * 2);
    a2 = take<__nv_bfloat16>(P * (N1 / 2) * 2);
    a2_q = take<uint8_t>(P * (N1 / 2));
    a2_s = take<float>(P * (N1 / 2 / 128 + 1) * 4);
    c3 = take<__nv_bfloat16>(P * K1 * 2);
  }
};

// The grouped GEMM kind of a weight mode (0 bf16, 1 fp8 w8a8, 2 fp8 weights x bf16 activations, 3 4-bit weights x bf16
// activations); the pair-GEMV kernel's MODE is the weight mode itself (0..2: 4-bit weights run on the grouped path only).
constexpr int kWmodeW4 = 3;
int moe_gemm_kind(int wmode) {
  return wmode == 1 ? cb::KIND_FP8 : (wmode == 2 ? cb::KIND_SOFT : (wmode == kWmodeW4 ? cb::KIND_W4 : cb::KIND_16));
}

}  // namespace

extern "C" int64_t chitu_b200_moe_gate_workspace_bytes(int T, int E) { return GateWs(nullptr, T, E).end; }

extern "C" int chitu_b200_moe_gate(const void* x, const void* w, const void* bias, int bias_dtype, int T,
                                   int dim, int E, int n_groups, int topk_groups, int topk,
                                   int score_sigmoid, float route_scale, void* out_weights,
                                   int64_t* out_indices, int out_stride, void* workspace,
                                   int64_t workspace_bytes, void* stream) {
  CB_ARG(x && w && out_weights && out_indices && out_stride >= topk);
  CB_ARG(T >= 0 && dim > 0 && dim % 8 == 0 && E > 0 && topk > 0 && topk <= E && topk <= 32);
  CB_ARG(n_groups >= 1 && n_groups <= 64 && E % n_groups == 0 && topk_groups >= 1 && topk_groups <= n_groups);
  CB_ARG(bias == nullptr || bias_dtype == CB_F32 || bias_dtype == CB_BF16);
  if (T == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  // gate logits: one weight-streaming wgmma GEMM over all tokens (the old per-token in-kernel GEMV
  // re-read the 3.67 MB gate matrix once per token: 360 us per layer at bs=16)
  const __nv_bfloat16* logits = nullptr;
  if (workspace && workspace_bytes >= chitu_b200_moe_gate_workspace_bytes(T, E) && cb::tc_supported(cb::KIND_16, T, E, dim)) {
    __nv_bfloat16* lg = GateWs(workspace, T, E).logits;
    if (T <= 16 && dim <= 256 * kGateVecIters * 8) {
      // decode batches: one CTA per pair of experts, no split-K (see gate_logits_kernel)
      const dim3 grid((E + 1) / 2), block(256);
      const __nv_bfloat16* xb = (const __nv_bfloat16*)x;
      const __nv_bfloat16* wb = (const __nv_bfloat16*)w;
      if (T <= 1) cb::launch_k(gate_logits_kernel<1>, grid, block, 0, st, xb, wb, lg, T, dim, E);
      else if (T <= 4) cb::launch_k(gate_logits_kernel<4>, grid, block, 0, st, xb, wb, lg, T, dim, E);
      else if (T <= 8) cb::launch_k(gate_logits_kernel<8>, grid, block, 0, st, xb, wb, lg, T, dim, E);
      else cb::launch_k(gate_logits_kernel<16>, grid, block, 0, st, xb, wb, lg, T, dim, E);
      CB_LAUNCHED(1);
    } else {
      int rc = cb::tc_linear16(x, w, nullptr, nullptr, lg, T, E, dim, CB_BF16, workspace, cb::tc_workspace_bytes(T, E), st);
      if (rc) return rc;
    }
    logits = lg;
  }
  const size_t smem = (size_t)dim * 2 + (size_t)(2 * E + n_groups) * 4 + (size_t)topk * 4 + 16;
  const int rc = launch_smem<moe_gate_kernel, kGateSmemBound>(
      __func__, dim3(T), dim3(256), smem, st, (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, bias,
      (int)(bias_dtype == CB_F32), dim, E, n_groups, topk_groups, topk, score_sigmoid, route_scale,
      (__nv_bfloat16*)out_weights, out_indices, logits, out_stride);
  if (rc) return rc;
  CB_LAUNCHED(1);
  return 0;
}

// ---- invoke_fused_moe_kernel (fused_moe.py:796-891; kernel :62-307) as a stand-alone entry ------------------
// Blocks of `block_m` entries of sorted_token_ids (moe_align_block_size's output) share expert expert_ids[block];
// entry r reads A[sorted_ids[r] / top_k] and writes C.view(-1, N)[sorted_ids[r]] (x topk_weights[sorted_ids[r]] when
// mul_routed_weight); entries >= numel are padding.  Here: gather (+ per_token_group_quant_fp8 for fp8_w8a8) the A rows
// into sorted order, build the (block, n-tile) list on the device, run the grouped wgmma GEMM with an output-row
// indirection.
__global__ void moe_blocks_prepare_kernel(const int32_t* __restrict__ sorted_ids, const int32_t* __restrict__ expert_ids,
                                          const int32_t* __restrict__ npp, int EM, int numel, int block_m, int E, int N,
                                          const void* __restrict__ topk_w, int topk_w_f32, int mul_routed,
                                          int* __restrict__ out_rows, float* __restrict__ row_scale, int* __restrict__ num_tiles,
                                          int* __restrict__ tile_wrow, int* __restrict__ tile_xrow, int* __restrict__ tile_cnt) {
  cb::pdl_prologue();
  const int rows = min(*npp, EM);
  const int nblk = rows / block_m, nt = N / 128;
  const int gid = blockIdx.x * blockDim.x + threadIdx.x, gsz = gridDim.x * blockDim.x;
  // active blocks are compacted by a serial scan of thread 0 (a few hundred blocks at most): blocks whose expert is not
  // on this rank (expert_map == -1) produce no tile; their output rows are zeroed by the gather kernel
  if (gid == 0) {
    int na = 0;
    for (int b = 0; b < nblk; ++b) {
      const int e = expert_ids[b];
      if (e < 0 || e >= E) continue;
      for (int i = 0; i < nt; ++i) {
        tile_wrow[na * nt + i] = e * N + i * 128;
        tile_xrow[na * nt + i] = b * block_m;
        tile_cnt[na * nt + i] = block_m;
      }
      ++na;
    }
    *num_tiles = na * nt;
  }
  for (int r = gid; r < EM; r += gsz) {
    const int id = r < rows ? sorted_ids[r] : numel;
    const bool valid = id < numel;
    const int e = r < rows ? expert_ids[r / block_m] : -1;
    out_rows[r] = (valid && e >= 0 && e < E) ? id : -1;
    float w = 1.f;
    if (valid && mul_routed)
      w = topk_w_f32 ? reinterpret_cast<const float*>(topk_w)[id] : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(topk_w)[id]);
    row_scale[r] = w;
  }
}

// one warp per (sorted entry, 128-group of K): copy / quantise the A row of the entry; padding entries become zero rows;
// entries whose block's expert is absent write a zero OUTPUT row (fused_moe.py:160-176)
__global__ void moe_rows_gather_kernel(const __nv_bfloat16* __restrict__ A, const int32_t* __restrict__ sorted_ids,
                                       const int32_t* __restrict__ expert_ids, const int32_t* __restrict__ npp, int EM,
                                       int numel, int top_k, int block_m, int E, int K, int N, int quant,
                                       uint8_t* __restrict__ xq, float* __restrict__ xs, __nv_bfloat16* __restrict__ xb,
                                       __nv_bfloat16* __restrict__ C) {
  cb::pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int groups = K / 128;
  const int64_t gidx = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int rows = min(*npp, EM);
  if (gidx >= (int64_t)rows * groups) return;
  const int r = (int)(gidx / groups), gk = (int)(gidx - (int64_t)r * groups);
  const int id = sorted_ids[r];
  const int e = expert_ids[r / block_m];
  if (id < numel && (e < 0 || e >= E)) {
    for (int n = gk * 32 + lane; n < N; n += groups * 32) C[(int64_t)id * N + n] = __float2bfloat16_rn(0.f);
  }
  uint2 raw = make_uint2(0u, 0u);
  if (id < numel) raw = *reinterpret_cast<const uint2*>(A + (int64_t)(id / top_k) * K + gk * 128 + lane * 4);
  if (!quant) {
    *reinterpret_cast<uint2*>(xb + (int64_t)r * K + gk * 128 + lane * 4) = raw;
    return;
  }
  const float v[4] = {bf16lo(raw.x), bf16hi(raw.x), bf16lo(raw.y), bf16hi(raw.y)};
  const E4m3Word<4> g = e4m3_group_quant<E4m3Group::kPerTokenGroup>(v);
  *reinterpret_cast<uint32_t*>(xq + (int64_t)r * K + gk * 128 + lane * 4) = g.bits[0];
  if (lane == 0) xs[(int64_t)r * groups + gk] = g.scale;
}

extern "C" int64_t chitu_b200_moe_grouped_gemm_workspace_bytes(int EM, int N, int K) {
  return BlocksWs(nullptr, EM, N, K).end + 256;
}

extern "C" int chitu_b200_moe_grouped_gemm(const void* A, const void* B, void* C, const float* B_scale, const void* topk_weights,
                                           int topk_w_dtype, const int32_t* sorted_token_ids, const int32_t* expert_ids,
                                           const int32_t* num_tokens_post_padded, int EM, int numel, int mul_routed_weight,
                                           int top_k, int block_m, int E, int N, int K, int wmode, void* workspace,
                                           int64_t workspace_bytes, void* stream) {
  CB_ARG(A && B && C && sorted_token_ids && expert_ids && num_tokens_post_padded && workspace);
  CB_ARG(EM >= 0 && numel >= 0 && top_k >= 1 && E > 0 && N > 0 && K > 0 && wmode >= 0 && wmode <= 2);
  CB_ARG(block_m == 16 || block_m == 32 || block_m == 64 || block_m == 128);
  // moe_rows_gather_kernel copies / quantises whole 128-column groups of A
  CB_ARG(N % 128 == 0 && K % 128 == 0 && (wmode == 0 || B_scale));
  EM -= EM % block_m;     // num_tokens_post_padded is a multiple of block_m, so whole blocks cover every valid entry
  CB_ARG(!mul_routed_weight || topk_weights);
  CB_ARG(topk_w_dtype == CB_BF16 || topk_w_dtype == CB_F32);
  if (EM == 0 || numel == 0) return 0;
  CB_ARG(workspace_bytes >= chitu_b200_moe_grouped_gemm_workspace_bytes(EM, N, K));
  if (!cb::tma_available()) return cb::fail(-3, "moe_grouped_gemm: TMA is not available");
  cudaStream_t st = (cudaStream_t)stream;
  const BlocksWs ws(workspace, EM, N, K);
  CB_ARG(ws.tiles <= cb::tc_max_tiles());
  const int quant = wmode == 1;
  cb::launch_k(moe_blocks_prepare_kernel, dim3(cdiv(EM, 256)), dim3(256), 0, st, sorted_token_ids, expert_ids,
               num_tokens_post_padded, EM, numel, block_m, E, N, topk_weights, (int)(topk_w_dtype == CB_F32),
               mul_routed_weight, ws.out_rows, ws.row_scale, ws.num_tiles, ws.t_w, ws.t_x, ws.t_c);
  CB_LAUNCHED(1);
  cb::launch_k(moe_rows_gather_kernel, dim3(cdiv((int64_t)EM * (K / 128), 8)), dim3(256), 0, st, (const __nv_bfloat16*)A,
               sorted_token_ids, expert_ids, num_tokens_post_padded, EM, numel, top_k, block_m, E, K, N, quant, ws.xs,
               ws.xs_s, (__nv_bfloat16*)ws.xs, (__nv_bfloat16*)C);
  CB_LAUNCHED(1);
  return cb::tc_grouped_gemm(moe_gemm_kind(wmode), ws.xs, ws.xs_s, B, B_scale, nullptr, nullptr, C, EM, E, N, K, block_m, ws.num_tiles,
                             ws.t_w, ws.t_x, ws.t_c, mul_routed_weight ? ws.row_scale : nullptr, ws.out_rows, workspace,
                             cb::tc_workspace_bytes(128, 128), st);
}

extern "C" int64_t chitu_b200_moe_workspace_bytes(int T, int topk, int E, int N1, int K1) {
  const int64_t P = (int64_t)T * topk;
  const int64_t pair = PairWs(nullptr, T, P, N1, K1).end, grouped = GroupedWs(nullptr, P, E, N1, K1).end;
  return (pair > grouped ? pair : grouped) + 256;
}

// rows per chunk (= wgmma N of the grouped GEMMs): twice the mean number of routed rows per expert, 16 .. 128
static int moe_chunk_rows(int64_t P, int E) {
  int BN = 16;
  while (BN < 128 && BN < 2 * (int)((P + E - 1) / E)) BN *= 2;
  return BN;
}

// The 4-bit operands of weight mode 3: bf16 scales and uint8 zeros (null: every zero is 8), [E, N, K / 128] each.
struct W4Operands {
  const void *w1_s, *w2_s;
  const uint8_t *w1_z, *w2_z;
};

// w1_s / w2_s: the fp8 block scales of weight modes 1 and 2; w4: the scales and zeros of weight mode 3.
static int fused_experts_impl(const void* x, const void* w1, const void* w2, const float* w1_s,
                              const float* w2_s, const W4Operands& w4, const void* topk_w, int topk_w_dtype,
                              const void* topk_ids, int ids_dtype, int T, int topk, int E, int N1,
                              int K1, int wmode, void* out, const void* residual, void* workspace,
                              int64_t workspace_bytes, void* stream, void* comm) {
  CB_ARG(x && w1 && w2 && topk_w && topk_ids && (out || comm) && workspace);
  CB_ARG(T >= 0 && topk > 0 && E > 0 && N1 > 0 && N1 % 2 == 0 && K1 > 0);
  CB_ARG(wmode >= 0 && wmode <= kWmodeW4);
  CB_ARG(wmode == 0 || wmode == kWmodeW4 || (w1_s && w2_s));
  CB_ARG(wmode != kWmodeW4 || (w4.w1_s && w4.w2_s));
  CB_ARG(topk_w_dtype == CB_BF16 || topk_w_dtype == CB_F32);
  CB_ARG(ids_dtype == CB_I32 || ids_dtype == CB_I64);
  CB_ARG(K1 % 16 == 0 && (N1 / 2) % 16 == 0);
  if (wmode == 1) CB_ARG(K1 % 128 == 0 && (N1 / 2) % 128 == 0);
  CB_ARG(workspace_bytes >= chitu_b200_moe_workspace_bytes(T, topk, E, N1, K1));
  // 4-bit weights run on the grouped wgmma path only (one group of 128 per pipeline stage of both GEMMs)
  if (wmode == kWmodeW4 && !(N1 % 256 == 0 && K1 % 128 == 0 && (N1 / 2) % 128 == 0))
    return cb::fail(-2, "fused_experts_w4a16: needs N1 %% 256 == 0, K1 %% 128 == 0 and (N1 / 2) %% 128 == 0 "
                        "(N1 = %d, K1 = %d)", N1, K1);
  if (T == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t P = (int64_t)T * topk;
  const int N2 = N1 / 2;
  CB_ARG(P <= 65535);
  const int w_f32 = topk_w_dtype == CB_F32, ids_i64 = ids_dtype == CB_I64;

  // ---- grouped wgmma path: sort pairs by expert, stream every distinct expert once ----
  const int BN = moe_chunk_rows(P, E);
  const int64_t chunks = E + P / 16 + 1;
  const bool grouped = P <= kPlanMaxPairs && E <= kPlanThreads && N1 % 256 == 0 && K1 % 128 == 0 &&
                       (wmode != 2 || (N1 / 2) % 128 == 0) && chunks * (N1 / 128) <= cb::tc_max_tiles() &&
                       chunks * (K1 / 128) <= cb::tc_max_tiles() && cb::tma_available();
  if (!grouped && wmode == kWmodeW4)
    return cb::fail(-2, "fused_experts_w4a16: the grouped wgmma path cannot run (T=%d topk=%d E=%d N1=%d K1=%d; it needs "
                        "T * topk <= %d, E <= %d and TMA), and 4-bit weights have no other path", T, topk, E, N1, K1,
                    kPlanMaxPairs, kPlanThreads);
  if (grouped) {
    const GroupedWs ws(workspace, P, E, N1, K1);
    const MoePlan& pl = ws.pl;
    const int quant = wmode == 1, gkind = moe_gemm_kind(wmode);
    const size_t psm = (size_t)moe_plan_smem_ints(P, E) * sizeof(int);
    int rc = ids_i64
        ? launch_smem<moe_plan_kernel<int64_t>, kPlanSmemBound>(__func__, dim3(1), dim3(kPlanThreads), psm, st,
                                                                (const int64_t*)topk_ids, topk_w, w_f32, (int)P, E, N1, K1, BN, pl)
        : launch_smem<moe_plan_kernel<int32_t>, kPlanSmemBound>(__func__, dim3(1), dim3(kPlanThreads), psm, st,
                                                                (const int32_t*)topk_ids, topk_w, w_f32, (int)P, E, N1, K1, BN, pl);
    if (rc) return rc;
    CB_LAUNCHED(1);
    cb::launch_k(moe_gather_quant_kernel, dim3(cdiv(P * (K1 / 128), 8)), dim3(256), 0, st, (const __nv_bfloat16*)x,
                 (const int*)pl.pair_sorted, (const int*)pl.seg_start, E, topk, K1, quant, ws.xs, ws.xs_s,
                 (__nv_bfloat16*)ws.xs);
    CB_LAUNCHED(1);
    rc = cb::tc_grouped_gemm(gkind, ws.xs, ws.xs_s, w1, w1_s, w4.w1_s, w4.w1_z, ws.c1, (int)P, E, N1, K1, BN, pl.num_tiles1, pl.tile1_wrow,
                             pl.tile1_xrow, pl.tile1_cnt, nullptr, nullptr, workspace, cb::tc_workspace_bytes(128, 128), st);
    if (rc) return rc;
    cb::launch_k(moe_silu_quant_kernel, dim3(cdiv(P * (N2 / 128), 8)), dim3(256), 0, st, (const __nv_bfloat16*)ws.c1,
                 (const int*)pl.seg_start, E, N2, quant, ws.a2, ws.a2_s, (__nv_bfloat16*)ws.a2);
    CB_LAUNCHED(1);
    rc = cb::tc_grouped_gemm(gkind, ws.a2, ws.a2_s, w2, w2_s, w4.w2_s, w4.w2_z, ws.c3, (int)P, E, K1, N2, BN, pl.num_tiles2, pl.tile2_wrow,
                             pl.tile2_xrow, pl.tile2_cnt, pl.w_sorted, nullptr, workspace, cb::tc_workspace_bytes(128, 128),
                             st);
    if (rc) return rc;
    int cblocks = cdiv((int64_t)T * K1 / 2, 256);
    if (cblocks > 132 * 8) cblocks = 132 * 8;
    PushDev push;
    memset(&push, 0, sizeof(push));
    if (comm) {
      rc = cb::comm_push_desc(comm, &push);
      if (rc) return rc;
    }
    cb::launch_k(moe_combine_kernel, dim3(cblocks), dim3(256), 0, st, (const __nv_bfloat16*)ws.c3, (const int*)pl.pos,
                 (__nv_bfloat16*)out, T, topk, K1, (const __nv_bfloat16*)residual, comm ? 1 : 0, push);
    CB_LAUNCHED(1);
    return 0;
  }
  if (comm) return cb::fail(-2, "fused_experts_ar: only the grouped wgmma path pushes (T=%d topk=%d E=%d N1=%d K1=%d)", T, topk, E, N1, K1);

  // ---- pair-GEMV path: both GEMMs run the kernel of the weight mode, mode 1 on activations quantised per 128-group ----
  const PairWs ws(workspace, T, P, N1, K1);
  const auto gemv = wmode == 1 ? moe_pair_gemv_kernel<1> : (wmode == 2 ? moe_pair_gemv_kernel<2> : moe_pair_gemv_kernel<0>);
  int rc;
  // GEMM1
  if (wmode == 1) {
    rc = chitu_b200_act_quant_fp8(x, ws.a1_q, ws.a1_s, T, K1, 128, 1, 1e-10f, CB_BF16, stream);
    if (rc) return rc;
  }
  cb::launch_k(gemv, dim3(cdiv(N1, 16), (unsigned)P), dim3(256), 0, st, wmode == 1 ? (const void*)ws.a1_q : x,
               wmode == 1 ? ws.a1_s : nullptr, (const uint8_t*)w1, wmode ? w1_s : nullptr, topk_ids, ids_i64, topk_w,
               w_f32, 0, topk, E, N1, K1, ws.c1);
  CB_LAUNCHED(1);
  rc = chitu_b200_silu_and_mul(ws.c1, ws.a2, P, N2, CB_BF16, stream);
  if (rc) return rc;
  // GEMM2 (x routed weight)
  if (wmode == 1) {
    rc = chitu_b200_act_quant_fp8(ws.a2, ws.a2_q, ws.a2_s, P, N2, 128, 1, 1e-10f, CB_BF16, stream);
    if (rc) return rc;
  }
  cb::launch_k(gemv, dim3(cdiv(K1, 16), (unsigned)P), dim3(256), 0, st, wmode == 1 ? (const void*)ws.a2_q : ws.a2,
               wmode == 1 ? ws.a2_s : nullptr, (const uint8_t*)w2, wmode ? w2_s : nullptr, topk_ids, ids_i64, topk_w,
               w_f32, 1, 1, E, K1, N2, ws.c3);
  CB_LAUNCHED(1);
  int blocks = cdiv((int64_t)T * K1, 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  cb::launch_k(moe_sum_kernel, dim3(blocks), dim3(256), 0, st, ws.c3, (__nv_bfloat16*)out, T, topk, K1);
  CB_LAUNCHED(1);
  if (residual) return chitu_b200_add(out, residual, out, (int64_t)T * K1, CB_BF16, stream);
  return 0;
}

extern "C" int chitu_b200_fused_experts(const void* x, const void* w1, const void* w2, const float* w1_s,
                                        const float* w2_s, const void* topk_w, int topk_w_dtype,
                                        const void* topk_ids, int ids_dtype, int T, int topk, int E, int N1,
                                        int K1, int wmode, void* out, const void* residual, void* workspace,
                                        int64_t workspace_bytes, void* stream) {
  CB_ARG(out && wmode >= 0 && wmode <= 2);
  return fused_experts_impl(x, w1, w2, w1_s, w2_s, W4Operands{}, topk_w, topk_w_dtype, topk_ids, ids_dtype, T, topk, E, N1,
                            K1, wmode, out, residual, workspace, workspace_bytes, stream, nullptr);
}

// fused_experts over 4-bit weights (W4A16, groups of 128): the grouped path of chitu_b200_fused_experts with the W4 kind of
// the grouped GEMM; the plan, gather, SiLU and combine kernels are the bf16 mode's.
extern "C" int chitu_b200_fused_experts_w4a16(const void* x, const void* w1, const void* w1_scales, const uint8_t* w1_zeros,
                                              const void* w2, const void* w2_scales, const uint8_t* w2_zeros,
                                              const void* topk_w, int topk_w_dtype, const void* topk_ids, int ids_dtype,
                                              int T, int topk, int E, int N1, int K1, void* out, const void* residual,
                                              void* workspace, int64_t workspace_bytes, void* stream) {
  CB_ARG(out);
  return fused_experts_impl(x, w1, w2, nullptr, nullptr, W4Operands{w1_scales, w2_scales, w1_zeros, w2_zeros}, topk_w,
                            topk_w_dtype, topk_ids, ids_dtype, T, topk, E, N1, K1, kWmodeW4, out, residual, workspace,
                            workspace_bytes, stream, nullptr);
}

// fused_experts whose result (this rank's partial of the MoE block) is pushed into every rank's all-reduce area from the
// combine kernel instead of being written to `out`; reduce with chitu_b200_allreduce_consume(comm, ...).
extern "C" int chitu_b200_fused_experts_ar(const void* x, const void* w1, const void* w2, const float* w1_s,
                                           const float* w2_s, const void* topk_w, int topk_w_dtype,
                                           const void* topk_ids, int ids_dtype, int T, int topk, int E, int N1,
                                           int K1, int wmode, void* comm, void* workspace, int64_t workspace_bytes,
                                           void* stream) {
  CB_ARG(comm && K1 % 2 == 0 && (int64_t)T * K1 * 2 <= cb::comm_slot_bytes(comm) && wmode >= 0 && wmode <= 2);
  return fused_experts_impl(x, w1, w2, w1_s, w2_s, W4Operands{}, topk_w, topk_w_dtype, topk_ids, ids_dtype, T, topk, E, N1,
                            K1, wmode, nullptr, nullptr, workspace, workspace_bytes, stream, comm);
}

CB_DEFINE_TL_SETTER(moe)
