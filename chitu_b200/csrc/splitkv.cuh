// The split-KV ("flash decoding") workspace contract of the attention kernels: GQA decode and the absorb-o merge
// (attention.cu), MLA decode (mla_tc.cu), GQA paged prefill (gqa_prefill.cu), MLA paged prefill (mla_prefill.cu) and
// the device-side split plan (core.cu).
//
// A kernel that splits the keys of `rows` partial rows (B * H) into S splits writes, from the start of the workspace,
//   o_part [rows, S, dv] fp32, each split normalised by its own softmax sum
//   lse    [rows, S]     fp32, log2 domain (m + log2(l)), -inf for a split that saw no key
// and a merge weights the S partials of a row by split_weights below.  The last kPlanBytes of the workspace hold the
// split plan that chitu_b200_attn_plan writes for the MLA decode kernel.
#pragma once
#include "common.cuh"

namespace cb {

// the merges keep one weight per split in shared memory (s_w of merge_splits_kernel, s_mw of mla_absorb_o_kernel)
constexpr int kMaxSplits = 128;
constexpr int kMlaC = 512;      // absorbed MLA: kv_lora_rank, the head dim of its partials

// the plan is int32 words, the magic written last: keys per split (whole pages), the most splits of one request, the
// splits of the batch, and the B, page size and head count it was made for
constexpr int kPlanBytes = 256;
constexpr int32_t kPlanMagic = 0x504c414e;   // "PLAN"
enum PlanWord { kPlanWordMagic, kPlanWordKeysPerSplit, kPlanWordMaxSplits, kPlanWordTotalSplits, kPlanWordBatch,
                kPlanWordPageSize, kPlanWordHeads };

inline int64_t split_kv_bytes(int64_t rows, int dv, int splits) {
  return rows * splits * (dv + 1) * (int64_t)sizeof(float) + kPlanBytes;
}

inline int32_t* split_kv_plan(void* workspace, int64_t workspace_bytes) {   // null when the workspace cannot hold it
  return workspace && workspace_bytes >= kPlanBytes ? (int32_t*)((uint8_t*)workspace + workspace_bytes - kPlanBytes)
                                                    : nullptr;
}

struct SplitKv { float* o_part; float* lse; int32_t* plan; };
// the partials of `splits` splits and the plan inside `workspace` (all null without one)
inline SplitKv split_kv_carve(void* workspace, int64_t workspace_bytes, int64_t rows, int dv, int splits) {
  float* o_part = (float*)workspace;
  return {o_part, o_part ? o_part + rows * splits * dv : nullptr, split_kv_plan(workspace, workspace_bytes)};
}

// the largest split count <= `splits` whose partials fit the workspace (at least 1)
inline int splits_that_fit(int splits, int64_t rows, int dv, int64_t workspace_bytes) {
  while (splits > 1 && split_kv_bytes(rows, dv, splits) > workspace_bytes) --splits;
  return splits;
}

// split count for a kernel with `slots` resident CTAs on the GPU: minimise waves x (keys per split + a fixed
// per-CTA cost worth ~192 keys).  Waves are whole: a CTA streams at its SM's rate however empty the GPU is
// (measured over split counts: bs=16 128 CTAs x 4096 keys beat every split; bs=1 wants ~one full wave).
inline int pick_splits_waves(int ctas_without_split, int max_len, int slots) {
  int by_len = (max_len + 127) / 128;
  if (by_len > 64) by_len = 64;
  int best = 1;
  double best_cost = 1e30;
  for (int s = 1; s <= by_len; ++s) {
    const int ctas = ctas_without_split * s;
    const int waves = (ctas + slots - 1) / slots;
    const double cost = waves * ((double)max_len / s + 192.0) + (s > 1 ? 64.0 : 0.0);   // + the merge launch
    if (cost < best_cost - 1e-9) { best_cost = cost; best = s; }
  }
  return best;
}

inline int pick_splits(int ctas_without_split, int max_len, int min_keys_per_split, int max_splits) {
  int want = (132 * 4 + ctas_without_split - 1) / ctas_without_split;  // ~4 CTAs per SM
  int by_len = (max_len + min_keys_per_split - 1) / min_keys_per_split;
  int s = want < by_len ? want : by_len;
  if (s > max_splits) s = max_splits;
  if (s < 1) s = 1;
  return s;
}

// KV splits of the wgmma MLA decode kernel (1 CTA per SM): one wave of CTAs, whole pages, at least two pages per split,
// and the partials must fit the workspace.  Deterministic in its arguments: the merging absorb-o kernel recomputes it.
inline int mla_num_splits(int B, int H, int max_len, int64_t workspace_bytes) {
  const int hgroups = cdiv(H, 16);
  int want = 132 / (B * hgroups);
  const int pages = cdiv(max_len, 64);
  int by_len = pages / 2;
  int splits = want < by_len ? want : by_len;
  if (splits > kMaxSplits) splits = kMaxSplits;
  if (splits < 1) splits = 1;
  return splits_that_fit(splits, (int64_t)B * H, kMlaC, workspace_bytes);
}

// One warp turns the `n` split LSEs of a row into its merge weights w[s] = exp2(lse[s] - max) / sum: 0 for a split
// that saw no key, all 0 when no split did.  merge_splits_kernel and the fused merge of mla_absorb_o_kernel both call
// it and then add the splits in ascending order, so the two merges give bit-identical results.
__device__ __forceinline__ void split_weights(const float* lse, int n, float* w, int lane) {
  float mx = -INFINITY;
  for (int s = lane; s < n; s += 32) mx = fmaxf(mx, lse[s]);
  mx = warp_max(mx);
  float den = 0.f;
  for (int s = lane; s < n; s += 32) {
    const float ls = lse[s];
    const float wv = ls == -INFINITY ? 0.f : exp2f(ls - mx);
    w[s] = wv;
    den += wv;
  }
  den = warp_sum(den);
  const float inv = den > 0.f ? 1.f / den : 0.f;
  for (int s = lane; s < n; s += 32) w[s] *= inv;
}

// LSE-weighted merge of the partials of `rows` rows into out [rows, dv] (attention.cu).  Built for bf16 and fp16 with
// dv 64 and 128, and for bf16 with dv 512; anything else returns a negative status without launching.
int launch_merge_splits(const float* o_part, const float* lse, void* out, int rows, int splits, int dv, int dtype,
                        cudaStream_t st);

}  // namespace cb
