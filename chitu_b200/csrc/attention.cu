// Paged-KV decode attention, split-KV ("flash decoding").
//
//  * gqa_paged_decode : AttnBackend.attn_with_kvcache with a block_table (attn_backend.py:92-164,
//    FlashAttn impl :208-243) — GQA, in-place append of the new token, page gather through the
//    block table, online softmax in fp32, LSE-weighted merge of the splits.  Head dim 128 with
//    power-of-two pages runs on tensor cores (gqa_decode_mmaT_kernel, optional fused rotary);
//    head dim 64 and other page sizes run on the SIMT kernel (gqa_decode_kernel).
//  * gqa_contiguous_attn : the same without a block table, over a [Bc, S, Hkv, D] cache (any S): the contiguous
//    variants of both decode kernels for seqlen_q == 1 (head dim 128 always on tensor cores), gqa_prefill.cu's for
//    seqlen_q > 1.
//  * gqa_paged_attn_fp8kv : the paged cache in fp8 e4m3 (half the KV bytes): the e4m3 instance of the tensor-core
//    decode kernel for seqlen_q == 1 (gqa_decode_mmaT_e4m3_kernel), gqa_prefill.cu's e4m3 instance for seqlen_q > 1.
//    The three entries check their arguments; gqa_decode() launches seqlen_q == 1 for all of them, gqa_prefill()
//    (gqa_prefill.cu) seqlen_q > 1.
//  * merge_splits_kernel : the LSE-weighted merge of split-KV partials, for GQA decode, MLA decode
//    (mla_tc.cu) and the GQA and MLA paged prefills (gqa_prefill.cu, mla_prefill.cu).  The workspace
//    layout, the split counts, the split plan and the merge weights are defined once in splitkv.cuh.
//  * MLA absorb-o (it can also merge the MLA decode partials) and mla_prep (rotary, kv_norm and
//    absorb-q in one launch).
//
// The GQA kernels never read the cache row of the token being appended: the CTA that owns that
// position takes it from `k_new` directly and split 0 writes it to the cache -> no RAW hazard.
// The reference fixes NUM_KV_SPLITS = 4 (attn_backend.py:735) -> 4 CTAs at B=1; here the split
// count is sized from the SM count so the 132 SMs of an H100 are busy at B=1.

#include "common.cuh"
#include "splitkv.cuh"
#include "tc_ptx.cuh"

using namespace cb;

namespace {

constexpr float kLog2e = 1.4426950408889634f;

template <typename T, int DV>
__global__ void merge_splits_kernel(const float* __restrict__ o_part, const float* __restrict__ lse,
                                    T* __restrict__ out, int num_splits) {
  cb::pdl_prologue();
  __shared__ float s_w[kMaxSplits];               // normalised split weights
  const int64_t bh = blockIdx.x;  // b * H + h
  const float* l = lse + bh * num_splits;
  if (threadIdx.x < 32) split_weights(l, num_splits, s_w, threadIdx.x);
  __syncthreads();
  const float* base = o_part + bh * num_splits * DV;
  for (int d = threadIdx.x; d < DV; d += blockDim.x) {
    float acc = 0.f;
    int s = 0;
    for (; s + 8 <= num_splits; s += 8) {          // 8 independent L2 loads in flight
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = base[(int64_t)(s + i) * DV + d];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc = fmaf(s_w[s + i], v[i], acc);
    }
    for (; s < num_splits; ++s) acc = fmaf(s_w[s], base[(int64_t)s * DV + d], acc);
    out[bh * DV + d] = io<T>::from_f(acc);
  }
}

// --------------------------------------------------------------------------------------------
// GQA: one CTA per (split, kv head, request); 4 warps interleave over keys, a lane owns D/32
// consecutive dims, G = Hq/Hkv query heads share every K/V row that is loaded.
// --------------------------------------------------------------------------------------------
// CONTIG: the cache is [Bc, cache_rows, Hkv, D] and request b owns the rows from b * rows_sb (rows of Hkv * D) instead
// of the pages of its block-table row.  Its length is clamped to cache_rows, so no key at or past cache_rows is read, and
// a new row at cache_rows or past it is not written.
template <typename T, int D, int G, bool CONTIG>
__device__ __forceinline__ void gqa_decode_cta(
    const T* __restrict__ q, T* __restrict__ k_cache, T* __restrict__ v_cache,
    const T* __restrict__ k_new, const T* __restrict__ v_new, int64_t k_new_sb, int64_t v_new_sb,
    const int32_t* __restrict__ seqlens,
    const int32_t* __restrict__ block_table, int bt_stride, int64_t rows_sb, int cache_rows, int Hq, int Hkv,
    int page_size, float scale, int num_splits, float* __restrict__ o_part, float* __restrict__ lse,
    T* __restrict__ out) {
  cb::pdl_prologue();
  constexpr int VEC = D / 32;
  const int split = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int L_cache = CONTIG ? min(seqlens[b], cache_rows) : seqlens[b];
  const int L = L_cache + (k_new ? 1 : 0);
  const int chunk = (L + num_splits - 1) / num_splits;
  const int begin = split * chunk;
  const int end = min(begin + chunk, L);
  const int32_t* bt = block_table + (int64_t)b * bt_stride;

  auto cache_row = [&](int key) -> int64_t {           // row of (key, kvh) in units of D
    if constexpr (CONTIG) return ((int64_t)b * rows_sb + key) * Hkv + kvh;
    const int page = bt[key / page_size];
    return ((int64_t)page * page_size + key % page_size) * Hkv + kvh;
  };

  // in-place append of the new token (true page_size indexing, as flash_attn_with_kvcache does)
  if (k_new && split == 0 && warp == 0 && (!CONTIG || L_cache < cache_rows)) {
    const int64_t row = cache_row(L_cache);
    const T* ks = k_new + (int64_t)b * k_new_sb + kvh * D;
    const T* vs = v_new + (int64_t)b * v_new_sb + kvh * D;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      k_cache[row * D + lane * VEC + i] = ks[lane * VEC + i];
      v_cache[row * D + lane * VEC + i] = vs[lane * VEC + i];
    }
  }

  float qv[G][VEC], acc[G][VEC], m[G], l[G];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const T* qp = q + ((int64_t)b * Hq + kvh * G + g) * D + lane * VEC;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      qv[g][i] = io<T>::to_f(qp[i]) * (scale * kLog2e);
      acc[g][i] = 0.f;
    }
    m[g] = -INFINITY;
    l[g] = 0.f;
  }

  for (int key0 = begin + warp * 2; key0 < end; key0 += 8) {
    float kf[2][VEC], vf[2][VEC];
    bool valid[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int key = key0 + j;
      valid[j] = key < end;
      const T *kp, *vp;
      if (valid[j] && key < L_cache) {
        const int64_t row = cache_row(key);
        kp = k_cache + row * D + lane * VEC;
        vp = v_cache + row * D + lane * VEC;
      } else {  // the token being appended (or a masked slot: loads are harmless, result unused)
        kp = k_new ? k_new + (int64_t)b * k_new_sb + kvh * D + lane * VEC : k_cache + lane * VEC;
        vp = v_new ? v_new + (int64_t)b * v_new_sb + kvh * D + lane * VEC : v_cache + lane * VEC;
      }
      if constexpr (VEC == 4) {
        uint2 kr = *reinterpret_cast<const uint2*>(kp);
        uint2 vr = *reinterpret_cast<const uint2*>(vp);
        const T* tag = nullptr;
        float2 a = unpack2(kr.x, tag), c = unpack2(kr.y, tag);
        kf[j][0] = a.x; kf[j][1] = a.y; kf[j][2] = c.x; kf[j][3] = c.y;
        a = unpack2(vr.x, tag); c = unpack2(vr.y, tag);
        vf[j][0] = a.x; vf[j][1] = a.y; vf[j][2] = c.x; vf[j][3] = c.y;
      } else {
        const T* tag = nullptr;
        float2 a = unpack2(*reinterpret_cast<const uint32_t*>(kp), tag);
        float2 c = unpack2(*reinterpret_cast<const uint32_t*>(vp), tag);
        kf[j][0] = a.x; kf[j][1] = a.y;
        vf[j][0] = c.x; vf[j][1] = c.y;
      }
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      if (!valid[j]) continue;  // warp-uniform
#pragma unroll
      for (int g = 0; g < G; ++g) {
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < VEC; ++i) s = fmaf(qv[g][i], kf[j][i], s);
        s = warp_sum(s);
        const float mn = fmaxf(m[g], s);
        const float corr = exp2f(m[g] - mn);
        const float p = exp2f(s - mn);
        l[g] = l[g] * corr + p;
#pragma unroll
        for (int i = 0; i < VEC; ++i) acc[g][i] = fmaf(p, vf[j][i], acc[g][i] * corr);
        m[g] = mn;
      }
    }
  }

  // merge the 4 warps through shared memory
  __shared__ float s_m[4][G], s_l[4][G];
  __shared__ float s_acc[4][G][D];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    if (lane == 0) { s_m[warp][g] = m[g]; s_l[warp][g] = l[g]; }
#pragma unroll
    for (int i = 0; i < VEC; ++i) s_acc[warp][g][lane * VEC + i] = acc[g][i];
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < G * D; idx += 128) {
    const int g = idx / D, d = idx - g * D;
    float mx = fmaxf(fmaxf(s_m[0][g], s_m[1][g]), fmaxf(s_m[2][g], s_m[3][g]));
    float num = 0.f, den = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      if (s_m[w][g] == -INFINITY) continue;
      float sc = exp2f(s_m[w][g] - mx);
      num = fmaf(sc, s_acc[w][g][d], num);
      den = fmaf(sc, s_l[w][g], den);
    }
    const int h = kvh * G + g;
    const float o = den > 0.f ? num / den : 0.f;
    if (num_splits == 1) {
      out[((int64_t)b * Hq + h) * D + d] = io<T>::from_f(o);
    } else {
      const int64_t pi = ((int64_t)b * Hq + h) * num_splits + split;
      o_part[pi * D + d] = o;
      if (d == 0) lse[pi] = den > 0.f ? mx + log2f(den) : -INFINITY;
    }
  }
}

template <typename T, int D, int G>
__global__ void __launch_bounds__(128) gqa_decode_kernel(
    const T* __restrict__ q, T* __restrict__ k_cache, T* __restrict__ v_cache,
    const T* __restrict__ k_new, const T* __restrict__ v_new, int64_t k_new_sb, int64_t v_new_sb,
    const int32_t* __restrict__ seqlens,
    const int32_t* __restrict__ block_table, int bt_stride, int Hq, int Hkv, int page_size, float scale,
    int num_splits, float* __restrict__ o_part, float* __restrict__ lse, T* __restrict__ out) {
  gqa_decode_cta<T, D, G, false>(q, k_cache, v_cache, k_new, v_new, k_new_sb, v_new_sb, seqlens, block_table, bt_stride,
                                 0, 0, Hq, Hkv, page_size, scale, num_splits, o_part, lse, out);
}

template <typename T, int D, int G>
__global__ void __launch_bounds__(128) gqa_decode_contig_kernel(
    const T* __restrict__ q, T* __restrict__ k_cache, T* __restrict__ v_cache,
    const T* __restrict__ k_new, const T* __restrict__ v_new, int64_t k_new_sb, int64_t v_new_sb,
    const int32_t* __restrict__ seqlens, int64_t rows_sb, int cache_rows, int Hq, int Hkv, float scale,
    int num_splits, float* __restrict__ o_part, float* __restrict__ lse, T* __restrict__ out) {
  gqa_decode_cta<T, D, G, true>(q, k_cache, v_cache, k_new, v_new, k_new_sb, v_new_sb, seqlens, nullptr, 0, rows_sb,
                                cache_rows, Hq, Hkv, 1, scale, num_splits, o_part, lse, out);
}

__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
template <typename T>
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1);
template <>
__device__ __forceinline__ void mma16816<__nv_bfloat16>(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <>
__device__ __forceinline__ void mma16816<__half>(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// src_bytes = 0 zero-fills the 16 bytes (masked rows must be finite: 0 * NaN would poison P·V)
__device__ __forceinline__ void cp_async16_g(uint32_t smem_addr, const void* gmem, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_addr), "l"(gmem), "r"(src_bytes));
}

// --------------------------------------------------------------------------------------------
// GQA, tensor-core version (D = 128, power-of-two pages) with the KEYS as the MMA M dimension
// ("swap-AB"): S^T = K Q^T and O^T = V^T P^T.  One CTA per (split, kv head, request).  Each warp
// streams its own tiles of K and V through a private cp.async ring in shared memory (no block-level
// barrier in the main loop); K tiles are read with ldmatrix, V tiles with ldmatrix.trans, and rows
// are XOR-swizzled in 16-byte chunks so both are bank-conflict free.  A split covers whole tiles, the
// warps take them round robin, and the warps are merged through shared memory at the end.
// With G <= 8 query heads per kv head the head dimension fits the n = 8 side of m16n8k16 exactly, so
// a 32-key tile costs 32 MMAs instead of the 64 (half of them on zero padding rows) of heads as M,
// and the O accumulator is 32 registers instead of 64.  P^T is produced from the S^T accumulator
// fragments with movmatrix.trans (8x8 b16 transpose in registers); FA2-style register softmax.
// --------------------------------------------------------------------------------------------
constexpr int kGqaD = 128;
// 4 warps x 3 stages x 32 keys (one warp per scheduler) left the kernel latency bound (ncu r1: 3.45 TB/s, no pipe
// above 20 %); 8 warps x 3 stages x 16 keys doubles the warps per scheduler.
constexpr int kGqaTile = 16;      // keys per tile
constexpr int kGqaStages = 3;     // cp.async stages per warp
constexpr int kGqaWarps = 8;      // warps per CTA
constexpr int kGqaCtas = 1;       // resident CTAs per SM
constexpr int kGqaSmemBytes = kGqaWarps * kGqaStages * 2 * (kGqaTile * kGqaD * 2);   // [warp][stage][K tile | V tile]

__device__ __forceinline__ uint32_t movmatrix_trans(uint32_t a) {
  uint32_t d;
  asm volatile("movmatrix.sync.aligned.m8n8.trans.b16 %0, %1;" : "=r"(d) : "r"(a));
  return d;
}

// Smem of the e4m3-cache instances: per warp the ring of e4m3 tiles and one K | V tile pair in the io dtype.
constexpr int kGqaE4m3SmemBytes = kGqaWarps * (kGqaStages * 2 * (kGqaTile * kGqaD) + 2 * (kGqaTile * kGqaD * 2));

// CONTIG: the contiguous cache of gqa_decode_cta, with no page shift, so any cache_rows runs on tensor cores.
// C: the cache element, T or uint8_t (e4m3).  With e4m3 the ring stages e4m3 tiles (half the bytes per key) and each
// warp converts its tile into the io-dtype swizzled tile the MMA path reads; the new row is rounded to e4m3 once, and
// that value is both stored and staged.  Same tiles and splits as the io-dtype cache, so on e4m3-representable data
// the result is bit-identical.
template <typename T, typename C, int G, bool CONTIG>
__device__ __forceinline__ void gqa_decode_mmaT_cta(
    const T* __restrict__ q, C* __restrict__ k_cache, C* __restrict__ v_cache, const T* __restrict__ k_new,
    const T* __restrict__ v_new, int64_t k_new_sb, int64_t v_new_sb,
    const int32_t* __restrict__ seqlens, const int32_t* __restrict__ block_table, int bt_stride, int Hq, int Hkv,
    int page_shift, float scale, int num_splits, float* __restrict__ o_part, float* __restrict__ lse,
    T* __restrict__ out, int64_t q_sb, const float* __restrict__ cosp, const float* __restrict__ sinp, int64_t rows_sb,
    int cache_rows) {
  static_assert(G <= 8, "heads of one kv group are the n = 8 side of the MMA");
  constexpr bool kE4m3 = sizeof(C) == 1;
  static_assert(!(kE4m3 && CONTIG), "the e4m3 cache is paged");
  // Sequence lengths and the block table are written only by kernels that do not trigger dependents early (torch copies,
  // decode_prepare), so they are read before griddepcontrol.wait.  The K/V rows are not: the appends, the scatter and the
  // decode kernels (this one included) trigger early and write the cache after their own wait, so a cache row may still
  // be in flight until this kernel's wait returns.  No tile is loaded before it; the first tiles are only prefetched
  // into L2, which binds no value (the loads after the wait read through L2, where the writer's stores land).
  cb::pdl_launch_dependents();
  constexpr int D = kGqaD;
  constexpr int kTileBytes = kGqaTile * D * 2;              // K tile bytes (V the same)
  constexpr int kRingTile = kGqaTile * D * sizeof(C);       // bytes of a staged K tile
  constexpr int MT = kGqaTile / 16;                         // key m-tiles per tile
  extern __shared__ __align__(128) uint8_t gqa_smem[];      // [warp][stage][K tile | V tile] (e4m3: + [K | V] io)
  const int split = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int page_size = 1 << page_shift;
  const int L_cache = CONTIG ? min(seqlens[b], cache_rows) : seqlens[b];
  const int L = L_cache + (k_new ? 1 : 0);
  const int chunk = (((L + num_splits - 1) / num_splits) + kGqaTile - 1) / kGqaTile * kGqaTile;
  const int begin = split * chunk;
  const int end = min(begin + chunk, L);
  const int32_t* bt = block_table + (int64_t)b * bt_stride;

  const uint32_t smem_warp = (uint32_t)__cvta_generic_to_shared(gqa_smem) +
                             warp * (kGqaStages * 2 * kRingTile + (kE4m3 ? 2 * kTileBytes : 0));
  const int ntiles_total = end > begin ? (end - begin + kGqaTile - 1) / kGqaTile : 0;
  // tiles warp, warp + kGqaWarps, ...
  const int my_tiles = ntiles_total > warp ? (ntiles_total - warp + kGqaWarps - 1) / kGqaWarps : 0;

  auto cache_row = [&](int key) -> int64_t {    // row of (key, kvh) in units of D
    if constexpr (CONTIG) return ((int64_t)b * rows_sb + key) * Hkv + kvh;
    return ((int64_t)bt[key >> page_shift] * page_size + (key & (page_size - 1))) * Hkv + kvh;
  };
  auto issue = [&](int ti, int stage) {
    const int key0 = begin + (warp + kGqaWarps * ti) * kGqaTile;
    if constexpr (kE4m3) {                   // rows of 128 bytes, unswizzled; the appended and masked rows are zero
      const uint32_t sk = smem_warp + stage * (2 * kRingTile), sv = sk + kRingTile;
#pragma unroll
      for (int i = 0; i < kGqaTile / 4; ++i) {
        const int c = i * 32 + lane;         // 16-byte chunk id within the tile: row = c/8, col = c%8
        const int r = c >> 3, cc = c & 7;
        const int key = key0 + r;
        const C *ksrc = k_cache, *vsrc = v_cache;
        int nbytes = 0;
        if (key < L_cache && key < end) {
          const int64_t row = cache_row(key);
          ksrc = k_cache + row * D;
          vsrc = v_cache + row * D;
          nbytes = 16;
        }
        cp_async16_g(sk + c * 16, ksrc + cc * 16, nbytes);
        cp_async16_g(sv + c * 16, vsrc + cc * 16, nbytes);
      }
      cp_async_commit();
    } else {
      const uint32_t sk = smem_warp + stage * (2 * kTileBytes), sv = sk + kTileBytes;
#pragma unroll
      for (int i = 0; i < kGqaTile / 2; ++i) {
        const int c = i * 32 + lane;         // 16-byte chunk id within the tile: row = c/16, col = c%16
        const int r = c >> 4, cc = c & 15;
        const int key = key0 + r;
        const T *ksrc = k_cache, *vsrc = v_cache;
        int nbytes = 16;
        if (key < L_cache && key < end) {
          const int64_t row = cache_row(key);
          ksrc = k_cache + row * D;
          vsrc = v_cache + row * D;
        } else if (key < end) {              // the token being appended (key == L_cache)
          ksrc = k_new + (int64_t)b * k_new_sb + kvh * D;
          vsrc = v_new + (int64_t)b * v_new_sb + kvh * D;
        } else {
          nbytes = 0;                        // masked row: zero fill
        }
        const uint32_t off = r * 256 + ((cc ^ (r & 7)) << 4);
        cp_async16_g(sk + off, ksrc + cc * 8, nbytes);
        cp_async16_g(sv + off, vsrc + cc * 8, nbytes);
      }
      cp_async_commit();
    }
  };

  // the K and V rows of the tiles the prologue below stages, as 128-byte lines into L2
  constexpr int kRowLines = D * (int)sizeof(C) / 128;
#pragma unroll
  for (int s = 0; s < kGqaStages - 1; ++s) {
    const int key0 = begin + (warp + kGqaWarps * s) * kGqaTile;
#pragma unroll
    for (int i = lane; i < 2 * kGqaTile * kRowLines; i += 32) {
      const int key = key0 + i % kGqaTile, line = i / kGqaTile;
      if (s < my_tiles && key < L_cache && key < end) {
        const C* src = (line & 1 ? v_cache : k_cache) + cache_row(key) * D;
        asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const uint8_t*>(src) + (line >> 1) * 128));
      }
    }
  }
  cb::pdl_wait();
  cb::tl_stamp();

  // Fused rotary (cosp != null; apply_rotary_pos_emb "llama" = interleaved pairs, ops.py:311-326, arithmetic of
  // rotary_interleaved_vec_kernel): q is rotated in the MMA fragments (a 32-bit fragment word IS one (2i, 2i+1) pair),
  // the new k row is rotated once per warp (lane = dims 4*lane .. 4*lane+3) for the append and for the staged tile.
  auto rot_pair = [&](uint32_t w, int pair) -> uint32_t {
    const float c = cosp[(int64_t)b * (D / 2) + pair], sn = sinp[(int64_t)b * (D / 2) + pair];
    const T* pr = reinterpret_cast<const T*>(&w);
    const float x0 = io<T>::to_f(pr[0]), x1 = io<T>::to_f(pr[1]);
    const float o0 = __fmaf_rn(x0, c, -__fmul_rn(x1, sn));
    const float o1 = __fmaf_rn(x1, c, __fmul_rn(x0, sn));
    T po[2] = {io<T>::from_f(o0), io<T>::from_f(o1)};
    return *reinterpret_cast<const uint32_t*>(po);
  };
  uint2 k_rot = make_uint2(0u, 0u);
  if (k_new) {
    k_rot = reinterpret_cast<const uint2*>(k_new + (int64_t)b * k_new_sb + kvh * D)[lane];
    if (cosp) { k_rot.x = rot_pair(k_rot.x, 2 * lane); k_rot.y = rot_pair(k_rot.y, 2 * lane + 1); }
  }
  // e4m3: the new row rounded once; k8 / v8 are stored, their decoded values kd / vd replace the zero-filled staged row
  uint32_t k8 = 0u, v8 = 0u;
  uint2 kd = make_uint2(0u, 0u), vd = make_uint2(0u, 0u);
  if (kE4m3 && k_new) {
    const uint2 vr = reinterpret_cast<const uint2*>(v_new + (int64_t)b * v_new_sb + kvh * D)[lane];
    k8 = io2_to_e4m3x2<T>(k_rot.x) | io2_to_e4m3x2<T>(k_rot.y) << 16;
    v8 = io2_to_e4m3x2<T>(vr.x) | io2_to_e4m3x2<T>(vr.y) << 16;
    E4m3<T>::to_io(k8, kd.x, kd.y);
    E4m3<T>::to_io(v8, vd.x, vd.y);
  }
  if (k_new && split == 0 && warp == 0 && (!CONTIG || L_cache < cache_rows)) {   // in-place append (true page_size indexing)
    int64_t row;
    if constexpr (CONTIG) {
      row = ((int64_t)b * rows_sb + L_cache) * Hkv + kvh;
    } else {
      const int page = bt[L_cache >> page_shift];
      row = ((int64_t)page * page_size + (L_cache & (page_size - 1))) * Hkv + kvh;
    }
    if constexpr (kE4m3) {
      reinterpret_cast<uint32_t*>(k_cache + row * D)[lane] = k8;
      reinterpret_cast<uint32_t*>(v_cache + row * D)[lane] = v8;
    } else {
      const uint2* vs = reinterpret_cast<const uint2*>(v_new + (int64_t)b * v_new_sb + kvh * D);
      reinterpret_cast<uint2*>(k_cache + row * D)[lane] = k_rot;
      reinterpret_cast<uint2*>(v_cache + row * D)[lane] = vs[lane];
    }
  }

  // Q^T fragments (B operand, k = 16 dims x n = 8 heads): head g of the group, zero for g >= G
  uint32_t qb[8][2];
  {
    const T* q0 = q + (int64_t)b * q_sb + (int64_t)(kvh * G + g) * D;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      qb[ks][0] = g < G ? *reinterpret_cast<const uint32_t*>(q0 + ks * 16 + 2 * t) : 0u;
      qb[ks][1] = g < G ? *reinterpret_cast<const uint32_t*>(q0 + ks * 16 + 2 * t + 8) : 0u;
      if (cosp && g < G) {
        qb[ks][0] = rot_pair(qb[ks][0], ks * 8 + t);
        qb[ks][1] = rot_pair(qb[ks][1], ks * 8 + t + 4);
      }
    }
  }
  // O^T accumulators: m-tile dt = dims 16*dt..16*dt+15; [0],[1] = (dim g, heads 2t, 2t+1), [2],[3] = dim g+8
  float o[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float m1 = -INFINITY, m0 = -INFINITY, l0 = 0.f, l1 = 0.f;     // heads 2t and 2t+1 (log2 domain max)
  const float sc = scale * kLog2e;

  for (int s = 0; s < kGqaStages - 1; ++s) {
    if (s < my_tiles) issue(s, s);
    else cp_async_commit();
  }
  for (int ti = 0; ti < my_tiles; ++ti) {
    const int stage = ti % kGqaStages;
    if (ti + kGqaStages - 1 < my_tiles) issue(ti + kGqaStages - 1, (ti + kGqaStages - 1) % kGqaStages);
    else cp_async_commit();
    cp_async_wait<kGqaStages - 1>();
    __syncwarp();
    const uint32_t sk = smem_warp + (kE4m3 ? kGqaStages : stage) * (2 * kRingTile), sv = sk + kTileBytes;
    const int key0 = begin + (warp + kGqaWarps * ti) * kGqaTile;
    if constexpr (kE4m3) {
      // the staged e4m3 tiles -> io tiles: lane converts 16-byte chunks (16 dims of one key) into two swizzled chunks
      const uint32_t rk = smem_warp + stage * (2 * kRingTile);
#pragma unroll
      for (int kv = 0; kv < 2; ++kv) {
#pragma unroll
        for (int i = 0; i < kGqaTile / 4; ++i) {
          const int c = i * 32 + lane, r = c >> 3, cc = c & 7;
          uint32_t w[4], h[8];
          asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];"
                       : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "r"(rk + kv * kRingTile + c * 16));
#pragma unroll
          for (int j = 0; j < 4; ++j) E4m3<T>::to_io(w[j], h[2 * j], h[2 * j + 1]);
          const uint32_t dst = sk + kv * kTileBytes + r * 256;
          asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};"
                       ::"r"(dst + (((2 * cc) ^ (r & 7)) << 4)), "r"(h[0]), "r"(h[1]), "r"(h[2]), "r"(h[3]) : "memory");
          asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};"
                       ::"r"(dst + (((2 * cc + 1) ^ (r & 7)) << 4)), "r"(h[4]), "r"(h[5]), "r"(h[6]), "r"(h[7]) : "memory");
        }
      }
      if (k_new && L_cache >= key0 && L_cache < key0 + kGqaTile && L_cache < end) {
        const int r = L_cache - key0;
        const uint32_t a = sk + r * 256 + (((lane >> 1) ^ (r & 7)) << 4) + (lane & 1) * 8;
        asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(kd.x), "r"(kd.y) : "memory");
        asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a + kTileBytes), "r"(vd.x), "r"(vd.y) : "memory");
      }
      __syncwarp();
    } else if (cosp && k_new && L_cache >= key0 && L_cache < key0 + kGqaTile && L_cache < end) {
      // the appended row was staged un-rotated from k_new: overwrite it with the rotated row
      const int r = L_cache - key0;
      const uint32_t a = sk + r * 256 + (((lane >> 1) ^ (r & 7)) << 4) + (lane & 1) * 8;
      asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(k_rot.x), "r"(k_rot.y) : "memory");
      __syncwarp();
    }

    // ---- S^T = K Q^T : MT m-tiles (16 keys each) x 8 k-steps; even / odd k-steps accumulate separately
    //      so that a 16-key tile still has two independent MMA chains ----
    float sacc[MT][4], sodd[MT][4];
#pragma unroll
    for (int j = 0; j < MT; ++j) {
      sacc[j][0] = sacc[j][1] = sacc[j][2] = sacc[j][3] = 0.f;
      sodd[j][0] = sodd[j][1] = sodd[j][2] = sodd[j][3] = 0.f;
    }
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        // A matrices: {keys 0-7, d lo}, {keys 8-15, d lo}, {keys 0-7, d hi}, {keys 8-15, d hi}
        const int r = mt * 16 + (((lane >> 3) & 1) << 3) + (lane & 7);
        const int cc = ks * 2 + (lane >> 4);
        uint32_t ka[4];
        ldsm_x4(ka, sk + r * 256 + ((cc ^ (r & 7)) << 4));
        if (ks & 1) mma16816<T>(sodd[mt], ka, qb[ks][0], qb[ks][1]);
        else mma16816<T>(sacc[mt], ka, qb[ks][0], qb[ks][1]);
      }
    }
    // ---- online softmax: this thread holds heads 2t (m0, l0) and 2t+1 (m1, l1) for keys 16mt+g, 16mt+g+8 ----
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      const bool ok_lo = key0 + mt * 16 + g < end, ok_hi = key0 + mt * 16 + g + 8 < end;
      sacc[mt][0] = ok_lo ? (sacc[mt][0] + sodd[mt][0]) * sc : -INFINITY;
      sacc[mt][1] = ok_lo ? (sacc[mt][1] + sodd[mt][1]) * sc : -INFINITY;
      sacc[mt][2] = ok_hi ? (sacc[mt][2] + sodd[mt][2]) * sc : -INFINITY;
      sacc[mt][3] = ok_hi ? (sacc[mt][3] + sodd[mt][3]) * sc : -INFINITY;
      mx0 = fmaxf(mx0, fmaxf(sacc[mt][0], sacc[mt][2]));
      mx1 = fmaxf(mx1, fmaxf(sacc[mt][1], sacc[mt][3]));
    }
#pragma unroll
    for (int off = 4; off < 32; off <<= 1) {
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, off));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, off));
    }
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);     // finite: every tile has >= 1 valid key
    const float c0 = exp2f(m0 - mn0), c1 = exp2f(m1 - mn1);
    m0 = mn0; m1 = mn1;
    l0 *= c0; l1 *= c1;
#pragma unroll
    for (int j = 0; j < 8; ++j) { o[j][0] *= c0; o[j][1] *= c1; o[j][2] *= c0; o[j][3] *= c1; }
    uint32_t pb[MT][2];                      // P^T as B operand (k = 16 keys x n = 8 heads)
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      const float p0 = exp2f(sacc[mt][0] - mn0), p1 = exp2f(sacc[mt][1] - mn1);
      const float p2 = exp2f(sacc[mt][2] - mn0), p3 = exp2f(sacc[mt][3] - mn1);
      l0 += p0 + p2;
      l1 += p1 + p3;
      const T* tag = nullptr;
      pb[mt][0] = movmatrix_trans(pack2(p0, p1, tag));   // (keys 2t, 2t+1;   head g)
      pb[mt][1] = movmatrix_trans(pack2(p2, p3, tag));   // (keys 2t+8, 2t+9; head g)
    }
    // ---- O^T += V^T P^T : 8 m-tiles (16 dims each) x MT k-steps (16 keys each) ----
#pragma unroll
    for (int kk = 0; kk < MT; ++kk) {
#pragma unroll
      for (int dt = 0; dt < 8; ++dt) {
        // trans matrices: {keys 0-7, d lo}, {keys 0-7, d hi}, {keys 8-15, d lo}, {keys 8-15, d hi}
        const int r = kk * 16 + ((lane >> 4) << 3) + (lane & 7);
        const int cc = dt * 2 + ((lane >> 3) & 1);
        uint32_t va[4];
        ldsm_x4_trans(va, sv + r * 256 + ((cc ^ (r & 7)) << 4));
        mma16816<T>(o[dt], va, pb[kk][0], pb[kk][1]);
      }
    }
    __syncwarp();
  }
  cp_async_wait<0>();

  // finish the row sums across the 8 key lanes of a head, then merge the warps through shared memory
#pragma unroll
  for (int off = 4; off < 32; off <<= 1) {
    l0 += __shfl_xor_sync(0xffffffffu, l0, off);
    l1 += __shfl_xor_sync(0xffffffffu, l1, off);
  }
  __syncthreads();                            // all warps are done with their staging buffers
  constexpr int DS = D + 4;                   // padded head stride: heads 2t land in different banks
  float* s_o = reinterpret_cast<float*>(gqa_smem);                 // [kGqaWarps][G][DS]
  float* s_m = s_o + kGqaWarps * G * DS;                                // [kGqaWarps][G]
  float* s_l = s_m + kGqaWarps * G;                                     // [kGqaWarps][G]
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int h = 2 * t + e;
    if (h < G) {
      if (g == 0) { s_m[warp * G + h] = e ? m1 : m0; s_l[warp * G + h] = e ? l1 : l0; }
#pragma unroll
      for (int dt = 0; dt < 8; ++dt) {
        s_o[(warp * G + h) * DS + dt * 16 + g] = o[dt][e];
        s_o[(warp * G + h) * DS + dt * 16 + g + 8] = o[dt][2 + e];
      }
    }
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < G * D; idx += kGqaWarps * 32) {
    const int gg = idx / D, d = idx - gg * D;
    float mx = -INFINITY;
#pragma unroll
    for (int w = 0; w < kGqaWarps; ++w) mx = fmaxf(mx, s_m[w * G + gg]);
    float num = 0.f, den = 0.f;
#pragma unroll
    for (int w = 0; w < kGqaWarps; ++w) {
      const float mw = s_m[w * G + gg];
      if (mw == -INFINITY) continue;
      const float f = exp2f(mw - mx);
      num = fmaf(f, s_o[(w * G + gg) * DS + d], num);
      den = fmaf(f, s_l[w * G + gg], den);
    }
    const int h = kvh * G + gg;
    const float ov = den > 0.f ? num / den : 0.f;
    if (num_splits == 1) {
      out[((int64_t)b * Hq + h) * D + d] = io<T>::from_f(ov);
    } else {
      const int64_t pi = ((int64_t)b * Hq + h) * num_splits + split;
      o_part[pi * D + d] = ov;
      if (d == 0) lse[pi] = den > 0.f ? mx + log2f(den) : -INFINITY;
    }
  }
}

template <typename T, int G>
__global__ void __launch_bounds__(kGqaWarps * 32, kGqaCtas) gqa_decode_mmaT_kernel(
    const T* __restrict__ q, T* __restrict__ k_cache, T* __restrict__ v_cache, const T* __restrict__ k_new,
    const T* __restrict__ v_new, int64_t k_new_sb, int64_t v_new_sb,
    const int32_t* __restrict__ seqlens, const int32_t* __restrict__ block_table, int bt_stride, int Hq, int Hkv,
    int page_shift, float scale, int num_splits, float* __restrict__ o_part, float* __restrict__ lse,
    T* __restrict__ out, int64_t q_sb, const float* __restrict__ cosp, const float* __restrict__ sinp) {
  gqa_decode_mmaT_cta<T, T, G, false>(q, k_cache, v_cache, k_new, v_new, k_new_sb, v_new_sb, seqlens, block_table,
                                      bt_stride, Hq, Hkv, page_shift, scale, num_splits, o_part, lse, out, q_sb, cosp,
                                      sinp, 0, 0);
}

template <typename T, int G>
__global__ void __launch_bounds__(kGqaWarps * 32, kGqaCtas) gqa_decode_mmaT_e4m3_kernel(
    const T* __restrict__ q, uint8_t* __restrict__ k_cache, uint8_t* __restrict__ v_cache, const T* __restrict__ k_new,
    const T* __restrict__ v_new, int64_t k_new_sb, int64_t v_new_sb,
    const int32_t* __restrict__ seqlens, const int32_t* __restrict__ block_table, int bt_stride, int Hq, int Hkv,
    int page_shift, float scale, int num_splits, float* __restrict__ o_part, float* __restrict__ lse,
    T* __restrict__ out, int64_t q_sb, const float* __restrict__ cosp, const float* __restrict__ sinp) {
  gqa_decode_mmaT_cta<T, uint8_t, G, false>(q, k_cache, v_cache, k_new, v_new, k_new_sb, v_new_sb, seqlens,
                                            block_table, bt_stride, Hq, Hkv, page_shift, scale, num_splits, o_part, lse,
                                            out, q_sb, cosp, sinp, 0, 0);
}

template <typename T, int G>
__global__ void __launch_bounds__(kGqaWarps * 32, kGqaCtas) gqa_decode_mmaT_contig_kernel(
    const T* __restrict__ q, T* __restrict__ k_cache, T* __restrict__ v_cache, const T* __restrict__ k_new,
    const T* __restrict__ v_new, int64_t k_new_sb, int64_t v_new_sb, const int32_t* __restrict__ seqlens,
    int64_t rows_sb, int cache_rows, int Hq, int Hkv, float scale, int num_splits, float* __restrict__ o_part,
    float* __restrict__ lse, T* __restrict__ out) {
  gqa_decode_mmaT_cta<T, T, G, true>(q, k_cache, v_cache, k_new, v_new, k_new_sb, v_new_sb, seqlens, nullptr, 0, Hq,
                                     Hkv, 0, scale, num_splits, o_part, lse, out, (int64_t)Hq * kGqaD, nullptr, nullptr,
                                     rows_sb, cache_rows);
}

// The seqlen_q == 1 path of the three GQA entries, for arguments the entry has checked (B > 0): the split count
// (tensor cores: whole waves of kGqaCtas CTAs per SM; SIMT: ~4 CTAs per SM), shrunk to the workspace (none: 1 split),
// the attention and, with a split, the merge, logged as `entry`.  The paged layouts read block_table, bt_stride and
// page_size, the contiguous one rows_sb and cache_rows; q_sb and the rotary tables reach the paged tensor-core kernels.
int gqa_decode(const char* entry, KvLayout layout, bool tc, const void* q, int64_t q_sb, void* k_cache, void* v_cache,
               const void* k_new, const void* v_new, int64_t k_new_sb, int64_t v_new_sb, const float* rope_cos,
               const float* rope_sin, const int32_t* cache_seqlens, const int32_t* block_table, int bt_stride,
               int page_size, int64_t rows_sb, int cache_rows, int B, int Hq, int Hkv, int D, int max_len,
               float softmax_scale, void* out, void* workspace, int64_t workspace_bytes, int dtype, cudaStream_t st) {
  int splits = tc ? pick_splits_waves(B * Hkv, max_len, 132 * kGqaCtas) : pick_splits(B * Hkv, max_len, 256, 64);
  splits = workspace ? splits_that_fit(splits, (int64_t)B * Hq, D, workspace_bytes) : 1;
  const SplitKv part = split_kv_carve(workspace, workspace_bytes, (int64_t)B * Hq, D, splits);
  int page_shift = 0;                                       // the paged tensor-core kernels' power-of-two page
  if (tc && layout != KvLayout::kContiguous)
    while ((1 << page_shift) < page_size) ++page_shift;
  const dim3 grid(splits, Hkv, B), tc_block(kGqaWarps * 32), simt_block(128);
  int rc = dispatch_io_g(dtype, Hq / Hkv, [&](auto t, auto g) {
    using T = decltype(t);
    constexpr int G = decltype(g)::value;
    const T *qt = (const T*)q, *kn = (const T*)k_new, *vn = (const T*)v_new;
    T *kc = (T*)k_cache, *vc = (T*)v_cache, *o = (T*)out;
    float *op = part.o_part, *lse = part.lse;
    if (layout == KvLayout::kPagedE4m3)
      return launch_smem<gqa_decode_mmaT_e4m3_kernel<T, G>>(
          entry, grid, tc_block, kGqaE4m3SmemBytes, st, qt, (uint8_t*)k_cache, (uint8_t*)v_cache, kn, vn, k_new_sb,
          v_new_sb, cache_seqlens, block_table, bt_stride, Hq, Hkv, page_shift, softmax_scale, splits, op, lse, o, q_sb,
          rope_cos, rope_sin);
    if (layout == KvLayout::kContiguous && tc)
      return launch_smem<gqa_decode_mmaT_contig_kernel<T, G>>(
          entry, grid, tc_block, kGqaSmemBytes, st, qt, kc, vc, kn, vn, k_new_sb, v_new_sb, cache_seqlens, rows_sb,
          cache_rows, Hq, Hkv, softmax_scale, splits, op, lse, o);
    if (layout == KvLayout::kContiguous)
      launch_k(gqa_decode_contig_kernel<T, 64, G>, grid, simt_block, 0, st, qt, kc, vc, kn, vn, k_new_sb, v_new_sb,
               cache_seqlens, rows_sb, cache_rows, Hq, Hkv, softmax_scale, splits, op, lse, o);
    else if (tc)
      return launch_smem<gqa_decode_mmaT_kernel<T, G>>(
          entry, grid, tc_block, kGqaSmemBytes, st, qt, kc, vc, kn, vn, k_new_sb, v_new_sb, cache_seqlens, block_table,
          bt_stride, Hq, Hkv, page_shift, softmax_scale, splits, op, lse, o, q_sb, rope_cos, rope_sin);
    else
      launch_k(D == 128 ? gqa_decode_kernel<T, 128, G> : gqa_decode_kernel<T, 64, G>, grid, simt_block, 0, st, qt, kc,
               vc, kn, vn, k_new_sb, v_new_sb, cache_seqlens, block_table, bt_stride, Hq, Hkv, page_size,
               softmax_scale, splits, op, lse, o);
    return 0;
  });
  if (rc) return rc;
  CB_LAUNCHED_AS(entry, 1);
  if (splits > 1) {
    rc = launch_merge_splits(part.o_part, part.lse, out, B * Hq, splits, D, dtype, st);
    if (rc) return rc;
    CB_LAUNCHED_AS(entry, 1);
  }
  return 0;
}

}  // namespace

extern "C" int64_t chitu_b200_attn_workspace_bytes(int batch, int heads, int head_dim_v, int max_splits) {
  return split_kv_bytes((int64_t)batch * heads, head_dim_v, max_splits);
}

namespace cb {
int launch_merge_splits(const float* o_part, const float* lse, void* out, int rows, int splits, int dv, int dtype,
                        cudaStream_t st) {
#define MERGE(T, DV, THREADS) \
  launch_k(merge_splits_kernel<T, DV>, dim3(rows), dim3(THREADS), 0, st, o_part, lse, (T*)out, splits)
  if (dtype == CB_BF16 && dv == 128) MERGE(__nv_bfloat16, 128, 128);
  else if (dtype == CB_BF16 && dv == 64) MERGE(__nv_bfloat16, 64, 64);
  else if (dtype == CB_BF16 && dv == kMlaC) MERGE(__nv_bfloat16, kMlaC, 256);
  else if (dtype == CB_F16 && dv == 128) MERGE(__half, 128, 128);
  else if (dtype == CB_F16 && dv == 64) MERGE(__half, 64, 64);
  else return fail(-1, "merge_splits: no merge kernel for dtype %d, head dim %d", dtype, dv);
#undef MERGE
  return 0;
}
}  // namespace cb

extern "C" int chitu_b200_gqa_paged_decode(const void* q, void* k_cache, void* v_cache, const void* k_new,
                                           const void* v_new, int64_t k_new_sb, int64_t v_new_sb,
                                           const int32_t* cache_seqlens,
                                           const int32_t* block_table, int bt_stride, int B, int Hq,
                                           int Hkv, int D, int page_size, int max_seqlen_hint,
                                           float softmax_scale, void* out, void* workspace,
                                           int64_t workspace_bytes, int dtype, void* stream) {
  return chitu_b200_gqa_paged_decode_rope(q, (int64_t)Hq * D, k_cache, v_cache, k_new, v_new, k_new_sb, v_new_sb, nullptr,
                                          nullptr, cache_seqlens, block_table, bt_stride, B, Hq, Hkv, D, page_size,
                                          max_seqlen_hint, softmax_scale, out, workspace, workspace_bytes, dtype, stream);
}

extern "C" int chitu_b200_gqa_paged_decode_rope(const void* q, int64_t q_sb, void* k_cache, void* v_cache,
                                                const void* k_new, const void* v_new, int64_t k_new_sb,
                                                int64_t v_new_sb, const float* rope_cos, const float* rope_sin,
                                                const int32_t* cache_seqlens, const int32_t* block_table,
                                                int bt_stride, int B, int Hq, int Hkv, int D, int page_size,
                                                int max_seqlen_hint, float softmax_scale, void* out, void* workspace,
                                                int64_t workspace_bytes, int dtype, void* stream) {
  if (int rc = check_gqa_operands(__func__, q, k_cache, v_cache, cache_seqlens, out, k_new, v_new, k_new_sb, 0,
                                  v_new_sb, 0, false, dtype))
    return rc;
  CB_ARG(block_table);
  CB_ARG((rope_cos == nullptr) == (rope_sin == nullptr) && q_sb >= (int64_t)Hq * D && q_sb % 2 == 0);
  CB_ARG(B >= 0 && Hq > 0 && Hkv > 0 && Hq % Hkv == 0 && page_size > 0 && bt_stride > 0);
  CB_ARG(D == 64 || D == 128);
  if (B == 0) return 0;
  const int G = Hq / Hkv;
  CB_ARG(G == 1 || G == 2 || G == 4 || G == 8);
  const bool tc = D == kGqaD && (page_size & (page_size - 1)) == 0;
  if (!tc && (rope_cos || q_sb != (int64_t)Hq * D))
    return fail(-2, "gqa_paged_decode_rope: fused rotary / strided q need head_dim 128 and a power-of-two page");
  const int max_len = max_seqlen_hint > 0 ? max_seqlen_hint : bt_stride * page_size;
  return gqa_decode(__func__, KvLayout::kPaged, tc, q, q_sb, k_cache, v_cache, k_new, v_new, k_new_sb, v_new_sb,
                    rope_cos, rope_sin, cache_seqlens, block_table, bt_stride, page_size, 0, 0, B, Hq, Hkv, D, max_len,
                    softmax_scale, out, workspace, workspace_bytes, dtype, (cudaStream_t)stream);
}

// flash_attn_with_kvcache without a block table (include/chitu_b200.h): sq == 1 runs the decode kernels' contiguous
// variants here, sq > 1 the multi-token kernel's (gqa_prefill.cu).
extern "C" int chitu_b200_gqa_contiguous_attn(const void* q, void* k_cache, void* v_cache, int64_t cache_sb,
                                              int cache_rows, const void* k_new, const void* v_new, int64_t k_new_sb,
                                              int64_t k_new_st, int64_t v_new_sb, int64_t v_new_st,
                                              const int32_t* cache_seqlens, int B, int sq, int Hq, int Hkv, int D,
                                              int max_seqlen_hint, int causal, float softmax_scale, void* out,
                                              void* workspace, int64_t workspace_bytes, int dtype, void* stream) {
  if (int rc = check_gqa_operands(__func__, q, k_cache, v_cache, cache_seqlens, out, k_new, v_new, k_new_sb, k_new_st,
                                  v_new_sb, v_new_st, sq > 1, dtype))
    return rc;
  CB_ARG(B >= 0 && B <= 65535 && sq >= 1 && Hq > 0 && Hkv > 0 && Hkv <= 65535 && Hq % Hkv == 0);
  const int G = Hq / Hkv;
  CB_ARG(G == 1 || G == 2 || G == 4 || G == 8);
  CB_ARG(D == 128 || (D == 64 && sq == 1));
  const int64_t row = (int64_t)Hkv * D;                     // elements of one cache position
  CB_ARG(cache_rows >= 1 && cache_sb >= cache_rows * row && cache_sb % row == 0 && cache_sb % 8 == 0);
  CB_ARG(workspace == nullptr || (uintptr_t)workspace % 16 == 0);
  if (B == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int max_len = max_seqlen_hint > 0 ? max_seqlen_hint : cache_rows;
  const int64_t rows_sb = cache_sb / row;
  if (sq > 1)
    return gqa_prefill(__func__, "gqa_contiguous_prefill", KvLayout::kContiguous, q, k_cache, v_cache, k_new, v_new,
                       k_new_sb, k_new_st, v_new_sb, v_new_st, cache_seqlens, nullptr, 0, 0, 0, rows_sb, cache_rows, B,
                       sq, Hq, Hkv, max_len, causal, softmax_scale, out, workspace, workspace_bytes, dtype, st);
  return gqa_decode(__func__, KvLayout::kContiguous, D == kGqaD, q, (int64_t)Hq * D, k_cache, v_cache, k_new, v_new,
                    k_new_sb, v_new_sb, nullptr, nullptr, cache_seqlens, nullptr, 0, 0, rows_sb, cache_rows, B, Hq, Hkv,
                    D, max_len, softmax_scale, out, workspace, workspace_bytes, dtype, st);
}

// flash_attn_with_kvcache (paged) over an e4m3 cache (include/chitu_b200.h): sq == 1 runs the e4m3 instance of the
// tensor-core decode kernel here, sq > 1 the multi-token kernel's (gqa_prefill.cu).
extern "C" int chitu_b200_gqa_paged_attn_fp8kv(const void* q, int64_t q_sb, void* k_cache, void* v_cache,
                                               const void* k_new, const void* v_new, int64_t k_new_sb, int64_t k_new_st,
                                               int64_t v_new_sb, int64_t v_new_st, const float* rope_cos,
                                               const float* rope_sin, const int32_t* cache_seqlens,
                                               const int32_t* block_table, int bt_stride, int B, int sq, int Hq,
                                               int Hkv, int D, int page_size, int num_blocks, int max_seqlen_hint,
                                               int causal, float softmax_scale, void* out, void* workspace,
                                               int64_t workspace_bytes, int dtype, void* stream) {
  if (int rc = check_gqa_operands(__func__, q, k_cache, v_cache, cache_seqlens, out, k_new, v_new, k_new_sb, k_new_st,
                                  v_new_sb, v_new_st, sq > 1, dtype))
    return rc;
  CB_ARG(block_table && (rope_cos == nullptr) == (rope_sin == nullptr));
  CB_ARG(B >= 0 && B <= 65535 && sq >= 1 && Hq > 0 && Hkv > 0 && Hkv <= 65535 && Hq % Hkv == 0);
  const int G = Hq / Hkv;
  CB_ARG(G == 1 || G == 2 || G == 4 || G == 8);
  CB_ARG(D == kGqaD);
  CB_ARG(bt_stride > 0 && num_blocks > 0 && page_size >= 64 && page_size % 64 == 0 &&
         (page_size & (page_size - 1)) == 0 && (int64_t)num_blocks * page_size <= 0x7fffffff);
  CB_ARG(rope_cos == nullptr || sq == 1);
  CB_ARG((int64_t)sq * Hq <= 0x7fffffff / D && q_sb % 8 == 0 &&
         (sq == 1 ? q_sb >= (int64_t)Hq * D : q_sb == (int64_t)sq * Hq * D));
  CB_ARG(workspace == nullptr || (uintptr_t)workspace % 16 == 0);
  if (B == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int max_len = max_seqlen_hint > 0 ? max_seqlen_hint : bt_stride * page_size;
  if (sq > 1)
    return gqa_prefill(__func__, "gqa_paged_prefill_e4m3", KvLayout::kPagedE4m3, q, k_cache, v_cache, k_new, v_new,
                       k_new_sb, k_new_st, v_new_sb, v_new_st, cache_seqlens, block_table, bt_stride, page_size,
                       num_blocks, 0, 0, B, sq, Hq, Hkv, max_len, causal, softmax_scale, out, workspace,
                       workspace_bytes, dtype, st);
  return gqa_decode(__func__, KvLayout::kPagedE4m3, true, q, q_sb, k_cache, v_cache, k_new, v_new, k_new_sb, v_new_sb,
                    rope_cos, rope_sin, cache_seqlens, block_table, bt_stride, page_size, 0, 0, B, Hq, Hkv, D, max_len,
                    softmax_scale, out, workspace, workspace_bytes, dtype, st);
}

// ============================================================================================
// MLA weight absorption (the two torch.einsum of AttentionDeepSeekV3, model_deepseek_v3.py:529-531
// and :697; SURVEY K8): wkv_b (bf16, [H, dn + dv, C]) is W_UK = [:, :dn] and W_UV = [:, dn:].
//   absorb_q : q'[b,h,c] = sum_d q_nope[b,h,d] * W_UK[h,d,c]        ("shd,hdc->shc", a role of mla_prep below)
//   absorb_o : o[b,h,d]  = sum_c x[b,h,c]     * W_UV[h,d,c]        ("bshc,hdc->bshd")
// Both stream the 2 MB of per-rank absorbed weights once for all tokens (fp32 accumulate).
// ============================================================================================
// CTA = (head, token chunk): warp w computes output dims [w*dv/8, (w+1)*dv/8) (one W_UV row at a time,
// lanes stride C); with dv == 128 the head's 128 outputs are exactly one act_quant group, so the fp8
// payload + scale of the following `wo` linear can be produced here (q_out != null).
// With `o_part` != null the latent input is the split-KV partials of the attention kernel and the LSE-weighted merge
// (merge_splits_kernel's arithmetic: split_weights, the same fmaf order, one bf16 rounding) happens while staging: the
// merge launch and its [B,H,C] round trip disappear.
template <int MT>
__global__ void __launch_bounds__(256) mla_absorb_o_kernel(const __nv_bfloat16* __restrict__ x,
                                                          const __nv_bfloat16* __restrict__ w,
                                                          __nv_bfloat16* __restrict__ out, uint8_t* __restrict__ q_out,
                                                          float* __restrict__ q_scales, int B, int H, int dn,
                                                          int dv, int C, const float* __restrict__ o_part,
                                                          const float* __restrict__ lse, int num_splits,
                                                          __nv_bfloat16* __restrict__ x_out) {
  cb::pdl_launch_dependents();
  __shared__ float s_o[MT][128];
  __shared__ float s_mw[MT][kMaxSplits];                        // normalised split weights
  extern __shared__ __align__(16) uint8_t s_x_raw[];            // [MT][C] bf16 latent outputs of this head
  __nv_bfloat16* s_x = reinterpret_cast<__nv_bfloat16*>(s_x_raw);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int h = blockIdx.x;
  const int b0 = blockIdx.y * MT;
  // W_UV rows in flight per warp: all 2 x RU 16-byte loads of a block of rows are issued before the first FMA (the old
  // RU = 4 loop with the loads inside the c loop was a chain of 8 dependent L2 round trips: 19 us for 2 MB of weights).
  // The first block is requested BEFORE griddepcontrol.wait: the weights are immutable, so their HBM / L2 latency hides
  // under the tail of the attention kernel (in-graph timeline r2 call 10: this kernel was 14-15 us at bs = 1 and 16).
  constexpr int RU = 8;
  const int rows_per_warp = dv / 8;
  uint4 wv[2][RU];
  if (C == 512) {
#pragma unroll
    for (int cc = 0; cc < 2; ++cc)
#pragma unroll
      for (int u = 0; u < RU; ++u)
        wv[cc][u] = ld_stream(w + ((int64_t)h * (dn + dv) + dn + warp * rows_per_warp + u) * C + cc * 256 + lane * 8);
  }
  cb::pdl_wait();
  cb::tl_stamp();
  if (o_part) {
    for (int m = warp; m < MT; m += 8) {                        // warp m: the split weights of token b0 + m
      const int b = min(b0 + m, B - 1);
      split_weights(lse + ((int64_t)b * H + h) * num_splits, num_splits, s_mw[m], lane);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < MT * (C / 4); i += 256) {
      const int m = i / (C / 4), c4 = i - m * (C / 4);
      const int b = min(b0 + m, B - 1);
      const float* base = o_part + ((int64_t)b * H + h) * num_splits * C + c4 * 4;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      int sp = 0;
      for (; sp + 8 <= num_splits; sp += 8) {                   // 8 independent L2 loads in flight
        float4 v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = *reinterpret_cast<const float4*>(base + (int64_t)(sp + u) * C);
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const float wv_ = s_mw[m][sp + u];
          acc.x = fmaf(wv_, v[u].x, acc.x); acc.y = fmaf(wv_, v[u].y, acc.y);
          acc.z = fmaf(wv_, v[u].z, acc.z); acc.w = fmaf(wv_, v[u].w, acc.w);
        }
      }
      for (; sp + 4 <= num_splits; sp += 4) {                   // 4 independent L2 loads in flight
        float4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = *reinterpret_cast<const float4*>(base + (int64_t)(sp + u) * C);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const float wv = s_mw[m][sp + u];
          acc.x = fmaf(wv, v[u].x, acc.x); acc.y = fmaf(wv, v[u].y, acc.y);
          acc.z = fmaf(wv, v[u].z, acc.z); acc.w = fmaf(wv, v[u].w, acc.w);
        }
      }
      for (; sp < num_splits; ++sp) {
        const float4 v = *reinterpret_cast<const float4*>(base + (int64_t)sp * C);
        const float wv = s_mw[m][sp];
        acc.x = fmaf(wv, v.x, acc.x); acc.y = fmaf(wv, v.y, acc.y);
        acc.z = fmaf(wv, v.z, acc.z); acc.w = fmaf(wv, v.w, acc.w);
      }
      const __nv_bfloat16* tag = nullptr;
      const uint2 pk = make_uint2(pack2(acc.x, acc.y, tag), pack2(acc.z, acc.w, tag));
      *reinterpret_cast<uint2*>(s_x + m * C + c4 * 4) = pk;
      if (x_out && b0 + m < B) *reinterpret_cast<uint2*>(x_out + ((int64_t)(b0 + m) * H + h) * C + c4 * 4) = pk;
    }
  } else {
    for (int i = threadIdx.x; i < MT * (C / 8); i += 256) {
      const int m = i / (C / 8), ch = i - m * (C / 8);
      const int b = min(b0 + m, B - 1);
      reinterpret_cast<uint4*>(s_x)[i] = *reinterpret_cast<const uint4*>(x + ((int64_t)b * H + h) * C + ch * 8);
    }
  }
  __syncthreads();
  for (int rr = 0; rr < rows_per_warp; rr += RU) {
    const int d0 = warp * rows_per_warp + rr;
    float acc[RU][MT];
#pragma unroll
    for (int u = 0; u < RU; ++u)
#pragma unroll
      for (int m = 0; m < MT; ++m) acc[u][m] = 0.f;
    if (C == 512) {
      if (rr > 0) {                                             // block 0 was requested before the dependency wait
#pragma unroll
        for (int cc = 0; cc < 2; ++cc)
#pragma unroll
          for (int u = 0; u < RU; ++u)
            wv[cc][u] = ld_stream(w + ((int64_t)h * (dn + dv) + dn + d0 + u) * C + cc * 256 + lane * 8);
      }
#pragma unroll
      for (int cc = 0; cc < 2; ++cc) {
#pragma unroll
        for (int m = 0; m < MT; ++m) {
          const uint4 xv = *reinterpret_cast<const uint4*>(s_x + m * C + cc * 256 + lane * 8);
          const uint32_t xx[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
          for (int u = 0; u < RU; ++u) {
            const uint32_t ww[4] = {wv[cc][u].x, wv[cc][u].y, wv[cc][u].z, wv[cc][u].w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              acc[u][m] = fmaf(bf16lo(ww[i]), bf16lo(xx[i]), acc[u][m]);
              acc[u][m] = fmaf(bf16hi(ww[i]), bf16hi(xx[i]), acc[u][m]);
            }
          }
        }
      }
    } else {
      for (int c = lane * 8; c < C; c += 256) {
        uint4 wg[RU];
#pragma unroll
        for (int u = 0; u < RU; ++u)
          wg[u] = *reinterpret_cast<const uint4*>(w + ((int64_t)h * (dn + dv) + dn + d0 + u) * C + c);
#pragma unroll
        for (int m = 0; m < MT; ++m) {
          const uint4 xv = *reinterpret_cast<const uint4*>(s_x + m * C + c);
          const uint32_t xx[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
          for (int u = 0; u < RU; ++u) {
            const uint32_t ww[4] = {wg[u].x, wg[u].y, wg[u].z, wg[u].w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              acc[u][m] = fmaf(bf16lo(ww[i]), bf16lo(xx[i]), acc[u][m]);
              acc[u][m] = fmaf(bf16hi(ww[i]), bf16hi(xx[i]), acc[u][m]);
            }
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < RU; ++u)
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        const float v = warp_sum(acc[u][m]);
        if (lane == 0) s_o[m][d0 + u] = __bfloat162float(__float2bfloat16_rn(v));
      }
  }
  __syncthreads();
  // write bf16 and (optionally) the quantised group: warp m handles token b0+m (MT <= 8 warps)
  for (int m = warp; m < MT; m += 8) {
    if (b0 + m >= B) continue;
    for (int d0 = 0; d0 < dv; d0 += 128) {
      float v[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) v[i] = (d0 + lane * 4 + i < dv) ? s_o[m][d0 + lane * 4 + i] : 0.f;
      const int64_t o = ((int64_t)(b0 + m) * H + h) * dv + d0 + lane * 4;
      if (out) {
        const __nv_bfloat16* tag = nullptr;
        *reinterpret_cast<uint2*>(out + o) = make_uint2(pack2(v[0], v[1], tag), pack2(v[2], v[3], tag));
      }
      if (q_out) {
        const E4m3Word<4> g = e4m3_group_quant<E4m3Group::kActQuant>(v);
        *reinterpret_cast<uint32_t*>(q_out + o) = g.bits[0];
        if (lane == 0) q_scales[((int64_t)(b0 + m) * H + h) * (dv / 128) + d0 / 128] = g.scale;
      }
    }
  }
}

extern "C" int chitu_b200_mla_absorb_o_quant(const void* x, const void* wkv_b, void* out, void* q_out,
                                             float* q_scales, int B, int H, int dn, int dv, int C, void* stream) {
  CB_ARG(x && wkv_b && (out || q_out) && B >= 0 && H > 0 && dn > 0 && dv > 0 && C > 0 && C % 8 == 0);
  CB_ARG(dv == 128 && (q_out == nullptr) == (q_scales == nullptr));
  CB_ARG(((uintptr_t)x | (uintptr_t)wkv_b) % 16 == 0 && (uintptr_t)out % 8 == 0 && (uintptr_t)q_out % 4 == 0);
  if (B == 0) return 0;
  constexpr int MT = 2;          // tokens per CTA: 128 CTAs at bs = 16, one merge item per thread
  CB_ARG(dv % 32 == 0);
  dim3 grid(H, cdiv(B, MT));
  cb::launch_k(mla_absorb_o_kernel<MT>, grid, dim3(256), (size_t)MT * C * 2, (cudaStream_t)stream, (const __nv_bfloat16*)x,
               (const __nv_bfloat16*)wkv_b, (__nv_bfloat16*)out, (uint8_t*)q_out, q_scales, B, H, dn, dv, C,
               (const float*)nullptr, (const float*)nullptr, 0, (__nv_bfloat16*)nullptr);
  CB_LAUNCHED(1);
  return 0;
}

// absorb-o (+ act_quant) reading the split-KV partials that chitu_b200_mla_decode(out = NULL) left in `workspace`:
// merge + absorb + quantise in one launch.  `max_seqlen_hint`, B, H and the workspace must be the ones given to
// chitu_b200_mla_decode (the split count is recomputed from them).  x_out (optional): the merged latent output [B,H,C].
extern "C" int chitu_b200_mla_absorb_o_merge_quant(const void* workspace, int64_t workspace_bytes, int max_seqlen_hint,
                                                   const void* wkv_b, void* x_out, void* out, void* q_out, float* q_scales,
                                                   int B, int H, int dn, int dv, int C, void* stream) {
  CB_ARG(workspace && wkv_b && (out || q_out) && B >= 0 && H > 0 && dn > 0 && dv == 128 && C == kMlaC);
  CB_ARG((q_out == nullptr) == (q_scales == nullptr) && max_seqlen_hint > 0);
  CB_ARG(((uintptr_t)workspace | (uintptr_t)wkv_b) % 16 == 0 && ((uintptr_t)x_out | (uintptr_t)out) % 8 == 0 &&
         (uintptr_t)q_out % 4 == 0);                                   // float4 partials, uint4 weights, uint2 rows
  if (B == 0) return 0;
  const int splits = mla_num_splits(B, H, max_seqlen_hint, workspace_bytes);
  CB_ARG(split_kv_bytes((int64_t)B * H, kMlaC, splits) <= workspace_bytes);
  const auto [o_part, lse, plan] = split_kv_carve((void*)workspace, workspace_bytes, (int64_t)B * H, kMlaC, splits);
  constexpr int MT = 2;
  dim3 grid(H, cdiv(B, MT));
  cb::launch_k(mla_absorb_o_kernel<MT>, grid, dim3(256), (size_t)MT * C * 2, (cudaStream_t)stream,
               (const __nv_bfloat16*)nullptr, (const __nv_bfloat16*)wkv_b, (__nv_bfloat16*)out, (uint8_t*)q_out, q_scales, B,
               H, dn, dv, C, o_part, lse, splits, (__nv_bfloat16*)x_out);
  CB_LAUNCHED(1);
  return 0;
}


// ============================================================================================
// mla_prep: everything between the wq_b GEMM and the attention call of decode_forward_paged
// (model_deepseek_v3.py:489-531, 684-686) in ONE launch instead of three:
//   blocks [0, nA)      : q_abs = q_nope · W_UK                      (absorb_q role, see above)
//   blocks [nA, nA + B) : per token: q_pe <- rotary(q_pe), k_pe <- rotary(k_pe),
//                         new_kv = [kv_norm(kv) | k_pe]              (apply_rotary_pos_emb + RMSNorm + cat)
// ============================================================================================
template <int MT>
__global__ void __launch_bounds__(256) mla_prep_kernel(
    const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ kv_in, int64_t kv_sb,
    const __nv_bfloat16* __restrict__ kv_norm_w, const float* __restrict__ cosp, const float* __restrict__ sinp,
    const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ q_abs, __nv_bfloat16* __restrict__ q_pe,
    __nv_bfloat16* __restrict__ new_kv, int B, int H, int dn, int dv, int C, int R, float eps, int nA) {
  cb::pdl_prologue();
  extern __shared__ float s_abs[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int qk = dn + R;
  if ((int)blockIdx.x < nA) {
    // ---- absorb_q role: CTA = (64-column chunk, head, token chunk); the 8 warps split the dn reduction dim, a lane
    // owns two adjacent columns, and the partial sums are combined through shared memory ----
    const int ncx = C / 64;
    const int cx = blockIdx.x % ncx, h = (blockIdx.x / ncx) % H, z = blockIdx.x / (ncx * H);
    float* s_q = s_abs;
    float* s_red = s_abs + MT * dn;
    const int c = cx * 64 + lane * 2;
    const int b0 = z * MT;
    for (int i = threadIdx.x; i < MT * dn; i += 256) {
      const int m = i / dn, d = i - m * dn;
      s_q[i] = (b0 + m < B) ? __bfloat162float(q[((int64_t)(b0 + m) * H + h) * qk + d]) : 0.f;
    }
    __syncthreads();
    float acc0[MT], acc1[MT];
#pragma unroll
    for (int m = 0; m < MT; ++m) acc0[m] = acc1[m] = 0.f;
    const int dper = dn / 8;
    const __nv_bfloat16* wp = w + ((int64_t)h * (dn + dv) + warp * dper) * C + c;
    // all weight loads of a block of 16 rows are issued before the first FMA (one L2 round trip instead of four)
    for (int d0 = 0; d0 < dper; d0 += 16) {
      uint32_t uu[16];
#pragma unroll
      for (int i = 0; i < 16; ++i)
        uu[i] = d0 + i < dper ? *reinterpret_cast<const uint32_t*>(wp + (int64_t)(d0 + i) * C) : 0u;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        if (d0 + i >= dper) break;
        const float w0 = bf16lo(uu[i]), w1 = bf16hi(uu[i]);
#pragma unroll
        for (int m = 0; m < MT; ++m) {
          const float qv = s_q[m * dn + warp * dper + d0 + i];
          acc0[m] = fmaf(qv, w0, acc0[m]);
          acc1[m] = fmaf(qv, w1, acc1[m]);
        }
      }
    }
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      s_red[(warp * MT + m) * 64 + lane * 2] = acc0[m];
      s_red[(warp * MT + m) * 64 + lane * 2 + 1] = acc1[m];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < MT * 64; i += 256) {
      const int m = i / 64, cc = i - m * 64;
      float v = 0.f;
#pragma unroll
      for (int wq = 0; wq < 8; ++wq) v += s_red[(wq * MT + m) * 64 + cc];
      if (b0 + m < B) q_abs[((int64_t)(b0 + m) * H + h) * C + cx * 64 + cc] = __float2bfloat16_rn(v);
    }
    return;
  }
  // ---- token role ----
  const int b = blockIdx.x - nA;
  const __nv_bfloat16* kvr = kv_in + (int64_t)b * kv_sb;          // [C kv | R k_pe]
  __nv_bfloat16* nk = new_kv + (int64_t)b * (C + R);
  // kv_norm (fp32 math, one rounding)
  float ss = 0.f;
  for (int i = threadIdx.x; i < C; i += 256) {
    const float v = __bfloat162float(kvr[i]);
    ss += v * v;
  }
  __shared__ float red[8];
  ss = warp_sum(ss);
  if (lane == 0) red[warp] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += red[i];
  const float rinv = rsqrtf(tot / (float)C + eps);
  for (int i = threadIdx.x; i < C; i += 256)
    nk[i] = __float2bfloat16_rn(__bfloat162float(kvr[i]) * rinv * __bfloat162float(kv_norm_w[i]));
  // interleaved rotary on the H q_pe heads and on k_pe (fp32 cos/sin, one rounding)
  const int half = R / 2;
  for (int idx = threadIdx.x; idx < (H + 1) * half; idx += 256) {
    const int hh = idx / half, i = idx - hh * half;
    const float cs = cosp[(int64_t)b * half + i], sn = sinp[(int64_t)b * half + i];
    const __nv_bfloat16* src = hh < H ? q + ((int64_t)b * H + hh) * qk + dn : kvr + C;
    __nv_bfloat16* dst = hh < H ? q_pe + ((int64_t)b * H + hh) * R : nk + C;
    const float x0 = __bfloat162float(src[2 * i]), x1 = __bfloat162float(src[2 * i + 1]);
    dst[2 * i] = __float2bfloat16_rn(x0 * cs - x1 * sn);
    dst[2 * i + 1] = __float2bfloat16_rn(x1 * cs + x0 * sn);
  }
}

extern "C" int chitu_b200_mla_prep(const void* q, const void* kv_in, int64_t kv_sb, const void* kv_norm_w,
                                   const float* cos, const float* sin, const void* wkv_b, void* q_abs, void* q_pe,
                                   void* new_kv, int B, int H, int dn, int dv, int C, int R, float eps,
                                   void* stream) {
  CB_ARG(q && kv_in && kv_norm_w && cos && sin && wkv_b && q_abs && q_pe && new_kv);
  CB_ARG(B >= 0 && H > 0 && dn % 8 == 0 && C % 64 == 0 && R % 2 == 0);
  CB_ARG((uintptr_t)wkv_b % 4 == 0);                                   // W_UK column pairs are read as uint32
  if (B == 0) return 0;
  constexpr int MT = 16;
  const int nA = (C / 64) * H * cdiv(B, MT);
  const size_t smem = (size_t)(MT * dn + 8 * MT * 64) * 4;
  cb::launch_k(mla_prep_kernel<MT>, dim3(nA + B), dim3(256), smem, (cudaStream_t)stream, (const __nv_bfloat16*)q,
               (const __nv_bfloat16*)kv_in, kv_sb, (const __nv_bfloat16*)kv_norm_w, cos, sin,
               (const __nv_bfloat16*)wkv_b, (__nv_bfloat16*)q_abs, (__nv_bfloat16*)q_pe, (__nv_bfloat16*)new_kv, B, H,
               dn, dv, C, R, eps, nA);
  CB_LAUNCHED(1);
  return 0;
}

CB_DEFINE_TL_SETTER(attention)
