// Paged-KV decode attention, split-KV ("flash decoding"), SIMT implementation.
//
//  * gqa_paged_decode : AttnBackend.attn_with_kvcache with a block_table (attn_backend.py:92-164,
//    FlashAttn impl :208-243) — GQA, in-place append of the new token, page gather through the
//    block table, online softmax in fp32, LSE-weighted merge of the splits.
//  * mla_decode       : *.mla_attn_with_kvcache (attn_backend.py:707-774) = append (ops.py:50-91)
//    + absorbed-MLA split-KV attention (triton_decode_attention.py:20-130) + merge (:185-232).
//    V is a view of the first C columns of the same cache row, so each row is read once.
//
// Both kernels never read the cache row of the token being appended: the CTA that owns that
// position takes it from `k_new` directly and split 0 writes it to the cache -> no RAW hazard.
// The reference fixes NUM_KV_SPLITS = 4 (attn_backend.py:735) -> 4 CTAs at B=1; here the split
// count is sized from the SM count so the 132 SMs of an H100 are busy at B=1.
#include <stdlib.h>

#include "common.cuh"
#include "tc_ptx.cuh"

using namespace cb;

namespace {

constexpr float kLog2e = 1.4426950408889634f;

// partial layout in the workspace: o_part[B, H, S, Dv] fp32 (already normalised), lse[B, H, S]
// (log2 domain: m + log2(l)), S = num_splits.

template <typename T, int DV>
__global__ void merge_splits_kernel(const float* __restrict__ o_part, const float* __restrict__ lse,
                                    T* __restrict__ out, int num_splits) {
  cb::pdl_prologue();
  __shared__ float s_w[128];                      // normalised split weights (num_splits <= 128)
  const int64_t bh = blockIdx.x;  // b * H + h
  const float* l = lse + bh * num_splits;
  if (threadIdx.x < 32) {
    float mx = -INFINITY;
    for (int s = threadIdx.x; s < num_splits; s += 32) mx = fmaxf(mx, l[s]);
    mx = warp_max(mx);
    float den = 0.f;
    for (int s = threadIdx.x; s < num_splits; s += 32) {
      const float ls = l[s];
      const float wv = ls == -INFINITY ? 0.f : exp2f(ls - mx);
      s_w[s] = wv;
      den += wv;
    }
    den = warp_sum(den);
    const float inv = den > 0.f ? 1.f / den : 0.f;
    for (int s = threadIdx.x; s < num_splits; s += 32) s_w[s] *= inv;
  }
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
template <typename T, int D, int G>
__global__ void __launch_bounds__(128) gqa_decode_kernel(
    const T* __restrict__ q, T* __restrict__ k_cache, T* __restrict__ v_cache,
    const T* __restrict__ k_new, const T* __restrict__ v_new, int64_t k_new_sb, int64_t v_new_sb,
    const int32_t* __restrict__ seqlens,
    const int32_t* __restrict__ block_table, int bt_stride, int Hq, int Hkv, int page_size, float scale,
    int num_splits, float* __restrict__ o_part, float* __restrict__ lse, T* __restrict__ out) {
  cb::pdl_prologue();
  constexpr int VEC = D / 32;
  const int split = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int L_cache = seqlens[b];
  const int L = L_cache + (k_new ? 1 : 0);
  const int chunk = (L + num_splits - 1) / num_splits;
  const int begin = split * chunk;
  const int end = min(begin + chunk, L);
  const int32_t* bt = block_table + (int64_t)b * bt_stride;

  // in-place append of the new token (true page_size indexing, as flash_attn_with_kvcache does)
  if (k_new && split == 0 && warp == 0) {
    const int page = bt[L_cache / page_size];
    const int64_t row = ((int64_t)page * page_size + L_cache % page_size) * Hkv + kvh;
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
        const int page = bt[key / page_size];
        const int64_t row = ((int64_t)page * page_size + key % page_size) * Hkv + kvh;
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

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }

// --------------------------------------------------------------------------------------------
// GQA, tensor-core version (D = 128): one CTA (4 warps) per (split, kv head, request).
// Each warp streams its own 32-key tiles of K and V through a private 3-stage cp.async ring in
// shared memory (no block-level barrier in the main loop), computes S = Q K^T and O += P V with
// mma.sync.m16n8k16 (the G <= 16 query heads of the group are the 16 MMA rows, so every K/V byte
// is read once for all heads), FA2-style register softmax, and the four warps are merged at the end.
// K tiles are read with ldmatrix, V tiles with ldmatrix.trans; rows are XOR-swizzled in 16-byte
// chunks so both are bank-conflict free.
// --------------------------------------------------------------------------------------------
constexpr int kGqaD = 128;
// tile / pipeline / warp configuration (TILE keys per tile, STAGES cp.async stages per warp, WARPS warps per CTA)
// is a template parameter: 4 warps x 3 stages x 32 keys (one warp per scheduler) left the kernel latency bound
// (ncu r1: 3.45 TB/s, no pipe above 20 %); 8 warps x 3 stages x 16 keys doubles the warps per scheduler.

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

template <typename T, int G, int TILE, int STAGES, int WARPS, int CTAS>
__global__ void __launch_bounds__(WARPS * 32, CTAS) gqa_decode_mma_kernel(
    const T* __restrict__ q, T* __restrict__ k_cache, T* __restrict__ v_cache,
    const T* __restrict__ k_new, const T* __restrict__ v_new, int64_t k_new_sb, int64_t v_new_sb,
    const int32_t* __restrict__ seqlens, const int32_t* __restrict__ block_table, int bt_stride, int Hq, int Hkv,
    int page_shift, float scale, int num_splits, float* __restrict__ o_part, float* __restrict__ lse,
    T* __restrict__ out, int64_t q_sb, const float* __restrict__ cosp, const float* __restrict__ sinp) {
  cb::pdl_prologue();
  constexpr int D = kGqaD;
  constexpr int kGqaTile = TILE, kGqaStages = STAGES;
  constexpr int kTileBytes = kGqaTile * D * 2;              // K tile bytes (V the same)
  extern __shared__ __align__(128) uint8_t gqa_smem[];      // [warp][stage][K tile | V tile]
  const int split = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int page_size = 1 << page_shift;
  const int L_cache = seqlens[b];
  const int L = L_cache + (k_new ? 1 : 0);
  const int chunk = (((L + num_splits - 1) / num_splits) + kGqaTile - 1) / kGqaTile * kGqaTile;
  const int begin = split * chunk;
  const int end = min(begin + chunk, L);
  const int32_t* bt = block_table + (int64_t)b * bt_stride;

  if (k_new && split == 0 && warp == 0) {   // in-place append (true page_size indexing)
    const int page = bt[L_cache >> page_shift];
    const int64_t row = ((int64_t)page * page_size + (L_cache & (page_size - 1))) * Hkv + kvh;
    const uint2* ks = reinterpret_cast<const uint2*>(k_new + (int64_t)b * k_new_sb + kvh * D);
    const uint2* vs = reinterpret_cast<const uint2*>(v_new + (int64_t)b * v_new_sb + kvh * D);
    reinterpret_cast<uint2*>(k_cache + row * D)[lane] = ks[lane];
    reinterpret_cast<uint2*>(v_cache + row * D)[lane] = vs[lane];
  }

  // Q fragments (A operand, 16 x 128): rows >= G are zero padding
  uint32_t qa[8][4];
  {
    const T* q0 = q + (int64_t)b * q_sb + (int64_t)(kvh * G) * D;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const int c0 = ks * 16 + 2 * t;
      qa[ks][0] = g < G ? *reinterpret_cast<const uint32_t*>(q0 + g * D + c0) : 0u;
      qa[ks][1] = g + 8 < G ? *reinterpret_cast<const uint32_t*>(q0 + (g + 8) * D + c0) : 0u;
      qa[ks][2] = g < G ? *reinterpret_cast<const uint32_t*>(q0 + g * D + c0 + 8) : 0u;
      qa[ks][3] = g + 8 < G ? *reinterpret_cast<const uint32_t*>(q0 + (g + 8) * D + c0 + 8) : 0u;
    }
  }
  float o[16][4];
#pragma unroll
  for (int j = 0; j < 16; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;     // rows g and g+8 (log2 domain max)
  const float sc = scale * kLog2e;

  const uint32_t smem_warp = (uint32_t)__cvta_generic_to_shared(gqa_smem) + warp * (kGqaStages * 2 * kTileBytes);
  const int ntiles_total = end > begin ? (end - begin + kGqaTile - 1) / kGqaTile : 0;
  const int my_tiles = ntiles_total > warp ? (ntiles_total - warp + WARPS - 1) / WARPS : 0;   // tiles warp, warp+WARPS, ...

  auto issue = [&](int ti, int stage) {
    const int key0 = begin + (warp + WARPS * ti) * kGqaTile;
    const uint32_t sk = smem_warp + stage * (2 * kTileBytes), sv = sk + kTileBytes;
#pragma unroll
    for (int i = 0; i < kGqaTile / 2; ++i) {
      const int c = i * 32 + lane;           // 16-byte chunk id within the tile: row = c/16, col = c%16
      const int r = c >> 4, cc = c & 15;
      const int key = key0 + r;
      const T *ksrc = k_cache, *vsrc = v_cache;
      int nbytes = 16;
      if (key < L_cache && key < end) {
        const int page = bt[key >> page_shift];
        const int64_t row = ((int64_t)page * page_size + (key & (page_size - 1))) * Hkv + kvh;
        ksrc = k_cache + row * D;
        vsrc = v_cache + row * D;
      } else if (key < end) {                // the token being appended (key == L_cache)
        ksrc = k_new + (int64_t)b * k_new_sb + kvh * D;
        vsrc = v_new + (int64_t)b * v_new_sb + kvh * D;
      } else {
        nbytes = 0;                          // masked row: zero fill
      }
      const uint32_t off = r * 256 + ((cc ^ (r & 7)) << 4);
      cp_async16_g(sk + off, ksrc + cc * 8, nbytes);
      cp_async16_g(sv + off, vsrc + cc * 8, nbytes);
    }
    cp_async_commit();
  };

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
    const uint32_t sk = smem_warp + stage * (2 * kTileBytes), sv = sk + kTileBytes;
    const int key0 = begin + (warp + WARPS * ti) * kGqaTile;
    constexpr int NT = kGqaTile / 8;          // score n-tiles (8 keys each)

    // ---- S = Q K^T : NT n-tiles x 8 k-steps ----
    float sacc[NT][4];
#pragma unroll
    for (int j = 0; j < NT; ++j) sacc[j][0] = sacc[j][1] = sacc[j][2] = sacc[j][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
      for (int jp = 0; jp < NT / 2; ++jp) {  // pairs of n-tiles: keys 16*jp .. 16*jp+15
        // matrices: {keys 0-7, d lo}, {keys 0-7, d hi}, {keys 8-15, d lo}, {keys 8-15, d hi}
        const int r = jp * 16 + ((lane >> 4) << 3) + (lane & 7);
        const int cc = ks * 2 + ((lane >> 3) & 1);
        uint32_t kb[4];
        ldsm_x4(kb, sk + r * 256 + ((cc ^ (r & 7)) << 4));
        mma16816<T>(sacc[jp * 2], qa[ks], kb[0], kb[1]);
        mma16816<T>(sacc[jp * 2 + 1], qa[ks], kb[2], kb[3]);
      }
    }
    // ---- online softmax (rows g, g+8; this thread holds keys 8j+2t, 8j+2t+1) ----
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const bool ok = key0 + j * 8 + 2 * t + e < end;
        sacc[j][e] = ok ? sacc[j][e] * sc : -INFINITY;
        sacc[j][2 + e] = ok ? sacc[j][2 + e] * sc : -INFINITY;
        mx0 = fmaxf(mx0, sacc[j][e]);
        mx1 = fmaxf(mx1, sacc[j][2 + e]);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);     // finite: every tile has >= 1 valid key
    const float c0 = exp2f(m0 - mn0), c1 = exp2f(m1 - mn1);
    m0 = mn0; m1 = mn1;
    l0 *= c0; l1 *= c1;
#pragma unroll
    for (int j = 0; j < 16; ++j) { o[j][0] *= c0; o[j][1] *= c0; o[j][2] *= c1; o[j][3] *= c1; }
    uint32_t pa[NT / 2][4];                  // P as A operand: NT/2 k-steps of 16 keys
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      const float p0 = exp2f(sacc[j][0] - mn0), p1 = exp2f(sacc[j][1] - mn0);
      const float p2 = exp2f(sacc[j][2] - mn1), p3 = exp2f(sacc[j][3] - mn1);
      l0 += p0 + p1;
      l1 += p2 + p3;
      const T* tag = nullptr;
      pa[j >> 1][(j & 1) * 2] = pack2(p0, p1, tag);          // (row g,   keys 8j+2t..)
      pa[j >> 1][(j & 1) * 2 + 1] = pack2(p2, p3, tag);      // (row g+8, keys 8j+2t..)
    }
    // ---- O += P V : 16 n-tiles (8 dims each) x 2 k-steps (16 keys each) ----
#pragma unroll
    for (int kk = 0; kk < NT / 2; ++kk) {
#pragma unroll
      for (int dp = 0; dp < 8; ++dp) {        // pairs of d n-tiles: dims 16*dp .. 16*dp+15
        // trans matrices: {keys 0-7, d lo}, {keys 8-15, d lo}, {keys 0-7, d hi}, {keys 8-15, d hi}
        const int r = kk * 16 + (((lane >> 3) & 1) << 3) + (lane & 7);
        const int cc = dp * 2 + (lane >> 4);
        uint32_t vb[4];
        ldsm_x4_trans(vb, sv + r * 256 + ((cc ^ (r & 7)) << 4));
        mma16816<T>(o[dp * 2], pa[kk], vb[0], vb[1]);
        mma16816<T>(o[dp * 2 + 1], pa[kk], vb[2], vb[3]);
      }
    }
    __syncwarp();
  }
  cp_async_wait<0>();

  // finish the row sums across the 4 lanes of a row, then merge the 4 warps through shared memory
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  __syncthreads();                            // all warps are done with their staging buffers
  float* s_o = reinterpret_cast<float*>(gqa_smem);                 // [WARPS][G][D]
  float* s_m = s_o + WARPS * G * D;                                 // [WARPS][G]
  float* s_l = s_m + WARPS * G;                                     // [WARPS][G]
  if (g < G) {
    if (t == 0) { s_m[warp * G + g] = m0; s_l[warp * G + g] = l0; }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      s_o[(warp * G + g) * D + j * 8 + 2 * t] = o[j][0];
      s_o[(warp * G + g) * D + j * 8 + 2 * t + 1] = o[j][1];
    }
  }
  if (g + 8 < G) {
    if (t == 0) { s_m[warp * G + g + 8] = m1; s_l[warp * G + g + 8] = l1; }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      s_o[(warp * G + g + 8) * D + j * 8 + 2 * t] = o[j][2];
      s_o[(warp * G + g + 8) * D + j * 8 + 2 * t + 1] = o[j][3];
    }
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < G * D; idx += WARPS * 32) {
    const int gg = idx / D, d = idx - gg * D;
    float mx = -INFINITY;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) mx = fmaxf(mx, s_m[w * G + gg]);
    float num = 0.f, den = 0.f;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) {
      const float mw = s_m[w * G + gg];
      if (mw == -INFINITY) continue;
      const float f = exp2f(mw - mx);
      num = fmaf(f, s_o[(w * G + gg) * D + d], num);
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

// --------------------------------------------------------------------------------------------
// GQA, tensor-core version with the KEYS as the MMA M dimension ("swap-AB"): S^T = K Q^T and
// O^T = V^T P^T.  With G <= 8 query heads per kv head the head dimension fits the n = 8 side of
// m16n8k16 exactly, so a 32-key tile costs 32 MMAs instead of the 64 (half of them on zero padding
// rows) of the heads-as-M kernel above, and the O accumulator is 32 registers instead of 64.
// P^T is produced from the S^T accumulator fragments with movmatrix.trans (8x8 b16 transpose in
// registers).  Staging, swizzle, split handling and the warp merge are those of the kernel above.
// --------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t movmatrix_trans(uint32_t a) {
  uint32_t d;
  asm volatile("movmatrix.sync.aligned.m8n8.trans.b16 %0, %1;" : "=r"(d) : "r"(a));
  return d;
}
template <typename T>
__device__ __forceinline__ void mma16816r(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  mma16816<T>(d, a, b0, b1);
}

template <typename T, int G, int TILE, int STAGES, int WARPS, int CTAS>
__global__ void __launch_bounds__(WARPS * 32, CTAS) gqa_decode_mmaT_kernel(
    const T* __restrict__ q, T* __restrict__ k_cache, T* __restrict__ v_cache, const T* __restrict__ k_new,
    const T* __restrict__ v_new, int64_t k_new_sb, int64_t v_new_sb,
    const int32_t* __restrict__ seqlens, const int32_t* __restrict__ block_table, int bt_stride, int Hq, int Hkv,
    int page_shift, float scale, int num_splits, float* __restrict__ o_part, float* __restrict__ lse,
    T* __restrict__ out, int64_t q_sb, const float* __restrict__ cosp, const float* __restrict__ sinp) {
  static_assert(G <= 8, "heads of one kv group are the n = 8 side of the MMA");
  // The K/V pages are only written by earlier decode steps and by this kernel; sequence lengths and the block table by
  // kernels that do not trigger dependents early: the first tiles of every warp are put in flight BEFORE
  // griddepcontrol.wait (they overlap the tail of the qkv GEMM); q / k_new / v_new (the previous kernel's output) are
  // only touched after it.
  cb::pdl_launch_dependents();
  constexpr int D = kGqaD;
  constexpr int kTileBytes = TILE * D * 2;                  // K tile bytes (V the same)
  constexpr int MT = TILE / 16;                             // key m-tiles per tile
  extern __shared__ __align__(128) uint8_t gqa_smem[];      // [warp][stage][K tile | V tile]
  const int split = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int page_size = 1 << page_shift;
  const int L_cache = seqlens[b];
  const int L = L_cache + (k_new ? 1 : 0);
  const int chunk = (((L + num_splits - 1) / num_splits) + TILE - 1) / TILE * TILE;
  const int begin = split * chunk;
  const int end = min(begin + chunk, L);
  const int32_t* bt = block_table + (int64_t)b * bt_stride;

  const uint32_t smem_warp = (uint32_t)__cvta_generic_to_shared(gqa_smem) + warp * (STAGES * 2 * kTileBytes);
  const int ntiles_total = end > begin ? (end - begin + TILE - 1) / TILE : 0;
  const int my_tiles = ntiles_total > warp ? (ntiles_total - warp + WARPS - 1) / WARPS : 0;   // tiles warp, warp+WARPS, ...

  auto issue = [&](int ti, int stage) {
    const int key0 = begin + (warp + WARPS * ti) * TILE;
    const uint32_t sk = smem_warp + stage * (2 * kTileBytes), sv = sk + kTileBytes;
#pragma unroll
    for (int i = 0; i < TILE / 2; ++i) {
      const int c = i * 32 + lane;           // 16-byte chunk id within the tile: row = c/16, col = c%16
      const int r = c >> 4, cc = c & 15;
      const int key = key0 + r;
      const T *ksrc = k_cache, *vsrc = v_cache;
      int nbytes = 16;
      if (key < L_cache && key < end) {
        const int page = bt[key >> page_shift];
        const int64_t row = ((int64_t)page * page_size + (key & (page_size - 1))) * Hkv + kvh;
        ksrc = k_cache + row * D;
        vsrc = v_cache + row * D;
      } else if (key < end) {                // the token being appended (key == L_cache)
        ksrc = k_new + (int64_t)b * k_new_sb + kvh * D;
        vsrc = v_new + (int64_t)b * v_new_sb + kvh * D;
      } else {
        nbytes = 0;                          // masked row: zero fill
      }
      const uint32_t off = r * 256 + ((cc ^ (r & 7)) << 4);
      cp_async16_g(sk + off, ksrc + cc * 8, nbytes);
      cp_async16_g(sv + off, vsrc + cc * 8, nbytes);
    }
    cp_async_commit();
  };

  // tiles that lie completely inside the cached part of the sequence can be fetched before the previous kernel is done
  bool early[STAGES - 1];
#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    early[s] = s < my_tiles && begin + (warp + WARPS * s + 1) * TILE <= min(L_cache, end);
    if (early[s]) issue(s, s);
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
  if (k_new && split == 0 && warp == 0) {   // in-place append (true page_size indexing)
    const int page = bt[L_cache >> page_shift];
    const int64_t row = ((int64_t)page * page_size + (L_cache & (page_size - 1))) * Hkv + kvh;
    const uint2* vs = reinterpret_cast<const uint2*>(v_new + (int64_t)b * v_new_sb + kvh * D);
    reinterpret_cast<uint2*>(k_cache + row * D)[lane] = k_rot;
    reinterpret_cast<uint2*>(v_cache + row * D)[lane] = vs[lane];
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
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;     // heads 2t and 2t+1 (log2 domain max)
  const float sc = scale * kLog2e;

  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < my_tiles && !early[s]) issue(s, s);
    else if (!early[s]) cp_async_commit();
  }
  for (int ti = 0; ti < my_tiles; ++ti) {
    const int stage = ti % STAGES;
    if (ti + STAGES - 1 < my_tiles) issue(ti + STAGES - 1, (ti + STAGES - 1) % STAGES);
    else cp_async_commit();
    cp_async_wait<STAGES - 1>();
    __syncwarp();
    const uint32_t sk = smem_warp + stage * (2 * kTileBytes), sv = sk + kTileBytes;
    const int key0 = begin + (warp + WARPS * ti) * TILE;
    if (cosp && k_new && L_cache >= key0 && L_cache < key0 + TILE && L_cache < end) {
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
  float* s_o = reinterpret_cast<float*>(gqa_smem);                 // [WARPS][G][DS]
  float* s_m = s_o + WARPS * G * DS;                                // [WARPS][G]
  float* s_l = s_m + WARPS * G;                                     // [WARPS][G]
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
  for (int idx = threadIdx.x; idx < G * D; idx += WARPS * 32) {
    const int gg = idx / D, d = idx - gg * D;
    float mx = -INFINITY;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) mx = fmaxf(mx, s_m[w * G + gg]);
    float num = 0.f, den = 0.f;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) {
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

// --------------------------------------------------------------------------------------------
// MLA (C = 512 latent dims, R = 64 rope dims): one CTA per (split, 16-head group, request).
// K rows ([C+R] bf16 = 1152 B) are staged through shared memory with cp.async (double buffered,
// 16 keys per tile) so the four warps — each owning 4 heads — share one HBM read of every row.
// A lane owns latent dims [16*lane, 16*lane+16) and rope dims [2*lane, 2*lane+2).
// --------------------------------------------------------------------------------------------
constexpr int kMlaC = 512, kMlaR = 64, kMlaRow = kMlaC + kMlaR;
constexpr int kMlaTile = 16;   // keys per smem tile
constexpr int kMlaHPW = 4;     // heads per warp


__global__ void __launch_bounds__(128) mla_decode_kernel(
    const __nv_bfloat16* __restrict__ q_nope, const __nv_bfloat16* __restrict__ q_pe,
    __nv_bfloat16* __restrict__ kv_cache, const __nv_bfloat16* __restrict__ new_kv,
    const int32_t* __restrict__ seqlens_excl, const int32_t* __restrict__ block_table, int bt_stride,
    int H, int page_size, float scale, int num_splits, float* __restrict__ o_part,
    float* __restrict__ lse, __nv_bfloat16* __restrict__ out) {
  cb::pdl_prologue();
  __shared__ __align__(16) __nv_bfloat16 s_k[2][kMlaTile][kMlaRow];
  const int split = blockIdx.x, hg = blockIdx.y, b = blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int L_cache = seqlens_excl[b];
  const int L = L_cache + (new_kv ? 1 : 0);
  const int chunk = (((L + num_splits - 1) / num_splits) + kMlaTile - 1) / kMlaTile * kMlaTile;
  const int begin = split * chunk;
  const int end = min(begin + chunk, L);
  const int32_t* bt = block_table + (int64_t)b * bt_stride;

  // append (reference semantics incl. the literal-64 page arithmetic are handled by the caller
  // passing page_size == 64 for MLA, backend.py:234-237; here true page_size indexing is used)
  if (new_kv && split == 0 && hg == 0) {
    const int page = bt[L_cache / page_size];
    __nv_bfloat16* dst = kv_cache + ((int64_t)page * page_size + L_cache % page_size) * kMlaRow;
    const __nv_bfloat16* src = new_kv + (int64_t)b * kMlaRow;
    for (int i = threadIdx.x; i < kMlaRow / 8; i += 128)
      reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
  }

  const int h0 = hg * 16 + warp * kMlaHPW;
  float qn[kMlaHPW][16], qp[kMlaHPW][2], acc[kMlaHPW][16], m[kMlaHPW], l[kMlaHPW];
  const float qs = scale * kLog2e;
#pragma unroll
  for (int g = 0; g < kMlaHPW; ++g) {
    const int h = min(h0 + g, H - 1);
    const __nv_bfloat16* a = q_nope + ((int64_t)b * H + h) * kMlaC + lane * 16;
    const __nv_bfloat16* p = q_pe + ((int64_t)b * H + h) * kMlaR + lane * 2;
#pragma unroll
    for (int i = 0; i < 16; ++i) { qn[g][i] = __bfloat162float(a[i]) * qs; acc[g][i] = 0.f; }
    qp[g][0] = __bfloat162float(p[0]) * qs;
    qp[g][1] = __bfloat162float(p[1]) * qs;
    m[g] = -INFINITY;
    l[g] = 0.f;
  }

  auto issue_tile = [&](int tile_begin, int buf) {
    // 16 rows x 72 chunks of 16 B = 1152 chunks, 9 per thread
    for (int c = threadIdx.x; c < kMlaTile * (kMlaRow / 8); c += 128) {
      const int r = c / (kMlaRow / 8), cc = c - r * (kMlaRow / 8);
      const int key = tile_begin + r;
      const __nv_bfloat16* src;
      if (key < L_cache && key < end) {
        const int page = bt[key / page_size];
        src = kv_cache + ((int64_t)page * page_size + key % page_size) * kMlaRow;
      } else if (new_kv) {
        src = new_kv + (int64_t)b * kMlaRow;          // the appended token / masked filler
      } else {
        src = kv_cache;                               // masked filler (never used)
      }
      cp_async16(&s_k[buf][r][cc * 8], src + cc * 8);
    }
    cp_async_commit();
  };

  const int ntiles = end > begin ? (end - begin + kMlaTile - 1) / kMlaTile : 0;
  if (ntiles > 0) issue_tile(begin, 0);
  for (int t = 0; t < ntiles; ++t) {
    const int buf = t & 1;
    if (t + 1 < ntiles) {
      issue_tile(begin + (t + 1) * kMlaTile, buf ^ 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const int nk = min(kMlaTile, end - (begin + t * kMlaTile));
    for (int r = 0; r < nk; ++r) {
      const uint4* kr = reinterpret_cast<const uint4*>(&s_k[buf][r][lane * 16]);
      uint4 k0 = kr[0], k1 = kr[1];
      uint32_t kpe = *reinterpret_cast<const uint32_t*>(&s_k[buf][r][kMlaC + lane * 2]);
      const uint32_t kw[8] = {k0.x, k0.y, k0.z, k0.w, k1.x, k1.y, k1.z, k1.w};
      float kf[16];
#pragma unroll
      for (int i = 0; i < 8; ++i) { kf[2 * i] = bf16lo(kw[i]); kf[2 * i + 1] = bf16hi(kw[i]); }
      const float kp0 = bf16lo(kpe), kp1 = bf16hi(kpe);
#pragma unroll
      for (int g = 0; g < kMlaHPW; ++g) {
        float s = qp[g][0] * kp0;
        s = fmaf(qp[g][1], kp1, s);
#pragma unroll
        for (int i = 0; i < 16; ++i) s = fmaf(qn[g][i], kf[i], s);
        s = warp_sum(s);
        const float mn = fmaxf(m[g], s);
        const float corr = exp2f(m[g] - mn);
        // p stays fp32 (the reference rounds it to bf16 first, triton_decode_attention.py:113)
        const float p = exp2f(s - mn);
        l[g] = l[g] * corr + p;
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[g][i] = fmaf(p, kf[i], acc[g][i] * corr);
        m[g] = mn;
      }
    }
    __syncthreads();
  }

#pragma unroll
  for (int g = 0; g < kMlaHPW; ++g) {
    const int h = h0 + g;
    if (h >= H) continue;
    const float inv = l[g] > 0.f ? 1.f / l[g] : 0.f;
    if (num_splits == 1) {
      __nv_bfloat16* o = out + ((int64_t)b * H + h) * kMlaC + lane * 16;
#pragma unroll
      for (int i = 0; i < 16; ++i) o[i] = __float2bfloat16_rn(acc[g][i] * inv);
    } else {
      const int64_t pi = ((int64_t)b * H + h) * num_splits + split;
      float* o = o_part + pi * kMlaC + lane * 16;
#pragma unroll
      for (int i = 0; i < 16; ++i) o[i] = acc[g][i] * inv;
      if (lane == 0) lse[pi] = l[g] > 0.f ? m[g] + log2f(l[g]) : -INFINITY;
    }
  }
}

// one CTA per SM kernels: ~3 CTAs per SM in total, >= 256 keys per split
// --------------------------------------------------------------------------------------------
// MLA, tensor-core version (C = 512, R = 64, page = 64, H <= 16 heads per CTA).
//   * warp 4 (producer): one elected lane stages each 64-key page with 9 TMA boxes
//     ([64 rows x 128 B], 128B-swizzled) into a 2-stage shared-memory ring (mbarrier full/empty);
//     the compressed-KV row is read ONCE and serves both as K (576 dims) and as V (first 512 dims).
//   * warps 0-3 (compute): all 16 heads are the 16 rows of one mma.sync tile.  S = Q K^T is split
//     over the keys (warp w: keys 16w..16w+15, 72 MMAs), the row max is exchanged through shared
//     memory, P (bf16) goes to shared memory once, and O += P V is split over the latent dims
//     (warp w: dims 128w..128w+127, 64 MMAs) so the accumulators stay at 64 registers per thread.
//   * the token being appended is patched into the staged tile from `new_kv` (its cache row is
//     written by split 0 for later steps, never read in this launch); rows past the sequence end
//     are zero-filled in shared memory so that 0 * garbage cannot poison P·V.
// --------------------------------------------------------------------------------------------
constexpr int kMtTile = 64;                               // keys per tile == page size
constexpr int kMtBox = kMtTile * 128;                     // one TMA box: 64 rows x 128 B
constexpr int kMtStageBytes = 9 * kMtBox;                 // 73,728 B
constexpr int kMtStages = 2;
constexpr int kMtQBytes = 9 * 16 * 128;                   // Q: 16 rows x 576 dims, same blocked layout
constexpr int kMtPBytes = 16 * 128;                       // P: 16 rows x 64 keys bf16

// byte offset of (row, 16-byte chunk c of column block b) inside a [blocks][rows][128 B] swizzled tile
__device__ __forceinline__ uint32_t sw_off(int rows_per_block, int b, int row, int c) {
  return (uint32_t)(b * rows_per_block * 128 + row * 128 + ((c ^ (row & 7)) << 4));
}

__global__ void __launch_bounds__(160, 1) mla_decode_mma_kernel(
    const __grid_constant__ CUtensorMap map_kv, const __nv_bfloat16* __restrict__ q_nope,
    const __nv_bfloat16* __restrict__ q_pe, __nv_bfloat16* __restrict__ kv_cache,
    const __nv_bfloat16* __restrict__ new_kv, const int32_t* __restrict__ seqlens_excl,
    const int32_t* __restrict__ block_table, int bt_stride, int H, float scale, int num_splits,
    float* __restrict__ o_part, float* __restrict__ lse, __nv_bfloat16* __restrict__ out) {
  extern __shared__ __align__(1024) uint8_t mla_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(mla_smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_kv = smem;                                         // [stages][9][64][128 B]
  uint8_t* s_q = s_kv + kMtStages * kMtStageBytes;              // [9][16][128 B]
  uint8_t* s_p = s_q + kMtQBytes;                               // [16][128 B]
  float* s_max = reinterpret_cast<float*>(s_p + kMtPBytes);     // [4 warps][16 rows]
  float* s_sum = s_max + 64;                                    // [4 warps][16 rows] (epilogue)
  __shared__ __align__(8) uint64_t full_bar[kMtStages], empty_bar[kMtStages];

  const int split = blockIdx.x, hg = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  constexpr int C = kMlaC, R = kMlaR, ROW = kMlaRow;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kMtStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_kv) : "memory");
  }
  cb::pdl_launch_dependents();
  __syncthreads();
  cb::pdl_wait();
  cb::tl_stamp();

  const int L_cache = seqlens_excl[b];
  const int L = L_cache + (new_kv ? 1 : 0);
  const int chunk = (((L + num_splits - 1) / num_splits) + kMtTile - 1) / kMtTile * kMtTile;
  const int begin = split * chunk;
  const int end = min(begin + chunk, L);
  const int ntiles = end > begin ? (end - begin + kMtTile - 1) / kMtTile : 0;
  const int32_t* bt = block_table + (int64_t)b * bt_stride;
  const int h0 = hg * 16;

  if (new_kv && split == 0 && hg == 0 && warp < 4) {     // append for the following steps
    const int page = bt[L_cache / kMtTile];
    __nv_bfloat16* dst = kv_cache + ((int64_t)page * kMtTile + L_cache % kMtTile) * ROW;
    const __nv_bfloat16* src = new_kv + (int64_t)b * ROW;
    for (int i = threadIdx.x; i < ROW / 8; i += 128)
      reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
  }

  if (warp == 4) {
    // ================= TMA producer =================
    if (elect_one()) {
      const uint64_t pol = l2_policy_evict_first();
      for (int it = 0; it < ntiles; ++it) {
        const int s = it % kMtStages;
        mbar_wait(&empty_bar[s], ((it / kMtStages) & 1) ^ 1);
        mbar_expect_tx(&full_bar[s], kMtStageBytes);
        const int key0 = begin + it * kMtTile;
        const int row0 = bt[key0 / kMtTile] * kMtTile;
#pragma unroll
        for (int cb_ = 0; cb_ < 9; ++cb_)
          tma_load_2d(s_kv + s * kMtStageBytes + cb_ * kMtBox, &map_kv, &full_bar[s], cb_ * 64, row0, pol);
      }
    }
    return;
  }

  // ================= compute warps =================
  // Q -> shared memory in the blocked + swizzled layout ([9][16 rows][128 B]); rows >= H are zero
  for (int i = threadIdx.x; i < 16 * (ROW / 8); i += 128) {
    const int row = i / (ROW / 8), ch = i - row * (ROW / 8);      // 72 chunks of 16 B per row
    uint4 v = make_uint4(0, 0, 0, 0);
    if (h0 + row < H) {
      const __nv_bfloat16* src = ch < C / 8 ? q_nope + ((int64_t)b * H + h0 + row) * C + ch * 8
                                            : q_pe + ((int64_t)b * H + h0 + row) * R + (ch - C / 8) * 8;
      v = *reinterpret_cast<const uint4*>(src);
    }
    *reinterpret_cast<uint4*>(s_q + sw_off(16, ch >> 3, row, ch & 7)) = v;
  }
  asm volatile("bar.sync 1, 128;" ::: "memory");

  float o[16][4];
#pragma unroll
  for (int j = 0; j < 16; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  const float sc = scale * kLog2e;
  const uint32_t sq_a = smem_u32(s_q), sp_a = smem_u32(s_p);

  for (int it = 0; it < ntiles; ++it) {
    const int s = it % kMtStages;
    const int key0 = begin + it * kMtTile;
    const int nvalid = min(kMtTile, end - key0);
    uint8_t* tile = s_kv + s * kMtStageBytes;
    const uint32_t tile_a = smem_u32(tile);
    mbar_wait(&full_bar[s], (it / kMtStages) & 1);
    // patch the appended token / zero the rows past the end (generic-proxy writes after the TMA landed)
    const int patch_row = (new_kv && L_cache >= key0 && L_cache < key0 + kMtTile) ? L_cache - key0 : -1;
    if (patch_row >= 0 || nvalid < kMtTile) {
      if (patch_row >= 0) {
        for (int i = threadIdx.x; i < ROW / 8; i += 128)
          *reinterpret_cast<uint4*>(tile + sw_off(kMtTile, i >> 3, patch_row, i & 7)) =
              *reinterpret_cast<const uint4*>(new_kv + (int64_t)b * ROW + i * 8);
      }
      for (int i = threadIdx.x; i < (kMtTile - nvalid) * (ROW / 8); i += 128) {
        const int row = nvalid + i / (ROW / 8), ch = i % (ROW / 8);
        *reinterpret_cast<uint4*>(tile + sw_off(kMtTile, ch >> 3, row, ch & 7)) = make_uint4(0, 0, 0, 0);
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");
    }

    // ---- S[16 x 16 keys of this warp] = Q K^T over 576 dims: 9 column blocks x 4 k-steps ----
    float sacc[2][4];
#pragma unroll
    for (int j = 0; j < 2; ++j) sacc[j][0] = sacc[j][1] = sacc[j][2] = sacc[j][3] = 0.f;
#pragma unroll
    for (int cbk = 0; cbk < 9; ++cbk) {
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        uint32_t qa[4], kb[4];
        {   // A: Q rows 0-15, dims 64*cbk + 16*ks .. +15 : matrices {r0-7,lo},{r8-15,lo},{r0-7,hi},{r8-15,hi}
          const int row = ((lane >> 3) & 1) * 8 + (lane & 7);
          const int c = ks * 2 + (lane >> 4);
          ldsm_x4(qa, sq_a + sw_off(16, cbk, row, c));
        }
        {   // B: keys 16w..16w+15 : matrices {k0-7,lo},{k0-7,hi},{k8-15,lo},{k8-15,hi}
          const int row = warp * 16 + ((lane >> 4) << 3) + (lane & 7);
          const int c = ks * 2 + ((lane >> 3) & 1);
          ldsm_x4(kb, tile_a + sw_off(kMtTile, cbk, row, c));
        }
        mma16816<__nv_bfloat16>(sacc[0], qa, kb[0], kb[1]);
        mma16816<__nv_bfloat16>(sacc[1], qa, kb[2], kb[3]);
      }
    }
    // ---- scale, mask, row max over this warp's keys, exchange across warps ----
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const bool ok = warp * 16 + j * 8 + 2 * t + e < nvalid;
        sacc[j][e] = ok ? sacc[j][e] * sc : -INFINITY;
        sacc[j][2 + e] = ok ? sacc[j][2 + e] * sc : -INFINITY;
        mx0 = fmaxf(mx0, sacc[j][e]);
        mx1 = fmaxf(mx1, sacc[j][2 + e]);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    if (t == 0) { s_max[warp * 16 + g] = mx0; s_max[warp * 16 + g + 8] = mx1; }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    float tm0 = fmaxf(fmaxf(s_max[g], s_max[16 + g]), fmaxf(s_max[32 + g], s_max[48 + g]));
    float tm1 = fmaxf(fmaxf(s_max[g + 8], s_max[24 + g]), fmaxf(s_max[40 + g], s_max[56 + g]));
    const float mn0 = fmaxf(m0, tm0), mn1 = fmaxf(m1, tm1);          // finite: key0 < end
    const float c0 = exp2f(m0 - mn0), c1 = exp2f(m1 - mn1);
    m0 = mn0; m1 = mn1;
    l0 *= c0; l1 *= c1;
    // ---- P (bf16) -> shared memory [16 rows][64 keys], swizzled ----
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const float p0 = exp2f(sacc[j][0] - mn0), p1 = exp2f(sacc[j][1] - mn0);
      const float p2 = exp2f(sacc[j][2] - mn1), p3 = exp2f(sacc[j][3] - mn1);
      l0 += p0 + p1;
      l1 += p2 + p3;
      const int key = warp * 16 + j * 8 + 2 * t;                       // even -> 4-byte aligned pair
      const __nv_bfloat16* tag = nullptr;
      *reinterpret_cast<uint32_t*>(s_p + sw_off(16, 0, g, key >> 3) + (key & 7) * 2) = pack2(p0, p1, tag);
      *reinterpret_cast<uint32_t*>(s_p + sw_off(16, 0, g + 8, key >> 3) + (key & 7) * 2) = pack2(p2, p3, tag);
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) { o[j][0] *= c0; o[j][1] *= c0; o[j][2] *= c1; o[j][3] *= c1; }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    // ---- O[16 x dims 128w..128w+127] += P[16 x 64] V[64 x 128] ----
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t pa[4];
      {
        const int row = ((lane >> 3) & 1) * 8 + (lane & 7);
        const int c = kk * 2 + (lane >> 4);
        ldsm_x4(pa, sp_a + sw_off(16, 0, row, c));
      }
#pragma unroll
      for (int dp = 0; dp < 8; ++dp) {        // dims 128w + 16dp .. +15 : column block 2w + dp/4
        const int row = kk * 16 + (((lane >> 3) & 1) << 3) + (lane & 7);
        const int c = (dp & 3) * 2 + (lane >> 4);
        uint32_t vb[4];
        ldsm_x4_trans(vb, tile_a + sw_off(kMtTile, warp * 2 + (dp >> 2), row, c));
        mma16816<__nv_bfloat16>(o[dp * 2], pa, vb[0], vb[1]);
        mma16816<__nv_bfloat16>(o[dp * 2 + 1], pa, vb[2], vb[3]);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);      // this warp is done with the stage
  }

  // ---- epilogue: row sums across the quad and the 4 warps, normalise, write ----
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  asm volatile("bar.sync 1, 128;" ::: "memory");
  if (t == 0) { s_sum[warp * 16 + g] = l0; s_sum[warp * 16 + g + 8] = l1; }
  asm volatile("bar.sync 1, 128;" ::: "memory");
  const float lt0 = s_sum[g] + s_sum[16 + g] + s_sum[32 + g] + s_sum[48 + g];
  const float lt1 = s_sum[g + 8] + s_sum[24 + g] + s_sum[40 + g] + s_sum[56 + g];
  const float inv0 = lt0 > 0.f ? 1.f / lt0 : 0.f, inv1 = lt1 > 0.f ? 1.f / lt1 : 0.f;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int row = g + half * 8;
    const int h = h0 + row;
    if (h >= H) continue;
    const float inv = half ? inv1 : inv0;
    if (num_splits == 1) {
      __nv_bfloat16* op = out + ((int64_t)b * H + h) * C + warp * 128;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        __nv_bfloat162 v = __floats2bfloat162_rn(o[j][half * 2] * inv, o[j][half * 2 + 1] * inv);
        *reinterpret_cast<__nv_bfloat162*>(op + j * 8 + 2 * t) = v;
      }
    } else {
      const int64_t pi = ((int64_t)b * H + h) * num_splits + split;
      float* op = o_part + pi * C + warp * 128;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        *reinterpret_cast<float2*>(op + j * 8 + 2 * t) = make_float2(o[j][half * 2] * inv, o[j][half * 2 + 1] * inv);
      if (warp == 0 && t == 0) {
        const float lt = half ? lt1 : lt0, mm = half ? m1 : m0;
        lse[pi] = lt > 0.f ? mm + log2f(lt) : -INFINITY;
      }
    }
  }
}

inline int pick_splits_1cta(int ctas_without_split, int max_len) {
  int want = (132 * 3 + ctas_without_split - 1) / ctas_without_split;
  int by_len = (max_len + 255) / 256;
  int s = want < by_len ? want : by_len;
  if (s > 64) s = 64;
  return s < 1 ? 1 : s;
}

// split count for a kernel with `slots` resident CTAs on the GPU: minimise waves x (keys per split + a fixed
// per-CTA cost worth ~192 keys).  Waves are whole: a CTA streams at its SM's rate however empty the GPU is
// (measured, scripts/gqa_sweep.py: bs=16 128 CTAs x 4096 keys beat every split; bs=1 wants ~one full wave).
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

}  // namespace

extern "C" int64_t chitu_b200_attn_workspace_bytes(int batch, int heads, int head_dim_v, int max_splits) {
  return (int64_t)batch * heads * max_splits * (head_dim_v + 1) * (int64_t)sizeof(float) + 256;
}

static int splits_that_fit(int splits, int B, int H, int DV, int64_t workspace_bytes) {
  while (splits > 1 && chitu_b200_attn_workspace_bytes(B, H, DV, splits) > workspace_bytes) --splits;
  return splits;
}

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
  CB_ARG(q && k_cache && v_cache && cache_seqlens && block_table && out);
  CB_ARG((rope_cos == nullptr) == (rope_sin == nullptr) && q_sb >= (int64_t)Hq * D && q_sb % 2 == 0);
  CB_ARG((k_new == nullptr) == (v_new == nullptr));
  CB_ARG(B >= 0 && Hq > 0 && Hkv > 0 && Hq % Hkv == 0 && page_size > 0 && bt_stride > 0);
  CB_ARG(D == 64 || D == 128);
  CB_ARG(k_new == nullptr || (k_new_sb % 4 == 0 && v_new_sb % 4 == 0));
  CB_ARG(dtype == CB_BF16 || dtype == CB_F16);
  if (B == 0) return 0;
  const int G = Hq / Hkv;
  CB_ARG(G == 1 || G == 2 || G == 4 || G == 8);
  int max_len = max_seqlen_hint > 0 ? max_seqlen_hint : bt_stride * page_size;
  int splits = pick_splits(B * Hkv, max_len, 256, 64);
  splits = workspace ? splits_that_fit(splits, B, Hq, D, workspace_bytes) : 1;
  float* o_part = (float*)workspace;
  float* lse = o_part ? o_part + (int64_t)B * Hq * splits * D : nullptr;
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid(splits, Hkv, B);
  const int impl_simt = getenv("CHITU_B200_GQA_SIMT") ? 1 : 0;   // debugging / A-B profiling switch

  const bool pow2 = (page_size & (page_size - 1)) == 0;
  if (D == 128 && pow2 && impl_simt == 0) {
    int page_shift = 0;
    while ((1 << page_shift) < page_size) ++page_shift;
    // configuration (A/B switch CHITU_B200_GQA_CFG, split override CHITU_B200_GQA_SPLITS):
    //   heads-as-M kernel  0: 4 warps x 3 stages x 32 keys, 1 CTA/SM   1: 8 x 3 x 16, 1 CTA/SM   2: 4 x 3 x 16, 2 CTA/SM
    //   keys-as-M kernel   4: 4 x 3 x 32, 1 CTA/SM   5: 8 x 3 x 16, 1 CTA/SM (default)   6: 4 x 3 x 16, 2 CTA/SM
    //                      7: 6 x 2 x 32, 1 CTA/SM   8: 2 x 3 x 32, 2 CTA/SM
    const char* e_cfg = getenv("CHITU_B200_GQA_CFG");
    const char* e_spl = getenv("CHITU_B200_GQA_SPLITS");
    const int gqa_cfg = e_cfg ? atoi(e_cfg) : 5;
    if (rope_cos && gqa_cfg < 4) return fail(-2, "gqa_paged_decode_rope: the heads-as-M kernel has no fused rotary");
    const int ctas_per_sm = (gqa_cfg == 2 || gqa_cfg == 6 || gqa_cfg == 8) ? 2 : 1;
    splits = e_spl ? atoi(e_spl) : pick_splits_waves(B * Hkv, max_len, 132 * ctas_per_sm);
    if (splits < 1) splits = 1;
    splits = workspace ? splits_that_fit(splits, B, Hq, D, workspace_bytes) : 1;
    lse = o_part ? o_part + (int64_t)B * Hq * splits * D : nullptr;
    grid = dim3(splits, Hkv, B);
#define LAUNCH_MMA_CFG(KERNEL, T, GG, TILE, STAGES, WARPS, CTAS)                                               \
  do {                                                                                                 \
    const size_t smem = (size_t)WARPS * STAGES * 2 * (TILE * kGqaD * 2);                               \
    static bool attr = false;                                                                          \
    if (!attr) {                                                                                       \
      CB_CUDA(cudaFuncSetAttribute(KERNEL<T, GG, TILE, STAGES, WARPS, CTAS>,                           \
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));           \
      attr = true;                                                                                     \
    }                                                                                                  \
    cb::launch_k(KERNEL<T, GG, TILE, STAGES, WARPS, CTAS>, dim3(grid), dim3(WARPS * 32), smem, st,      \
        (const T*)q, (T*)k_cache, (T*)v_cache, (const T*)k_new, (const T*)v_new, k_new_sb, v_new_sb,   \
        cache_seqlens, block_table, bt_stride, Hq, Hkv, page_shift, softmax_scale, splits, o_part, lse, \
        (T*)out, q_sb, rope_cos, rope_sin);                                                            \
  } while (0)
#define LAUNCH_MMA(T, GG)                                                                   \
  do {                                                                                      \
    switch (gqa_cfg) {                                                                      \
      case 0: LAUNCH_MMA_CFG(gqa_decode_mma_kernel, T, GG, 32, 3, 4, 1); break;             \
      case 1: LAUNCH_MMA_CFG(gqa_decode_mma_kernel, T, GG, 16, 3, 8, 1); break;             \
      case 2: LAUNCH_MMA_CFG(gqa_decode_mma_kernel, T, GG, 16, 3, 4, 2); break;             \
      case 4: LAUNCH_MMA_CFG(gqa_decode_mmaT_kernel, T, GG, 32, 3, 4, 1); break;            \
      case 5: LAUNCH_MMA_CFG(gqa_decode_mmaT_kernel, T, GG, 16, 3, 8, 1); break;            \
      case 6: LAUNCH_MMA_CFG(gqa_decode_mmaT_kernel, T, GG, 16, 3, 4, 2); break;            \
      case 7: LAUNCH_MMA_CFG(gqa_decode_mmaT_kernel, T, GG, 32, 2, 6, 1); break;            \
      case 8: LAUNCH_MMA_CFG(gqa_decode_mmaT_kernel, T, GG, 32, 3, 2, 2); break;            \
      default: LAUNCH_MMA_CFG(gqa_decode_mmaT_kernel, T, GG, 16, 3, 8, 1); break;           \
    }                                                                                       \
  } while (0)
#define DISPATCH_MMA(T)                 \
  switch (G) {                          \
    case 1: LAUNCH_MMA(T, 1); break;    \
    case 2: LAUNCH_MMA(T, 2); break;    \
    case 4: LAUNCH_MMA(T, 4); break;    \
    default: LAUNCH_MMA(T, 8); break;   \
  }
    if (dtype == CB_BF16) { DISPATCH_MMA(__nv_bfloat16); } else { DISPATCH_MMA(__half); }
#undef DISPATCH_MMA
#undef LAUNCH_MMA
#undef LAUNCH_MMA_CFG
  } else {
    if (rope_cos || q_sb != (int64_t)Hq * D)
      return fail(-2, "gqa_paged_decode_rope: fused rotary / strided q need head_dim 128 and a power-of-two page");
#define LAUNCH_GQA(T, DD, GG)                                                                       \
  cb::launch_k(gqa_decode_kernel<T, DD, GG>, dim3(grid), dim3(128), 0, st,                                                \
      (const T*)q, (T*)k_cache, (T*)v_cache, (const T*)k_new, (const T*)v_new, k_new_sb, v_new_sb,  \
      cache_seqlens,                                                                                \
      block_table, bt_stride, Hq, Hkv, page_size, softmax_scale, splits, o_part, lse, (T*)out)
#define DISPATCH_G(T, DD)                         \
  switch (G) {                                    \
    case 1: LAUNCH_GQA(T, DD, 1); break;          \
    case 2: LAUNCH_GQA(T, DD, 2); break;          \
    case 4: LAUNCH_GQA(T, DD, 4); break;          \
    default: LAUNCH_GQA(T, DD, 8); break;         \
  }
    if (dtype == CB_BF16) {
      if (D == 128) { DISPATCH_G(__nv_bfloat16, 128) } else { DISPATCH_G(__nv_bfloat16, 64) }
    } else {
      if (D == 128) { DISPATCH_G(__half, 128) } else { DISPATCH_G(__half, 64) }
    }
#undef DISPATCH_G
#undef LAUNCH_GQA
  }
  CB_LAUNCHED(1);
  if (splits > 1) {
    if (dtype == CB_BF16) {
      if (D == 128) cb::launch_k(merge_splits_kernel<__nv_bfloat16, 128>, dim3(B * Hq), dim3(128), 0, st, o_part, lse, (__nv_bfloat16*)out, splits);
      else cb::launch_k(merge_splits_kernel<__nv_bfloat16, 64>, dim3(B * Hq), dim3(64), 0, st, o_part, lse, (__nv_bfloat16*)out, splits);
    } else {
      if (D == 128) cb::launch_k(merge_splits_kernel<__half, 128>, dim3(B * Hq), dim3(128), 0, st, o_part, lse, (__half*)out, splits);
      else cb::launch_k(merge_splits_kernel<__half, 64>, dim3(B * Hq), dim3(64), 0, st, o_part, lse, (__half*)out, splits);
    }
    CB_LAUNCHED(1);
  }
  return 0;
}

namespace cb {
int mla_decode_tc_launch(const void* q_nope, const void* q_pe, void* kv_cache, const void* new_kv,
                         const int32_t* seqlens_excl, const int32_t* block_table, int bt_stride, int B, int H,
                         int num_blocks, int num_splits, float scale, void* out, float* o_part, float* lse,
                         const int32_t* plan, cudaStream_t st);
// KV splits of the wgmma MLA kernel (1 CTA per SM): one wave of CTAs, whole pages, at least two pages per split, and
// the partials must fit the workspace.  Deterministic in its arguments: the merging absorb-o kernel recomputes it.
int mla_tc_num_splits(int B, int H, int max_len, int64_t workspace_bytes) {
  const int hgroups = cdiv(H, 16);
  int want = 132 / (B * hgroups);
  const int pages = cdiv(max_len, 64);
  int by_len = pages / 2;
  int splits = want < by_len ? want : by_len;
  if (splits > 128) splits = 128;
  if (splits < 1) splits = 1;
  if (workspace_bytes <= 0) return 1;
  while (splits > 1 && chitu_b200_attn_workspace_bytes(B, H, 512, splits) > workspace_bytes) --splits;
  return splits;
}
}  // namespace cb

extern "C" int chitu_b200_mla_num_splits(int B, int H, int max_seqlen_hint, int64_t workspace_bytes) {
  return cb::mla_tc_num_splits(B, H, max_seqlen_hint, workspace_bytes);
}

extern "C" int chitu_b200_mla_decode(const void* q_nope, const void* q_pe, void* kv_cache,
                                     const void* new_kv, const int32_t* seqlens_excl,
                                     const int32_t* block_table, int bt_stride, int B, int H, int C, int R,
                                     int page_size, int num_blocks, int max_seqlen_hint, float softmax_scale, void* out,
                                     void* workspace, int64_t workspace_bytes, void* stream) {
  CB_ARG(q_nope && q_pe && kv_cache && seqlens_excl && block_table);
  CB_ARG(B >= 0 && H > 0 && page_size > 0 && bt_stride > 0 && num_blocks > 0);
  if (C != kMlaC || R != kMlaR)
    return fail(-1, "mla_decode: only kv_lora_rank=512, qk_rope_head_dim=64 is built (got %d,%d)", C, R);
  if (B == 0) return 0;
  const int hgroups = cdiv(H, 16);
  int max_len = max_seqlen_hint > 0 ? max_seqlen_hint : bt_stride * page_size;
  cudaStream_t st = (cudaStream_t)stream;
  // implementation (A/B switch CHITU_B200_MLA_IMPL): 0 / unset = wgmma kernel (mla_tc.cu), 1 = mma.sync kernel,
  // 2 = SIMT kernel; pages other than 64 tokens only run on the SIMT kernel
  static const int impl_env = getenv("CHITU_B200_MLA_IMPL") ? atoi(getenv("CHITU_B200_MLA_IMPL"))
                                                            : (getenv("CHITU_B200_MLA_SIMT") ? 2 : 0);
  const bool tma_ok = page_size == kMtTile && cb::tma_available();
  const bool use_tc = tma_ok && impl_env == 0;
  const bool use_mma = tma_ok && impl_env == 1;
  if (use_tc) {
    const int splits = cb::mla_tc_num_splits(B, H, max_len, workspace ? workspace_bytes : 0);
    float* o_part = (float*)workspace;
    float* lse = o_part ? o_part + (int64_t)B * H * splits * kMlaC : nullptr;
    // a split plan written by chitu_b200_attn_plan for this step (last 256 bytes of the workspace) overrides the
    // hint-derived keys per split: ragged batches get splits of equal size instead of equal count
    const int32_t* plan = workspace ? (const int32_t*)((const uint8_t*)workspace + workspace_bytes - 256) : nullptr;
    int rc = cb::mla_decode_tc_launch(q_nope, q_pe, kv_cache, new_kv, seqlens_excl, block_table, bt_stride, B, H, num_blocks,
                                      splits, softmax_scale, out, o_part, lse, plan, st);
    if (rc) return rc;
    if (splits > 1 && out) {        // out == NULL: the caller merges (chitu_b200_mla_absorb_o_merge_quant)
      cb::launch_k(merge_splits_kernel<__nv_bfloat16, kMlaC>, dim3(B * H), dim3(256), 0, st, o_part, lse, (__nv_bfloat16*)out, splits);
      CB_LAUNCHED(1);
    }
    return 0;
  }
  if (!out) return fail(-1, "mla_decode: out == NULL (deferred merge) needs the wgmma kernel (page 64, TMA)");
  int splits;
  float *o_part, *lse;
  if (use_mma) {
    // one CTA per SM (2 x 72 KB page stages): ~2 CTAs per SM in total, whole pages per split
    int want = (132 * 2 + B * hgroups - 1) / (B * hgroups);
    // at least 4 pages per CTA: a one-page split has no pipeline and makes the merge a long chain of
    // dependent L2 round trips (65 splits at bs=1 cost 14 us in the merge alone)
    int by_len = (max_len + 4 * kMtTile - 1) / (4 * kMtTile);
    splits = want < by_len ? want : by_len;
    if (splits > 128) splits = 128;
    if (splits < 1) splits = 1;
    splits = workspace ? splits_that_fit(splits, B, H, kMlaC, workspace_bytes) : 1;
    o_part = (float*)workspace;
    lse = o_part ? o_part + (int64_t)B * H * splits * kMlaC : nullptr;
    CUtensorMap map;
    // the cache as a 2-D [num_rows, 576] bf16 tensor; rows beyond the allocation are never addressed
    const int64_t rows = (int64_t)num_blocks * page_size;
    int rc = cb::make_tma_map_2d(&map, kv_cache, rows, kMlaRow, 2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, kMtTile);
    if (rc) return rc;
    const size_t smem = 1024 + kMtStages * kMtStageBytes + kMtQBytes + kMtPBytes + 512;
    static bool attr = false;
    if (!attr) {
      CB_CUDA(cudaFuncSetAttribute(mla_decode_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      attr = true;
    }
    dim3 grid(splits, hgroups, B);
    cb::launch_k(mla_decode_mma_kernel, grid, dim3(160), smem, st, map, (const __nv_bfloat16*)q_nope,
                 (const __nv_bfloat16*)q_pe, (__nv_bfloat16*)kv_cache, (const __nv_bfloat16*)new_kv, seqlens_excl,
                 block_table, bt_stride, H, softmax_scale, splits, o_part, lse, (__nv_bfloat16*)out);
  } else {
    splits = pick_splits(B * hgroups, max_len, 64, 128);
    splits = workspace ? splits_that_fit(splits, B, H, kMlaC, workspace_bytes) : 1;
    o_part = (float*)workspace;
    lse = o_part ? o_part + (int64_t)B * H * splits * kMlaC : nullptr;
    dim3 grid(splits, hgroups, B);
    cb::launch_k(mla_decode_kernel, dim3(grid), dim3(128), 0, st, (const __nv_bfloat16*)q_nope, (const __nv_bfloat16*)q_pe,
                 (__nv_bfloat16*)kv_cache, (const __nv_bfloat16*)new_kv, seqlens_excl, block_table, bt_stride, H,
                 page_size, softmax_scale, splits, o_part, lse, (__nv_bfloat16*)out);
  }
  CB_LAUNCHED(1);
  if (splits > 1) {
    cb::launch_k(merge_splits_kernel<__nv_bfloat16, kMlaC>, dim3(B * H), dim3(256), 0, st, o_part, lse, (__nv_bfloat16*)out, splits);
    CB_LAUNCHED(1);
  }
  return 0;
}


// ============================================================================================
// MLA weight absorption (the two torch.einsum of AttentionDeepSeekV3, model_deepseek_v3.py:529-531
// and :697; SURVEY K8): wkv_b (bf16, [H, dn + dv, C]) is W_UK = [:, :dn] and W_UV = [:, dn:].
//   absorb_q : q'[b,h,c] = sum_d q_nope[b,h,d] * W_UK[h,d,c]        ("shd,hdc->shc")
//   absorb_o : o[b,h,d]  = sum_c x[b,h,c]     * W_UV[h,d,c]        ("bshc,hdc->bshd")
// Both stream the 2 MB of per-rank absorbed weights once for all tokens (fp32 accumulate).
// ============================================================================================
// CTA = (64-column chunk of C, head): 8 warps split the dn reduction dim (16 d each), a lane owns two
// adjacent columns; partial sums are combined through shared memory.  W_UK is read once (2 MB per rank).
template <int MT>
__global__ void __launch_bounds__(256) mla_absorb_q_kernel(const __nv_bfloat16* __restrict__ q, int64_t q_sb,
                                                          int64_t q_sh, const __nv_bfloat16* __restrict__ w,
                                                          __nv_bfloat16* __restrict__ out, int B, int H, int dn,
                                                          int dv, int C) {
  cb::pdl_prologue();
  extern __shared__ float s_abs[];               // [MT][dn] q  |  [8 warps][MT][64] partial sums
  float* s_q = s_abs;
  float* s_red = s_abs + MT * dn;
  const int h = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = blockIdx.x * 64 + lane * 2;
  const int b0 = blockIdx.z * MT;
  for (int i = threadIdx.x; i < MT * dn; i += 256) {
    const int m = i / dn, d = i - m * dn;
    s_q[i] = (b0 + m < B) ? __bfloat162float(q[(int64_t)(b0 + m) * q_sb + (int64_t)h * q_sh + d]) : 0.f;
  }
  __syncthreads();
  float acc0[MT], acc1[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) acc0[m] = acc1[m] = 0.f;
  const int dper = dn / 8;                        // d slice of this warp
  const __nv_bfloat16* wp = w + ((int64_t)h * (dn + dv) + warp * dper) * C + c;
  if (c < C) {
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
    if (b0 + m < B && blockIdx.x * 64 + cc < C)
      out[((int64_t)(b0 + m) * H + h) * C + blockIdx.x * 64 + cc] = __float2bfloat16_rn(v);
  }
}

// CTA = (head, token chunk): warp w computes output dims [w*dv/8, (w+1)*dv/8) (one W_UV row at a time,
// lanes stride C); with dv == 128 the head's 128 outputs are exactly one act_quant group, so the fp8
// payload + scale of the following `wo` linear can be produced here (q_out != null).
// With `o_part` != null the latent input is the split-KV partials of the attention kernel and the LSE-weighted merge
// (merge_splits_kernel's arithmetic: same weights, same fmaf order, one bf16 rounding) happens while staging: the merge
// launch and its [B,H,C] round trip disappear.
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
  __shared__ float s_mw[MT][128];                               // normalised split weights (num_splits <= 128)
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
      const float* l = lse + ((int64_t)b * H + h) * num_splits;
      float mx = -INFINITY;
      for (int sp = lane; sp < num_splits; sp += 32) mx = fmaxf(mx, l[sp]);
      mx = warp_max(mx);
      float den = 0.f;
      for (int sp = lane; sp < num_splits; sp += 32) {
        const float ls = l[sp];
        const float wv = ls == -INFINITY ? 0.f : exp2f(ls - mx);
        s_mw[m][sp] = wv;
        den += wv;
      }
      den = warp_sum(den);
      const float inv = den > 0.f ? 1.f / den : 0.f;
      for (int sp = lane; sp < num_splits; sp += 32) s_mw[m][sp] *= inv;
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
        float amax = fmaxf(fmaxf(fabsf(v[0]), fabsf(v[1])), fmaxf(fabsf(v[2]), fabsf(v[3])));
        amax = warp_max(amax);
        const float sc = __fdiv_rn(amax, 448.0f);
        uint32_t packed = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) packed |= (uint32_t)float_to_fp8(__fdiv_rn(v[i], sc)) << (8 * i);
        *reinterpret_cast<uint32_t*>(q_out + o) = packed;
        if (lane == 0) q_scales[((int64_t)(b0 + m) * H + h) * (dv / 128) + d0 / 128] = sc;
      }
    }
  }
}

extern "C" int chitu_b200_mla_absorb_q(const void* q_nope, int64_t q_sb, int64_t q_sh, const void* wkv_b,
                                       void* out, int B, int H, int dn, int dv, int C, void* stream) {
  CB_ARG(q_nope && wkv_b && out && B >= 0 && H > 0 && dn > 0 && dv > 0 && C > 0 && C % 2 == 0);
  if (B == 0) return 0;
  constexpr int MT = 16;
  CB_ARG(dn % 8 == 0);
  dim3 grid(cdiv(C, 64), H, cdiv(B, MT));
  cb::launch_k(mla_absorb_q_kernel<MT>, grid, dim3(256), (size_t)(MT * dn + 8 * MT * 64) * 4, (cudaStream_t)stream,
               (const __nv_bfloat16*)q_nope, q_sb, q_sh, (const __nv_bfloat16*)wkv_b, (__nv_bfloat16*)out, B, H, dn, dv, C);
  CB_LAUNCHED(1);
  return 0;
}

extern "C" int chitu_b200_mla_absorb_o(const void* x, const void* wkv_b, void* out, int B, int H, int dn, int dv,
                                       int C, void* stream) {
  return chitu_b200_mla_absorb_o_quant(x, wkv_b, out, nullptr, nullptr, B, H, dn, dv, C, stream);
}

extern "C" int chitu_b200_mla_absorb_o_quant(const void* x, const void* wkv_b, void* out, void* q_out,
                                             float* q_scales, int B, int H, int dn, int dv, int C, void* stream) {
  CB_ARG(x && wkv_b && (out || q_out) && B >= 0 && H > 0 && dn > 0 && dv > 0 && C > 0 && C % 8 == 0);
  CB_ARG(dv == 128 && (q_out == nullptr) == (q_scales == nullptr));
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
  if (B == 0) return 0;
  const int splits = cb::mla_tc_num_splits(B, H, max_seqlen_hint, workspace_bytes);
  CB_ARG(splits <= 128);
  const float* o_part = (const float*)workspace;
  const float* lse = o_part + (int64_t)B * H * splits * kMlaC;
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
    // ---- absorb_q role: CTA = (64-column chunk, head, token chunk) ----
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
