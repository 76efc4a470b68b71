// Absorbed-MLA prefill attention on the Hopper tensor cores (sm_90a): wgmma + TMA + mbarrier.
//
// Replaces the flash_attn / SDPA delegation of AttnBackend.attn_varlen_func (FlashAttnBackend, attn_backend.py:193-206)
// for the call DeepSeek's prefill makes (model_deepseek_v3.py:588-602): absorbed MLA in MQA form,
//   q [Tq, H, 576] = [q_nope . W_uk | q_pe],  k [Tk, 1, 576] = [kv_norm(kv) | k_pe],  v [Tk, 1, 512] = kv_norm(kv),
// ragged batch by cu_seqlens_q / cu_seqlens_k, flash_attn_varlen_func semantics: fp32 scores and softmax, P rounded to
// bf16 before P.V, causal mask aligned bottom-right (query i sees keys j <= i + Lk - Lq), rows that see no key are 0.
//
// Mapping: q is flattened to [Tq * H, 576] rows, token-major (row r of a sequence is token r / H, head r % H), and one
// CTA owns 64 rows of one sequence.  Both products are SWAPPED, as in the decode kernel (mla_tc.cu), so the 64 rows are
// the wgmma N dimension:
//   S^T[64 keys x 64 rows]  = K[64 x 576] . Q^T           A = staged K chunk (K-major), B = staged Q chunk
//   O^T[512 dims x 64 rows] += V^T[512 x 64] . P^T         A = staged V chunks read MN-major, B = P[64 rows x 64 keys]
// O^T is 128 fp32 registers per thread for 256 dims, so the dims are split over two warpgroups (256 threads):
//   WG0 (warps 0-3)  S^T, the online softmax (fp32, log2 domain), P -> shared memory, O^T for dims 0..255
//   WG1 (warps 4-7)  O^T for dims 256..511: waits for P of the tile, applies WG0's rescale factors, P.V
// There is no producer warp: with a third warpgroup the launch bound caps every thread at 168 registers, which spills
// WG0 (O^T + S^T + row sums).  Instead each TMA load is issued by the warpgroup that frees its slot, one tile ahead:
//   K chunks of tile i+1   by WG1 once P(i) is published (WG0 has finished S(i), so the K slots are free)
//   V chunks 0-3 / 4-7     by WG0 / WG1 right after their own P.V of tile i
// so K(i+1) streams in during softmax(i) and P.V(i), and V(i+1) during S(i+1).
// Shared memory: 17 x 8 KB chunk slots (one 64-key tile: 9 K + 8 V boxes [64 rows x 128 B]) + Q 72 KB + P 8 KB
// = 216 KB + 1 KB alignment.  The Q tile is reused at the end to stage the bf16 output for 16-byte coalesced stores.
// Scheduling: a 1-D grid of (row tile, sequence) with the LAST row tiles first: under the causal mask they see the most
// keys, so the long CTAs start in the first wave and the short ones fill in behind them.
// Deterministic: every key of a row is reduced by one CTA in a fixed order (no split over keys).
//
// Paged variant (mla_paged_prefill_kernel, behind AttnBackend.mla_attn_with_kvcache with seqlen_q = sq > 1:
// multi-token-prediction verification, chunked prefill on a cached prefix): the same CTA over the paged latent cache
// [num_blocks * 64, 576].  Request b's sq * H rows are row tiles as above (Lq = sq, Lk = seqlens_excl[b] (+ sq)); key
// tile t is page block_table[b, t], K and V boxes come from the one cache map.  The paged append (core.cu) writes the
// new rows first (PDL orders the two).  In the tile holding Lk the V rows >= Lk (unwritten slots, maybe NaN) are zeroed
// in shared memory before P.V.  When row tiles x B CTAs cannot fill the GPU the keys are split; each split writes normalised fp32
// partials + LSE (splitkv.cuh, rows = B * sq * H, staged through the ring) and launch_merge_splits merges them.  The
// split count depends on host values only, so this variant is deterministic too.
#include <cuda.h>
#include <limits.h>

#include "common.cuh"
#include "splitkv.cuh"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace cb {
namespace {

constexpr int kC = 512, kR = 64, kRow = kC + kR;
constexpr int kTile = 64;                      // keys per tile
constexpr int kRows = 64;                      // query rows (token, head) per CTA
constexpr int kSlot = 64 * 128;                // 8 KB: one TMA box [64 rows x 128 B]
constexpr int kKC = kRow / 64, kVC = kC / 64;  // 9 K chunks, 8 V chunks per key tile
constexpr int kTC = kKC + kVC;                 // chunk c of every tile lives in slot c
constexpr int kQBytes = kKC * kSlot;           // Q as 9 K-major chunks [64 rows x 128 B]
constexpr int kPBytes = kRows * 128;           // P as [64 rows x 64 keys] bf16, K-major
constexpr int kSmemBytes = kTC * kSlot + kQBytes + kPBytes;
constexpr int kOutPitch = kC * 2 + 16;         // staged output row in bytes (padded: the 4 rows a store touches differ in bank)
static_assert(kRows * kOutPitch <= kQBytes, "the output tile is staged in the Q buffer");
constexpr int kPartPitch = kC + 4;             // staged fp32 split-partial row in floats (a warp's stores differ in bank)
static_assert(kRows * kPartPitch * 4 <= kTC * kSlot, "the fp32 partial tile is staged in the ring");
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kRescaleThreshold = 8.f;       // log2 domain
constexpr int kThreads = 256;

// one 64-key tile's chunks [c_begin, c_end) into their slots (issued by one thread).  e4m3: each chunk is a 4 KB box
// [64 rows x 64 B] that lands in the upper half of its slot, where expand_e4m3 finds it.
template <bool kFp8 = false>
__device__ __forceinline__ void load_chunks(const CUtensorMap* mk, const CUtensorMap* mv, uint8_t* s_ring, uint64_t* full,
                                            int c_begin, int c_end, int row, uint64_t pol) {
  constexpr int kLand = kFp8 ? kSlot / 2 : 0;
  for (int c = c_begin; c < c_end; ++c) {
    mbar_expect_tx(&full[c], kSlot - kLand);
    if (c < kKC) tma_load_2d(s_ring + c * kSlot + kLand, mk, &full[c], c * 64, row, pol);
    else tma_load_2d(s_ring + c * kSlot + kLand, mv, &full[c], (c - kKC) * 64, row, pol);
  }
}

// e4m3: the box in the upper half of `slot` expanded in place into the swizzled bf16 chunk [64 rows x 128 B] by one
// warpgroup (t: thread in it, named barrier kBar), exact; rows >= zero_from are written as 0.  Thread t expands 16
// bytes (row r, elements 16 u .. 16 u + 15) into bf16 units 2u, 2u + 1 of row r.  Every thread reads its 32 bytes
// before the barrier and writes after it: the chunk's upper half is the box.  The caller fences and syncs before the
// wgmma reads the chunk.
template <int kBar>
__device__ __forceinline__ void expand_e4m3(uint8_t* slot, int t, int zero_from) {
  uint4 x[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) x[j] = *reinterpret_cast<const uint4*>(slot + kSlot / 2 + (j * 128 + t) * 16);
  asm volatile("bar.sync %0, 128;" ::"n"(kBar) : "memory");
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int task = j * 128 + t, r = task >> 2, u = task & 3;
    if (r >= zero_from) x[j] = make_uint4(0, 0, 0, 0);
    uint4 y0, y1;
    E4m3<__nv_bfloat16>::to_io(x[j].x, y0.x, y0.y);
    E4m3<__nv_bfloat16>::to_io(x[j].y, y0.z, y0.w);
    E4m3<__nv_bfloat16>::to_io(x[j].z, y1.x, y1.y);
    E4m3<__nv_bfloat16>::to_io(x[j].w, y1.z, y1.w);
    *reinterpret_cast<uint4*>(slot + sw128(r, 2 * u)) = y0;
    *reinterpret_cast<uint4*>(slot + sw128(r, 2 * u + 1)) = y1;
  }
}

// One CTA of either variant.  Contiguous (kPaged = false): sequence b's rows and keys start at cu_q[b] / cu_k[b], map_q
// holds q as [Tq * H, 576].  Paged: request b has sq query tokens at q row b * sq * H (map_q = q_nope [., 512], map_qpe
// = q_pe [., 64]), Lk = seqlens_excl[b] (+ sq when appended) keys, key tile t is cache page block_table[b, t], and the
// CTA takes split `split` of its key tiles.  KV: the paged cache's element type, bf16 or e4m3 (the chunks are expanded
// to bf16 in place, so the MMA code is the same).
template <bool kPaged, typename KV = __nv_bfloat16>
__device__ __forceinline__ void mla_prefill_cta(
    const CUtensorMap* map_q, const CUtensorMap* map_qpe, const CUtensorMap* map_k, const CUtensorMap* map_v,
    const int32_t* __restrict__ cu_q, const int32_t* __restrict__ cu_k, const int32_t* __restrict__ seqlens_excl,
    const int32_t* __restrict__ block_table, int bt_stride, int sq, int appended, int splits, int B, int H,
    int row_tiles, int causal, float scale, float* __restrict__ o_part, float* __restrict__ lse,
    __nv_bfloat16* __restrict__ out) {
  constexpr bool kFp8 = std::is_same_v<KV, __nv_fp8_e4m3>;
  static_assert(kPaged || !kFp8, "the e4m3 cache is paged");
  extern __shared__ __align__(1024) uint8_t mla_prefill_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(mla_prefill_smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_ring = smem;                                   // [kTC][64 rows][128 B]  K / V chunks of one tile
  uint8_t* s_q = s_ring + kTC * kSlot;                      // [9][64 rows][128 B]; output staging at the end
  uint8_t* s_p = s_q + kQBytes;                             // [64 rows][128 B]
  __shared__ __align__(8) uint64_t full_b[kTC], q_bar, p_full, p_empty;
  __shared__ float red[4][kRows];                           // per-warp row partials: tile max, then the final row sum
  __shared__ float s_m[kRows];                              // running row max (log2 domain)
  __shared__ float s_alpha[kRows];                          // O rescale factor of the tile whose P is in s_p
  __shared__ float s_inv[kRows];                            // 1 / row sum (0 for a row that sees no key)

  const int b = blockIdx.x % B;
  int tile, split = 0;
  if constexpr (kPaged) {
    split = blockIdx.x / B % splits;
    tile = row_tiles - 1 - blockIdx.x / B / splits;
  } else {
    tile = row_tiles - 1 - blockIdx.x / B;                  // last row tiles (most causal work) first
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool wg0 = __shfl_sync(0xffffffffu, threadIdx.x / 128, 0) == 0;   // warp-uniform for the compiler (wgmma paths)

  cb::pdl_prologue();                                       // q, k, v and the lengths are written by earlier kernels
  int q0, Lq, k0 = 0, Lk;                                   // q0: first query token of the sequence
  if constexpr (kPaged) {
    q0 = b * sq;
    Lq = sq;
    Lk = seqlens_excl[b] + (appended ? sq : 0);
  } else {
    q0 = cu_q[b];
    Lq = cu_q[b + 1] - q0;
    k0 = cu_k[b];
    Lk = cu_k[b + 1] - k0;
  }
  const int nrows = Lq * H;
  const int r0 = tile * kRows;
  if (r0 >= nrows) return;                                  // uniform over the CTA
  const int rlast = min(r0 + kRows, nrows) - 1;
  // keys visible to row r (token r / H) are [0, lim(r)); lim is non-decreasing in r
  auto lim = [&](int r) { return causal ? max(0, min(Lk, r / H + 1 + Lk - Lq)) : max(Lk, 0); };
  const int nkeys = lim(rlast);
  const int all_see = lim(r0);                              // keys below this are visible to every row of the tile
  const int ntiles = (nkeys + kTile - 1) / kTile;
  int t_begin = 0, t_end = ntiles;                          // this CTA's key tiles
  if constexpr (kPaged) {
    const int per_split = (ntiles + splits - 1) / splits;
    t_begin = min(ntiles, split * per_split);
    t_end = min(ntiles, t_begin + per_split);
  }
  // paged: first cache row of key tile t (read by the thread that issues the tile's loads)
  auto page_row = [&](int t) { return block_table[(int64_t)b * bt_stride + t] * kTile; };
  const uint64_t pol_kv = l2_policy_evict_last();           // K / V are re-read by every row tile of the sequence

  if (threadIdx.x == 0) {
    for (int i = 0; i < kTC; ++i) mbar_init(&full_b[i], 1);
    mbar_init(&q_bar, 1);
    mbar_init(&p_full, 1);
    mbar_init(&p_empty, 4);                                 // one arrival per WG1 warp
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    if (t_end > t_begin) {
      mbar_expect_tx(&q_bar, kQBytes);
      if constexpr (kPaged) {
        for (int c = 0; c < kVC; ++c) tma_load_2d(s_q + c * kSlot, map_q, &q_bar, c * 64, q0 * H + r0, l2_policy_evict_first());
        tma_load_2d(s_q + kVC * kSlot, map_qpe, &q_bar, 0, q0 * H + r0, l2_policy_evict_first());
      } else {
        for (int c = 0; c < kKC; ++c) tma_load_2d(s_q + c * kSlot, map_q, &q_bar, c * 64, q0 * H + r0, l2_policy_evict_first());
      }
      load_chunks<kFp8>(map_k, map_v, s_ring, full_b, 0, kTC, kPaged ? page_row(t_begin) : k0, pol_kv);
    }
  }
  if (threadIdx.x < kRows) s_m[threadIdx.x] = -INFINITY;
  __syncthreads();

  const int krow = (warp & 3) * 16 + (lane >> 2);           // fragment rows krow, krow + 8: keys of S^T, dims of O^T
  const int qd = 2 * (lane & 3);                            // fragment columns 8 nb + qd + j: query rows of the tile
  const uint32_t ring_a = smem_u32(s_ring), q_a = smem_u32(s_q), p_a = smem_u32(s_p);
  const int vc0 = wg0 ? 0 : 4;                              // this warpgroup's V chunks (64 dims each)
  float o[4][32];                                           // O^T tile m: dims 64 (vc0 + m) + krow (+8), rows as S^T
#pragma unroll
  for (int m = 0; m < 4; ++m)
#pragma unroll
    for (int e = 0; e < 32; ++e) o[m][e] = 0.f;
  float l_part[16];                                         // WG0: this thread's share of the row sums, x = 2 nb + j
#pragma unroll
  for (int x = 0; x < 16; ++x) l_part[x] = 0.f;

  if (wg0 && t_end > t_begin) mbar_wait(&q_bar, 0);
  const float sc = scale * kLog2e;
  for (int it = 0; it < t_end - t_begin; ++it) {
    const uint32_t ph = it & 1;                             // phase of every chunk slot for tile it
    const bool more = t_begin + it + 1 < t_end;
    const int key0 = (t_begin + it) * kTile;
    // contiguous: rows past the sequence are masked; past the tensor, zero
    const int next_row = kPaged ? 0 : k0 + (it + 1) * kTile;
    if (wg0) {
      // ---- S^T = K . Q^T over the 9 chunks of 64 dims ----
      if constexpr (kFp8) {                                 // K rows past Lk keep their bytes: masked below
        for (int c = 0; c < kKC; ++c) {
          mbar_wait(&full_b[c], ph);
          expand_e4m3<1>(s_ring + c * kSlot, threadIdx.x, kTile);
        }
        fence_async_smem();
        asm volatile("bar.sync 1, 128;" ::: "memory");
      }
      float s[32];
#pragma unroll
      for (int e = 0; e < 32; ++e) s[e] = 0.f;
      wgmma_fence();
      for (int c = 0; c < kKC; ++c) {
        mbar_wait(&full_b[c], ph);
#pragma unroll
        for (int k = 0; k < 4; ++k)
          WgmmaN<64>::bf16<0>(s, make_sw128_desc(ring_a + c * kSlot + 32 * k, 16, 1024),
                              make_sw128_desc(q_a + c * kSlot + 32 * k, 16, 1024), (c | k) != 0);
      }
      wgmma_commit();
      wgmma_wait<0>();

      // ---- scale, mask (only tiles that reach past some row's last visible key), per-row tile max ----
      if (key0 + kTile > all_see) {
#pragma unroll
        for (int x = 0; x < 16; ++x) {
          const int lr = lim(r0 + 8 * (x >> 1) + qd + (x & 1));
          const int e = 4 * (x >> 1) + (x & 1);
          s[e] = key0 + krow < lr ? s[e] * sc : -INFINITY;
          s[e + 2] = key0 + krow + 8 < lr ? s[e + 2] * sc : -INFINITY;
        }
      } else {
#pragma unroll
        for (int e = 0; e < 32; ++e) s[e] *= sc;
      }
#pragma unroll
      for (int x = 0; x < 16; ++x) {
        const int e = 4 * (x >> 1) + (x & 1);
        const float mx = rows_max(fmaxf(s[e], s[e + 2]));
        if (lane < 4) red[warp][8 * (x >> 1) + qd + (x & 1)] = mx;
      }
      mbar_wait(&p_empty, ph ^ 1);                          // WG1 is done with P / alpha of tile it - 1
      asm volatile("bar.sync 1, 128;" ::: "memory");
      // ---- running max: moved only when a row's max grew by more than 2^8 (exact result: P, l, O share it) ----
      if (threadIdx.x < kRows) {
        const int r = threadIdx.x;
        const float mt = fmaxf(fmaxf(red[0][r], red[1][r]), fmaxf(red[2][r], red[3][r]));
        const float mo = s_m[r];
        float a = 1.f;
        if (mt > mo + kRescaleThreshold) {                  // also the first finite max (mo = -inf): a = 0
          a = exp2f(mo - mt);
          s_m[r] = mt;
        }
        s_alpha[r] = a;
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");
      // ---- P = exp2(S - m) -> bf16 -> shared memory as P[row][key] (K-major, swizzled) ----
      bool need = false;
#pragma unroll
      for (int x = 0; x < 16; ++x) {
        const int r = 8 * (x >> 1) + qd + (x & 1);
        const float m = s_m[r];
        const float mr = m == -INFINITY ? 0.f : m;          // a row with no visible key so far: P = 0
        const float a = s_alpha[r];
        need |= a != 1.f;
        const int e = 4 * (x >> 1) + (x & 1);
        const float p0 = exp2f(s[e] - mr), p1 = exp2f(s[e + 2] - mr);
        l_part[x] = l_part[x] * a + p0 + p1;
        *reinterpret_cast<__nv_bfloat16*>(s_p + sw128(r, krow >> 3) + (krow & 7) * 2) = __float2bfloat16_rn(p0);
        *reinterpret_cast<__nv_bfloat16*>(s_p + sw128(r, (krow >> 3) + 1) + (krow & 7) * 2) = __float2bfloat16_rn(p1);
      }
      if (need) {
#pragma unroll
        for (int x = 0; x < 16; ++x) {
          const float a = s_alpha[8 * (x >> 1) + qd + (x & 1)];
          const int e = 4 * (x >> 1) + (x & 1);
#pragma unroll
          for (int m = 0; m < 4; ++m) { o[m][e] *= a; o[m][e + 2] *= a; }
        }
      }
      fence_async_smem();
      asm volatile("bar.sync 1, 128;" ::: "memory");       // P complete; red / s_m free for the next tile
      if (threadIdx.x == 0) mbar_arrive(&p_full);
    } else {
      // ---- WG1: the K slots are free once P(it) is published; then the rescale WG0 decided for this tile ----
      mbar_wait(&p_full, ph);
      if (more && threadIdx.x == 128)
        load_chunks<kFp8>(map_k, map_v, s_ring, full_b, 0, kKC, kPaged ? page_row(t_begin + it + 1) : next_row, pol_kv);
      float al[16];
      bool need = false;
#pragma unroll
      for (int x = 0; x < 16; ++x) {
        al[x] = s_alpha[8 * (x >> 1) + qd + (x & 1)];
        need |= al[x] != 1.f;
      }
      if (need) {
#pragma unroll
        for (int x = 0; x < 16; ++x) {
          const int e = 4 * (x >> 1) + (x & 1);
#pragma unroll
          for (int m = 0; m < 4; ++m) { o[m][e] *= al[x]; o[m][e + 2] *= al[x]; }
        }
      }
    }
    if constexpr (kFp8) {
      // ---- e4m3: this warpgroup's V chunks expanded, with the rows of keys >= Lk zeroed as below ----
      for (int m = 0; m < 4; ++m) {
        const int c = kKC + vc0 + m;
        mbar_wait(&full_b[c], ph);
        if (wg0) expand_e4m3<1>(s_ring + c * kSlot, threadIdx.x, Lk - key0);
        else expand_e4m3<3>(s_ring + c * kSlot, threadIdx.x - 128, Lk - key0);
      }
      fence_async_smem();
      if (wg0) asm volatile("bar.sync 1, 128;" ::: "memory");
      else asm volatile("bar.sync 3, 128;" ::: "memory");
    } else if constexpr (kPaged) {
      // ---- the tile holding Lk: V rows of keys >= Lk are unwritten cache slots (maybe NaN) and 0 * NaN would poison
      // O, so they are zeroed (whole 128 B rows: the swizzle permutes within a row) in this warpgroup's V chunks ----
      if (key0 + kTile > Lk) {
        for (int m = 0; m < 4; ++m) {
          const int c = kKC + vc0 + m;
          mbar_wait(&full_b[c], ph);
          for (int u = (Lk - key0) * 8 + (threadIdx.x & 127); u < kTile * 8; u += 128)
            *reinterpret_cast<uint4*>(s_ring + c * kSlot + u * 16) = make_uint4(0, 0, 0, 0);
        }
        fence_async_smem();
        if (wg0) asm volatile("bar.sync 1, 128;" ::: "memory");
        else asm volatile("bar.sync 3, 128;" ::: "memory");
      }
    }
    // ---- O^T += V^T . P^T over this warpgroup's 4 V chunks, each a 64-dim M tile read MN-major ----
    wgmma_fence();
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int c = kKC + vc0 + m;
      mbar_wait(&full_b[c], ph);
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)                        // 16 keys = two 8-row groups of the chunk
        WgmmaN<64>::bf16<1>(o[m], make_sw128_desc(ring_a + c * kSlot + ks * 2048, kSlot, 1024),
                            make_sw128_desc(p_a + 32 * ks, 16, 1024), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    if (!wg0 && lane == 0) mbar_arrive(&p_empty);
    if (more) {                                             // this warpgroup's V slots are free: load tile it + 1's
      if (wg0) asm volatile("bar.sync 1, 128;" ::: "memory");
      else asm volatile("bar.sync 3, 128;" ::: "memory");
      if ((threadIdx.x & 127) == 0)
        load_chunks<kFp8>(map_k, map_v, s_ring, full_b, kKC + vc0, kKC + vc0 + 4,
                          kPaged ? page_row(t_begin + it + 1) : next_row, pol_kv);
    }
  }

  // ---- epilogue: row sums (WG0), O^T / l -> bf16 staged in the Q buffer -> 16-byte coalesced stores ----
  if (wg0) {
#pragma unroll
    for (int x = 0; x < 16; ++x) {
      const float ls = rows_sum(l_part[x]);
      if (lane < 4) red[warp][8 * (x >> 1) + qd + (x & 1)] = ls;
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    if (threadIdx.x < kRows) {
      const int r = threadIdx.x;
      const float l = (red[0][r] + red[1][r]) + (red[2][r] + red[3][r]);
      s_inv[r] = l > 0.f ? 1.f / l : 0.f;
      if constexpr (kPaged) s_m[r] = l > 0.f ? s_m[r] + log2f(l) : -INFINITY;   // the split's LSE (log2 domain)
    }
  }
  __syncthreads();                                          // s_inv ready; Q no longer read by any wgmma
  if constexpr (kPaged) {
    if (splits > 1) {
      // ---- split partials: O^T / l as fp32 rows staged in the ring (free: no load is in flight after the last tile)
      // -> 16-byte coalesced stores in the splitkv.cuh layout, row = q0 * H + r0 + r ----
      float* stage = reinterpret_cast<float*>(s_ring);
#pragma unroll
      for (int x = 0; x < 16; ++x) {
        const int r = 8 * (x >> 1) + qd + (x & 1);
        const float inv = s_inv[r];
        const int e = 4 * (x >> 1) + (x & 1);
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          stage[r * kPartPitch + 64 * (vc0 + m) + krow] = o[m][e] * inv;
          stage[r * kPartPitch + 64 * (vc0 + m) + krow + 8] = o[m][e + 2] * inv;
        }
      }
      __syncthreads();
      for (int u = threadIdx.x; u < kRows * (kC / 4); u += kThreads) {
        const int r = u / (kC / 4), c4 = u % (kC / 4);
        if (r0 + r > rlast) break;                          // rows are consecutive in u
        const int64_t row = (int64_t)q0 * H + r0 + r;
        *reinterpret_cast<float4*>(o_part + (row * splits + split) * kC + c4 * 4) =
            *reinterpret_cast<const float4*>(stage + r * kPartPitch + c4 * 4);
        if (c4 == 0) lse[row * splits + split] = s_m[r];
      }
      return;
    }
  }
#pragma unroll
  for (int x = 0; x < 16; ++x) {
    const int r = 8 * (x >> 1) + qd + (x & 1);
    const float inv = s_inv[r];
    const int e = 4 * (x >> 1) + (x & 1);
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      uint8_t* dst = s_q + r * kOutPitch + (64 * (vc0 + m) + krow) * 2;
      *reinterpret_cast<__nv_bfloat16*>(dst) = __float2bfloat16_rn(o[m][e] * inv);
      *reinterpret_cast<__nv_bfloat16*>(dst + 16) = __float2bfloat16_rn(o[m][e + 2] * inv);
    }
  }
  __syncthreads();
  __nv_bfloat16* orow = out + ((int64_t)q0 * H + r0) * kC;
  for (int u = threadIdx.x; u < kRows * (kC / 8); u += kThreads) {
    const int r = u / (kC / 8), cu = u % (kC / 8);
    if (r0 + r <= rlast)
      *reinterpret_cast<uint4*>(orow + (int64_t)r * kC + cu * 8) = *reinterpret_cast<const uint4*>(s_q + r * kOutPitch + cu * 16);
  }
}

__global__ void __launch_bounds__(kThreads, 1) mla_prefill_kernel(
    const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
    const __grid_constant__ CUtensorMap map_v, const int32_t* __restrict__ cu_q, const int32_t* __restrict__ cu_k, int B,
    int H, int row_tiles, int causal, float scale, __nv_bfloat16* __restrict__ out) {
  mla_prefill_cta<false>(&map_q, nullptr, &map_k, &map_v, cu_q, cu_k, nullptr, nullptr, 0, 0, 0, 1, B, H, row_tiles,
                         causal, scale, nullptr, nullptr, out);
}

// K and V are the same cache rows: map_kv serves the 9 K boxes and, again, the first 8 as V (the second read of a page
// is expected to hit L2)
__global__ void __launch_bounds__(kThreads, 1) mla_paged_prefill_kernel(
    const __grid_constant__ CUtensorMap map_qn, const __grid_constant__ CUtensorMap map_qpe,
    const __grid_constant__ CUtensorMap map_kv, const int32_t* __restrict__ seqlens_excl,
    const int32_t* __restrict__ block_table, int bt_stride, int B, int sq, int H, int appended, int row_tiles,
    int splits, int causal, float scale, float* __restrict__ o_part, float* __restrict__ lse,
    __nv_bfloat16* __restrict__ out) {
  mla_prefill_cta<true>(&map_qn, &map_qpe, &map_kv, &map_kv, nullptr, nullptr, seqlens_excl, block_table, bt_stride, sq,
                        appended, splits, B, H, row_tiles, causal, scale, o_part, lse, out);
}

// The same over an e4m3 cache: map_kv holds the cache as bytes, box = [64 rows x 64 B], no swizzle
__global__ void __launch_bounds__(kThreads, 1) mla_paged_prefill_e4m3_kernel(
    const __grid_constant__ CUtensorMap map_qn, const __grid_constant__ CUtensorMap map_qpe,
    const __grid_constant__ CUtensorMap map_kv, const int32_t* __restrict__ seqlens_excl,
    const int32_t* __restrict__ block_table, int bt_stride, int B, int sq, int H, int appended, int row_tiles,
    int splits, int causal, float scale, float* __restrict__ o_part, float* __restrict__ lse,
    __nv_bfloat16* __restrict__ out) {
  mla_prefill_cta<true, __nv_fp8_e4m3>(&map_qn, &map_qpe, &map_kv, &map_kv, nullptr, nullptr, seqlens_excl, block_table,
                                       bt_stride, sq, appended, splits, B, H, row_tiles, causal, scale, o_part, lse,
                                       out);
}

}  // namespace
}  // namespace cb

// flash_attn_varlen_func for absorbed MLA (include/chitu_b200.h).
extern "C" int chitu_b200_mla_prefill(const void* q, const void* k, int64_t k_sb, const void* v, int64_t v_sb,
                                      const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k, int B, int H,
                                      int total_q, int total_k, int max_seqlen_q, int causal, float softmax_scale,
                                      void* out, void* stream) {
  using namespace cb;
  CB_ARG(q && k && v && cu_seqlens_q && cu_seqlens_k && out);
  CB_ARG(B >= 0 && H >= 1 && max_seqlen_q >= 0 && total_q >= 0 && total_k >= 0);
  CB_ARG(k_sb >= kRow && v_sb >= kC && k_sb % 8 == 0 && v_sb % 8 == 0);          // TMA: 16-byte row strides
  CB_ARG(((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out) % 16 == 0); // TMA / vector stores: 16-byte bases
  CB_ARG((int64_t)total_q * H <= INT_MAX && (int64_t)max_seqlen_q * H <= INT_MAX - kRows);   // int32 TMA row coordinates
  if (B == 0 || total_q == 0 || max_seqlen_q == 0) return 0;
  const int row_tiles = cdiv((int64_t)max_seqlen_q * H, kRows);
  if ((int64_t)row_tiles * B > INT_MAX)
    return fail(-1, "mla_prefill: %d sequences x %d row tiles exceed the grid", B, row_tiles);
  CUtensorMap mq, mk, mv;
  // total_k == 0: no sequence has a key, the K / V maps are never read (one row keeps them encodable)
  const int64_t krows = total_k > 0 ? total_k : 1;
  int rc = make_tma_map_2d(&mq, q, (int64_t)total_q * H, kRow, 2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, kRows);
  if (!rc) rc = make_tma_map_2d(&mk, k, krows, kRow, 2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, kTile, k_sb);
  if (!rc) rc = make_tma_map_2d(&mv, v, krows, kC, 2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, kTile, v_sb);
  if (rc) return rc;
  rc = launch_smem<mla_prefill_kernel>(__func__, dim3(row_tiles * B), dim3(kThreads), 1024 + kSmemBytes,
                                       (cudaStream_t)stream, mq, mk, mv, cu_seqlens_q, cu_seqlens_k, B, H, row_tiles,
                                       causal ? 1 : 0, softmax_scale, (__nv_bfloat16*)out);
  if (rc) return rc;
  CB_LAUNCHED(1);
  return 0;
}

namespace cb {
// chitu_b200_mla_paged_prefill (e4m3 = false) and the sq > 1 form of chitu_b200_mla_attn_fp8kv (e4m3: kv_cache holds
// e4m3 bytes, the new rows are stored by the e4m3 append).  Argument checks and launches report under `entry`, the
// other refusals under `tag`.
int mla_paged_prefill(const char* entry, const char* tag, bool e4m3, const void* q_nope, const void* q_pe,
                      void* kv_cache, const void* new_kv, const int32_t* seqlens_excl, const int32_t* block_table,
                      int bt_stride, int B, int sq, int H, int C, int R, int page_size, int num_blocks,
                      int max_seqlen_hint, int causal, float softmax_scale, void* out, void* workspace,
                      int64_t workspace_bytes, cudaStream_t st) {
  CB_ARG_AS(entry, q_nope && q_pe && kv_cache && seqlens_excl && block_table && out);
  CB_ARG_AS(entry, B >= 0 && sq >= 1 && H >= 1 && bt_stride > 0 && num_blocks > 0);
  if (C != kC || R != kR)
    return fail(-1, "%s: only kv_lora_rank=512, qk_rope_head_dim=64 is built (got %d,%d)", tag, C, R);
  if (page_size != kTile) return fail(-1, "%s: page_size must be 64 (got %d)", tag, page_size);
  CB_ARG_AS(entry, ((uintptr_t)q_nope | (uintptr_t)q_pe | (uintptr_t)kv_cache | (uintptr_t)new_kv | (uintptr_t)out |
                    (uintptr_t)workspace) % 16 == 0);                           // TMA / vector accesses: 16-byte bases
  CB_ARG_AS(entry, (int64_t)B * sq * H <= INT_MAX && (int64_t)num_blocks * kTile <= INT_MAX);   // int32 TMA rows
  if (B == 0) return 0;

  const int row_tiles = cdiv((int64_t)sq * H, kRows);
  const int max_len = max_seqlen_hint > 0 ? max_seqlen_hint : bt_stride * kTile;
  // the decode kernels' wave rule on this kernel's CTAs (1 per SM), shrunk to the workspace (none: 1 split)
  const int64_t rows = (int64_t)B * sq * H;
  int splits = pick_splits_waves(row_tiles * B, max_len, 132);
  splits = workspace ? splits_that_fit(splits, rows, kC, workspace_bytes) : 1;
  if ((int64_t)row_tiles * splits * B > INT_MAX)
    return fail(-1, "%s: %d requests x %d row tiles x %d splits exceed the grid", tag, B, row_tiles, splits);
  if (!tma_available()) return fail(-3, "%s: TMA is not available", tag);
  const auto [o_part, lse, plan] = split_kv_carve(splits > 1 ? workspace : nullptr, workspace_bytes, rows, kC, splits);

  CUtensorMap mqn, mqp, mkv;
  int rc = make_tma_map_2d(&mqn, q_nope, rows, kC, 2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, kRows);
  if (!rc) rc = make_tma_map_2d(&mqp, q_pe, rows, kR, 2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, kRows);
  if (!rc && e4m3)    // one box per 64-element chunk, landed in half of its slot
    rc = make_tma_map_2d(&mkv, kv_cache, (int64_t)num_blocks * kTile, kRow, 1, CU_TENSOR_MAP_DATA_TYPE_UINT8, kTile, 0,
                         64);
  else if (!rc)
    rc = make_tma_map_2d(&mkv, kv_cache, (int64_t)num_blocks * kTile, kRow, 2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16,
                         kTile);
  if (rc) return rc;

  if (new_kv) {       // the B * sq new latent rows first, pages indexed with a literal 64 as the reference's append does
    const int64_t row_bytes = kRow * 2;
    if (e4m3)
      launch_paged_append_e4m3({kv_cache, new_kv, sq * row_bytes, row_bytes}, {}, kRow, CB_BF16, seqlens_excl, nullptr,
                               block_table, bt_stride, B, sq, kTile, st);
    else
      launch_paged_append({kv_cache, new_kv, sq * row_bytes, row_bytes}, {}, row_bytes, seqlens_excl, nullptr,
                          block_table, bt_stride, B, sq, kTile, 64, st);
    CB_LAUNCHED_AS(entry, 1);
  }
  const dim3 grid(row_tiles * splits * B), block(kThreads);
  const int appended = new_kv ? 1 : 0;
  causal = causal ? 1 : 0;
  if (e4m3)
    rc = launch_smem<mla_paged_prefill_e4m3_kernel>(entry, grid, block, 1024 + kSmemBytes, st, mqn, mqp, mkv,
                                                    seqlens_excl, block_table, bt_stride, B, sq, H, appended,
                                                    row_tiles, splits, causal, softmax_scale, o_part, lse,
                                                    (__nv_bfloat16*)out);
  else
    rc = launch_smem<mla_paged_prefill_kernel>(entry, grid, block, 1024 + kSmemBytes, st, mqn, mqp, mkv, seqlens_excl,
                                               block_table, bt_stride, B, sq, H, appended, row_tiles, splits, causal,
                                               softmax_scale, o_part, lse, (__nv_bfloat16*)out);
  if (rc) return rc;
  CB_LAUNCHED_AS(entry, 1);
  if (splits > 1) {
    rc = launch_merge_splits(o_part, lse, out, (int)rows, splits, kC, CB_BF16, st);
    if (rc) return rc;
    CB_LAUNCHED_AS(entry, 1);
  }
  return 0;
}
}  // namespace cb

// mla_attn_with_kvcache with more than one query token per request (include/chitu_b200.h).
extern "C" int chitu_b200_mla_paged_prefill(const void* q_nope, const void* q_pe, void* kv_cache, const void* new_kv,
                                            const int32_t* seqlens_excl, const int32_t* block_table, int bt_stride,
                                            int B, int sq, int H, int C, int R, int page_size, int num_blocks,
                                            int max_seqlen_hint, int causal, float softmax_scale, void* out,
                                            void* workspace, int64_t workspace_bytes, void* stream) {
  return cb::mla_paged_prefill(__func__, "mla_paged_prefill", false, q_nope, q_pe, kv_cache, new_kv, seqlens_excl,
                               block_table, bt_stride, B, sq, H, C, R, page_size, num_blocks, max_seqlen_hint, causal,
                               softmax_scale, out, workspace, workspace_bytes, (cudaStream_t)stream);
}

// mla_attn_with_kvcache over an e4m3 paged latent cache (include/chitu_b200.h): sq == 1 the decode kernel, sq > 1 the
// multi-token kernel, both with the cache type as a compile-time parameter of the bf16 kernels' CTA.
extern "C" int chitu_b200_mla_attn_fp8kv(const void* q_nope, const void* q_pe, void* kv_cache, const void* new_kv,
                                         const int32_t* seqlens_excl, const int32_t* block_table, int bt_stride, int B,
                                         int sq, int H, int C, int R, int page_size, int num_blocks,
                                         int max_seqlen_hint, int causal, float softmax_scale, void* out,
                                         void* workspace, int64_t workspace_bytes, void* stream) {
  CB_ARG(sq >= 1);
  if (sq == 1)      // one token: causal changes nothing (its only row sees every key)
    return cb::mla_decode(__func__, __func__, true, q_nope, q_pe, kv_cache, new_kv, seqlens_excl, block_table,
                          bt_stride, B, H, C, R, page_size, num_blocks, max_seqlen_hint, softmax_scale, out, workspace,
                          workspace_bytes, (cudaStream_t)stream);
  return cb::mla_paged_prefill(__func__, __func__, true, q_nope, q_pe, kv_cache, new_kv, seqlens_excl, block_table,
                               bt_stride, B, sq, H, C, R, page_size, num_blocks, max_seqlen_hint, causal, softmax_scale,
                               out, workspace, workspace_bytes, (cudaStream_t)stream);
}

CB_DEFINE_TL_SETTER(mla_prefill)
