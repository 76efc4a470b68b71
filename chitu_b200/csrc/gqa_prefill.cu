// GQA attention over the paged KV cache for more than one query token per request (sm_90a): wgmma + TMA + mbarrier.
//
// AttnBackend.attn_with_kvcache with seqlen_q > 1 (attn_backend.py:92-164, FlashAttn impl :208-243, i.e.
// flash_attn_with_kvcache): chunked prefill, prefill on top of a cached prefix, speculative verification.
//   q [B, sq, Hq, 128], k_cache / v_cache [num_blocks, page, Hkv, 128], new k / v [B, sq, Hkv, 128] appended in place at
//   positions cache_seqlens[b] + i (true page indexing), attention over Lk = cache_seqlens[b] (+ sq) keys, fp32 scores and
//   softmax, P rounded to the io dtype before P.V, causal mask aligned bottom-right (query i sees keys j <= i + Lk - sq),
//   rows that see no key are 0.
//
// Two launches (three with a split): the append kernel writes the sq new rows first, so the attention kernel reads
// every key from the cache and never races the append (PDL: a kernel touches memory only after its predecessor is done).
//
// Attention mapping: one CTA owns (request b, kv head, 64 query rows r = i * G + j: token i, query head j of the kv
// head's group), so each K / V tile is staged once for the G heads.  The rows are the wgmma M dimension:
//   S[64 rows x 64 keys]    = Q[64 x 128] . K^T     A = Q tile (staged once), B = K tile, both K-major in shared memory
//   O[64 rows x 128 dims] += P[64 x 64] . V          A = P in registers, B = V tile read MN-major
// One warpgroup (128 threads) does everything.  A thread holds two rows of S, P and O (32 + 16 packed + 64 registers),
// so the row max and the online softmax stay in registers with two lane shuffles, and P never goes through shared
// memory: the S accumulator fragment is the A fragment of P.V.  Thread 0 streams the K / V tiles by TMA through a
// 2-stage mbarrier ring and refills a slot once its P.V has finished (one CTA barrier per tile).  Two CTAs per SM
// overlap one CTA's softmax with the other's MMAs.
// TMA: a 3-D map over the cache, dims (128, Hkv, num_blocks * page), box (64 dims, 1 head, 64 keys) = one [64 x 128 B]
// swizzled chunk of one head inside one page (page % 64 == 0); a tile is 2 K + 2 V chunks.
// Paging safety: only block_table[b, 0 .. ceil(Lk / page) - 1] is read; V rows of keys >= Lk in the last tile are zeroed
// in shared memory before P.V (unused slots may hold NaN, and 0 * NaN would poison O); their scores are replaced by -inf.
// Shared memory: Q 16 KB + 2 x 32 KB ring = 80 KB + 1 KB alignment.
// Non-paged cache (chitu_b200_gqa_contiguous_attn, no block table): the same CTA compiled with a 4-D map over
// [B, S, Hkv, 128] caches (gqa_prefill_contig_kernel); TMA zero-fills keys >= S, so any S works.
// e4m3 cache (chitu_b200_gqa_paged_attn_fp8kv, gqa_prefill_e4m3_kernel): UINT8 maps, one [64 keys x 128 B] box per K and
// per V tile in a 2-stage ring, converted by the warpgroup into one io-dtype stage; the same 80 KB of shared memory.
// Split over keys when (row tiles x Hkv x B) CTAs cannot fill the GPU: split s of a CTA takes an equal share of the
// CTA's key tiles and writes normalised fp32 partials + LSE to the workspace as [B, sq * Hq, S, 128] (the decode
// layout with H = sq * Hq), merged by attention.cu's merge_splits_kernel.  Deterministic: the split count depends on
// host values only and every partial is reduced in a fixed order.
// gqa_prefill() launches all three layouts: for chitu_b200_gqa_paged_prefill here and for the multi-token paths of
// chitu_b200_gqa_contiguous_attn and chitu_b200_gqa_paged_attn_fp8kv (attention.cu), which check their arguments.
#include <cuda.h>
#include <limits.h>

#include "common.cuh"
#include "splitkv.cuh"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace cb {
namespace {

constexpr int kD = 128;
constexpr int kTile = 64;                      // keys per tile
constexpr int kRows = 64;                      // query rows (token, head) per CTA
constexpr int kSlot = 64 * 128;                // 8 KB: one TMA box [64 rows x 128 B]
constexpr int kStages = 2;
constexpr int kStageBytes = 4 * kSlot;         // K dims 0-63, 64-127, V dims 0-63, 64-127
constexpr int kQBytes = 2 * kSlot;
constexpr int kSmemBytes = kQBytes + kStages * kStageBytes;
constexpr int kOutPitch = kD + 4;              // staged fp32 output row in floats (the rows a warp touches differ in bank)
static_assert(kRows * kOutPitch * 4 <= kStages * kStageBytes, "the output tile is staged in the ring");
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kRescaleThreshold = 8.f;       // log2 domain
constexpr int kThreads = 128;
constexpr int kCtasPerSm = 2;

__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5}], [%2], %6;"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "l"(policy)
      : "memory");
}

// S = Q . K^T (both operands in shared memory, K-major) and O += P . V (P in registers as the A operand, V read
// MN-major: the B operand transposed)
template <typename T> struct Mma;
template <> struct Mma<__nv_bfloat16> {
  static __device__ __forceinline__ void qk(float (&d)[32], uint64_t a, uint64_t b, int acc) {
    WgmmaN<64>::bf16<0>(d, a, b, acc);
  }
  static __device__ __forceinline__ void pv(float (&d)[64], const uint32_t (&a)[4], uint64_t b) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, 1;\n\t}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
  }
};
template <> struct Mma<__half> {
  static __device__ __forceinline__ void qk(float (&d)[32], uint64_t a, uint64_t b, int acc) {
    WgmmaN<64>::f16<0>(d, a, b, acc);
  }
  static __device__ __forceinline__ void pv(float (&d)[64], const uint32_t (&a)[4], uint64_t b) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, 1;\n\t}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
  }
};

__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], %7;"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(policy)
      : "memory");
}

// CONTIG: the maps are 4-D over a contiguous cache, (128, Hkv, cache_rows, B) with the cache's batch stride, and key
// tile t of request b is the box at (c, kvh, 64 t, b).  Rows at or past cache_rows are zero-filled by TMA, so no box
// reads another request's rows; block_table, bt_stride and page are unused.
// C: the cache element, T or uint8_t (e4m3, paged only).  With e4m3 the maps are UINT8 (128 B = 128 dims, 1, keys) and
// a tile is one [64 keys x 128 B] K box and one V box in a 2-stage e4m3 ring behind a single io-dtype stage: the
// warpgroup converts each box into the two 64-dim io chunks the wgmmas read (V rows of keys >= Lk become 0 there), so
// shared memory stays at kSmemBytes.
template <typename T, typename C, int G, bool CONTIG>
__device__ __forceinline__ void gqa_prefill_cta(
    const CUtensorMap& map_k, const CUtensorMap& map_v, const T* __restrict__ q,
    const int32_t* __restrict__ cache_seqlens, const int32_t* __restrict__ block_table, int bt_stride, int sq, int Hq,
    int Hkv, int page, int appended, int causal, float scale, int row_tiles, int splits, float* __restrict__ o_part,
    float* __restrict__ lse, T* __restrict__ out) {
  extern __shared__ __align__(1024) uint8_t gqa_prefill_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(gqa_prefill_smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_q = smem;                                      // [2][64 rows][128 B]
  uint8_t* s_ring = s_q + kQBytes;                          // [kStages][K0 K1 V0 V1][64 keys][128 B]; output staging
  constexpr bool kE4m3 = sizeof(C) == 1;
  static_assert(!(kE4m3 && CONTIG), "the e4m3 cache is paged");
  static_assert(kStageBytes + kStages * 2 * kSlot == kStages * kStageBytes, "e4m3: one io stage + the e4m3 ring");
  uint8_t* s_e4m3 = s_ring + kStageBytes;                   // e4m3: [kStages][K V][64 keys][128 B]
  __shared__ __align__(8) uint64_t kfull[kStages], vfull[kStages];
  __shared__ float s_lse[kRows];                            // row LSE (log2 domain) for the split partials

  const int split = blockIdx.x % splits;
  const int tile = row_tiles - 1 - blockIdx.x / splits;     // last row tiles (most causal work) first
  const int kvh = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  cb::pdl_prologue();                                       // q, the lengths and the appended rows come from earlier kernels
  const int Lk = cache_seqlens[b] + (appended ? sq : 0);
  const int nrows = sq * G;
  const int r0 = tile * kRows;
  const int rlast = min(r0 + kRows, nrows) - 1;
  // keys visible to row r (token r / G) are [0, lim(r)); lim is non-decreasing in r
  auto lim = [&](int r) { return causal ? max(0, min(Lk, r / G + 1 + Lk - sq)) : max(Lk, 0); };
  const int all_see = lim(r0);                              // keys below this are visible to every row of the tile
  const int ntiles = (lim(rlast) + kTile - 1) / kTile;
  const int per_split = (ntiles + splits - 1) / splits;
  const int t_begin = min(ntiles, split * per_split), t_end = min(ntiles, t_begin + per_split);
  const uint64_t pol_kv = l2_policy_evict_last();           // K / V are re-read by every row tile and kv-head group

  auto load_tile = [&](int t) {                             // key tile t into its ring slot (one thread)
    const int slot = (t - t_begin) % kStages;
    const int key0 = t * kTile;
    if constexpr (CONTIG) {
      uint8_t* dst = s_ring + slot * kStageBytes;
      mbar_expect_tx(&kfull[slot], 2 * kSlot);
      tma_load_4d(dst, &map_k, &kfull[slot], 0, kvh, key0, b, pol_kv);
      tma_load_4d(dst + kSlot, &map_k, &kfull[slot], 64, kvh, key0, b, pol_kv);
      mbar_expect_tx(&vfull[slot], 2 * kSlot);
      tma_load_4d(dst + 2 * kSlot, &map_v, &vfull[slot], 0, kvh, key0, b, pol_kv);
      tma_load_4d(dst + 3 * kSlot, &map_v, &vfull[slot], 64, kvh, key0, b, pol_kv);
      return;
    }
    const int prow = block_table[(int64_t)b * bt_stride + key0 / page] * page + key0 % page;
    if constexpr (kE4m3) {
      uint8_t* dst = s_e4m3 + slot * 2 * kSlot;
      mbar_expect_tx(&kfull[slot], kSlot);
      tma_load_3d(dst, &map_k, &kfull[slot], 0, kvh, prow, pol_kv);
      mbar_expect_tx(&vfull[slot], kSlot);
      tma_load_3d(dst + kSlot, &map_v, &vfull[slot], 0, kvh, prow, pol_kv);
      return;
    }
    uint8_t* dst = s_ring + slot * kStageBytes;
    mbar_expect_tx(&kfull[slot], 2 * kSlot);
    tma_load_3d(dst, &map_k, &kfull[slot], 0, kvh, prow, pol_kv);
    tma_load_3d(dst + kSlot, &map_k, &kfull[slot], 64, kvh, prow, pol_kv);
    mbar_expect_tx(&vfull[slot], 2 * kSlot);
    tma_load_3d(dst + 2 * kSlot, &map_v, &vfull[slot], 0, kvh, prow, pol_kv);
    tma_load_3d(dst + 3 * kSlot, &map_v, &vfull[slot], 64, kvh, prow, pol_kv);
  };

  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&kfull[i], 1);
      mbar_init(&vfull[i], 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    for (int t = t_begin; t < min(t_end, t_begin + kStages); ++t) load_tile(t);
  }
  // Q rows of the tile -> two K-major swizzled chunks (dims 0-63, 64-127); rows past the request are zero
  for (int u = threadIdx.x; u < kRows * 16; u += kThreads) {
    const int r = u >> 4, c = u & 15;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r0 + r < nrows) {
      const int i = (r0 + r) / G, j = (r0 + r) % G;
      v = *reinterpret_cast<const uint4*>(q + (((int64_t)b * sq + i) * Hq + kvh * G + j) * kD + c * 8);
    }
    *reinterpret_cast<uint4*>(s_q + (c >> 3) * kSlot + sw128(r, c & 7)) = v;
  }
  fence_async_smem();
  __syncthreads();

  // accumulator fragments: this thread holds rows rw and rw + 8 of the tile (x = 0, 1) and columns 8 nb + qd + j
  const int rw = warp * 16 + (lane >> 2);
  const int qd = 2 * (lane & 3);
  const int lim_r[2] = {lim(r0 + rw), lim(r0 + rw + 8)};
  const uint32_t ring_a = smem_u32(s_ring), q_a = smem_u32(s_q);
  float o[64];                                              // O[row x][dim 8 nb + qd + j] = o[4 nb + 2 x + j]
#pragma unroll
  for (int e = 0; e < 64; ++e) o[e] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};                  // running row max (log2 domain), the same in a lane quad
  float l_run[2] = {0.f, 0.f};                              // this thread's share of the row sums

  // e4m3: one [64 keys x 128 B] box (16-byte unit c = dims 16c .. 16c+15) -> units 2c, 2c+1 of io chunk c / 4; rows at
  // or past `valid` are written as 0
  auto e4m3_to_io = [&](const uint8_t* src, uint8_t* dst, int valid) {
    for (int u = threadIdx.x; u < kTile * 8; u += kThreads) {
      const int r = u >> 3, c = u & 7;
      uint4 lo = make_uint4(0, 0, 0, 0), hi = make_uint4(0, 0, 0, 0);
      if (r < valid) {
        const uint4 w = *reinterpret_cast<const uint4*>(src + sw128(r, c));
        E4m3<T>::to_io(w.x, lo.x, lo.y);
        E4m3<T>::to_io(w.y, lo.z, lo.w);
        E4m3<T>::to_io(w.z, hi.x, hi.y);
        E4m3<T>::to_io(w.w, hi.z, hi.w);
      }
      uint8_t* d = dst + (c >> 2) * kSlot;
      *reinterpret_cast<uint4*>(d + sw128(r, (2 * c) & 7)) = lo;
      *reinterpret_cast<uint4*>(d + sw128(r, (2 * c + 1) & 7)) = hi;
    }
    fence_async_smem();
    __syncthreads();
  };

  const float sc = scale * kLog2e;
  for (int t = t_begin; t < t_end; ++t) {
    const int slot = (t - t_begin) % kStages;
    const uint32_t ph = ((t - t_begin) / kStages) & 1;
    const uint32_t st_a = ring_a + (kE4m3 ? 0 : slot) * kStageBytes;
    // ---- S = Q . K^T over the 2 chunks of 64 dims ----
    float s[32];
    mbar_wait(&kfull[slot], ph);
    if constexpr (kE4m3) e4m3_to_io(s_e4m3 + slot * 2 * kSlot, s_ring, kTile);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < 2; ++c)
#pragma unroll
      for (int k = 0; k < 4; ++k)
        Mma<T>::qk(s, make_sw128_desc(q_a + c * kSlot + 32 * k, 16, 1024),
                   make_sw128_desc(st_a + c * kSlot + 32 * k, 16, 1024), (c | k) != 0);
    wgmma_commit();
    wgmma_wait<0>();

    // ---- scale, mask (a select, so a NaN score of an unwritten slot never survives) ----
    const int key0 = t * kTile;
    if (key0 + kTile > all_see) {
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        const int key = key0 + 8 * (e >> 2) + qd + (e & 1);
        s[e] = key < lim_r[(e >> 1) & 1] ? s[e] * sc : -INFINITY;
      }
    } else {
#pragma unroll
      for (int e = 0; e < 32; ++e) s[e] *= sc;
    }
    // ---- online softmax in registers: the row max moves only when it grew by more than 2^8 (exact result: P, l and
    // O share it); P = exp2(S - m) rounded to the io dtype, packed as the A fragments of the P.V product ----
    uint32_t pa[4][4];
#pragma unroll
    for (int x = 0; x < 2; ++x) {
      float mx = -INFINITY;
#pragma unroll
      for (int nb = 0; nb < 8; ++nb) mx = fmaxf(mx, fmaxf(s[4 * nb + 2 * x], s[4 * nb + 2 * x + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      if (mx > m_run[x] + kRescaleThreshold) {              // also the first finite max (m_run = -inf): a = 0
        const float a = exp2f(m_run[x] - mx);
        m_run[x] = mx;
        l_run[x] *= a;
#pragma unroll
        for (int nb = 0; nb < 16; ++nb) { o[4 * nb + 2 * x] *= a; o[4 * nb + 2 * x + 1] *= a; }
      }
      const float mr = m_run[x] == -INFINITY ? 0.f : m_run[x];   // a row with no visible key so far: P = 0
#pragma unroll
      for (int nb = 0; nb < 8; ++nb) {
        const float p0 = exp2f(s[4 * nb + 2 * x] - mr), p1 = exp2f(s[4 * nb + 2 * x + 1] - mr);
        l_run[x] += p0 + p1;
        pa[nb >> 1][2 * (nb & 1) + x] = pack2(p0, p1, (const T*)nullptr);
      }
    }
    // ---- V rows of keys past the sequence (unwritten slots, possibly NaN) -> 0 before P.V reads them ----
    if constexpr (kE4m3) {
      mbar_wait(&vfull[slot], ph);
      e4m3_to_io(s_e4m3 + slot * 2 * kSlot + kSlot, s_ring + 2 * kSlot, Lk - key0);
      if (threadIdx.x == 0 && t + kStages < t_end) load_tile(t + kStages);     // both boxes of the slot are converted
    } else {
      if (key0 + kTile > Lk) {
        mbar_wait(&vfull[slot], ph);
        uint4* v0 = reinterpret_cast<uint4*>(s_ring + slot * kStageBytes + 2 * kSlot);
        for (int u = threadIdx.x; u < 2 * kTile * 8; u += kThreads) {
          const int c = u / (kTile * 8), key = (u / 8) % kTile;
          if (key0 + key >= Lk) v0[c * (kSlot / 16) + key * 8 + (u & 7)] = make_uint4(0, 0, 0, 0);
        }
        fence_async_smem();
        __syncthreads();
      }
      mbar_wait(&vfull[slot], ph);
    }
    // ---- O += P . V: 4 steps of 16 keys, N = 128 dims over the two V chunks (64-dim blocks kSlot apart) ----
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) Mma<T>::pv(o, pa[ks], make_sw128_desc(st_a + 2 * kSlot + ks * 2048, kSlot, 1024));
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();                                        // the slot is free
    if (!kE4m3 && threadIdx.x == 0 && t + kStages < t_end) load_tile(t + kStages);
  }

  // ---- epilogue: row sums over the lane quad, O / l staged as fp32 rows in the ring -> coalesced stores ----
  float inv[2];
#pragma unroll
  for (int x = 0; x < 2; ++x) {
    float l = l_run[x];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    inv[x] = l > 0.f ? 1.f / l : 0.f;
    if ((lane & 3) == 0) s_lse[rw + 8 * x] = l > 0.f ? m_run[x] + log2f(l) : -INFINITY;
  }
  float* stage = reinterpret_cast<float*>(s_ring);
#pragma unroll
  for (int nb = 0; nb < 16; ++nb)
#pragma unroll
    for (int x = 0; x < 2; ++x)
      *reinterpret_cast<float2*>(stage + (rw + 8 * x) * kOutPitch + 8 * nb + qd) =
          make_float2(o[4 * nb + 2 * x] * inv[x], o[4 * nb + 2 * x + 1] * inv[x]);
  __syncthreads();
  for (int u = threadIdx.x; u < kRows * (kD / 4); u += kThreads) {
    const int r = u / (kD / 4), c4 = u % (kD / 4);
    if (r0 + r > rlast) break;                              // rows are consecutive in u
    const int i = (r0 + r) / G, j = (r0 + r) % G;
    const int64_t row = ((int64_t)b * sq + i) * Hq + kvh * G + j;   // = b * (sq * Hq) + (i * Hq + h)
    const float4 v = *reinterpret_cast<const float4*>(stage + r * kOutPitch + c4 * 4);
    if (splits == 1) {
      uint2 w;
      w.x = pack2(v.x, v.y, (const T*)nullptr);
      w.y = pack2(v.z, v.w, (const T*)nullptr);
      *reinterpret_cast<uint2*>(out + row * kD + c4 * 4) = w;
    } else {
      *reinterpret_cast<float4*>(o_part + (row * splits + split) * kD + c4 * 4) = v;
      if (c4 == 0) lse[row * splits + split] = s_lse[r];
    }
  }
}

template <typename T, int G>
__global__ void __launch_bounds__(kThreads, kCtasPerSm) gqa_prefill_kernel(
    const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v, const T* __restrict__ q,
    const int32_t* __restrict__ cache_seqlens, const int32_t* __restrict__ block_table, int bt_stride, int sq, int Hq,
    int Hkv, int page, int appended, int causal, float scale, int row_tiles, int splits, float* __restrict__ o_part,
    float* __restrict__ lse, T* __restrict__ out) {
  gqa_prefill_cta<T, T, G, false>(map_k, map_v, q, cache_seqlens, block_table, bt_stride, sq, Hq, Hkv, page, appended,
                                  causal, scale, row_tiles, splits, o_part, lse, out);
}

template <typename T, int G>
__global__ void __launch_bounds__(kThreads, kCtasPerSm) gqa_prefill_e4m3_kernel(
    const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v, const T* __restrict__ q,
    const int32_t* __restrict__ cache_seqlens, const int32_t* __restrict__ block_table, int bt_stride, int sq, int Hq,
    int Hkv, int page, int appended, int causal, float scale, int row_tiles, int splits, float* __restrict__ o_part,
    float* __restrict__ lse, T* __restrict__ out) {
  gqa_prefill_cta<T, uint8_t, G, false>(map_k, map_v, q, cache_seqlens, block_table, bt_stride, sq, Hq, Hkv, page,
                                        appended, causal, scale, row_tiles, splits, o_part, lse, out);
}

template <typename T, int G>
__global__ void __launch_bounds__(kThreads, kCtasPerSm) gqa_prefill_contig_kernel(
    const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v, const T* __restrict__ q,
    const int32_t* __restrict__ cache_seqlens, int sq, int Hq, int Hkv, int appended, int causal, float scale,
    int row_tiles, int splits, float* __restrict__ o_part, float* __restrict__ lse, T* __restrict__ out) {
  gqa_prefill_cta<T, T, G, true>(map_k, map_v, q, cache_seqlens, nullptr, 0, sq, Hq, Hkv, kTile, appended, causal,
                                 scale, row_tiles, splits, o_part, lse, out);
}

}  // namespace

int gqa_prefill(const char* entry, const char* name, KvLayout layout, const void* q, void* k_cache, void* v_cache,
                const void* k_new, const void* v_new, int64_t k_new_sb, int64_t k_new_st, int64_t v_new_sb,
                int64_t v_new_st, const int32_t* cache_seqlens, const int32_t* block_table, int bt_stride,
                int page_size, int num_blocks, int64_t rows_sb, int cache_rows, int B, int sq, int Hq, int Hkv,
                int max_len, int causal, float softmax_scale, void* out, void* workspace, int64_t workspace_bytes,
                int dtype, cudaStream_t st) {
  if (!tma_available()) return fail(-3, "%s: TMA is not available", entry);
  const int G = Hq / Hkv;
  const int row_tiles = cdiv((int64_t)sq * G, kRows);
  const int64_t rows = (int64_t)B * sq * Hq;
  // the decode kernels' wave rule on this kernel's CTAs, shrunk to the workspace (none: 1 split)
  int splits = pick_splits_waves(row_tiles * Hkv * B, max_len, 132 * kCtasPerSm);
  splits = workspace ? splits_that_fit(splits, rows, kD, workspace_bytes) : 1;
  if ((int64_t)row_tiles * splits > INT_MAX)
    return fail(-1, "%s: %d row tiles x %d splits exceed the grid", entry, row_tiles, splits);
  const SplitKv part = split_kv_carve(splits > 1 ? workspace : nullptr, workspace_bytes, rows, kD, splits);

  // the caches as (128 dims, Hkv, keys[, B]) with a box of 128 B of dims x 1 head x 64 keys: paged (keys = num_blocks *
  // page, a box lies inside one page), contiguous (keys = cache_rows, 4-D with the batch stride), e4m3 paged (UINT8)
  const bool contig = layout == KvLayout::kContiguous, e4m3 = layout == KvLayout::kPagedE4m3;
  const int esize = e4m3 ? 1 : 2;
  const cuuint64_t dims[4] = {(cuuint64_t)kD, (cuuint64_t)Hkv,
                              contig ? (cuuint64_t)cache_rows : (cuuint64_t)num_blocks * page_size, (cuuint64_t)B};
  const cuuint64_t strides[3] = {(cuuint64_t)kD * esize, (cuuint64_t)Hkv * kD * esize,
                                 (cuuint64_t)rows_sb * Hkv * kD * esize};
  const CUtensorMapDataType tdt = e4m3              ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                  : dtype == CB_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                     : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUtensorMap mk, mv;
  int rc = make_tma_map_nd(&mk, k_cache, contig ? 4 : 3, dims, strides, esize, tdt, kTile);
  if (!rc) rc = make_tma_map_nd(&mv, v_cache, contig ? 4 : 3, dims, strides, esize, tdt, kTile);
  if (rc) return rc;

  if (k_new) {                                              // the sq new k / v rows first
    const PagedAppend kc{k_cache, k_new, k_new_sb * 2, k_new_st * 2}, vc{v_cache, v_new, v_new_sb * 2, v_new_st * 2};
    if (contig)
      launch_contiguous_append(kc, vc, (int64_t)Hkv * kD * 2, cache_seqlens, nullptr, rows_sb, cache_rows, B, sq, st);
    else if (e4m3)
      launch_paged_append_e4m3(kc, vc, Hkv * kD, dtype, cache_seqlens, nullptr, block_table, bt_stride, B, sq,
                               page_size, st);
    else                                                    // true page indexing
      launch_paged_append(kc, vc, (int64_t)Hkv * kD * 2, cache_seqlens, nullptr, block_table, bt_stride, B, sq,
                          page_size, page_size, st);
    CB_LAUNCHED_AS(name, 1);
  }

  const int smem = 1024 + kSmemBytes;
  const dim3 grid(row_tiles * splits, Hkv, B), block(kThreads);
  const int appended = k_new ? 1 : 0;
  causal = causal ? 1 : 0;
  rc = dispatch_io_g(dtype, G, [&](auto t, auto g) {
    using T = decltype(t);
    constexpr int GG = decltype(g)::value;
    const T* qt = (const T*)q;
    float *op = part.o_part, *lse = part.lse;
    if (contig)
      return launch_smem<gqa_prefill_contig_kernel<T, GG>>(entry, grid, block, smem, st, mk, mv, qt, cache_seqlens, sq,
                                                           Hq, Hkv, appended, causal, softmax_scale, row_tiles, splits,
                                                           op, lse, (T*)out);
    if (e4m3)
      return launch_smem<gqa_prefill_e4m3_kernel<T, GG>>(entry, grid, block, smem, st, mk, mv, qt, cache_seqlens,
                                                         block_table, bt_stride, sq, Hq, Hkv, page_size, appended,
                                                         causal, softmax_scale, row_tiles, splits, op, lse, (T*)out);
    return launch_smem<gqa_prefill_kernel<T, GG>>(entry, grid, block, smem, st, mk, mv, qt, cache_seqlens, block_table,
                                                  bt_stride, sq, Hq, Hkv, page_size, appended, causal, softmax_scale,
                                                  row_tiles, splits, op, lse, (T*)out);
  });
  if (rc) return rc;
  CB_LAUNCHED_AS(name, 1);
  if (splits > 1) {
    rc = launch_merge_splits(part.o_part, part.lse, out, B * sq * Hq, splits, kD, dtype, st);
    if (rc) return rc;
    CB_LAUNCHED_AS(name, 1);
  }
  return 0;
}

}  // namespace cb

// flash_attn_with_kvcache (paged) with seqlen_q >= 1 (include/chitu_b200.h).
extern "C" int chitu_b200_gqa_paged_prefill(const void* q, void* k_cache, void* v_cache, const void* k_new,
                                            const void* v_new, int64_t k_new_sb, int64_t k_new_st, int64_t v_new_sb,
                                            int64_t v_new_st, const int32_t* cache_seqlens, const int32_t* block_table,
                                            int bt_stride, int B, int sq, int Hq, int Hkv, int D, int page_size,
                                            int num_blocks, int max_seqlen_hint, int causal, float softmax_scale,
                                            void* out, void* workspace, int64_t workspace_bytes, int dtype,
                                            void* stream) {
  using namespace cb;
  if (int rc = check_gqa_operands(__func__, q, k_cache, v_cache, cache_seqlens, out, k_new, v_new, k_new_sb, k_new_st,
                                  v_new_sb, v_new_st, true, dtype))
    return rc;
  CB_ARG(block_table);
  CB_ARG(B >= 0 && B <= 65535 && sq >= 1 && Hq > 0 && Hkv > 0 && Hkv <= 65535 && Hq % Hkv == 0);
  CB_ARG(bt_stride > 0 && num_blocks > 0);
  CB_ARG(D == kD);
  CB_ARG(page_size > 0 && page_size % kTile == 0 && (int64_t)num_blocks * page_size <= INT_MAX);
  const int G = Hq / Hkv;
  CB_ARG(G == 1 || G == 2 || G == 4 || G == 8);
  CB_ARG((int64_t)sq * Hq <= INT_MAX / kD);
  CB_ARG(workspace == nullptr || (uintptr_t)workspace % 16 == 0);
  if (B == 0) return 0;
  const int max_len = max_seqlen_hint > 0 ? max_seqlen_hint : bt_stride * page_size;
  return gqa_prefill(__func__, __func__, KvLayout::kPaged, q, k_cache, v_cache, k_new, v_new, k_new_sb, k_new_st,
                     v_new_sb, v_new_st, cache_seqlens, block_table, bt_stride, page_size, num_blocks, 0, 0, B, sq, Hq,
                     Hkv, max_len, causal, softmax_scale, out, workspace, workspace_bytes, dtype, (cudaStream_t)stream);
}

CB_DEFINE_TL_SETTER(gqa_prefill)
