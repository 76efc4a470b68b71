// Absorbed-MLA paged decode on the Hopper tensor cores (sm_90a): wgmma + TMA + mbarrier.
//
// Replaces third_party/FlashMLA (flash_api.cpp:73-75) and triton_decode_attention.py:20-290 behind
// AttnBackend.mla_attn_with_kvcache (attn_backend.py:536-572 / 707-774).  Same arithmetic as the reference:
// scores = (q_nope.k_c + q_pe.k_pe) * scale in fp32, softmax in fp32, P rounded to bf16 before P.V
// (triton_decode_attention.py:113), V = the first 512 columns of the SAME cache row, split-KV partials merged by LSE.
//
// Mapping (one CTA per (KV split, 16-head group, request), 1 CTA / SM, 5 warps):
//   both products are SWAPPED so that the 16 local heads (tp = 8) are the wgmma N dimension:
//     S^T[64 keys x 16 heads]  = K[64 x 576] . Q^T       A = staged K chunk, K-major (wgmma M = 64 = one page)
//     O^T[512 dims x 16 heads] += V^T[512 x 64] . P^T     A = the SAME staged chunks read MN-major (dims contiguous),
//                                                         8 M tiles of 64 dims, B = P[16 heads x 64 keys] K-major
//   so a cache row is read from HBM exactly once and the tensor pipe does 36 + 32 tiny MMAs per 64-key page.
//   warp 4   TMA producer: one page = 9 boxes [64 keys x 128 B] (128B swizzle); the 8 latent chunks go through a ring of
//            22 x 8 KB slots (2.75 pages in flight), the rope chunk through its own 3-slot ring (it is released right
//            after Q.K^T).  KV streaming starts BEFORE griddepcontrol.wait: cache rows are only written by earlier decode
//            steps and by this kernel, so the stream overlaps the tail of the previous kernel (PDL).
//   warps 0-3 one warpgroup: Q.K^T (S^T in registers: 2 keys x 4 heads per thread), softmax, P -> shared memory, P.V
//            (O^T in registers: 8 tiles x 2 dims x 4 heads per thread).  Per-head running max across the 64 keys by
//            shuffles + one shared-memory exchange between the 4 warps; O^T is only rescaled when a head's max moved
//            by more than 2^8 (the exact result is recovered at the end: P, l and O share the same reference max).
#include <cuda.h>

#include "common.cuh"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace cb {
namespace {

constexpr int kC = 512, kR = 64, kRow = kC + kR;
constexpr int kTile = 64;                      // keys per tile == page size
constexpr int kSlot = kTile * 128;             // 8 KB: one TMA box [64 keys x 128 B]
constexpr int kNSM = 22;                       // main ring slots
constexpr int kNSR = 3;                        // rope ring slots
constexpr int kQBytes = 9 * 16 * 128;          // Q as 9 K-major chunks of [16 heads x 128 B]
constexpr int kPBytes = 16 * 128;              // P as [16 heads x 64 keys] bf16, K-major
constexpr int kSmemBytes = kNSM * kSlot + kNSR * kSlot + kQBytes + 2 * kPBytes;
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kRescaleThreshold = 8.f;       // log2 domain
constexpr int kThreads = 160;                  // warpgroup (warps 0-3) + producer warp

__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// byte offset of the 16-byte unit `unit` of row `row` in a [rows x 128 B] 128B-swizzled tile
__device__ __forceinline__ uint32_t sw128(int row, int unit) { return (uint32_t)(row * 128 + ((unit ^ (row & 7)) << 4)); }

// dev tool (profiling build only, -DCB_TIMELINE): %globaltimer at fixed points of every CTA, 32 slots per CTA, read by
// scripts/mla_probe.py.  The product library compiles these to nothing.
#ifdef CB_TIMELINE
static __device__ unsigned long long* d_mla_probe = nullptr;
__device__ __forceinline__ void probe(int idx) {
  unsigned long long* b = d_mla_probe;
  if (b != nullptr) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    b[(((int64_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * 32 + idx] = t;
  }
}
#else
__device__ __forceinline__ void probe(int) {}
#endif

// max / sum over the 8 lanes that share lane % 4 (the key rows of one wgmma fragment column)
__device__ __forceinline__ float rows_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 4));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 8));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 16));
}
__device__ __forceinline__ float rows_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 8);
  return v + __shfl_xor_sync(0xffffffffu, v, 16);
}
// value h of a 16-entry register array without dynamic register indexing
__device__ __forceinline__ float pick16(const float (&v)[16], int h) {
  float r = v[0];
#pragma unroll
  for (int i = 1; i < 16; ++i) r = (h == i) ? v[i] : r;
  return r;
}

__global__ void __launch_bounds__(kThreads, 1) mla_decode_tc_kernel(
    const __grid_constant__ CUtensorMap map_kv, const __nv_bfloat16* __restrict__ q_nope,
    const __nv_bfloat16* __restrict__ q_pe, __nv_bfloat16* __restrict__ kv_cache,
    const __nv_bfloat16* __restrict__ new_kv, const int32_t* __restrict__ seqlens_excl,
    const int32_t* __restrict__ block_table, int bt_stride, int H, float scale, int num_splits,
    float* __restrict__ o_part, float* __restrict__ lse, __nv_bfloat16* __restrict__ out,
    const int32_t* __restrict__ plan) {
  extern __shared__ __align__(1024) uint8_t mla_tc_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(mla_tc_smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_ring = smem;                                   // [kNSM][64 keys][128 B]   latent chunks
  uint8_t* s_rope = s_ring + kNSM * kSlot;                  // [kNSR][64 keys][128 B]   rope chunk
  uint8_t* s_q = s_rope + kNSR * kSlot;                     // [9][16 heads][128 B]
  uint8_t* s_p = s_q + kQBytes;                             // [2][16 heads][128 B]
  __shared__ __align__(8) uint64_t full_m[kNSM], empty_m[kNSM], full_r[kNSR], empty_r[kNSR], raw_bar;
  __shared__ float red_max[4][16], red_sum[4][16];

  const int split = blockIdx.x, hg = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h0 = hg * 16;

  if (threadIdx.x == 0) {
    probe(0);
    for (int i = 0; i < kNSM; ++i) { mbar_init(&full_m[i], 1); mbar_init(&empty_m[i], 1); }
    for (int i = 0; i < kNSR; ++i) { mbar_init(&full_r[i], 1); mbar_init(&empty_r[i], 1); }
    mbar_init(&raw_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_kv) : "memory");
  }
  cb::pdl_launch_dependents();
  __syncthreads();

  // sequence lengths and the block table are written only by kernels that do not trigger dependents early (torch copies,
  // the decode-prepare kernel): they are stable here even before griddepcontrol.wait
  const int L_cache = seqlens_excl[b];
  const int L = L_cache + (new_kv ? 1 : 0);
  int per = (((L + num_splits - 1) / num_splits) + kTile - 1) / kTile * kTile;           // keys per split, whole pages
  // length-aware plan of chitu_b200_attn_plan (written by a kernel that does not trigger dependents early): equal-size
  // splits over a ragged batch; splits past a request's end do nothing (their LSE is -inf)
  // (only a plan made for THIS launch shape — same batch, same head count — is honoured)
  if (plan && plan[0] == 0x504c414e && plan[5] == kTile && plan[4] == (int)gridDim.z && plan[6] == H && plan[1] >= per &&
      (L + plan[1] - 1) / plan[1] <= num_splits)
    per = plan[1];
  const int begin = split * per;
  const int end = min(begin + per, L);
  const int ntiles = end > begin ? (end - begin + kTile - 1) / kTile : 0;
  const int32_t* bt = block_table + (int64_t)b * bt_stride;

  if (warp == 4) {
    // ================= TMA producer (whole warp: lane 0 issues, all lanes patch the tail page) =================
    const uint64_t pol = l2_policy_evict_first();
    uint32_t raw_phase = 0;
    bool waited = false;
    for (int it = 0; it < ntiles; ++it) {
      const int key0 = begin + it * kTile;
      const int row0 = bt[key0 / kTile] * kTile;
      const int valid_rows = min(kTile, L - key0);                         // rows >= valid_rows must read as zero
      const int rnew = (new_kv && L - 1 >= key0 && L - 1 < key0 + kTile) ? L - 1 - key0 : -1;
      const bool tail = valid_rows < kTile || rnew >= 0;
      const int rs = it % kNSR;
      if (!tail) {
        for (int c = 0; c < 8; ++c) {
          const int g = it * 8 + c, s = g % kNSM;
          mbar_wait(&empty_m[s], ((g / kNSM) & 1) ^ 1);
          if (lane == 0) {
            if (it == 0 && c == 0) probe(30);
            mbar_expect_tx(&full_m[s], kSlot);
            tma_load_2d(s_ring + s * kSlot, &map_kv, &full_m[s], c * 64, row0, pol);
          }
        }
        mbar_wait(&empty_r[rs], ((it / kNSR) & 1) ^ 1);
        if (lane == 0) {
          mbar_expect_tx(&full_r[rs], kSlot);
          tma_load_2d(s_rope + rs * kSlot, &map_kv, &full_r[rs], 8 * 64, row0, pol);
        }
      } else {
        // the page that holds the end of the sequence (at most one per CTA): load all nine boxes, then overwrite the row
        // of the token being appended from `new_kv` (its cache write may not have landed) and zero the rows past the end
        // (0 * garbage must not poison P.V), then publish.
        for (int c = 0; c < 8; ++c) {
          const int g = it * 8 + c, s = g % kNSM;
          mbar_wait(&empty_m[s], ((g / kNSM) & 1) ^ 1);
        }
        mbar_wait(&empty_r[rs], ((it / kNSR) & 1) ^ 1);
        if (lane == 0) {
          mbar_expect_tx(&raw_bar, 9 * kSlot);
          for (int c = 0; c < 8; ++c)
            tma_load_2d(s_ring + ((it * 8 + c) % kNSM) * kSlot, &map_kv, &raw_bar, c * 64, row0, pol);
          tma_load_2d(s_rope + rs * kSlot, &map_kv, &raw_bar, 8 * 64, row0, pol);
        }
        if (!waited) { cb::pdl_wait(); waited = true; }                     // new_kv is written by the previous kernel
        mbar_wait(&raw_bar, raw_phase);
        raw_phase ^= 1;
        for (int c = 0; c < 9; ++c) {
          uint8_t* dst = c < 8 ? s_ring + ((it * 8 + c) % kNSM) * kSlot : s_rope + rs * kSlot;
          if (rnew >= 0 && lane < 8)
            *reinterpret_cast<uint4*>(dst + sw128(rnew, lane)) =
                *reinterpret_cast<const uint4*>(new_kv + (int64_t)b * kRow + c * 64 + lane * 8);
          for (int i = valid_rows * 8 + lane; i < kTile * 8; i += 32)       // whole rows: the swizzle permutes within a row
            *reinterpret_cast<uint4*>(dst + (i >> 3) * 128 + ((i & 7) << 4)) = make_uint4(0, 0, 0, 0);
        }
        fence_async_smem();
        __syncwarp();
        if (lane == 0) {
          for (int c = 0; c < 8; ++c) mbar_arrive(&full_m[(it * 8 + c) % kNSM]);
          mbar_arrive(&full_r[rs]);
        }
      }
    }
  } else {
    // ================= warpgroup: Q.K^T, softmax, P.V, epilogue =================
    const int t = threadIdx.x;                               // 0..127
    const int krow = warp * 16 + (lane >> 2);                // fragment rows krow, krow + 8: keys of S^T, dims of O^T tiles
    const int hc = 2 * (lane & 3);                           // fragment columns hc + 8 nb + j: heads
    // ---- Q -> shared memory (K-major, swizzled); rows >= H are zero ----
    cb::pdl_wait();
    cb::tl_stamp();
    if (t == 0) probe(1);
    {
      // 16 heads x 72 units of 16 B = 9 units per thread: all nine global loads are issued before the first shared-memory
      // store
      uint4 v[9];
#pragma unroll
      for (int j = 0; j < 9; ++j) {
        const int i = j * 128 + t;
        const int h = i / 72, u = i - h * 72;
        const int c = u >> 3, uu = u & 7;                    // chunk (64 elements), unit within the 128 B row
        v[j] = make_uint4(0, 0, 0, 0);
        if (h0 + h < H) {
          if (c < 8) v[j] = *reinterpret_cast<const uint4*>(q_nope + ((int64_t)b * H + h0 + h) * kC + c * 64 + uu * 8);
          else v[j] = *reinterpret_cast<const uint4*>(q_pe + ((int64_t)b * H + h0 + h) * kR + uu * 8);
        }
      }
#pragma unroll
      for (int j = 0; j < 9; ++j) {
        const int i = j * 128 + t;
        const int h = i / 72, u = i - h * 72;
        *reinterpret_cast<uint4*>(s_q + (u >> 3) * 2048 + sw128(h, u & 7)) = v[j];
      }
    }
    fence_async_smem();
    asm volatile("bar.sync 1, 128;" ::: "memory");
    if (t == 0) probe(2);
    if (new_kv && split == 0 && hg == 0) {                   // append for the following steps (ops.py:50-91)
      const int page = bt[L_cache / kTile];
      __nv_bfloat16* dst = kv_cache + ((int64_t)page * kTile + L_cache % kTile) * kRow;
      const __nv_bfloat16* src = new_kv + (int64_t)b * kRow;
      for (int i = t; i < kRow / 8; i += 128) reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
    }

    const uint32_t ring_a = smem_u32(s_ring), rope_a = smem_u32(s_rope), q_a = smem_u32(s_q), p_a = smem_u32(s_p);
    const float sc = scale * kLog2e;
    float m_run[16];                                         // identical in every thread
    float l_part[4];                                         // this thread's keys, heads hc + 8 (e >> 1) + (e & 1)
    float o[8][8];                                           // O^T tile m: dims 64 m + krow (+8), heads as S^T
#pragma unroll
    for (int h = 0; h < 16; ++h) m_run[h] = -INFINITY;
#pragma unroll
    for (int i = 0; i < 4; ++i) l_part[i] = 0.f;
#pragma unroll
    for (int m = 0; m < 8; ++m)
#pragma unroll
      for (int e = 0; e < 8; ++e) o[m][e] = 0.f;

    for (int it = 0; it < ntiles; ++it) {
      // ---- S^T = K . Q^T over the 8 latent chunks and the rope chunk ----
      float s[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) s[e] = 0.f;
      wgmma_fence();
      for (int c = 0; c < 8; ++c) {
        const int g = it * 8 + c, sl = g % kNSM;
        mbar_wait(&full_m[sl], (g / kNSM) & 1);
#pragma unroll
        for (int k = 0; k < 4; ++k)
          WgmmaN<16>::bf16<0>(s, make_sw128_desc(ring_a + sl * kSlot + 32 * k, 16, 1024),
                              make_sw128_desc(q_a + c * 2048 + 32 * k, 16, 1024), (c | k) != 0);
      }
      const int rs = it % kNSR;
      mbar_wait(&full_r[rs], (it / kNSR) & 1);
#pragma unroll
      for (int k = 0; k < 4; ++k)
        WgmmaN<16>::bf16<0>(s, make_sw128_desc(rope_a + rs * kSlot + 32 * k, 16, 1024),
                            make_sw128_desc(q_a + 8 * 2048 + 32 * k, 16, 1024), 1);
      wgmma_commit();
      wgmma_wait<0>();
      if (t == 0) {
        mbar_arrive(&empty_r[rs]);                           // the rope chunk is not needed by P.V
        if (it < 12) probe(3 + 2 * it);
      }

      // ---- per-head tile maximum over the 64 keys (finite: every tile has a valid key) ----
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const bool valid = begin + it * kTile + krow + 8 * ((e >> 1) & 1) < end;
        s[e] = valid ? s[e] * sc : -INFINITY;
      }
#pragma unroll
      for (int x = 0; x < 4; ++x) {                          // x = 2 nb + j
        const int e = 4 * (x >> 1) + (x & 1);
        const float mx = rows_max(fmaxf(s[e], s[e + 2]));
        if (lane < 4) red_max[warp][hc + 8 * (x >> 1) + (x & 1)] = mx;
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");
      // rescale only when some head moved by > 2^8
      float mt[16];
      bool need = false;
#pragma unroll
      for (int h = 0; h < 16; ++h) {
        mt[h] = fmaxf(fmaxf(red_max[0][h], red_max[1][h]), fmaxf(red_max[2][h], red_max[3][h]));
        need |= mt[h] > m_run[h] + kRescaleThreshold;
      }
      float alpha[16];
      if (need) {
#pragma unroll
        for (int h = 0; h < 16; ++h) {
          const float mn = fmaxf(m_run[h], mt[h]);
          alpha[h] = exp2f(m_run[h] - mn);                   // 0 on the first tile (m_run = -inf)
          m_run[h] = mn;
        }
      }
      // ---- P = exp2(S - m) -> bf16 -> shared memory as P[head][key] (K-major, swizzled) ----
      uint8_t* pb = s_p + (it & 1) * kPBytes;
#pragma unroll
      for (int x = 0; x < 4; ++x) {
        const int h = hc + 8 * (x >> 1) + (x & 1);
        const float mr = pick16(m_run, h);
        const int e = 4 * (x >> 1) + (x & 1);
        const float p0 = exp2f(s[e] - mr), p1 = exp2f(s[e + 2] - mr);       // 0 for masked keys
        l_part[x] = (need ? l_part[x] * pick16(alpha, h) : l_part[x]) + p0 + p1;
        *reinterpret_cast<__nv_bfloat16*>(pb + sw128(h, krow >> 3) + (krow & 7) * 2) = __float2bfloat16_rn(p0);
        *reinterpret_cast<__nv_bfloat16*>(pb + sw128(h, (krow + 8) >> 3) + (krow & 7) * 2) = __float2bfloat16_rn(p1);
      }
      if (need && it > 0) {
        float al[4];
#pragma unroll
        for (int x = 0; x < 4; ++x) al[x] = pick16(alpha, hc + 8 * (x >> 1) + (x & 1));
#pragma unroll
        for (int m = 0; m < 8; ++m)
#pragma unroll
          for (int e = 0; e < 8; ++e) o[m][e] *= al[2 * (e >> 2) + (e & 1)];
      }
      fence_async_smem();
      asm volatile("bar.sync 1, 128;" ::: "memory");          // P complete; red_max free for the next tile
      if (t == 0 && it < 12) probe(4 + 2 * it);

      // ---- O^T += V^T . P^T: the 8 latent chunks of the page, each a 64-dim M tile read MN-major ----
      wgmma_fence();
#pragma unroll
      for (int m = 0; m < 8; ++m) {
        const int sl = (it * 8 + m) % kNSM;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)                       // 16 keys = two 8-row groups of the chunk
          WgmmaN<16>::bf16<1>(o[m], make_sw128_desc(ring_a + sl * kSlot + ks * 2048, kSlot, 1024),
                              make_sw128_desc(p_a + (it & 1) * kPBytes + 32 * ks, 16, 1024), 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
      if (t == 0)
        for (int m = 0; m < 8; ++m) mbar_arrive(&empty_m[(it * 8 + m) % kNSM]);
    }

    // ---- epilogue: row sums across the 64 keys, O^T / l -> out (one split) or normalised partial + log2-sum-exp ----
#pragma unroll
    for (int x = 0; x < 4; ++x) {
      const float ls = rows_sum(l_part[x]);
      if (lane < 4) red_sum[warp][hc + 8 * (x >> 1) + (x & 1)] = ls;
    }
    if (t == 0) probe(28);
    asm volatile("bar.sync 1, 128;" ::: "memory");
    const bool direct = num_splits == 1 && out != nullptr;   // out == NULL: partials even for one split (deferred merge)
    float inv[4];
#pragma unroll
    for (int x = 0; x < 4; ++x) {
      const int h = hc + 8 * (x >> 1) + (x & 1);
      const float l = (red_sum[0][h] + red_sum[1][h]) + (red_sum[2][h] + red_sum[3][h]);
      inv[x] = (ntiles > 0 && l > 0.f) ? 1.f / l : 0.f;
    }
#pragma unroll
    for (int m = 0; m < 8; ++m) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int x = 2 * (e >> 2) + (e & 1);
        const int h = hc + 8 * (x >> 1) + (x & 1);
        const int dim = m * 64 + krow + 8 * ((e >> 1) & 1);
        if (h0 + h >= H) continue;
        const float v = o[m][e] * inv[x];
        if (direct) out[((int64_t)b * H + h0 + h) * kC + dim] = __float2bfloat16_rn(v);
        else o_part[(((int64_t)b * H + h0 + h) * num_splits + split) * kC + dim] = v;
      }
    }
    if (!direct && t < 16 && h0 + t < H) {
      const float l = (red_sum[0][t] + red_sum[1][t]) + (red_sum[2][t] + red_sum[3][t]);
      lse[((int64_t)b * H + h0 + t) * num_splits + split] = (ntiles > 0 && l > 0.f) ? pick16(m_run, t) + log2f(l) : -INFINITY;
    }
    if (t == 0) probe(29);
  }
}

}  // namespace

// q_nope [B,H,512], q_pe [B,H,64], kv_cache [num_blocks,64,576] bf16; new_kv [B,576] or null; seqlens_excl [B] int32;
// block_table [B, bt_stride] int32.  num_splits == 1: out [B,H,512] bf16; else o_part [B,H,splits,512] fp32 (normalised)
// and lse [B,H,splits] (log2 domain) — the layout merge_splits_kernel / the merging absorb-o kernel consume.
int mla_decode_tc_launch(const void* q_nope, const void* q_pe, void* kv_cache, const void* new_kv,
                         const int32_t* seqlens_excl, const int32_t* block_table, int bt_stride, int B, int H,
                         int num_blocks, int num_splits, float scale, void* out, float* o_part, float* lse,
                         const int32_t* plan, cudaStream_t st) {
  CUtensorMap map;
  // the cache as a 2-D [num_rows, 576] bf16 tensor, box = [64 rows x 64 elements (128 B)]
  int rc = make_tma_map_2d(&map, kv_cache, (int64_t)num_blocks * kTile, kRow, 2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, kTile);
  if (rc) return rc;
  const size_t smem = 1024 + (size_t)kSmemBytes;
  static bool attr = false;
  if (!attr) {
    CB_CUDA(cudaFuncSetAttribute(mla_decode_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = true;
  }
  dim3 grid(num_splits, cdiv(H, 16), B);
  launch_k(mla_decode_tc_kernel, grid, dim3(kThreads), smem, st, map, (const __nv_bfloat16*)q_nope,
           (const __nv_bfloat16*)q_pe, (__nv_bfloat16*)kv_cache, (const __nv_bfloat16*)new_kv, seqlens_excl, block_table,
           bt_stride, H, scale, num_splits, o_part, lse, (__nv_bfloat16*)out, plan);
  CB_LAUNCHED(1);
  return 0;
}

}  // namespace cb

CB_DEFINE_TL_SETTER(mla_tc)
#ifdef CB_TIMELINE
extern "C" int chitu_b200_debug_mla_probe(unsigned long long* p) {      // p: uint64 [CTAs * 32], zero-filled; NULL disarms
  return (int)cudaMemcpyToSymbol(cb::d_mla_probe, &p, sizeof(p));
}
#endif
