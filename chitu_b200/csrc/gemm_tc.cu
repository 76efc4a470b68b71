// wgmma + TMA weight-streaming skinny GEMM for decode linears (sm_90a).
//
//   y[M,N] = x[M,K] · W[N,K]^T        M = decode tokens (1..256), N x K = nn.Linear weight
//
// Swap-AB mapping (SURVEY §7.3-1): the WEIGHT tile is the wgmma "A" operand (128 rows = two warpgroups of M = 64), the
// tokens are the wgmma "N" dimension (BN = 16/32/64/128), so one 128 B stage row of K consumes 16 KB of weights however
// small the batch is; the tensor pipe is mostly idle and the kernel is a pure HBM stream:
//   warps 0-7: two consumer warpgroups — warpgroup g multiplies weight rows [64 g, 64 g + 64) of the tile with the
//              tokens, accumulators in registers (BN / 2 per thread), then runs the epilogue for its rows.
//              FP8: every 128-K block is multiplied into a fresh accumulator and added with a_s[m,kb]*b_s[n/128,kb]
//              applied to the fp32 partial product exactly as the reference does (triton_kernels.py:357);
//              bf16 / int8: one accumulator per work item.
//   warp 8   : TMA producer — cp.async.bulk.tensor.2d, 128B-swizzled boxes W[128 rows x 128 B] and X[BN rows x 128 B]
//              into an S-stage shared-memory ring (mbarrier full/empty), weights with an L2 evict-first policy (read
//              exactly once), activations evict-last.
//   soft fp8 : 8 more warps convert each fp8 weight stage to bf16 for the bf16 MMA.
// Split-K fills the SMs when N/128 tiles are too few: fp32 (int32) partials go to a workspace, the last CTA of a tile
// half (atomic ticket) reduces them in split order -> deterministic.
//
// Reference semantics implemented here:
//   kind 0: F.linear bf16/fp16 (+bias fp32-joined, +residual as a separate rounding)
//   kind 1: fp8_gemm_deepseek_v3 (ops.py:452-483, triton_kernels.py:303-365)
//   kind 2: w8a8gemm.mm / w8a8gemv.mv (quantize/w8a8.py:105,120,125)
#include <cuda.h>

#include <stdlib.h>

#include <mutex>
#include <type_traits>

#include "common.cuh"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace cb {

namespace {

enum { KIND_16 = 0, KIND_FP8 = 1, KIND_I8 = 2, KIND_SOFT = 3 };   // SOFT: fp8 weights -> bf16 in shared memory, bf16 MMA

constexpr int kTileN = 128;        // weight rows per CTA tile (two wgmma M = 64 halves)
constexpr int kStageRowBytes = 128;  // bytes of K per stage row (one 128B swizzle atom)
constexpr int kMmaThreads = 256;   // two consumer warpgroups; the producer warp and the converter warps follow
constexpr int kGeomCache = 256;   // grouped mode: tiles whose geometry a CTA stages in shared memory

__device__ __forceinline__ uint64_t make_kmajor_sw128_desc(uint32_t smem_addr) { return make_sw128_desc(smem_addr, 16, 1024); }

// ---------------------------------------------------------------------------------------------
// Persistent stream-K schedule.  The global work list is the sequence of pipeline stages
//   g = tile * S + s        (tile = m_chunk * n_tiles + n_tile, S = stages per tile)
// split into gridDim.x equal contiguous ranges, one per CTA (one CTA per SM).  A CTA therefore
// streams a contiguous run of weight bytes, its TMA ring never drains between tiles, and all
// SMs finish within one stage of each other.  A tile whose stages are shared by several CTAs is
// reduced through fp32 (int32) partials: contributor `ord` writes partial[tile][ord], takes a
// ticket, the last one sums ords 0..count-1 in order (deterministic) and writes the output.
// ---------------------------------------------------------------------------------------------
struct Params {
  int M, N, K;              // tokens, out features, reduction (elements)
  int S;                    // stages per tile = ceil(K * elem / 128)
  int n_tiles, m_chunks;
  int per;                  // stages per CTA (dense mode; grouped mode derives it on the device)
  int kblocks;              // fp8: ceil(K/128) (scale columns)
  int out_dtype;            // CB_BF16 | CB_F16
  int prefetch;             // dense mode: stream weight tiles before griddepcontrol.wait (A/B: CHITU_B200_GEMM_PREFETCH=0)
  int act_pairs;            // kind 0: weight rows (2i, 2i+1) = (gate_i, up_i); out[m, i] = SiluAndMul -> [M, N/2]
  int has_push;             // row-parallel linear of a tensor-parallel layer: the bf16 result is stored into every rank's
  PushDev push;             // push area instead of `out`, as epoch-tagged words (comm.cu allreduce_consume_kernel)
  const float* a_s;         // fp8: [M, kblocks]         i8: a_scales [M]
  const float* b_s;         // fp8: [ceil(N/128), kblocks] i8: b_scales [N]
  const void* bias;         // [N] (io dtype; i8: fp16) or null
  const void* residual;     // [M, N] io dtype or null (kind 0 only)
  void* out;                // [M, N]
  float* partial;           // [gridDim.x][2 slots][BN][128] fp32 (int32 bits for i8): a CTA has at most
                            // two partially covered tiles (its first and its last work item)
  int* tickets;             // [tiles][2 halves], zero on entry, zero on exit
  // ---- grouped (MoE experts) mode: the tile list lives in device memory (g_num_tiles != null) ----
  const int* g_num_tiles;   // number of active (expert, n-tile) tiles
  const int* g_tile_wrow;   // [tiles] first weight row of the tile in the stacked [E*Ng, K] matrix
  const int* g_tile_xrow;   // [tiles] first (expert-sorted) activation row of the tile's expert
  const int* g_tile_cnt;    // [tiles] tokens routed to the tile's expert (<= BN)
  int g_ncols;              // Ng = output features per expert (row stride of the sorted output)
  const float* g_row_scale; // [rows] routed weight per sorted row (GEMM2, fused_moe.py:290-292) or null
  const int* g_out_rows;    // [rows] output row of sorted row r (the reference writes C.view(-1,N)[sorted_ids[r]],
                            // fused_moe.py:296-306), negative = padding row: nothing is written; null = r itself
};

template <int KIND, int BN>
struct Cfg {
  static constexpr bool kSoft = KIND == KIND_SOFT;
  static constexpr int kStageW = kTileN * kStageRowBytes;                     // 16 KB
  // soft fp8: a stage is 128 K-elements = 128 B of fp8 weights per row but 256 B of bf16 activations (two swizzle atoms)
  static constexpr int kStageX = BN * kStageRowBytes * (kSoft ? 2 : 1);
  static constexpr int kStageBytes = kStageW + kStageX;
  // soft fp8: ring of converted (bf16) weight tiles, [2 atoms][128 rows][128 B] each, between the converter warps and
  // the MMA warpgroups
  static constexpr int kCvtStages = kSoft ? 3 : 0;
  static constexpr int kCvtBytes = 2 * kTileN * kStageRowBytes;               // 32 KB
  // 3 converter warps: with the producer warp they fill a third warpgroup, so the block stays at 384 threads (registers
  // are budgeted per 128 threads; more converter threads would cut every consumer thread to 128 registers)
  static constexpr int kCvtThreads = kSoft ? 96 : 0;
  static constexpr int kCvtRing = kSoft ? kCvtStages : 1;                     // modulus of the converter ring
  // one CTA per SM with the deepest ring that fits
  static constexpr int kBudget = 200 * 1024 - kCvtStages * kCvtBytes;
  static constexpr int kStages = (kBudget / kStageBytes) > 10 ? 10 : (kBudget / kStageBytes);
  static constexpr int kProducerWarp = kMmaThreads / 32;
  static constexpr int kCvtWarp0 = kProducerWarp + 1;                         // first converter warp
  static constexpr int kThreads = kMmaThreads + 32 + kCvtThreads;
};

struct WorkItem {
  int tile, s_lo, s_hi;
};
// Work items of a CTA whose global stage range is [g_begin, g_end): only the first item can start inside a
// tile, every later one starts at a tile boundary (one division per CTA, none per item).
struct ItemIter {
  int g, g_end, S, tile, s_lo;
  __device__ __forceinline__ ItemIter(int g_begin, int g_end_, int S_) : g(g_begin), g_end(g_end_), S(S_) {
    tile = g_begin / S_;
    s_lo = g_begin - tile * S_;
  }
  __device__ __forceinline__ bool valid() const { return g < g_end; }
  __device__ __forceinline__ WorkItem item() const {
    WorkItem w;
    w.tile = tile;
    w.s_lo = s_lo;
    w.s_hi = min(S, s_lo + (g_end - g));
    return w;
  }
  __device__ __forceinline__ void next() {
    g += min(S, s_lo + (g_end - g)) - s_lo;
    ++tile;
    s_lo = 0;
  }
};

// Epilogue variants are separate instantiations: folding SiluAndMul / the NVLink push into the plain kernel as run-time
// branches grows the code of every dense GEMM.
enum { EPI_PLAIN = 0, EPI_PAIRS = 1, EPI_PUSH = 2, EPI_ROWS = 3 };   // ROWS: Params::g_out_rows (grouped mode only)

// one 128 B K slice of a stage: D[64 weight rows x BN tokens] (+)= W[64 x K] . X[BN x K]^T
// (KIND_16 multiplies fp16 operands when `f16`, bf16 otherwise)
template <int KIND, int BN, typename Acc>
__device__ __forceinline__ void mma_k(Acc (&d)[BN / 2], uint64_t a, uint64_t b, int accumulate, bool f16) {
  if constexpr (KIND == KIND_FP8) WgmmaN<BN>::e4m3(d, a, b, accumulate);
  else if constexpr (KIND == KIND_I8) WgmmaN<BN>::s8(d, a, b, accumulate);
  else if constexpr (KIND == KIND_SOFT) WgmmaN<BN>::template bf16<0>(d, a, b, accumulate);
  else if (f16) WgmmaN<BN>::template f16<0>(d, a, b, accumulate);
  else WgmmaN<BN>::template bf16<0>(d, a, b, accumulate);
}

template <int KIND, int BN, int EPI>
__global__ void __launch_bounds__((Cfg<KIND, BN>::kThreads), 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_x, const Params p) {
  using C = Cfg<KIND, BN>;
  using Acc = typename std::conditional<KIND == KIND_I8, int32_t, float>::type;
  constexpr bool kPairs = EPI == EPI_PAIRS;       // Params::act_pairs
  constexpr bool kPush = EPI == EPI_PUSH;         // Params::has_push
  constexpr int NR = BN / 2;                      // accumulators per thread
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // dynamic smem base is only guaranteed 16 B aligned: round up to the 1024 B the swizzle needs
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_w = smem;
  uint8_t* smem_x = smem + C::kStages * C::kStageW;
  uint8_t* smem_c = smem_x + C::kStages * C::kStageX;          // soft fp8: converted weight tiles
  __shared__ __align__(8) uint64_t full_bar[C::kStages], empty_bar[C::kStages];
  __shared__ __align__(8) uint64_t cvt_full[C::kSoft ? C::kCvtStages : 1], cvt_empty[C::kSoft ? C::kCvtStages : 1];
  __shared__ int s_is_last[2];
  __shared__ int4 s_geom[kGeomCache];             // grouped mode: {wrow, xrow, cnt, out col} of this CTA's first tiles

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = p.S;
  const bool grouped = p.g_num_tiles != nullptr;
  int total, per;
  if (grouped) {
    pdl_wait();                                   // the tile list is produced by the previous kernel
    total = *p.g_num_tiles * S;
    per = (total + (int)gridDim.x - 1) / (int)gridDim.x;
    if (per < 4) per = 4;                         // >= 64 KB of weights per CTA
    if (per * 8 < S) per = (S + 7) / 8;           // <= 8 CTAs per tile
    if (S * 4 <= per) per = (per + S - 1) / S * S;  // short reductions: whole tiles only, no fix-up traffic
  } else {
    total = p.n_tiles * p.m_chunks * S;
    per = p.per;
  }
  const int g_begin = min((int)blockIdx.x * per, total);
  const int g_end = min(g_begin + per, total);
  constexpr int kElemsPerStage = KIND == KIND_16 ? 64 : 128;   // K elements per pipeline stage
  // grouped mode: the tile geometry lives in device memory; reading it per tile puts an L2 round trip in front of every
  // tile of the producer and of the epilogue (the K = 256 down projection's tiles are only two stages long).  Stage this
  // CTA's share once.
  const int geom_t0 = g_begin / S;
  if (grouped && g_end > g_begin) {
    const int nt = min((g_end - 1) / S - geom_t0 + 1, kGeomCache);
    for (int i = threadIdx.x; i < nt; i += C::kThreads)
      s_geom[i] = make_int4(p.g_tile_wrow[geom_t0 + i], p.g_tile_xrow[geom_t0 + i], p.g_tile_cnt[geom_t0 + i],
                            p.g_tile_wrow[geom_t0 + i] % p.g_ncols);
  }
  auto geom = [&](int tile) -> int4 {
    const int i = tile - geom_t0;
    if (i < kGeomCache) return s_geom[i];
    return make_int4(p.g_tile_wrow[tile], p.g_tile_xrow[tile], p.g_tile_cnt[tile], p.g_tile_wrow[tile] % p.g_ncols);
  };

  if (threadIdx.x == 0) {
    for (int i = 0; i < C::kStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 2); }
    if (C::kSoft)
      for (int i = 0; i < C::kCvtStages; ++i) { mbar_init(&cvt_full[i], 1); mbar_init(&cvt_empty[i], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp == C::kProducerWarp && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_x) : "memory");
  }
  pdl_launch_dependents();
  __syncthreads();
  // everything above (barrier init, tensormap prefetch) overlapped the previous kernel's tail.  The WEIGHTS are never
  // written by a preceding kernel, so the producer also starts streaming them now — up to the whole ring (10 x 16 KB per
  // SM) is in flight or landed before the activations exist; everything else waits here for the previous kernel to
  // complete and flush.
  if (warp == C::kProducerWarp) {
    // ================= TMA producer =================
    if (elect_one()) {
      const uint64_t pol_w = l2_policy_evict_first(), pol_x = l2_policy_evict_last();
      int pre = 0;                                  // stages whose weight tile was issued before griddepcontrol.wait
      if (!grouped && p.prefetch) {
        int it = 0;
        for (ItemIter ii(g_begin, g_end, S); ii.valid() && it < C::kStages; ii.next()) {
          const WorkItem w = ii.item();
          const int n0 = (w.tile % p.n_tiles) * kTileN;
          for (int st = w.s_lo; st < w.s_hi && it < C::kStages; ++st, ++it) {
            mbar_expect_tx_only(&full_bar[it], C::kStageW);        // first ring pass: every slot is free
            tma_load_2d(smem_w + it * C::kStageW, &map_w, &full_bar[it], st * kElemsPerStage, n0, pol_w);
          }
        }
        pre = it;
      }
      pdl_wait();
      int it = 0;
      for (ItemIter ii(g_begin, g_end, S); ii.valid(); ii.next()) {
        const WorkItem w = ii.item();
        int n0, m0;
        if (grouped) { const int4 ge = geom(w.tile); n0 = ge.x; m0 = ge.y; }
        else { n0 = (w.tile % p.n_tiles) * kTileN; m0 = (w.tile / p.n_tiles) * BN; }
        for (int st = w.s_lo; st < w.s_hi; ++st, ++it) {
          const int s = it % C::kStages;
          const uint32_t ph = (it / C::kStages) & 1;
          const int kc = st * kElemsPerStage;
          if (it < pre) {
            mbar_expect_tx(&full_bar[s], C::kStageX);              // the arrival of the phase; weights already issued
          } else {
            mbar_wait(&empty_bar[s], ph ^ 1);
            mbar_expect_tx(&full_bar[s], C::kStageBytes);
            tma_load_2d(smem_w + s * C::kStageW, &map_w, &full_bar[s], kc, n0, pol_w);
          }
          tma_load_2d(smem_x + s * C::kStageX, &map_x, &full_bar[s], kc, m0, pol_x);
          if (C::kSoft)   // second 64-element atom of the bf16 activations
            tma_load_2d(smem_x + s * C::kStageX + BN * kStageRowBytes, &map_x, &full_bar[s], kc + 64, m0, pol_x);
        }
      }
    }
  } else if (C::kSoft && warp >= C::kCvtWarp0) {
    // ================= soft fp8: weight converter (3 warps) =================
    // soft_fp8_gemm_deepseek_v3 (triton_kernels.py:388-508): w_bf16 = bf16(fp8 bits as fp32 * (s * 2^120)) == the value
    // bf16(fp32(fp8) * s) for every finite fp8 weight; the stage's [128 rows x 128 B] fp8 tile (one 128x128 scale block)
    // becomes two 128B-swizzled bf16 atoms [128 rows x 64 elements], 1024 units of 16 fp8 weights.
    const int ct = threadIdx.x - C::kCvtWarp0 * 32;            // 0..95
    int it = 0;
    for (ItemIter ii(g_begin, g_end, S); ii.valid(); ii.next()) {
      const WorkItem w = ii.item();
      const int w_row0 = grouped ? geom(w.tile).x : (w.tile % p.n_tiles) * kTileN;
      const float* srow = p.b_s + (int64_t)(w_row0 / kTileN) * p.kblocks;
      float sc_next = srow[w.s_lo];
      for (int st = w.s_lo; st < w.s_hi; ++st, ++it) {
        const int s = it % C::kStages, c = it % C::kCvtRing;
        const float sc = sc_next;
        if (st + 1 < w.s_hi) sc_next = srow[st + 1];
        mbar_wait(&full_bar[s], (it / C::kStages) & 1);
        mbar_wait(&cvt_empty[c], ((it / C::kCvtRing) & 1) ^ 1);
        const uint8_t* src = smem_w + s * C::kStageW;
        uint8_t* dst = smem_c + c * C::kCvtBytes;
#pragma unroll 2
        for (int unit = ct; unit < 1024; unit += C::kCvtThreads) {   // row = unit / 8, 16 elements each
          const int r = unit >> 3, u = unit & 7;
          const uint4 v = *reinterpret_cast<const uint4*>(src + r * 128 + ((u ^ (r & 7)) << 4));
          const uint32_t vw[4] = {v.x, v.y, v.z, v.w};
          uint32_t o[8];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float2 lo = fp8x2_to_float2((uint16_t)(vw[q] & 0xffffu)), hi = fp8x2_to_float2((uint16_t)(vw[q] >> 16));
            const __nv_bfloat16* tag = nullptr;
            o[2 * q] = pack2(lo.x * sc, lo.y * sc, tag);
            o[2 * q + 1] = pack2(hi.x * sc, hi.y * sc, tag);
          }
          uint8_t* drow = dst + (u >> 2) * (kTileN * kStageRowBytes) + r * 128;
          const int du = 2 * (u & 3);
          *reinterpret_cast<uint4*>(drow + ((du ^ (r & 7)) << 4)) = make_uint4(o[0], o[1], o[2], o[3]);
          *reinterpret_cast<uint4*>(drow + (((du + 1) ^ (r & 7)) << 4)) = make_uint4(o[4], o[5], o[6], o[7]);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        asm volatile("bar.sync 5, %0;" ::"n"(C::kCvtThreads) : "memory");
        if (ct == 0) mbar_arrive(&cvt_full[c]);
      }
    }
  } else if (warp < C::kProducerWarp) {
    // ================= MMA + epilogue: consumer warpgroup `wg` owns weight rows [64 wg, 64 wg + 64) of every tile ==========
    pdl_wait();
    tl_stamp();
    const int wg = warp >> 2;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);     // tile rows r0 and r0 + 8 (wgmma fragment rows)
    const int cl = 2 * (lane & 3);                               // token columns 8 nb + cl + {0, 1}
    const bool signal = (threadIdx.x & 127) == 0;                // arrives on the ring barriers for its warpgroup
    const bool f16 = KIND == KIND_16 && p.out_dtype == CB_F16;
    auto row_of = [&](int e) { return r0 + 8 * ((e >> 1) & 1); };
    auto col_of = [&](int e) { return 8 * (e >> 2) + cl + (e & 1); };

    // final conversion of one element: m = activation / output row, n = output column, ld = row stride
    const uint32_t push_calls = kPush ? *p.push.calls : 0u;       // reduces completed so far: slot and epoch of this one
    const int64_t push_off = kPush ? push_area(p.push, push_calls) : 0;
    auto finish = [&](int m, int n, int ld, float v_f, int v_i) {
      int mo = m;
      if constexpr (EPI == EPI_ROWS) {
        mo = p.g_out_rows[m];
        if (mo < 0) return;
      }
      const int64_t o = (int64_t)mo * ld + n;
      if (KIND == KIND_I8) {
        float v = (float)v_i * p.a_s[m] * p.b_s[n];
        __half h = __float2half_rn(v);
        if (p.bias) h = __hadd(h, reinterpret_cast<const __half*>(p.bias)[n]);
        reinterpret_cast<__half*>(p.out)[o] = h;
      } else if (p.out_dtype == CB_BF16) {
        float v = v_f;
        if (p.g_row_scale) v *= p.g_row_scale[m];
        if (p.bias) v += __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.bias)[n]);
        if (p.residual) v = __bfloat162float(__float2bfloat16_rn(v)) + __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.residual)[o]);
        reinterpret_cast<__nv_bfloat16*>(p.out)[o] = __float2bfloat16_rn(v);
      } else {
        float v = v_f;
        if (p.bias) v += __half2float(reinterpret_cast<const __half*>(p.bias)[n]);
        if (p.residual) v = __half2float(__float2half_rn(v)) + __half2float(reinterpret_cast<const __half*>(p.residual)[o]);
        reinterpret_cast<__half*>(p.out)[o] = __float2half_rn(v);
      }
    };

    // tile geometry: weight row block (scale row), activation rows, valid tokens, output addressing
    struct Geo { int w_row0, m0, cnt, ocol0, ld, last_row; };
    auto geo_of = [&](const WorkItem& w) -> Geo {
      Geo ge;
      if (grouped) {
        const int4 t = geom(w.tile);
        ge.w_row0 = t.x; ge.m0 = t.y; ge.cnt = t.z;
        ge.ocol0 = t.w;
        ge.ld = p.g_ncols;
        ge.last_row = ge.m0 + ge.cnt - 1;
      } else {
        ge.w_row0 = (w.tile % p.n_tiles) * kTileN;
        ge.m0 = (w.tile / p.n_tiles) * BN;
        ge.cnt = min(BN, p.M - ge.m0);
        ge.ocol0 = ge.w_row0;
        ge.ld = p.N;
        ge.last_row = p.M - 1;
      }
      return ge;
    };
    // fp8 block scales of one 128-wide K block, fetched ONE BLOCK AHEAD of the MMA that needs them (loaded after the
    // wait they are an exposed L2 round trip per K block).  The BN activation scales are spread over the lanes
    // (token j -> lane j % 32) and broadcast by shuffle.
    constexpr int AV = (BN + 31) / 32;
    auto fetch_scales = [&](const Geo& ge, int kb, float& bsc, float (&av)[AV]) {
      bsc = p.b_s[(int64_t)(ge.w_row0 / kTileN) * p.kblocks + kb];
#pragma unroll
      for (int i = 0; i < AV; ++i) {
        const int j = BN < 32 ? (lane & (BN - 1)) : i * 32 + lane;
        const int m = min(ge.m0 + j, ge.last_row);
        av[i] = p.a_s[(int64_t)m * p.kblocks + kb];
      }
    };

    int it = 0;                                   // pipeline stage counter (same sequence as the producer's)
    ItemIter ii(g_begin, g_end, S);
    float bsc_n = 0.f, av_n[AV];
#pragma unroll
    for (int i = 0; i < AV; ++i) av_n[i] = 0.f;
    Geo ge = {0, 0, 0, 0, 0, 0};
    if (ii.valid()) {
      ge = geo_of(ii.item());
      if (KIND == KIND_FP8) fetch_scales(ge, ii.item().s_lo, bsc_n, av_n);
    }
    while (ii.valid()) {
      const WorkItem w = ii.item();
      ii.next();
      const bool have_next = ii.valid();
      const Geo gn = have_next ? geo_of(ii.item()) : ge;
      const int m0 = ge.m0, cnt = ge.cnt, ld = ge.ld;

      Acc d[NR];
      float acc[NR];
#pragma unroll
      for (int e = 0; e < NR; ++e) { d[e] = 0; acc[e] = 0.f; }
      for (int st = w.s_lo; st < w.s_hi; ++st, ++it) {
        const int s = it % C::kStages;
        const float bsc = bsc_n;
        float av[AV];
#pragma unroll
        for (int i = 0; i < AV; ++i) av[i] = av_n[i];
        if (KIND == KIND_FP8) {
          if (st + 1 < w.s_hi) fetch_scales(ge, st + 1, bsc_n, av_n);
          else if (have_next) fetch_scales(gn, ii.item().s_lo, bsc_n, av_n);
        }
        mbar_wait(&full_bar[s], (it / C::kStages) & 1);
        const int first = KIND == KIND_FP8 || st == w.s_lo;     // fp8: a fresh accumulator per K block
        wgmma_fence();
        if constexpr (C::kSoft) {
          // A = the bf16 tile the converter warps produced from this stage's fp8 weights (two 64-element atoms)
          const int c = it % C::kCvtRing;
          mbar_wait(&cvt_full[c], (it / C::kCvtRing) & 1);
          const uint32_t a0 = smem_u32(smem_c + c * C::kCvtBytes) + wg * 64 * kStageRowBytes;
          const uint32_t b0 = smem_u32(smem_x + s * C::kStageX);
#pragma unroll
          for (int k = 0; k < 8; ++k)
            mma_k<KIND, BN>(d, make_kmajor_sw128_desc(a0 + (k >> 2) * (kTileN * kStageRowBytes) + 32 * (k & 3)),
                            make_kmajor_sw128_desc(b0 + (k >> 2) * (BN * kStageRowBytes) + 32 * (k & 3)),
                            (first && k == 0) ? 0 : 1, f16);
          wgmma_commit();
          wgmma_wait<0>();
          if (signal) mbar_arrive(&cvt_empty[c]);
        } else {
          const uint32_t a0 = smem_u32(smem_w + s * C::kStageW) + wg * 64 * kStageRowBytes;
          const uint32_t b0 = smem_u32(smem_x + s * C::kStageX);
#pragma unroll
          for (int k = 0; k < 4; ++k)     // 4 x 32 B of K per 128 B stage row
            mma_k<KIND, BN>(d, make_kmajor_sw128_desc(a0 + 32 * k), make_kmajor_sw128_desc(b0 + 32 * k),
                            (first && k == 0) ? 0 : 1, f16);
          wgmma_commit();
          wgmma_wait<0>();
        }
        if (signal) mbar_arrive(&empty_bar[s]);
        if constexpr (KIND == KIND_FP8) {
#pragma unroll
          for (int e = 0; e < NR; ++e) {
            // (dot * a_s) * b_s as the reference does (triton_kernels.py:357)
            const int col = col_of(e);
            const float as = __shfl_sync(0xffffffffu, av[(e >> 2) >> 2], col & 31);
            acc[e] = fmaf(d[e] * as, bsc, acc[e]);
          }
        }
      }
      float vals[NR];                             // i8: raw int32 bits kept in the float register
#pragma unroll
      for (int e = 0; e < NR; ++e) {
        if constexpr (KIND == KIND_FP8) vals[e] = acc[e];
        else if constexpr (KIND == KIND_I8) vals[e] = __int_as_float(d[e]);
        else vals[e] = d[e];
      }

      const bool whole = (w.s_lo == 0 && w.s_hi == S);
      auto n_ok = [&](int e) { return grouped ? true : (ge.ocol0 + row_of(e) < p.N); };
      // SiluAndMul fused into the epilogue (fused_moe.py:24-39; FeedForward gate_up -> silu * mul): with the gate / up rows
      // of the merged weight interleaved at load time, rows 2i and 2i+1 of the tile (lanes l and l ^ 4) hold g and u of the
      // same output element.  Same roundings as the two separate launches: g, u -> bf16 (the GEMM's output), silu(g) ->
      // bf16, product -> bf16.
      auto emit_pairs = [&](const float (&v)[NR]) {
#pragma unroll
        for (int e = 0; e < NR; ++e) {
          const float other = __shfl_xor_sync(0xffffffffu, v[e], 4);
          const int n = ge.ocol0 + row_of(e), j = col_of(e);
          if (n_ok(e) && ((lane >> 2) & 1) == 0 && j < cnt) {
            const float g = __bfloat162float(__float2bfloat16_rn(v[e])), u = __bfloat162float(__float2bfloat16_rn(other));
            const float sl = __bfloat162float(__float2bfloat16_rn(g / (1.f + expf(-g))));
            reinterpret_cast<__nv_bfloat16*>(p.out)[(int64_t)(m0 + j) * (ld >> 1) + (n >> 1)] = __float2bfloat16_rn(sl * u);
          }
        }
      };
      // tensor-parallel partial (EPI_PUSH): bf16 pairs (adjacent output features = lanes l and l ^ 4) straight into
      // every rank's push area over NVLink, each 8-byte word tagged with the reduce's epoch (comm.cu)
      auto emit_push = [&](const float (&v)[NR]) {
#pragma unroll
        for (int e = 0; e < NR; ++e) {
          const float other = __shfl_xor_sync(0xffffffffu, v[e], 4);
          const int n = ge.ocol0 + row_of(e), j = col_of(e);
          if (n_ok(e) && ((lane >> 2) & 1) == 0 && j < cnt) {
            const __nv_bfloat16* tag = nullptr;
            push_word(p.push, push_off + ((((int64_t)(m0 + j) * ld + n) >> 1) << 3), pack2(v[e], other, tag), push_calls + 1u);
          }
        }
      };
      auto emit = [&](const float (&v)[NR]) {
        if constexpr (kPairs) {
          emit_pairs(v);
        } else if constexpr (kPush) {
          emit_push(v);
        } else {
#pragma unroll
          for (int e = 0; e < NR; ++e)
            if (n_ok(e) && col_of(e) < cnt) finish(m0 + col_of(e), ge.ocol0 + row_of(e), ld, v[e], __float_as_int(v[e]));
        }
      };
      if (whole) {
        emit(vals);
      } else {
        // contributors of this tile: CTAs whose ranges intersect [tile*S, (tile+1)*S); CTA c keeps the
        // partial of its FIRST work item in slot 0 and of any later (necessarily last) item in slot 1
        const int c_first = (w.tile * S) / per;
        const int c_last = ((w.tile + 1) * S - 1) / per;
        const int count = c_last - c_first + 1;
        const int my_slot = ((int)blockIdx.x * per) / S == w.tile ? 0 : 1;
        float* mine = p.partial + ((int64_t)blockIdx.x * 2 + my_slot) * (BN * kTileN);
#pragma unroll
        for (int e = 0; e < NR; ++e) mine[col_of(e) * kTileN + row_of(e)] = vals[e];
        __threadfence();
        // named barrier of this warpgroup (ids 1..2), 128 threads; each half of the tile has its own ticket
        asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
        if (signal) {
          const int prev = atomicAdd(&p.tickets[w.tile * 2 + wg], 1);
          s_is_last[wg] = (prev == count - 1);
          if (prev == count - 1) p.tickets[w.tile * 2 + wg] = 0;   // self-reset for the next launch / graph replay
        }
        asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
        const bool last = s_is_last[wg] != 0;
        asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");   // s_is_last may be rewritten by the next item
        if (last) {
          __threadfence();
          // all loads of one contributor are independent -> issued back to back (a serial loop is one L2 round trip
          // per load)
          float tot[NR];
#pragma unroll
          for (int e = 0; e < NR; ++e) tot[e] = 0.f;
          // CB contributors per round trip, summed in contributor order -> deterministic
          constexpr int CB = BN <= 16 ? 8 : (BN <= 32 ? 4 : (BN <= 64 ? 2 : 1));
          for (int c0 = c_first; c0 <= c_last; c0 += CB) {
            float v[CB][NR];
#pragma unroll
            for (int cc = 0; cc < CB; ++cc) {
              const int c = min(c0 + cc, c_last);
              const int slot = (c * per) / S == w.tile ? 0 : 1;
              const float* base = p.partial + ((int64_t)c * 2 + slot) * (BN * kTileN);
#pragma unroll
              for (int e = 0; e < NR; ++e) v[cc][e] = __ldcg(&base[col_of(e) * kTileN + row_of(e)]);
            }
#pragma unroll
            for (int cc = 0; cc < CB; ++cc) {
              if (c0 + cc > c_last) break;
#pragma unroll
              for (int e = 0; e < NR; ++e) {
                if (KIND == KIND_I8) tot[e] = __int_as_float(__float_as_int(tot[e]) + __float_as_int(v[cc][e]));
                else tot[e] += v[cc][e];
              }
            }
          }
          emit(tot);
        }
      }
      ge = gn;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
}  // namespace

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)f;
  });
  return fn;
}

bool tma_available() { return get_encode() != nullptr; }

int make_tma_map_2d(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int elem_bytes,
                    CUtensorMapDataType dt, int box_rows) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return fail(-3, "cuTensorMapEncodeTiled is not available from the driver");
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * elem_bytes};
  cuuint32_t box[2] = {(cuuint32_t)(128 / elem_bytes), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(-3, "cuTensorMapEncodeTiled failed (CUresult %d) rows=%lld cols=%lld", (int)r, (long long)rows, (long long)cols);
  return 0;
}

namespace {

int make_map(CUtensorMap* map, const void* base, int rows, int K, int elem_bytes, CUtensorMapDataType dt, int box_rows) {
  return make_tma_map_2d(map, base, rows, K, elem_bytes, dt, box_rows);
}

int pick_bn(int M) { return M <= 16 ? 16 : M <= 32 ? 32 : M <= 64 ? 64 : 128; }

constexpr int kMaxTickets = 65536;          // tiles; two tickets (one per 64-row half) each
int g_num_sms = 0;

int num_sms() {
  if (g_num_sms == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
      g_num_sms = n;
    else
      g_num_sms = 132;
  }
  return g_num_sms;
}

// tickets + two partial slots of [BN][128] fp32 per CTA
constexpr int64_t kTicketBytes = (int64_t)kMaxTickets * 2 * 4;
int64_t ws_bytes_for(int grid, int BN) { return kTicketBytes + (int64_t)grid * 2 * BN * kTileN * 4; }

template <int KIND, int BN, int EPI>
int launch_epi(const CUtensorMap& mw, const CUtensorMap& mx, Params& p, int grid, cudaStream_t st) {
  using C = Cfg<KIND, BN>;
  size_t smem = 1024 + (size_t)C::kStages * C::kStageBytes + (size_t)C::kCvtStages * C::kCvtBytes;
  // opt-in dynamic shared memory: static (barriers, tile geometry) + dynamic must stay within 227 KB
  static size_t attr_bytes = 0;
  if (smem > attr_bytes) {
    CB_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<KIND, BN, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_bytes = smem;
  }
  cb::launch_k(tc_gemm_kernel<KIND, BN, EPI>, dim3(grid), dim3(C::kThreads), smem, st, mw, mx, p);
  CB_LAUNCHED(1);
  return 0;
}

template <int KIND, int BN>
int launch(const CUtensorMap& mw, const CUtensorMap& mx, Params& p, int grid, cudaStream_t st) {
  if (p.act_pairs) {
    if constexpr (KIND == KIND_16) return launch_epi<KIND, BN, EPI_PAIRS>(mw, mx, p, grid, st);
    else return fail(-2, "tc gemm: the SiluAndMul epilogue is built for bf16 weights only");
  }
  if (p.has_push) {
    if constexpr (KIND == KIND_16 || KIND == KIND_FP8) return launch_epi<KIND, BN, EPI_PUSH>(mw, mx, p, grid, st);
    else return fail(-2, "tc gemm: the push epilogue is built for bf16 and fp8 weights only");
  }
  if (p.g_out_rows) {
    if constexpr (KIND != KIND_I8) return launch_epi<KIND, BN, EPI_ROWS>(mw, mx, p, grid, st);
    else return fail(-2, "tc gemm: output-row indirection is not built for int8");
  }
  return launch_epi<KIND, BN, EPI_PLAIN>(mw, mx, p, grid, st);
}

template <int KIND>
int dispatch_bn(int BN, const CUtensorMap& mw, const CUtensorMap& mx, Params& p, int grid, cudaStream_t st) {
  switch (BN) {
    case 16: return launch<KIND, 16>(mw, mx, p, grid, st);
    case 32: return launch<KIND, 32>(mw, mx, p, grid, st);
    case 64: return launch<KIND, 64>(mw, mx, p, grid, st);
    default: return launch<KIND, 128>(mw, mx, p, grid, st);
  }
}

int run(int kind, const void* x, const void* w, Params& p, int elem, CUtensorMapDataType dt, void* ws, int64_t ws_bytes,
        cudaStream_t st, int x_elem = 0, CUtensorMapDataType x_dt = CU_TENSOR_MAP_DATA_TYPE_UINT8) {
  static const int prefetch_env = getenv("CHITU_B200_GEMM_PREFETCH") ? atoi(getenv("CHITU_B200_GEMM_PREFETCH")) : 1;
  p.prefetch = prefetch_env;
  const int BN = pick_bn(p.M);
  p.n_tiles = cdiv(p.N, kTileN);
  p.m_chunks = cdiv(p.M, BN);
  p.S = cdiv((int64_t)p.K * elem, kStageRowBytes);
  p.kblocks = cdiv(p.K, 128);
  const int tiles = p.n_tiles * p.m_chunks;
  if (tiles > kMaxTickets) return fail(-2, "tc_gemm: too many tiles (%d)", tiles);
  const int64_t total = (int64_t)tiles * p.S;
  const int sms = num_sms();
  int grid = sms;
  if (grid > total) grid = (int)total;
  // at least 4 stages (64 KB of weights) per CTA, otherwise the prologue dominates; and at most 8 CTAs
  // per tile, otherwise the last arriver's reduction of the partials dominates (gate GEMM: 28 -> 8)
  if (total / grid < 4) grid = (int)(total / 4 > 0 ? total / 4 : 1);
  p.per = (int)((total + grid - 1) / grid);
  if (p.per * 8 < p.S) p.per = (p.S + 7) / 8;
  grid = (int)((total + p.per - 1) / p.per);
  // Sharing tiles between CTAs costs a partial write + ticket + a reduction round trip (~3.5 us measured);
  // streaming one 16 KB stage costs ~0.15 us per CTA.  Small GEMMs are faster with whole tiles per CTA.
  const int whole_per = p.S * (int)((tiles + sms - 1) / sms);
  const double t_split = 0.15 * p.per + 3.5, t_whole = 0.15 * whole_per;
  const bool no_ws = !ws || ws_bytes < ws_bytes_for(grid, BN);
  if ((p.per % p.S) != 0 && (no_ws || t_whole <= t_split)) {
    p.per = whole_per;
    grid = (int)((total + p.per - 1) / p.per);
  }
  p.tickets = (int*)ws;
  p.partial = ws ? (float*)((uint8_t*)ws + kTicketBytes) : nullptr;
  CUtensorMap mw, mx;
  int rc = make_map(&mw, w, p.N, p.K, elem, dt, kTileN);
  if (rc) return rc;
  rc = x_elem ? make_map(&mx, x, p.M, p.K, x_elem, x_dt, BN) : make_map(&mx, x, p.M, p.K, elem, dt, BN);
  if (rc) return rc;
  if (kind == KIND_16) return dispatch_bn<KIND_16>(BN, mw, mx, p, grid, st);
  if (kind == KIND_FP8) return dispatch_bn<KIND_FP8>(BN, mw, mx, p, grid, st);
  if (kind == KIND_SOFT) return dispatch_bn<KIND_SOFT>(BN, mw, mx, p, grid, st);
  return dispatch_bn<KIND_I8>(BN, mw, mx, p, grid, st);
}

}  // namespace

int64_t tc_max_tiles() { return kMaxTickets; }

bool tc_supported(int kind, int M, int N, int K) {
  if (M < 1 || N < 1 || K < 1) return false;
  const int elem = kind == KIND_16 ? 2 : 1;
  if (((int64_t)K * elem) % 16 != 0) return false;          // TMA row pitch
  if ((kind == KIND_FP8 || kind == KIND_SOFT) && K % 128 != 0) return false;   // one scale block per pipeline stage
  return tma_available();
}

int64_t tc_workspace_bytes(int M, int N) {
  (void)N;
  return ws_bytes_for(num_sms(), pick_bn(M));
}

// Grouped (MoE experts) GEMM: sorted activations xs [rows, K], stacked weights w [E*Ng, K]; tile list in
// device memory (see Params).  kind: KIND_16 (bf16 x bf16) or KIND_FP8 (block-scaled, a_s [rows, K/128],
// b_s [E*Ng/128, K/128]).  max_tokens_per_expert bounds wgmma N.  Output: sorted rows [rows, Ng] bf16.
int tc_grouped_gemm(int kind, const void* xs, const float* a_s, const void* w, const float* b_s, void* out, int rows,
                    int E, int Ng, int K, int max_tokens_per_expert, const int* g_num_tiles, const int* g_tile_wrow,
                    const int* g_tile_xrow, const int* g_tile_cnt, const float* row_scale, const int* out_rows, void* ws,
                    int64_t ws_bytes, cudaStream_t st) {
  Params p{};
  const int elem = kind == KIND_16 ? 2 : 1;             // weight bytes per element
  p.M = rows; p.N = Ng; p.K = K;
  p.S = cdiv((int64_t)K * elem, kStageRowBytes);
  p.kblocks = cdiv(K, 128);
  p.out_dtype = CB_BF16; p.a_s = a_s; p.b_s = b_s; p.out = out;
  p.g_num_tiles = g_num_tiles; p.g_tile_wrow = g_tile_wrow; p.g_tile_xrow = g_tile_xrow; p.g_tile_cnt = g_tile_cnt;
  p.g_ncols = Ng; p.g_row_scale = row_scale; p.g_out_rows = out_rows;
  const int BN = pick_bn(max_tokens_per_expert);      // rows per chunk: the plan cuts larger experts into chunks
  if (max_tokens_per_expert > 128) return fail(-2, "tc_grouped_gemm: more than 128 rows per chunk");
  if (Ng % kTileN != 0) return fail(-2, "tc_grouped_gemm: expert width %d is not a multiple of 128", Ng);
  if (kind != KIND_16 && K % 128 != 0) return fail(-2, "tc_grouped_gemm: fp8 weights need K %% 128 == 0 (K = %d)", K);
  const int grid = num_sms();
  if (!ws || ws_bytes < ws_bytes_for(grid, BN)) return fail(-2, "tc_grouped_gemm: workspace too small");
  p.tickets = (int*)ws;
  p.partial = (float*)((uint8_t*)ws + kTicketBytes);
  CUtensorMap mw, mx;
  const CUtensorMapDataType wdt = kind == KIND_16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8;
  const bool x16 = kind != KIND_FP8;                  // bf16 activations (bf16 and soft-fp8 kinds)
  int rc = make_tma_map_2d(&mw, w, (int64_t)E * Ng, K, elem, wdt, kTileN);
  if (rc) return rc;
  rc = make_tma_map_2d(&mx, xs, rows, K, x16 ? 2 : 1, x16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, BN);
  if (rc) return rc;
  if (kind == KIND_16) return dispatch_bn<KIND_16>(BN, mw, mx, p, grid, st);
  if (kind == KIND_SOFT) return dispatch_bn<KIND_SOFT>(BN, mw, mx, p, grid, st);
  return dispatch_bn<KIND_FP8>(BN, mw, mx, p, grid, st);
}

int tc_linear16(const void* x, const void* w, const void* bias, const void* residual, void* y, int M, int N, int K,
                int dtype, void* ws, int64_t ws_bytes, cudaStream_t st, void* comm) {
  Params p{};
  p.M = M; p.N = N; p.K = K;
  p.out_dtype = dtype; p.bias = bias; p.residual = residual; p.out = y;
  if (comm) {
    int rc = comm_push_desc(comm, &p.push);
    if (rc) return rc;
    p.has_push = 1;
  }
  return run(KIND_16, x, w, p, 2, dtype == CB_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
             ws, ws_bytes, st);
}

// y[M, N/2] = SiluAndMul(x . W^T) with W's rows interleaved (gate_0, up_0, gate_1, up_1, ...); bf16 only
int tc_linear16_silu_pairs(const void* x, const void* w, void* y, int M, int N, int K, void* ws, int64_t ws_bytes,
                           cudaStream_t st) {
  Params p{};
  p.M = M; p.N = N; p.K = K;
  p.out_dtype = CB_BF16; p.out = y; p.act_pairs = 1;
  return run(KIND_16, x, w, p, 2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, ws, ws_bytes, st);
}

int tc_fp8_gemm(const void* a, const float* a_s, const void* b, const float* b_s, void* c, int M, int N, int K,
                const void* residual, void* ws, int64_t ws_bytes, cudaStream_t st, void* comm) {
  Params p{};
  p.M = M; p.N = N; p.K = K;
  p.out_dtype = CB_BF16; p.a_s = a_s; p.b_s = b_s; p.out = c; p.residual = residual;
  if (comm) {
    int rc = comm_push_desc(comm, &p.push);
    if (rc) return rc;
    p.has_push = 1;
  }
  return run(KIND_FP8, a, b, p, 1, CU_TENSOR_MAP_DATA_TYPE_UINT8, ws, ws_bytes, st);
}

// soft_fp8_gemm_deepseek_v3 (ops.py:486-511): a bf16 [M,K], b fp8 [N,K] + block scales -> c bf16 [M,N]
int tc_soft_fp8_gemm(const void* a, const void* b, const float* b_s, void* c, int M, int N, int K, void* ws,
                     int64_t ws_bytes, cudaStream_t st) {
  Params p{};
  p.M = M; p.N = N; p.K = K;
  p.out_dtype = CB_BF16; p.b_s = b_s; p.out = c;
  return run(KIND_SOFT, a, b, p, 1, CU_TENSOR_MAP_DATA_TYPE_UINT8, ws, ws_bytes, st, 2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
}

int tc_w8a8_gemm(void* out, const int8_t* a, const int8_t* b, const float* a_scales, const float* b_scales,
                 const void* bias, int M, int N, int K, void* ws, int64_t ws_bytes, cudaStream_t st) {
  Params p{};
  p.M = M; p.N = N; p.K = K;
  p.out_dtype = CB_F16; p.a_s = a_scales; p.b_s = b_scales; p.bias = bias; p.out = out;
  return run(KIND_I8, a, b, p, 1, CU_TENSOR_MAP_DATA_TYPE_UINT8, ws, ws_bytes, st);
}

}  // namespace cb

CB_DEFINE_TL_SETTER(gemm_tc)
