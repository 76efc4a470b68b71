// One-shot all-reduce over NVLink peer memory, fused with the residual add and the RMSNorm (+ FP8
// activation quantisation) that follow every tensor-parallel linear of the decode step.
//
// Reference: RowParallelLinear.forward -> torch.distributed.all_reduce (tensor_parallel.py:157-169) and the
// MoE all_reduce (model_deepseek_v3.py:1011), each followed by `x = x + ...` and the next block's RMSNorm
// (model_deepseek_v3.py:1100-1114): NCCL all-reduce + add + norm (+ act_quant) = 3-4 launches and a
// 15-20 us small-message latency, 122 times per DeepSeek step (SURVEY §5.8).  Here: ONE kernel.
//
//   * every rank owns a symmetric buffer (cudaMalloc + CUDA IPC, mapped into all peers) with two slots;
//   * CTA `row` copies its rank's partial row into the local slot, publishes a per-(row, rank) flag to every
//     peer (st.release.sys), waits for the W flags of its row (ld.acquire.sys), then PULLS the row from all
//     W ranks over NVLink (ld.global on peer pointers), sums in rank order in fp32 (deterministic, identical
//     on all ranks), rounds, adds the residual, writes h and the RMSNorm / fp8 outputs of h;
//   * slots alternate per call and flags carry an epoch, both from a per-row device counter, so the kernel
//     is CUDA-graph replayable and needs no second barrier (a rank can only reach call i+2 after all peers
//     finished reading call i).
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

using namespace cb;

namespace {

constexpr int kMaxWorld = cb::kPushMaxWorld;
constexpr int kMaxRows = 256;

struct Comm {
  int rank, world;
  int64_t slot_bytes;                 // bytes of one slot
  uint8_t* buf[kMaxWorld];            // symmetric data buffers (2 slots each), index = rank
  uint32_t* flags[kMaxWorld];         // [2 slots][kMaxRows][kMaxWorld]
  uint32_t* counters;                 // local: [kMaxRows] calls so far, then [1] status word
  void* local_buf;
  void* local_flags;
  uint64_t timeout_ns;
  int grid_cap;                       // resident CTAs of the kernel on this device (persistent grid bound)
  // push mode: producers (GEMM / expert-combine epilogues) store their bf16 partial rows straight into EVERY rank's
  // push area [2 slots][W sources][2 * slot_bytes] as 8-byte {2 x bf16, epoch} words (the data carries its own flag:
  // no fence, no arrival counter)
  uint8_t* pbuf[kMaxWorld];
  uint32_t* pflags[kMaxWorld];        // local only: [16] = consumer CTAs done, [17] = calls so far (epoch = calls + 1)
};

struct CommDev {
  int rank, world;
  int64_t slot_bytes;
  uint8_t* buf[kMaxWorld];
  uint32_t* flags[kMaxWorld];
  uint32_t* counters;
  uint32_t* status;                   // local: [0] != 0 after a peer wait timed out (see chitu_b200_comm_status)
  uint64_t timeout_ns;                // 0 = wait for ever (NCCL's behaviour)
};

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// one CTA per row; dim % 8 == 0, dim <= 8192 (4 uint4 per thread)
__global__ void __launch_bounds__(256) allreduce_norm_kernel(CommDev c, const __nv_bfloat16* __restrict__ partial,
                                                             const __nv_bfloat16* __restrict__ residual,
                                                             __nv_bfloat16* __restrict__ h_out,
                                                             const __nv_bfloat16* __restrict__ norm_w,
                                                             __nv_bfloat16* __restrict__ y, uint8_t* __restrict__ q,
                                                             float* __restrict__ qs, int dim, float eps, int rows) {
  cb::pdl_prologue();
  constexpr int kIt = 4;
  const int tid = threadIdx.x, lane = tid & 31;
  const int nvec = dim / 8;                               // uint4 (8 bf16) per row
  __shared__ uint32_t s_n;
  __shared__ float red[8];
  // Persistent grid: gridDim.x <= the number of CTAs that are resident at once on EVERY rank, each CTA walks its rows in
  // increasing order.  A CTA waiting for row r's peers therefore never blocks a lower row of another rank from being
  // scheduled (the protocol needs the CTA of row r alive on all ranks, not in-order block dispatch).
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
  __syncthreads();
  if (tid == 0) s_n = c.counters[row];
  __syncthreads();
  const uint32_t n = s_n;
  const int slot = n & 1;
  const uint32_t epoch = (n >> 1) + 1;
  const int64_t row_off = (int64_t)slot * c.slot_bytes + (int64_t)row * dim * 2;

  // phase 1: my partial row -> my symmetric slot
  uint4* mine = reinterpret_cast<uint4*>(c.buf[c.rank] + row_off);
  const uint4* src = reinterpret_cast<const uint4*>(partial + (int64_t)row * dim);
#pragma unroll
  for (int it = 0; it < kIt; ++it) {
    const int i = it * 256 + tid;
    if (i < nvec) mine[i] = src[i];
  }
  // release pattern: the CTA barrier orders every thread's slot stores before thread `tid`'s
  // st.release.sys of the flag (cumulativity), so no per-thread system fence is needed
  __syncthreads();
  // phase 2: publish / wait (per row, per source rank)
  if (tid < c.world) {
    uint32_t* f = c.flags[tid] + ((int64_t)slot * kMaxRows + row) * kMaxWorld + c.rank;
    st_release_sys(f, epoch);
    const uint32_t* mineflag = c.flags[c.rank] + ((int64_t)slot * kMaxRows + row) * kMaxWorld + tid;
    // A peer may legitimately be late by seconds (a long prefill, a lazy compile, a debugger): like NCCL, wait.  The
    // timeout (CHITU_B200_COMM_TIMEOUT_S, default 600 s, 0 = for ever) is for DEAD peers only: it raises the status word
    // the host can poll (chitu_b200_comm_status) and then traps, so the failure is loud instead of a silent hang.
    uint64_t t0 = 0;
    for (uint32_t spin = 0;; ++spin) {
      if (ld_acquire_sys(mineflag) == epoch) break;
      if ((spin & 0xfff) == 0xfff && c.timeout_ns) {
        uint64_t t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        if (t0 == 0) t0 = t;
        else if (t - t0 > c.timeout_ns) {
          atomicExch(c.status, 1u + (uint32_t)tid);          // which peer never arrived
          __threadfence_system();
          __trap();
        }
      }
    }
  }
  __syncthreads();
  // phase 3: pull the row from every rank — ALL loads are issued before the first add, so the W peers cost
  // one NVLink round trip instead of W (measured: 34 us -> per all-reduce at W=8 with the serial loop);
  // the sum is still formed in rank order (deterministic, identical on all ranks)
  float acc[kIt][8];
#pragma unroll
  for (int it = 0; it < kIt; ++it)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[it][j] = 0.f;
  {
    uint4 v[kMaxWorld][kIt];
#pragma unroll
    for (int r = 0; r < kMaxWorld; ++r) {
      const uint4* pr = reinterpret_cast<const uint4*>(c.buf[r < c.world ? r : c.rank] + row_off);
#pragma unroll
      for (int it = 0; it < kIt; ++it) {
        const int i = it * 256 + tid;
        v[r][it] = make_uint4(0, 0, 0, 0);
        // volatile: never served from a stale L1 line of an earlier use of this slot
        if (r < c.world && i < nvec)
          asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                       : "=r"(v[r][it].x), "=r"(v[r][it].y), "=r"(v[r][it].z), "=r"(v[r][it].w) : "l"(pr + i));
      }
    }
#pragma unroll
    for (int r = 0; r < kMaxWorld; ++r) {
      if (r < c.world) {
#pragma unroll
        for (int it = 0; it < kIt; ++it) {
          const uint32_t u[4] = {v[r][it].x, v[r][it].y, v[r][it].z, v[r][it].w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            acc[it][2 * j] += bf16lo(u[j]);
            acc[it][2 * j + 1] += bf16hi(u[j]);
          }
        }
      }
    }
  }
  // phase 4: round (the all-reduced tensor is bf16), + residual, write h; RMSNorm (+ fp8 quant) of h
  float ss = 0.f;
#pragma unroll
  for (int it = 0; it < kIt; ++it) {
    const int i = it * 256 + tid;
    if (i < nvec) {
      uint4 rv = make_uint4(0, 0, 0, 0);
      if (residual) rv = reinterpret_cast<const uint4*>(residual + (int64_t)row * dim)[i];
      const uint32_t ru[4] = {rv.x, rv.y, rv.z, rv.w};
      uint32_t ou[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float a = __bfloat162float(__float2bfloat16_rn(acc[it][2 * j]));
        float b = __bfloat162float(__float2bfloat16_rn(acc[it][2 * j + 1]));
        if (residual) {
          a = __bfloat162float(__float2bfloat16_rn(a + bf16lo(ru[j])));
          b = __bfloat162float(__float2bfloat16_rn(b + bf16hi(ru[j])));
        }
        acc[it][2 * j] = a;
        acc[it][2 * j + 1] = b;
        ss += a * a + b * b;
        const __nv_bfloat16* tag = nullptr;
        ou[j] = pack2(a, b, tag);
      }
      if (h_out) reinterpret_cast<uint4*>(h_out + (int64_t)row * dim)[i] = make_uint4(ou[0], ou[1], ou[2], ou[3]);
    }
  }
  if (tid == 0) c.counters[row] = n + 1;
  if (!norm_w) continue;
  ss = warp_sum(ss);
  if (lane == 0) red[tid >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) tot += red[i];
  const float rinv = rsqrtf(tot / (float)dim + eps);
#pragma unroll
  for (int it = 0; it < kIt; ++it) {
    const int i = it * 256 + tid;
    if (i < nvec) {                                     // warp-uniform when dim % 256 == 0 ... handled per lane
      const uint4 wv = reinterpret_cast<const uint4*>(norm_w)[i];
      const uint32_t wu[4] = {wv.x, wv.y, wv.z, wv.w};
      float o[8];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        o[2 * j] = __bfloat162float(__float2bfloat16_rn(acc[it][2 * j] * rinv * bf16lo(wu[j])));
        o[2 * j + 1] = __bfloat162float(__float2bfloat16_rn(acc[it][2 * j + 1] * rinv * bf16hi(wu[j])));
      }
      if (y) {
        const __nv_bfloat16* tag = nullptr;
        reinterpret_cast<uint4*>(y + (int64_t)row * dim)[i] =
            make_uint4(pack2(o[0], o[1], tag), pack2(o[2], o[3], tag), pack2(o[4], o[5], tag), pack2(o[6], o[7], tag));
      }
      if (q) {                                          // 16 lanes x 8 elements = one 128-wide group
        float amax = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(o[j]));
#pragma unroll
        for (int off = 8; off > 0; off >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, off));
        const float sc = __fdiv_rn(amax, 448.0f);
        uint32_t p0 = 0, p1 = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          p0 |= (uint32_t)float_to_fp8(__fdiv_rn(o[j], sc)) << (8 * j);
          p1 |= (uint32_t)float_to_fp8(__fdiv_rn(o[4 + j], sc)) << (8 * j);
        }
        reinterpret_cast<uint2*>(q + (int64_t)row * dim)[i] = make_uint2(p0, p1);
        if ((lane & 15) == 0) qs[(int64_t)row * (dim / 128) + (i >> 4)] = sc;
      }
    }
  }
  }   // persistent row loop
}


// ---------------------------------------------------------------------------------------------------------------
// Push mode, the local half (SURVEY 5.8 "fused with their collectives"): the row-parallel GEMM / expert combine of EVERY
// rank stored its bf16 partial into THIS rank's push area from its epilogue, over NVLink, as 8-byte words
//   { bf16 x[2k], bf16 x[2k+1], uint32 epoch }        epoch = number of reduces completed so far + 1
// (an aligned 8-byte store arrives whole, so a word whose epoch matches carries valid data: the protocol of NCCL's LL
// mode).  No fence and no arrival counter on the producer side: the first version, one system-scope fence + release
// counter per tile, was 6-9 us per reduce SLOWER than the pull kernel above on 2 GPUs (r2 mgpu2).  Here: poll the words
// of a row until every source's epoch matches, then everything is local: sum the W partials in rank order (fp32,
// deterministic, identical on all ranks), round, add the residual, write h, RMSNorm (+ fp8 quant).  One NVLink one-way
// trip per reduce instead of the copy + flag round trip + pull.
// Slots alternate with the call count: a rank can be at most one call ahead of a peer (it cannot finish reduce n + 1
// before that peer pushed its partial of n + 1, which the peer does after consuming n), so call n + 2 never overwrites
// words of call n that are still being read.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kConsumeThreads = 512;
__global__ void __launch_bounds__(kConsumeThreads) allreduce_consume_kernel(CommDev c, const uint8_t* __restrict__ pbuf,
                                                                            uint32_t* __restrict__ pflags,
                                                                            const __nv_bfloat16* __restrict__ residual,
                                                                            __nv_bfloat16* __restrict__ h_out,
                                                                            const __nv_bfloat16* __restrict__ norm_w,
                                                                            __nv_bfloat16* __restrict__ y, uint8_t* __restrict__ q,
                                                                            float* __restrict__ qs, int dim, float eps, int rows) {
  cb::pdl_prologue();
  constexpr int kIt = 2, NT = kConsumeThreads;       // 512 threads x 2 vectors x 8 elements = 8192 >= dim
  constexpr int kBatch = 4;                          // sources polled per round trip
  const int tid = threadIdx.x, lane = tid & 31;
  const int nvec = dim / 8;
  __shared__ float red[NT / 32];
  const uint32_t ncall = pflags[17];
  const int slot = ncall & 1;
  const uint32_t epoch = ncall + 1;
  const int64_t ll_bytes = 2 * c.slot_bytes;
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    float acc[kIt][8];
#pragma unroll
    for (int it = 0; it < kIt; ++it)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[it][j] = 0.f;
    for (int r0 = 0; r0 < c.world; r0 += kBatch) {
      uint4 v[kBatch][kIt][2];
      uint64_t t0 = 0;
      for (uint32_t spin = 0;; ++spin) {
        bool ok = true;
#pragma unroll
        for (int rr = 0; rr < kBatch; ++rr) {
          const int r = r0 + rr;
          const uint4* pr = reinterpret_cast<const uint4*>(pbuf + ((int64_t)slot * c.world + (r < c.world ? r : 0)) * ll_bytes +
                                                           (int64_t)row * dim * 4);
#pragma unroll
          for (int it = 0; it < kIt; ++it) {
            const int i = it * NT + tid;
            if (r < c.world && i < nvec) {
#pragma unroll
              for (int hh = 0; hh < 2; ++hh)
                asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                             : "=r"(v[rr][it][hh].x), "=r"(v[rr][it][hh].y), "=r"(v[rr][it][hh].z), "=r"(v[rr][it][hh].w)
                             : "l"(pr + 2 * i + hh));
            }
          }
        }
#pragma unroll
        for (int rr = 0; rr < kBatch; ++rr)
#pragma unroll
          for (int it = 0; it < kIt; ++it)
            if (r0 + rr < c.world && it * NT + tid < nvec)
              ok &= v[rr][it][0].y == epoch && v[rr][it][0].w == epoch && v[rr][it][1].y == epoch && v[rr][it][1].w == epoch;
        if (ok) break;
        if ((spin & 0x3ff) == 0x3ff && c.timeout_ns) {
          uint64_t t;
          asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
          if (t0 == 0) t0 = t;
          else if (t - t0 > c.timeout_ns) {
            atomicExch(c.status, 1u + (uint32_t)r0);
            __threadfence_system();
            __trap();
          }
        }
      }
#pragma unroll
      for (int rr = 0; rr < kBatch; ++rr) {
        if (r0 + rr < c.world) {
#pragma unroll
          for (int it = 0; it < kIt; ++it) {
            if (it * NT + tid < nvec) {
              const uint32_t u[4] = {v[rr][it][0].x, v[rr][it][0].z, v[rr][it][1].x, v[rr][it][1].z};
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                acc[it][2 * j] += bf16lo(u[j]);
                acc[it][2 * j + 1] += bf16hi(u[j]);
              }
            }
          }
        }
      }
    }
    float ss = 0.f;
#pragma unroll
    for (int it = 0; it < kIt; ++it) {
      const int i = it * NT + tid;
      if (i < nvec) {
        uint4 rv = make_uint4(0, 0, 0, 0);
        if (residual) rv = reinterpret_cast<const uint4*>(residual + (int64_t)row * dim)[i];
        const uint32_t ru[4] = {rv.x, rv.y, rv.z, rv.w};
        uint32_t ou[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float a = __bfloat162float(__float2bfloat16_rn(acc[it][2 * j]));
          float b = __bfloat162float(__float2bfloat16_rn(acc[it][2 * j + 1]));
          if (residual) {
            a = __bfloat162float(__float2bfloat16_rn(a + bf16lo(ru[j])));
            b = __bfloat162float(__float2bfloat16_rn(b + bf16hi(ru[j])));
          }
          acc[it][2 * j] = a;
          acc[it][2 * j + 1] = b;
          ss += a * a + b * b;
          const __nv_bfloat16* tag = nullptr;
          ou[j] = pack2(a, b, tag);
        }
        if (h_out) reinterpret_cast<uint4*>(h_out + (int64_t)row * dim)[i] = make_uint4(ou[0], ou[1], ou[2], ou[3]);
      }
    }
    if (norm_w) {
      ss = warp_sum(ss);
      __syncthreads();
      if (lane == 0) red[tid >> 5] = ss;
      __syncthreads();
      float tot = 0.f;
#pragma unroll
      for (int i = 0; i < NT / 32; ++i) tot += red[i];
      const float rinv = rsqrtf(tot / (float)dim + eps);
#pragma unroll
      for (int it = 0; it < kIt; ++it) {
        const int i = it * NT + tid;
        if (i < nvec) {
          const uint4 wv = reinterpret_cast<const uint4*>(norm_w)[i];
          const uint32_t wu[4] = {wv.x, wv.y, wv.z, wv.w};
          float o[8];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            o[2 * j] = __bfloat162float(__float2bfloat16_rn(acc[it][2 * j] * rinv * bf16lo(wu[j])));
            o[2 * j + 1] = __bfloat162float(__float2bfloat16_rn(acc[it][2 * j + 1] * rinv * bf16hi(wu[j])));
          }
          if (y) {
            const __nv_bfloat16* tag = nullptr;
            reinterpret_cast<uint4*>(y + (int64_t)row * dim)[i] =
                make_uint4(pack2(o[0], o[1], tag), pack2(o[2], o[3], tag), pack2(o[4], o[5], tag), pack2(o[6], o[7], tag));
          }
          if (q) {
            float amax = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(o[j]));
#pragma unroll
            for (int off = 8; off > 0; off >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, off));
            const float sc = __fdiv_rn(amax, 448.0f);
            uint32_t p0 = 0, p1 = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              p0 |= (uint32_t)float_to_fp8(__fdiv_rn(o[j], sc)) << (8 * j);
              p1 |= (uint32_t)float_to_fp8(__fdiv_rn(o[4 + j], sc)) << (8 * j);
            }
            reinterpret_cast<uint2*>(q + (int64_t)row * dim)[i] = make_uint2(p0, p1);
            if ((lane & 15) == 0) qs[(int64_t)row * (dim / 128) + (i >> 4)] = sc;
          }
        }
      }
    }
  }
  // the last CTA to finish advances the call count (= the epoch the producers of the next reduce will tag with)
  __syncthreads();
  if (tid == 0) {
    const uint32_t prev = atomicAdd(&pflags[16], 1u);
    if (prev == gridDim.x - 1) {
      pflags[16] = 0u;
      __threadfence();
      pflags[17] = ncall + 1;
    }
  }
}

}  // namespace

namespace cb {
// producers: the push descriptor of a communicator (device pointers of every rank's push area / arrival counters)
int comm_push_desc(void* handle, void* out_desc) {
  if (!handle || !out_desc) return fail(-1, "comm_push_desc: null argument");
  Comm* c = (Comm*)handle;
  PushDev d;
  memset(&d, 0, sizeof(d));
  for (int r = 0; r < kMaxWorld; ++r) d.base[r] = c->pbuf[r];
  d.calls = c->pflags[c->rank] + 17;
  d.world = c->world; d.rank = c->rank; d.ll_bytes = 2 * c->slot_bytes;
  memcpy(out_desc, &d, sizeof(d));
  return 0;
}
int64_t comm_slot_bytes(void* handle) { return handle ? ((Comm*)handle)->slot_bytes : 0; }
}  // namespace cb

namespace {
}  // namespace

extern "C" int chitu_b200_comm_create(int rank, int world, int64_t slot_bytes, void** handle_out,
                                      uint8_t* ipc_out /* 128 bytes */) {
  CB_ARG(handle_out && ipc_out && rank >= 0 && world >= 1 && world <= kMaxWorld && rank < world && slot_bytes > 0);
  Comm* c = new Comm();
  memset(c, 0, sizeof(Comm));
  c->rank = rank;
  c->world = world;
  c->slot_bytes = (slot_bytes + 255) / 256 * 256;
  const size_t fbytes = (size_t)2 * kMaxRows * kMaxWorld * sizeof(uint32_t) + 64 * sizeof(uint32_t);
  CB_CUDA(cudaMalloc(&c->local_buf, (size_t)2 * c->slot_bytes * (1 + 2 * world)));   // pull slots + LL push area
  CB_CUDA(cudaMalloc(&c->local_flags, fbytes));
  CB_CUDA(cudaMalloc((void**)&c->counters, (kMaxRows + 1) * sizeof(uint32_t)));
  CB_CUDA(cudaMemset(c->local_buf, 0, (size_t)2 * c->slot_bytes * (1 + 2 * world)));
  CB_CUDA(cudaMemset(c->local_flags, 0, fbytes));
  CB_CUDA(cudaMemset(c->counters, 0, (kMaxRows + 1) * sizeof(uint32_t)));
  {
    const char* e = getenv("CHITU_B200_COMM_TIMEOUT_S");
    const double sec = e ? atof(e) : 600.0;
    c->timeout_ns = sec > 0 ? (uint64_t)(sec * 1e9) : 0;
    int dev = 0, sms = 132, per_sm = 1;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, allreduce_norm_kernel, 256, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
    c->grid_cap = sms * per_sm;
  }
  CB_CUDA(cudaDeviceSynchronize());
  c->buf[rank] = (uint8_t*)c->local_buf;
  c->flags[rank] = (uint32_t*)c->local_flags;
  c->pbuf[rank] = (uint8_t*)c->local_buf + (size_t)2 * c->slot_bytes;
  c->pflags[rank] = (uint32_t*)c->local_flags + (size_t)2 * kMaxRows * kMaxWorld;
  cudaIpcMemHandle_t h0, h1;
  CB_CUDA(cudaIpcGetMemHandle(&h0, c->local_buf));
  CB_CUDA(cudaIpcGetMemHandle(&h1, c->local_flags));
  memcpy(ipc_out, &h0, 64);
  memcpy(ipc_out + 64, &h1, 64);
  *handle_out = c;
  return 0;
}

extern "C" int chitu_b200_comm_connect(void* handle, const uint8_t* all_ipc /* world x 128 bytes */) {
  CB_ARG(handle && all_ipc);
  Comm* c = (Comm*)handle;
  for (int r = 0; r < c->world; ++r) {
    if (r == c->rank) continue;
    cudaIpcMemHandle_t h0, h1;
    memcpy(&h0, all_ipc + (size_t)r * 128, 64);
    memcpy(&h1, all_ipc + (size_t)r * 128 + 64, 64);
    void *p0 = nullptr, *p1 = nullptr;
    CB_CUDA(cudaIpcOpenMemHandle(&p0, h0, cudaIpcMemLazyEnablePeerAccess));
    CB_CUDA(cudaIpcOpenMemHandle(&p1, h1, cudaIpcMemLazyEnablePeerAccess));
    c->buf[r] = (uint8_t*)p0;
    c->flags[r] = (uint32_t*)p1;
    c->pbuf[r] = (uint8_t*)p0 + (size_t)2 * c->slot_bytes;
    c->pflags[r] = (uint32_t*)p1 + (size_t)2 * kMaxRows * kMaxWorld;
  }
  return 0;
}

// 0 = healthy; 1 + r = the wait for peer r timed out (the kernel trapped after raising it).  Synchronous small copy.
extern "C" int chitu_b200_comm_status(void* handle) {
  if (!handle) return -1;
  Comm* c = (Comm*)handle;
  uint32_t v = 0;
  if (cudaMemcpy(&v, c->counters + kMaxRows, sizeof(v), cudaMemcpyDeviceToHost) != cudaSuccess) return -2;
  return (int)v;
}

extern "C" int chitu_b200_comm_destroy(void* handle) {
  if (!handle) return 0;
  Comm* c = (Comm*)handle;
  for (int r = 0; r < c->world; ++r) {
    if (r == c->rank) continue;
    if (c->buf[r]) cudaIpcCloseMemHandle(c->buf[r]);
    if (c->flags[r]) cudaIpcCloseMemHandle(c->flags[r]);
  }
  cudaFree(c->local_buf);
  cudaFree(c->local_flags);
  cudaFree(c->counters);
  delete c;
  return 0;
}

extern "C" int chitu_b200_allreduce_residual_rmsnorm(void* handle, const void* partial, const void* residual,
                                                     void* h_out, const void* norm_w, void* y, void* q,
                                                     float* q_scales, int rows, int dim, float eps, void* stream) {
  CB_ARG(handle && partial && rows >= 0 && rows <= kMaxRows && dim > 0 && dim % 8 == 0 && dim <= 8192);
  CB_ARG(h_out || norm_w);
  CB_ARG((q == nullptr) == (q_scales == nullptr));
  CB_ARG(q == nullptr || (norm_w && dim % 256 == 0));
  Comm* c = (Comm*)handle;
  CB_ARG((int64_t)rows * dim * 2 <= c->slot_bytes);
  if (rows == 0) return 0;
  CommDev d;
  d.rank = c->rank; d.world = c->world; d.slot_bytes = c->slot_bytes; d.counters = c->counters;
  d.status = c->counters + kMaxRows; d.timeout_ns = c->timeout_ns;
  for (int r = 0; r < kMaxWorld; ++r) { d.buf[r] = c->buf[r]; d.flags[r] = c->flags[r]; }
  const int grid = rows < c->grid_cap ? rows : c->grid_cap;
  cb::launch_k(allreduce_norm_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, d,
               (const __nv_bfloat16*)partial, (const __nv_bfloat16*)residual, (__nv_bfloat16*)h_out,
               (const __nv_bfloat16*)norm_w, (__nv_bfloat16*)y, (uint8_t*)q, q_scales, dim, eps, rows);
  CB_LAUNCHED(1);
  return 0;
}

// Push-mode reduce (see allreduce_consume_kernel) of the [rows, dim] partials the producing call (chitu_b200_fp8_gemm_ar /
// chitu_b200_linear_bf16_ar / chitu_b200_fused_experts_ar) of every rank pushed.
extern "C" int chitu_b200_allreduce_consume(void* handle, const void* residual, void* h_out, const void* norm_w,
                                            void* y, void* q, float* q_scales, int rows, int dim, float eps, void* stream) {
  CB_ARG(handle && rows >= 0 && rows <= kMaxRows && dim > 0 && dim % 8 == 0 && dim <= 8192);
  CB_ARG(h_out || norm_w);
  CB_ARG((q == nullptr) == (q_scales == nullptr));
  CB_ARG(q == nullptr || (norm_w && dim % 256 == 0));
  Comm* c = (Comm*)handle;
  CB_ARG((int64_t)rows * dim * 2 <= c->slot_bytes);
  if (rows == 0) return 0;
  CommDev d;
  d.rank = c->rank; d.world = c->world; d.slot_bytes = c->slot_bytes; d.counters = c->counters;
  d.status = c->counters + kMaxRows; d.timeout_ns = c->timeout_ns;
  for (int r = 0; r < kMaxWorld; ++r) { d.buf[r] = c->buf[r]; d.flags[r] = c->flags[r]; }
  const int grid = rows < c->grid_cap ? rows : c->grid_cap;
  cb::launch_k(allreduce_consume_kernel, dim3(grid), dim3(kConsumeThreads), 0, (cudaStream_t)stream, d,
               (const uint8_t*)c->pbuf[c->rank], c->pflags[c->rank], (const __nv_bfloat16*)residual, (__nv_bfloat16*)h_out, (const __nv_bfloat16*)norm_w,
               (__nv_bfloat16*)y, (uint8_t*)q, q_scales, dim, eps, rows);
  CB_LAUNCHED(1);
  return 0;
}

CB_DEFINE_TL_SETTER(comm)
