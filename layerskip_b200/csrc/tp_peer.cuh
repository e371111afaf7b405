// tp_peer.cuh — one-shot collectives over peer-mapped HBM (NVLink / NVSwitch) for the
// tensor-parallel engine.  This is the DEFAULT data path under tensor parallelism
// (LSK_TP_ONESHOT selects the protocol, 0 = NCCL; engine.cu: emit_allreduce_resid /
// emit_gemm_push_resid).  The fence + flag protocol described first is mode 3; the LL protocol
// further down (modes 1 and 2) is the default.
//
// Why: a round of the TP engine performs 2 x [(d+1) E + (L-E)] all-reduces of <= 16 x hidden fp32
// (SURVEY.md §8(e): 176 per round at 13B) plus d+1 arg-max exchanges, every one on the critical
// path of a batch-1 decode.  At these sizes (8 ... 512 KiB) a collective is pure latency: far
// more than the few microseconds of weight streaming per instance.  Here every rank owns a small region of HBM
// that all peers map (CUDA IPC), and ONE kernel per instance
//     pushes its partial rows into every peer's region (plain stores over NVLink),
//     raises a flag per (source rank, CTA) with release semantics at system scope,
//     waits for the peers' flags (acquire), sums the partials in RANK ORDER and adds the residual.
// No NCCL call remains in the round.  Summing in rank order makes every rank compute bit-identical
// residual streams (the ranks must agree on every arg-max); for two ranks it is also bit-identical
// to the NCCL path (a + b).
//
// Hazards and why they do not occur:
//  * data slots and flags are addressed by an EPOCH that lives in device memory and advances once
//    per instance, so the kernels are CUDA-graph safe (no host-baked sequence numbers);
//  * flags are monotonic (never reset): a fast peer that already signalled instance i+1 still
//    satisfies "flag >= i";
//  * data is double-buffered by epoch parity: a peer can only start instance i+2 after finishing
//    i+1, which needs MY push of i+1, which I issue after my instance i has completed (stream
//    order, every kernel waits on its predecessor) -> nobody overwrites a slot that is being read;
//  * every CTA of the grid is resident before any dependent kernel is scheduled (PDL launches the
//    dependents only once all CTAs have started), grids are <= 64 small CTAs -> the spin cannot
//    starve the CTAs it is waiting for;
//  * a peer that died would make the others spin forever: the wait has a ~2 s clock budget, then
//    raises a host-visible error flag and falls through (the host turns it into an error code).
#pragma once
#include "common.cuh"

namespace lsk {

constexpr int kMaxPeers = 8;
constexpr int kMaxArCtas = 64;
constexpr int kMaxGemmCtas = 160;                       // >= SM count: one flag per GEMM CTA
constexpr int kArThreads = 256;
constexpr int kArVecPerCta = 512;                       // float4 elements per CTA slice
constexpr long long kPeerTimeoutCycles = 4000000000LL;  // ~2 s at 1.9 GHz

// Byte offsets inside one rank's peer-visible region.
struct PeerRegionLayout {
  size_t ar_data;    // float  [2 parities][tp][kMaxRows * hidden]   (fence + flag protocol)
  size_t ll_data;    // LL lines [2 parities][tp][kMaxRows * hidden / 2] x 16 B: {v0, flag, v1, flag}
  size_t ar_flags;   // uint32 [tp][kMaxArCtas]
  size_t g_data;     // uint32 [2 parities][tp][32]   (16 fp32 values + 16 int32 indices)
  size_t g_flags;    // uint32 [tp]
  size_t gemm_flags; // uint32 [tp][kMaxGemmCtas]  (fused mode: raised by the GEMM's epilogue)
  size_t local;      // owner only: uint32 ar_epoch, int32 ar_ticket, uint32 g_epoch
  size_t total;
};
__host__ __device__ inline PeerRegionLayout peer_region_layout(int tp, int hidden) {
  PeerRegionLayout L;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t at = off; off += (bytes + 255) & ~(size_t)255; return at; };
  L.ar_data = take((size_t)2 * tp * kMaxRows * hidden * 4);
  L.ll_data = take((size_t)2 * tp * kMaxRows * hidden * 8);
  L.ar_flags = take((size_t)tp * kMaxArCtas * 4);
  L.g_data = take((size_t)2 * tp * 32 * 4);
  L.g_flags = take((size_t)tp * 4);
  L.gemm_flags = take((size_t)tp * kMaxGemmCtas * 4);
  L.local = take(16);
  L.total = off;
  return L;
}

struct PeerComm {
  unsigned char* base[kMaxPeers];   // base[r]: rank r's region (own allocation or IPC mapping)
  int rank, size, hidden;
  int* error;                       // mapped pinned host word: != 0 after a wait timed out
};

// base[r] with a run-time r, without forcing the by-value struct into local memory
__device__ __forceinline__ unsigned char* peer_base(const PeerComm& pc, int r) {
  unsigned char* p = pc.base[0];
#pragma unroll
  for (int k = 1; k < kMaxPeers; ++k)
    if (r == k) p = pc.base[k];
  return p;
}

__device__ __forceinline__ void st_release_sys(unsigned int* p, unsigned int v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_sys(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// spin until *flag has reached `epoch` (wrap-safe); false on timeout
__device__ __forceinline__ bool peer_wait(const unsigned int* flag, unsigned int epoch) {
  const long long t0 = clock64();
  while ((int)(ld_acquire_sys(flag) - epoch) < 0)
    if (clock64() - t0 > kPeerTimeoutCycles) return false;
  return true;
}

// hidden rows x[0 .. n4*4) += sum over ranks of partial_r   (partial = this rank's contribution,
// the fp32 output of a row-parallel GEMM; llama: after o_proj and after down_proj)
__global__ void __launch_bounds__(kArThreads)
tp_allreduce_resid_kernel(const PeerComm pc, const float* __restrict__ partial,
                          float* __restrict__ x, int n4) {
  pdl_launch_dependents();
  pdl_wait();
  const PeerRegionLayout L = peer_region_layout(pc.size, pc.hidden);
  unsigned char* mine = peer_base(pc, pc.rank);
  volatile unsigned int* epoch_p = reinterpret_cast<volatile unsigned int*>(mine + L.local);
  int* ticket_p = reinterpret_cast<int*>(mine + L.local + 4);
  const unsigned int epoch = *epoch_p + 1u;
  const size_t slot4 = (size_t)kMaxRows * pc.hidden / 4;          // float4 per (parity, rank) slot
  const size_t par4 = (size_t)(epoch & 1u) * pc.size * slot4;
  const int tid = threadIdx.x, c = blockIdx.x;
  const int i0 = c * kArVecPerCta;
  const int i1 = (i0 + kArVecPerCta < n4) ? i0 + kArVecPerCta : n4;
  const float4* p4 = reinterpret_cast<const float4*>(partial);

  // 1. push this CTA's slice of my partial into my slot of every peer's region
  for (int i = i0 + tid; i < i1; i += kArThreads) {
    const float4 v = __ldcg(p4 + i);
#pragma unroll
    for (int r = 0; r < kMaxPeers; ++r) {
      if (r >= pc.size || r == pc.rank) continue;
      float4* dst = reinterpret_cast<float4*>(pc.base[r] + L.ar_data) + par4 + (size_t)pc.rank * slot4 + i;
      *dst = v;
    }
  }
  __threadfence_system();
  __syncthreads();

  // 2. thread r: tell rank r "slice c of instance `epoch` from me is complete", then wait for its
  if (tid < pc.size && tid != pc.rank) {
    st_release_sys(reinterpret_cast<unsigned int*>(peer_base(pc, tid) + L.ar_flags) + pc.rank * kMaxArCtas + c, epoch);
    if (!peer_wait(reinterpret_cast<const unsigned int*>(mine + L.ar_flags) + tid * kMaxArCtas + c, epoch))
      *reinterpret_cast<volatile int*>(pc.error) = 1;
  }
  __syncthreads();

  // 3. sum in rank order (identical on every rank) and add to the residual stream
  const float4* recv = reinterpret_cast<const float4*>(mine + L.ar_data) + par4;
  float4* x4 = reinterpret_cast<float4*>(x);
  for (int i = i0 + tid; i < i1; i += kArThreads) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int r = 0; r < pc.size; ++r) {
      const float4 v = (r == pc.rank) ? __ldcg(p4 + i) : __ldcg(recv + (size_t)r * slot4 + i);
      if (r == 0) acc = v;
      else { acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w; }
    }
    float4 h = x4[i];
    h.x += acc.x; h.y += acc.y; h.z += acc.z; h.w += acc.w;
    x4[i] = h;
  }

  // 4. the last CTA to finish advances the epoch (every CTA has read it by then)
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    const int t = atomicAdd(ticket_p, 1);
    if (t == (int)gridDim.x - 1) {
      *ticket_p = 0;
      *epoch_p = epoch;
      __threadfence();
    }
  }
}

// ---------------------------------------------------------------------------------------------
// LL ("low latency") variants: the flag travels INSIDE the data.  A 16-byte line carries two fp32
// values and the instance's epoch twice — {v0, epoch, v1, epoch} — and 8-byte aligned halves are
// single-copy atomic, so a reader that sees the epoch in both halves has the values: no
// __threadfence_system(), no separate flag store, no second NVLink round trip.  The element a
// thread pushes is the element it reduces, so the kernel needs no intra-CTA synchronisation
// either.  Cost: 2x the bytes on NVLink (229 KiB per peer for a 7 x 4096 block: ~0.5 us).
// Same hazards argument as above (epoch in device memory, two parities, monotone instances).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void ll_store(uint4* p, float v0, float v1, unsigned int flag) {
  asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(__float_as_uint(v0)),
               "r"(flag), "r"(__float_as_uint(v1)), "r"(flag) : "memory");
}
// spin until both halves of the line carry `flag`; false on timeout
__device__ __forceinline__ bool ll_load(const uint4* p, unsigned int flag, float& v0, float& v1) {
  const long long t0 = clock64();
  uint4 q;
  for (;;) {
    asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(q.x), "=r"(q.y), "=r"(q.z), "=r"(q.w) : "l"(p) : "memory");
    if (q.y == flag && q.w == flag) break;
    if (clock64() - t0 > kPeerTimeoutCycles) { v0 = v1 = 0.f; return false; }
  }
  v0 = __uint_as_float(q.x);
  v1 = __uint_as_float(q.z);
  return true;
}

// last CTA to finish advances the epoch (every CTA read it at its start)
__device__ __forceinline__ void peer_advance_epoch(volatile unsigned int* epoch_p, int* ticket_p,
                                                   unsigned int epoch) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const int t = atomicAdd(ticket_p, 1);
    if (t == (int)gridDim.x - 1) {
      *ticket_p = 0;
      *epoch_p = epoch;
      __threadfence();
    }
  }
}

// x[0 .. 2*n2) += sum over ranks (rank order) of partial_r.  One launch = push + reduce.
__global__ void __launch_bounds__(kArThreads)
tp_allreduce_ll_kernel(const PeerComm pc, const float* __restrict__ partial, float* __restrict__ x, int n2) {
  pdl_launch_dependents();
  pdl_wait();
  const PeerRegionLayout L = peer_region_layout(pc.size, pc.hidden);
  unsigned char* mine = peer_base(pc, pc.rank);
  volatile unsigned int* epoch_p = reinterpret_cast<volatile unsigned int*>(mine + L.local);
  int* ticket_p = reinterpret_cast<int*>(mine + L.local + 4);
  const unsigned int epoch = *epoch_p + 1u;
  const size_t slot = (size_t)kMaxRows * pc.hidden / 2;             // lines per (parity, rank)
  const size_t par = (size_t)(epoch & 1u) * pc.size * slot;
  const float2* p2 = reinterpret_cast<const float2*>(partial);
  float2* x2 = reinterpret_cast<float2*>(x);
  const uint4* recv = reinterpret_cast<const uint4*>(mine + L.ll_data) + par;
  bool ok = true;
  for (int i = blockIdx.x * kArThreads + threadIdx.x; i < n2; i += gridDim.x * kArThreads) {
    const float2 own = __ldcg(p2 + i);
#pragma unroll
    for (int r = 0; r < kMaxPeers; ++r) {
      if (r >= pc.size || r == pc.rank) continue;
      ll_store(reinterpret_cast<uint4*>(pc.base[r] + L.ll_data) + par + (size_t)pc.rank * slot + i, own.x, own.y, epoch);
    }
    float2 h = x2[i];                                              // overlaps the NVLink flight
    float2 acc = make_float2(0.f, 0.f);
    for (int r = 0; r < pc.size; ++r) {
      float v0 = own.x, v1 = own.y;
      if (r != pc.rank) ok &= ll_load(recv + (size_t)r * slot + i, epoch, v0, v1);
      if (r == 0) acc = make_float2(v0, v1);
      else { acc.x += v0; acc.y += v1; }
    }
    h.x += acc.x; h.y += acc.y;
    x2[i] = h;
  }
  if (!ok) *reinterpret_cast<volatile int*>(pc.error) = 1;
  peer_advance_epoch(epoch_p, ticket_p, epoch);
}

// Fused mode: the row-parallel GEMM's epilogue (gemm_skinny.cuh, EPI_PUSH) wrote LL lines of its
// output tiles into slot [parity][its rank] of EVERY rank's region (its own included) while it
// was still streaming weights.  This kernel only polls the lines, sums in rank order and adds the
// residual — the NVLink transfer overlapped the GEMM tile by tile.
__global__ void __launch_bounds__(kArThreads)
tp_finish_ll_kernel(const PeerComm pc, float* __restrict__ x, int n2) {
  pdl_launch_dependents();
  pdl_wait();
  const PeerRegionLayout L = peer_region_layout(pc.size, pc.hidden);
  unsigned char* mine = peer_base(pc, pc.rank);
  volatile unsigned int* epoch_p = reinterpret_cast<volatile unsigned int*>(mine + L.local);
  int* ticket_p = reinterpret_cast<int*>(mine + L.local + 4);
  const unsigned int epoch = *epoch_p + 1u;
  const size_t slot = (size_t)kMaxRows * pc.hidden / 2;
  const uint4* recv = reinterpret_cast<const uint4*>(mine + L.ll_data) + (size_t)(epoch & 1u) * pc.size * slot;
  float2* x2 = reinterpret_cast<float2*>(x);
  bool ok = true;
  for (int i = blockIdx.x * kArThreads + threadIdx.x; i < n2; i += gridDim.x * kArThreads) {
    float2 h = x2[i];
    float2 acc = make_float2(0.f, 0.f);
    for (int r = 0; r < pc.size; ++r) {
      float v0, v1;
      ok &= ll_load(recv + (size_t)r * slot + i, epoch, v0, v1);
      if (r == 0) acc = make_float2(v0, v1);
      else { acc.x += v0; acc.y += v1; }
    }
    h.x += acc.x; h.y += acc.y;
    x2[i] = h;
  }
  if (!ok) *reinterpret_cast<volatile int*>(pc.error) = 1;
  peer_advance_epoch(epoch_p, ticket_p, epoch);
}

// Vocab-parallel LM head: this rank's best (value, index) per row from its arg-max candidates,
// exchanged with every peer -> gath_val / gath_idx [tp][kMaxRows] on every rank (what the
// finalize / accept kernels consume).  One CTA.
__global__ void __launch_bounds__(256)
tp_gather_best_kernel(const PeerComm pc, const float* __restrict__ cand_val,
                      const int* __restrict__ cand_idx, int n_cand, int rows,
                      float* __restrict__ gath_val, int* __restrict__ gath_idx) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_val[kMaxRows];
  __shared__ int s_idx[kMaxRows];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid < kMaxRows) { s_val[tid] = -INFINITY; s_idx[tid] = 0x7fffffff; }
  __syncthreads();
  for (int row = warp; row < rows; row += 8) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int k = lane; k < n_cand; k += 32) {
      const float v = cand_val[k * kMaxRows + row];
      const int i = cand_idx[k * kMaxRows + row];
      if (better(v, i, bv, bi)) { bv = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { s_val[row] = bv; s_idx[row] = bi; }
  }
  __syncthreads();

  const PeerRegionLayout L = peer_region_layout(pc.size, pc.hidden);
  unsigned char* mine = peer_base(pc, pc.rank);
  volatile unsigned int* epoch_p = reinterpret_cast<volatile unsigned int*>(mine + L.local + 8);
  const unsigned int epoch = *epoch_p + 1u;
  const int par = (int)(epoch & 1u);
  for (int k = tid; k < pc.size * 32; k += 256) {
    const int r = k >> 5, j = k & 31;
    if (r == pc.rank) continue;
    const unsigned int word = j < 16 ? __float_as_uint(s_val[j]) : (unsigned int)s_idx[j - 16];
    reinterpret_cast<unsigned int*>(peer_base(pc, r) + L.g_data)[(par * pc.size + pc.rank) * 32 + j] = word;
  }
  __threadfence_system();
  __syncthreads();
  if (tid < pc.size && tid != pc.rank) {
    st_release_sys(reinterpret_cast<unsigned int*>(peer_base(pc, tid) + L.g_flags) + pc.rank, epoch);
    if (!peer_wait(reinterpret_cast<const unsigned int*>(mine + L.g_flags) + tid, epoch))
      *reinterpret_cast<volatile int*>(pc.error) = 1;
  }
  __syncthreads();
  const unsigned int* recv = reinterpret_cast<const unsigned int*>(mine + L.g_data) + (size_t)par * pc.size * 32;
  for (int k = tid; k < pc.size * kMaxRows; k += 256) {
    const int r = k / kMaxRows, row = k % kMaxRows;
    float v;
    int i;
    if (r == pc.rank) { v = s_val[row]; i = s_idx[row]; }
    else { v = __uint_as_float(__ldcg(recv + r * 32 + row)); i = (int)__ldcg(recv + r * 32 + 16 + row); }
    gath_val[r * kMaxRows + row] = v;
    gath_idx[r * kMaxRows + row] = i;
  }
  __syncthreads();
  if (tid == 0) *epoch_p = epoch;
}

}  // namespace lsk
