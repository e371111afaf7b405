// lmhead_tc.cuh — LM head on the Hopper tensor cores (wgmma), OPT-IN (LSK_LMHEAD_TC=1).
// The default LM head is gemm_skinny_kernel<NT, PRO_RMS, EPI_LMHEAD> (mma.sync).
//
//   logits[v, m] = sum_k Wlm[v, k] * rmsnorm(x)[m, k]        v: local vocab rows, m <= 16 tokens
//
// This is the one GEMM of the decode path whose N side is large enough (vocab >= 32000: 250+
// tiles of 128 rows) for a 128-row tile to keep every SM busy without split-K, so it is where a
// warpgroup MMA fits (DESIGN.md §3.1 explains why the layer GEMMs stay on 16-row mma.sync fragments).
// Swap-AB: the WEIGHTS are the A operand (128 vocab rows per tile, K-major, streamed by TMA bulk
// copies into a shared-memory ring), the normalised activations are the B operand (N = 16 token
// columns, K-major, resident in shared memory); the fp32 accumulators live in registers.
//
// Roles (384 threads = 3 warpgroups): warp 0 lane 0 = TMA producer (the rest of warpgroup 0
// idles); warpgroups 1 and 2 = consumers, each owning 64 vocab rows of every tile: RMSNorm
// prologue, wgmma.m64n16k16 over the ring, then logits store + running arg-max from registers
// with the engine's "lowest index wins" rule.
//
// Shared-memory operand layouts (no-swizzle K-major: 8 rows x 16 B core matrices):
//   A stage  = 128 rows x 64 k = 16 KiB, packed by pack_canonical_kernel exactly as it lies in
//              HBM: core(row group i = 0..15, k chunk j = 0..7) at (i * 8 + j) * 128 B
//              -> descriptor LBO = 128 B (next k chunk), SBO = 1024 B (next 8 rows)
//   B (whole K) = core(k chunk j, token group i = 0..1) at (j * 2 + i) * 128 B
//              -> descriptor LBO = 256 B, SBO = 128 B
//   one wgmma consumes K = 16 (two k chunks): per stage 4 MMAs, descriptors advance by
//   256 B (A) and 512 B (B); consumer warpgroup g starts 8 row groups (8 KiB) into the A stage.
#pragma once
#include "gemm_skinny.cuh"

namespace lsk {

constexpr int kTcThreads = 384;
constexpr int kTcConsumerThreads = 256;                      // warpgroups 1 and 2
constexpr int kTcTileRows = 128;
constexpr int kTcStageK = 64;
constexpr int kTcStageBytes = kTcTileRows * kTcStageK * 2;   // 16 KiB
constexpr int kTcTokens = 16;                                // MMA N
constexpr int kTcMaxStages = 6;
constexpr int BAR_TC_CONS = 9;                               // named barrier of the consumer warpgroups
constexpr int kTcHeaderBytes = 2048;                         // mbarriers, small scratch
constexpr long long kTcTimeoutCycles = 2000000000LL;         // ~1 s: trap instead of hanging

struct LmHeadTcArgs {
  const unsigned char* W;     // canonical-packed weights [n_tiles][K / 64][16 KiB]
  int n_tiles;                // ceil(local vocab / 128)
  int K;                      // hidden (multiple of 64)
  int M;                      // valid token rows (<= 16)
  int n_stages;               // ring depth
  const float* x_f32;         // residual rows [M][x_ld]
  int x_ld;
  const __nv_bfloat16* norm_w;
  float eps;
  float* logits;              // optional [M][logits_ld]
  int logits_ld;
  int n_valid_rows;           // local vocab rows
  int vocab_off;              // global id of local row 0
  float* part_val;            // [grid][16]
  int* part_idx;
};

__host__ __device__ inline size_t lmhead_tc_smem_bytes(int K, int n_stages) {
  return (size_t)kTcHeaderBytes + (size_t)n_stages * kTcStageBytes + (size_t)kTcTokens * K * 2;
}

// ---- wgmma primitives (PTX ISA: "Asynchronous Warpgroup Level Matrix Multiply-Accumulate")
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// shared-memory matrix descriptor: start address, leading / stride byte offsets, layout type in
// bits 62-63 (0 = no swizzle, 1 = 128-byte swizzle)
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes,
                                               uint32_t layout) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32) | ((uint64_t)layout << 62);
}

// D[64 x 16] (+)= A[64 x 16] * B[16 x 16]^T, bf16 in, fp32 accumulate, both operands K-major in
// shared memory.  Accumulator fragment: d[j] holds row 16 (warp % 4) + lane / 4 + 8 ((j & 3) >> 1),
// column 8 (j >> 2) + 2 (lane % 4) + (j & 1) — the mma.sync C layout repeated over N / 8.
__device__ __forceinline__ void wgmma_m64n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(accumulate));
}

// bounded mbarrier wait: a protocol bug must surface as a launch failure, not as a hung GPU
__device__ __forceinline__ void mbar_wait_bounded(uint64_t* bar, uint32_t parity) {
  const long long t0 = clock64();
  uint32_t done = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    if (!done && clock64() - t0 > kTcTimeoutCycles) __trap();
  }
}

// natural [rows, K] bf16 -> canonical tiles (see header); rows >= n_rows are zero
__global__ void pack_canonical_kernel(const __nv_bfloat16* __restrict__ src, int64_t src_ld, int64_t row0,
                                      int64_t n_rows, int64_t K, uint4* __restrict__ dst, int64_t n_tiles) {
  const int64_t kst = K / kTcStageK;
  const int64_t total = n_tiles * kst * (kTcStageBytes / 16);
  for (int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; c < total; c += (int64_t)gridDim.x * blockDim.x) {
    const int64_t blk = c / (kTcStageBytes / 16);          // (tile, k stage)
    const int in = (int)(c % (kTcStageBytes / 16));        // 16-byte chunk inside the stage
    const int64_t tile = blk / kst, s = blk % kst;
    const int core = in >> 3, r = in & 7;                  // core = i * 8 + j
    const int i = core >> 3, j = core & 7;
    const int64_t row = tile * kTcTileRows + i * 8 + r;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (row < n_rows) v = *reinterpret_cast<const uint4*>(src + (row0 + row) * src_ld + s * kTcStageK + j * 8);
    dst[c] = v;
  }
}

__global__ void __launch_bounds__(kTcThreads, 1)
lmhead_tc_kernel(const LmHeadTcArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty_bar = full_bar + kTcMaxStages;
  float* stat = reinterpret_cast<float*>(smem + 256);       // [8 warps][16] + rstd[16]   (576 B)
  float* xval = reinterpret_cast<float*>(smem + 1024);      // [8 warps][16] cross-warp arg-max
  int* xi = reinterpret_cast<int*>(smem + 1536);            // [8 warps][16]
  unsigned char* ring = smem + kTcHeaderBytes;
  unsigned char* xb = ring + (size_t)a.n_stages * kTcStageBytes;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int NS = a.n_stages;
  const int n_kst = a.K / kTcStageK;

  if (tid == 0) {
    for (int s = 0; s < NS; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kTcConsumerThreads); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  pdl_launch_dependents();
  if (warp < 4) {
    if (tid == 0) {
      // ============================================================ TMA PRODUCER (weights are static:
      // it runs ahead of the PDL dependency, like gemm_producer)
      uint32_t q = 0;
      for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x)
        for (int s = 0; s < n_kst; ++s, ++q) {
          const int st = q % NS;
          mbar_wait_bounded(&empty_bar[st], ((q / NS) & 1) ^ 1);
          mbar_arrive_expect_tx(&full_bar[st], kTcStageBytes);
          tma_bulk_g2s(ring + (size_t)st * kTcStageBytes,
                       a.W + ((size_t)tile * n_kst + s) * kTcStageBytes, kTcStageBytes, &full_bar[st]);
        }
    }
    pdl_wait();                                      // completion stays transitive along the PDL chain
    return;
  }
  pdl_wait();
  // ---------------------------------------------------------------- prologue (consumers): RMSNorm
  // of the token rows -> bf16 B operand in the canonical K-major layout.  The producer must NOT
  // take part: its progress depends on the MMAs, which depend on this prologue.
  const int ctid = tid - 128, cwarp = warp - 4, wg = cwarp >> 2;
  const int nvec = a.K >> 2;
  for (int m = 0; m < a.M; ++m) {
    const float4* xr = reinterpret_cast<const float4*>(a.x_f32 + (size_t)m * a.x_ld);
    float ss = 0.f;
    for (int idx = ctid; idx < nvec; idx += kTcConsumerThreads) {
      const float4 v = xr[idx];
      ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    ss = warp_sum(ss);
    if (lane == 0) stat[cwarp * 16 + m] = ss;
  }
  bar_sync(BAR_TC_CONS, kTcConsumerThreads);
  if (ctid < a.M) {
    float tot = 0.f;
    for (int w = 0; w < kTcConsumerThreads / 32; ++w) tot += stat[w * 16 + ctid];
    stat[8 * 16 + ctid] = rsqrtf(tot / (float)a.K + a.eps);
  }
  bar_sync(BAR_TC_CONS, kTcConsumerThreads);
  for (int m = 0; m < kTcTokens; ++m) {
    const float rstd = m < a.M ? stat[8 * 16 + m] : 0.f;
    const float4* xr = reinterpret_cast<const float4*>(a.x_f32 + (size_t)(m < a.M ? m : 0) * a.x_ld);
    for (int idx = ctid; idx < nvec; idx += kTcConsumerThreads) {   // 4 consecutive k: half a 16-B chunk
      uint2 o = make_uint2(0u, 0u);
      if (m < a.M) {
        const float4 v = xr[idx];
        const uint2 wv = *reinterpret_cast<const uint2*>(a.norm_w + idx * 4);
        o.x = pack_bf16x2(bf16_lo(wv.x) * (v.x * rstd), bf16_hi(wv.x) * (v.y * rstd));
        o.y = pack_bf16x2(bf16_lo(wv.y) * (v.z * rstd), bf16_hi(wv.y) * (v.w * rstd));
      }
      const int k = idx * 4, j = k >> 3;
      *reinterpret_cast<uint2*>(xb + ((size_t)j * 2 + (m >> 3)) * 128 + (m & 7) * 16 + (k & 7) * 2) = o;
    }
  }
  // generic-proxy writes -> visible to the tensor core's async-proxy reads
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  bar_sync(BAR_TC_CONS, kTcConsumerThreads);

  // ================================================================ MMA + EPILOGUE (64 rows per warpgroup)
  const uint32_t xb_addr = smem_u32(xb);
  const int r_lo = (cwarp & 3) * 16 + (lane >> 2);   // accumulator rows r_lo and r_lo + 8 of this warpgroup
  float best_v[4];                                   // tokens 8 (i >> 1) + 2 (lane % 4) + (i & 1)
  int best_i[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { best_v[i] = -INFINITY; best_i[i] = 0x7fffffff; }
  uint32_t q = 0;
  for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
    float d[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) d[j] = 0.f;
    for (int s = 0; s < n_kst; ++s, ++q) {
      const int st = q % NS;
      mbar_wait_bounded(&full_bar[st], (q / NS) & 1);
      const uint32_t a_addr = smem_u32(ring + (size_t)st * kTcStageBytes) + wg * 8192;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kTcStageK / 16; ++k)
        wgmma_m64n16(d, wgmma_desc(a_addr + k * 256, 128, 1024, 0),
                     wgmma_desc(xb_addr + (uint32_t)(s * 8 + k * 2) * 256, 256, 128, 0), (s > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      if (s > 0) {                                   // the previous stage's MMAs are done reading it
        wgmma_wait<1>();
        mbar_arrive(&empty_bar[(q - 1) % NS]);
      }
    }
    wgmma_wait<0>();
    mbar_arrive(&empty_bar[(q - 1) % NS]);
    const int row0 = tile * kTcTileRows + wg * 64 + r_lo;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int m = 8 * (j >> 2) + 2 * (lane & 3) + (j & 1);
      const int orow = row0 + 8 * ((j & 3) >> 1);
      const int bi_slot = 2 * (j >> 2) + (j & 1);
      if (m < a.M && orow < a.n_valid_rows) {
        if (a.logits != nullptr) a.logits[(size_t)m * a.logits_ld + orow] = d[j];
        if (better(d[j], orow, best_v[bi_slot], best_i[bi_slot])) { best_v[bi_slot] = d[j]; best_i[bi_slot] = orow; }
      }
    }
  }
  // lanes with the same lane % 4 hold the same tokens: reduce over lane / 4, then across warps
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best_v[i], o);
      const int oi = __shfl_xor_sync(0xffffffffu, best_i[i], o);
      if (better(ov, oi, best_v[i], best_i[i])) { best_v[i] = ov; best_i[i] = oi; }
    }
  }
  if (lane < 4) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = 8 * (i >> 1) + 2 * lane + (i & 1);
      xval[cwarp * kTcTokens + m] = best_v[i];
      xi[cwarp * kTcTokens + m] = best_i[i];
    }
  }
  bar_sync(BAR_TC_CONS, kTcConsumerThreads);
  if (ctid < a.M) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int w = 0; w < kTcConsumerThreads / 32; ++w)
      if (better(xval[w * kTcTokens + ctid], xi[w * kTcTokens + ctid], bv, bi)) {
        bv = xval[w * kTcTokens + ctid];
        bi = xi[w * kTcTokens + ctid];
      }
    a.part_val[blockIdx.x * kMaxRows + ctid] = bv;
    a.part_idx[blockIdx.x * kMaxRows + ctid] = (bi == 0x7fffffff) ? 0x7fffffff : bi + a.vocab_off;
  }
}

}  // namespace lsk
