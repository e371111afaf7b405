// gemm_skinny.cuh — weight-streaming "skinny" GEMM for decode shapes:
//     y[m, n] = sum_k x[m, k] * W[n, k]        m <= 16 tokens,  W bf16 [N, K] (HF layout)
// HBM-bound by construction (arithmetic intensity <= 16 flop/B).  PRE-SHUFFLED weights are
// streamed by the TMA engine (1-D cp.async.bulk, global -> shared, mbarrier completion) through
// a multi-stage shared-memory ring: ~100 KB per SM in flight with no L1 miss tracking involved
// (a plain LDG path cannot keep enough bytes in flight per SM to reach HBM bandwidth).  Consumer warps
// lift mma.sync A-fragments out of the ring with conflict-free 128-bit shared loads; the (tiny)
// activation block is resident in shared memory as the B operand.
//
// Packed weight layout (built once by pack_rows_kernel, see engine.cu):
//   tile   = 16 consecutive output rows,  super-block (sb) = 32 consecutive k
//   for each (tile, sb): 2 MMAs x 32 lanes x 16 B   = 1 KiB, contiguous, tile-major
//   lane (g = lane/4, t = lane%4), MMA j holds  a0..a3 =
//        W[g   ][32sb + 8t + 4j + {0,1}],  W[g+8][.. same ..],
//        W[g   ][32sb + 8t + 4j + {2,3}],  W[g+8][.. same ..]
//   i.e. the physical k order inside a super-block is permuted so that a lane's B operand for
//   both MMAs is ONE 128-bit shared-memory load of x[token g][32sb + 8t .. 8t+7].
//
// Numerics are batch-invariant: an output element is accumulated in the same order whatever
// the number of token rows, so a row computed alone (draft / AR, m = 1) is bit-identical to
// the same row computed inside a verify block (m = D+1).
#pragma once
#include "common.cuh"
#include "tp_peer.cuh"

namespace lsk {

enum { PRO_RMS = 0, PRO_BF16 = 1 };
// EPI_PUSH (tensor parallel, opt-in): like EPI_STORE, but the fp32 tile goes straight into every
// rank's peer-visible region over NVLink while the kernel is still streaming (tp_peer.cuh)
// EPI_QKV_SEQS (batched rounds): EPI_QKV on the rows of several sequences (GemmArgs::seq_rows); a
// separate instantiation, so the single-sequence epilogue stays as it is
enum { EPI_QKV = 0, EPI_RESID = 1, EPI_STORE = 2, EPI_SILU = 3, EPI_LMHEAD = 4, EPI_PUSH = 5, EPI_QKV_SEQS = 6 };

constexpr int kGemmWarps = 16;                       // consumer warps (LDS + MMA)
constexpr int kEpiWarps = 3;                         // reduction / epilogue warps
constexpr int kConsumerThreads = kGemmWarps * 32;    // 512
constexpr int kEpiThreads = kEpiWarps * 32;          // 96
constexpr int kGemmThreads = kConsumerThreads + 32 + kEpiThreads;   // + 1 producer warp = 640
constexpr int kWorkThreads = kConsumerThreads + kEpiThreads;        // everyone but the producer
constexpr int kProducerWarp = kGemmWarps;            // warp 16
#ifndef LSK_STAGE_SBS
#define LSK_STAGE_SBS 16
#endif
constexpr int kStageSbs = LSK_STAGE_SBS;             // super-blocks (1 KiB each) per ring stage
constexpr int kStageBytes = kStageSbs * 1024;
constexpr int kMaxStages = 128 / LSK_STAGE_SBS;      // ring capped at 128 KiB
constexpr int kMaxTilesPerPass = 2;

// named barriers (0 is __syncthreads)
enum { BAR_FULL0 = 1, BAR_FULL1 = 2, BAR_EMPTY0 = 3, BAR_EMPTY1 = 4, BAR_EPI = 5, BAR_CONS = 6,
       BAR_WORK = 7 };
__device__ __forceinline__ void bar_sync(int id, int n) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory");
}
__device__ __forceinline__ void bar_arrive(int id, int n) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory");
}
struct GemmArgs {
  const uint4* W;       // packed weights
  int n_tiles;          // N / 16
  int nsb;              // K / 32
  int K;
  int M;                // valid token rows
  // ---- schedule (host-planned, see plan_gemm in engine.cu)
  int tiles_per_pass;   // 1 or 2 tiles accumulated side by side (needed when K is chunked)
  int n_chunks;         // K chunks whose activations are resident at a time
  int kc_sbs;           // super-blocks per chunk (multiple of kStageSbs unless n_chunks == 1)
  int n_stages;         // ring depth
  int xs_rows;          // activation rows resident in shared memory (= M; absent rows read as 0)
  // ---- prologue
  const float* x_f32;   // PRO_RMS: residual-stream rows [M][x_ld] fp32
  int x_ld;
  const __nv_bfloat16* norm_w;
  float eps;
  const __nv_bfloat16* x_bf16;  // PRO_BF16: activations [M][xb_ld]
  int xb_ld;
  // ---- epilogue: RESID (+=) / STORE (=)
  float* out_f32;
  int out_ld;
  // ---- SILU: act[m][8*tile + r] = silu(gate) * up
  __nv_bfloat16* act;
  int act_ld;
  // ---- QKV: RoPE, q -> q_out, k/v -> paged cache
  __nv_bfloat16* q_out;
  int q_ld;
  __nv_bfloat16* kpool;  // layer base
  __nv_bfloat16* vpool;
  const int* page_table;
  const int* base_len;
  int pos_off;
  // EPI_QKV_SEQS: row m belongs to sequence s = m / seq_rows, sits at position
  // base_len[s * len_stride] + pos_off + m % seq_rows and writes through the page-table view
  // page_table + s * seq_pages (EPI_QKV: every row is one sequence's, at *base_len + pos_off + m)
  int seq_rows, len_stride, seq_pages;
  const float2* rope;    // [max_pos][head_dim / 2] (cos, sin)
  int head_dim;
  int q_rows;            // local q rows (heads * head_dim)
  int kv_rows;           // local kv rows
  int n_kv_heads;        // local
  // ---- LMHEAD
  float* logits;         // optional [M][logits_ld]
  int logits_ld;
  int n_valid_rows;      // local vocab rows (<= n_tiles*16)
  int vocab_off;         // global id of local row 0
  float* part_val;       // [grid][16]
  int* part_idx;
};

// EPI_QKV_SEQS: position of token row m, and the first page-table entry of its sequence's view in
// *view
__device__ __forceinline__ int qkv_seq_pos(const GemmArgs& a, int m, int* view) {
  const int s = m / a.seq_rows;
  *view = s * a.seq_pages;
  return a.base_len[s * a.len_stride] + a.pos_off + (m - s * a.seq_rows);
}

__host__ __device__ inline int gemm_x_stride_bytes(int kcols) {
  return ((2 * kcols + 127) / 128) * 128 + 64;   // == 64 (mod 128): conflict-free LDS.128
}

// shared-memory carve-up (host and device must agree).  Fixed part: mbarriers + ring; the
// SCRATCH region behind it holds, per GEMM, the activation block, the partial-tile slots, RMS
// statistics and the LM-head logits tile.
constexpr int kBarBytes = 1024;
struct GemmScratch {
  size_t xs, red, stat, lg, total;
};
__host__ __device__ inline GemmScratch gemm_scratch_layout(int NT, int xs_rows, int kc_cols, int tpp, int epi) {
  GemmScratch L;
  size_t off = 0;
  L.xs = off;   off += (size_t)xs_rows * gemm_x_stride_bytes(kc_cols);
  L.red = off;  off += (size_t)2 * tpp * kGemmWarps * NT * 128 * 4;
  L.stat = off; off += (size_t)(kGemmWarps + kEpiWarps + 1) * NT * 8 * 4;
  L.lg = off;   if (epi == EPI_LMHEAD) off += (size_t)NT * 8 * (tpp * 16) * 4;
  L.total = (off + 127) & ~(size_t)127;
  return L;
}
__host__ __device__ inline size_t gemm_smem_total(int n_stages, size_t scratch_bytes) {
  return (size_t)kBarBytes + (size_t)n_stages * kStageBytes + scratch_bytes;
}

// Per-CTA pipeline context shared by the three warp roles.
struct GemmCtx {
  unsigned char* ring;
  uint64_t* full_bar;
  uint64_t* empty_bar;
  unsigned char* scratch;
  int NS;
};
__device__ __forceinline__ GemmCtx make_ctx(unsigned char* smem, int n_stages) {
  GemmCtx c;
  c.full_bar = reinterpret_cast<uint64_t*>(smem);
  c.empty_bar = c.full_bar + kMaxStages;
  c.ring = smem + kBarBytes;
  c.scratch = c.ring + (size_t)n_stages * kStageBytes;
  c.NS = n_stages;
  return c;
}
__device__ __forceinline__ void ctx_init_barriers(const GemmCtx& c) {   // one thread
  for (int s = 0; s < c.NS; ++s) {
    mbar_init(&c.full_bar[s], 1);
    mbar_init(&c.empty_bar[s], kGemmWarps);
  }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// ---------------------------------------------------------------------------------------------
// PRODUCER (one lane): walk this CTA's weight byte stream, tile after tile in 16 KiB stages, and
// issue TMA bulk copies into the ring as slots free up.  `q` counts stages over the kernel's
// lifetime.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void gemm_producer(const GemmArgs& a, const GemmCtx& c, uint32_t& q) {
  const int TPP = a.tiles_per_pass;
  const int n_slots = (a.n_tiles + TPP - 1) / TPP;
  for (int slot = blockIdx.x; slot < n_slots; slot += gridDim.x) {
    for (int kc = 0; kc < a.n_chunks; ++kc) {
      const int sb_lo = kc * a.kc_sbs;
      const int sb_hi = min(a.nsb, sb_lo + a.kc_sbs);
      for (int j = 0; j < TPP; ++j) {
        const int tile = slot * TPP + j;
        if (tile >= a.n_tiles) break;
        const unsigned char* src = reinterpret_cast<const unsigned char*>(a.W) +
                                   ((size_t)tile * a.nsb + sb_lo) * 1024;
        for (int sb = sb_lo; sb < sb_hi; sb += kStageSbs, ++q) {
          const int cnt = min(kStageSbs, sb_hi - sb);
          const int s = q % c.NS;
          mbar_wait(&c.empty_bar[s], ((q / c.NS) & 1) ^ 1);
          mbar_arrive_expect_tx(&c.full_bar[s], (uint32_t)cnt * 1024);
          tma_bulk_g2s(c.ring + (size_t)s * kStageBytes, src + (size_t)(sb - sb_lo) * 1024,
                       (uint32_t)cnt * 1024, &c.full_bar[s]);
        }
      }
    }
  }
}

// fills the resident activation chunk kc (bf16 source); callers sync around it
template <int NT>
__device__ __forceinline__ void gemm_load_x_bf16(const GemmArgs& a, unsigned char* xs, int XS,
                                                 int kc_cols, int kc, int ltid, int nthreads) {
  const int col0 = kc * kc_cols;
  const int cols = min(a.K - col0, kc_cols);
  const int nvec = cols >> 3;                // uint4 (8 bf16) per row
  const int zvec = kc_cols >> 3;
  // four rows per step: their loads are issued together (one L2 round trip per step instead of
  // one per row)
  for (int m0 = 0; m0 < a.xs_rows; m0 += 4) {
    for (int idx = ltid; idx < zvec; idx += nthreads) {
      uint4 v[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        v[r] = make_uint4(0, 0, 0, 0);
        if (m0 + r < a.M && idx < nvec)
          v[r] = *reinterpret_cast<const uint4*>(a.x_bf16 + (size_t)(m0 + r) * a.xb_ld + col0 + idx * 8);
      }
#pragma unroll
      for (int r = 0; r < 4; ++r)
        if (m0 + r < a.xs_rows) *reinterpret_cast<uint4*>(xs + (size_t)(m0 + r) * XS + idx * 16) = v[r];
    }
  }
}

// K-chunked RMSNorm mode: chunk kc of the fp32 residual rows -> normalised bf16 activation chunk,
// with the rstd the prologue left in `rstd[m]`; same rounding as the resident mode
// (bf16(w * (x * rstd)), modeling_llama.py:52-70).  Four rows per step, loads issued together.
template <int NT>
__device__ __forceinline__ void gemm_load_x_rms(const GemmArgs& a, unsigned char* xs, int XS, int kc_cols,
                                                int kc, const float* rstd, int ltid, int nthreads) {
  const int col0 = kc * kc_cols;
  const int cols = min(a.K - col0, kc_cols);
  const int nvec = cols >> 2;                // float4 per row in this chunk
  const int zvec = kc_cols >> 2;
  for (int m0 = 0; m0 < a.xs_rows; m0 += 4) {
    for (int idx = ltid; idx < zvec; idx += nthreads) {
      float4 v[4];
      uint2 wv = make_uint2(0, 0);
      if (idx < nvec) wv = *reinterpret_cast<const uint2*>(a.norm_w + col0 + idx * 4);
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        v[r] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (m0 + r < a.M && idx < nvec)
          v[r] = *reinterpret_cast<const float4*>(a.x_f32 + (size_t)(m0 + r) * a.x_ld + col0 + idx * 4);
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int m = m0 + r;
        if (m >= a.xs_rows) continue;
        uint2 o = make_uint2(0u, 0u);
        if (m < a.M && idx < nvec) {
          const float rs = rstd[m];
          o.x = pack_bf16x2(bf16_lo(wv.x) * (v[r].x * rs), bf16_hi(wv.x) * (v[r].y * rs));
          o.y = pack_bf16x2(bf16_lo(wv.y) * (v[r].z * rs), bf16_hi(wv.y) * (v[r].w * rs));
        }
        *reinterpret_cast<uint2*>(xs + (size_t)m * XS + idx * 8) = o;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// PROLOGUE (consumer + epilogue warps, kWorkThreads): activations -> bf16 rows in scratch.
// Ends with a BAR_WORK sync.
// ---------------------------------------------------------------------------------------------
// PRO_RMS: the norm weights are WEIGHTS — the stand-alone kernel loads them before the PDL
// dependency resolves (gemm_preload_norm) and hands them in through `wreg`.
__device__ __forceinline__ void gemm_preload_norm(const GemmArgs& a, int wtid, uint2 (&wreg)[4]) {
  const int nvec = a.K >> 2;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = wtid + i * kWorkThreads;
    wreg[i] = idx < nvec ? *reinterpret_cast<const uint2*>(a.norm_w + idx * 4) : make_uint2(0, 0);
  }
}

// ROWS residual rows at a time: each thread pulls its VEC float4 slices of all ROWS rows into
// registers at once, the group's sums of squares are reduced across the work threads (2 barriers),
// and the rows are normalised out of registers into the activation block.
template <int NT, int ROWS, int VEC, bool STATS_ONLY = false>
__device__ __forceinline__ void rms_rows_group(const GemmArgs& a, unsigned char* xs, int XS, int kc_cols,
                                               float* stat, int wtid, int swarp, int lane,
                                               const uint2 (&wreg)[4]) {
  constexpr int kStatWarps = kGemmWarps + kEpiWarps;
  const int nvec = a.K >> 2;
#pragma unroll 1
  for (int m0 = 0; m0 < a.xs_rows; m0 += ROWS) {
    float4 v[ROWS][VEC];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      const float4* xr = reinterpret_cast<const float4*>(a.x_f32 + (size_t)(m0 + r) * a.x_ld);
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const int idx = wtid + i * kWorkThreads;
        v[r][i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (m0 + r < a.M && idx < nvec) v[r][i] = xr[idx];
      }
    }
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      float ss = 0.f;
#pragma unroll
      for (int i = 0; i < VEC; ++i)
        ss += v[r][i].x * v[r][i].x + v[r][i].y * v[r][i].y + v[r][i].z * v[r][i].z + v[r][i].w * v[r][i].w;
      ss = warp_sum(ss);
      if (lane == 0) stat[swarp * (NT * 8) + m0 + r] = ss;
    }
    bar_sync(BAR_WORK, kWorkThreads);
    if (wtid < ROWS) {
      float tot = 0.f;
      for (int w = 0; w < kStatWarps; ++w) tot += stat[w * (NT * 8) + m0 + wtid];
      stat[kStatWarps * NT * 8 + m0 + wtid] = rsqrtf(tot / (float)a.K + a.eps);
    }
    bar_sync(BAR_WORK, kWorkThreads);
    if (STATS_ONLY) continue;                  // K-chunked mode: rows are normalised per chunk later
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      const int m = m0 + r;
      if (m >= a.xs_rows) continue;
      if (m < a.M) {
        const float rstd = stat[kStatWarps * NT * 8 + m];
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          const int idx = wtid + i * kWorkThreads;
          if (idx < nvec) {
            const float4 x4 = v[r][i];
            const uint2 wv = wreg[i];
            uint2 o;
            o.x = pack_bf16x2(bf16_lo(wv.x) * (x4.x * rstd), bf16_hi(wv.x) * (x4.y * rstd));
            o.y = pack_bf16x2(bf16_lo(wv.y) * (x4.z * rstd), bf16_hi(wv.y) * (x4.w * rstd));
            *reinterpret_cast<uint2*>(xs + (size_t)m * XS + idx * 8) = o;
          }
        }
      } else {
        for (int idx = wtid; idx < (kc_cols >> 3); idx += kWorkThreads)
          *reinterpret_cast<uint4*>(xs + (size_t)m * XS + idx * 16) = make_uint4(0, 0, 0, 0);
      }
    }
  }
}

template <int NT, int PRO>
__device__ __forceinline__ void gemm_prologue(const GemmArgs& a, const GemmCtx& c, int epi,
                                              int wtid, int swarp, int lane, const uint2 (&wreg)[4]) {
  const int kc_cols = a.kc_sbs * 32;
  const GemmScratch L = gemm_scratch_layout(NT, a.xs_rows, kc_cols, a.tiles_per_pass, epi);
  const int XS = gemm_x_stride_bytes(kc_cols);
  unsigned char* xs = c.scratch + L.xs;
  float* stat = reinterpret_cast<float*>(c.scratch + L.stat);
  constexpr int kStatWarps = kGemmWarps + kEpiWarps;
  if (PRO == PRO_RMS) {
    // RMSNorm of the fp32 residual rows -> bf16 (rounding point of a bf16 HF model:
    // modeling_llama.py:52-70).  n_chunks == 1 here.  Rows are processed FOUR at a time: each thread
    // pulls its <= 4 float4 slices of all four rows into registers at once (one L2 round trip per
    // group instead of two per row), reduces, and normalises out of registers.
    // K <= 4864: 2 slices per thread and row -> groups of 4 rows; larger K: 4 slices -> groups of 2.
    // (Groups of 8 rows would need 64 live registers, which spill inside the 96-register budget of
    // the 640-thread CTA.)
    // K-chunked (n_chunks > 1: 16-row blocks at hidden > 4096): only the statistics here — the SAME
    // reduction as the resident mode, so a row's rstd does not depend on how the block is staged —
    // and gemm_load_x_rms normalises each chunk when the consumers swap it in.
    if (a.n_chunks > 1) {
      if ((a.K >> 2) <= 2 * kWorkThreads) rms_rows_group<NT, 4, 2, true>(a, xs, XS, kc_cols, stat, wtid, swarp, lane, wreg);
      else rms_rows_group<NT, 2, 4, true>(a, xs, XS, kc_cols, stat, wtid, swarp, lane, wreg);
    } else if ((a.K >> 2) <= 2 * kWorkThreads) rms_rows_group<NT, 4, 2>(a, xs, XS, kc_cols, stat, wtid, swarp, lane, wreg);
    else rms_rows_group<NT, 2, 4>(a, xs, XS, kc_cols, stat, wtid, swarp, lane, wreg);
  } else if (a.n_chunks == 1) {
    gemm_load_x_bf16<NT>(a, xs, XS, kc_cols, 0, wtid, kWorkThreads);
  }
  bar_sync(BAR_WORK, kWorkThreads);
}

// ---------------------------------------------------------------------------------------------
// CONSUMER warps (0..15): warp w owns super-block w of every stage (interleaved 16-way K split).
// ---------------------------------------------------------------------------------------------
template <int NT>
__device__ __forceinline__ void gemm_consume(const GemmArgs& a, const GemmCtx& c, int epi,
                                             uint32_t& q, int tid, int warp, int lane) {
  const int TPP = a.tiles_per_pass;
  const int kc_cols = a.kc_sbs * 32;
  const GemmScratch L = gemm_scratch_layout(NT, a.xs_rows, kc_cols, TPP, epi);
  const int XS = gemm_x_stride_bytes(kc_cols);
  unsigned char* xs = c.scratch + L.xs;
  float* red = reinterpret_cast<float*>(c.scratch + L.red);
  const int kRedFloats = TPP * kGemmWarps * NT * 128;     // one buffer
  const int g = lane >> 2, t = lane & 3;
  const int n_slots = (a.n_tiles + TPP - 1) / TPP;
  const int NS = c.NS;
  const unsigned char* xlane = xs + (size_t)g * XS + t * 16;
  bool row_ok[NT];                       // rows beyond xs_rows are not resident: B fragment = 0
#pragma unroll
  for (int n = 0; n < NT; ++n) row_ok[n] = (n * 8 + g) < a.xs_rows;
  int it = 0;
  for (int slot = blockIdx.x; slot < n_slots; slot += gridDim.x, ++it) {
    float acc[kMaxTilesPerPass][NT][2][4];
#pragma unroll
    for (int j = 0; j < kMaxTilesPerPass; ++j)
#pragma unroll
      for (int n = 0; n < NT; ++n)
#pragma unroll
        for (int h = 0; h < 2; ++h) acc[j][n][h][0] = acc[j][n][h][1] = acc[j][n][h][2] = acc[j][n][h][3] = 0.f;

    for (int kc = 0; kc < a.n_chunks; ++kc) {
      if (a.n_chunks > 1) {            // swap the resident activation chunk
        bar_sync(BAR_CONS, kConsumerThreads);
        if (a.x_f32 != nullptr && a.norm_w != nullptr) {   // PRO_RMS, K-chunked
          const float* rstd = reinterpret_cast<const float*>(c.scratch + L.stat) + (kGemmWarps + kEpiWarps) * NT * 8;
          gemm_load_x_rms<NT>(a, xs, XS, kc_cols, kc, rstd, tid, kConsumerThreads);
        } else {
          gemm_load_x_bf16<NT>(a, xs, XS, kc_cols, kc, tid, kConsumerThreads);
        }
        bar_sync(BAR_CONS, kConsumerThreads);
      }
      const int sb_lo = kc * a.kc_sbs;
      const int sb_hi = min(a.nsb, sb_lo + a.kc_sbs);
#pragma unroll
      for (int j = 0; j < kMaxTilesPerPass; ++j) {
        if (j < TPP && slot * TPP + j < a.n_tiles) {
          for (int sb = sb_lo; sb < sb_hi; sb += kStageSbs, ++q) {
            const int s = q % NS;
            mbar_wait(&c.full_bar[s], (q / NS) & 1);
#pragma unroll
            for (int w2 = 0; w2 < (kStageSbs + kGemmWarps - 1) / kGemmWarps; ++w2) {
              const int wsb = warp + w2 * kGemmWarps;        // this warp's super-block(s) in the stage
              if (wsb < kStageSbs && sb + wsb < sb_hi) {
                const unsigned char* ap = c.ring + (size_t)s * kStageBytes + wsb * 1024 + lane * 16;
                const uint4 a0 = *reinterpret_cast<const uint4*>(ap);
                const uint4 a1 = *reinterpret_cast<const uint4*>(ap + 512);
#pragma unroll
                for (int n = 0; n < NT; ++n) {
                  uint4 b = make_uint4(0, 0, 0, 0);
                  if (row_ok[n])
                    b = *reinterpret_cast<const uint4*>(
                        xlane + (size_t)n * 8 * XS + (size_t)(sb + wsb - sb_lo) * 64);
                  mma_bf16_16816(acc[j][n][0], a0.x, a0.y, a0.z, a0.w, b.x, b.y);
                  mma_bf16_16816(acc[j][n][1], a1.x, a1.y, a1.z, a1.w, b.z, b.w);
                }
              }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&c.empty_bar[s]);
          }
        }
      }
    }

    const int buf = it & 1;
    if (it >= 2) bar_sync(BAR_EMPTY0 + buf, kWorkThreads);   // epilogue released this slot
    float* rbase = red + buf * kRedFloats;
#pragma unroll
    for (int j = 0; j < kMaxTilesPerPass; ++j) {
      if (j < TPP) {
#pragma unroll
        for (int n = 0; n < NT; ++n) {
          float* r = rbase + (((j * kGemmWarps + warp) * NT + n) * 16) * 8;
          *reinterpret_cast<float2*>(r + g * 8 + 2 * t) =
              make_float2(acc[j][n][0][0] + acc[j][n][1][0], acc[j][n][0][1] + acc[j][n][1][1]);
          *reinterpret_cast<float2*>(r + (g + 8) * 8 + 2 * t) =
              make_float2(acc[j][n][0][2] + acc[j][n][1][2], acc[j][n][0][3] + acc[j][n][1][3]);
        }
      }
    }
    bar_arrive(BAR_FULL0 + buf, kWorkThreads);
  }
}

// ---------------------------------------------------------------------------------------------
// EPILOGUE warps (17..19): fixed-order reduction over the 16 K-slices + fused epilogue.
// ---------------------------------------------------------------------------------------------
template <int NT, int EPI>
__device__ __forceinline__ void gemm_epilogue_role(const GemmArgs& a, const GemmCtx& c, int etid,
                                                   int ewarp, int lane,
                                                   const PeerComm* pc = nullptr) {
  const int TPP = a.tiles_per_pass;
  const int kc_cols = a.kc_sbs * 32;
  const GemmScratch L = gemm_scratch_layout(NT, a.xs_rows, kc_cols, TPP, EPI);
  float* red = reinterpret_cast<float*>(c.scratch + L.red);
  float* lg = reinterpret_cast<float*>(c.scratch + L.lg);
  const int kRedFloats = TPP * kGemmWarps * NT * 128;
  const int n_slots = (a.n_tiles + TPP - 1) / TPP;
  constexpr int kRowsPerEwarp = (NT * 8 + kEpiWarps - 1) / kEpiWarps;
  float best_v[kRowsPerEwarp];                    // LMHEAD: running arg-max, rows ewarp + 3*i
  int best_i[kRowsPerEwarp];
#pragma unroll
  for (int i = 0; i < kRowsPerEwarp; ++i) { best_v[i] = -INFINITY; best_i[i] = 0x7fffffff; }

  // EPI_PUSH: where this rank's slot lives inside every rank's region for the current instance
  // (LL lines, tp_peer.cuh: {v0, epoch, v1, epoch} — the flag travels inside the data)
  unsigned int push_epoch = 0;
  size_t push_line0 = 0, push_ll = 0;
  if (EPI == EPI_PUSH) {
    const PeerRegionLayout PL = peer_region_layout(pc->size, pc->hidden);
    push_epoch = *reinterpret_cast<volatile unsigned int*>(peer_base(*pc, pc->rank) + PL.local) + 1u;
    push_line0 = ((size_t)(push_epoch & 1u) * pc->size + pc->rank) * ((size_t)kMaxRows * pc->hidden / 2);
    push_ll = PL.ll_data;
  }

  int it = 0;
  for (int slot = blockIdx.x; slot < n_slots; slot += gridDim.x, ++it) {
    const int buf = it & 1;
    // EPI_RESID: fetch the old residual values of this slot BEFORE waiting for the tile, so the
    // tail of the kernel has no dependent global round trip (each element has one owner thread)
    constexpr int kMaxItems = (kMaxTilesPerPass * NT * 128 + kEpiThreads - 1) / kEpiThreads;
    float old_resid[kMaxItems];
    if (EPI == EPI_RESID) {
#pragma unroll
      for (int k = 0; k < kMaxItems; ++k) {
        const int itx = etid + k * kEpiThreads;
        old_resid[k] = 0.f;
        if (itx < TPP * NT * 128) {
          const int row = itx & 15, tok = (itx >> 4) & 7, n = (itx >> 7) % NT, j = (itx >> 7) / NT;
          const int m = n * 8 + tok, tile = slot * TPP + j;
          if (m < a.M && tile < a.n_tiles) old_resid[k] = a.out_f32[(size_t)m * a.out_ld + tile * 16 + row];
        }
      }
    }
    // EPI_QKV: RoPE factors and KV page of this thread's items, fetched BEFORE the tile arrives
    // (the committed length is constant while the kernel runs) — same idea as old_resid
    constexpr bool kSeqs = EPI == EPI_QKV_SEQS;
    constexpr int kQkvItems = (kMaxTilesPerPass * NT * 64 + kEpiThreads - 1) / kEpiThreads;
    float2 q_cs[kQkvItems];
    int q_page[kQkvItems];
    if (EPI == EPI_QKV || kSeqs) {
      const int base_pos = kSeqs ? 0 : *a.base_len + a.pos_off;
      const int half = a.head_dim >> 1;
#pragma unroll
      for (int k = 0; k < kQkvItems; ++k) {
        const int itx = etid + k * kEpiThreads;
        q_cs[k] = make_float2(1.f, 0.f);
        q_page[k] = 0;
        if (itx < TPP * NT * 64) {
          const int tok = itx & 7, r = (itx >> 3) & 7, n = (itx >> 6) % NT, j = (itx >> 6) / NT;
          const int m = n * 8 + tok, tile = slot * TPP + j;
          if (m < a.M && tile < a.n_tiles) {
            const int pr = tile * 16;
            int pos = base_pos + m, view = 0;
            if (kSeqs) pos = qkv_seq_pos(a, m, &view);
            if (pr < a.q_rows + a.kv_rows) {
              const int rel = pr < a.q_rows ? pr : pr - a.q_rows;
              q_cs[k] = a.rope[(size_t)pos * half + ((rel % a.head_dim) >> 4) * 8 + r];
            }
            if (pr >= a.q_rows) q_page[k] = a.page_table[view + (pos >> 6)];
          }
        }
      }
    }
    bar_sync(BAR_FULL0 + buf, kWorkThreads);
    const float* rbase = red + buf * kRedFloats;
    auto ksum = [&](int j, int n, int row, int tok) {
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < kGemmWarps; ++k)
        s += rbase[(((j * kGemmWarps + k) * NT + n) * 16 + row) * 8 + tok];
      return s;
    };

    if (EPI == EPI_QKV || kSeqs || EPI == EPI_SILU) {
      const int items = TPP * NT * 64;
#pragma unroll
      for (int kq = 0; kq < kQkvItems; ++kq) {
        const int itx = etid + kq * kEpiThreads;
        if (itx >= items) continue;
        const int tok = itx & 7, r = (itx >> 3) & 7, n = (itx >> 6) % NT, j = (itx >> 6) / NT;
        const int m = n * 8 + tok;
        const int tile = slot * TPP + j;
        if (m >= a.M || tile >= a.n_tiles) continue;
        const float lo = ksum(j, n, r, tok), hi = ksum(j, n, r + 8, tok);
        if (EPI == EPI_SILU) {
          const float sg = lo / (1.f + __expf(-lo));
          a.act[(size_t)m * a.act_ld + tile * 8 + r] = __float2bfloat16_rn(sg * hi);
        } else {
          const int pr = tile * 16;                     // first packed row of the tile
          int view;
          const int pos = kSeqs ? qkv_seq_pos(a, m, &view) : *a.base_len + a.pos_off + m;
          const int HD = a.head_dim, half = HD >> 1;
          if (pr < a.q_rows + a.kv_rows) {              // q or k: rotary pair (d, d + HD/2)
            const bool is_q = pr < a.q_rows;
            const int rel = is_q ? pr : pr - a.q_rows;
            const int head = rel / HD, tt = (rel % HD) >> 4;
            const int d = tt * 8 + r;
            const float2 cs = q_cs[kq];
            const float o_lo = lo * cs.x - hi * cs.y;
            const float o_hi = hi * cs.x + lo * cs.y;
            if (is_q) {
              __nv_bfloat16* qd = a.q_out + (size_t)m * a.q_ld + head * HD;
              qd[d] = __float2bfloat16_rn(o_lo);
              qd[d + half] = __float2bfloat16_rn(o_hi);
            } else {
              const int page = q_page[kq];
              a.kpool[kv_elem_offset(HD, page, a.n_kv_heads, head, pos & 63, d)] = __float2bfloat16_rn(o_lo);
              a.kpool[kv_elem_offset(HD, page, a.n_kv_heads, head, pos & 63, d + half)] = __float2bfloat16_rn(o_hi);
            }
          } else {                                       // v: natural order, no rotation
            const int rel = pr - a.q_rows - a.kv_rows;
            const int head = rel / HD, d0 = rel % HD;
            const int page = q_page[kq];
            a.vpool[kv_elem_offset(HD, page, a.n_kv_heads, head, pos & 63, d0 + r)] = __float2bfloat16_rn(lo);
            a.vpool[kv_elem_offset(HD, page, a.n_kv_heads, head, pos & 63, d0 + r + 8)] = __float2bfloat16_rn(hi);
          }
        }
      }
    } else {
      const int items = TPP * NT * 128;
#pragma unroll
      for (int k = 0; k < kMaxItems; ++k) {
        const int itx = etid + k * kEpiThreads;
        if (itx >= items) continue;
        const int row = itx & 15, tok = (itx >> 4) & 7, n = (itx >> 7) % NT, j = (itx >> 7) / NT;
        const int m = n * 8 + tok;
        const int tile = slot * TPP + j;
        if (tile >= a.n_tiles) continue;
        const int orow = tile * 16 + row;
        const float v = (m < a.M) ? ksum(j, n, row, tok) : 0.f;
        if (EPI == EPI_RESID) {
          if (m < a.M) a.out_f32[(size_t)m * a.out_ld + orow] = old_resid[k] + v;
        } else if (EPI == EPI_STORE) {
          if (m < a.M) a.out_f32[(size_t)m * a.out_ld + orow] = v;
        } else if (EPI == EPI_PUSH) {
          // rows (orow, orow + 1) of one token -> one 16-byte line to every rank (own included);
          // `items` is a multiple of 32 and `tile` is warp-uniform, so the shuffle is convergent
          const float vn = __shfl_down_sync(0xffffffffu, v, 1);
          if (m < a.M && !(row & 1)) {
            const size_t line = push_line0 + ((size_t)m * pc->hidden + orow) / 2;
#pragma unroll
            for (int r = 0; r < kMaxPeers; ++r)
              if (r < pc->size)
                ll_store(reinterpret_cast<uint4*>(pc->base[r] + push_ll) + line, v, vn, push_epoch);
          }
        } else {  // LMHEAD
          if (m < a.M && a.logits != nullptr && orow < a.n_valid_rows)
            a.logits[(size_t)m * a.logits_ld + orow] = v;
          lg[m * (TPP * 16) + j * 16 + row] = v;
        }
      }
      if (EPI == EPI_LMHEAD) {
        bar_sync(BAR_EPI, kEpiThreads);
#pragma unroll
        for (int i = 0; i < kRowsPerEwarp; ++i) {
          const int m = ewarp + i * kEpiWarps;
          if (m < NT * 8 && m < a.M) {
            float bv = -INFINITY;
            int bi = 0x7fffffff;
            for (int cidx = lane; cidx < TPP * 16; cidx += 32) {
              const int orow = slot * TPP * 16 + cidx;
              if (orow < a.n_valid_rows && orow < a.n_tiles * 16) {
                const float v = lg[m * (TPP * 16) + cidx];
                if (better(v, orow, bv, bi)) { bv = v; bi = orow; }
              }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
              const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
              const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
              if (better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
            }
            if (better(bv, bi, best_v[i], best_i[i])) { best_v[i] = bv; best_i[i] = bi; }
          }
        }
        bar_sync(BAR_EPI, kEpiThreads);   // lg is rewritten by the next slot
      }
    }
    if (slot + 2 * gridDim.x < n_slots) bar_arrive(BAR_EMPTY0 + buf, kWorkThreads);
  }

  if (EPI == EPI_LMHEAD) {
#pragma unroll
    for (int i = 0; i < kRowsPerEwarp; ++i) {
      const int m = ewarp + i * kEpiWarps;
      if (m < NT * 8 && m < a.M && lane == 0) {
        a.part_val[blockIdx.x * kMaxRows + m] = best_v[i];
        a.part_idx[blockIdx.x * kMaxRows + m] =
            (best_i[i] == 0x7fffffff) ? 0x7fffffff : best_i[i] + a.vocab_off;
      }
    }
  }
}

// Everything a non-producer thread does for one GEMM (prologue, then its role).
template <int NT, int PRO, int EPI>
__device__ __forceinline__ void gemm_work(const GemmArgs& a, const GemmCtx& c, uint32_t& q,
                                          int tid, int warp, int lane,
                                          const uint2* pre_wreg = nullptr,
                                          const PeerComm* pc = nullptr) {
  const int wtid = (warp < kGemmWarps) ? tid : tid - 32;   // 0..607 over consumers + epilogue
  const int swarp = (warp < kGemmWarps) ? warp : warp - 1;
  uint2 wreg[4];
  if (PRO == PRO_RMS) {
    if (pre_wreg != nullptr) {
#pragma unroll
      for (int i = 0; i < 4; ++i) wreg[i] = pre_wreg[i];
    } else {
      gemm_preload_norm(a, wtid, wreg);
    }
  }
  gemm_prologue<NT, PRO>(a, c, EPI, wtid, swarp, lane, wreg);
  if (warp < kGemmWarps) gemm_consume<NT>(a, c, EPI, q, tid, warp, lane);
  else gemm_epilogue_role<NT, EPI>(a, c, tid - kConsumerThreads - 32, warp - kGemmWarps - 1, lane, pc);
}

// Stand-alone kernel (one CTA per SM, persistent over tiles; 20 warps):
//   warp 16      : PRODUCER (starts before the previous kernel has finished: PDL)
//   warps 0..15  : CONSUMERS
//   warps 17..19 : EPILOGUE
template <int NT, int PRO, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_skinny_kernel(const GemmArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const GemmCtx c = make_ctx(smem, a.n_stages);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) ctx_init_barriers(c);
  __syncthreads();
  uint32_t q = 0;
  if (warp == kProducerWarp) {
    pdl_launch_dependents();
    if (lane == 0) gemm_producer(a, c, q);
    pdl_wait();   // completion stays transitive along the PDL chain
    return;
  }
  pdl_launch_dependents();
  uint2 wreg[4];
  if (PRO == PRO_RMS) gemm_preload_norm(a, (warp < kGemmWarps) ? tid : tid - 32, wreg);
  pdl_wait();
  gemm_work<NT, PRO, EPI>(a, c, q, tid, warp, lane, PRO == PRO_RMS ? wreg : nullptr);
}

// Tensor-parallel row-parallel GEMM whose epilogue pushes its tiles to every rank (EPI_PUSH).
template <int NT>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_skinny_push_kernel(const GemmArgs a, const __grid_constant__ PeerComm pc) {
  extern __shared__ __align__(128) unsigned char smem[];
  const GemmCtx c = make_ctx(smem, a.n_stages);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) ctx_init_barriers(c);
  __syncthreads();
  uint32_t q = 0;
  if (warp == kProducerWarp) {
    pdl_launch_dependents();
    if (lane == 0) gemm_producer(a, c, q);
    pdl_wait();
    return;
  }
  pdl_launch_dependents();
  pdl_wait();
  gemm_work<NT, PRO_BF16, EPI_PUSH>(a, c, q, tid, warp, lane, nullptr, &pc);
}

}  // namespace lsk
