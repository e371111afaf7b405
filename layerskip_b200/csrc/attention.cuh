// attention.cuh — paged split-KV attention for decode / verify blocks (<= 16 query tokens).
//
// One CTA = (kv head, split); no thread-block clusters (see the split merge below).  The query
// rows of a CTA are all tokens x all q-heads that share the kv head (GQA), processed 16 rows at a
// time as the M side of mma.sync m16n8k16.  A split owns the 64-key groups  s, s + n_splits, ...
// (by ABSOLUTE key index, so the partition seen by a query at position p does not depend on how
// many rows are in flight — this keeps the result batch-invariant).  Rounding points mirror a bf16
// HF model: q/k/v bf16, scores and softmax fp32, probabilities rounded to bf16 for P.V, fp32
// accumulate (transformers modeling_llama.py:187-221).
//
// Data movement (round 2): a (page, kv head) block of K or V is CONTIGUOUS in the pool and
// pre-swizzled (common.cuh: kv_elem_offset), so one TMA bulk copy per block lands it in shared
// memory ready for conflict-free fragment loads — no LDG -> STS staging, no register round trip.
// The committed context (keys < *base_len) cannot change while a round's graph runs, so the bulk
// copies of every FULLY committed key group are issued BEFORE griddepcontrol.wait: they overlap
// the tail of the QKV projection that precedes this kernel, and after the wait only the query
// fragments and the one boundary group (the keys this round appended) are still to be fetched.
//
// Partials (m, l, O) are merged in fixed order: the 4 warps of a CTA through shared memory, then
// the splits: every split publishes its partial rows to global memory, and the LAST split of the kv
// head to arrive (per-head arrival counter) merges all of them in split order.  Deterministic.  No
// thread-block clusters: a cluster has to fit inside one GPC, and on the 132-SM H100 only 30
// clusters of 4 (39 of 3) are resident at one CTA per SM, so a clustered 7B grid (32 x 4) or 13B
// grid (40 x 3) would leave clusters for a second wave.  Unclustered, the grid is resident at once.
#pragma once
#include "common.cuh"

namespace lsk {

constexpr int kAttnThreads = 128;
constexpr int kKeyGroup = 64;                 // keys per pipeline stage (== one KV page)
constexpr int kAttnMaxStages = 4;             // K/V stages in flight per CTA (AttnArgs::n_stages of them used)
constexpr int kAttnHeader = 128;              // mbarriers, then the merger flag
constexpr int kMaxSplits = 8;

struct AttnArgs {
  const __nv_bfloat16* q;      // [M][q_ld] post-RoPE
  int q_ld;
  __nv_bfloat16* out;          // [M][out_ld]
  int out_ld;
  const __nv_bfloat16* kpool;  // layer base
  const __nv_bfloat16* vpool;
  const int* page_table;
  const int* base_len;         // committed length: constant while the enclosing graph runs
  int pos_off;
  int M;
  int group;                   // q heads per kv head
  int n_kv_heads;              // local
  int n_splits;
  float scale;                 // head_dim^-0.5
  int rows_pad;                // group * M rounded up to 16
  int merge_off;               // byte offset of the warp-merge buffer (== stage 0 when aliased)
  int part_off;                // byte offset of this CTA's partial (O, then m/l)
  int reload_per_rb;           // 1: the merge buffer aliases the stages -> K/V re-fetched per row block
  int out_canon;               // 1: `out` is a canonical K-major operand (rows = tokens) for prefill_tc.cuh
  int n_stages;                // K/V ring depth (2 .. kAttnMaxStages)
  float* part;                 // [n_kv_heads][n_splits][rows_pad][HD + 2] published partials (O, then m/l)
  unsigned int* arrive;        // [n_kv_heads] splits done; zero between launches (the merger resets it)
};

// Piece grid (attn_piece_kernel): blockIdx.z selects pieces[z] = (chunk row of its first query row,
// rows, position of that row, first logical page of its page-table view).  q, the canonical output
// and the partials are addressed by chunk row; AttnArgs::M is the largest piece's rows,
// AttnArgs::arrive holds [pieces][n_kv_heads] counters.
// Sequence grid (batched rounds, pieces == nullptr): piece z is sequence z's seq_rows rows, chunk row
// z * seq_rows, at position *(base_len + z * len_stride) + pos_off + i, over its page-table view
// page_table + z * seq_pages.  Packed scoring's pieces all read *base_len (len_stride 0).
struct AttnPieces {
  const int4* pieces;
  int part_rows;               // row stride of AttnArgs::part: rows_pad of all the launch's rows
  int seq_rows, len_stride, seq_pages;
};

// floats of AttnArgs::part for a launch
__host__ inline size_t attn_part_floats(int n_kv_heads, int n_splits, int rows_pad, int hd) {
  return (size_t)n_kv_heads * n_splits * rows_pad * (hd + 2);
}

// shared-memory plan of one launch (host and device agree through AttnArgs offsets)
struct AttnSmemPlan {
  int merge_off, part_off, reload_per_rb, n_stages;
  size_t total;
};
__host__ inline AttnSmemPlan attn_smem_plan(int hd, int group, int M, int kAttnStages = 2) {
  AttnSmemPlan p;
  p.n_stages = kAttnStages;
  const int R = group * M;
  const int rows_pad = (R + 15) / 16 * 16;
  const int stage_bytes = 2 * kKeyGroup * hd * 2;
  const int merge_bytes = 4 * 16 * hd * 4 + 4 * 16 * 2 * 4;
  const int stages_end = kAttnHeader + kAttnStages * stage_bytes;
  // one row block: the merge buffer may reuse stage memory (nothing is re-read afterwards)
  p.reload_per_rb = (R <= 16 && merge_bytes <= kAttnStages * stage_bytes) ? 1 : 0;
  p.merge_off = p.reload_per_rb ? kAttnHeader : stages_end;
  p.part_off = p.reload_per_rb ? stages_end : stages_end + ((merge_bytes + 127) & ~127);
  p.total = (size_t)p.part_off + (size_t)rows_pad * (hd + 2) * 4;
  return p;
}

__device__ __forceinline__ void team_sync() {
  asm volatile("bar.sync 8, %0;" ::"r"(kAttnThreads) : "memory");
}

// Fixed-order merge of the splits' partials for one (row, 16-dim segment); `ml(s)` / `o(s)` return
// split s's (m, l) pair and O segment (published in global memory, read past L1).  SP = compile-time
// bound on the number of splits: with SP <= 4 every value (4 (m, l) pairs + 16 float4) is requested
// up front — ONE round trip instead of a chain of five; same arithmetic in the same order either way.
template <int HD, int SP, typename FML, typename FO>
__device__ __forceinline__ void merge_splits_write(const AttnArgs& a, int kvh, int row, int dseg, int tok0,
                                                   FML ml, FO o) {
  float ms[SP], ls[SP];
#pragma unroll
  for (int s = 0; s < SP; ++s) {
    ms[s] = -INFINITY; ls[s] = 0.f;
    if (s < a.n_splits) { const float* p = ml(s); ms[s] = __ldcg(p); ls[s] = __ldcg(p + 1); }
  }
  float acc[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = 0.f;
  float ll = 0.f;
  if (SP <= 4) {
    float4 v[4][SP];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int s = 0; s < SP; ++s)
        v[i][s] = (s < a.n_splits) ? __ldcg(reinterpret_cast<const float4*>(o(s)) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    float mm = -INFINITY;
#pragma unroll
    for (int s = 0; s < SP; ++s) mm = fmaxf(mm, ms[s]);
    float f[SP];
#pragma unroll
    for (int s = 0; s < SP; ++s) {
      f[s] = (ms[s] == -INFINITY) ? 0.f : __expf(ms[s] - mm);
      if (s < a.n_splits) ll += ls[s] * f[s];
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int s = 0; s < SP; ++s) {
        if (s < a.n_splits) {
          acc[4 * i] += v[i][s].x * f[s]; acc[4 * i + 1] += v[i][s].y * f[s];
          acc[4 * i + 2] += v[i][s].z * f[s]; acc[4 * i + 3] += v[i][s].w * f[s];
        }
      }
  } else {
    // all (m, l) pairs first, then the O segments in batches of independent loads
    float mm = -INFINITY;
#pragma unroll
    for (int s = 0; s < SP; ++s) mm = fmaxf(mm, ms[s]);
    float f[SP];
#pragma unroll
    for (int s = 0; s < SP; ++s) {
      f[s] = (ms[s] == -INFINITY) ? 0.f : __expf(ms[s] - mm);
      if (s < a.n_splits) ll += ls[s] * f[s];
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float4 v[SP];
#pragma unroll
      for (int s = 0; s < SP; ++s)
        v[s] = (s < a.n_splits) ? __ldcg(reinterpret_cast<const float4*>(o(s)) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int s = 0; s < SP; ++s) {
        if (s < a.n_splits) {
          acc[4 * i] += v[s].x * f[s]; acc[4 * i + 1] += v[s].y * f[s];
          acc[4 * i + 2] += v[s].z * f[s]; acc[4 * i + 3] += v[s].w * f[s];
        }
      }
    }
  }
  const float inv = 1.f / ll;
  const int tok = tok0 + row / a.group, hq = kvh * a.group + row % a.group;
  if (a.out_canon) {           // two 16-byte chunks of the O projection's B operand
    unsigned char* base = reinterpret_cast<unsigned char*>(a.out);
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      uint4 v;
      v.x = pack_bf16x2(acc[8 * c] * inv, acc[8 * c + 1] * inv);
      v.y = pack_bf16x2(acc[8 * c + 2] * inv, acc[8 * c + 3] * inv);
      v.z = pack_bf16x2(acc[8 * c + 4] * inv, acc[8 * c + 5] * inv);
      v.w = pack_bf16x2(acc[8 * c + 6] * inv, acc[8 * c + 7] * inv);
      *reinterpret_cast<uint4*>(base + canon_offset(tok, hq * HD + dseg + 8 * c)) = v;
    }
    return;
  }
  __nv_bfloat16* op = a.out + (size_t)tok * a.out_ld + hq * HD + dseg;
#pragma unroll
  for (int i = 0; i < 16; i += 2)
    *reinterpret_cast<uint32_t*>(op + i) = pack_bf16x2(acc[i] * inv, acc[i + 1] * inv);
}

// PIECES: one launch covers several independent query pieces (packed scoring); blockIdx.z selects
// the piece, whose rows, positions, page-table view and partials rows come from a.pieces.  A row's
// arithmetic is the same as in a launch of its own.
template <int HD, bool PIECES>
__device__ __forceinline__ void attn_split_body(const AttnArgs& a, const AttnPieces& pz) {
  constexpr int KS = HD / 16;                   // k steps of Q.K^T
  constexpr int DT = HD / 8;                    // n8 tiles of the output
  constexpr int CH = HD / 8;                    // 16-byte chunks per K/V row
  constexpr int kGroupBytes = kKeyGroup * HD * 2;
  constexpr int kStageBytes = 2 * kGroupBytes;  // K block, then V block
  extern __shared__ __align__(128) unsigned char dsm[];
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(dsm);
  uint64_t* empty_bar = full_bar + kAttnMaxStages;
  unsigned char* stages = dsm + kAttnHeader;
  const int kAttnStages = a.n_stages;
  float* mo = reinterpret_cast<float*>(dsm + a.merge_off);       // [4 warps][16 rows][HD]
  float* mml = mo + 4 * 16 * HD;                                  // [4][16][2]
  float* po = reinterpret_cast<float*>(dsm + a.part_off);        // [rows_pad][HD]
  float* pml = po + (size_t)a.rows_pad * HD;                      // [rows_pad][2]
  int* last = reinterpret_cast<int*>(empty_bar + kAttnMaxStages); // header word behind the mbarriers
  const int kvh = blockIdx.x, split = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  // this CTA's query rows: the whole launch, or piece blockIdx.z (chunk row tok0)
  const int z = blockIdx.z;
  const int4 pc = !PIECES ? make_int4(0, 0, 0, 0)
                  : pz.pieces ? pz.pieces[z] : make_int4(z * pz.seq_rows, pz.seq_rows, a.pos_off, z * pz.seq_pages);
  const int* base_len = PIECES ? a.base_len + z * pz.len_stride : a.base_len;
  const int tok0 = pc.x;
  const int M = PIECES ? pc.y : a.M;
  const int pos_off = PIECES ? pc.z : a.pos_off;
  const int* page_table = PIECES ? a.page_table + pc.w : a.page_table;
  const __nv_bfloat16* qb = PIECES ? a.q + (size_t)tok0 * a.q_ld : a.q;

  if (tid == 0) {
    for (int s = 0; s < kAttnStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_launch_dependents();

  // ---- everything below up to pdl_wait() reads only data that is constant while the enclosing
  // graph runs: the committed length, the page table, and K/V rows below the committed length
  const int len0 = *base_len;
  const int base = len0 + pos_off;                   // position of token row 0
  const int n_keys = base + M;                       // keys visible to the last row
  const int n_kgroups = (n_keys + kKeyGroup - 1) / kKeyGroup;
  const int n_mine = split < n_kgroups ? (n_kgroups - split + a.n_splits - 1) / a.n_splits : 0;
  const int R = a.group * M;                         // real query rows (token-major)
  const int n_rb = (R + 15) / 16;
  const bool reload = a.reload_per_rb != 0 || n_mine > kAttnStages;   // K/V re-fetched per row block
  int issued = 0;                                                    // (thread 0) items handed to the TMA engine

  auto issue = [&](int item) {       // thread 0 only
    const int j = item % n_mine;
    const int kg = split + j * a.n_splits;
    const int st = item % kAttnStages;
    mbar_wait(&empty_bar[st], ((item / kAttnStages) & 1) ^ 1);
    const int page = page_table[kg];                 // kKeyGroup == kPageTokens
    const size_t blk = (size_t)(page * a.n_kv_heads + kvh) * kPageTokens * HD;
    unsigned char* dst = stages + (size_t)st * kStageBytes;
    mbar_arrive_expect_tx(&full_bar[st], kStageBytes);
    tma_bulk_g2s(dst, a.kpool + blk, kGroupBytes, &full_bar[st]);
    tma_bulk_g2s(dst + kGroupBytes, a.vpool + blk, kGroupBytes, &full_bar[st]);
  };
  if (tid == 0) {
    // fully committed groups of the first row block, as deep as the ring
    while (issued < n_mine && issued < kAttnStages &&
           (split + issued * a.n_splits + 1) * kKeyGroup <= len0) {
      issue(issued);
      ++issued;
    }
  }
  pdl_wait();

  int item = 0;
  for (int rb = 0; rb < n_rb; ++rb) {
    // ---- Q fragments for rows rb*16 + {g, g+8}
    uint32_t qf[KS][4];
    {
      const int r0 = rb * 16 + g, r1 = r0 + 8;
      const __nv_bfloat16* q0 = nullptr;
      const __nv_bfloat16* q1 = nullptr;
      if (r0 < R) q0 = qb + (size_t)(r0 / a.group) * a.q_ld + (kvh * a.group + r0 % a.group) * HD;
      if (r1 < R) q1 = qb + (size_t)(r1 / a.group) * a.q_ld + (kvh * a.group + r1 % a.group) * HD;
#pragma unroll
      for (int k = 0; k < KS; ++k) {
        qf[k][0] = q0 ? *reinterpret_cast<const uint32_t*>(q0 + k * 16 + 2 * t) : 0u;
        qf[k][1] = q1 ? *reinterpret_cast<const uint32_t*>(q1 + k * 16 + 2 * t) : 0u;
        qf[k][2] = q0 ? *reinterpret_cast<const uint32_t*>(q0 + k * 16 + 8 + 2 * t) : 0u;
        qf[k][3] = q1 ? *reinterpret_cast<const uint32_t*>(q1 + k * 16 + 8 + 2 * t) : 0u;
      }
    }
    const int row0 = rb * 16 + g, row1 = row0 + 8;
    const int lim0 = (row0 < R) ? base + row0 / a.group : -1;   // last visible key index
    const int lim1 = (row1 < R) ? base + row1 / a.group : -1;

    float o[DT][4];
#pragma unroll
    for (int d = 0; d < DT; ++d) o[d][0] = o[d][1] = o[d][2] = o[d][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

    const bool loads_now = reload || rb == 0;
    const int item0 = reload ? rb * n_mine : 0;       // first item of this row block
    for (int j = 0; j < n_mine; ++j) {
      const int kg = split + j * a.n_splits;
      item = item0 + j;
      if (tid == 0 && loads_now) {                    // keep the ring topped up (this row block only)
        const int hi = min(item0 + n_mine, item + kAttnStages);
        if (issued < item0) issued = item0;
        while (issued < hi) { issue(issued); ++issued; }
      }
      __syncwarp();
      const int st = item % kAttnStages;
      mbar_wait(&full_bar[st], (item / kAttnStages) & 1);
      const unsigned char* ks = stages + (size_t)st * kStageBytes;
      const unsigned char* vs = ks + kGroupBytes;

      // ---- S = Q K^T for this warp's 16 keys (two n8 tiles); key row r, logical chunk c lives at
      // physical chunk c ^ swz(r): 8 rows x one chunk per access phase -> conflict-free
      float s[2][4];
#pragma unroll
      for (int n = 0; n < 2; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
#pragma unroll
      for (int n = 0; n < 2; ++n) {
        const int key = warp * 16 + n * 8 + g;
        const int swz = kv_chunk_swizzle(HD, key);
        const unsigned char* kr = ks + key * (HD * 2) + t * 4;
#pragma unroll
        for (int k = 0; k < KS; ++k) {
          const uint32_t b0 = *reinterpret_cast<const uint32_t*>(kr + (((2 * k) ^ swz) << 4));
          const uint32_t b1 = *reinterpret_cast<const uint32_t*>(kr + (((2 * k + 1) ^ swz) << 4));
          mma_bf16_16816(s[n], qf[k][0], qf[k][1], qf[k][2], qf[k][3], b0, b1);
        }
      }
      // ---- scale + causal mask + online softmax (rows g and g+8)
      const int key0 = kg * kKeyGroup + warp * 16 + 2 * t;
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int n = 0; n < 2; ++n) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int kidx = key0 + n * 8 + c;
          s[n][c] = (kidx <= lim0) ? s[n][c] * a.scale : -INFINITY;
          s[n][2 + c] = (kidx <= lim1) ? s[n][2 + c] * a.scale : -INFINITY;
          mx0 = fmaxf(mx0, s[n][c]);
          mx1 = fmaxf(mx1, s[n][2 + c]);
        }
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float nm0 = fmaxf(m0, mx0), nm1 = fmaxf(m1, mx1);
      const float sc0 = (nm0 == -INFINITY) ? 1.f : __expf(m0 - nm0);
      const float sc1 = (nm1 == -INFINITY) ? 1.f : __expf(m1 - nm1);
      m0 = nm0;
      m1 = nm1;
      float p[2][4];
#pragma unroll
      for (int n = 0; n < 2; ++n) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          p[n][c] = (nm0 == -INFINITY) ? 0.f : __expf(s[n][c] - nm0);
          p[n][2 + c] = (nm1 == -INFINITY) ? 0.f : __expf(s[n][2 + c] - nm1);
        }
      }
      l0 = l0 * sc0 + p[0][0] + p[0][1] + p[1][0] + p[1][1];
      l1 = l1 * sc1 + p[0][2] + p[0][3] + p[1][2] + p[1][3];
#pragma unroll
      for (int d = 0; d < DT; ++d) {
        o[d][0] *= sc0; o[d][1] *= sc0; o[d][2] *= sc1; o[d][3] *= sc1;
      }
      // ---- O += P V  (P as bf16 A fragments, V through ldmatrix.trans).  Keys past the last
      // visible one have p == 0 exactly; their V rows are stale-but-finite pool contents.
      const uint32_t pa0 = pack_bf16x2(p[0][0], p[0][1]);
      const uint32_t pa1 = pack_bf16x2(p[0][2], p[0][3]);
      const uint32_t pa2 = pack_bf16x2(p[1][0], p[1][1]);
      const uint32_t pa3 = pack_bf16x2(p[1][2], p[1][3]);
      {
        const int mat = lane >> 3;
        const int key = warp * 16 + (mat & 1) * 8 + (lane & 7);
        const int swz = kv_chunk_swizzle(HD, key);
        const unsigned char* vrow = vs + key * (HD * 2);
#pragma unroll
        for (int d = 0; d < DT; d += 2) {
          uint32_t vb[4];
          ldmatrix_x4_trans(vb, vrow + (((d + (mat >> 1)) ^ swz) << 4));
          mma_bf16_16816(o[d], pa0, pa1, pa2, pa3, vb[0], vb[1]);
          mma_bf16_16816(o[d + 1], pa0, pa1, pa2, pa3, vb[2], vb[3]);
        }
      }
      if (loads_now) {                                // this warp is done with the stage
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[st]);
      }
    }
    (void)CH;

    // ---- merge the 4 warps (fixed order) through shared memory
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    team_sync();   // every warp has consumed its stages (the merge buffer may alias them)
#pragma unroll
    for (int d = 0; d < DT; ++d) {
      *reinterpret_cast<float2*>(mo + ((warp * 16 + g) * HD) + d * 8 + 2 * t) = make_float2(o[d][0], o[d][1]);
      *reinterpret_cast<float2*>(mo + ((warp * 16 + g + 8) * HD) + d * 8 + 2 * t) = make_float2(o[d][2], o[d][3]);
    }
    if (t == 0) {
      mml[(warp * 16 + g) * 2] = m0;
      mml[(warp * 16 + g) * 2 + 1] = l0;
      mml[(warp * 16 + g + 8) * 2] = m1;
      mml[(warp * 16 + g + 8) * 2 + 1] = l1;
    }
    team_sync();
    for (int it = tid; it < 16 * (HD / 16); it += kAttnThreads) {
      // item -> (row = it / (HD/16), 16 dims)
      const int row = it / (HD / 16), dseg = (it % (HD / 16)) * 16;
      float mm = -INFINITY;
      for (int w = 0; w < 4; ++w) mm = fmaxf(mm, mml[(w * 16 + row) * 2]);
      float ll = 0.f;
      float acc[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[i] = 0.f;
      for (int w = 0; w < 4; ++w) {
        const float mw = mml[(w * 16 + row) * 2];
        const float f = (mw == -INFINITY) ? 0.f : __expf(mw - mm);
        ll += mml[(w * 16 + row) * 2 + 1] * f;
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[i] += mo[(w * 16 + row) * HD + dseg + i] * f;
      }
      const size_t prow = (size_t)(rb * 16 + row);
      float* pp = po + prow * HD + dseg;
#pragma unroll
      for (int i = 0; i < 16; i += 4)
        *reinterpret_cast<float4*>(pp + i) = make_float4(acc[i], acc[i + 1], acc[i + 2], acc[i + 3]);
      if (dseg == 0) {
        pml[prow * 2] = mm;
        pml[prow * 2 + 1] = ll;
      }
    }
    team_sync();   // merge buffer free before the next row block refills the stages
    // generic-proxy accesses of the (aliased) merge buffer are ordered before the next bulk copies
    if (tid == 0 && rb + 1 < n_rb) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }

  // ---- publish this split's partial rows (same layout as po / pml)
  // (a piece's rows sit at chunk row tok0 of partials laid out for a whole chunk, part_rows rows)
  const int prows = PIECES ? pz.part_rows : a.rows_pad;
  const size_t part_floats = (size_t)prows * (HD + 2);
  const size_t o_off = PIECES ? (size_t)a.group * tok0 * HD : 0;
  const size_t ml_off = (size_t)prows * HD + (PIECES ? (size_t)a.group * tok0 * 2 : 0);
  unsigned int* arrive = PIECES ? a.arrive + (size_t)blockIdx.z * a.n_kv_heads : a.arrive;
  float* gp = a.part + (size_t)(kvh * a.n_splits + split) * part_floats;
  for (int i = tid; i < R * (HD / 4); i += kAttnThreads)
    reinterpret_cast<float4*>(gp + o_off)[i] = reinterpret_cast<const float4*>(po)[i];
  for (int i = tid; i < 2 * R; i += kAttnThreads) gp[ml_off + i] = pml[i];
  __threadfence();
  __syncthreads();
  if (tid == 0) *last = atomicAdd(&arrive[kvh], 1u) == (unsigned)(a.n_splits - 1);
  __syncthreads();
  if (!*last) return;

  // ---- the last split of the kv head merges every split's partial, in split order
  __threadfence();
  constexpr int SEG = HD / 16;
  const float* hp = a.part + (size_t)kvh * a.n_splits * part_floats;
  for (int it = tid; it < R * SEG; it += kAttnThreads) {
    const int row = it / SEG, dseg = (it % SEG) * 16;
    auto f_ml = [&](int s) { return hp + s * part_floats + ml_off + row * 2; };
    auto f_o = [&](int s) { return hp + s * part_floats + o_off + (size_t)row * HD + dseg; };
    if (a.n_splits <= 4) merge_splits_write<HD, 4>(a, kvh, row, dseg, tok0, f_ml, f_o);
    else merge_splits_write<HD, kMaxSplits>(a, kvh, row, dseg, tok0, f_ml, f_o);
  }
  if (tid == 0) arrive[kvh] = 0u;   // every split has arrived: ready for the next launch
}

template <int HD>
__global__ void __launch_bounds__(kAttnThreads)
attn_split_kernel(const AttnArgs a) {
  attn_split_body<HD, false>(a, AttnPieces{nullptr, 0});
}

// grid (kv heads, splits, pieces): every piece of a packed prompt-pass chunk, or every sequence of a
// batched round, in one launch
template <int HD>
__global__ void __launch_bounds__(kAttnThreads)
attn_piece_kernel(const AttnArgs a, const AttnPieces pz) {
  attn_split_body<HD, true>(a, pz);
}

}  // namespace lsk
