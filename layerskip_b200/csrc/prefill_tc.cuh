// prefill_tc.cuh — the prompt pass on the Hopper tensor cores (wgmma).
//
// The reference's prefill is `forward_early` / `forward_remainder` on s = T_p rows
// (self_speculation/llama_model_utils.py:213-276, 363-383): a real contraction, unlike the decode
// steps.  The decode kernel (gemm_skinny.cuh) carries at most 16 token rows, i.e. one pass over
// the weights per 16 prompt tokens; here a pass carries 128 tokens:
//
//     out[tok, f] = sum_k act[tok, k] * W[f, k]          tok < 128 per launch, f = output feature
//
// Swap-AB warpgroup MMA: the WEIGHTS are the A operand (128 output features per tile), the
// ACTIVATIONS the B operand (N = 128 tokens), both K-major in the SWIZZLE_128B layout below and
// both streamed by TMA bulk copies (16 KiB per operand per 64-wide k stage) through one shared-
// memory ring; the fp32 accumulators D[128 features x 128 tokens] live in the registers of the
// two consumer warpgroups (64 features each: wgmma.m64n128k16, 64 floats per thread).  Weights
// come from HBM once per launch; the activation block (<= 128 x K bf16) is re-read per feature
// tile from L2.  A 7B layer at 128 tokens moves 405 MB of weights for 52 GFLOP: HBM-bound on
// an H100 (the prompt costs ONE weight pass per 128 tokens instead of eight).
//
// Roles (384 threads, as lmhead_tc.cuh): warp 0 lane 0 = TMA producer, warpgroups 1 and 2 =
// MMA issue + epilogue straight from the accumulator registers.  The ring keeps streaming while
// the consumers run the epilogue of a tile.
//
// Operand layouts (common.cuh: canon_offset): K-major SWIZZLE_128B — stage (128 rows x 64 k) =
//   16 KiB, row r at r*128 B, 16-byte chunk c of a row stored at c ^ (r & 7).  Descriptor: layout
//   type 1 (128-byte swizzle), SBO = 1024 B (next 8-row atom), LBO unused (16 B); one wgmma eats
//   K = 16 = 32 bytes of a row: 4 MMAs per stage, start address advancing by 32 B.  Consumer
//   warpgroup g reads A rows 64 g .. 64 g + 63 (8 atoms = 8 KiB into the stage).  Stages must sit
//   on 1024-byte boundaries (the swizzle pattern is anchored to the address).
//   Weights: [tile][k stage][16 KiB], packed once with the SAME row permutations as the decode
//   layout (rotary pairs / gate-up pairs sit 8 rows apart: one accumulator thread holds both rows
//   of a pair).  Activations: [k stage][16 KiB] with rows = tokens, written in this layout by
//   the producing kernel.
//
// Grid: one CTA per work item wave; a work item = (feature tile, k split).  Row-parallel GEMMs with
// few feature tiles (O / down projections: hidden / 128 = 32 tiles at 7B) split K so that ~all SMs
// stream weights; their fp32 partial tiles go to per-split buffers that the NEXT kernel
// (rms_canon_kernel: residual add + RMSNorm) sums in fixed order — deterministic, no atomics.
#pragma once
#include "lmhead_tc.cuh"
#include "misc_kernels.cuh"

namespace lsk {

constexpr int kPfTokens = 128;                 // UMMA N: token rows per prefill pass
constexpr int kPfStageBytes = 2 * kTcStageBytes;   // A stage + B stage
constexpr int kPfMaxStages = 6;

// PF_EPI_QKV_MAP: the QKV epilogue with per-row positions and page-table views (row_map): token
// rows of several sequences packed into one chunk
enum { PF_EPI_QKV = 0, PF_EPI_STORE = 2, PF_EPI_SILU = 3, PF_EPI_QKV_MAP = 4 };

struct PrefillGemmArgs {
  const unsigned char* W;      // canonical weights [n_tiles][n_kst][16 KiB]
  const unsigned char* X;      // canonical activations [n_kst][16 KiB] (rows = tokens)
  int n_tiles;                 // ceil(n_rows / 128)
  int n_rows;                  // valid output features
  int n_kst;                   // K / 64 (K padded to 64)
  int M;                       // valid token rows (<= 128)
  int n_stages;
  int k_splits;                // work items per tile (STORE only; 1 otherwise)
  // STORE: out_f32[k split][tok][f]  (split stride = kPfTokens * out_ld floats)
  float* out_f32;
  int out_ld;
  // SILU: act canonical [inter_pad / 64][16 KiB]; packed rows (16-row groups: 8 gate, 8 up)
  unsigned char* act_canon;
  // QKV: RoPE, q -> q_out natural [tok][q_ld], k/v -> paged pool
  __nv_bfloat16* q_out;
  int q_ld;
  __nv_bfloat16* kpool;
  __nv_bfloat16* vpool;
  const int* page_table;
  int pos0;                    // position of token row 0 (prefill: base length is 0)
  const float2* rope;
  int head_dim;
  int q_rows, kv_rows, n_kv_heads;
  const int2* row_map;         // QKV_MAP: per token row (position, first logical page of its page-table view)
};

// + 1 KiB: the ring is aligned up to 1024 bytes inside the dynamic shared memory
__host__ __device__ inline size_t prefill_tc_smem_bytes(int n_stages) {
  return (size_t)kTcHeaderBytes + 1024 + (size_t)n_stages * kPfStageBytes;
}

// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T (bf16 in, fp32 accumulate, both K-major in shared
// memory); fragment layout as wgmma_m64n16 (lmhead_tc.cuh), 16 column groups of 8
__device__ __forceinline__ void wgmma_m64n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate));
}

// natural [rows, K] bf16 -> canonical tiles with a row permutation (`mode`: misc_kernels.cuh map_row)
// and an input-column slice (tensor-parallel row-parallel GEMMs); dst rows beyond n_rows and k
// beyond K are zero.  Packed row pr of dst = source row map^-1: we iterate SOURCE rows and scatter.
__global__ void pack_canonical_rows_kernel(const __nv_bfloat16* __restrict__ src, int64_t src_ld,
                                           int64_t src_row0, int64_t src_col0, int64_t n_rows, int64_t K,
                                           unsigned char* __restrict__ dst, int64_t dst_row0, int mode,
                                           int64_t n_kst, int hd) {
  const int64_t chunks = K >> 3;                               // 16-byte chunks per source row
  const int64_t total = n_rows * chunks;
  for (int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; c < total; c += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = c / chunks, kc = c % chunks;
    const uint4 v = *reinterpret_cast<const uint4*>(src + (src_row0 + r) * src_ld + src_col0 + kc * 8);
    const int64_t pr = dst_row0 + map_row(mode, r, hd);
    const int64_t tile = pr >> 7;
    *reinterpret_cast<uint4*>(dst + (size_t)tile * n_kst * kTcStageBytes + canon_offset((int)(pr & 127), (int)(kc * 8))) = v;
  }
}

// x[tok] += sum of the `n_part` partial rows (fixed order; the split-K / tensor-parallel partials of
// the previous row-parallel GEMM), written back, then RMSNorm -> bf16 activations in the operand
// layout (the rounding point of a bf16 HF model, modeling_llama.py:52-70).  One CTA per token row.
__global__ void __launch_bounds__(256)
rms_canon_kernel(float* __restrict__ x, int x_ld, const float* __restrict__ part, int n_part, size_t part_stride,
                 const __nv_bfloat16* __restrict__ norm_w, float eps, int K, unsigned char* __restrict__ dst) {
  __shared__ float s_part[8];
  pdl_launch_dependents();
  pdl_wait();
  const int tok = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float4* xr = reinterpret_cast<float4*>(x + (size_t)tok * x_ld);
  const int nvec = K >> 2;
  float ss = 0.f;
  for (int i = tid; i < nvec; i += 256) {
    float4 v = xr[i];
    for (int p = 0; p < n_part; ++p) {
      const float4 d = *reinterpret_cast<const float4*>(part + (size_t)p * part_stride + (size_t)tok * x_ld + i * 4);
      v.x += d.x; v.y += d.y; v.z += d.z; v.w += d.w;
    }
    if (n_part > 0) xr[i] = v;
    ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  ss = warp_sum(ss);
  if (lane == 0) s_part[warp] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += s_part[w];
  const float rstd = rsqrtf(tot / (float)K + eps);
  if (dst == nullptr) return;                       // residual update only
  for (int i = tid; i < nvec; i += 256) {
    const float4 v = xr[i];                         // own writes: same thread, same address
    const uint2 wv = *reinterpret_cast<const uint2*>(norm_w + i * 4);
    uint2 o;
    o.x = pack_bf16x2(bf16_lo(wv.x) * (v.x * rstd), bf16_hi(wv.x) * (v.y * rstd));
    o.y = pack_bf16x2(bf16_lo(wv.y) * (v.z * rstd), bf16_hi(wv.y) * (v.w * rstd));
    *reinterpret_cast<uint2*>(dst + canon_offset(tok, i * 4)) = o;
  }
}

// tensor parallel: out[tok] = sum of the local split-K partials (fixed order), all-reduced afterwards
__global__ void __launch_bounds__(256)
reduce_partials_kernel(const float* __restrict__ part, int n_part, size_t part_stride, int ld, int K,
                       float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int tok = blockIdx.x;
  for (int i = threadIdx.x; i < (K >> 2); i += 256) {
    float4 v = *reinterpret_cast<const float4*>(part + (size_t)tok * ld + i * 4);
    for (int p = 1; p < n_part; ++p) {
      const float4 d = *reinterpret_cast<const float4*>(part + (size_t)p * part_stride + (size_t)tok * ld + i * 4);
      v.x += d.x; v.y += d.y; v.z += d.z; v.w += d.w;
    }
    *reinterpret_cast<float4*>(out + (size_t)tok * ld + i * 4) = v;
  }
}

template <int EPI>
__global__ void __launch_bounds__(kTcThreads, 1)
prefill_gemm_tc_kernel(const PrefillGemmArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty_bar = full_bar + kPfMaxStages;
  unsigned char* ring = smem + kTcHeaderBytes + ((1024u - (smem_u32(smem) + kTcHeaderBytes) % 1024u) % 1024u);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int NS = a.n_stages;
  const int KS = (EPI == PF_EPI_STORE && a.k_splits > 1) ? a.k_splits : 1;
  const int n_items = a.n_tiles * KS;

  if (tid == 0) {
    for (int s = 0; s < NS; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kTcConsumerThreads); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  pdl_launch_dependents();
  pdl_wait();          // the activations (B operand) are the previous kernel's output

  if (warp < 4) {
    if (tid == 0) {
      // ============================================================ TMA PRODUCER
      uint32_t q = 0;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int tile = item / KS, ks = item - tile * KS;
        const int s_lo = (int)((long long)a.n_kst * ks / KS), s_hi = (int)((long long)a.n_kst * (ks + 1) / KS);
        for (int s = s_lo; s < s_hi; ++s, ++q) {
          const int st = q % NS;
          mbar_wait_bounded(&empty_bar[st], ((q / NS) & 1) ^ 1);
          mbar_arrive_expect_tx(&full_bar[st], kPfStageBytes);
          unsigned char* dst = ring + (size_t)st * kPfStageBytes;
          tma_bulk_g2s(dst, a.W + ((size_t)tile * a.n_kst + s) * kTcStageBytes, kTcStageBytes, &full_bar[st]);
          tma_bulk_g2s(dst + kTcStageBytes, a.X + (size_t)s * kTcStageBytes, kTcStageBytes, &full_bar[st]);
        }
      }
    }
    return;
  }

  // ================================================================ CONSUMERS (2 warpgroups x 64 features)
  const int wg = (warp - 4) >> 2;
  const int r_lo = ((warp - 4) & 3) * 16 + (lane >> 2);   // accumulator rows r_lo, r_lo + 8 of this warpgroup
  uint32_t q = 0;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int tile = item / KS, ks = item - tile * KS;
    const int s_lo = (int)((long long)a.n_kst * ks / KS), s_hi = (int)((long long)a.n_kst * (ks + 1) / KS);
    float d[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) d[j] = 0.f;
    for (int s = s_lo; s < s_hi; ++s, ++q) {
      const int st = q % NS;
      mbar_wait_bounded(&full_bar[st], (q / NS) & 1);
      const uint32_t a_addr = smem_u32(ring + (size_t)st * kPfStageBytes) + wg * 8192;
      const uint32_t b_addr = smem_u32(ring + (size_t)st * kPfStageBytes) + kTcStageBytes;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kTcStageK / 16; ++k)
        wgmma_m64n128(d, wgmma_desc(a_addr + k * 32, 16, 1024, 1), wgmma_desc(b_addr + k * 32, 16, 1024, 1),
                      (s > s_lo || k > 0) ? 1u : 0u);
      wgmma_commit();
      if (s > s_lo) {                                 // the previous stage's MMAs are done reading it
        wgmma_wait<1>();
        mbar_arrive(&empty_bar[(q - 1) % NS]);
      }
    }
    wgmma_wait<0>();
    if (s_hi > s_lo) mbar_arrive(&empty_bar[(q - 1) % NS]);

    // d[4 n + c] = (row r_lo, token 8 n + 2 (lane % 4) + c), d[4 n + 2 + c] = (row r_lo + 8, same token):
    // the lower and upper row of a gate/up or rotary pair are in the same thread
    const int prow = tile * kTcTileRows + wg * 64 + r_lo;   // packed output row (feature), lower of the pair
    const bool valid_lo = prow < a.n_rows, valid_hi = prow + 8 < a.n_rows;
    if (EPI == PF_EPI_STORE) {
      float* outp = a.out_f32 + (size_t)ks * kPfTokens * a.out_ld + prow;
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        const int tok = 8 * (j >> 2) + 2 * (lane & 3) + (j & 1);
        const bool hi = (j & 2) != 0;
        if (tok < a.M && (hi ? valid_hi : valid_lo)) outp[(size_t)tok * a.out_ld + (hi ? 8 : 0)] = d[j];
      }
    } else if (EPI == PF_EPI_SILU) {
      // 16-row groups: rows 0..7 gate, rows 8..15 up of the same 8 features (MAP_GATE / MAP_UP)
      const int kidx = (prow >> 4) * 8 + (prow & 7);
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        if (j & 2) continue;
        const int tok = 8 * (j >> 2) + 2 * (lane & 3) + (j & 1);
        if (tok < a.M && valid_lo) {
          const float g = d[j], u = d[j + 2];
          const float sg = g / (1.f + __expf(-g));
          *reinterpret_cast<__nv_bfloat16*>(a.act_canon + canon_offset(tok, kidx)) = __float2bfloat16_rn(sg * u);
        }
      }
    } else {  // PF_EPI_QKV, PF_EPI_QKV_MAP
      // a pair never straddles q / k / v or a head (all are multiples of head_dim >= 32 rows)
      const int HD = a.head_dim, half = HD >> 1;
      const bool is_q = prow < a.q_rows, is_k = !is_q && prow < a.q_rows + a.kv_rows;
      const int rel = is_q ? prow : (is_k ? prow - a.q_rows : prow - a.q_rows - a.kv_rows);
      const int head = rel / HD, inhead = rel - head * HD;
      const bool rot = is_q || is_k;
      const int dp = (inhead >> 4) * 8 + (inhead & 7);          // pair index (q / k rows)
      const int dd_lo = rot ? dp : inhead, dd_hi = rot ? dp + half : inhead + 8;
      const float2* __restrict__ rope = a.rope;
      __nv_bfloat16* __restrict__ pool = is_k ? a.kpool : a.vpool;
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        if (j & 2) continue;
        const int tok = 8 * (j >> 2) + 2 * (lane & 3) + (j & 1);
        if (tok >= a.M || !valid_lo) continue;
        int pos = a.pos0 + tok;
        const int* page_table = a.page_table;
        if (EPI == PF_EPI_QKV_MAP) {
          const int2 rm = a.row_map[tok];
          pos = rm.x;
          page_table += rm.y;
        }
        // lower row of the pair holds x[d] (lo), upper row x[d + half] (hi):
        //   out_lo = lo cos - hi sin,  out_hi = hi cos + lo sin   (rotate_half, modeling_llama.py:138-168)
        const float lo = d[j], hi = d[j + 2];
        float out_lo = lo, out_hi = hi;
        if (rot) {
          const float2 cs = __ldg(rope + (size_t)pos * half + dp);
          out_lo = lo * cs.x - hi * cs.y;
          out_hi = hi * cs.x + lo * cs.y;
        }
        if (is_q) {
          __nv_bfloat16* qo = a.q_out + (size_t)tok * a.q_ld + head * HD;
          qo[dd_lo] = __float2bfloat16_rn(out_lo);
          qo[dd_hi] = __float2bfloat16_rn(out_hi);
        } else {
          const int page = page_table[pos >> 6];
          pool[kv_elem_offset(HD, page, a.n_kv_heads, head, pos & 63, dd_lo)] = __float2bfloat16_rn(out_lo);
          if (valid_hi) pool[kv_elem_offset(HD, page, a.n_kv_heads, head, pos & 63, dd_hi)] = __float2bfloat16_rn(out_hi);
        }
      }
    }
  }
}

}  // namespace lsk
