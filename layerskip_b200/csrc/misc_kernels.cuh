// misc_kernels.cuh — small kernels around the two streaming kernels: weight repacking, RoPE
// table, embedding gather, arg-max finalisation, accept / commit, residual add.
#pragma once
#include "common.cuh"

namespace lsk {

// ---------------------------------------------------------------------------------------
// weight repacking: HF row-major [rows, cols] bf16 (a [n_rows, K] slice of it) -> the
// fragment-major layout documented in gemm_skinny.cuh.
// ---------------------------------------------------------------------------------------
enum { MAP_PLAIN = 0, MAP_ROPE_HEADS = 1, MAP_GATE = 2, MAP_UP = 3 };

__host__ __device__ inline int64_t map_row(int mode, int64_t r, int hd = 128) {
  switch (mode) {
    case MAP_ROPE_HEADS: {  // rotary pair (d, d + hd/2) -> rows (r, r+8) of one 16-row tile
      const int64_t half = hd >> 1;
      const int64_t head = r / hd, d = r % hd;
      const int64_t dd = d % half, tt = dd >> 3;
      return head * hd + tt * 16 + (d >= half ? 8 : 0) + (dd & 7);
    }
    case MAP_GATE: return (r >> 3) * 16 + (r & 7);
    case MAP_UP: return (r >> 3) * 16 + 8 + (r & 7);
    default: return r;
  }
}

__host__ __device__ inline int64_t packed_elem_offset(int64_t pr, int64_t k, int64_t nsb) {
  const int64_t tile = pr >> 4, rr = pr & 15, g = rr & 7, hi = rr >> 3;
  const int64_t sb = k >> 5, kk = k & 31, t = kk >> 3, j = (kk >> 2) & 1, q = (kk >> 1) & 1,
                half = kk & 1;
  const int64_t reg = q * 2 + hi, lane = g * 4 + t;
  return ((((tile * nsb + sb) * 2 + j) * 32 + lane) * 4 + reg) * 2 + half;
}

// K = source columns taken (even); K_dst = padded K of the packed matrix (multiple of 32; columns
// K .. K_dst-1 keep whatever dst holds: the engine zero-fills its weight buffers at allocation)
__global__ void pack_rows_kernel(const __nv_bfloat16* __restrict__ src, int64_t src_ld,
                                 int64_t src_row0, int64_t src_col0, int64_t n_rows, int64_t K,
                                 __nv_bfloat16* __restrict__ dst, int64_t dst_row0, int mode,
                                 int64_t K_dst, int hd) {
  const int64_t nsb = K_dst >> 5;
  const int64_t pairs = n_rows * (K >> 1);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < pairs;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / (K >> 1), k = (i % (K >> 1)) * 2;
    const uint32_t v = *reinterpret_cast<const uint32_t*>(
        src + (src_row0 + r) * src_ld + src_col0 + k);
    const int64_t pr = dst_row0 + map_row(mode, r, hd);
    *reinterpret_cast<uint32_t*>(dst + packed_elem_offset(pr, k, nsb)) = v;
  }
}

// ---------------------------------------------------------------------------------------
// embedding gather: hidden[row] = float(embed[token])   (llama_model_utils.py:182,242,310)
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void embed_row(const __nv_bfloat16* __restrict__ embed, int hidden,
                                          int token, float* __restrict__ dst, int tid,
                                          int nthreads) {
  const uint2* src = reinterpret_cast<const uint2*>(embed + (size_t)token * hidden);
  for (int i = tid; i < (hidden >> 2); i += nthreads) {
    const uint2 v = src[i];
    *reinterpret_cast<float4*>(dst + i * 4) =
        make_float4(bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y));
  }
}

// rows [0, n): tokens from `ids` (device array) — prompt chunks and the round's first row.
__global__ void embed_tokens_kernel(const __nv_bfloat16* __restrict__ embed, int hidden,
                                    const int* __restrict__ ids, float* __restrict__ rows,
                                    int row_ld) {
  pdl_launch_dependents();
  pdl_wait();
  embed_row(embed, hidden, ids[blockIdx.x], rows + (size_t)blockIdx.x * row_ld, threadIdx.x,
            blockDim.x);
}

// ---------------------------------------------------------------------------------------
// KV slot copy (prefix-shared scoring): entry blockIdx.x = (src page, dst page, t) copies token
// slots [0, t) of one (layer blockIdx.y, K or V, kv head) block from the src page to the dst page.
// The slots of a (page, kv head) block are contiguous rows and are copied slot for slot, so the
// swizzle inside each row (kv_elem_offset) carries over unchanged.
// grid (entries, layers, 2 * n_kv_heads)
// ---------------------------------------------------------------------------------------
__global__ void kv_copy_slots_kernel(const int4* __restrict__ entries, __nv_bfloat16* __restrict__ kpool,
                                     __nv_bfloat16* __restrict__ vpool, size_t layer_elems, int n_kv_heads,
                                     int hd) {
  pdl_launch_dependents();
  pdl_wait();
  const int4 en = entries[blockIdx.x];
  const int head = blockIdx.z >> 1;
  __nv_bfloat16* pool = ((blockIdx.z & 1) ? vpool : kpool) + (size_t)blockIdx.y * layer_elems;
  const uint4* src = reinterpret_cast<const uint4*>(pool + kv_elem_offset(hd, en.x, n_kv_heads, head, 0, 0));
  uint4* dst = reinterpret_cast<uint4*>(pool + kv_elem_offset(hd, en.y, n_kv_heads, head, 0, 0));
  const int n = en.z * hd / 8;
  for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}

// Candidate arg-max reduction for token row `row` (warp-wide, fixed order).
__device__ __forceinline__ int reduce_candidates(const float* __restrict__ val,
                                                 const int* __restrict__ idx, int n_cand,
                                                 int row, int lane) {
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int c = lane; c < n_cand; c += 32) {
    const float v = val[c * kMaxRows + row];
    const int i = idx[c * kMaxRows + row];
    if (better(v, i, bv, bi)) { bv = v; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
  }
  return bi;
}

// Draft step tail: token = argmax(LM-head partials of row 0) -> st->tok[slot]; embed it into
// the next hidden row.  Every CTA reduces redundantly and embeds one slice.
// (decode_next_token greedy branch llama_model_utils.py:120-122 + the `.item()` /
//  re-upload at self_speculation_generator.py:140-145, kept on device.)
__global__ void finalize_embed_kernel(const float* __restrict__ cand_val,
                                      const int* __restrict__ cand_idx, int n_cand,
                                      DevState* __restrict__ st, int slot,
                                      const __nv_bfloat16* __restrict__ embed, int hidden,
                                      float* __restrict__ dst_row) {
  __shared__ int s_tok;
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x < 32) {
    const int tok = reduce_candidates(cand_val, cand_idx, n_cand, 0, threadIdx.x);
    if (threadIdx.x == 0) {
      s_tok = tok;
      if (blockIdx.x == 0) st->tok[slot] = tok;
    }
  }
  __syncthreads();
  const int per = (hidden / 4 + gridDim.x - 1) / gridDim.x;   // float4 per CTA
  const int lo = blockIdx.x * per, hi = min(hidden / 4, lo + per);
  const uint2* src = reinterpret_cast<const uint2*>(embed + (size_t)s_tok * hidden);
  for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    const uint2 v = src[i];
    *reinterpret_cast<float4*>(dst_row + i * 4) =
        make_float4(bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y));
  }
}

// Batched rounds: sequence s's rows are row_ld floats apart.  embed_seq_tokens_kernel embeds
// st[s].tok[0] into rows + s * row_ld (grid n_seqs); finalize_embed_seqs_kernel is
// finalize_embed_kernel for candidate row s = blockIdx.y: its token goes to st[s].tok[slot] and is
// embedded into rows + s * row_ld (grid (slices, n_seqs)).
__global__ void embed_seq_tokens_kernel(const __nv_bfloat16* __restrict__ embed, int hidden,
                                        const DevState* __restrict__ st, float* __restrict__ rows,
                                        int row_ld) {
  pdl_launch_dependents();
  pdl_wait();
  embed_row(embed, hidden, st[blockIdx.x].tok[0], rows + (size_t)blockIdx.x * row_ld, threadIdx.x,
            blockDim.x);
}

__global__ void finalize_embed_seqs_kernel(const float* __restrict__ cand_val,
                                           const int* __restrict__ cand_idx, int n_cand,
                                           DevState* __restrict__ st, int slot,
                                           const __nv_bfloat16* __restrict__ embed, int hidden,
                                           float* __restrict__ rows, int row_ld) {
  __shared__ int s_tok;
  pdl_launch_dependents();
  pdl_wait();
  const int s = blockIdx.y;
  if (threadIdx.x < 32) {
    const int tok = reduce_candidates(cand_val, cand_idx, n_cand, s, threadIdx.x);
    if (threadIdx.x == 0) {
      s_tok = tok;
      if (blockIdx.x == 0) st[s].tok[slot] = tok;
    }
  }
  __syncthreads();
  const int per = (hidden / 4 + gridDim.x - 1) / gridDim.x;   // float4 per CTA
  const int lo = blockIdx.x * per, hi = min(hidden / 4, lo + per);
  const uint2* src = reinterpret_cast<const uint2*>(embed + (size_t)s_tok * hidden);
  float* dst_row = rows + (size_t)s * row_ld;
  for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    const uint2 v = src[i];
    *reinterpret_cast<float4*>(dst_row + i * 4) =
        make_float4(bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y));
  }
}

// Per-generation constants on the device.
struct GenParams {
  int n_eos;
  int eos[8];
  int sample;
  float temperature;
  int top_k;
  float top_p;
  unsigned long long seed;
};

// Mirror of lsk_round_out, written by the accept kernel into mapped pinned host memory.
struct RoundResult {
  int n_drafted, n_matches, n_emitted, kv_len;
  int draft_ids[kMaxRows];
  int emitted_ids[kMaxRows];
  int verified_ids[kMaxRows];
  float conf[kMaxRows];   // adaptive rounds: confidence of each kept draft
  int seq;   // written last: host-visible completion stamp
};

__device__ __forceinline__ bool is_eos(const GenParams& gp, int tok) {
  for (int i = 0; i < gp.n_eos; ++i)
    if (gp.eos[i] == tok) return true;
  return false;
}

// Greedy accept + commit (self_speculation_generator.py:185-190, 203-205, 219-221):
//   verified[j] = argmax of verify row j;  n = longest prefix with draft[j] == verified[j];
//   emitted = draft[:n] + [verified[n]];  every layer's KV length becomes len + n + 1.
// The draft loop's early stop on EOS (:146-148) is restated as "drafts after the first EOS do
// not exist": d_actual = index of first EOS + 1.  Rows past d_actual were computed but, the
// attention being causal, cannot influence rows <= d_actual; their KV entries lie beyond the
// committed length and are overwritten later.
// An adaptive round (d_stop != nullptr) drafted *d_stop tokens of the d it has rows for: drafts
// after the first EOS or the first unsure token do not exist either, and their confidences go out.
// thread-0 part of the greedy accept: compares drafts with the verifier's arg-maxes, commits.
__device__ __forceinline__ void accept_commit(const int* s_ver, int d, DevState* __restrict__ st,
                                              const GenParams& g, RoundResult* __restrict__ res,
                                              int seq, int* __restrict__ hist = nullptr,
                                              const int* __restrict__ d_stop = nullptr) {
  const int d_lim = d_stop != nullptr ? *d_stop : d;
  int d_act = d_lim;
  for (int i = 0; i < d_lim; ++i)
    if (is_eos(g, st->tok[1 + i])) { d_act = i + 1; break; }
  if (d_stop != nullptr)
    for (int i = 0; i < d_act; ++i) res->conf[i] = st->conf[i];
  int n = 0;
  while (n < d_act && st->tok[1 + n] == s_ver[n]) ++n;
  res->n_drafted = d_act;
  res->n_matches = n;
  res->n_emitted = n + 1;
  for (int i = 0; i < d_act; ++i) res->draft_ids[i] = st->tok[1 + i];
  for (int i = 0; i <= d_act; ++i) res->verified_ids[i] = s_ver[i];
  for (int i = 0; i < n; ++i) res->emitted_ids[i] = st->tok[1 + i];
  res->emitted_ids[n] = s_ver[n];
  for (int i = 0; i <= d; ++i) st->verified[i] = s_ver[i];
  if (hist != nullptr)                       // token history for the n-gram ban (prompt ids + output)
    for (int i = 0; i <= n; ++i) hist[st->n_prompt + st->n_out + i] = res->emitted_ids[i];
  st->len += n + 1;
  st->n_out += n + 1;
  st->tok[0] = s_ver[n];
  st->step_count += 1;
  res->kv_len = st->len;
  __threadfence_system();
  *reinterpret_cast<volatile int*>(&res->seq) = seq;
}

__global__ void accept_greedy_kernel(const float* __restrict__ cand_val,
                                     const int* __restrict__ cand_idx, int n_cand, int d,
                                     DevState* __restrict__ st, const GenParams* __restrict__ gp,
                                     RoundResult* __restrict__ res, int seq, int* __restrict__ hist,
                                     const int* __restrict__ d_stop) {
  __shared__ int s_ver[kMaxRows];
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int row = warp; row <= d; row += blockDim.x >> 5) {
    const int tok = reduce_candidates(cand_val, cand_idx, n_cand, row, lane);
    if (lane == 0) s_ver[row] = tok;
  }
  __syncthreads();
  if (threadIdx.x == 0) accept_commit(s_ver, d, st, *gp, res, seq, hist, d_stop);
}

// Batched round: one CTA per sequence s = blockIdx.x, whose verify rows are candidate rows
// s * (d + 1) .. s * (d + 1) + d.  An active sequence accepts and commits as a round of d_seq[s]
// drafts would (accept_commit with d_seq[s] as d_stop: its rows past d_seq[s] are causally invisible
// to the kept ones) into st[s] and res[s]; an inactive one commits nothing and reports no tokens.
__global__ void accept_greedy_seqs_kernel(const float* __restrict__ cand_val,
                                          const int* __restrict__ cand_idx, int n_cand, int d,
                                          DevState* __restrict__ st, const GenParams* __restrict__ gp,
                                          RoundResult* __restrict__ res, const int* __restrict__ d_seq,
                                          const int* __restrict__ active) {
  __shared__ int s_ver[kMaxRows];
  pdl_launch_dependents();
  pdl_wait();
  const int s = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int row = warp; row <= d; row += blockDim.x >> 5) {
    const int tok = reduce_candidates(cand_val, cand_idx, n_cand, s * (d + 1) + row, lane);
    if (lane == 0) s_ver[row] = tok;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  if (active[s]) {
    accept_commit(s_ver, d, &st[s], *gp, &res[s], 0, nullptr, &d_seq[s]);
    return;
  }
  RoundResult* r = &res[s];
  r->n_drafted = r->n_matches = r->n_emitted = 0;
  r->kv_len = st[s].len;
  __threadfence_system();
  *reinterpret_cast<volatile int*>(&r->seq) = 0;
}

// Autoregressive commit (autoregressive_generator.py:62-76): token = argmax(row 0).
__device__ __forceinline__ void ar_commit(int tok, DevState* __restrict__ st,
                                          RoundResult* __restrict__ res, int seq, int* __restrict__ hist = nullptr) {
  if (hist != nullptr) hist[st->n_prompt + st->n_out] = tok;
  st->tok[0] = tok;
  st->len += 1;
  st->n_out += 1;
  st->step_count += 1;
  res->n_drafted = 0;
  res->n_matches = 0;
  res->n_emitted = 1;
  res->emitted_ids[0] = tok;
  res->verified_ids[0] = tok;
  res->kv_len = st->len;
  __threadfence_system();
  *reinterpret_cast<volatile int*>(&res->seq) = seq;
}

__global__ void ar_commit_kernel(const float* __restrict__ cand_val,
                                 const int* __restrict__ cand_idx, int n_cand,
                                 DevState* __restrict__ st, RoundResult* __restrict__ res,
                                 int seq, int* __restrict__ hist) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x < 32) {
    const int tok = reduce_candidates(cand_val, cand_idx, n_cand, 0, threadIdx.x);
    if (threadIdx.x == 0) ar_commit(tok, st, res, seq, hist);
  }
}

// Tensor-parallel helpers: per-rank best candidate per row (so one all-gather of 16 pairs per
// rank suffices), and the residual add that follows the all-reduce of a row-parallel GEMM.
__global__ void rank_best_kernel(const float* __restrict__ cand_val,
                                 const int* __restrict__ cand_idx, int n_cand, int rows,
                                 float* __restrict__ out_val, int* __restrict__ out_idx) {
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int row = warp; row < rows; row += blockDim.x >> 5) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int c = lane; c < n_cand; c += 32) {
      const float v = cand_val[c * kMaxRows + row];
      const int i = cand_idx[c * kMaxRows + row];
      if (better(v, i, bv, bi)) { bv = v; bi = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { out_val[row] = bv; out_idx[row] = bi; }
  }
}

// Tensor-parallel sampling: all-gathered vocab shards [tp][M][vl_pad] -> rows [M][vocab]
// (vocab = tp * vl; the padding columns of every shard are dropped).
__global__ void tp_logits_rows_kernel(const float* __restrict__ gath, int tp, int M, int vl,
                                      int vl_pad, float* __restrict__ full, int ld) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.y;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < tp * vl; j += gridDim.x * blockDim.x) {
    const int r = j / vl, c = j - r * vl;
    full[(size_t)row * ld + j] = gath[((size_t)r * M + row) * vl_pad + c];
  }
}

__global__ void residual_add_kernel(float* __restrict__ hidden, int ld,
                                    const float* __restrict__ delta, int delta_ld, int n_cols) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.y;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (n_cols >> 2);
       i += gridDim.x * blockDim.x) {
    float4 h = *reinterpret_cast<float4*>(hidden + (size_t)row * ld + i * 4);
    const float4 dl = *reinterpret_cast<const float4*>(delta + (size_t)row * delta_ld + i * 4);
    h.x += dl.x; h.y += dl.y; h.z += dl.z; h.w += dl.w;
    *reinterpret_cast<float4*>(hidden + (size_t)row * ld + i * 4) = h;
  }
}

__global__ void set_state_kernel(DevState* st, int len, int tok0, int n_out, int n_prompt) {
  st->len = len;
  st->tok[0] = tok0;
  st->n_out = n_out;
  st->n_prompt = n_prompt;
}

// ---------------------------------------------------------------------------------------
// NoRepeatNGramLogitsProcessor on the device (transformers generation/logits_process.py:
// `_calc_banned_ngram_tokens`; the reference builds it at generator_base.py:77-85).  Row `row` of
// `logits` predicts the token after  seq = hist[0 .. n_prompt + n_out) ++ draft[0 .. j0 + row):
// every token that would complete an n-gram already present in seq gets -inf.  With
// len(seq) + 1 < n nothing is banned (HF's early return); n == 1 bans every token already seen.
// `logits` holds this rank's vocabulary shard [vocab_off, vocab_off + v_local).
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ngram_ban_kernel(float* __restrict__ logits, int ld, int v_local, int vocab_off, const int* __restrict__ hist,
                 const DevState* __restrict__ st, int n, int j0) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x, j = j0 + row;
  const int hlen = st->n_prompt + st->n_out;
  const int L = hlen + j;                                   // tokens in seq
  if (L + 1 < n) return;
  auto tok_at = [&](int i) { return i < hlen ? hist[i] : st->tok[1 + i - hlen]; };
  float* lrow = logits + (size_t)row * ld;
  for (int i = threadIdx.x; i + n - 1 < L; i += blockDim.x) {   // n-gram seq[i .. i+n-1] exists
    bool same = true;
    for (int k = 0; k < n - 1 && same; ++k) same = tok_at(i + k) == tok_at(L - (n - 1) + k);
    if (same) {
      const int banned = tok_at(i + n - 1) - vocab_off;
      if (banned >= 0 && banned < v_local) lrow[banned] = -INFINITY;
    }
  }
}

// arg-max of every logits row (lowest index wins ties) -> one candidate per row, in the layout the
// finalize / accept kernels consume with n_cand == 1.  Used when the logits had to be materialised
// (n-gram ban) instead of taking the arg-max inside the LM-head epilogue.
__global__ void __launch_bounds__(1024)
argmax_rows_kernel(const float* __restrict__ logits, int ld, int v_local, int vocab_off,
                   float* __restrict__ out_val, int* __restrict__ out_idx) {
  __shared__ float s_v[32];
  __shared__ int s_i[32];
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x;
  const float* lrow = logits + (size_t)row * ld;
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int c = threadIdx.x; c < v_local; c += blockDim.x) {
    const float v = lrow[c];
    if (better(v, c, bv, bi)) { bv = v; bi = c; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = bv; s_i[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x < 32) {
    bv = s_v[threadIdx.x];
    bi = s_i[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (threadIdx.x == 0) {
      out_val[row] = bv;
      out_idx[row] = (bi == 0x7fffffff) ? 0x7fffffff : bi + vocab_off;
    }
  }
}

// ---------------------------------------------------------------------------------------
// Teacher-forced scoring: per logits row, log softmax at the target id and the arg-max (lowest
// id wins ties).  One CTA per row, one pass over the `vocab` valid columns (pad columns
// [vocab, ld) are never read): every thread keeps a running (max m, sum s of exp(v - m)) and its
// best (value, id); threads merge by a fixed xor tree, warps in index order, so the result is
// bit-reproducible.  logprob = logit[target] - (m + log s), with expf / logf (not the intrinsics).
// ---------------------------------------------------------------------------------------
constexpr int kLogprobThreads = 512;

__device__ __forceinline__ void lse_merge(float& m, float& s, float om, float os) {
  const float nm = fmaxf(m, om);
  if (nm == -INFINITY) return;                                   // both empty
  s = (m == -INFINITY ? 0.f : s * expf(m - nm)) + (om == -INFINITY ? 0.f : os * expf(om - nm));
  m = nm;
}

__global__ void __launch_bounds__(kLogprobThreads)
logprob_rows_kernel(const float* __restrict__ logits, int ld, int vocab, const int* __restrict__ targets,
                    float* __restrict__ logprob, int* __restrict__ greedy) {
  __shared__ float s_m[kLogprobThreads / 32], s_s[kLogprobThreads / 32], s_bv[kLogprobThreads / 32];
  __shared__ int s_bi[kLogprobThreads / 32];
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* lrow = logits + (size_t)row * ld;
  float m = -INFINITY, s = 0.f, bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int c = threadIdx.x; c < vocab; c += kLogprobThreads) {
    const float v = lrow[c];
    if (better(v, c, bv, bi)) { bv = v; bi = c; }
    if (v == -INFINITY) continue;
    if (v > m) { s = s * expf(m - v) + 1.f; m = v; }             // expf(-inf) = 0 on the first element
    else s += expf(v - m);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    lse_merge(m, s, om, os);
    if (better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
  }
  if (lane == 0) { s_m[warp] = m; s_s[warp] = s; s_bv[warp] = bv; s_bi[warp] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kLogprobThreads / 32; ++w) {
      lse_merge(m, s, s_m[w], s_s[w]);
      if (better(s_bv[w], s_bi[w], bv, bi)) { bv = s_bv[w]; bi = s_bi[w]; }
    }
    logprob[row] = lrow[targets[row]] - (m + logf(s));
    if (greedy != nullptr) greedy[row] = bi;
  }
}

}  // namespace lsk
