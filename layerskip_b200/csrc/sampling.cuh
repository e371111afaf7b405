// sampling.cuh — the reference's sampling branch on the device:
//   decode_next_token  (llama_model_utils.py:109-131): logits / T -> top-k (if > 0) -> top-p
//                      (always) -> softmax -> multinomial
//   rejection test     (self_speculation_generator.py:191-199) + max_fn residual (:27-29)
// Distributions are what must agree with the reference (its RNG stream cannot: torch's CPU
// generator vs a counter-based Philox here), so tests compare the filtered probability rows
// exactly and acceptance statistics within binomial error.
#pragma once
#include "common.cuh"
#include "misc_kernels.cuh"

namespace lsk {

constexpr int kSampleThreads = 1024;

// ---- Philox4x32-10 (Salmon et al.), counter-based: (seed, step, row, purpose) -> 4 x u32
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}
__device__ __forceinline__ float u01(uint32_t x) { return (float)(x >> 8) * (1.0f / 16777216.0f); }

enum { RNG_DRAFT = 1, RNG_VERIFY = 2, RNG_ACCEPT = 3, RNG_RESID = 4 };

__device__ __forceinline__ float rng_uniform(const GenParams& gp, int step, int row, int purpose) {
  const uint4 r = philox4x32_10(make_uint4((uint32_t)step, (uint32_t)row, (uint32_t)purpose, 0x4c534bu),
                                make_uint2((uint32_t)gp.seed, (uint32_t)(gp.seed >> 32)));
  return u01(r.x);
}
// The same draw with the key given explicitly: batched rounds key each sequence by its own seed.
__device__ __forceinline__ float rng_uniform(unsigned long long seed, int step, int row, int purpose) {
  const uint4 r = philox4x32_10(make_uint4((uint32_t)step, (uint32_t)row, (uint32_t)purpose, 0x4c534bu),
                                make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  return u01(r.x);
}

// ---- block-wide helpers (blockDim.x == kSampleThreads), deterministic order
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  float t = (threadIdx.x < (kSampleThreads >> 5)) ? red[threadIdx.x] : 0.f;
  if (w == 0) {
    t = warp_sum(t);
    if (l == 0) red[32] = t;
  }
  __syncthreads();
  return red[32];
}
__device__ __forceinline__ float block_max(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  float t = (threadIdx.x < (kSampleThreads >> 5)) ? red[threadIdx.x] : -INFINITY;
  if (w == 0) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, o));
    if (l == 0) red[32] = t;
  }
  __syncthreads();
  return red[32];
}

// order-preserving key of a float (for radix selection)
__device__ __forceinline__ uint32_t fkey(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// Inverse-CDF draw over weights w[0..V) in index order (torch.multinomial's distribution): the
// token whose interval of the running sum holds target = u * total.  Contiguous chunk per thread;
// before_t is the fp32 block scan of the chunk sums.  In fp32 before_t + local_t is not
// before_{t+1}, so intervals [before_t, before_t + local_t) would leave gaps and overlaps of a few
// ulps at thread boundaries.  Instead the LAST thread with a positive chunk sum and before_t <=
// target owns the target (a max over thread ids: one owner, whatever the order), and walks its own
// chunk: the first token whose running sum exceeds target, else the chunk's last positive weight.
// An all-zero row has no owner: token 0.
__device__ int block_sample_index(const float* __restrict__ w, int V, float u, float* red,
                                  int* s_pick) {
  const int chunk = (V + kSampleThreads - 1) / kSampleThreads;
  const int lo = threadIdx.x * chunk, hi = min(V, lo + chunk);
  float local = 0.f;
  for (int j = lo; j < hi; ++j) local += w[j];
  // exclusive scan of `local` over threads: warp scan + scan of warp totals
  const int wp = threadIdx.x >> 5, l = threadIdx.x & 31;
  float incl = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float n = __shfl_up_sync(0xffffffffu, incl, o);
    if (l >= o) incl += n;
  }
  __syncthreads();
  if (l == 31) red[wp] = incl;
  __syncthreads();
  if (wp == 0) {
    float t = red[l];
    float ti = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float n = __shfl_up_sync(0xffffffffu, ti, o);
      if (l >= o) ti += n;
    }
    red[64 + l] = ti - t;              // exclusive prefix of warp totals
    if (l == 31) red[32] = ti;         // grand total
  }
  if (threadIdx.x == 0) *s_pick = -1;  // holds the owning thread first, then its pick
  __syncthreads();
  const float total = red[32];
  const float target = u * total;
  const float before = red[64 + wp] + (incl - local);
  if (local > 0.f && target >= before) atomicMax(s_pick, (int)threadIdx.x);
  __syncthreads();
  const int owner = *s_pick;
  __syncthreads();
  if (owner < 0) return 0;
  if ((int)threadIdx.x == owner) {
    float run = before;
    int pick = lo;
    for (int j = lo; j < hi; ++j) {
      const float wj = w[j];
      if (wj > 0.f) {
        pick = j;
        run += wj;
        if (target < run) break;
      }
    }
    *s_pick = pick;
  }
  __syncthreads();
  return *s_pick;
}

// block_sample_index alone (lsk_test_draw): CTA i draws from w[0..V) at u[i].
__global__ void __launch_bounds__(kSampleThreads)
draw_index_kernel(const float* __restrict__ w, int V, const float* __restrict__ u, int* __restrict__ picks) {
  __shared__ float red[96 + 32];
  __shared__ int s_pick;
  const int pick = block_sample_index(w, V, u[blockIdx.x], red, &s_pick);
  if (threadIdx.x == 0) picks[blockIdx.x] = pick;
}

// The warp of decode_next_token on one logits row lg[0 .. V) by one CTA of kSampleThreads: logits
// / T -> top-k threshold -> softmax -> nucleus -> renormalised probabilities in pr[0 .. V).  Shared
// by the sampling path and the acceptance kernels below, so a predicted acceptance probability
// uses the arithmetic generation draws from.  Ends with a barrier: pr is then readable by the
// whole CTA.  Shared scratch: red [96 + 32], hist [512], s_prefix, s_g.
// The nucleus masses are summed as integers (probability * 2^43, truncated; two 32-bit limbs per
// bucket, hist[b] the high and hist[256 + b] the low 12 bits, neither of which can overflow below a
// vocabulary of 2^20): the atomic bucket sums then do not depend on the order the threads arrive in,
// so a row whose mass sits on top_p keeps the same support every time.
constexpr float kMassScale = 8796093022208.f;   // 2^43
__device__ __forceinline__ void warp_row(const float* __restrict__ lg, int V, float temperature, int top_k,
                                         float top_p, float* __restrict__ pr, float* red, uint32_t* hist,
                                         uint32_t& s_prefix, float& s_g) {
  const float inv_t = 1.0f / temperature;

  // ---- top-k threshold (HF TopKLogitsWarper: drop scores < k-th largest)
  float kth = -INFINITY;
  if (top_k > 0 && top_k < V) {
    __shared__ int cnt[256];
    uint32_t prefix = 0;
    int need = top_k;                    // how many keys >= threshold still to take
    for (int level = 3; level >= 0; --level) {
      for (int i = threadIdx.x; i < 256; i += kSampleThreads) cnt[i] = 0;
      __syncthreads();
      const uint32_t hi_mask = level == 3 ? 0u : (0xffffffffu << (8 * (level + 1)));
      for (int j = threadIdx.x; j < V; j += kSampleThreads) {
        const uint32_t k = fkey(lg[j] * inv_t);
        if ((k & hi_mask) == (prefix & hi_mask)) atomicAdd(&cnt[(k >> (8 * level)) & 255], 1);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        int b = 255, acc = 0;
        for (; b > 0; --b) {
          if (acc + cnt[b] >= need) break;
          acc += cnt[b];
        }
        need -= acc;
        s_prefix = prefix | ((uint32_t)b << (8 * level));
      }
      __syncthreads();
      prefix = s_prefix;
      if (threadIdx.x == 0) { /* need is thread-0 private; broadcast via smem */ s_g = (float)need; }
      __syncthreads();
      need = (int)s_g;
    }
    const uint32_t kb = (prefix & 0x80000000u) ? (prefix & 0x7fffffffu) : ~prefix;
    kth = __uint_as_float(kb);
  }

  // ---- softmax numerator of the (top-k filtered) row
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < V; j += kSampleThreads) {
    const float v = lg[j] * inv_t;
    if (v >= kth) mx = fmaxf(mx, v);
  }
  mx = block_max(mx, red);
  float z = 0.f;
  for (int j = threadIdx.x; j < V; j += kSampleThreads) {
    const float v = lg[j] * inv_t;
    const float e = (v >= kth) ? __expf(v - mx) : 0.f;
    pr[j] = e;
    z += e;
  }
  z = block_sum(z, red);
  const float inv_z = 1.0f / z;

  // ---- nucleus: keep token i iff the mass of strictly larger tokens is < top_p
  uint32_t kstar = 0;                    // keep keys >= kstar
  if (top_p >= 0.f && top_p < 1.0f) {
    __shared__ unsigned long long s_mass;
    const unsigned long long p_fix = (unsigned long long)((double)top_p * (double)kMassScale);
    uint32_t prefix = 0;
    unsigned long long G = 0;            // mass above the bucket being refined
    for (int level = 3; level >= 0; --level) {
      for (int i = threadIdx.x; i < 512; i += kSampleThreads) hist[i] = 0u;
      __syncthreads();
      const uint32_t hi_mask = level == 3 ? 0u : (0xffffffffu << (8 * (level + 1)));
      for (int j = threadIdx.x; j < V; j += kSampleThreads) {
        const float p = pr[j] * inv_z;
        const uint32_t k = __float_as_uint(p);       // p >= 0: bit order == value order
        if (p > 0.f && (k & hi_mask) == (prefix & hi_mask))
        {
          const unsigned long long q = __float2ull_rz(p * kMassScale);
          const int b = (k >> (8 * level)) & 255;
          atomicAdd(&hist[b], (uint32_t)(q >> 12));
          atomicAdd(&hist[256 + b], (uint32_t)q & 4095u);
        }
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        int b = 255;
        unsigned long long g = G;
        for (; b > 0; --b) {
          const unsigned long long h = ((unsigned long long)hist[b] << 12) + hist[256 + b];
          if (g + h >= p_fix) break;
          g += h;
        }
        s_mass = g;
        s_prefix = prefix | ((uint32_t)b << (8 * level));
      }
      __syncthreads();
      prefix = s_prefix;
      G = s_mass;
    }
    kstar = prefix;
  }
  {  // min_tokens_to_keep = 1: the arg-max (numerator exp(0) = 1) always survives
    const uint32_t kmax = __float_as_uint(inv_z);
    if (kstar > kmax) kstar = kmax;
  }
  float z2 = 0.f;
  for (int j = threadIdx.x; j < V; j += kSampleThreads) {
    const float e = pr[j];
    const bool keep = e > 0.f && __float_as_uint(e * inv_z) >= kstar;
    z2 += keep ? e : 0.f;
  }
  z2 = block_sum(z2, red);
  const float inv_z2 = 1.0f / z2;
  for (int j = threadIdx.x; j < V; j += kSampleThreads) {
    const float e = pr[j];
    const bool keep = e > 0.f && __float_as_uint(e * inv_z) >= kstar;
    pr[j] = keep ? e * inv_z2 : 0.f;
  }
  __syncthreads();
}

// One row per CTA: logits -> warped probabilities (written out) -> sampled token.
//   grid.x rows; row r reads logits + r*ld, writes probs + r*V and tok_out[r].
__global__ void __launch_bounds__(kSampleThreads)
warp_and_sample_kernel(const float* __restrict__ logits, int ld, int V,
                       const GenParams* __restrict__ gpp, const DevState* __restrict__ st,
                       float* __restrict__ probs, int* __restrict__ tok_out, int purpose,
                       int row_base) {
  __shared__ float red[96 + 32];
  __shared__ uint32_t hist[512];
  __shared__ uint32_t s_prefix;
  __shared__ float s_g;
  __shared__ int s_pick;
  pdl_launch_dependents();
  pdl_wait();
  const GenParams gp = *gpp;
  const int row = blockIdx.x;
  float* pr = probs + (size_t)row * V;
  warp_row(logits + (size_t)row * ld, V, gp.temperature, gp.top_k, gp.top_p, pr, red, hist, s_prefix, s_g);

  // ---- multinomial draw
  const float u = rng_uniform(gp, st->step_count, row_base + row, purpose);
  const int tok = block_sample_index(pr, V, u, red, &s_pick);
  if (threadIdx.x == 0) tok_out[row] = tok;
}

// ---------------------------------------------------------------------------------------------
// Acceptance probability of a sampled draft (lsk_score_exits).  The accept test u < min(1, p_L(t)
// / p_E(t)) with t ~ p_E accepts with probability alpha = sum_v min(p_E(v), p_L(v)), p the warped
// distributions of one position at the exit E and at full depth.  The warp settings travel by
// value: a scoring call never touches a generation's GenParams.
// ---------------------------------------------------------------------------------------------
struct WarpParams {
  float temperature;
  int top_k;
  float top_p;
};

// grid.x rows: row r of logits (ld floats apart, V valid columns) -> warped row at probs + r*V
__global__ void __launch_bounds__(kSampleThreads)
warp_rows_kernel(const float* __restrict__ logits, int ld, int V, WarpParams wp, float* __restrict__ probs) {
  __shared__ float red[96 + 32];
  __shared__ uint32_t hist[512];
  __shared__ uint32_t s_prefix;
  __shared__ float s_g;
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x;
  warp_row(logits + (size_t)row * ld, V, wp.temperature, wp.top_k, wp.top_p, probs + (size_t)row * V, red, hist,
           s_prefix, s_g);
}

// grid.x full-depth rows: warp row r of logits into scratch + r*V, then for every draft exit j
// accept[j * accept_ld + r] = sum_v min(p_draft[j * draft_stride + r*V + v], p_full(v)): per-thread
// strided sums merged by block_sum, a fixed order, so the result is bit-reproducible.
__global__ void __launch_bounds__(kSampleThreads)
accept_prob_kernel(const float* __restrict__ logits, int ld, int V, WarpParams wp,
                   const float* __restrict__ p_draft, size_t draft_stride, int n_draft,
                   float* __restrict__ scratch, float* __restrict__ accept, size_t accept_ld) {
  __shared__ float red[96 + 32];
  __shared__ uint32_t hist[512];
  __shared__ uint32_t s_prefix;
  __shared__ float s_g;
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x;
  float* pv = scratch + (size_t)row * V;
  warp_row(logits + (size_t)row * ld, V, wp.temperature, wp.top_k, wp.top_p, pv, red, hist, s_prefix, s_g);
  for (int j = 0; j < n_draft; ++j) {
    const float* pd = p_draft + j * draft_stride + (size_t)row * V;
    float s = 0.f;
    for (int v = threadIdx.x; v < V; v += kSampleThreads) s += fminf(pd[v], pv[v]);
    s = block_sum(s, red);
    if (threadIdx.x == 0) accept[j * accept_ld + row] = s;
  }
}

// Rejection test + commit for the sampling path (self_speculation_generator.py:191-221).
__global__ void __launch_bounds__(kSampleThreads)
accept_sample_kernel(const float* __restrict__ p_draft, const float* __restrict__ p_verify, int V,
                     int d, DevState* __restrict__ st, const GenParams* __restrict__ gpp,
                     RoundResult* __restrict__ res, float* __restrict__ scratch, int seq,
                     int* __restrict__ hist, const int* __restrict__ d_stop) {
  __shared__ float red[96 + 32];
  __shared__ int s_pick;
  __shared__ int s_n, s_dact, s_reject;
  pdl_launch_dependents();
  pdl_wait();
  const GenParams gp = *gpp;
  if (threadIdx.x == 0) {
    // adaptive rounds: only the first *d_stop drafts exist (accept_commit)
    const int d_lim = d_stop != nullptr ? *d_stop : d;
    int d_act = d_lim;
    for (int i = 0; i < d_lim; ++i)
      if (is_eos(gp, st->tok[1 + i])) { d_act = i + 1; break; }
    if (d_stop != nullptr)
      for (int i = 0; i < d_act; ++i) res->conf[i] = st->conf[i];
    int n = 0, reject = -1;
    for (int i = 0; i < d_act; ++i) {
      const int t = st->tok[1 + i];
      const float pv = p_verify[(size_t)i * V + t], pd = p_draft[(size_t)i * V + t];
      const float u = rng_uniform(gp, st->step_count, i, RNG_ACCEPT);
      if (u < fminf(1.0f, pv / pd)) ++n;
      else { reject = i; break; }
    }
    s_n = n; s_dact = d_act; s_reject = reject;
  }
  __syncthreads();
  const int n = s_n, d_act = s_dact, reject = s_reject;
  int bonus;
  if (reject >= 0) {
    // resample from norm(max(p_v - p_d, 0))   (max_fn, :27-29)
    const float* pv = p_verify + (size_t)reject * V;
    const float* pd = p_draft + (size_t)reject * V;
    for (int j = threadIdx.x; j < V; j += kSampleThreads) scratch[j] = fmaxf(pv[j] - pd[j], 0.f);
    __syncthreads();
    const float u = rng_uniform(gp, st->step_count, reject, RNG_RESID);
    bonus = block_sample_index(scratch, V, u, red, &s_pick);
  } else {
    bonus = st->verified[n];             // the verifier's own draw at row n (= d_act)
  }
  if (threadIdx.x == 0) {
    res->n_drafted = d_act;
    res->n_matches = n;
    res->n_emitted = n + 1;
    for (int i = 0; i < d_act; ++i) res->draft_ids[i] = st->tok[1 + i];
    for (int i = 0; i <= d_act; ++i) res->verified_ids[i] = st->verified[i];
    res->verified_ids[n] = bonus;
    for (int i = 0; i < n; ++i) res->emitted_ids[i] = st->tok[1 + i];
    res->emitted_ids[n] = bonus;
    if (hist != nullptr)
      for (int i = 0; i <= n; ++i) hist[st->n_prompt + st->n_out + i] = res->emitted_ids[i];
    st->len += n + 1;
    st->n_out += n + 1;
    st->tok[0] = bonus;
    st->step_count += 1;
    res->kv_len = st->len;
    __threadfence_system();
    *reinterpret_cast<volatile int*>(&res->seq) = seq;
  }
}

// ---------------------------------------------------------------------------------------------
// Batched sampled rounds (lsk_round_batch after lsk_prefill_batch_seeded).  Sequence s owns rows
// s * seq_rows .. s * seq_rows + seq_rows - 1 of probs_d / probs_v (seq_rows = d + 1) and draws
// with its own seed seeds[s] at its own step count, with the counters a round of that sequence
// alone uses, so each sequence's draws do not depend on the rest of the batch.
// ---------------------------------------------------------------------------------------------
// warp_and_sample_kernel for several sequences: CTA r serves sequence s = r / rows_per_seq and its
// row j = r % rows_per_seq.  It warps logits row r, writes the warped row to probs row
// s * seq_rows + row_base + j, draws with counter (st[s].step_count, row_base + j, purpose) into
// tok_out[s * (DevState ints) + j] (tok_out points into st[0]) and, when `embed` is set, embeds
// the token into emb_rows + s * emb_ld.
//   draft step i: grid B, rows_per_seq 1, row_base i, tok_out &st[0].tok[1 + i];
//   verify:       grid B * seq_rows, rows_per_seq seq_rows, row_base 0, tok_out &st[0].verified[0].
__global__ void __launch_bounds__(kSampleThreads)
warp_and_sample_seqs_kernel(const float* __restrict__ logits, int ld, int V,
                            const GenParams* __restrict__ gpp, const DevState* __restrict__ st,
                            const unsigned long long* __restrict__ seeds, int rows_per_seq, int seq_rows,
                            int row_base, int purpose, float* __restrict__ probs, int* __restrict__ tok_out,
                            const __nv_bfloat16* __restrict__ embed, int hidden,
                            float* __restrict__ emb_rows, int emb_ld) {
  __shared__ float red[96 + 32];
  __shared__ uint32_t hist[512];
  __shared__ uint32_t s_prefix;
  __shared__ float s_g;
  __shared__ int s_pick;
  pdl_launch_dependents();
  pdl_wait();
  const GenParams gp = *gpp;
  const int r = blockIdx.x;
  const int s = r / rows_per_seq, j = r - s * rows_per_seq;
  float* pr = probs + ((size_t)s * seq_rows + row_base + j) * V;
  warp_row(logits + (size_t)r * ld, V, gp.temperature, gp.top_k, gp.top_p, pr, red, hist, s_prefix, s_g);
  const float u = rng_uniform(seeds[s], st[s].step_count, row_base + j, purpose);
  const int tok = block_sample_index(pr, V, u, red, &s_pick);
  if (threadIdx.x == 0) tok_out[(size_t)s * (sizeof(DevState) / sizeof(int)) + j] = tok;
  if (embed != nullptr) embed_row(embed, hidden, tok, emb_rows + (size_t)s * emb_ld, threadIdx.x, blockDim.x);
}

// accept_sample_kernel for a batch: CTA s serves sequence s, whose drafts are rows s * (d + 1) .. of
// probs_d and verify rows the same rows of probs_v.  An active sequence runs the rejection test and
// residual resample with its own seed and d_seq[s] as d_stop (as accept_greedy_seqs_kernel), and
// commits into st[s] / res[s]; its residual goes to probs_d row s * (d + 1) + d, which no draft
// writes.  An inactive sequence commits nothing and reports no tokens.  The body restates
// accept_sample_kernel's rather than sharing it: routing that kernel through a common function
// changes its instructions.
__global__ void __launch_bounds__(kSampleThreads)
accept_sample_seqs_kernel(float* __restrict__ probs_d, const float* __restrict__ probs_v, int V, int d,
                          DevState* __restrict__ sts, const GenParams* __restrict__ gpp,
                          const unsigned long long* __restrict__ seeds, RoundResult* __restrict__ ress,
                          const int* __restrict__ d_seq, const int* __restrict__ active) {
  __shared__ float red[96 + 32];
  __shared__ int s_pick;
  __shared__ int s_n, s_dact, s_reject;
  pdl_launch_dependents();
  pdl_wait();
  const int s = blockIdx.x;
  DevState* st = &sts[s];
  RoundResult* res = &ress[s];
  if (!active[s]) {
    if (threadIdx.x == 0) {
      res->n_drafted = res->n_matches = res->n_emitted = 0;
      res->kv_len = st->len;
      __threadfence_system();
      *reinterpret_cast<volatile int*>(&res->seq) = 0;
    }
    return;
  }
  const GenParams gp = *gpp;
  const unsigned long long seed = seeds[s];
  const float* p_draft = probs_d + (size_t)s * (d + 1) * V;
  const float* p_verify = probs_v + (size_t)s * (d + 1) * V;
  if (threadIdx.x == 0) {
    const int d_lim = d_seq[s];
    int d_act = d_lim;
    for (int i = 0; i < d_lim; ++i)
      if (is_eos(gp, st->tok[1 + i])) { d_act = i + 1; break; }
    int n = 0, reject = -1;
    for (int i = 0; i < d_act; ++i) {
      const int t = st->tok[1 + i];
      const float pv = p_verify[(size_t)i * V + t], pd = p_draft[(size_t)i * V + t];
      const float u = rng_uniform(seed, st->step_count, i, RNG_ACCEPT);
      if (u < fminf(1.0f, pv / pd)) ++n;
      else { reject = i; break; }
    }
    s_n = n; s_dact = d_act; s_reject = reject;
  }
  __syncthreads();
  const int n = s_n, d_act = s_dact, reject = s_reject;
  int bonus;
  if (reject >= 0) {
    // resample from norm(max(p_v - p_d, 0))   (max_fn, :27-29)
    float* scratch = probs_d + ((size_t)s * (d + 1) + d) * V;
    const float* pv = p_verify + (size_t)reject * V;
    const float* pd = p_draft + (size_t)reject * V;
    for (int j = threadIdx.x; j < V; j += kSampleThreads) scratch[j] = fmaxf(pv[j] - pd[j], 0.f);
    __syncthreads();
    const float u = rng_uniform(seed, st->step_count, reject, RNG_RESID);
    bonus = block_sample_index(scratch, V, u, red, &s_pick);
  } else {
    bonus = st->verified[n];             // the verifier's own draw at row n (= d_act)
  }
  if (threadIdx.x == 0) {
    res->n_drafted = d_act;
    res->n_matches = n;
    res->n_emitted = n + 1;
    for (int i = 0; i < d_act; ++i) res->draft_ids[i] = st->tok[1 + i];
    for (int i = 0; i <= d_act; ++i) res->verified_ids[i] = st->verified[i];
    res->verified_ids[n] = bonus;
    for (int i = 0; i < n; ++i) res->emitted_ids[i] = st->tok[1 + i];
    res->emitted_ids[n] = bonus;
    st->len += n + 1;
    st->n_out += n + 1;
    st->tok[0] = bonus;
    st->step_count += 1;
    res->kv_len = st->len;
    __threadfence_system();
    *reinterpret_cast<volatile int*>(&res->seq) = 0;
  }
}

// AR commit when the token was sampled into st->verified[0].
__global__ void ar_commit_sampled_kernel(DevState* __restrict__ st, RoundResult* __restrict__ res,
                                         int seq, int* __restrict__ hist) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) {
    const int tok = st->verified[0];
    if (hist != nullptr) hist[st->n_prompt + st->n_out] = tok;
    st->tok[0] = tok;
    st->len += 1;
    st->n_out += 1;
    st->step_count += 1;
    res->n_drafted = 0; res->n_matches = 0; res->n_emitted = 1;
    res->emitted_ids[0] = tok; res->verified_ids[0] = tok;
    res->kv_len = st->len;
    __threadfence_system();
    *reinterpret_cast<volatile int*>(&res->seq) = seq;
  }
}

// ---------------------------------------------------------------------------------------------
// Confidence-threshold drafting (lsk_round_adaptive).  After draft step j has chosen tok[1 + j]:
//   conf[j] = the probability of that token under the distribution it was chosen from:
//             greedy   softmax(logits row)[arg-max] = 1 / sum_v exp(l_v - max_v l_v)  (T = 1, after the
//                      n-gram ban when there is one), a log-sum-exp over the CTAs' column slices;
//             sampling probs[tok], the warped row warp_and_sample_kernel drew from.
//   The round stops after draft j (d_stop = j + 1) when it is an EOS, when conf[j] < min_conf, or
//   when j + 1 == d_max; otherwise d_stop = d_max until a later step stops it.  `next` is the graph
//   conditional that runs step j + 1: set to 1 to go on (its default at every launch is 0).
// Step 0 also zeroes hidden rows 2 .. d_max: only later draft steps write them, and the verify runs
// layers >= E on every row, so a row the round skips must hold finite values (0 x NaN in P.V would
// reach the kept rows).  Causality keeps those rows out of the kept ones.
// The slices' (max, sum) partials are merged in CTA order by the last CTA to arrive, so the result
// does not depend on timing; it resets the arrival counter for the next launch.
// ---------------------------------------------------------------------------------------------
constexpr int kConfThreads = 512;
constexpr int kConfMaxCtas = 64;
constexpr int kConfCols = 4096;          // columns per CTA (grid = ceil(V / kConfCols), <= kConfMaxCtas)

struct ConfScratch {
  float m[kConfMaxCtas], s[kConfMaxCtas];
  unsigned int arrive;
};

__global__ void __launch_bounds__(kConfThreads)
draft_confidence_kernel(const float* __restrict__ logits, const float* __restrict__ probs, int V,
                        DevState* __restrict__ st, const GenParams* __restrict__ gpp, ConfScratch* __restrict__ cs,
                        int j, int d_max, float* __restrict__ hidden, int hidden_ld,
                        cudaGraphConditionalHandle next, int has_next) {
  __shared__ float s_m[kConfThreads / 32], s_s[kConfThreads / 32];
  __shared__ int s_last;
  pdl_launch_dependents();
  pdl_wait();
  if (j == 0) {
    const int n4 = (d_max - 1) * (hidden_ld >> 2);
    float4* dst = reinterpret_cast<float4*>(hidden + 2 * (size_t)hidden_ld);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x)
      dst[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float conf;
  if (logits != nullptr) {
    const int per = (V + gridDim.x - 1) / gridDim.x;
    const int lo = blockIdx.x * per, hi = min(V, lo + per);
    float m = -INFINITY, s = 0.f;
    for (int c = lo + threadIdx.x; c < hi; c += kConfThreads) {
      const float v = logits[c];
      if (v == -INFINITY) continue;
      if (v > m) { s = s * expf(m - v) + 1.f; m = v; }
      else s += expf(v - m);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
      lse_merge(m, s, om, os);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { s_m[warp] = m; s_s[warp] = s; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kConfThreads / 32; ++w) lse_merge(m, s, s_m[w], s_s[w]);
      cs->m[blockIdx.x] = m;
      cs->s[blockIdx.x] = s;
      __threadfence();
      s_last = atomicAdd(&cs->arrive, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last || threadIdx.x != 0) return;
    __threadfence();
    m = __ldcg(&cs->m[0]);
    s = __ldcg(&cs->s[0]);
    for (int b = 1; b < gridDim.x; ++b) lse_merge(m, s, __ldcg(&cs->m[b]), __ldcg(&cs->s[b]));
    cs->arrive = 0;
    conf = 1.0f / s;
  } else {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    conf = probs[st->tok[1 + j]];
  }
  if (j > 0 && st->d_stop <= j) return;   // eager launches only: an earlier draft already ended the round
  const GenParams gp = *gpp;
  st->conf[j] = conf;
  const bool stop = j + 1 == d_max || is_eos(gp, st->tok[1 + j]) || conf < st->min_conf;
  st->d_stop = stop ? j + 1 : d_max;
  if (has_next) cudaGraphSetConditional(next, stop ? 0u : 1u);
}

// ---------------------------------------------------------------------------------------------
// Confidence-threshold drafting for a batch (lsk_round_batch_adaptive).  Draft step j of sequence
// s = blockIdx.y: the confidence of its draft row and the solo stop rule, with d_seq[s] for d_max,
// into st[s] and d_stop[s] (what the batched accept kernels take as their d_seq).  Sequence s drafts
// at step j iff it is active and j < its d_stop (j < d_seq[s] at step 0); a sequence that stopped
// still has its rows computed while others draft on, but its d_stop and confidences stay as they
// were.  Draft step j + 1 runs iff some active sequence has d_stop > j + 1: the last sequence to be
// decided sets the conditional (an OR over the final d_stop values, so the vote does not depend on
// timing).  Greedy confidences partition, walk and merge the columns exactly as
// draft_confidence_kernel (grid.x = its grid), so they are bit-identical to a solo round's; sampled
// ones read probs row s * seq_rows + j (grid.x = 1).  Step 0 zeroes hidden rows 2 .. d of every
// sequence (rows s * seq_rows + 2 .., d = seq_rows - 1), for the reason draft_confidence_kernel
// gives.  The body restates draft_confidence_kernel's rather than sharing it, which would change
// that kernel's instructions.
// ---------------------------------------------------------------------------------------------
struct ConfSeqsScratch {
  float m[kMaxRows][kConfMaxCtas], s[kMaxRows][kConfMaxCtas];
  unsigned int arrive[kMaxRows];         // column slices of sequence s merged in this launch
  unsigned int decided;                  // sequences decided in this launch
  int d_stop[kMaxRows];                  // drafts sequence s keeps (seeded from d_seq at step 0)
  float min_conf;                        // the batch's threshold, set by the host before each round
};

__global__ void __launch_bounds__(kConfThreads)
draft_confidence_seqs_kernel(const float* __restrict__ logits, int ld, const float* __restrict__ probs, int V,
                             int seq_rows, DevState* __restrict__ sts, const GenParams* __restrict__ gpp,
                             RoundResult* __restrict__ ress, ConfSeqsScratch* __restrict__ cs,
                             const int* __restrict__ d_seq, const int* __restrict__ active, int j,
                             float* __restrict__ hidden, int hidden_ld, cudaGraphConditionalHandle next,
                             int has_next) {
  __shared__ float s_m[kConfThreads / 32], s_s[kConfThreads / 32];
  __shared__ int s_last;
  pdl_launch_dependents();
  pdl_wait();
  const int q = blockIdx.y;
  if (j == 0) {
    const int n4 = (seq_rows - 2) * (hidden_ld >> 2);
    float4* dst = reinterpret_cast<float4*>(hidden + ((size_t)q * seq_rows + 2) * hidden_ld);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x)
      dst[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  DevState* st = &sts[q];
  float conf;
  if (logits != nullptr) {
    const float* row = logits + (size_t)q * ld;
    const int per = (V + gridDim.x - 1) / gridDim.x;
    const int lo = blockIdx.x * per, hi = min(V, lo + per);
    float m = -INFINITY, s = 0.f;
    for (int c = lo + threadIdx.x; c < hi; c += kConfThreads) {
      const float v = row[c];
      if (v == -INFINITY) continue;
      if (v > m) { s = s * expf(m - v) + 1.f; m = v; }
      else s += expf(v - m);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
      lse_merge(m, s, om, os);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { s_m[warp] = m; s_s[warp] = s; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kConfThreads / 32; ++w) lse_merge(m, s, s_m[w], s_s[w]);
      cs->m[q][blockIdx.x] = m;
      cs->s[q][blockIdx.x] = s;
      __threadfence();
      s_last = atomicAdd(&cs->arrive[q], 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last || threadIdx.x != 0) return;
    __threadfence();
    m = __ldcg(&cs->m[q][0]);
    s = __ldcg(&cs->s[q][0]);
    for (int b = 1; b < gridDim.x; ++b) lse_merge(m, s, __ldcg(&cs->m[q][b]), __ldcg(&cs->s[q][b]));
    cs->arrive[q] = 0;
    conf = 1.0f / s;
  } else {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    conf = probs[((size_t)q * seq_rows + j) * V + st->tok[1 + j]];
  }
  // one thread per sequence from here on
  const int d_lim = d_seq[q];
  const int prev = j == 0 ? d_lim : cs->d_stop[q];
  if (active[q] && j < prev) {
    const GenParams gp = *gpp;
    st->conf[j] = conf;
    ress[q].conf[j] = conf;              // the sampled accept does not copy confidences
    const bool stop = j + 1 == d_lim || is_eos(gp, st->tok[1 + j]) || conf < cs->min_conf;
    st->d_stop = cs->d_stop[q] = stop ? j + 1 : d_lim;
  } else if (j == 0) {
    st->d_stop = cs->d_stop[q] = prev;
  }
  __threadfence();
  if (atomicAdd(&cs->decided, 1u) != gridDim.y - 1) return;
  __threadfence();
  cs->decided = 0;
  if (!has_next) return;
  unsigned int go = 0;
  for (int r = 0; r < (int)gridDim.y; ++r)
    if (active[r] && __ldcg(&cs->d_stop[r]) > j + 1) go = 1u;
  cudaGraphSetConditional(next, go);
}

}  // namespace lsk
