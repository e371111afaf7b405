/*
 * lsk.h — C ABI of the H100-native LayerSkip self-speculative decoding engine (liblsk.so).
 *
 * The reference (facebookresearch/LayerSkip) has NO FFI: its hot path is Python calling
 * HuggingFace modules.  This ABI is what a binding for that path would bind; each entry point
 * names the reference code it replaces (paths relative to the reference root).  Plain C types
 * only — device pointers travel as `const void*`, streams are owned by the engine.  Every call
 * returns 0 on success or a negative lsk_status; the text is available from lsk_last_error().
 * Not re-entrant: one host thread drives one engine (the reference is single-threaded too,
 * self_speculation/generator_base.py:97-130).
 */
#ifndef LSK_H_
#define LSK_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LSK_ABI_VERSION 2
#define LSK_MAX_SPEC 15      /* D_max: verify handles up to 16 rows (D+1)                    */
#define LSK_MAX_EOS 8

typedef enum {
  LSK_OK = 0,
  LSK_ERR_INVALID = -1,      /* bad argument / unsupported shape                             */
  LSK_ERR_CUDA = -2,         /* CUDA runtime error (message has the CUDA string)             */
  LSK_ERR_STATE = -3,        /* call order violated (e.g. round before prefill)              */
  LSK_ERR_NCCL = -4,
  LSK_ERR_NOMEM = -5,
  LSK_ERR_CTX = -6           /* sequence would exceed max_ctx                                */
} lsk_status;

/* flags */
#define LSK_FLAG_KEEP_LOGITS 1u  /* also store fp32 logits (needed for sampling / debug reads) */
#define LSK_FLAG_NO_PDL 2u       /* disable programmatic dependent launch                    */
#define LSK_FLAG_NO_GRAPH 4u     /* launch kernels eagerly instead of replaying CUDA graphs  */
#define LSK_FLAG_NO_PREFILL_TC 8u /* keep only the decode-layout weights: the prompt pass runs 16 rows at a time on the decode kernels instead of 128 rows at a time on wgmma (saves the second, canonical-layout weight copy) */
#define LSK_FLAG_TP_NCCL 16u     /* tp_size > 1: use NCCL all-reduce instead of the one-shot kernels over peer-mapped HBM */

/* Llama architecture + engine sizing.  Replaces what the reference reads off the HF model
 * object (`model.config`, generate.py:54-67). */
typedef struct {
  int32_t vocab, hidden, inter, n_layers, n_heads, n_kv_heads, head_dim;
  float rms_eps, rope_theta;
  int32_t max_ctx;           /* prompt + generated tokens the KV pool must hold              */
  int32_t tp_rank, tp_size;  /* tensor-parallel shard of this process (1 process per GPU)    */
  int32_t attn_splits;       /* split-KV factor (0 = default)                                */
  uint32_t flags;
  /* RoPE frequency scaling (HF `rope_scaling` / `rope_parameters`, transformers
   * modeling_rope_utils.py: _compute_linear_scaling_rope_parameters, _compute_llama3_parameters):
   * 0 default, 1 linear (inv_freq / factor), 2 llama3 (Llama-3.1 / 3.2 checkpoints such as
   * facebook/layerskip-llama3.2-1B, the reference's own test model, tests/tests_constants.py:9). */
  int32_t rope_scaling;
  float rope_factor, rope_low_freq_factor, rope_high_freq_factor;
  int32_t rope_original_max_pos;
} lsk_config;
#define LSK_ROPE_DEFAULT 0
#define LSK_ROPE_LINEAR 1
#define LSK_ROPE_LLAMA3 2

/* Which HF tensor a weight descriptor carries (names as in
 * transformers LlamaForCausalLM.state_dict(); call sites llama_model_utils.py:182,193,204-205). */
typedef enum {
  LSK_W_EMBED = 0,           /* model.embed_tokens.weight            [vocab, hidden]          */
  LSK_W_FINAL_NORM = 1,      /* model.norm.weight                    [hidden]                 */
  LSK_W_LM_HEAD = 2,         /* lm_head.weight                       [vocab, hidden]          */
  LSK_W_LN1 = 3,             /* layers.i.input_layernorm.weight      [hidden]                 */
  LSK_W_Q = 4, LSK_W_K = 5, LSK_W_V = 6, LSK_W_O = 7,   /* self_attn.{q,k,v,o}_proj.weight     */
  LSK_W_LN2 = 8,             /* layers.i.post_attention_layernorm.weight                      */
  LSK_W_GATE = 9, LSK_W_UP = 10, LSK_W_DOWN = 11         /* mlp.{gate,up,down}_proj.weight      */
} lsk_weight_role;

/* One full (unsharded) bf16 tensor in DEVICE memory, row-major [rows, cols] as HF stores it.
 * The engine slices its tensor-parallel shard, repacks it into its own HBM layout and does not
 * keep the pointer: the caller may free the tensor when lsk_load_weights returns. */
typedef struct {
  int32_t role;              /* lsk_weight_role                                              */
  int32_t layer;             /* decoder layer index, ignored for embed / final norm / head   */
  const void* data;          /* device pointer, bf16                                         */
  int64_t rows, cols;
} lsk_weight_desc;

/* Per-generation settings: `GenerationConfig` (self_speculation/generator_base.py:33-49) plus the
 * eos list built at generator_base.py:106. */
typedef struct {
  int32_t exit_layer;        /* E; <= 0 means "all layers" for lsk_ar_step                   */
  int32_t max_steps;
  int32_t n_eos;
  int32_t eos_ids[LSK_MAX_EOS];
  int32_t sample;            /* 0 greedy (arg-max), 1 sampling                               */
  float temperature;
  int32_t top_k;
  float top_p;
  int32_t no_repeat_ngram_size; /* > 0: NoRepeatNGramLogitsProcessor on the device (generator_base.py:77-85;
                              * transformers logits_process.py _calc_banned_ngram_tokens) over
                              * prompt + output + drafts; 0 = off                              */
  uint64_t seed;             /* counter-based RNG seed for the sampling path                 */
} lsk_generation;

/* What one speculation round produced — everything
 * SelfSpeculativeGenerationStrategy.single_step_speculation returns or streams
 * (self_speculation_generator.py:102-229): the draft ids (for SpeculativeTextStreamer, :158-161),
 * number_of_matches (:185-199), the tokens appended to output_ids (:203-205). */
typedef struct {
  int32_t n_drafted;                     /* D_actual (EOS can end the draft loop early)       */
  int32_t n_matches;
  int32_t n_emitted;                     /* n_matches + 1                                     */
  int32_t kv_len;                        /* committed context after the round                 */
  int32_t draft_ids[LSK_MAX_SPEC + 1];
  int32_t emitted_ids[LSK_MAX_SPEC + 1]; /* draft[:n] + [verified[n]]                         */
  int32_t verified_ids[LSK_MAX_SPEC + 1];
} lsk_round_out;

typedef struct lsk_engine lsk_engine;

int lsk_abi_version(void);
const char* lsk_last_error(void);

/* Engine lifetime.  Allocates packed-weight storage, the paged KV pool, scratch and streams on
 * the CURRENT CUDA device.  Replaces model placement in generate.py:54-67. */
int lsk_create(const lsk_config* cfg, lsk_engine** out);
void lsk_destroy(lsk_engine* e);

/* Tensor-parallel wiring (configs with tp_size > 1): rank 0 calls lsk_comm_unique_id, the host
 * side broadcasts the 128 bytes, every rank calls lsk_comm_init.  The reference has no
 * equivalent (generate.py:50-52 exits on non-zero ranks). */
int lsk_comm_unique_id(uint8_t id_out[128]);
int lsk_comm_init(lsk_engine* e, const uint8_t id[128]);

/* Weight ingest: HF tensors -> packed / sharded HBM layout.  Synchronous. */
int lsk_load_weights(lsk_engine* e, const lsk_weight_desc* descs, int32_t n);
/* 1 when every tensor the architecture needs has been loaded. */
int lsk_weights_complete(const lsk_engine* e);

/* Start a generation: reset lengths, store E / eos / sampling.  Replaces the state reset at
 * self_speculation_generator.py:41-50. */
int lsk_begin(lsk_engine* e, const lsk_generation* gen);

/* Prompt ingestion from HOST memory (ids[n], n >= 1).  Runs ids[0..n-2] through all layers (the
 * work the reference does inside its first forward_early + forward_remainder,
 * llama_model_utils.py:251-261, 363-383) so that afterwards every round has the steady-state
 * shape: one pending input token (ids[n-1]) and kv_len == n-1 in every layer. */
int lsk_prefill(lsk_engine* e, const int32_t* ids, int32_t n);

/* One draft / verify / accept / commit round with d_req speculations
 * (self_speculation_generator.py:102-229; the caller applies the max_steps clamp of :63-66).
 * d_req == 0 is the reference's tail round.  Blocks until the round's result is on the host. */
int lsk_round(lsk_engine* e, int32_t d_req, lsk_round_out* out);

/* A round that stops drafting when the early-exit head is unsure (Hugging Face assisted
 * generation's assistant_confidence_threshold).  The confidence of draft i is the probability of
 * the token it chose under the distribution it chose from: softmax(logits)[arg-max] at temperature
 * 1 when greedy, the warped draft row's probability of the drawn token when sampling (both after
 * the n-gram ban, if any).  n_drafted = 1 + the first i whose draft is an EOS or has confidence
 * < min_confidence, else d_max; the stopping draft is kept.  The draft steps after it do not run
 * (graph mode; LSK_FLAG_NO_GRAPH runs them and ignores their results).
 * The result, and the state left behind, are bit-identical to lsk_round(e, n_drafted, out) from
 * the same state; min_confidence == 0 gives lsk_round(e, d_max, out).
 * draft_conf_out (host, may be NULL, LSK_MAX_SPEC entries) receives confidences 0 .. n_drafted-1.
 * Same preconditions and errors as lsk_round with d_max for d_req; also LSK_ERR_INVALID for
 * min_confidence outside [0, 1] or NaN, and for tp_size > 1. */
int lsk_round_adaptive(lsk_engine* e, int32_t d_max, float min_confidence, lsk_round_out* out,
                       float* draft_conf_out);

/* Batched generation: n_seqs prompts share every weight pass of a round.  The batch shares
 * the KV pool: sequence s owns a slot of P = n_pages / n_seqs whole 64-token pages, logical pages
 * [s*P, (s+1)*P), and its position p is logical position s*64*P + p (LSK_DBG_KROW / LSK_DBG_VROW
 * read it there).  Every active sequence's round and the state it leaves are bit-identical to
 * lsk_round(e, d_seq[s]) run on that sequence alone (lsk_begin + lsk_prefill of its prompt, then the
 * same earlier rounds; with sampling, lsk_begin with seed = seeds[s]).  After lsk_begin with
 * no_repeat_ngram_size == 0, tp_size == 1 and 1 <= exit_layer <= n_layers; n_seqs in [1, max_rows].
 * With sample == 1 the batch must be prefilled by lsk_prefill_batch_seeded (lsk_prefill_batch then
 * returns LSK_ERR_INVALID).
 *
 * lsk_prefill_batch: prompt j is ids[offsets[j] .. offsets[j+1]-1] (offsets[0] == 0), length >= 1;
 * each is prefilled into its own slot exactly as lsk_prefill would prefill it alone (same routes,
 * same bits).  slot_positions_out (may be NULL): positions per slot, 64 * P.  LSK_ERR_CTX when a
 * prompt + 1 does not fit its slot.  Ends any single-sequence generation: lsk_round,
 * lsk_round_adaptive and lsk_ar_step return LSK_ERR_STATE until the next lsk_prefill.
 *
 * lsk_round_batch: one round for every sequence, n_seqs * (d_req + 1) <= max_rows.  d_seq (may be NULL:
 * all d_req) holds each sequence's draft count in [0, d_req]; active (may be NULL: all active) flags
 * the sequences that commit.  An inactive sequence commits nothing: outs[s] has n_drafted = n_matches
 * = n_emitted = 0 and kv_len unchanged (its rows still run, writing K/V only inside its own slot above
 * its committed length).  LSK_ERR_CTX when some sequence, active or not, has kv_len + d_req + 2 above
 * its slot's positions; LSK_ERR_STATE after any lsk_prefill or scoring call since the batch's
 * prefill.  outs: n_seqs records.
 *
 * lsk_prefill_batch_seeded: lsk_prefill_batch with one Philox seed per sequence (seeds: n_seqs
 * values).  Sequence s draws, accepts and resamples exactly as a solo generation begun with seed =
 * seeds[s], at its own step count, so a (prompt, seed) pair gives the same tokens whatever it is
 * batched with.  A greedy generation ignores the seeds, as lsk_begin's seed. */
int lsk_prefill_batch(lsk_engine* e, const int32_t* ids, const int32_t* offsets, int32_t n_seqs,
                      int32_t* slot_positions_out);
int lsk_prefill_batch_seeded(lsk_engine* e, const int32_t* ids, const int32_t* offsets, int32_t n_seqs,
                             const uint64_t* seeds, int32_t* slot_positions_out);
int lsk_round_batch(lsk_engine* e, int32_t d_req, const int32_t* d_seq, const int32_t* active,
                    lsk_round_out* outs);

/* lsk_round_batch with confidence-threshold drafting (lsk_round_adaptive's stop rule) for every
 * sequence: d_max takes d_req's place, and sequence s stops drafting after draft j when that draft is
 * an EOS, when its confidence is below min_confidence (one threshold for the whole batch), or when
 * j + 1 == d_seq[s].  Draft step j >= 1 runs (graph mode) iff some active sequence has not stopped
 * before it; a sequence that stopped still has its rows computed while others draft on, causally
 * invisible to its kept rows.  Every active sequence's round, confidences and committed K/V rows are
 * bit-identical to lsk_round_adaptive(e, d_seq[s], min_confidence) of that sequence alone (and so to
 * lsk_round(e, n_drafted)); an inactive one behaves as in lsk_round_batch.  min_confidence == 0 gives
 * lsk_round_batch(e, d_max, d_seq, active); d_max == 0 is lsk_round_batch(e, 0, ...).
 * LSK_FLAG_NO_GRAPH runs every draft step, with the same results.
 * draft_conf_out (host, may be NULL): [n_seqs][LSK_MAX_SPEC] floats; sequence s receives the
 * confidences of its outs[s].n_drafted kept drafts.
 * Same preconditions, state rules and errors as lsk_round_batch; also LSK_ERR_INVALID for
 * min_confidence outside [0, 1] or NaN. */
int lsk_round_batch_adaptive(lsk_engine* e, int32_t d_max, const int32_t* d_seq, const int32_t* active,
                             float min_confidence, lsk_round_out* outs, float* draft_conf_out);

/* One autoregressive step on the same engine (autoregressive_generator.py:44-67): all layers, or
 * layers < E when the generation's exit_layer > 0.  Returns the chosen token; the caller decides
 * about EOS exactly as the reference does (:66-67). */
int lsk_ar_step(lsk_engine* e, int32_t* token_out);

/* Teacher-forced scoring of ids[0..n-1] (2 <= n <= max_ctx), single GPU (tp_size == 1).
 * For i in 0 .. n-2:
 *   logprob_out[i] = log softmax(logits after ids[0..i])[ids[i+1]]   (fp32)
 *   greedy_out[i]  = arg-max token of that row, lowest id on ties    (may be NULL)
 * exit_layer E in [1, n_layers] runs layers [0, E) and then the final norm and LM head, as the
 * draft does (forward_early, llama_model_utils.py:271-273); E <= 0 means all layers (forward,
 * :155-209).  Host pointers.  Synchronous; lsk_last_device_ms gives its device time.  It reuses the
 * KV pool, so it ends any generation in progress: lsk_round / lsk_ar_step / lsk_debug_forward_rows
 * return LSK_ERR_STATE until the next lsk_prefill.  It needs neither lsk_begin nor
 * LSK_FLAG_KEEP_LOGITS; with that flag, LSK_DBG_LOGITS afterwards holds the last LM-head slice. */
int lsk_score(lsk_engine* e, const int32_t* ids, int32_t n, int32_t exit_layer,
              float* logprob_out, int32_t* greedy_out);

/* Teacher-forced scoring of n_seqs sequences in one call, single GPU, wgmma prompt pass required.
 * Sequence j is ids[offsets[j] .. offsets[j+1]-1], 2 <= length <= max_ctx, offsets[0] == 0.  Outputs
 * are concatenated in input order: sequence j's (length_j - 1) entries start at offsets[j] - j and
 * mean exactly what lsk_score's do.  greedy_out may be NULL.  Same state rules as lsk_score.
 * The rows of all sequences are packed into shared 128-token prompt-pass chunks; every entry is
 * bit-identical to lsk_score of that sequence alone on the wgmma route (sequences of more than
 * max_rows + 1 ids). */
int lsk_score_batch(lsk_engine* e, const int32_t* ids, const int32_t* offsets, int32_t n_seqs,
                    int32_t exit_layer, float* logprob_out, int32_t* greedy_out);

/* Teacher-forced scoring of continuations that share contexts, single GPU, wgmma prompt pass
 * required.  Prefix p is prefix_ids[prefix_offsets[p] .. prefix_offsets[p+1]-1] and branch b is
 * branch_ids[branch_offsets[b] .. branch_offsets[b+1]-1], each at least 1 id (both offset arrays
 * start at 0 and increase); branch b continues prefix branch_prefix[b] and scores P + B, with
 * len(P) + len(B) <= max_ctx.  Every prefix has at least one branch; branches come in any order.
 * Outputs have one entry per branch id, concatenated in input order (branch b owns
 * [branch_offsets[b], branch_offsets[b+1])): entry i of branch b is the log-probability of B[i]
 * after P + B[:i], and greedy_out (may be NULL) the arg-max token there.  These are bit-identical
 * to entries len(P)-1 .. len(P)+len(B)-2 of lsk_score_batch of P + B.  A prefix's rows run once
 * per group, writing K/V only; its own ids are not scored.  Same state rules as lsk_score. */
int lsk_score_prefixed(lsk_engine* e, const int32_t* prefix_ids, const int32_t* prefix_offsets,
                       int32_t n_prefixes, const int32_t* branch_ids, const int32_t* branch_offsets,
                       const int32_t* branch_prefix, int32_t n_branches, int32_t exit_layer,
                       float* logprob_out, int32_t* greedy_out);

/* Teacher-forced scoring of ids[0..n-1] at n_exits exit layers in ONE pass, single GPU.  exits is
 * strictly increasing, each in [1, n_layers], 1 <= n_exits <= LSK_MAX_EXITS.  Layers below each
 * exit run once: the heads of the earlier exits run inside the pass of the deepest one.
 *   logprob_out[j][i], greedy_out[j][i]  ([n_exits][n-1]; greedy may be NULL) are bit-identical to
 *                                         lsk_score(ids, n, exits[j]) entry i
 *   accept_out[j][i]  ([n_exits-1][n-1], may be NULL) = sum_v min(p_E(v), p_L(v)) for the row
 *                     predicting ids[i+1]: p_E, p_L the warped (temperature, top-k, top-p)
 *                     distributions at exit exits[j] and at full depth, i.e. the probability that
 *                     the accept test of sampled self-speculation (self_speculation_generator.py:
 *                     191-199) accepts a draft drawn at that exit.  It needs sampling->sample == 1,
 *                     temperature > 0, no_repeat_ngram_size == 0 (the ban is not modelled) and
 *                     exits[n_exits-1] == n_layers.  Only temperature, top_k and top_p are read.
 * sampling may be NULL when accept_out is.  Same state rules as lsk_score. */
#define LSK_MAX_EXITS 32
int lsk_score_exits(lsk_engine* e, const int32_t* ids, int32_t n, const int32_t* exits, int32_t n_exits,
                    const lsk_generation* sampling, float* logprob_out, int32_t* greedy_out,
                    float* accept_out);

/* Queries / debugging (parity tests). */
int lsk_kv_len(const lsk_engine* e, int32_t* len_out);
/* Teacher-forced block: the m given ids as one block at positions kv_len .. kv_len+m-1 through
 * every layer and the LM head — `forward` (llama_model_utils.py:155-209) on top of the committed
 * context; logits of the m rows are then readable through LSK_DBG_LOGITS (needs
 * LSK_FLAG_KEEP_LOGITS).  Nothing is committed. */
int lsk_debug_forward_rows(lsk_engine* e, const int32_t* ids_host, int32_t m);
typedef enum {
  LSK_DBG_HIDDEN = 0,        /* fp32 [16, hidden] residual-stream rows of the last launch     */
  LSK_DBG_LOGITS = 1,        /* fp32 [16, vocab_local] (needs LSK_FLAG_KEEP_LOGITS)           */
  LSK_DBG_KROW = 2,          /* bf16->fp32 K cache rows [count][head_dim], n_floats = count*head_dim: layer, index = kv_head*max_ctx + pos0; positions pos0 .. pos0+count-1 (<= max_ctx) */
  LSK_DBG_VROW = 3,
  LSK_DBG_PROBS_DRAFT = 4,   /* fp32 [16, vocab] warped (T, top-k, top-p) draft distributions     */
  LSK_DBG_PROBS_VERIFY = 5,  /* fp32 [16, vocab] warped verifier distributions of the last round */
  LSK_DBG_RESIDUAL = 6,      /* fp32 [vocab] max(p_verify - p_draft, 0) of the last rejected draft (unnormalised; self_speculation_generator.py:27-29 max_fn before its division) */
  LSK_DBG_ARGMAX = 7         /* fp32 [rows][2] (logit, token id) the engine picks greedily per row of the last LM head, n_floats = 2*rows (<= 32): its candidates merged as the accept kernels merge them */
} lsk_debug_what;
int lsk_debug_read(lsk_engine* e, int32_t what, int32_t layer, int64_t index,
                   float* dst_host, int64_t n_floats);
/* Replace the (identity) logical->physical KV page map with a permutation: proves the paged
 * indirection.  Only valid before lsk_prefill. */
int lsk_debug_set_page_table(lsk_engine* e, const int32_t* pages, int32_t n_pages);

/* Bytes of HBM the engine streams for one (d, ctx) round / AR step — the algorithmic-bytes
 * model of SURVEY.md §8(d), per GPU (tensor-parallel shards included). */
int lsk_round_bytes(const lsk_engine* e, int32_t d, int32_t ctx, double* bytes_out);
int lsk_ar_bytes(const lsk_engine* e, int32_t ctx, double* bytes_out);
/* Kernels launched (or replayed through graphs) since lsk_create; device time of the last
 * lsk_round / lsk_ar_step / lsk_prefill measured with CUDA events on the engine's stream. */
int lsk_launch_count(const lsk_engine* e, int64_t* count_out);
int lsk_last_device_ms(const lsk_engine* e, float* ms_out);

/* Same work as lsk_round, launched eagerly with a CUDA-event pair around every kernel so the
 * device time can be attributed per kernel class: 0 qkv, 1 attention, 2 o-proj, 3 gate/up,
 * 4 down, 5 lm-head, 6 small kernels, 7 collectives.  class_ms / class_launches have 8 entries.
 * Measurement aid for bench.py's roofline section; the numbers include launch gaps that graph
 * replay + programmatic dependent launch hide in lsk_round. */
int lsk_profile_round(lsk_engine* e, int32_t d_req, lsk_round_out* out, float* class_ms,
                      int64_t* class_launches, float* total_ms);

/* Host-side launch schedule of one weight-streaming GEMM (pure host logic; works without a GPU):
 * how many activation columns are resident at a time, tiles accumulated side by side, TMA ring
 * depth, grid.  pro: 0 RMSNorm prologue, 1 bf16 copy; epi: 0 qkv/rope, 1 residual add, 2 store,
 * 3 silu*up, 4 lm-head arg-max. */
typedef struct {
  int32_t ok, nt, tiles_per_pass, n_chunks, chunk_cols, ring_stages, stage_bytes, grid, block;
  int32_t n_tiles;
  int64_t smem_bytes, smem_limit;
} lsk_gemm_plan;
int lsk_plan_gemm(int64_t n_rows, int64_t k, int32_t m, int32_t pro, int32_t epi, int32_t sm_count,
                  lsk_gemm_plan* out);

/* Host-side launch plan of the attention kernel (pure host logic): split-KV factor (an engine
 * constant: results are batch-invariant only for a fixed partition), K/V ring depth, grid, shared
 * memory incl. the one-CTA-per-SM floor, 16-row blocks per CTA.  n_heads / n_kv_heads_local are the
 * tensor-parallel shard's head counts with the same GQA ratio as the model.  ok = 0 when `m` rows
 * do not fit, and for every `m` when the layout cannot run at all: a 16-token launch of its
 * (head_dim, n_heads / n_kv_heads_local) does not fit shared memory (lsk_create refuses it). */
typedef struct {
  int32_t ok, n_splits, ring_stages, grid, block, row_blocks, kv_refetched_per_row_block;
  int64_t smem_bytes, smem_limit;
} lsk_attn_plan;
int lsk_plan_attention(int32_t head_dim, int32_t n_heads, int32_t n_kv_heads_local, int32_t m,
                       int32_t sm_count, lsk_attn_plan* out);

/* Device memory of one engine (one rank), in bytes per category: the packed layer weights (both
 * layouts), the embedding and final norm, the LM head (both layouts), the paged KV pool, and
 * everything else; total is their sum. */
typedef struct {
  int64_t weights, embed, lm_head, kv_pool, scratch, total;
} lsk_memory_plan;
/* What an engine is asked to do beyond what lsk_create allocates (a zeroed struct: nothing). */
typedef struct {
  int32_t lm_head_tc;        /* the opt-in wgmma LM head was asked for (LSK_LMHEAD_TC=1)          */
  int32_t sampling;          /* lsk_begin with sample = 1                                         */
  int32_t ngram_ban;         /* lsk_begin with no_repeat_ngram_size > 0                           */
  int32_t adaptive;          /* lsk_round_adaptive (lsk_round_batch_adaptive with batch_seqs)     */
  int32_t score_exits;       /* scoring with up to this many exits (lsk_score: 1), <= LSK_MAX_EXITS */
  int32_t accept_exits;      /* lsk_score_exits with accept_out, up to this many exits            */
  int32_t packed_scoring;    /* lsk_score_batch or lsk_score_prefixed                             */
  int32_t tp_peer;           /* tp_size > 1: lsk_comm_init's peer region of the one-shot collectives */
  int32_t batch_seqs;        /* lsk_prefill_batch with up to this many sequences, <= 16 (any count
                              * allocates the same buffers; with `sampling`, also the seeds; with
                              * `adaptive`, also lsk_round_batch_adaptive's confidence scratch)   */
} lsk_memory_uses;
/* Host-side plan of the device memory an engine with config `cfg` on a GPU with `sm_count` SMs
 * allocates at lsk_create plus for `uses` (pure host logic; works without a GPU).  The flags it
 * reads from cfg are the ones lsk_create reads; it refuses the configs lsk_create refuses, with the
 * same codes and messages. */
int lsk_plan_memory(const lsk_config* cfg, int32_t sm_count, const lsk_memory_uses* uses,
                    lsk_memory_plan* out);
/* The device memory the engine holds now, per category. */
int lsk_memory_in_use(const lsk_engine* e, lsk_memory_plan* out);

/* Stand-alone kernel entry points used by the micro-benchmarks and unit tests: run the skinny
 * GEMM (y[m, n] = x[m, k] . W[n, k]^T, fp32 out) on packed weights / the split-KV attention on
 * caller-provided device buffers. */
int lsk_test_pack(const void* w_bf16_dev, int64_t n, int64_t k, void* packed_out_dev);
int lsk_test_gemm(const void* packed_dev, int64_t n, int64_t k, const void* x_bf16_dev,
                  int32_t m, float* y_dev, int32_t iters, float* avg_ms_out);
/* Paged split-KV attention alone: m query rows at positions ctx-m .. ctx-1 attend causally to keys
 * 0 .. ctx-1 (modeling_llama.py:187-221 eager attention).  q / out: [m][n_heads*head_dim] bf16,
 * k / v: natural [n_kv_heads][ctx][head_dim] bf16 (k already rotated) — the entry point builds the
 * engine's paged, swizzled pool from them; page_perm_host (nullable) permutes logical->physical
 * pages.  m <= 16 runs one decode block; 16 < m <= 128 runs the prompt pass's launches for one
 * chunk at position ctx-m (canonical output, returned unpacked in the same [m][n_heads*head_dim]
 * layout).  All other pointers are device pointers. */
int lsk_test_attn(const void* q_dev, const void* k_dev, const void* v_dev, int32_t n_heads,
                  int32_t n_kv_heads, int32_t head_dim, int32_t ctx, int32_t m, int32_t n_splits,
                  const int32_t* page_perm_host, void* out_dev, int32_t iters, float* avg_ms_out);
/* The same attention over several sequences in one launch, as a batched round (lsk_round_batch)
 * launches it: sequence s has seq_rows query rows (q / out rows s * seq_rows ..) at positions
 * ctx_host[s] - seq_rows .. ctx_host[s] - 1, and its keys k / v natural
 * [n_seqs][n_kv_heads][slot_positions][head_dim] bf16 fill logical pages [s * P, (s + 1) * P) of one
 * pool, P = slot_positions / 64; page_perm_host (nullable) permutes all n_seqs * P pages.  Refuses
 * n_seqs * seq_rows > 16, ctx_host[s] outside [seq_rows, slot_positions], a slot that is not a
 * multiple of 64 and n_splits outside [1, 8]. */
int lsk_test_attn_seqs(const void* q_dev, const void* k_dev, const void* v_dev, int32_t n_heads,
                       int32_t n_kv_heads, int32_t head_dim, int32_t n_seqs, int32_t seq_rows,
                       const int32_t* ctx_host, int32_t slot_positions, int32_t n_splits,
                       const int32_t* page_perm_host, void* out_dev);
/* wgmma LM head (csrc/lmhead_tc.cuh, opt-in): logits[m, n] = rmsnorm(x)[m, :] . W[n, :] with
 * W natural bf16 [n, k], x fp32 [m, k], norm_w bf16 [k]; writes fp32 logits [m, n] and per row the
 * arg-max (lowest index wins).  All pointers are device pointers. */
int lsk_test_lmhead_tc(const void* w_bf16_dev, int64_t n, int64_t k, const float* x_f32_dev,
                       const void* norm_w_bf16_dev, float eps, int32_t m, float* logits_dev,
                       float* best_val_dev, int32_t* best_idx_dev, int32_t iters, float* avg_ms_out);
/* The scoring kernel alone (csrc/misc_kernels.cuh: logprob_rows_kernel) on device buffers: logits
 * [rows][ld] fp32 with only the first `vocab` columns of each row valid, targets [rows]; writes
 * logprob [rows] and the per-row arg-max greedy [rows] (nullable). */
int lsk_test_logprob(const float* logits_dev, int32_t rows, int32_t vocab, int32_t ld,
                     const int32_t* targets_dev, float* logprob_dev, int32_t* greedy_dev);
/* The acceptance kernels alone (csrc/sampling.cuh: warp_rows_kernel, accept_prob_kernel) on device
 * buffers: draft and full-depth logits [rows][ld] fp32, the first `vocab` columns valid; writes
 * accept_dev[r] = sum_v min of the two rows' warped distributions (temperature, top_k, top_p of
 * `sampling`, temperature > 0). */
int lsk_test_accept(const float* logits_draft_dev, const float* logits_verify_dev, int32_t rows,
                    int32_t vocab, int32_t ld, const lsk_generation* sampling, float* accept_dev);
/* The sampling kernels alone (csrc/sampling.cuh).  `_dev` pointers are device pointers, the others
 * host pointers.  Of `sampling` the draw reads temperature (> 0), top_k, top_p and seed, the accept
 * test seed, n_eos and eos_ids.  The random number of a draw is Philox4x32-10 at counter (step
 * count, row, purpose, 0x4c534b) under key (seed low, seed high): u = (first word >> 8) * 2^-24;
 * purposes: 1 draft draw, 2 verifier draw, 3 accept test, 4 residual draw.
 *
 * lsk_test_draw: the inverse-CDF draw (block_sample_index) over weights_dev[vocab] (fp32, >= 0, any
 * total), once per u_dev[i] in [0, 1): picks_dev[i] = the token whose interval of the running sum
 * holds u * total; 0 for an all-zero row. */
int lsk_test_draw(const float* weights_dev, int32_t vocab, const float* u_dev, int32_t n, int32_t* picks_dev);
/* lsk_test_sample: warp_and_sample_kernel, the kernel generation draws with, on logits_dev [rows][ld]
 * (the first `vocab` columns valid), n_steps times with step counts step0 .. step0 + n_steps - 1:
 * row r draws at counter row row_base + r.  probs_dev [rows][vocab] receives the warped rows (of the
 * first step; they do not depend on the step), tokens_dev [n_steps][rows] the drawn tokens. */
int lsk_test_sample(const float* logits_dev, int32_t rows, int32_t vocab, int32_t ld,
                    const lsk_generation* sampling, int32_t step0, int32_t n_steps, int32_t purpose,
                    int32_t row_base, float* probs_dev, int32_t* tokens_dev);
/* lsk_test_accept_sample: accept_sample_kernel (rejection test, residual resample, commit) on warped
 * rows p_draft_dev [d][vocab] and p_verify_dev [d + 1][vocab], 1 <= d <= LSK_MAX_SPEC, n_steps times.
 * Step s starts from a fresh state (committed length kv_len0, step count step0 + s) holding the draft
 * tokens draft_ids [s][d] and the verifier's draws verified_ids [s][d + 1], and fills out[s];
 * residual_dev [vocab] is the kernel's residual scratch, left as the last rejecting step wrote it. */
int lsk_test_accept_sample(const float* p_draft_dev, const float* p_verify_dev, int32_t vocab, int32_t d,
                           const int32_t* draft_ids, const int32_t* verified_ids,
                           const lsk_generation* sampling, int32_t kv_len0, int32_t step0, int32_t n_steps,
                           lsk_round_out* out, float* residual_dev);

#ifdef __cplusplus
}
#endif
#endif /* LSK_H_ */
