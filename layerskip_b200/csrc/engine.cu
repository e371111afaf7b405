// engine.cu — liblsk: C ABI (include/lsk.h) + host-side orchestration of the sm_90a kernels.
//
// The engine owns: packed weights, the paged KV pool, scratch activations, the device-resident
// generation state, one stream and a cache of CUDA graphs (one per (E, d_req) round shape).
// A speculation round is ONE graph replay and ONE host synchronisation.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <nccl.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <atomic>
#include <functional>
#include <map>
#include <string>
#include <vector>

#include "../../include/lsk.h"
#include "attention.cuh"
#include "common.cuh"
#include "gemm_skinny.cuh"
#include "tp_peer.cuh"
#include "lmhead_tc.cuh"
#include "prefill_tc.cuh"
#include "misc_kernels.cuh"
#include "sampling.cuh"

using namespace lsk;

// ---------------------------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------------------------
static thread_local std::string g_last_error;

static int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return code;
}

#define CU(expr)                                                                         \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess)                                                               \
      return fail(LSK_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),  \
                  __FILE__, __LINE__);                                                   \
  } while (0)

#define NC(expr)                                                                         \
  do {                                                                                   \
    ncclResult_t _r = (expr);                                                            \
    if (_r != ncclSuccess)                                                               \
      return fail(LSK_ERR_NCCL, "%s failed: %s (%s:%d)", #expr, ncclGetErrorString(_r),  \
                  __FILE__, __LINE__);                                                   \
  } while (0)

#define TRY(expr)            \
  do {                       \
    int _s = (expr);         \
    if (_s != LSK_OK) return _s; \
  } while (0)

// ---------------------------------------------------------------------------------------------
// device memory
// ---------------------------------------------------------------------------------------------
// The categories of lsk_memory_plan, in its field order.
enum MemCat { MEM_WEIGHTS = 0, MEM_EMBED, MEM_LM_HEAD, MEM_KV_POOL, MEM_SCRATCH, MEM_CATS };
struct MemBuf {
  size_t bytes;
  MemCat cat;
};

// Owner of device allocations: every pointer it hands out is recorded with its size and category
// until it is freed, and whatever it still holds is freed when it is destroyed.
class DeviceMem {
 public:
  cudaStream_t stream = nullptr;       // zero fills are enqueued here
  DeviceMem() = default;
  DeviceMem(const DeviceMem&) = delete;
  DeviceMem& operator=(const DeviceMem&) = delete;
  ~DeviceMem() { release(); }

  // b.bytes at *p, zero-filled on `stream` when `zero`.  On failure *p is null.
  template <typename T>
  int alloc(T** p, const MemBuf& b, bool zero = false) {
    const cudaError_t er = cudaMalloc((void**)p, b.bytes);
    if (er != cudaSuccess) {
      *p = nullptr;
      cudaGetLastError();
      return fail(LSK_ERR_NOMEM, "cudaMalloc of %zu bytes failed: %s", b.bytes, cudaGetErrorString(er));
    }
    held_.push_back({(void*)*p, b});
    if (zero) CU(cudaMemsetAsync(*p, 0, b.bytes, stream));
    return LSK_OK;
  }
  void free(void* p) {
    for (size_t i = 0; i < held_.size(); ++i)
      if (held_[i].p == p) {
        cudaFree(p);
        held_.erase(held_.begin() + i);
        return;
      }
  }
  void release() {
    for (const Held& h : held_) cudaFree(h.p);
    held_.clear();
  }
  void bytes_held(int64_t* cat) const {
    for (const Held& h : held_) cat[h.b.cat] += (int64_t)h.b.bytes;
  }

 private:
  struct Held {
    void* p;
    MemBuf b;
  };
  std::vector<Held> held_;
};

// ---------------------------------------------------------------------------------------------
// engine
// ---------------------------------------------------------------------------------------------
struct LayerWeights {
  __nv_bfloat16* wqkv = nullptr;  // packed [(q_rows + 2 kv_rows), hidden]
  __nv_bfloat16* wo = nullptr;    // packed [hidden, q_rows]
  __nv_bfloat16* wgu = nullptr;   // packed [2 * inter_l, hidden]  (gate/up interleaved by 8)
  __nv_bfloat16* wd = nullptr;    // packed [hidden, inter_l]
  __nv_bfloat16* ln1 = nullptr;
  __nv_bfloat16* ln2 = nullptr;
  // tensor-core prefill (prefill_tc.cuh): second copy in the canonical K-major tile layout
  unsigned char* wqkv_c = nullptr;
  unsigned char* wo_c = nullptr;
  unsigned char* wgu_c = nullptr;
  unsigned char* wd_c = nullptr;
  unsigned loaded = 0;            // bit per role
};

struct GemmPlan {
  int n_tiles = 0, nsb = 0, K = 0;
};

// What an engine derives from its config, the SM count and which of its two optional paths it
// takes: host arithmetic only (engine_shape), so lsk_plan_memory needs no device.
struct EngineShape {
  // local (tensor-parallel shard) dimensions
  int heads_l = 0, kv_heads_l = 0, q_rows = 0, kv_rows = 0, inter_l = 0, vocab_l = 0,
      vocab_l_pad = 0, vocab_off = 0, group = 0, inter_l_pad = 0;
  int n_pages = 0, max_pos = 0, n_splits = 0;
  size_t pool_layer_elems = 0;
  // opt-in wgmma LM head (lmhead_tc.cuh): a second, canonical-layout copy of the head weights
  bool lm_tc = false;
  int lm_tc_tiles = 0, lm_tc_grid = 0, lm_tc_stages = 0;
  int lm_cand = 0;                     // candidates produced by the wgmma LM head (its grid)
  // tensor-core prefill: 128-token passes (on unless LSK_FLAG_NO_PREFILL_TC / LSK_PREFILL_TC=0)
  bool pf_tc = false;
  int pf_stages = 0;
  int kst_h = 0, kst_q = 0, kst_i = 0;          // 64-wide k stages of hidden / q_rows / inter_l
  int pf_t_qkv = 0, pf_t_h = 0, pf_t_gu = 0;     // 128-row tiles of qkv / hidden / gate-up outputs
};

// Every device buffer an engine can hold, with its size and category (mem_table): create_into, the
// buffers allocated on first use and lsk_plan_memory all read their sizes from here.
struct AttnBufs {
  MemBuf part, arrive;                 // attention split partials, per-kv-head arrival counters
};
struct MemTable {
  // at create, per layer; the canonical copies (*_c) with the prompt pass
  MemBuf wqkv, wo, wgu, wd, norm, wqkv_c, wo_c, wgu_c, wd_c;
  // at create with the prompt pass: [128][hidden] fp32 rows (hidden_p, tp_buf_p), O / down partials,
  // q rows and the canonical activations
  MemBuf rows_p, part_p, q_p, xn_c, attn_c, act_c;
  MemBuf embed, final_norm, lm_head, lm_head_tc;   // lm_head_tc with the wgmma LM head
  MemBuf kv_pool;                                   // each of kpool, vpool
  MemBuf page_table, rope, hidden, qbuf, act, tp_buf;   // qbuf: also attn_out
  AttnBufs attn;
  MemBuf cand, gath, row_best, d_zero, d_prompt, state, gen_dev;   // cand / gath / row_best: each of val, idx
  // on first use
  MemBuf logits;          // at create with LSK_FLAG_KEEP_LOGITS; sampling, the n-gram ban, adaptive rounds, scoring
  MemBuf vocab_rows;      // [16][vocab] fp32: probs_d, probs_v, logits_full (TP), exits_pv
  MemBuf samp_scratch, logits_gath, conf_scratch;
  MemBuf score_rows;      // per exit, each of score_lp, score_greedy
  MemBuf accept_rows, draft_rows;                   // per draft exit: exits_accept, exits_pd
  MemBuf batch_buf, view_table, piece_arrive;       // packed scoring
  MemBuf batch_state, batch_ctl, batch_arrive;      // batched rounds
  MemBuf batch_seeds;                               // batched sampled rounds
  MemBuf conf_seqs;                                 // batched adaptive rounds
  MemBuf peer_region;                               // lsk_comm_init with the one-shot collectives
};

struct lsk_engine : EngineShape {
  lsk_config cfg{};
  int sm_count = 0;
  int max_rows = kMaxRows;             // token rows one step can carry (8 when 16 do not fit)
  bool use_pdl = true, use_graph = true, keep_logits = false;
  bool pdl_break = false;              // launch the next kernel without the PDL attribute (graph conditional boundary)
  bool adaptive = false;               // enqueueing an adaptive round: draft heads materialise their logits

  std::vector<LayerWeights> layers;
  __nv_bfloat16* embed = nullptr;      // [vocab, hidden] natural (replicated)
  __nv_bfloat16* final_norm = nullptr;
  __nv_bfloat16* lm_head = nullptr;    // packed [vocab_l_pad, hidden]
  unsigned char* lm_head_tc = nullptr;   // wgmma LM head: [lm_tc_tiles][hidden / 64][16 KiB]
  unsigned globals_loaded = 0;
  float* hidden_p = nullptr;             // [128][hidden] fp32 residual rows of a prompt chunk
  float* tp_buf_p = nullptr;             // [128][hidden] fp32 row-parallel partial sums (TP)
  float* part_p = nullptr;               // [4 k-splits][128][hidden] fp32 partial tiles of the O / down GEMMs
  __nv_bfloat16* q_p = nullptr;          // [128][q_rows]
  unsigned char* xn_c = nullptr;         // canonical activations: RMS-normed rows   [kst_h][16 KiB]
  unsigned char* attn_c = nullptr;       //                        attention output   [kst_q][16 KiB]
  unsigned char* act_c = nullptr;        //                        silu(gate) * up    [kst_i][16 KiB]

  __nv_bfloat16* kpool = nullptr;      // [layer][page][kv_head][64][128]
  __nv_bfloat16* vpool = nullptr;
  int* page_table = nullptr;
  std::vector<int> page_table_host;    // host copy of page_table (prefix-shared scoring builds its views from it)
  float2* rope = nullptr;

  float* hidden = nullptr;             // [16][hidden] fp32 residual-stream rows
  __nv_bfloat16* qbuf = nullptr;       // [16][q_rows]
  __nv_bfloat16* attn_out = nullptr;   // [16][q_rows]
  float* attn_part = nullptr;          // attention: published split partials (AttnArgs::part)
  size_t attn_part_cap = 0;            // floats
  unsigned int* attn_arrive = nullptr; // attention: per-kv-head arrival counters (AttnArgs::arrive)
  __nv_bfloat16* act = nullptr;        // [16][inter_l]
  float* tp_buf = nullptr;             // [16][hidden] row-parallel partial sums (TP)
  float* logits = nullptr;             // [16][vocab_l_pad] (optional)
  float* logits_gath = nullptr;        // TP sampling: [tp][16][vocab_l_pad] all-gathered shards
  float* logits_full = nullptr;        // TP sampling: [16][vocab] rows every rank samples from
  float* probs_d = nullptr;            // sampling: [16][vocab] warped draft distributions
  float* probs_v = nullptr;            // sampling: [16][vocab] warped verifier distributions
  float* samp_scratch = nullptr;       // sampling: [vocab] residual weights
  float* cand_val = nullptr;           // [n_cand_max][16]
  int* cand_idx = nullptr;
  float* gath_val = nullptr;           // TP: [tp_size][16]
  int* gath_idx = nullptr;
  float* ban_val = nullptr;            // n-gram ban: [16] arg-max of the banned logits rows (n_cand == 1 layout)
  int* ban_idx = nullptr;
  float* rank_val = nullptr;           // TP: [16]
  int* rank_idx = nullptr;
  int* d_zero = nullptr;
  int* d_prompt = nullptr;             // [max_ctx] prompt ids
  // scoring (allocated on first use; the result arrays grow with the number of exits)
  int score_cap = 0;                   // exits the result arrays hold
  float* score_lp = nullptr;           // [score_cap][max_pos] log-probabilities (packed scoring: row 0)
  int* score_greedy = nullptr;         // [score_cap][max_pos] arg-max ids
  int* batch_buf = nullptr;            // packed scoring: [8][max_pos] row ids, targets, row maps, pieces of a group
  unsigned int* piece_arrive = nullptr;  // packed scoring: [128 pieces][kv heads] attention arrival counters
  int* view_table = nullptr;           // packed scoring: [max_pos] physical pages of a group's page-table views
  int accept_cap = 0;                  // draft exits the acceptance buffers hold
  float* exits_accept = nullptr;       // [accept_cap][max_pos] acceptance probabilities
  float* exits_pd = nullptr;           // [accept_cap][128 or 16 rows][vocab] warped draft rows of the current chunk
  float* exits_pv = nullptr;           // [16][vocab] warped full-depth rows of the current slice
  DevState* state = nullptr;
  GenParams* gen_dev = nullptr;
  RoundResult* res_host = nullptr;     // mapped pinned
  RoundResult* res_dev = nullptr;      // device alias of res_host
  // batched rounds (lsk_prefill_batch / lsk_round_batch; allocated on first use)
  int batch_n = 0;                     // sequences of the batch in progress; 0: none
  std::vector<int> batch_len;          // host mirror of each sequence's committed length
  DevState* bstate = nullptr;          // [kMaxRows] per-sequence generation state
  int* batch_ctl = nullptr;            // [2][kMaxRows] the round's d_seq, then its active flags
  unsigned int* batch_arrive = nullptr;  // [kMaxRows][kv heads] attention arrival counters
  bool batch_seeded = false;           // the batch was prefilled with one Philox seed per sequence
  unsigned long long* batch_seeds = nullptr;  // [kMaxRows] those seeds (sampled batches; first use)
  RoundResult* bres_host = nullptr;    // [kMaxRows] mapped pinned
  RoundResult* bres_dev = nullptr;     // device alias of bres_host

  GemmPlan p_qkv, p_o, p_gu, p_d, p_lm;
  const float* cur_cand_val = nullptr;  // candidates of the last enqueued LM head (epilogue's, or the banned rows' arg-max)
  const int* cur_cand_idx = nullptr;
  int cur_n_cand = 0;

  cudaStream_t stream = nullptr;
  cudaStream_t body_stream = nullptr;  // captures the bodies of an adaptive round's conditional nodes
  ConfScratch* conf_scratch = nullptr; // draft_confidence_kernel's partials and arrival counter
  ConfSeqsScratch* conf_seqs = nullptr;  // draft_confidence_seqs_kernel's partials, counters, d_stop, threshold
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  std::map<long long, cudaGraphExec_t> graphs;
  ncclComm_t comm = nullptr;
  // one-shot collectives over peer-mapped HBM (tp_peer.cuh); opt-in, NCCL otherwise
  bool want_peer = false, peer_ok = false;
  unsigned ablate = 0;                   // LSK_ABLATE: timing-only diagnostics, kernel classes NOT launched
  int peer_mode = 1;                     // 1: push kernel after the GEMM; 2: push fused into the GEMM epilogue
  PeerComm peer{};
  void* peer_region = nullptr;           // this rank's peer-visible allocation
  void* peer_opened[kMaxPeers] = {};     // IPC mappings of the other ranks' regions
  int* peer_err_host = nullptr;          // mapped pinned: set by a kernel whose wait timed out

  lsk_generation gen{};
  bool began = false, prefilled = false;
  int host_len = 0;                    // host mirror of the committed KV length
  int64_t launches = 0;
  int64_t capture_launches = 0;        // launches recorded while capturing the current graph
  std::map<long long, int64_t> graph_launches;
  float last_ms = 0.f;
  // per-kernel-class timing (lsk_profile_round): events around every launch, eager mode
  bool profiling = false;
  int cur_class = 0;
  std::vector<std::pair<int, std::pair<cudaEvent_t, cudaEvent_t>>> prof_events;

  MemTable sizes;                      // set by create_into
  DeviceMem mem;                       // every device buffer above

  lsk_engine() = default;
  lsk_engine(const lsk_engine&) = delete;
  lsk_engine& operator=(const lsk_engine&) = delete;
  // lsk_destroy; also releases the temporary engines of the stand-alone test entry points on every
  // return path.  Fields that were never set are skipped.
  ~lsk_engine() {
    if (stream) cudaStreamSynchronize(stream);
    for (auto& kv : graphs) cudaGraphExecDestroy(kv.second);
    for (void* p : peer_opened) if (p) cudaIpcCloseMemHandle(p);
    if (comm) ncclCommDestroy(comm);
    mem.release();
    if (peer_err_host) cudaFreeHost(peer_err_host);
    if (res_host) cudaFreeHost(res_host);
    if (bres_host) cudaFreeHost(bres_host);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (stream) cudaStreamDestroy(stream);
    if (body_stream) cudaStreamDestroy(body_stream);
    cudaGetLastError();   // a half-built engine may have left a sticky-free error behind
  }
};

enum { CLS_QKV = 0, CLS_ATTN = 1, CLS_O = 2, CLS_GATEUP = 3, CLS_DOWN = 4, CLS_LMHEAD = 5, CLS_MISC = 6, CLS_COMM = 7, CLS_COUNT = 8 };

static constexpr int kSmemMax = 227 * 1024;

// ---------------------------------------------------------------------------------------------
// launch helpers
// ---------------------------------------------------------------------------------------------
// One piece of work enqueued on the engine's stream: counted as one launch and, when profiling,
// timed by an event pair under kernel class `cls`.  Every kernel goes through it by way of
// launch(); the NCCL all-reduces call it directly.
template <typename F>
static auto stream_op(lsk_engine* e, int cls, F enqueue) -> decltype(enqueue()) {
  e->launches += 1;
  e->capture_launches += 1;
  if (!e->profiling) return enqueue();
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  cudaEventRecord(a, e->stream);
  auto err = enqueue();
  cudaEventRecord(b, e->stream);
  e->prof_events.push_back({cls, {a, b}});
  return err;
}

// Kernel launch: programmatic dependent launch attribute on every kernel, class = e->cur_class.
// A programmatic edge cannot cross into or out of a graph conditional body: the first kernel of a
// body and the first kernel after one are launched without it (e->pdl_break).
template <typename... KArgs, typename... Args>
static cudaError_t launch(lsk_engine* e, void (*kern)(KArgs...), dim3 grid, dim3 block,
                          size_t smem, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = e->stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = (e->use_pdl && !e->pdl_break) ? 1 : 0;
  e->pdl_break = false;
  return stream_op(e, e->cur_class, [&]() { return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...); });
}

// Opt kernel `Kern` in to kSmemMax of dynamic shared memory, once per device (the attribute is per
// DEVICE: one process may drive engines on several GPUs).  Done lazily at the launch site: the
// stand-alone test entry points launch through an engine that lsk_create never set up.
template <auto Kern>
static cudaError_t allow_max_smem() {
  static std::atomic<uint64_t> configured{0};
  int dev = 0;
  cudaError_t err = cudaGetDevice(&dev);
  if (err != cudaSuccess) return err;
  const uint64_t bit = 1ull << (dev & 63);
  if (configured.load(std::memory_order_relaxed) & bit) return cudaSuccess;
  err = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax);
  if (err == cudaSuccess) configured.fetch_or(bit, std::memory_order_relaxed);
  return err;
}

// ---------------------------------------------------------------------------------------------
// GEMM planning / dispatch
// ---------------------------------------------------------------------------------------------
static GemmPlan make_plan(int n_rows, int K) {
  GemmPlan p;
  p.n_tiles = n_rows / 16;
  p.K = K;
  p.nsb = K / 32;
  return p;
}

// Per-launch schedule: how much of K is resident (activation chunk), how many tiles are
// accumulated side by side, and how deep the TMA ring can be in the remaining shared memory.
struct GemmSched {
  int tpp = 1, n_chunks = 1, kc_sbs = 0, n_stages = 0, grid = 0;
  size_t smem = 0;
  bool ok = false;
};
static GemmSched plan_sched(int NT, int M, int pro, int epi, const GemmPlan& p, int sm_count) {
  GemmSched best;
  for (int want = 1; want <= 16; ++want) {
    // RMSNorm prologue: whole rows resident whenever that fits; otherwise (16-row blocks at hidden
    // > 4096) the statistics are computed up front and the rows are normalised chunk by chunk
    if (pro == PRO_RMS && want == 2 && best.ok) break;   // whole rows fit: keep the resident mode
    int kc = (p.nsb + want - 1) / want;
    if (want > 1) kc = (kc + kStageSbs - 1) / kStageSbs * kStageSbs;
    const int n_chunks = (p.nsb + kc - 1) / kc;
    const int tpp = n_chunks > 1 ? kMaxTilesPerPass : 1;
    const GemmScratch L = gemm_scratch_layout(NT, M, kc * 32, tpp, epi);
    for (int st = kMaxStages; st >= 2; --st) {
      if (gemm_smem_total(st, L.total) <= (size_t)kSmemMax) {
        if (!best.ok || st > best.n_stages) {
          best.ok = true; best.tpp = tpp; best.n_chunks = n_chunks; best.kc_sbs = kc;
          best.n_stages = st; best.smem = gemm_smem_total(st, L.total);
        }
        break;
      }
    }
    if (best.ok && best.n_stages >= 5) break;   // >= 80 KiB in flight per SM
  }
  if (best.ok) {
    const int n_slots = (p.n_tiles + best.tpp - 1) / best.tpp;
    best.grid = n_slots < sm_count ? n_slots : sm_count;
    // Tile quantisation: with g CTAs the kernel lasts ceil(n_slots / g) slot-times.  Among the
    // CTA counts that reach the minimum number of waves, take the SMALLEST one that wastes the
    // fewest slots (e.g. 768 tiles: 128 CTAs x 6 instead of 132 CTAs of which 108 run a 6th tile
    // alone) — the TMA ring lets ~85 % of the SMs saturate HBM.
    if (n_slots > sm_count) {
      const int waves = (n_slots + sm_count - 1) / sm_count;
      int g = (n_slots + waves - 1) / waves;          // smallest CTA count with that many waves
      const int lo = sm_count * 4 / 5;
      if (g < lo) g = lo;
      best.grid = g;
    }
  }
  return best;
}

static void apply_sched(GemmArgs& a, const GemmPlan& p, const GemmSched& sc) {
  a.n_tiles = p.n_tiles;
  a.nsb = p.nsb;
  a.K = p.K;
  a.tiles_per_pass = sc.tpp;
  a.n_chunks = sc.n_chunks;
  a.kc_sbs = sc.kc_sbs;
  a.n_stages = sc.n_stages;
  a.xs_rows = a.M;
}

template <int NT, int PRO, int EPI>
static int launch_gemm_t(lsk_engine* e, const GemmPlan& p, GemmArgs& a) {
  const GemmSched sc = plan_sched(NT, a.M, PRO, EPI, p, e->sm_count);
  if (!sc.ok)
    return fail(LSK_ERR_INVALID, "skinny GEMM does not fit shared memory (K=%d, NT=%d)", p.K, NT);
  apply_sched(a, p, sc);
  CU((allow_max_smem<gemm_skinny_kernel<NT, PRO, EPI>>()));
  CU(launch(e, gemm_skinny_kernel<NT, PRO, EPI>, dim3(sc.grid), dim3(kGemmThreads), sc.smem, a));
  return LSK_OK;
}

template <int PRO, int EPI>
static int launch_gemm(lsk_engine* e, const GemmPlan& p, GemmArgs a) {
  const int NT = a.M <= 8 ? 1 : 2;
  if (NT == 1) return launch_gemm_t<1, PRO, EPI>(e, p, a);
  if (plan_sched(2, a.M, PRO, EPI, p, e->sm_count).ok) return launch_gemm_t<2, PRO, EPI>(e, p, a);
  return fail(LSK_ERR_INVALID, "%d token rows need the 16-row kernel, which does not fit next to K=%d "
              "(hidden sizes > 4096 support at most 8 rows, i.e. num_speculations <= 7)", a.M, p.K);
}

// Tensor parallel: x[0..M) += sum over ranks of tp_buf (the fp32 partial of a row-parallel GEMM).
// Peer mode 1 (default, tp_peer.cuh): ONE kernel pushes the partial to every peer over NVLink as
// LL lines (flag inside the data), polls theirs and adds the rank-ordered sum to the residual.
// Peer mode 3: the fence + flag protocol (A/B).  Without peer access: NCCL all-reduce + residual add,
// timed by its own event pair so that `comm` never reads 0.
static int ll_grid(int n2, int sm_count) {
  int g = (n2 + kArThreads - 1) / kArThreads;
  return g < 1 ? 1 : (g > sm_count ? sm_count : g);      // every CTA resident at once (spin-wait safety)
}
static int emit_allreduce_resid_nccl(lsk_engine* e, float* buf, float* x, int M) {
  const lsk_config& c = e->cfg;
  NC(stream_op(e, CLS_COMM, [&]() {
    return ncclAllReduce(buf, buf, (size_t)M * c.hidden, ncclFloat, ncclSum, e->comm, e->stream);
  }));
  e->cur_class = CLS_MISC;
  CU(launch(e, residual_add_kernel, dim3(8, M), dim3(256), 0, x, c.hidden, (const float*)buf, c.hidden, c.hidden));
  return LSK_OK;
}
static int emit_allreduce_resid(lsk_engine* e, float* x, int M) {
  const lsk_config& c = e->cfg;
  if (e->peer_ok && e->peer_mode == 3) {
    e->cur_class = CLS_COMM;
    const int n4 = M * c.hidden / 4;
    const int grid = (n4 + kArVecPerCta - 1) / kArVecPerCta;      // <= kMaxArCtas (hidden <= 8192)
    CU(launch(e, tp_allreduce_resid_kernel, dim3(grid), dim3(kArThreads), 0, e->peer,
              (const float*)e->tp_buf, x, n4));
    return LSK_OK;
  }
  if (e->peer_ok) {
    e->cur_class = CLS_COMM;
    const int n2 = M * c.hidden / 2;
    CU(launch(e, tp_allreduce_ll_kernel, dim3(ll_grid(n2, e->sm_count)), dim3(kArThreads), 0, e->peer,
              (const float*)e->tp_buf, x, n2));
    return LSK_OK;
  }
  return emit_allreduce_resid_nccl(e, e->tp_buf, x, M);
}

// Fused variant (peer_mode 2): the row-parallel GEMM pushes its tiles to every rank from its
// epilogue as LL lines while it is still streaming weights (gemm_skinny_push_kernel); a small
// kernel polls the lines of all ranks and adds the rank-ordered sum to the residual rows.
static int emit_gemm_push_resid(lsk_engine* e, const GemmPlan& p, GemmArgs a, float* x) {
  const lsk_config& c = e->cfg;
  const int NT = a.M <= 8 ? 1 : 2;
  const GemmSched sc = plan_sched(NT, a.M, PRO_BF16, EPI_PUSH, p, e->sm_count);
  if (!sc.ok) return fail(LSK_ERR_INVALID, "skinny GEMM does not fit shared memory (K=%d, NT=%d)", p.K, NT);
  apply_sched(a, p, sc);
  if (NT == 1) {
    CU(allow_max_smem<gemm_skinny_push_kernel<1>>());
    CU(launch(e, gemm_skinny_push_kernel<1>, dim3(sc.grid), dim3(kGemmThreads), sc.smem, a, e->peer));
  } else {
    CU(allow_max_smem<gemm_skinny_push_kernel<2>>());
    CU(launch(e, gemm_skinny_push_kernel<2>, dim3(sc.grid), dim3(kGemmThreads), sc.smem, a, e->peer));
  }
  e->cur_class = CLS_COMM;
  const int n2 = a.M * c.hidden / 2;
  CU(launch(e, tp_finish_ll_kernel, dim3(ll_grid(n2, e->sm_count)), dim3(kArThreads), 0, e->peer, x, n2));
  return LSK_OK;
}

// Host-side launch plan of the attention kernel (pure host logic; lsk_plan_attention exposes it):
// split count = engine constant (batch invariance), ring depth as deep as shared memory allows, and a
// shared-memory floor that gives a one-wave grid a whole SM per CTA.
static int attn_default_splits(int sm_count, int kv_heads_local) {
  return std::max(1, std::min(4, sm_count / std::max(1, kv_heads_local)));
}
struct AttnLaunchPlan {
  AttnSmemPlan sp;
  int stages;
  size_t smem;
  bool ok;
};
static AttnLaunchPlan plan_attention_launch(int head_dim, int group, int M, int kv_heads_local, int n_splits,
                                            int want_stages, int sm_count) {
  AttnLaunchPlan p;
  int st = want_stages;
  while (st > 2 && attn_smem_plan(head_dim, group, M, st).total > (size_t)kSmemMax) --st;
  p.sp = attn_smem_plan(head_dim, group, M, st);
  p.stages = st;
  p.ok = p.sp.total <= (size_t)kSmemMax;
  p.smem = p.sp.total;
  if (kv_heads_local * n_splits <= sm_count && p.smem < (size_t)116 * 1024) p.smem = (size_t)116 * 1024;
  return p;
}
// Shared memory of the smallest launch a (head_dim, group) layout must run: the prompt pass launches
// at least 16 tokens at a time (prompt_attn_rows) and a verify block carries up to kMaxRows = 16, both
// at the 2-stage ring.  A layout above kSmemMax is refused by lsk_create.
static size_t attn_layout_smem(int head_dim, int group) { return attn_smem_plan(head_dim, group, 16, 2).total; }

// Attention over the paged cache: grid (kv heads, splits), the last split of a head to finish
// merges; head_dim selects the instantiation, the shared-memory plan depends on (group, M).
// pz: the piece grid (kv heads, splits, pieces) of attn_piece_kernel, with a.M the largest piece's rows.
template <int HD>
static int launch_attention_t(lsk_engine* e, AttnArgs& a, const AttnPieces* pz, int n_pieces) {
  const int grid_z = pz ? n_pieces : 1;
  const AttnLaunchPlan lp = plan_attention_launch(HD, a.group, a.M, a.n_kv_heads * grid_z, a.n_splits, kAttnMaxStages,
                                                  e->sm_count);
  const AttnSmemPlan& sp = lp.sp;
  a.n_stages = lp.stages;
  if (!lp.ok)
    return fail(LSK_ERR_INVALID, "attention: %d query rows per kv head do not fit shared memory", a.group * a.M);
  a.rows_pad = (a.group * a.M + 15) / 16 * 16;
  a.merge_off = sp.merge_off; a.part_off = sp.part_off; a.reload_per_rb = sp.reload_per_rb;
  if (attn_part_floats(a.n_kv_heads, a.n_splits, pz ? pz->part_rows : a.rows_pad, HD) > e->attn_part_cap)
    return fail(LSK_ERR_INVALID, "attention: %d query rows per kv head exceed the partials buffer", a.group * a.M);
  // counters per (piece, kv head): packed scoring's pieces, or a batched round's sequences
  a.part = e->attn_part; a.arrive = pz ? (pz->pieces ? e->piece_arrive : e->batch_arrive) : e->attn_arrive;
  // lp.smem: a grid that fits one wave gets a whole SM per CTA (> half of the SM's shared memory):
  // the CTAs then spread over the SMs instead of sharing a few SMs' load bandwidth
  const dim3 grid(a.n_kv_heads, a.n_splits, grid_z);
  if (pz) {
    CU(allow_max_smem<attn_piece_kernel<HD>>());
    CU(launch(e, attn_piece_kernel<HD>, grid, dim3(kAttnThreads), lp.smem, a, *pz));
  } else {
    CU(allow_max_smem<attn_split_kernel<HD>>());
    CU(launch(e, attn_split_kernel<HD>, grid, dim3(kAttnThreads), lp.smem, a));
  }
  return LSK_OK;
}
static int launch_attention(lsk_engine* e, AttnArgs& a, int head_dim, const AttnPieces* pz = nullptr, int n_pieces = 0) {
  switch (head_dim) {
    case 128: return launch_attention_t<128>(e, a, pz, n_pieces);
    case 64: return launch_attention_t<64>(e, a, pz, n_pieces);
    case 32: return launch_attention_t<32>(e, a, pz, n_pieces);
    default: return fail(LSK_ERR_INVALID, "head_dim %d unsupported (32, 64 or 128)", head_dim);
  }
}

// Split partials + arrival counters of the attention kernel, sized for `rows` query tokens per
// launch (the engine's: the prompt pass's 128) at `n_splits`.
static AttnBufs attn_bufs(int kv_heads, int group, int head_dim, int n_splits, int rows) {
  return {{attn_part_floats(kv_heads, n_splits, (group * rows + 15) / 16 * 16, head_dim) * 4, MEM_SCRATCH},
          {(size_t)kv_heads * 4, MEM_SCRATCH}};
}
// The counters start at zero.
static int alloc_attn_partials(lsk_engine* e, const AttnBufs& b) {
  TRY(e->mem.alloc(&e->attn_part, b.part));
  e->attn_part_cap = b.part.bytes / 4;
  return e->mem.alloc(&e->attn_arrive, b.arrive, true);
}

// Rows of several sequences in one launch (batched rounds, single GPU): n_seqs sequences of seq_rows
// rows each, sequence s's rows first at hidden row row0 + s * x_ld / hidden, its committed length at
// base_len[s * len_stride] and its page-table view at page_table + s * seq_pages.  The activations
// between the GEMMs (q, attention output, act) stay contiguous.
struct SeqRows {
  int n_seqs, seq_rows, len_stride, seq_pages, x_ld;
};

// ---------------------------------------------------------------------------------------------
// one decoder layer on hidden rows [row0, row0 + M) at positions *base_len + pos_off + i
//   (HF LlamaDecoderLayer as called at llama_model_utils.py:193-201,253-261,354-362,375-383)
// With `sr` the M rows are sr->n_seqs sequences' (SeqRows), x_ld floats apart.
// ---------------------------------------------------------------------------------------------
static int enqueue_layer(lsk_engine* e, int li, int row0, int M, const int* base_len, int pos_off,
                         const SeqRows* sr = nullptr) {
  const lsk_config& c = e->cfg;
  LayerWeights& L = e->layers[li];
  float* x = e->hidden + (size_t)row0 * c.hidden;
  const int x_ld = sr ? sr->x_ld : c.hidden;
  __nv_bfloat16* kp = e->kpool + (size_t)li * e->pool_layer_elems;
  __nv_bfloat16* vp = e->vpool + (size_t)li * e->pool_layer_elems;
  const bool tp = c.tp_size > 1;

  if (!(e->ablate & (1u << CLS_QKV))) {  // RMSNorm -> QKV -> RoPE -> KV append
    e->cur_class = CLS_QKV;
    GemmArgs a{};
    a.W = reinterpret_cast<const uint4*>(L.wqkv);
    a.M = M;
    a.x_f32 = x; a.x_ld = x_ld; a.norm_w = L.ln1; a.eps = c.rms_eps;
    a.q_out = e->qbuf; a.q_ld = e->q_rows;
    a.kpool = kp; a.vpool = vp; a.page_table = e->page_table;
    a.base_len = base_len; a.pos_off = pos_off; a.rope = e->rope; a.head_dim = c.head_dim;
    a.q_rows = e->q_rows; a.kv_rows = e->kv_rows; a.n_kv_heads = e->kv_heads_l;
    if (sr) {
      a.seq_rows = sr->seq_rows; a.len_stride = sr->len_stride; a.seq_pages = sr->seq_pages;
      TRY((launch_gemm<PRO_RMS, EPI_QKV_SEQS>(e, e->p_qkv, a)));
    } else {
      TRY((launch_gemm<PRO_RMS, EPI_QKV>(e, e->p_qkv, a)));
    }
  }
  if (!(e->ablate & (1u << CLS_ATTN))) {  // attention over the paged cache
    e->cur_class = CLS_ATTN;
    AttnArgs a{};
    a.q = e->qbuf; a.q_ld = e->q_rows; a.out = e->attn_out; a.out_ld = e->q_rows;
    a.kpool = kp; a.vpool = vp; a.page_table = e->page_table;
    a.base_len = base_len; a.pos_off = pos_off; a.M = M; a.group = e->group;
    a.n_kv_heads = e->kv_heads_l; a.n_splits = e->n_splits;
    a.scale = 1.0f / sqrtf((float)c.head_dim);
    if (sr) {   // one piece per sequence (attn_piece_kernel's sequence grid)
      a.M = sr->seq_rows;
      const AttnPieces pz{nullptr, (e->group * M + 15) / 16 * 16, sr->seq_rows, sr->len_stride, sr->seq_pages};
      TRY(launch_attention(e, a, c.head_dim, &pz, sr->n_seqs));
    } else {
      TRY(launch_attention(e, a, c.head_dim));
    }
  }
  if (!(e->ablate & (1u << CLS_O))) {  // O projection (+ residual, or all-reduce then residual under TP)
    e->cur_class = CLS_O;
    GemmArgs a{};
    a.W = reinterpret_cast<const uint4*>(L.wo);
    a.M = M;
    a.x_bf16 = e->attn_out; a.xb_ld = e->q_rows;
    if (!tp) {
      a.out_f32 = x; a.out_ld = x_ld;
      TRY((launch_gemm<PRO_BF16, EPI_RESID>(e, e->p_o, a)));
    } else if (e->peer_ok && e->peer_mode == 2) {
      TRY(emit_gemm_push_resid(e, e->p_o, a, x));
    } else {
      a.out_f32 = e->tp_buf; a.out_ld = c.hidden;
      TRY((launch_gemm<PRO_BF16, EPI_STORE>(e, e->p_o, a)));
      TRY(emit_allreduce_resid(e, x, M));
    }
  }
  if (!(e->ablate & (1u << CLS_GATEUP))) {  // RMSNorm -> gate/up -> SiLU * up
    e->cur_class = CLS_GATEUP;
    GemmArgs a{};
    a.W = reinterpret_cast<const uint4*>(L.wgu);
    a.M = M;
    a.x_f32 = x; a.x_ld = x_ld; a.norm_w = L.ln2; a.eps = c.rms_eps;
    a.act = e->act; a.act_ld = e->inter_l_pad;
    TRY((launch_gemm<PRO_RMS, EPI_SILU>(e, e->p_gu, a)));
  }
  if (!(e->ablate & (1u << CLS_DOWN))) {  // down projection (+ residual)
    e->cur_class = CLS_DOWN;
    GemmArgs a{};
    a.W = reinterpret_cast<const uint4*>(L.wd);
    a.M = M;
    a.x_bf16 = e->act; a.xb_ld = e->inter_l_pad;
    if (!tp) {
      a.out_f32 = x; a.out_ld = x_ld;
      TRY((launch_gemm<PRO_BF16, EPI_RESID>(e, e->p_d, a)));
    } else if (e->peer_ok && e->peer_mode == 2) {
      TRY(emit_gemm_push_resid(e, e->p_d, a, x));
    } else {
      a.out_f32 = e->tp_buf; a.out_ld = c.hidden;
      TRY((launch_gemm<PRO_BF16, EPI_STORE>(e, e->p_d, a)));
      TRY(emit_allreduce_resid(e, x, M));
    }
  }
  return LSK_OK;
}

// ---------------------------------------------------------------------------------------------
// prompt chunk of m <= 128 tokens at positions c0 .. c0+m-1 through every layer on the wgmma
// GEMMs (forward_early + forward_remainder of llama_model_utils.py:213-276 / 363-383 on s = T_p)
// ---------------------------------------------------------------------------------------------
template <int EPI>
static int launch_prefill_gemm(lsk_engine* e, PrefillGemmArgs& a) {
  a.n_stages = e->pf_stages;
  const int items = a.n_tiles * (EPI == PF_EPI_STORE && a.k_splits > 1 ? a.k_splits : 1);
  const int grid = items < e->sm_count ? items : e->sm_count;
  CU(launch(e, prefill_gemm_tc_kernel<EPI>, dim3(grid), dim3(kTcThreads), prefill_tc_smem_bytes(a.n_stages), a));
  return LSK_OK;
}

// Prompt-pass attention of m <= 128 token rows at positions c0 .. c0+m-1 (q: [m][q_ld]) over the keys
// 0 .. c0+m-1 of the paged cache.  The base length is the device zero `zero`, the positions come from
// pos_off, and the output goes to the canonical operand `out_canon` (rows = token index in the chunk)
// that the O projection of prefill_tc.cuh reads.  One launch per m_attn rows: as many as fit the
// attention kernel's shared-memory plan (a multiple of 16, so the canonical swizzle of row r0 + j
// equals that of row j).
static int prompt_attn_rows(int head_dim, int group) {
  for (int cand = kPfTokens; cand >= 16; cand -= 16)
    if (attn_smem_plan(head_dim, group, cand, 2).total <= (size_t)kSmemMax) return cand;
  return 16;
}
static int launch_prompt_attention(lsk_engine* e, const __nv_bfloat16* q, int q_ld, unsigned char* out_canon,
                                   const __nv_bfloat16* kp, const __nv_bfloat16* vp, const int* page_table,
                                   const int* zero, int c0, int m, int group, int n_kv_heads, int head_dim) {
  const int m_attn = prompt_attn_rows(head_dim, group);
  for (int r0 = 0; r0 < m; r0 += m_attn) {
    AttnArgs a{};
    a.q = q + (size_t)r0 * q_ld; a.q_ld = q_ld;
    // operand rows are addressed by token index inside the 128-row stage: shift by r0 rows
    a.out = reinterpret_cast<__nv_bfloat16*>(out_canon + canon_offset(r0, 0)); a.out_canon = 1;
    a.kpool = kp; a.vpool = vp; a.page_table = page_table;
    a.base_len = zero; a.pos_off = c0 + r0; a.M = (m - r0) < m_attn ? (m - r0) : m_attn;
    a.group = group; a.n_kv_heads = n_kv_heads; a.n_splits = e->n_splits;
    a.scale = 1.0f / sqrtf((float)head_dim);
    TRY(launch_attention(e, a, head_dim));
  }
  return LSK_OK;
}

// A chunk of rows from several sequences (packed scoring), device pointers at the chunk's first row:
// ids, per-row (position, first page), and the chunk's attention pieces (AttnPieces::pieces).  The
// first pages index page_table, the group's table of page-table views.
struct PackedChunk {
  const int* ids;
  const int2* row_map;
  const int4* pieces;
  int n_pieces, max_piece_rows;
  const int* page_table;
};

// Scoring at several exits in one pass (lsk_score_exits): at the top of layer layers[t] the first
// norm kernel has folded the pending partials into hidden_p, exactly as the final fold of a pass
// that stops there does, so head(t) reads the residual rows after layers [0, layers[t]).
struct ChunkTaps {
  const int* layers;             // strictly increasing, each in [1, n_run)
  int n;
  std::function<int(int)> head;
};

// Layers [0, n_run) run on the chunk.  The prompt pass (complete = false) stops the last of them
// once its K/V rows are written; scoring (complete = true) runs it to the end and folds the pending
// row-parallel partials into hidden_p, which then holds the residual rows the LM head reads.
// With `pk` the rows are a packed chunk: ids, positions and pages come from it, and one piece-grid
// attention launch per layer covers every piece (c0 is then unused).  With `taps` the heads of the
// earlier exits run inside the pass.
static int enqueue_prefill_chunk(lsk_engine* e, int c0, int m, int n_run, bool complete,
                                 const PackedChunk* pk = nullptr, const ChunkTaps* taps = nullptr) {
  const lsk_config& c = e->cfg;
  const bool tp = c.tp_size > 1;
  e->cur_class = CLS_MISC;
  CU(launch(e, embed_tokens_kernel, dim3(m), dim3(256), 0, (const __nv_bfloat16*)e->embed, c.hidden,
            pk ? pk->ids : (const int*)(e->d_prompt + c0), e->hidden_p, c.hidden));
  // row-parallel GEMMs (O / down): hidden / 128 feature tiles are too few to keep the SMs streaming
  // -> split K; the partial tiles are summed (fixed order) by the next rms_canon_kernel
  const int ks_o = std::max(1, std::min(std::min(4, e->kst_q), e->sm_count / e->pf_t_h));
  const int ks_d = std::max(1, std::min(std::min(4, e->kst_i), e->sm_count / e->pf_t_h));
  const size_t part_stride = (size_t)kPfTokens * c.hidden;
  // pending row-parallel partials that the next norm kernel has to add to the residual rows
  const float* pend = nullptr;
  int n_pend = 0;
  auto after_row_parallel = [&](int n_splits) -> int {
    if (!tp) { pend = e->part_p; n_pend = n_splits; return LSK_OK; }
    e->cur_class = CLS_COMM;
    CU(launch(e, reduce_partials_kernel, dim3(m), dim3(256), 0, (const float*)e->part_p, n_splits, part_stride,
              c.hidden, c.hidden, e->tp_buf_p));
    NC(stream_op(e, CLS_COMM, [&]() {
      return ncclAllReduce(e->tp_buf_p, e->tp_buf_p, (size_t)m * c.hidden, ncclFloat, ncclSum, e->comm, e->stream);
    }));
    pend = e->tp_buf_p; n_pend = 1;
    return LSK_OK;
  };
  for (int li = 0, tap = 0; li < n_run; ++li) {
    LayerWeights& L = e->layers[li];
    __nv_bfloat16* kp = e->kpool + (size_t)li * e->pool_layer_elems;
    __nv_bfloat16* vp = e->vpool + (size_t)li * e->pool_layer_elems;
    e->cur_class = CLS_QKV;
    CU(launch(e, rms_canon_kernel, dim3(m), dim3(256), 0, e->hidden_p, c.hidden, pend, n_pend, part_stride,
              (const __nv_bfloat16*)L.ln1, c.rms_eps, c.hidden, e->xn_c));
    if (taps && tap < taps->n && taps->layers[tap] == li) TRY(taps->head(tap++));
    {
      PrefillGemmArgs a{};
      a.W = L.wqkv_c; a.X = e->xn_c; a.n_tiles = e->pf_t_qkv; a.n_rows = e->q_rows + 2 * e->kv_rows;
      a.n_kst = e->kst_h; a.M = m; a.k_splits = 1;
      a.q_out = e->q_p; a.q_ld = e->q_rows; a.kpool = kp; a.vpool = vp; a.page_table = e->page_table;
      a.pos0 = c0; a.rope = e->rope; a.head_dim = c.head_dim;
      a.q_rows = e->q_rows; a.kv_rows = e->kv_rows; a.n_kv_heads = e->kv_heads_l;
      if (pk) {
        a.row_map = pk->row_map;
        a.page_table = pk->page_table;
        TRY(launch_prefill_gemm<PF_EPI_QKV_MAP>(e, a));
      } else {
        TRY(launch_prefill_gemm<PF_EPI_QKV>(e, a));
      }
    }
    // the prompt pass has no LM head (the reference discards those logits): once the last layer's
    // K/V rows are written nothing downstream is needed
    if (li + 1 == n_run && !complete) break;
    e->cur_class = CLS_ATTN;
    if (pk) {
      AttnArgs a{};
      a.q = e->q_p; a.q_ld = e->q_rows;
      a.out = reinterpret_cast<__nv_bfloat16*>(e->attn_c); a.out_canon = 1;
      a.kpool = kp; a.vpool = vp; a.page_table = pk->page_table; a.base_len = e->d_zero;
      a.M = pk->max_piece_rows; a.group = e->group; a.n_kv_heads = e->kv_heads_l; a.n_splits = e->n_splits;
      a.scale = 1.0f / sqrtf((float)c.head_dim);
      const AttnPieces pz{pk->pieces, (e->group * kPfTokens + 15) / 16 * 16};
      TRY(launch_attention(e, a, c.head_dim, &pz, pk->n_pieces));
    } else {
      TRY(launch_prompt_attention(e, e->q_p, e->q_rows, e->attn_c, kp, vp, e->page_table, e->d_zero, c0, m,
                                  e->group, e->kv_heads_l, c.head_dim));
    }
    e->cur_class = CLS_O;
    {
      PrefillGemmArgs a{};
      a.W = L.wo_c; a.X = e->attn_c; a.n_tiles = e->pf_t_h; a.n_rows = c.hidden; a.n_kst = e->kst_q; a.M = m;
      a.k_splits = ks_o; a.out_f32 = e->part_p; a.out_ld = c.hidden;
      TRY(launch_prefill_gemm<PF_EPI_STORE>(e, a));
      TRY(after_row_parallel(ks_o));
    }
    e->cur_class = CLS_GATEUP;
    CU(launch(e, rms_canon_kernel, dim3(m), dim3(256), 0, e->hidden_p, c.hidden, pend, n_pend, part_stride,
              (const __nv_bfloat16*)L.ln2, c.rms_eps, c.hidden, e->xn_c));
    {
      PrefillGemmArgs a{};
      a.W = L.wgu_c; a.X = e->xn_c; a.n_tiles = e->pf_t_gu; a.n_rows = 2 * e->inter_l; a.n_kst = e->kst_h; a.M = m;
      a.k_splits = 1; a.act_canon = e->act_c;
      TRY(launch_prefill_gemm<PF_EPI_SILU>(e, a));
    }
    e->cur_class = CLS_DOWN;
    {
      PrefillGemmArgs a{};
      a.W = L.wd_c; a.X = e->act_c; a.n_tiles = e->pf_t_h; a.n_rows = c.hidden; a.n_kst = e->kst_i; a.M = m;
      a.k_splits = ks_d; a.out_f32 = e->part_p; a.out_ld = c.hidden;
      TRY(launch_prefill_gemm<PF_EPI_STORE>(e, a));
      TRY(after_row_parallel(ks_d));
    }
  }
  if (complete) {   // residual update only (dst = nullptr): the final norm is the LM head's prologue
    e->cur_class = CLS_MISC;
    CU(launch(e, rms_canon_kernel, dim3(m), dim3(256), 0, e->hidden_p, c.hidden, pend, n_pend, part_stride,
              (const __nv_bfloat16*)e->final_norm, c.rms_eps, c.hidden, (unsigned char*)nullptr));
  }
  return LSK_OK;
}

// ---------------------------------------------------------------------------------------------
// small stages
// ---------------------------------------------------------------------------------------------
static int emit_embed(lsk_engine* e, const int* ids, float* rows, int n_rows) {
  const lsk_config& c = e->cfg;
  e->cur_class = CLS_MISC;
  CU(launch(e, embed_tokens_kernel, dim3(n_rows), dim3(256), 0, (const __nv_bfloat16*)e->embed, c.hidden,
            ids, rows, c.hidden));
  return LSK_OK;
}
static const float* cand_val_ptr(lsk_engine* e);
static const int* cand_idx_ptr(lsk_engine* e);
// what the sampling kernels read: the local logits, or under TP the gathered [16][vocab] rows
static const float* samp_logits(lsk_engine* e) { return e->cfg.tp_size > 1 ? e->logits_full : e->logits; }
static int samp_ld(lsk_engine* e) { return e->cfg.tp_size > 1 ? e->cfg.vocab : e->vocab_l_pad; }
static int n_cand(lsk_engine* e);
static int emit_finalize(lsk_engine* e, int slot, float* dst_row) {
  const lsk_config& c = e->cfg;
  e->cur_class = CLS_MISC;
  CU(launch(e, finalize_embed_kernel, dim3(8), dim3(128), 0, cand_val_ptr(e), cand_idx_ptr(e), n_cand(e),
            e->state, slot, (const __nv_bfloat16*)e->embed, c.hidden, dst_row));
  return LSK_OK;
}
// token history (prompt ids + emitted tokens) is kept on the device only when the n-gram ban needs it
static int* hist_ptr(lsk_engine* e) { return e->gen.no_repeat_ngram_size > 0 ? e->d_prompt : nullptr; }
static int emit_accept(lsk_engine* e, int d_spec, const int* d_stop) {
  e->cur_class = CLS_MISC;
  CU(launch(e, accept_greedy_kernel, dim3(1), dim3(256), 0, cand_val_ptr(e), cand_idx_ptr(e), n_cand(e), d_spec,
            e->state, (const GenParams*)e->gen_dev, e->res_dev, 0, hist_ptr(e), d_stop));
  return LSK_OK;
}
static int emit_ar_commit(lsk_engine* e) {
  e->cur_class = CLS_MISC;
  CU(launch(e, ar_commit_kernel, dim3(1), dim3(32), 0, cand_val_ptr(e), cand_idx_ptr(e), n_cand(e), e->state,
            e->res_dev, 0, hist_ptr(e)));
  return LSK_OK;
}

// Final RMSNorm + the mma.sync LM head on M fp32 residual rows at x (row stride x_ld; 0: hidden): arg-max
// candidates into cand_*, and the logits rows when `logits` is set.
static int launch_lm_head_gemm(lsk_engine* e, const float* x, int M, float* logits, int x_ld = 0) {
  const lsk_config& c = e->cfg;
  GemmArgs a{};
  a.W = reinterpret_cast<const uint4*>(e->lm_head);
  a.M = M;
  a.x_f32 = x; a.x_ld = x_ld ? x_ld : c.hidden;
  a.norm_w = e->final_norm; a.eps = c.rms_eps;
  a.logits = logits; a.logits_ld = e->vocab_l_pad;
  a.n_valid_rows = e->vocab_l; a.vocab_off = e->vocab_off;
  a.part_val = e->cand_val; a.part_idx = e->cand_idx;
  return launch_gemm<PRO_RMS, EPI_LMHEAD>(e, e->p_lm, a);
}

// final RMSNorm + LM head on rows [row0, row0+M): arg-max candidates (and optional logits).
// (llama_model_utils.py:204-205, 271-273, 386-387).  Afterwards e->cand_* / n_cand() hold one
// (value, index) per candidate per row.
// With no_repeat_ngram_size > 0 (NoRepeatNGramLogitsProcessor, generator_base.py:77-85) the logits
// are materialised, the tokens that would repeat an n-gram of the sequence so far are set to -inf
// (row r continues prompt ++ output ++ draft[0 .. j0 + r)), and the arg-max is taken from the
// banned rows instead of the LM-head epilogue.  x_ld: row stride of the M rows (0: hidden).
static int enqueue_lm_head(lsk_engine* e, int row0, int M, int j0, int x_ld = 0) {
  const lsk_config& c = e->cfg;
  if (!x_ld) x_ld = c.hidden;
  const bool ban = e->gen.no_repeat_ngram_size > 0;
  e->cur_class = CLS_LMHEAD;
  const float* x = e->hidden + (size_t)row0 * c.hidden;
  float* logits = (e->keep_logits || e->gen.sample || ban || e->adaptive) ? e->logits : nullptr;
  if (e->lm_tc) {
    if (!(e->ablate & (1u << CLS_LMHEAD))) {
      LmHeadTcArgs t{};
      t.W = e->lm_head_tc; t.n_tiles = e->lm_tc_tiles; t.K = c.hidden; t.M = M; t.n_stages = e->lm_tc_stages;
      t.x_f32 = x; t.x_ld = x_ld; t.norm_w = e->final_norm; t.eps = c.rms_eps;
      t.logits = logits; t.logits_ld = e->vocab_l_pad; t.n_valid_rows = e->vocab_l; t.vocab_off = e->vocab_off;
      t.part_val = e->cand_val; t.part_idx = e->cand_idx;
      CU(launch(e, lmhead_tc_kernel, dim3(e->lm_tc_grid), dim3(kTcThreads),
                lmhead_tc_smem_bytes(c.hidden, e->lm_tc_stages), t));
    }
  } else if (!(e->ablate & (1u << CLS_LMHEAD))) TRY(launch_lm_head_gemm(e, x, M, logits, x_ld));
  e->cur_class = CLS_MISC;
  const float* cv = e->cand_val;
  const int* ci = e->cand_idx;
  // one candidate per CTA of the launch: the skinny GEMM's grid depends on M (plan_sched, exactly as
  // launch_gemm picks it) and may be smaller than min(tiles, SMs) — candidates past it are never
  // written and must not be merged (a stale (0, 0) would beat a row whose logits are all negative)
  int ncand = e->lm_tc ? e->lm_cand : plan_sched(M <= 8 ? 1 : 2, M, PRO_RMS, EPI_LMHEAD, e->p_lm, e->sm_count).grid;
  if (ban) {
    CU(launch(e, ngram_ban_kernel, dim3(M), dim3(256), 0, e->logits, e->vocab_l_pad, e->vocab_l, e->vocab_off,
              (const int*)e->d_prompt, (const DevState*)e->state, (int)e->gen.no_repeat_ngram_size, j0));
    if (!e->gen.sample) {
      CU(launch(e, argmax_rows_kernel, dim3(M), dim3(1024), 0, (const float*)e->logits, e->vocab_l_pad, e->vocab_l,
                e->vocab_off, e->ban_val, e->ban_idx));
      cv = e->ban_val; ci = e->ban_idx; ncand = 1;
    }
  }
  e->cur_cand_val = cv; e->cur_cand_idx = ci; e->cur_n_cand = ncand;
  if (c.tp_size > 1 && e->gen.sample) {
    // every rank needs the whole distribution: all-gather the vocab shards of the M rows, lay them
    // out as [M][vocab]; all ranks then run the same warp / Philox draw and stay in lockstep.
    // (The all-gathers of this function are not counted as launches, unlike the all-reduces.)
    e->cur_class = CLS_COMM;
    NC(ncclAllGather(e->logits, e->logits_gath, (size_t)M * e->vocab_l_pad, ncclFloat, e->comm, e->stream));
    CU(launch(e, tp_logits_rows_kernel, dim3(32, M), dim3(256), 0, (const float*)e->logits_gath, c.tp_size, M,
              e->vocab_l, e->vocab_l_pad, e->logits_full, c.vocab));
    e->cur_class = CLS_MISC;
  }
  if (c.tp_size > 1 && e->peer_ok) {
    CU(launch(e, tp_gather_best_kernel, dim3(1), dim3(256), 0, e->peer, cv, ci, ncand, M, e->gath_val, e->gath_idx));
  } else if (c.tp_size > 1) {
    CU(launch(e, rank_best_kernel, dim3(1), dim3(256), 0, cv, ci, ncand, M, e->rank_val, e->rank_idx));
    NC(ncclAllGather(e->rank_val, e->gath_val, kMaxRows, ncclFloat, e->comm, e->stream));
    NC(ncclAllGather(e->rank_idx, e->gath_idx, kMaxRows, ncclInt32, e->comm, e->stream));
  }
  return LSK_OK;
}
// candidates of the LAST enqueued LM head (what the following finalize / accept kernel consumes)
static const float* cand_val_ptr(lsk_engine* e) { return e->cfg.tp_size > 1 ? e->gath_val : e->cur_cand_val; }
static const int* cand_idx_ptr(lsk_engine* e) { return e->cfg.tp_size > 1 ? e->gath_idx : e->cur_cand_idx; }
static int n_cand(lsk_engine* e) { return e->cfg.tp_size > 1 ? e->cfg.tp_size : e->cur_n_cand; }

// ---------------------------------------------------------------------------------------------
// round / AR-step command streams
// ---------------------------------------------------------------------------------------------
// Draft step i after its layers: the shared head on row i; its token becomes tok[i+1] and is
// embedded into row i+1.
static int enqueue_draft_token(lsk_engine* e, int i) {
  const lsk_config& c = e->cfg;
  TRY(enqueue_lm_head(e, i, 1, i));
  e->cur_class = CLS_MISC;
  if (!e->gen.sample) {
    TRY(emit_finalize(e, 1 + i, e->hidden + (size_t)(i + 1) * c.hidden));
  } else {
    // decode_next_token sampling branch (llama_model_utils.py:123-131): keep the warped
    // distribution of draft i (needed by the rejection test), draw tok[i+1], embed it.
    CU(launch(e, warp_and_sample_kernel, dim3(1), dim3(kSampleThreads), 0, samp_logits(e),
              samp_ld(e), c.vocab, (const GenParams*)e->gen_dev, (const DevState*)e->state,
              e->probs_d + (size_t)i * c.vocab, &e->state->tok[1 + i], (int)RNG_DRAFT, i));
    CU(launch(e, embed_tokens_kernel, dim3(1), dim3(256), 0, (const __nv_bfloat16*)e->embed, c.hidden,
              (const int*)&e->state->tok[1 + i], e->hidden + (size_t)(i + 1) * c.hidden, c.hidden));
  }
  return LSK_OK;
}

// Verify after the draft rows: layers >= E see [exit rows of the draft steps ; the last draft's row]
// = rows 0..d (:363-383), then the head and the accept / commit.  d_stop: see accept_commit.
static int enqueue_verify(lsk_engine* e, int E, int d, const int* d_stop) {
  const lsk_config& c = e->cfg;
  const int* len = &e->state->len;
  for (int l = E; l < c.n_layers; ++l) TRY(enqueue_layer(e, l, 0, d + 1, len, 0));
  TRY(enqueue_lm_head(e, 0, d + 1, 0));
  e->cur_class = CLS_MISC;
  if (!e->gen.sample) {
    TRY(emit_accept(e, d, d_stop));
  } else {
    CU(launch(e, warp_and_sample_kernel, dim3(d + 1), dim3(kSampleThreads), 0, samp_logits(e),
              samp_ld(e), c.vocab, (const GenParams*)e->gen_dev, (const DevState*)e->state,
              e->probs_v, &e->state->verified[0], (int)RNG_VERIFY, 0));
    CU(launch(e, accept_sample_kernel, dim3(1), dim3(kSampleThreads), 0, (const float*)e->probs_d,
              (const float*)e->probs_v, c.vocab, d, e->state, (const GenParams*)e->gen_dev, e->res_dev,
              e->samp_scratch, 0, hist_ptr(e), d_stop));
  }
  return LSK_OK;
}

static int enqueue_round(lsk_engine* e, int E, int d) {
  const int* len = &e->state->len;
  // row 0 <- embedding of the pending token (self_speculation_generator.py:122, input_ids)
  TRY(emit_embed(e, &e->state->tok[0], e->hidden, 1));
  // draft loop (:127-148): step i runs layers [0,E) on row i at position len+i, then the shared
  // head; its arg-max becomes tok[i+1] and is embedded into row i+1.
  for (int i = 0; i < d; ++i) {
    for (int l = 0; l < E; ++l) TRY(enqueue_layer(e, l, i, 1, len, i));
    TRY(enqueue_draft_token(e, i));
  }
  // verify (:164-174 -> llama_model_utils.py:280-391): the last drafted token has not been
  // through layers < E yet (:350-362) ...
  for (int l = 0; l < E; ++l) TRY(enqueue_layer(e, l, d, 1, len, d));
  // ... then layers >= E on rows 0..d
  return enqueue_verify(e, E, d, nullptr);
}

// Confidence and stop rule of draft step j (draft_confidence_kernel).
static int emit_draft_confidence(lsk_engine* e, int j, int d, cudaGraphConditionalHandle next, bool has_next) {
  const lsk_config& c = e->cfg;
  e->cur_class = CLS_MISC;
  const int grid = std::min(kConfMaxCtas, (c.vocab + kConfCols - 1) / kConfCols);
  const float* logits = e->gen.sample ? nullptr : (const float*)e->logits;
  const float* probs = e->gen.sample ? (const float*)e->probs_d + (size_t)j * c.vocab : nullptr;
  CU(launch(e, draft_confidence_kernel, dim3(grid), dim3(kConfThreads), 0, logits, probs, c.vocab, e->state,
            (const GenParams*)e->gen_dev, e->conf_scratch, j, d, e->hidden, c.hidden, next, (int)has_next));
  return LSK_OK;
}

// `body` enqueued as the body of a graph IF node on `cond` while e->stream is being captured (the
// body is captured on e->body_stream), or launched directly in eager mode.
template <typename F>
static int enqueue_if(lsk_engine* e, cudaGraphConditionalHandle cond, F body) {
  if (!e->use_graph) return body();
  cudaStreamCaptureStatus cs;
  cudaGraph_t graph = nullptr;
  const cudaGraphNode_t* deps = nullptr;
  size_t n_deps = 0;
  CU(cudaStreamGetCaptureInfo(e->stream, &cs, nullptr, &graph, &deps, &n_deps));
  if (cs != cudaStreamCaptureStatusActive) return fail(LSK_ERR_CUDA, "adaptive round: stream is not capturing");
  cudaGraphNodeParams p = {};
  p.type = cudaGraphNodeTypeConditional;
  p.conditional.handle = cond;
  p.conditional.type = cudaGraphCondTypeIf;
  p.conditional.size = 1;
  cudaGraphNode_t node;
  CU(cudaGraphAddNode(&node, graph, deps, n_deps, &p));
  CU(cudaStreamBeginCaptureToGraph(e->body_stream, p.conditional.phGraph_out[0], nullptr, nullptr, 0,
                                   cudaStreamCaptureModeRelaxed));
  cudaStream_t outer = e->stream;
  e->stream = e->body_stream;
  e->pdl_break = true;
  const int st = body();
  e->stream = outer;
  cudaGraph_t body_graph = nullptr;
  const cudaError_t ce = cudaStreamEndCapture(e->body_stream, &body_graph);
  if (st != LSK_OK) return st;
  if (ce != cudaSuccess) return fail(LSK_ERR_CUDA, "conditional body capture failed: %s", cudaGetErrorString(ce));
  CU(cudaStreamUpdateCaptureDependencies(e->stream, &node, 1, cudaStreamSetCaptureDependencies));
  e->pdl_break = true;
  return LSK_OK;
}

// Adaptive round (lsk_round_adaptive): the rows of enqueue_round(E, d), but draft step j >= 1 runs
// only while no earlier draft has stopped the round (draft_confidence_kernel).  Each conditional
// body j holds step j's head, token and stop test, then the layers < E of row j + 1, the token
// step j chose: both run iff j < d_stop.  For j = d - 1 those layers are the verify's row d.
// Step 0 and the layers of row 1 always run (d_stop >= 1).  Layers >= E run on rows 0..d whatever
// d_stop is; rows past d_stop are finite (zeroed by step 0) and causally invisible to the kept rows.
static int enqueue_round_adaptive(lsk_engine* e, int E, int d) {
  const int* len = &e->state->len;
  std::vector<cudaGraphConditionalHandle> cond(d, 0);
  if (e->use_graph) {
    cudaStreamCaptureStatus cs;
    cudaGraph_t graph = nullptr;
    CU(cudaStreamGetCaptureInfo(e->stream, &cs, nullptr, &graph, nullptr, nullptr));
    for (int j = 1; j < d; ++j) CU(cudaGraphConditionalHandleCreate(&cond[j], graph, 0, cudaGraphCondAssignDefault));
  }
  const bool graph = e->use_graph;
  TRY(emit_embed(e, &e->state->tok[0], e->hidden, 1));
  for (int l = 0; l < E; ++l) TRY(enqueue_layer(e, l, 0, 1, len, 0));
  TRY(enqueue_draft_token(e, 0));
  TRY(emit_draft_confidence(e, 0, d, graph && d > 1 ? cond[1] : 0, graph && d > 1));
  for (int l = 0; l < E; ++l) TRY(enqueue_layer(e, l, 1, 1, len, 1));
  for (int j = 1; j < d; ++j) {
    TRY(enqueue_if(e, cond[j], [&]() -> int {
      TRY(enqueue_draft_token(e, j));
      TRY(emit_draft_confidence(e, j, d, graph && j + 1 < d ? cond[j + 1] : 0, graph && j + 1 < d));
      for (int l = 0; l < E; ++l) TRY(enqueue_layer(e, l, j + 1, 1, len, j + 1));
      return LSK_OK;
    }));
  }
  return enqueue_verify(e, E, d, &e->state->d_stop);
}

// Batched round (lsk_round_batch): the rows of enqueue_round(E, d) for each of B sequences, every
// weight pass shared.  Sequence s owns hidden rows s * (d + 1) .. s * (d + 1) + d; draft step i runs
// row i of every sequence (B rows, (d + 1) * hidden floats apart), the verify's layers >= E run all
// B * (d + 1) rows, each sequence at its own positions, over its own KV slot (page-table view
// page_table + s * P).  The GEMMs are batch-invariant and the attention partition is fixed by
// absolute key index, so every row is computed as in a round of that sequence alone.
struct BatchRows {
  SeqRows draft, verify;
  int stride;                          // floats between two sequences' rows of one draft step
};
static BatchRows batch_rows(lsk_engine* e, int B, int d) {
  const lsk_config& c = e->cfg;
  const int len_stride = (int)(sizeof(DevState) / sizeof(int));
  const int P = e->n_pages / B;
  const int stride = (d + 1) * c.hidden;
  return {SeqRows{B, 1, len_stride, P, stride}, SeqRows{B, d + 1, len_stride, P, c.hidden}, stride};
}

// Draft step i's head on row i of every sequence; each sequence's token becomes its tok[1 + i] and is
// embedded into its row i + 1 (sampling: the warped row goes to probs_d row s * (d + 1) + i).
static int enqueue_draft_token_seqs(lsk_engine* e, int i, int B, int d, int stride) {
  const lsk_config& c = e->cfg;
  TRY(enqueue_lm_head(e, i, B, i, stride));
  e->cur_class = CLS_MISC;
  if (e->gen.sample) {
    CU(launch(e, warp_and_sample_seqs_kernel, dim3(B), dim3(kSampleThreads), 0, (const float*)e->logits,
              e->vocab_l_pad, c.vocab, (const GenParams*)e->gen_dev, (const DevState*)e->bstate,
              (const unsigned long long*)e->batch_seeds, 1, d + 1, i, (int)RNG_DRAFT, e->probs_d,
              &e->bstate->tok[1 + i], (const __nv_bfloat16*)e->embed, c.hidden,
              e->hidden + (size_t)(i + 1) * c.hidden, stride));
    return LSK_OK;
  }
  CU(launch(e, finalize_embed_seqs_kernel, dim3(8, B), dim3(128), 0, cand_val_ptr(e), cand_idx_ptr(e), n_cand(e),
            e->bstate, 1 + i, (const __nv_bfloat16*)e->embed, c.hidden, e->hidden + (size_t)(i + 1) * c.hidden,
            stride));
  return LSK_OK;
}

// The batch's verify after the draft rows: layers >= E on all B * (d + 1) rows, the head, and the
// accept, which keeps d_stop[s] drafts of active sequence s (lsk_round_batch: d_seq).
static int enqueue_verify_seqs(lsk_engine* e, int E, int B, int d, const BatchRows& rows, const int* d_stop) {
  const lsk_config& c = e->cfg;
  const int* len = &e->bstate->len;
  const int* active = (const int*)e->batch_ctl + kMaxRows;
  const GenParams* gp = e->gen_dev;
  for (int l = E; l < c.n_layers; ++l) TRY(enqueue_layer(e, l, 0, B * (d + 1), len, 0, &rows.verify));
  TRY(enqueue_lm_head(e, 0, B * (d + 1), 0));
  e->cur_class = CLS_MISC;
  if (e->gen.sample) {
    const unsigned long long* seeds = e->batch_seeds;
    CU(launch(e, warp_and_sample_seqs_kernel, dim3(B * (d + 1)), dim3(kSampleThreads), 0, (const float*)e->logits,
              e->vocab_l_pad, c.vocab, gp, (const DevState*)e->bstate, seeds, d + 1, d + 1, 0, (int)RNG_VERIFY,
              e->probs_v, &e->bstate->verified[0], (const __nv_bfloat16*)nullptr, 0, (float*)nullptr, 0));
    CU(launch(e, accept_sample_seqs_kernel, dim3(B), dim3(kSampleThreads), 0, e->probs_d, (const float*)e->probs_v,
              c.vocab, d, e->bstate, gp, seeds, e->bres_dev, d_stop, active));
    return LSK_OK;
  }
  CU(launch(e, accept_greedy_seqs_kernel, dim3(B), dim3(256), 0, cand_val_ptr(e), cand_idx_ptr(e), n_cand(e), d,
            e->bstate, gp, e->bres_dev, d_stop, active));
  return LSK_OK;
}

static int enqueue_round_batch(lsk_engine* e, int E, int B, int d) {
  const lsk_config& c = e->cfg;
  const int* len = &e->bstate->len;
  const BatchRows rows = batch_rows(e, B, d);
  e->cur_class = CLS_MISC;
  CU(launch(e, embed_seq_tokens_kernel, dim3(B), dim3(256), 0, (const __nv_bfloat16*)e->embed, c.hidden,
            (const DevState*)e->bstate, e->hidden, rows.stride));
  for (int i = 0; i < d; ++i) {
    for (int l = 0; l < E; ++l) TRY(enqueue_layer(e, l, i, B, len, i, &rows.draft));
    TRY(enqueue_draft_token_seqs(e, i, B, d, rows.stride));
  }
  for (int l = 0; l < E; ++l) TRY(enqueue_layer(e, l, d, B, len, d, &rows.draft));
  return enqueue_verify_seqs(e, E, B, d, rows, (const int*)e->batch_ctl);
}

// Confidences and stop rules of draft step j for every sequence (draft_confidence_seqs_kernel).
static int emit_draft_confidence_seqs(lsk_engine* e, int j, int B, int d, cudaGraphConditionalHandle next,
                                      bool has_next) {
  const lsk_config& c = e->cfg;
  e->cur_class = CLS_MISC;
  const bool sample = e->gen.sample;
  const int grid = sample ? 1 : std::min(kConfMaxCtas, (c.vocab + kConfCols - 1) / kConfCols);
  CU(launch(e, draft_confidence_seqs_kernel, dim3(grid, B), dim3(kConfThreads), 0,
            sample ? (const float*)nullptr : (const float*)e->logits, e->vocab_l_pad,
            sample ? (const float*)e->probs_d : (const float*)nullptr, c.vocab, d + 1, e->bstate,
            (const GenParams*)e->gen_dev, e->bres_dev, e->conf_seqs, (const int*)e->batch_ctl,
            (const int*)e->batch_ctl + kMaxRows, j, e->hidden, c.hidden, next, (int)has_next));
  return LSK_OK;
}

// Adaptive batched round (lsk_round_batch_adaptive): the rows of enqueue_round_batch(E, B, d) with the
// conditional bodies of enqueue_round_adaptive.  Body j holds step j's head and tokens for every
// sequence, the confidence kernel, then layers < E of row j + 1 of every sequence; it runs iff some
// active sequence is still drafting after step j - 1.  Step 0 and row 1's layers always run.  The
// accept keeps min(d_seq[s], the step sequence s stopped at) drafts: conf_seqs->d_stop.
static int enqueue_round_batch_adaptive(lsk_engine* e, int E, int B, int d) {
  const lsk_config& c = e->cfg;
  const int* len = &e->bstate->len;
  const BatchRows rows = batch_rows(e, B, d);
  std::vector<cudaGraphConditionalHandle> cond(d, 0);
  if (e->use_graph) {
    cudaStreamCaptureStatus cs;
    cudaGraph_t graph = nullptr;
    CU(cudaStreamGetCaptureInfo(e->stream, &cs, nullptr, &graph, nullptr, nullptr));
    for (int j = 1; j < d; ++j) CU(cudaGraphConditionalHandleCreate(&cond[j], graph, 0, cudaGraphCondAssignDefault));
  }
  const bool graph = e->use_graph;
  e->cur_class = CLS_MISC;
  CU(launch(e, embed_seq_tokens_kernel, dim3(B), dim3(256), 0, (const __nv_bfloat16*)e->embed, c.hidden,
            (const DevState*)e->bstate, e->hidden, rows.stride));
  for (int l = 0; l < E; ++l) TRY(enqueue_layer(e, l, 0, B, len, 0, &rows.draft));
  TRY(enqueue_draft_token_seqs(e, 0, B, d, rows.stride));
  TRY(emit_draft_confidence_seqs(e, 0, B, d, graph && d > 1 ? cond[1] : 0, graph && d > 1));
  for (int l = 0; l < E; ++l) TRY(enqueue_layer(e, l, 1, B, len, 1, &rows.draft));
  for (int j = 1; j < d; ++j) {
    TRY(enqueue_if(e, cond[j], [&]() -> int {
      TRY(enqueue_draft_token_seqs(e, j, B, d, rows.stride));
      TRY(emit_draft_confidence_seqs(e, j, B, d, graph && j + 1 < d ? cond[j + 1] : 0, graph && j + 1 < d));
      for (int l = 0; l < E; ++l) TRY(enqueue_layer(e, l, j + 1, B, len, j + 1, &rows.draft));
      return LSK_OK;
    }));
  }
  return enqueue_verify_seqs(e, E, B, d, rows, (const int*)e->conf_seqs->d_stop);
}

static int enqueue_ar(lsk_engine* e, int n_layers_run) {
  const lsk_config& c = e->cfg;
  const int* len = &e->state->len;
  TRY(emit_embed(e, &e->state->tok[0], e->hidden, 1));
  for (int l = 0; l < n_layers_run; ++l) TRY(enqueue_layer(e, l, 0, 1, len, 0));
  TRY(enqueue_lm_head(e, 0, 1, 0));
  e->cur_class = CLS_MISC;
  if (!e->gen.sample) {
    TRY(emit_ar_commit(e));
  } else {
    CU(launch(e, warp_and_sample_kernel, dim3(1), dim3(kSampleThreads), 0, samp_logits(e),
              samp_ld(e), c.vocab, (const GenParams*)e->gen_dev, (const DevState*)e->state,
              e->probs_v, &e->state->verified[0], (int)RNG_VERIFY, 0));
    CU(launch(e, ar_commit_sampled_kernel, dim3(1), dim3(32), 0, e->state, e->res_dev, 0, hist_ptr(e)));
  }
  return LSK_OK;
}

// Run `enqueue` either eagerly or as a cached CUDA graph keyed by `key`.  Completion is
// the ev1 event in both modes; the commit kernels' stamp (RoundResult::seq) is always 0.
template <typename F>
static int run_cached(lsk_engine* e, long long key, F enqueue) {
  CU(cudaEventRecord(e->ev0, e->stream));
  if (!e->use_graph) {
    TRY(enqueue());
  } else {
    auto it = e->graphs.find(key);
    if (it == e->graphs.end()) {
      cudaGraph_t graph = nullptr;
      const int64_t before = e->launches;
      e->capture_launches = 0;
      CU(cudaStreamBeginCapture(e->stream, cudaStreamCaptureModeThreadLocal));
      int st = enqueue();
      cudaError_t ce = cudaStreamEndCapture(e->stream, &graph);
      if (st != LSK_OK) { if (graph) cudaGraphDestroy(graph); return st; }
      if (ce != cudaSuccess) return fail(LSK_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(ce));
      cudaGraphExec_t exec = nullptr;
      CU(cudaGraphInstantiate(&exec, graph, 0));
      CU(cudaGraphDestroy(graph));
      e->graph_launches[key] = e->capture_launches;
      e->launches = before;   // captured, not executed
      it = e->graphs.emplace(key, exec).first;
    }
    CU(cudaGraphLaunch(it->second, e->stream));
    e->launches += e->graph_launches[key];
  }
  CU(cudaEventRecord(e->ev1, e->stream));
  CU(cudaEventSynchronize(e->ev1));
  CU(cudaEventElapsedTime(&e->last_ms, e->ev0, e->ev1));
  return LSK_OK;
}

// ---------------------------------------------------------------------------------------------
// shape, buffer sizes and memory plan (host only)
// ---------------------------------------------------------------------------------------------
// want_pf_tc / want_lm_tc: the prompt pass and the wgmma LM head are asked for; each is taken when
// the hidden size fits it.
static EngineShape engine_shape(const lsk_config& c, int sm_count, bool want_pf_tc, bool want_lm_tc) {
  EngineShape s;
  s.heads_l = c.n_heads / c.tp_size;
  s.kv_heads_l = c.n_kv_heads / c.tp_size;
  s.group = c.n_heads / c.n_kv_heads;
  s.q_rows = s.heads_l * c.head_dim;
  s.kv_rows = s.kv_heads_l * c.head_dim;
  s.inter_l = c.inter / c.tp_size;
  s.inter_l_pad = (s.inter_l + 31) / 32 * 32;   // K of the down projection (zero columns beyond inter_l)
  s.vocab_l = c.vocab / c.tp_size;
  s.vocab_l_pad = (s.vocab_l + 15) / 16 * 16;
  s.vocab_off = c.tp_rank * s.vocab_l;
  s.n_pages = (c.max_ctx + kPageTokens - 1) / kPageTokens;
  s.max_pos = s.n_pages * kPageTokens;
  // split-KV factor: a constant of the engine (results are batch-invariant only for a fixed
  // partition).  The kernel is bound by per-SM load bandwidth and barrier latency, so the grid is
  // ONE CTA per SM on as many SMs as possible — splits = floor(SMs / kv heads), at most 4 (7B: 32
  // heads x 4 splits; an 8-way split's merge costs more than extra SMs bring).
  s.n_splits = c.attn_splits > 0 ? c.attn_splits : attn_default_splits(sm_count, s.kv_heads_l);
  if (s.n_splits > 8) s.n_splits = 8;
  if (s.n_splits < 1) s.n_splits = 1;
  s.pool_layer_elems = (size_t)s.n_pages * s.kv_heads_l * kPageTokens * c.head_dim;
  if (want_lm_tc) {
    // wgmma LM head: needs hidden % 64 == 0 and the 16-token B operand + a >= 3-stage ring in
    // shared memory (hidden <= 5120)
    int st = kTcMaxStages;
    while (st >= 3 && lmhead_tc_smem_bytes(c.hidden, st) > (size_t)kSmemMax) --st;
    if (c.hidden % kTcStageK == 0 && st >= 3) {
      s.lm_tc = true;
      s.lm_tc_stages = st;
      s.lm_tc_tiles = (s.vocab_l + kTcTileRows - 1) / kTcTileRows;
      const int waves = (s.lm_tc_tiles + sm_count - 1) / sm_count;
      s.lm_tc_grid = (s.lm_tc_tiles + waves - 1) / waves;        // even waves
      s.lm_cand = s.lm_tc_grid;
    }
  }
  s.pf_tc = want_pf_tc && c.hidden % 64 == 0;
  s.pf_stages = kPfMaxStages;
  s.kst_h = c.hidden / 64;
  s.kst_q = (s.q_rows + 63) / 64;
  s.kst_i = (s.inter_l + 63) / 64;
  s.pf_t_qkv = (s.q_rows + 2 * s.kv_rows + 127) / 128;
  s.pf_t_h = (c.hidden + 127) / 128;
  s.pf_t_gu = (2 * s.inter_l + 127) / 128;
  return s;
}

static MemTable mem_table(const lsk_config& c, const EngineShape& s, int sm_count) {
  const size_t h = c.hidden, V = c.vocab, P = s.max_pos, R = kMaxRows;
  const MemCat W = MEM_WEIGHTS, S = MEM_SCRATCH;
  MemTable t;
  t.wqkv = {(size_t)(s.q_rows + 2 * s.kv_rows) * h * 2, W};
  t.wo = {h * s.q_rows * 2, W};
  t.wgu = {(size_t)2 * s.inter_l * h * 2, W};
  t.wd = {h * s.inter_l_pad * 2, W};
  t.norm = {h * 2, W};
  t.wqkv_c = {(size_t)s.pf_t_qkv * s.kst_h * kCanonStageBytes, W};
  t.wo_c = {(size_t)s.pf_t_h * s.kst_q * kCanonStageBytes, W};
  t.wgu_c = {(size_t)s.pf_t_gu * s.kst_h * kCanonStageBytes, W};
  t.wd_c = {(size_t)s.pf_t_h * s.kst_i * kCanonStageBytes, W};
  t.rows_p = {(size_t)kPfTokens * h * 4, S};
  t.part_p = {(size_t)4 * kPfTokens * h * 4, S};
  t.q_p = {(size_t)kPfTokens * s.q_rows * 2, S};
  t.xn_c = {(size_t)s.kst_h * kCanonStageBytes, S};
  t.attn_c = {(size_t)s.kst_q * kCanonStageBytes, S};
  t.act_c = {(size_t)s.kst_i * kCanonStageBytes, S};
  t.embed = {V * h * 2, MEM_EMBED};
  t.final_norm = {h * 2, MEM_EMBED};
  t.lm_head = {(size_t)s.vocab_l_pad * h * 2, MEM_LM_HEAD};
  t.lm_head_tc = {(size_t)s.lm_tc_tiles * kTcTileRows * h * 2, MEM_LM_HEAD};
  t.kv_pool = {s.pool_layer_elems * c.n_layers * 2, MEM_KV_POOL};
  t.page_table = {(size_t)s.n_pages * 4, S};
  t.rope = {P * (c.head_dim / 2) * sizeof(float2), S};
  t.hidden = {(R + 1) * h * 4, S};
  t.qbuf = {R * s.q_rows * 2, S};
  t.act = {R * s.inter_l_pad * 2, S};
  t.tp_buf = {R * h * 4, S};
  t.attn = attn_bufs(s.kv_heads_l, s.group, c.head_dim, s.n_splits, std::max(kMaxRows, kPfTokens));
  t.cand = {(size_t)sm_count * R * 4, S};
  t.gath = {(size_t)c.tp_size * R * 4, S};
  t.row_best = {R * 4, S};
  t.d_zero = {4, S};
  t.d_prompt = {P * 4, S};
  t.state = {sizeof(DevState), S};
  t.gen_dev = {sizeof(GenParams), S};
  t.logits = {R * s.vocab_l_pad * 4, S};
  t.vocab_rows = {R * V * 4, S};
  t.samp_scratch = {V * 4, S};
  t.logits_gath = {(size_t)c.tp_size * R * s.vocab_l_pad * 4, S};
  t.conf_scratch = {sizeof(ConfScratch), S};
  t.score_rows = {P * 4, S};
  t.accept_rows = {P * 4, S};
  t.draft_rows = {(size_t)(s.pf_tc ? kPfTokens : kMaxRows) * V * 4, S};
  t.batch_buf = {8 * P * 4, S};
  t.view_table = {P * 4, S};
  t.piece_arrive = {(size_t)kPfTokens * s.kv_heads_l * 4, S};
  t.batch_state = {(size_t)kMaxRows * sizeof(DevState), S};
  t.batch_ctl = {(size_t)2 * kMaxRows * 4, S};
  t.batch_arrive = {(size_t)kMaxRows * s.kv_heads_l * 4, S};
  t.batch_seeds = {(size_t)kMaxRows * 8, S};
  t.conf_seqs = {sizeof(ConfSeqsScratch), S};
  t.peer_region = {peer_region_layout(c.tp_size, c.hidden).total, S};
  return t;
}

// Bytes per category (MemCat order) of what create_into allocates, plus what the uses allocate.
static void plan_memory(const lsk_config& c, const EngineShape& s, const MemTable& t, const lsk_memory_uses& u,
                        int64_t* cat) {
  auto add = [&](const MemBuf& b, size_t n) { cat[b.cat] += (int64_t)(b.bytes * n); };
  const size_t L = c.n_layers;
  for (const MemBuf& b : {t.wqkv, t.wo, t.wgu, t.wd}) add(b, L);
  add(t.norm, 2 * L);
  if (s.pf_tc) {
    for (const MemBuf& b : {t.wqkv_c, t.wo_c, t.wgu_c, t.wd_c}) add(b, L);
    add(t.rows_p, 2);
    for (const MemBuf& b : {t.part_p, t.q_p, t.xn_c, t.attn_c, t.act_c}) add(b, 1);
  }
  for (const MemBuf& b : {t.embed, t.final_norm, t.lm_head}) add(b, 1);
  if (s.lm_tc) add(t.lm_head_tc, 1);
  add(t.kv_pool, 2);
  for (const MemBuf& b : {t.page_table, t.rope, t.hidden, t.act, t.tp_buf, t.attn.part, t.attn.arrive, t.d_zero,
                          t.d_prompt, t.state, t.gen_dev})
    add(b, 1);
  add(t.qbuf, 2);
  add(t.cand, 2);
  add(t.gath, 2);
  add(t.row_best, 4);
  const bool packed = u.packed_scoring && s.pf_tc;     // without the prompt pass the call is refused
  const int score_k = std::max({u.score_exits, u.accept_exits, packed ? 1 : 0});
  const int draft_k = u.accept_exits - 1;
  if ((c.flags & LSK_FLAG_KEEP_LOGITS) || u.sampling || u.ngram_ban || u.adaptive || score_k > 0) add(t.logits, 1);
  if (u.sampling) {
    add(t.vocab_rows, 2);
    add(t.samp_scratch, 1);
    if (c.tp_size > 1) {
      add(t.logits_gath, 1);
      add(t.vocab_rows, 1);
    }
  }
  if (u.adaptive) add(t.conf_scratch, 1);
  add(t.score_rows, 2 * (size_t)score_k);
  if (draft_k > 0) {
    add(t.accept_rows, draft_k);
    add(t.draft_rows, draft_k);
    add(t.vocab_rows, 1);
  }
  if (packed)
    for (const MemBuf& b : {t.batch_buf, t.view_table, t.piece_arrive}) add(b, 1);
  if (u.tp_peer && c.tp_size > 1) add(t.peer_region, 1);
  if (u.batch_seqs > 0)                                // sized for max_rows sequences, whatever the batch
    for (const MemBuf& b : {t.batch_state, t.batch_ctl, t.batch_arrive}) add(b, 1);
  if (u.batch_seqs > 0 && u.sampling) add(t.batch_seeds, 1);
  if (u.batch_seqs > 0 && u.adaptive) add(t.conf_seqs, 1);
}

static lsk_memory_plan plan_of(const int64_t* cat) {
  return {cat[MEM_WEIGHTS], cat[MEM_EMBED], cat[MEM_LM_HEAD], cat[MEM_KV_POOL], cat[MEM_SCRATCH],
          cat[MEM_WEIGHTS] + cat[MEM_EMBED] + cat[MEM_LM_HEAD] + cat[MEM_KV_POOL] + cat[MEM_SCRATCH]};
}

// Buffers allocated on first use: nothing to do once *p is allocated.  On failure *p stays null, so a
// later call tries again.
template <typename T>
static int alloc_once(lsk_engine* e, T** p, const MemBuf& b, bool zero = false) {
  return *p ? LSK_OK : e->mem.alloc(p, b, zero);
}
// The same for a buffer that grows: the old allocation (if any) is freed first.
template <typename T>
static int realloc_grown(lsk_engine* e, T** p, const MemBuf& b) {
  e->mem.free(*p);
  *p = nullptr;
  return e->mem.alloc(p, b);
}
static MemBuf times(MemBuf b, size_t n) { return {b.bytes * n, b.cat}; }
// [16][vocab_l_pad] logits rows: the n-gram ban, sampling, adaptive drafts and the scoring heads
static int ensure_logits(lsk_engine* e) { return alloc_once(e, &e->logits, e->sizes.logits); }

// Exit j's head on M residual rows at x: sequence rows r0 .., rows rc .. of the current chunk.
using ExitHead = std::function<int(int j, const float* x, int r0, int rc, int M)>;

// The prompt pass's route for rows 0 .. rows-1 of d_prompt (row i at position i) through layers
// [0, E): prompts longer than one decode block go through the wgmma GEMMs 128 tokens per weight pass
// (prefill_tc.cuh), short ones through the decode kernels in blocks of <= max_rows rows.  With k == 0
// this is the prompt pass: no heads, and a chunk's last layer stops once its K/V rows are written.
// With k > 0 the rows are scored at exits[0 .. k) (strictly increasing, exits[k - 1] == E), and
// exit j's head runs where that exit's own pass would have stopped: wgmma chunks run to the end, with
// a tap at the top of layer exits[j] for the earlier exits and the last head after the chunk, each on
// the chunk's max_rows slices; decode blocks run it after layer exits[j] - 1.
static int enqueue_prompt_rows(lsk_engine* e, int rows, int E, const int* exits, int k, const ExitHead& head) {
  if (e->pf_tc && rows > e->max_rows) {
    for (int c0 = 0; c0 < rows; c0 += kPfTokens) {
      const int m = std::min(rows - c0, kPfTokens);
      auto slices = [&](int j) -> int {
        for (int r0 = 0; r0 < m; r0 += e->max_rows)
          TRY(head(j, e->hidden_p + (size_t)r0 * e->cfg.hidden, c0 + r0, r0, std::min(m - r0, e->max_rows)));
        return LSK_OK;
      };
      const ChunkTaps taps{exits, k - 1, slices};
      TRY(enqueue_prefill_chunk(e, c0, m, E, k > 0, nullptr, k > 1 ? &taps : nullptr));
      if (k > 0) TRY(slices(k - 1));
    }
  } else {
    for (int c0 = 0; c0 < rows; c0 += e->max_rows) {
      const int m = std::min(rows - c0, e->max_rows);
      TRY(emit_embed(e, e->d_prompt + c0, e->hidden, m));
      for (int l = 0, j = 0; l < E; ++l) {
        TRY(enqueue_layer(e, l, 0, m, e->d_zero, c0));
        if (j < k && exits[j] == l + 1) TRY(head(j++, e->hidden, c0, 0, m));
      }
    }
  }
  return LSK_OK;
}

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" {

int lsk_abi_version(void) { return LSK_ABI_VERSION; }
const char* lsk_last_error(void) { return g_last_error.c_str(); }

static int create_into(lsk_engine* e, const lsk_config& c);

// The configs lsk_create and lsk_plan_memory accept.
static int check_config(const lsk_config& c) {
  if (c.head_dim != 128 && c.head_dim != 64 && c.head_dim != 32)
    return fail(LSK_ERR_INVALID, "head_dim %d unsupported (32, 64 or 128)", c.head_dim);
  if (c.rope_scaling < LSK_ROPE_DEFAULT || c.rope_scaling > LSK_ROPE_LLAMA3)
    return fail(LSK_ERR_INVALID, "rope_scaling %d unknown", c.rope_scaling);
  if (c.rope_scaling != LSK_ROPE_DEFAULT && !(c.rope_factor > 0.f))
    return fail(LSK_ERR_INVALID, "rope scaling needs factor > 0");
  if (c.rope_scaling == LSK_ROPE_LLAMA3 &&
      (!(c.rope_high_freq_factor > c.rope_low_freq_factor) || c.rope_original_max_pos < 1))
    return fail(LSK_ERR_INVALID, "llama3 rope scaling needs high_freq_factor > low_freq_factor and original_max_position_embeddings");
  if (c.tp_size < 1 || c.tp_rank < 0 || c.tp_rank >= c.tp_size) return fail(LSK_ERR_INVALID, "bad tp_rank/tp_size");
  if (c.n_heads % c.tp_size || c.n_kv_heads % c.tp_size || c.n_heads % c.n_kv_heads)
    return fail(LSK_ERR_INVALID, "heads (%d) / kv heads (%d) must divide by tp_size (%d)", c.n_heads, c.n_kv_heads, c.tp_size);
  if (attn_layout_smem(c.head_dim, c.n_heads / c.n_kv_heads) > (size_t)kSmemMax)
    return fail(LSK_ERR_INVALID, "attention: group %d (%d heads over %d kv heads) at head_dim %d needs %zu bytes of "
                "shared memory for a 16-token launch, more than the %d available", c.n_heads / c.n_kv_heads,
                c.n_heads, c.n_kv_heads, c.head_dim, attn_layout_smem(c.head_dim, c.n_heads / c.n_kv_heads), kSmemMax);
  if (c.inter % (c.tp_size * 8)) return fail(LSK_ERR_INVALID, "intermediate size %d must be a multiple of 8*tp_size", c.inter);
  if (c.hidden % 32 || c.hidden > 8192) return fail(LSK_ERR_INVALID, "hidden %d must be a multiple of 32 and <= 8192", c.hidden);
  if (c.vocab % c.tp_size) return fail(LSK_ERR_INVALID, "vocab must divide by tp_size");
  if (c.n_layers < 1 || c.max_ctx < 2) return fail(LSK_ERR_INVALID, "bad n_layers / max_ctx");
  return LSK_OK;
}

int lsk_create(const lsk_config* cfg, lsk_engine** out) {
  if (!cfg || !out) return fail(LSK_ERR_INVALID, "null argument");
  TRY(check_config(*cfg));
  // everything that can fail half-way runs in create_into(); a failure releases what was built
  lsk_engine* e = new lsk_engine();
  const int st = create_into(e, *cfg);
  if (st != LSK_OK) {
    const std::string why = g_last_error;
    lsk_destroy(e);
    g_last_error = why;
    return st;
  }
  *out = e;
  return LSK_OK;
}

int lsk_plan_memory(const lsk_config* cfg, int32_t sm_count, const lsk_memory_uses* uses, lsk_memory_plan* out) {
  if (!cfg || !uses || !out) return fail(LSK_ERR_INVALID, "null argument");
  TRY(check_config(*cfg));
  if (sm_count < 1) return fail(LSK_ERR_INVALID, "sm_count %d must be >= 1", sm_count);
  if (uses->score_exits < 0 || uses->score_exits > LSK_MAX_EXITS || uses->accept_exits < 0 ||
      uses->accept_exits > LSK_MAX_EXITS)
    return fail(LSK_ERR_INVALID, "score_exits and accept_exits must be in [0, %d]", LSK_MAX_EXITS);
  if (uses->batch_seqs < 0 || uses->batch_seqs > kMaxRows)
    return fail(LSK_ERR_INVALID, "batch_seqs must be in [0, %d]", kMaxRows);
  const EngineShape s = engine_shape(*cfg, sm_count, !(cfg->flags & LSK_FLAG_NO_PREFILL_TC), uses->lm_head_tc != 0);
  int64_t cat[MEM_CATS] = {};
  plan_memory(*cfg, s, mem_table(*cfg, s, sm_count), *uses, cat);
  *out = plan_of(cat);
  return LSK_OK;
}

int lsk_memory_in_use(const lsk_engine* e, lsk_memory_plan* out) {
  if (!e || !out) return fail(LSK_ERR_INVALID, "null argument");
  int64_t cat[MEM_CATS] = {};
  e->mem.bytes_held(cat);
  *out = plan_of(cat);
  return LSK_OK;
}

static int create_into(lsk_engine* e, const lsk_config& c) {
  e->cfg = c;
  int dev = 0;
  CU(cudaGetDevice(&dev));
  CU(cudaDeviceGetAttribute(&e->sm_count, cudaDevAttrMultiProcessorCount, dev));
  e->use_pdl = !(c.flags & LSK_FLAG_NO_PDL);
  e->use_graph = !(c.flags & LSK_FLAG_NO_GRAPH);
  e->keep_logits = (c.flags & LSK_FLAG_KEEP_LOGITS) != 0;
  // tensor-parallel collectives: one-shot kernels over peer-mapped HBM.  Default 2 = the
  // row-parallel GEMM pushes its tiles to every rank from its own epilogue as LL lines; 1 =
  // separate LL push + reduce kernel; 3 = fence + flag protocol; 0 = NCCL.  LSK_FLAG_TP_NCCL
  // forces NCCL from the API.
  {
    const char* env = getenv("LSK_TP_ONESHOT");
    const int mode = env ? atoi(env) : ((c.flags & LSK_FLAG_TP_NCCL) ? 0 : 2);
    e->want_peer = c.tp_size > 1 && mode != 0;
    e->peer_mode = (mode >= 1 && mode <= 3) ? mode : 2;
  }
  if (const char* env = getenv("LSK_ABLATE")) {
    // diagnostics only: the named kernel classes are not launched (results are garbage, the
    // round keeps its shape) so that t(full) - t(ablated) gives a class's cost INSIDE the graph
    static const char* names[] = {"qkv", "attn", "o", "gate_up", "down", "lm_head"};
    std::string list(env);
    for (size_t pos = 0; pos <= list.size();) {            // comma-separated, exact names
      const size_t end = std::min(list.find(',', pos), list.size());
      const std::string tok = list.substr(pos, end - pos);
      for (int i = 0; i < 6; ++i)
        if (tok == names[i]) e->ablate |= 1u << i;
      pos = end + 1;
    }
    if (e->ablate) fprintf(stderr, "[lsk] LSK_ABLATE=%s: kernel classes skipped, outputs are NOT valid\n", env);
  }
  const char* lm_env = getenv("LSK_LMHEAD_TC");
  const char* pf_env = getenv("LSK_PREFILL_TC");
  const bool want_lm_tc = lm_env && atoi(lm_env) != 0;
  static_cast<EngineShape&>(*e) = engine_shape(c, e->sm_count, !(c.flags & LSK_FLAG_NO_PREFILL_TC) &&
                                               !(pf_env && atoi(pf_env) == 0), want_lm_tc);
  // without the wgmma LM head's fit, stay on the mma.sync kernel, loudly
  if (want_lm_tc && !e->lm_tc)
    fprintf(stderr, "[lsk] LSK_LMHEAD_TC ignored: hidden %d does not fit the wgmma LM head\n", c.hidden);
  e->sizes = mem_table(c, *e, e->sm_count);

  e->p_qkv = make_plan(e->q_rows + 2 * e->kv_rows, c.hidden);
  e->p_o = make_plan(c.hidden, e->q_rows);
  e->p_gu = make_plan(2 * e->inter_l, c.hidden);
  e->p_d = make_plan(c.hidden, e->inter_l_pad);
  e->p_lm = make_plan(e->vocab_l_pad, c.hidden);
  e->max_rows = plan_sched(2, kMaxRows, PRO_RMS, EPI_QKV, e->p_qkv, e->sm_count).ok ? kMaxRows : 8;

  CU(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
  CU(cudaEventCreate(&e->ev0));
  CU(cudaEventCreate(&e->ev1));

  e->mem.stream = e->stream;

  const MemTable& t = e->sizes;
  auto alloc = [&](auto** p, const MemBuf& b) { return e->mem.alloc(p, b, true); };   // zero-filled
  e->layers.resize(c.n_layers);
  for (auto& L : e->layers) {
    TRY(alloc(&L.wqkv, t.wqkv));
    TRY(alloc(&L.wo, t.wo));
    TRY(alloc(&L.wgu, t.wgu));
    TRY(alloc(&L.wd, t.wd));
    TRY(alloc(&L.ln1, t.norm));
    TRY(alloc(&L.ln2, t.norm));
    if (e->pf_tc) {
      TRY(alloc(&L.wqkv_c, t.wqkv_c));
      TRY(alloc(&L.wo_c, t.wo_c));
      TRY(alloc(&L.wgu_c, t.wgu_c));
      TRY(alloc(&L.wd_c, t.wd_c));
    }
  }
  if (e->pf_tc) {
    TRY(alloc(&e->hidden_p, t.rows_p));
    TRY(alloc(&e->tp_buf_p, t.rows_p));
    TRY(alloc(&e->part_p, t.part_p));
    TRY(alloc(&e->q_p, t.q_p));
    TRY(alloc(&e->xn_c, t.xn_c));
    TRY(alloc(&e->attn_c, t.attn_c));
    TRY(alloc(&e->act_c, t.act_c));
    CU(cudaFuncSetAttribute(prefill_gemm_tc_kernel<PF_EPI_QKV>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax));
    CU(cudaFuncSetAttribute(prefill_gemm_tc_kernel<PF_EPI_STORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax));
    CU(cudaFuncSetAttribute(prefill_gemm_tc_kernel<PF_EPI_SILU>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax));
    CU(cudaFuncSetAttribute(prefill_gemm_tc_kernel<PF_EPI_QKV_MAP>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax));
  }
  TRY(alloc(&e->embed, t.embed));
  TRY(alloc(&e->final_norm, t.final_norm));
  TRY(alloc(&e->lm_head, t.lm_head));
  if (e->lm_tc) {
    TRY(alloc(&e->lm_head_tc, t.lm_head_tc));
    CU(cudaFuncSetAttribute(lmhead_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax));
  }
  TRY(alloc(&e->kpool, t.kv_pool));
  TRY(alloc(&e->vpool, t.kv_pool));
  TRY(alloc(&e->page_table, t.page_table));
  TRY(alloc(&e->rope, t.rope));
  TRY(alloc(&e->hidden, t.hidden));
  TRY(alloc(&e->qbuf, t.qbuf));
  TRY(alloc(&e->attn_out, t.qbuf));
  TRY(alloc_attn_partials(e, t.attn));
  TRY(alloc(&e->act, t.act));   // pad columns stay zero
  TRY(alloc(&e->tp_buf, t.tp_buf));
  if (e->keep_logits) TRY(alloc(&e->logits, t.logits));
  TRY(alloc(&e->cand_val, t.cand));
  TRY(alloc(&e->cand_idx, t.cand));
  TRY(alloc(&e->gath_val, t.gath));
  TRY(alloc(&e->gath_idx, t.gath));
  TRY(alloc(&e->ban_val, t.row_best));
  TRY(alloc(&e->ban_idx, t.row_best));
  TRY(alloc(&e->rank_val, t.row_best));
  TRY(alloc(&e->rank_idx, t.row_best));
  TRY(alloc(&e->d_zero, t.d_zero));
  TRY(alloc(&e->d_prompt, t.d_prompt));
  TRY(alloc(&e->state, t.state));
  TRY(alloc(&e->gen_dev, t.gen_dev));
  CU(cudaHostAlloc((void**)&e->res_host, sizeof(RoundResult), cudaHostAllocMapped));
  memset(e->res_host, 0, sizeof(RoundResult));
  CU(cudaHostGetDevicePointer((void**)&e->res_dev, e->res_host, 0));

  {  // identity page table + RoPE table (fp32 maths as HF: inv_freq, angle and cos/sin in fp32)
    std::vector<int> pt(e->n_pages);
    for (int i = 0; i < e->n_pages; ++i) pt[i] = i;
    CU(cudaMemcpyAsync(e->page_table, pt.data(), pt.size() * 4, cudaMemcpyHostToDevice, e->stream));
    e->page_table_host = pt;
    // inv_freq as transformers computes it (modeling_rope_utils.py): default theta^(-2i/d), then the
    // checkpoint's scaling rule; angle and cos/sin in fp32 like LlamaRotaryEmbedding.forward
    const int half = c.head_dim / 2;
    std::vector<float2> tab((size_t)e->max_pos * half);
    for (int d = 0; d < half; ++d) {
      float inv_freq = 1.0f / powf(c.rope_theta, (float)(2 * d) / (float)c.head_dim);
      if (c.rope_scaling == LSK_ROPE_LINEAR) {
        inv_freq /= c.rope_factor;
      } else if (c.rope_scaling == LSK_ROPE_LLAMA3) {
        const float old_len = (float)c.rope_original_max_pos;
        const float low_wavelen = old_len / c.rope_low_freq_factor, high_wavelen = old_len / c.rope_high_freq_factor;
        const float wavelen = 2.0f * (float)M_PI / inv_freq;
        float scaled = wavelen > low_wavelen ? inv_freq / c.rope_factor : inv_freq;
        if (!(wavelen < high_wavelen) && !(wavelen > low_wavelen)) {
          const float smooth = (old_len / wavelen - c.rope_low_freq_factor) /
                               (c.rope_high_freq_factor - c.rope_low_freq_factor);
          scaled = (1.0f - smooth) * scaled / c.rope_factor + smooth * scaled;
        }
        inv_freq = scaled;
      }
      for (int p = 0; p < e->max_pos; ++p) {
        const float ang = (float)p * inv_freq;
        tab[(size_t)p * half + d] = make_float2((float)cos((double)ang), (float)sin((double)ang));
      }
    }
    CU(cudaMemcpyAsync(e->rope, tab.data(), tab.size() * sizeof(float2), cudaMemcpyHostToDevice, e->stream));
    CU(cudaStreamSynchronize(e->stream));
  }
  return LSK_OK;
}

void lsk_destroy(lsk_engine* e) { delete e; }

int lsk_comm_unique_id(uint8_t id_out[128]) {
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId size");
  ncclUniqueId id;
  NC(ncclGetUniqueId(&id));
  memcpy(id_out, &id, 128);
  return LSK_OK;
}

// Map every rank's peer region into this process (CUDA IPC; the handles travel over the engine's
// own NCCL communicator) and switch the TP collectives to the one-shot kernels of tp_peer.cuh.
static int peer_setup(lsk_engine* e) {
  const int tp = e->cfg.tp_size, rank = e->cfg.tp_rank;
  if (tp > kMaxPeers) return fail(LSK_ERR_INVALID, "one-shot collectives support at most %d ranks", kMaxPeers);
  TRY(e->mem.alloc(&e->peer_region, e->sizes.peer_region, true));
  CU(cudaDeviceSynchronize());
  cudaIpcMemHandle_t mine;
  CU(cudaIpcGetMemHandle(&mine, e->peer_region));
  const size_t hb = sizeof(cudaIpcMemHandle_t);
  DeviceMem handles;                   // every rank's handle, on the device for the all-gather
  unsigned char* d_h = nullptr;
  TRY(handles.alloc(&d_h, {hb * tp, MEM_SCRATCH}));
  CU(cudaMemcpy(d_h + hb * rank, &mine, hb, cudaMemcpyHostToDevice));
  NC(ncclAllGather(d_h + hb * rank, d_h, hb, ncclUint8, e->comm, e->stream));
  CU(cudaStreamSynchronize(e->stream));
  std::vector<cudaIpcMemHandle_t> all(tp);
  CU(cudaMemcpy(all.data(), d_h, hb * tp, cudaMemcpyDeviceToHost));
  int local_ok = 1;
  std::string why;
  for (int r = 0; r < tp; ++r) {
    if (r == rank) { e->peer.base[r] = (unsigned char*)e->peer_region; continue; }
    void* p = nullptr;
    cudaError_t er = cudaIpcOpenMemHandle(&p, all[r], cudaIpcMemLazyEnablePeerAccess);
    if (er != cudaSuccess) {
      local_ok = 0;
      why = cudaGetErrorString(er);
      cudaGetLastError();
      continue;
    }
    e->peer_opened[r] = p;
    e->peer.base[r] = (unsigned char*)p;
  }
  CU(cudaHostAlloc((void**)&e->peer_err_host, sizeof(int), cudaHostAllocMapped));
  *e->peer_err_host = 0;
  CU(cudaHostGetDevicePointer((void**)&e->peer.error, e->peer_err_host, 0));
  e->peer.rank = rank;
  e->peer.size = tp;
  e->peer.hidden = e->cfg.hidden;
  // every rank must take the same path: agree on min(local_ok).  The all-reduce also keeps the
  // ranks together until every mapping exists (nobody pushes into a region before its owner has
  // zeroed it: all did, they produced a handle).
  const float mine_ok = (float)local_ok;
  CU(cudaMemcpyAsync(e->tp_buf, &mine_ok, 4, cudaMemcpyHostToDevice, e->stream));
  NC(ncclAllReduce(e->tp_buf, e->tp_buf, 1, ncclFloat, ncclMin, e->comm, e->stream));
  float all_ok = 0.f;
  CU(cudaMemcpyAsync(&all_ok, e->tp_buf, 4, cudaMemcpyDeviceToHost, e->stream));
  CU(cudaStreamSynchronize(e->stream));
  CU(cudaMemsetAsync(e->tp_buf, 0, 4, e->stream));
  if (all_ok < 0.5f) {
    fprintf(stderr, "[lsk] rank %d: peer mapping unavailable (%s): tensor-parallel collectives fall back to NCCL\n",
            rank, local_ok ? "another rank failed" : why.c_str());
    return LSK_OK;
  }
  e->peer_ok = true;
  return LSK_OK;
}

static int peer_check(lsk_engine* e) {
  if (e->peer_err_host && *(volatile int*)e->peer_err_host)
    return fail(LSK_ERR_NCCL, "one-shot TP collective timed out waiting for another rank");
  return LSK_OK;
}

int lsk_comm_init(lsk_engine* e, const uint8_t id_in[128]) {
  if (!e) return fail(LSK_ERR_INVALID, "null engine");
  if (e->cfg.tp_size == 1) return LSK_OK;
  ncclUniqueId id;
  memcpy(&id, id_in, 128);
  NC(ncclCommInitRank(&e->comm, e->cfg.tp_size, id, e->cfg.tp_rank));
  if (e->want_peer) TRY(peer_setup(e));
  return LSK_OK;
}

static int pack(lsk_engine* e, const __nv_bfloat16* src, int64_t src_ld, int64_t row0, int64_t col0,
                int64_t n_rows, int64_t K, __nv_bfloat16* dst, int64_t dst_row0, int mode, int64_t K_dst = 0) {
  if (K_dst == 0) K_dst = K;
  const int64_t pairs = n_rows * (K / 2);
  int blocks = (int)((pairs + 255) / 256);
  if (blocks > e->sm_count * 32) blocks = e->sm_count * 32;
  if (blocks < 1) blocks = 1;
  pack_rows_kernel<<<blocks, 256, 0, e->stream>>>(src, src_ld, row0, col0, n_rows, K, dst, dst_row0, mode, K_dst, e->cfg.head_dim);
  CU(cudaGetLastError());
  return LSK_OK;
}

static int pack_canon(lsk_engine* e, const __nv_bfloat16* src, int64_t src_ld, int64_t row0, int64_t col0,
                      int64_t n_rows, int64_t K, unsigned char* dst, int64_t dst_row0, int mode, int n_kst) {
  if (!e->pf_tc) return LSK_OK;
  const int64_t total = n_rows * (K / 8);
  int blocks = (int)((total + 255) / 256);
  if (blocks > e->sm_count * 32) blocks = e->sm_count * 32;
  if (blocks < 1) blocks = 1;
  pack_canonical_rows_kernel<<<blocks, 256, 0, e->stream>>>(src, src_ld, row0, col0, n_rows, K, dst, dst_row0, mode,
                                                            n_kst, e->cfg.head_dim);
  CU(cudaGetLastError());
  return LSK_OK;
}

int lsk_load_weights(lsk_engine* e, const lsk_weight_desc* descs, int32_t n) {
  if (!e || !descs) return fail(LSK_ERR_INVALID, "null argument");
  const lsk_config& c = e->cfg;
  const int r = c.tp_rank;
  for (int i = 0; i < n; ++i) {
    const lsk_weight_desc& d = descs[i];
    const __nv_bfloat16* src = static_cast<const __nv_bfloat16*>(d.data);
    auto expect = [&](int64_t rows, int64_t cols) -> int {
      if (d.rows != rows || d.cols != cols)
        return fail(LSK_ERR_INVALID, "weight role %d layer %d: shape [%lld,%lld], expected [%lld,%lld]",
                    d.role, d.layer, (long long)d.rows, (long long)d.cols, (long long)rows, (long long)cols);
      return LSK_OK;
    };
    const bool per_layer = d.role >= LSK_W_LN1;
    if (per_layer && (d.layer < 0 || d.layer >= c.n_layers)) return fail(LSK_ERR_INVALID, "bad layer %d", d.layer);
    LayerWeights* L = per_layer ? &e->layers[d.layer] : nullptr;
    const int64_t h = c.hidden, qd = (int64_t)c.n_heads * c.head_dim, kvd = (int64_t)c.n_kv_heads * c.head_dim;
    switch (d.role) {
      case LSK_W_EMBED:
        TRY(expect(c.vocab, h));
        CU(cudaMemcpyAsync(e->embed, src, (size_t)c.vocab * h * 2, cudaMemcpyDeviceToDevice, e->stream));
        e->globals_loaded |= 1u;
        break;
      case LSK_W_FINAL_NORM:
        TRY(expect(h, 1));
        CU(cudaMemcpyAsync(e->final_norm, src, h * 2, cudaMemcpyDeviceToDevice, e->stream));
        e->globals_loaded |= 2u;
        break;
      case LSK_W_LM_HEAD:
        TRY(expect(c.vocab, h));
        TRY(pack(e, src, h, (int64_t)r * e->vocab_l, 0, e->vocab_l, h, e->lm_head, 0, MAP_PLAIN));
        if (e->lm_tc) {
          pack_canonical_kernel<<<e->sm_count * 8, 256, 0, e->stream>>>(src, h, (int64_t)r * e->vocab_l, e->vocab_l, h,
                                                              reinterpret_cast<uint4*>(e->lm_head_tc), e->lm_tc_tiles);
          CU(cudaGetLastError());
        }
        e->globals_loaded |= 4u;
        break;
      case LSK_W_LN1:
        TRY(expect(h, 1));
        CU(cudaMemcpyAsync(L->ln1, src, h * 2, cudaMemcpyDeviceToDevice, e->stream));
        break;
      case LSK_W_LN2:
        TRY(expect(h, 1));
        CU(cudaMemcpyAsync(L->ln2, src, h * 2, cudaMemcpyDeviceToDevice, e->stream));
        break;
      case LSK_W_Q:
        TRY(expect(qd, h));
        TRY(pack(e, src, h, (int64_t)r * e->q_rows, 0, e->q_rows, h, L->wqkv, 0, MAP_ROPE_HEADS));
        TRY(pack_canon(e, src, h, (int64_t)r * e->q_rows, 0, e->q_rows, h, L->wqkv_c, 0, MAP_ROPE_HEADS, e->kst_h));
        break;
      case LSK_W_K:
        TRY(expect(kvd, h));
        TRY(pack(e, src, h, (int64_t)r * e->kv_rows, 0, e->kv_rows, h, L->wqkv, e->q_rows, MAP_ROPE_HEADS));
        TRY(pack_canon(e, src, h, (int64_t)r * e->kv_rows, 0, e->kv_rows, h, L->wqkv_c, e->q_rows, MAP_ROPE_HEADS, e->kst_h));
        break;
      case LSK_W_V:
        TRY(expect(kvd, h));
        TRY(pack(e, src, h, (int64_t)r * e->kv_rows, 0, e->kv_rows, h, L->wqkv, e->q_rows + e->kv_rows, MAP_PLAIN));
        TRY(pack_canon(e, src, h, (int64_t)r * e->kv_rows, 0, e->kv_rows, h, L->wqkv_c, e->q_rows + e->kv_rows, MAP_PLAIN, e->kst_h));
        break;
      case LSK_W_O:   // row-parallel: this rank's input features = its heads
        TRY(expect(h, qd));
        TRY(pack(e, src, qd, 0, (int64_t)r * e->q_rows, h, e->q_rows, L->wo, 0, MAP_PLAIN));
        TRY(pack_canon(e, src, qd, 0, (int64_t)r * e->q_rows, h, e->q_rows, L->wo_c, 0, MAP_PLAIN, e->kst_q));
        break;
      case LSK_W_GATE:
        TRY(expect(c.inter, h));
        TRY(pack(e, src, h, (int64_t)r * e->inter_l, 0, e->inter_l, h, L->wgu, 0, MAP_GATE));
        TRY(pack_canon(e, src, h, (int64_t)r * e->inter_l, 0, e->inter_l, h, L->wgu_c, 0, MAP_GATE, e->kst_h));
        break;
      case LSK_W_UP:
        TRY(expect(c.inter, h));
        TRY(pack(e, src, h, (int64_t)r * e->inter_l, 0, e->inter_l, h, L->wgu, 0, MAP_UP));
        TRY(pack_canon(e, src, h, (int64_t)r * e->inter_l, 0, e->inter_l, h, L->wgu_c, 0, MAP_UP, e->kst_h));
        break;
      case LSK_W_DOWN:
        TRY(expect(h, c.inter));
        TRY(pack(e, src, c.inter, 0, (int64_t)r * e->inter_l, h, e->inter_l, L->wd, 0, MAP_PLAIN, e->inter_l_pad));
        TRY(pack_canon(e, src, c.inter, 0, (int64_t)r * e->inter_l, h, e->inter_l, L->wd_c, 0, MAP_PLAIN, e->kst_i));
        break;
      default:
        return fail(LSK_ERR_INVALID, "unknown weight role %d", d.role);
    }
    if (L) L->loaded |= 1u << d.role;
  }
  CU(cudaStreamSynchronize(e->stream));
  return LSK_OK;
}

int lsk_weights_complete(const lsk_engine* e) {
  if (!e) return 0;
  if (e->globals_loaded != 7u) return 0;
  const unsigned need = (1u << LSK_W_LN1) | (1u << LSK_W_Q) | (1u << LSK_W_K) | (1u << LSK_W_V) |
                        (1u << LSK_W_O) | (1u << LSK_W_LN2) | (1u << LSK_W_GATE) | (1u << LSK_W_UP) |
                        (1u << LSK_W_DOWN);
  for (const auto& L : e->layers)
    if ((L.loaded & need) != need) return 0;
  return 1;
}

int lsk_begin(lsk_engine* e, const lsk_generation* gen) {
  if (!e || !gen) return fail(LSK_ERR_INVALID, "null argument");
  if (!lsk_weights_complete(e)) return fail(LSK_ERR_STATE, "weights not fully loaded");
  if (gen->n_eos < 0 || gen->n_eos > LSK_MAX_EOS) return fail(LSK_ERR_INVALID, "n_eos out of range");
  if (gen->exit_layer > e->cfg.n_layers) return fail(LSK_ERR_INVALID, "exit_layer > n_layers");
  if (gen->no_repeat_ngram_size < 0 || gen->no_repeat_ngram_size > 16)
    return fail(LSK_ERR_INVALID, "no_repeat_ngram_size must be in [0, 16]");
  if (gen->no_repeat_ngram_size > 0) TRY(ensure_logits(e));
  if (gen->sample) {
    if (!(gen->temperature > 0.f)) return fail(LSK_ERR_INVALID, "temperature must be > 0");
    TRY(ensure_logits(e));
    TRY(alloc_once(e, &e->probs_d, e->sizes.vocab_rows));
    TRY(alloc_once(e, &e->probs_v, e->sizes.vocab_rows));
    TRY(alloc_once(e, &e->samp_scratch, e->sizes.samp_scratch));
    if (e->cfg.tp_size > 1) {
      TRY(alloc_once(e, &e->logits_gath, e->sizes.logits_gath));
      TRY(alloc_once(e, &e->logits_full, e->sizes.vocab_rows));
    }
  }
  e->gen = *gen;
  GenParams gp{};
  gp.n_eos = gen->n_eos;
  for (int i = 0; i < gen->n_eos; ++i) gp.eos[i] = gen->eos_ids[i];
  gp.sample = gen->sample; gp.temperature = gen->temperature; gp.top_k = gen->top_k; gp.top_p = gen->top_p;
  gp.seed = gen->seed;
  CU(cudaMemcpyAsync(e->gen_dev, &gp, sizeof(gp), cudaMemcpyHostToDevice, e->stream));
  CU(cudaMemsetAsync(e->state, 0, sizeof(DevState), e->stream));
  CU(cudaStreamSynchronize(e->stream));
  e->began = true;
  e->prefilled = false;
  e->batch_n = 0;
  e->host_len = 0;
  return LSK_OK;
}

int lsk_prefill(lsk_engine* e, const int32_t* ids, int32_t n) {
  if (!e || !ids) return fail(LSK_ERR_INVALID, "null argument");
  if (!e->began) return fail(LSK_ERR_STATE, "lsk_begin must precede lsk_prefill");
  if (n < 1) return fail(LSK_ERR_INVALID, "empty prompt");
  if (n + 1 > e->cfg.max_ctx) return fail(LSK_ERR_CTX, "prompt of %d tokens exceeds max_ctx %d", n, e->cfg.max_ctx);
  for (int i = 0; i < n; ++i)
    if (ids[i] < 0 || ids[i] >= e->cfg.vocab) return fail(LSK_ERR_INVALID, "token id %d out of range", ids[i]);
  CU(cudaEventRecord(e->ev0, e->stream));
  CU(cudaMemcpyAsync(e->d_prompt, ids, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  // ids[0 .. n-2] through every layer; no LM head: the reference discards those logits too
  // (self_speculation_generator.py:177)
  TRY(enqueue_prompt_rows(e, n - 1, e->cfg.n_layers, nullptr, 0, {}));
  set_state_kernel<<<1, 1, 0, e->stream>>>(e->state, n - 1, ids[n - 1], 0, n);
  CU(cudaGetLastError());
  CU(cudaEventRecord(e->ev1, e->stream));
  CU(cudaEventSynchronize(e->ev1));
  CU(cudaEventElapsedTime(&e->last_ms, e->ev0, e->ev1));
  TRY(peer_check(e));
  e->host_len = n - 1;
  e->prefilled = true;
  e->batch_n = 0;
  return LSK_OK;
}

static void copy_result(const RoundResult& r, lsk_round_out* out) {
  out->n_drafted = r.n_drafted;
  out->n_matches = r.n_matches;
  out->n_emitted = r.n_emitted;
  out->kv_len = r.kv_len;
  for (int i = 0; i < kMaxRows; ++i) {
    out->draft_ids[i] = r.draft_ids[i];
    out->emitted_ids[i] = r.emitted_ids[i];
    out->verified_ids[i] = r.verified_ids[i];
  }
}

int lsk_round(lsk_engine* e, int32_t d_req, lsk_round_out* out) {
  if (!e || !out) return fail(LSK_ERR_INVALID, "null argument");
  if (!e->prefilled) return fail(LSK_ERR_STATE, "lsk_prefill must precede lsk_round");
  if (d_req < 0 || d_req + 1 > e->max_rows) return fail(LSK_ERR_INVALID, "d_req %d out of [0,%d]", d_req, e->max_rows - 1);
  const int E = e->gen.exit_layer;
  if (E < 1 || E > e->cfg.n_layers) return fail(LSK_ERR_INVALID, "self-speculation needs 1 <= exit_layer <= n_layers (got %d)", E);
  if (e->host_len + d_req + 2 > e->max_pos) return fail(LSK_ERR_CTX, "context %d + %d exceeds max_ctx", e->host_len, d_req + 1);
  const long long key = ((long long)E << 20) | ((long long)d_req << 8) | (e->gen.sample ? 4 : 0) | 1 |
                        ((long long)e->gen.no_repeat_ngram_size << 32);
  TRY(run_cached(e, key, [&]() { return enqueue_round(e, E, d_req); }));
  TRY(peer_check(e));
  copy_result(*e->res_host, out);
  e->host_len = out->kv_len;
  return LSK_OK;
}

// What every adaptive round needs before its first launch: the stream conditional bodies are captured
// on (graph mode; driver >= 12.4), draft_confidence_kernel's scratch, and the logits rows greedy drafts
// materialise.
static int prepare_adaptive(lsk_engine* e) {
  if (e->use_graph && !e->body_stream) {
    int drv = 0;
    CU(cudaDriverGetVersion(&drv));
    if (drv < 12040) return fail(LSK_ERR_CUDA, "adaptive rounds need CUDA graph conditional nodes (driver >= 12.4, found %d)", drv);
    CU(cudaStreamCreateWithFlags(&e->body_stream, cudaStreamNonBlocking));
  }
  TRY(alloc_once(e, &e->conf_scratch, e->sizes.conf_scratch, true));
  return ensure_logits(e);
}

int lsk_round_adaptive(lsk_engine* e, int32_t d_max, float min_confidence, lsk_round_out* out,
                       float* draft_conf_out) {
  if (!e || !out) return fail(LSK_ERR_INVALID, "null argument");
  if (!(min_confidence >= 0.f && min_confidence <= 1.f))
    return fail(LSK_ERR_INVALID, "min_confidence %g outside [0, 1]", (double)min_confidence);
  if (e->cfg.tp_size > 1) return fail(LSK_ERR_INVALID, "lsk_round_adaptive needs tp_size == 1");
  if (!e->prefilled) return fail(LSK_ERR_STATE, "lsk_prefill must precede lsk_round_adaptive");
  if (d_max < 0 || d_max + 1 > e->max_rows) return fail(LSK_ERR_INVALID, "d_max %d out of [0,%d]", d_max, e->max_rows - 1);
  const int E = e->gen.exit_layer;
  if (E < 1 || E > e->cfg.n_layers) return fail(LSK_ERR_INVALID, "self-speculation needs 1 <= exit_layer <= n_layers (got %d)", E);
  if (e->host_len + d_max + 2 > e->max_pos) return fail(LSK_ERR_CTX, "context %d + %d exceeds max_ctx", e->host_len, d_max + 1);
  if (d_max == 0) return lsk_round(e, 0, out);      // no draft to stop: the reference's tail round
  TRY(prepare_adaptive(e));
  // the threshold is read from device memory: one graph per round shape serves every threshold
  CU(cudaMemcpyAsync(&e->state->min_conf, &min_confidence, sizeof(float), cudaMemcpyHostToDevice, e->stream));
  const long long key = ((long long)E << 20) | ((long long)d_max << 8) | (e->gen.sample ? 4 : 0) | 8 | 1 |
                        ((long long)e->gen.no_repeat_ngram_size << 32);
  e->adaptive = true;
  const int st = run_cached(e, key, [&]() { return enqueue_round_adaptive(e, E, d_max); });
  e->adaptive = false;
  e->pdl_break = false;
  TRY(st);
  copy_result(*e->res_host, out);
  if (draft_conf_out)
    for (int i = 0; i < out->n_drafted; ++i) draft_conf_out[i] = e->res_host->conf[i];
  e->host_len = out->kv_len;
  return LSK_OK;
}

int lsk_ar_step(lsk_engine* e, int32_t* token_out) {
  if (!e || !token_out) return fail(LSK_ERR_INVALID, "null argument");
  if (!e->prefilled) return fail(LSK_ERR_STATE, "lsk_prefill must precede lsk_ar_step");
  if (e->host_len + 2 > e->max_pos) return fail(LSK_ERR_CTX, "context exceeds max_ctx");
  const int nl = (e->gen.exit_layer > 0 && e->gen.exit_layer <= e->cfg.n_layers) ? e->gen.exit_layer : e->cfg.n_layers;
  const long long key = ((long long)nl << 20) | (e->gen.sample ? 4 : 0) | 2 | ((long long)e->gen.no_repeat_ngram_size << 32);
  TRY(run_cached(e, key, [&]() { return enqueue_ar(e, nl); }));
  TRY(peer_check(e));
  *token_out = e->res_host->emitted_ids[0];
  e->host_len = e->res_host->kv_len;
  return LSK_OK;
}

// What a batch of sequences needs of the generation lsk_begin set up: greedy, or sampling with one seed
// per sequence (`seeded`); no n-gram ban, one GPU, a self-speculation exit layer.
static int check_batch_generation(const lsk_engine* e, bool seeded) {
  if (e->gen.sample && !seeded)
    return fail(LSK_ERR_INVALID, "batched sampling needs one seed per sequence: use lsk_prefill_batch_seeded");
  if (e->gen.no_repeat_ngram_size > 0)
    return fail(LSK_ERR_INVALID, "batched generation does not support the n-gram ban (no_repeat_ngram_size %d)",
                e->gen.no_repeat_ngram_size);
  if (e->cfg.tp_size > 1) return fail(LSK_ERR_INVALID, "batched generation needs tp_size 1 (got %d)", e->cfg.tp_size);
  const int E = e->gen.exit_layer;
  if (E < 1 || E > e->cfg.n_layers)
    return fail(LSK_ERR_INVALID, "self-speculation needs 1 <= exit_layer <= n_layers (got %d)", E);
  return LSK_OK;
}

// Sequence s of a batch of n sequences owns logical pages [s * P, (s + 1) * P) of the pool, P = n_pages / n:
// its position p is logical position s * 64 * P + p.
static int batch_slot_positions(const lsk_engine* e, int n) { return e->n_pages / n * kPageTokens; }

// lsk_prefill_batch (seeds == NULL) and lsk_prefill_batch_seeded
static int prefill_batch(lsk_engine* e, const int32_t* ids, const int32_t* offsets, int32_t n_seqs,
                         const uint64_t* seeds, int32_t* slot_positions_out) {
  if (!e || !ids || !offsets) return fail(LSK_ERR_INVALID, "null argument");
  if (!e->began) return fail(LSK_ERR_STATE, "lsk_begin must precede lsk_prefill_batch");
  TRY(check_batch_generation(e, seeds != nullptr));
  if (n_seqs < 1 || n_seqs > e->max_rows)
    return fail(LSK_ERR_INVALID, "n_seqs %d outside [1, %d]", n_seqs, e->max_rows);
  if (offsets[0] != 0) return fail(LSK_ERR_INVALID, "offsets[0] must be 0 (got %d)", offsets[0]);
  const int slot = batch_slot_positions(e, n_seqs);
  for (int j = 0; j < n_seqs; ++j) {
    const int n = offsets[j + 1] - offsets[j];
    if (n < 1) return fail(LSK_ERR_INVALID, "prompt %d is empty (offsets %d, %d)", j, offsets[j], offsets[j + 1]);
    for (int i = offsets[j]; i < offsets[j + 1]; ++i)
      if (ids[i] < 0 || ids[i] >= e->cfg.vocab) return fail(LSK_ERR_INVALID, "prompt %d: token id %d out of range", j, ids[i]);
    if (n + 1 > slot)
      return fail(LSK_ERR_CTX, "prompt %d of %d tokens does not fit its slot of %d positions (%d sequences)", j, n, slot,
                  n_seqs);
    // the slot rounds max_ctx up to whole pages: a prompt lsk_prefill refuses has no solo run to match
    if (n + 1 > e->cfg.max_ctx)
      return fail(LSK_ERR_CTX, "prompt %d of %d tokens exceeds max_ctx %d", j, n, e->cfg.max_ctx);
  }
  const MemTable& t = e->sizes;
  TRY(alloc_once(e, &e->bstate, t.batch_state));
  TRY(alloc_once(e, &e->batch_ctl, t.batch_ctl));
  TRY(alloc_once(e, &e->batch_arrive, t.batch_arrive, true));
  if (!e->bres_host) {
    CU(cudaHostAlloc((void**)&e->bres_host, kMaxRows * sizeof(RoundResult), cudaHostAllocMapped));
    memset(e->bres_host, 0, kMaxRows * sizeof(RoundResult));
    CU(cudaHostGetDevicePointer((void**)&e->bres_dev, e->bres_host, 0));
  }
  if (e->gen.sample) TRY(alloc_once(e, &e->batch_seeds, t.batch_seeds));
  e->prefilled = false;
  e->batch_n = 0;
  e->host_len = 0;
  CU(cudaEventRecord(e->ev0, e->stream));
  CU(cudaMemsetAsync(e->bstate, 0, t.batch_state.bytes, e->stream));
  // the rounds' graphs read the seeds from here: one captured graph serves every set of seeds
  if (e->gen.sample)
    CU(cudaMemcpyAsync(e->batch_seeds, seeds, (size_t)n_seqs * sizeof(uint64_t), cudaMemcpyHostToDevice, e->stream));
  // prompt j through lsk_prefill's route, over its slot's page-table view
  int* const table = e->page_table;
  for (int j = 0; j < n_seqs; ++j) {
    const int32_t* p = ids + offsets[j];
    const int n = offsets[j + 1] - offsets[j];
    CU(cudaMemcpyAsync(e->d_prompt, p, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
    e->page_table = table + (size_t)j * (slot / kPageTokens);
    const int st = enqueue_prompt_rows(e, n - 1, e->cfg.n_layers, nullptr, 0, {});
    e->page_table = table;
    TRY(st);
    set_state_kernel<<<1, 1, 0, e->stream>>>(e->bstate + j, n - 1, p[n - 1], 0, n);
    CU(cudaGetLastError());
  }
  CU(cudaEventRecord(e->ev1, e->stream));
  CU(cudaEventSynchronize(e->ev1));
  CU(cudaEventElapsedTime(&e->last_ms, e->ev0, e->ev1));
  e->batch_len.assign(n_seqs, 0);
  for (int j = 0; j < n_seqs; ++j) e->batch_len[j] = offsets[j + 1] - offsets[j] - 1;
  e->batch_n = n_seqs;
  e->batch_seeded = seeds != nullptr;
  if (slot_positions_out) *slot_positions_out = slot;
  return LSK_OK;
}

int lsk_prefill_batch(lsk_engine* e, const int32_t* ids, const int32_t* offsets, int32_t n_seqs,
                      int32_t* slot_positions_out) {
  return prefill_batch(e, ids, offsets, n_seqs, nullptr, slot_positions_out);
}

int lsk_prefill_batch_seeded(lsk_engine* e, const int32_t* ids, const int32_t* offsets, int32_t n_seqs,
                             const uint64_t* seeds, int32_t* slot_positions_out) {
  if (!seeds) return fail(LSK_ERR_INVALID, "null argument");
  return prefill_batch(e, ids, offsets, n_seqs, seeds, slot_positions_out);
}

// lsk_round_batch's and lsk_round_batch_adaptive's preconditions; fills ctl with the round's d_seq and
// active flags ([2][kMaxRows], batch_ctl's layout).
static int check_batch_round(lsk_engine* e, const char* fn, int32_t d_req, const int32_t* d_seq,
                             const int32_t* active, int* ctl) {
  if (!e->batch_n) return fail(LSK_ERR_STATE, "lsk_prefill_batch must precede %s", fn);
  TRY(check_batch_generation(e, e->batch_seeded));
  const int B = e->batch_n;
  if (d_req < 0 || B * (d_req + 1) > e->max_rows)
    return fail(LSK_ERR_INVALID, "%d sequences x (d_req %d + 1) rows exceed the %d rows of a step", B, d_req,
                e->max_rows);
  for (int s = 0; s < B; ++s) {
    ctl[s] = d_seq ? d_seq[s] : d_req;
    ctl[kMaxRows + s] = active ? (active[s] != 0) : 1;
    if (ctl[s] < 0 || ctl[s] > d_req)
      return fail(LSK_ERR_INVALID, "d_seq[%d] = %d outside [0, d_req %d]", s, ctl[s], d_req);
  }
  const int slot = batch_slot_positions(e, B);
  for (int s = 0; s < B; ++s)
    if (e->batch_len[s] + d_req + 2 > slot)
      return fail(LSK_ERR_CTX, "sequence %d: context %d + %d exceeds its slot of %d positions", s, e->batch_len[s],
                  d_req + 1, slot);
  return LSK_OK;
}

static void copy_batch_results(lsk_engine* e, lsk_round_out* outs) {
  for (int s = 0; s < e->batch_n; ++s) {
    copy_result(e->bres_host[s], &outs[s]);
    e->batch_len[s] = outs[s].kv_len;
  }
}

int lsk_round_batch(lsk_engine* e, int32_t d_req, const int32_t* d_seq, const int32_t* active,
                    lsk_round_out* outs) {
  if (!e || !outs) return fail(LSK_ERR_INVALID, "null argument");
  int ctl[2 * kMaxRows] = {};
  TRY(check_batch_round(e, "lsk_round_batch", d_req, d_seq, active, ctl));
  const int B = e->batch_n, E = e->gen.exit_layer;
  CU(cudaMemcpyAsync(e->batch_ctl, ctl, sizeof(ctl), cudaMemcpyHostToDevice, e->stream));
  const long long key = ((long long)E << 20) | ((long long)d_req << 8) | (e->gen.sample ? 4 : 0) | 16 | 1 |
                        ((long long)B << 40);
  TRY(run_cached(e, key, [&]() { return enqueue_round_batch(e, E, B, d_req); }));
  copy_batch_results(e, outs);
  return LSK_OK;
}

int lsk_round_batch_adaptive(lsk_engine* e, int32_t d_max, const int32_t* d_seq, const int32_t* active,
                             float min_confidence, lsk_round_out* outs, float* draft_conf_out) {
  if (!e || !outs) return fail(LSK_ERR_INVALID, "null argument");
  if (!(min_confidence >= 0.f && min_confidence <= 1.f))
    return fail(LSK_ERR_INVALID, "min_confidence %g outside [0, 1]", (double)min_confidence);
  int ctl[2 * kMaxRows] = {};
  TRY(check_batch_round(e, "lsk_round_batch_adaptive", d_max, d_seq, active, ctl));
  if (d_max == 0) return lsk_round_batch(e, 0, d_seq, active, outs);   // no draft to stop
  const int B = e->batch_n, E = e->gen.exit_layer;
  TRY(prepare_adaptive(e));
  TRY(alloc_once(e, &e->conf_seqs, e->sizes.conf_seqs, true));
  CU(cudaMemcpyAsync(e->batch_ctl, ctl, sizeof(ctl), cudaMemcpyHostToDevice, e->stream));
  // the threshold is read from device memory: one graph per round shape serves every threshold
  CU(cudaMemcpyAsync(&e->conf_seqs->min_conf, &min_confidence, sizeof(float), cudaMemcpyHostToDevice, e->stream));
  const long long key = ((long long)E << 20) | ((long long)d_max << 8) | (e->gen.sample ? 4 : 0) | 16 | 8 | 1 |
                        ((long long)B << 40);
  e->adaptive = true;
  const int st = run_cached(e, key, [&]() { return enqueue_round_batch_adaptive(e, E, B, d_max); });
  e->adaptive = false;
  e->pdl_break = false;
  TRY(st);
  copy_batch_results(e, outs);
  if (draft_conf_out)
    for (int s = 0; s < B; ++s)
      for (int i = 0; i < outs[s].n_drafted; ++i) draft_conf_out[(size_t)s * LSK_MAX_SPEC + i] = e->bres_host[s].conf[i];
  return LSK_OK;
}

int lsk_profile_round(lsk_engine* e, int32_t d_req, lsk_round_out* out, float* class_ms,
                      int64_t* class_launches, float* total_ms) {
  if (!e || !out || !class_ms || !class_launches) return fail(LSK_ERR_INVALID, "null argument");
  if (!e->prefilled) return fail(LSK_ERR_STATE, "lsk_prefill must precede lsk_profile_round");
  if (d_req < 0 || d_req > LSK_MAX_SPEC) return fail(LSK_ERR_INVALID, "d_req out of range");
  const int E = e->gen.exit_layer;
  if (E < 1 || E > e->cfg.n_layers) return fail(LSK_ERR_INVALID, "bad exit_layer");
  if (e->host_len + d_req + 2 > e->max_pos) return fail(LSK_ERR_CTX, "context exceeds max_ctx");
  e->profiling = true;
  e->prof_events.clear();
  CU(cudaEventRecord(e->ev0, e->stream));
  int st = enqueue_round(e, E, d_req);
  e->profiling = false;
  if (st != LSK_OK) return st;
  CU(cudaEventRecord(e->ev1, e->stream));
  CU(cudaEventSynchronize(e->ev1));
  CU(cudaEventElapsedTime(&e->last_ms, e->ev0, e->ev1));
  if (total_ms) *total_ms = e->last_ms;
  for (int i = 0; i < CLS_COUNT; ++i) { class_ms[i] = 0.f; class_launches[i] = 0; }
  for (auto& pe : e->prof_events) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, pe.second.first, pe.second.second);
    class_ms[pe.first] += ms;
    class_launches[pe.first] += 1;
    cudaEventDestroy(pe.second.first);
    cudaEventDestroy(pe.second.second);
  }
  e->prof_events.clear();
  copy_result(*e->res_host, out);
  e->host_len = out->kv_len;
  return LSK_OK;
}

// Teacher-forced block (parity tests): the m given token ids as rows 0..m-1 at positions
// len .. len+m-1 through ALL layers and the LM head (logits kept: needs LSK_FLAG_KEEP_LOGITS).
// Nothing is committed: the rows' K/V entries land beyond the committed length and are
// overwritten by the next real step.  This is forward() of llama_model_utils.py:155-209 on a
// block of m tokens on top of the committed context.
int lsk_debug_forward_rows(lsk_engine* e, const int32_t* ids, int32_t m) {
  if (!e || !ids) return fail(LSK_ERR_INVALID, "null argument");
  if (!e->prefilled) return fail(LSK_ERR_STATE, "lsk_prefill must precede lsk_debug_forward_rows");
  if (!e->keep_logits) return fail(LSK_ERR_STATE, "engine created without LSK_FLAG_KEEP_LOGITS");
  if (m < 1 || m > e->max_rows) return fail(LSK_ERR_INVALID, "m %d out of [1,%d]", m, e->max_rows);
  if (e->host_len + m + 1 > e->max_pos) return fail(LSK_ERR_CTX, "context exceeds max_ctx");
  const lsk_config& c = e->cfg;
  for (int i = 0; i < m; ++i)
    if (ids[i] < 0 || ids[i] >= c.vocab) return fail(LSK_ERR_INVALID, "token id %d out of range", ids[i]);
  CU(cudaMemcpyAsync(e->d_prompt, ids, (size_t)m * 4, cudaMemcpyHostToDevice, e->stream));
  e->cur_class = CLS_MISC;
  CU(launch(e, embed_tokens_kernel, dim3(m), dim3(256), 0, (const __nv_bfloat16*)e->embed, c.hidden,
            (const int*)e->d_prompt, e->hidden, c.hidden));
  for (int l = 0; l < c.n_layers; ++l) TRY(enqueue_layer(e, l, 0, m, &e->state->len, 0));
  const int keep_sample = e->gen.sample;
  e->gen.sample = 0;
  const int keep_ban = e->gen.no_repeat_ngram_size;
  e->gen.no_repeat_ngram_size = 0;
  const int st = enqueue_lm_head(e, 0, m, 0);
  e->gen.no_repeat_ngram_size = keep_ban;
  e->gen.sample = keep_sample;
  if (st != LSK_OK) return st;
  CU(cudaStreamSynchronize(e->stream));
  TRY(peer_check(e));
  return LSK_OK;
}

// Scoring buffers, allocated on first use: the logits rows, result rows for k exits (regrown when a
// call asks for more), and with `batch` packed scoring's group upload, arrival counters and view table.
static int alloc_scoring(lsk_engine* e, int k, bool batch) {
  const MemTable& t = e->sizes;
  TRY(ensure_logits(e));
  if (k > e->score_cap) {
    e->score_cap = 0;
    TRY(realloc_grown(e, &e->score_lp, times(t.score_rows, k)));
    TRY(realloc_grown(e, &e->score_greedy, times(t.score_rows, k)));
    e->score_cap = k;
  }
  if (batch) {
    TRY(alloc_once(e, &e->batch_buf, t.batch_buf));
    TRY(alloc_once(e, &e->view_table, t.view_table));
    TRY(alloc_once(e, &e->piece_arrive, t.piece_arrive, true));
  }
  return LSK_OK;
}

// lsk_score_exits' acceptance buffers for k - 1 draft exits: the acceptance rows and the warped draft
// rows of a chunk, plus the warped full-depth rows of a slice.  A call with more exits regrows them.
static int alloc_accept(lsk_engine* e, int k) {
  if (k - 1 <= e->accept_cap) return LSK_OK;
  const MemTable& t = e->sizes;
  e->accept_cap = 0;
  TRY(realloc_grown(e, &e->exits_accept, times(t.accept_rows, k - 1)));
  TRY(realloc_grown(e, &e->exits_pd, times(t.draft_rows, k - 1)));
  TRY(alloc_once(e, &e->exits_pv, t.vocab_rows));
  e->accept_cap = k - 1;
  return LSK_OK;
}

// LM head + log softmax on M residual rows at x: the log-probabilities of targets[0 .. M) and the
// arg-max ids go to lp / greedy (row 0 of score_lp / score_greedy unless given) from row r on.
static int enqueue_score_head(lsk_engine* e, const float* x, int M, const int* targets, int r,
                              float* lp = nullptr, int* greedy = nullptr) {
  e->cur_class = CLS_LMHEAD;
  TRY(launch_lm_head_gemm(e, x, M, e->logits));
  e->cur_class = CLS_MISC;
  CU(launch(e, logprob_rows_kernel, dim3(M), dim3(kLogprobThreads), 0, (const float*)e->logits, e->vocab_l_pad,
            e->vocab_l, targets, (lp ? lp : e->score_lp) + r, (greedy ? greedy : e->score_greedy) + r));
  return LSK_OK;
}

// Teacher-forced scoring of one sequence (forward / forward_early of llama_model_utils.py:155-276 on
// the whole sequence) at exits[0 .. k) in one pass: rows 0 .. n-2 take the prompt pass's route
// through layers [0, exits[k - 1]), and at every exit the final norm, the mma.sync LM head, then per
// row the log-probability of the next id and the arg-max.  Each exit's head runs where that exit's
// own pass would have stopped (enqueue_prompt_rows), so every row is bit-identical to a one-exit call
// at that exit.  With accept_out, each earlier exit's head also warps its logits into the chunk's
// draft rows, and the full-depth head computes the acceptance probability of every draft row against
// its own warped row.  The K/V rows overwrite the pool: any generation in progress ends here.
static int score_sequence(lsk_engine* e, const int32_t* ids, int n, const int32_t* exits, int k,
                          const lsk_generation* sampling, float* logprob_out, int32_t* greedy_out, float* accept_out) {
  TRY(alloc_scoring(e, k, false));
  if (accept_out) TRY(alloc_accept(e, k));
  const int rows = n - 1, V = e->cfg.vocab;
  const size_t P = (size_t)e->max_pos, pd_stride = e->sizes.draft_rows.bytes / 4;   // floats per draft exit
  const WarpParams wp = accept_out ? WarpParams{sampling->temperature, sampling->top_k, sampling->top_p}
                                   : WarpParams{1.f, 0, 1.f};
  e->prefilled = false;
  e->batch_n = 0;
  e->host_len = 0;
  auto head = [&](int j, const float* x, int r0, int rc, int M) -> int {
    TRY(enqueue_score_head(e, x, M, e->d_prompt + r0 + 1, r0, e->score_lp + j * P, e->score_greedy + j * P));
    if (!accept_out || k == 1) return LSK_OK;
    e->cur_class = CLS_MISC;
    if (j + 1 < k) {
      CU(launch(e, warp_rows_kernel, dim3(M), dim3(kSampleThreads), 0, (const float*)e->logits, e->vocab_l_pad, V,
                wp, e->exits_pd + j * pd_stride + (size_t)rc * V));
    } else {
      CU(launch(e, accept_prob_kernel, dim3(M), dim3(kSampleThreads), 0, (const float*)e->logits, e->vocab_l_pad, V,
                wp, (const float*)(e->exits_pd + (size_t)rc * V), pd_stride, k - 1, e->exits_pv,
                e->exits_accept + r0, P));
    }
    return LSK_OK;
  };
  CU(cudaEventRecord(e->ev0, e->stream));
  CU(cudaMemcpyAsync(e->d_prompt, ids, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  TRY(enqueue_prompt_rows(e, rows, exits[k - 1], exits, k, head));
  CU(cudaEventRecord(e->ev1, e->stream));
  CU(cudaMemcpy2DAsync(logprob_out, (size_t)rows * 4, e->score_lp, P * 4, (size_t)rows * 4, k,
                       cudaMemcpyDeviceToHost, e->stream));
  if (greedy_out)
    CU(cudaMemcpy2DAsync(greedy_out, (size_t)rows * 4, e->score_greedy, P * 4, (size_t)rows * 4, k,
                         cudaMemcpyDeviceToHost, e->stream));
  if (accept_out && k > 1)
    CU(cudaMemcpy2DAsync(accept_out, (size_t)rows * 4, e->exits_accept, P * 4, (size_t)rows * 4, k - 1,
                         cudaMemcpyDeviceToHost, e->stream));
  CU(cudaStreamSynchronize(e->stream));
  CU(cudaEventElapsedTime(&e->last_ms, e->ev0, e->ev1));
  return LSK_OK;
}

// Teacher-forced scoring of one sequence at full depth or at an early exit: score_sequence with the
// one exit E.
int lsk_score(lsk_engine* e, const int32_t* ids, int32_t n, int32_t exit_layer, float* logprob_out,
              int32_t* greedy_out) {
  if (!e || !ids || !logprob_out) return fail(LSK_ERR_INVALID, "null argument");
  const lsk_config& c = e->cfg;
  if (c.tp_size > 1) return fail(LSK_ERR_INVALID, "lsk_score needs tp_size 1: tensor-parallel scoring is not supported");
  if (n < 2) return fail(LSK_ERR_INVALID, "scoring needs at least 2 ids (got %d)", n);
  if (n > c.max_ctx) return fail(LSK_ERR_CTX, "sequence of %d ids exceeds max_ctx %d", n, c.max_ctx);
  if (exit_layer > c.n_layers) return fail(LSK_ERR_INVALID, "exit_layer %d > n_layers %d", exit_layer, c.n_layers);
  for (int i = 0; i < n; ++i)
    if (ids[i] < 0 || ids[i] >= c.vocab) return fail(LSK_ERR_INVALID, "token id %d out of range", ids[i]);
  if (!lsk_weights_complete(e)) return fail(LSK_ERR_STATE, "weights not fully loaded");
  const int32_t E = exit_layer <= 0 ? c.n_layers : exit_layer;
  return score_sequence(e, ids, n, &E, 1, nullptr, logprob_out, greedy_out, nullptr);
}

// Attention pieces of nr packed rows at group rows r .. r + nr - 1, positions pos0 .., first page
// `page`: maximal runs inside one 128-row chunk, cut to the m_attn rows one prompt-attention launch
// holds.  chunk_first[c] is the first piece of chunk c.
static void add_pieces(std::vector<int4>& pieces, std::vector<int>& chunk_first, int r, int nr, int pos0, int page,
                       int m_attn) {
  for (int i = 0; i < nr;) {
    const int row = r + i, chunk = row / kPfTokens;
    const int len = std::min(std::min(nr - i, (chunk + 1) * kPfTokens - row), m_attn);
    while ((int)chunk_first.size() <= chunk) chunk_first.push_back((int)pieces.size());
    pieces.push_back(make_int4(row - chunk * kPfTokens, len, pos0 + i, page));
    i += len;
  }
}

// The 128-row chunks of `rows` packed rows through layers [0, E): ids, row map and pieces on the
// device at d_ids / d_map / d_pieces, the pieces' host copy in pieces / chunk_first (with its final
// count), first pages indexing the view table `pages`.  With targets every chunk runs to the end and
// the score head runs on its max_rows slices (score_lp / score_greedy from row c0 on); without, the
// chunks are a prompt pass that only writes K/V.
static int enqueue_packed_chunks(lsk_engine* e, int rows, int E, const int* d_ids, const int2* d_map,
                                 const int4* d_pieces, const std::vector<int4>& pieces,
                                 const std::vector<int>& chunk_first, const int* d_tgt, const int* pages) {
  const int hidden = e->cfg.hidden;
  for (int ci = 0, c0 = 0; c0 < rows; ++ci, c0 += kPfTokens) {
    const int m = std::min(rows - c0, kPfTokens);
    PackedChunk pk{d_ids + c0, d_map + c0, d_pieces + chunk_first[ci], chunk_first[ci + 1] - chunk_first[ci], 0, pages};
    for (int p = chunk_first[ci]; p < chunk_first[ci + 1]; ++p) pk.max_piece_rows = std::max(pk.max_piece_rows, pieces[p].y);
    TRY(enqueue_prefill_chunk(e, c0, m, E, d_tgt != nullptr, &pk));
    if (!d_tgt) continue;
    for (int r0 = 0; r0 < m; r0 += e->max_rows)
      TRY(enqueue_score_head(e, e->hidden_p + (size_t)r0 * hidden, std::min(m - r0, e->max_rows), d_tgt + c0 + r0,
                             c0 + r0));
  }
  return LSK_OK;
}

// Packed scoring's input: a prefix P and the branches B that continue it, pointers into the caller's
// arrays; a branch's results go to the output arrays from row out_row on.
struct ScoreBranch { const int32_t* ids; int n, out_row; };
struct ScorePrefix { const int32_t* ids; int n; std::vector<ScoreBranch> br; };

// Teacher-forced scoring of branches that continue prefixes, on the wgmma prompt pass through layers
// [0, E).  Entry i of branch B on prefix P is the log-probability of B[i] after P + B[:i].  The
// prefixes with their branches are taken in order in groups, as many as the KV pool and the view
// table hold; a prefix whose branches do not all fit runs again in the next group.  With
// s = len(P) - 1 and t = s mod 64, a group runs in two phases:
//  * prefix phase: rows P[0 .. s) at positions 0 .. s - 1 write K/V only (the prompt pass: the last
//    layer stops after its QKV GEMM, no head);
//  * branch phase: rows [P[s]] + B[:-1] at positions s .. s + len(B) - 1 with targets B are scored.
// The rows of a phase are concatenated in input order and cut into 128-row chunks; one upload per
// group carries the row ids, the targets, the row maps (position, first page) and the pieces of every
// chunk: maximal runs of one sequence's rows inside a chunk, cut to the rows one prompt-attention
// launch holds.  Every sequence reads and writes keys through its own page-table view in view_table:
// a prefix's view is its own pages; a branch's view is the prefix's s / 64 full pages, then (t > 0) a
// page holding slots [0, t) of the prefix's partial page, then the branch's own pages.  The prefix's
// first branch in the group adopts that partial page in place (its rows write slots >= t only); every
// further branch gets a private copy of slots [0, t), made by one kv_copy_slots_kernel launch between
// the phases.  A later chunk of a sequence attends to the K/V rows its earlier chunks wrote, at the
// positions lsk_score puts them, so every row's arithmetic is that of lsk_score on P + B's wgmma route.
static int score_packed(lsk_engine* e, int E, const std::vector<ScorePrefix>& pre, float* logprob_out,
                        int32_t* greedy_out) {
  TRY(alloc_scoring(e, 1, true));
  const int m_attn = prompt_attn_rows(e->cfg.head_dim, e->group);
  e->prefilled = false;
  e->batch_n = 0;
  e->host_len = 0;

  struct Member { const ScorePrefix* p; int b0, b1; };   // a prefix with its branches [b0, b1) in the group
  std::vector<Member> grp;                 // the group being formed
  std::vector<int32_t> up, view;           // the group's upload to batch_buf, its page-table views
  std::vector<int4> pre_pieces, br_pieces, copies;
  std::vector<int> pre_first, br_first, pre_view, br_view, br_row;
  std::vector<float> lp_host;
  std::vector<int32_t> gr_host;
  // batch_buf sections start 16-byte aligned (row maps are int2, pieces and copies int4)
  auto section = [&](size_t n) { const size_t o = up.size(); up.resize(o + (n + 3) / 4 * 4, 0); return o; };
  auto run_group = [&](bool last) -> int {
    view.clear(); copies.clear(); pre_pieces.clear(); br_pieces.clear();
    pre_first.clear(); br_first.clear(); pre_view.clear(); br_view.clear(); br_row.clear();
    int logical = 0, rp = 0, rb = 0;
    auto new_page = [&]() { return e->page_table_host[logical++]; };
    for (const Member& g : grp) {
      const int s = g.p->n - 1, nf = s / kPageTokens, t = s % kPageTokens, pv = (int)view.size();
      pre_view.push_back(pv);
      for (int k = 0; k < (s + kPageTokens - 1) / kPageTokens; ++k) view.push_back(new_page());
      rp += s;
      for (int k = g.b0; k < g.b1; ++k) {
        const int nb = g.p->br[k].n, bv = (int)view.size(), n_view = (s + nb + kPageTokens - 1) / kPageTokens;
        for (int q = 0; q < nf; ++q) { const int page = view[pv + q]; view.push_back(page); }
        if (t > 0) {
          const int partial = view[pv + nf];
          if (k == g.b0) {
            view.push_back(partial);
          } else {
            const int page = new_page();
            view.push_back(page);
            copies.push_back(make_int4(partial, page, t, 0));
          }
        }
        while ((int)view.size() - bv < n_view) view.push_back(new_page());
        br_view.push_back(bv);
        br_row.push_back(rb);
        rb += nb;
      }
    }
    up.clear();
    const size_t o_pid = section(rp), o_pmap = section(2 * (size_t)rp);
    const size_t o_bid = section(rb), o_btgt = section(rb), o_bmap = section(2 * (size_t)rb);
    for (size_t gi = 0, r = 0, bi = 0; gi < grp.size(); ++gi) {
      const Member& g = grp[gi];
      const int32_t* P = g.p->ids;
      const int s = g.p->n - 1;
      for (int i = 0; i < s; ++i) {
        up[o_pid + r + i] = P[i];
        up[o_pmap + 2 * (r + i)] = i;
        up[o_pmap + 2 * (r + i) + 1] = pre_view[gi];
      }
      add_pieces(pre_pieces, pre_first, (int)r, s, 0, pre_view[gi], m_attn);
      r += s;
      for (int k = g.b0; k < g.b1; ++k, ++bi) {
        const int32_t* B = g.p->br[k].ids;
        const int lb = g.p->br[k].n, r0 = br_row[bi];
        for (int i = 0; i < lb; ++i) {
          up[o_bid + r0 + i] = i ? B[i - 1] : P[s];
          up[o_btgt + r0 + i] = B[i];
          up[o_bmap + 2 * (r0 + i)] = s + i;
          up[o_bmap + 2 * (r0 + i) + 1] = br_view[bi];
        }
        add_pieces(br_pieces, br_first, r0, lb, s, br_view[bi], m_attn);
      }
    }
    pre_first.push_back((int)pre_pieces.size());
    br_first.push_back((int)br_pieces.size());
    const size_t o_ppc = section(4 * pre_pieces.size()), o_bpc = section(4 * br_pieces.size());
    const size_t o_cp = section(4 * copies.size());
    memcpy(up.data() + o_ppc, pre_pieces.data(), pre_pieces.size() * sizeof(int4));
    memcpy(up.data() + o_bpc, br_pieces.data(), br_pieces.size() * sizeof(int4));
    memcpy(up.data() + o_cp, copies.data(), copies.size() * sizeof(int4));
    // every row owns a pool slot and needs at most 8 ints, so a group that fits the pool fits batch_buf
    if (up.size() > (size_t)8 * e->max_pos)
      return fail(LSK_ERR_INVALID, "packed scoring: group upload of %zu ints exceeds its buffer", up.size());
    CU(cudaMemcpyAsync(e->batch_buf, up.data(), up.size() * 4, cudaMemcpyHostToDevice, e->stream));
    CU(cudaMemcpyAsync(e->view_table, view.data(), view.size() * 4, cudaMemcpyHostToDevice, e->stream));
    const int* d = e->batch_buf;
    auto i2 = [&](size_t o) { return reinterpret_cast<const int2*>(d + o); };
    auto i4 = [&](size_t o) { return reinterpret_cast<const int4*>(d + o); };
    TRY(enqueue_packed_chunks(e, rp, E, d + o_pid, i2(o_pmap), i4(o_ppc), pre_pieces, pre_first, nullptr,
                              e->view_table));
    if (!copies.empty()) {
      e->cur_class = CLS_MISC;
      CU(launch(e, kv_copy_slots_kernel, dim3((unsigned)copies.size(), E, 2 * e->kv_heads_l), dim3(128), 0, i4(o_cp),
                e->kpool, e->vpool, e->pool_layer_elems, e->kv_heads_l, e->cfg.head_dim));
    }
    TRY(enqueue_packed_chunks(e, rb, E, d + o_bid, i2(o_bmap), i4(o_bpc), br_pieces, br_first, d + o_btgt,
                              e->view_table));
    if (last) CU(cudaEventRecord(e->ev1, e->stream));
    lp_host.resize(rb);
    gr_host.resize(rb);
    CU(cudaMemcpyAsync(lp_host.data(), e->score_lp, (size_t)rb * 4, cudaMemcpyDeviceToHost, e->stream));
    if (greedy_out)
      CU(cudaMemcpyAsync(gr_host.data(), e->score_greedy, (size_t)rb * 4, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    for (size_t gi = 0, bi = 0; gi < grp.size(); ++gi)
      for (int k = grp[gi].b0; k < grp[gi].b1; ++k, ++bi) {
        const ScoreBranch& b = grp[gi].p->br[k];
        memcpy(logprob_out + b.out_row, lp_host.data() + br_row[bi], (size_t)b.n * 4);
        if (greedy_out) memcpy(greedy_out + b.out_row, gr_host.data() + br_row[bi], (size_t)b.n * 4);
      }
    grp.clear();
    return LSK_OK;
  };

  CU(cudaEventRecord(e->ev0, e->stream));
  int pages = 0, views = 0;   // pool pages and view entries the group uses
  for (const ScorePrefix& p : pre) {
    const int s = p.n - 1, nf = s / kPageTokens, t = s % kPageTokens, own = (s + kPageTokens - 1) / kPageTokens;
    bool in_group = false;
    for (int b = 0; b < (int)p.br.size(); ++b) {
      const int n_view = (s + p.br[b].n + kPageTokens - 1) / kPageTokens;
      // the prefix's pages come with its first branch in a group, which adopts the partial page
      auto need_pages = [&]() { return in_group ? n_view - nf : own + n_view - nf - (t > 0 ? 1 : 0); };
      auto need_views = [&]() { return in_group ? n_view : own + n_view; };
      if (pages + need_pages() > e->n_pages || views + need_views() > e->max_pos) {
        TRY(run_group(false));
        pages = views = 0;
        in_group = false;
      }
      pages += need_pages();
      views += need_views();
      if (!in_group) grp.push_back({&p, b, b});
      in_group = true;
      ++grp.back().b1;
    }
  }
  TRY(run_group(true));
  CU(cudaEventElapsedTime(&e->last_ms, e->ev0, e->ev1));
  return LSK_OK;
}

// Teacher-forced scoring of many sequences on the wgmma prompt pass: sequence j is the branch
// ids[1 ..] of the one-id prefix ids[0], so it has no prefix rows, its view is its own pages in
// page-table order, and its rows are packed into shared 128-row chunks with the other sequences'
// (score_packed).  Every row's arithmetic is that of lsk_score on the same sequence's wgmma route.
int lsk_score_batch(lsk_engine* e, const int32_t* ids, const int32_t* offsets, int32_t n_seqs, int32_t exit_layer,
                    float* logprob_out, int32_t* greedy_out) {
  if (!e || !ids || !offsets || !logprob_out) return fail(LSK_ERR_INVALID, "null argument");
  const lsk_config& c = e->cfg;
  if (c.tp_size > 1)
    return fail(LSK_ERR_INVALID, "lsk_score_batch needs tp_size 1: tensor-parallel scoring is not supported");
  if (!e->pf_tc) return fail(LSK_ERR_INVALID, "lsk_score_batch needs the wgmma prompt pass, which this engine does not have");
  if (n_seqs < 1) return fail(LSK_ERR_INVALID, "n_seqs must be at least 1 (got %d)", n_seqs);
  if (exit_layer > c.n_layers) return fail(LSK_ERR_INVALID, "exit_layer %d > n_layers %d", exit_layer, c.n_layers);
  if (offsets[0] != 0) return fail(LSK_ERR_INVALID, "offsets[0] must be 0 (got %d)", offsets[0]);
  for (int j = 0; j < n_seqs; ++j) {
    if (offsets[j + 1] <= offsets[j])
      return fail(LSK_ERR_INVALID, "offsets are not increasing at sequence %d (%d, %d)", j, offsets[j], offsets[j + 1]);
    const int n = offsets[j + 1] - offsets[j];
    if (n < 2) return fail(LSK_ERR_INVALID, "sequence %d has %d id: scoring needs at least 2", j, n);
    if (n > c.max_ctx) return fail(LSK_ERR_CTX, "sequence %d of %d ids exceeds max_ctx %d", j, n, c.max_ctx);
    for (int i = offsets[j]; i < offsets[j + 1]; ++i)
      if (ids[i] < 0 || ids[i] >= c.vocab) return fail(LSK_ERR_INVALID, "sequence %d: token id %d out of range", j, ids[i]);
  }
  if (!lsk_weights_complete(e)) return fail(LSK_ERR_STATE, "weights not fully loaded");
  // sequence j's n_j - 1 results start at row offsets[j] - j
  std::vector<ScorePrefix> pre(n_seqs);
  for (int j = 0; j < n_seqs; ++j)
    pre[j] = {ids + offsets[j], 1, {{ids + offsets[j] + 1, offsets[j + 1] - offsets[j] - 1, offsets[j] - j}}};
  return score_packed(e, exit_layer <= 0 ? c.n_layers : exit_layer, pre, logprob_out, greedy_out);
}

// Teacher-forced scoring of branches that continue shared prefixes (score_packed): the results of
// branch b start at row branch_offsets[b], and are bit for bit those of lsk_score_batch on P + B.
int lsk_score_prefixed(lsk_engine* e, const int32_t* prefix_ids, const int32_t* prefix_offsets, int32_t n_prefixes,
                       const int32_t* branch_ids, const int32_t* branch_offsets, const int32_t* branch_prefix,
                       int32_t n_branches, int32_t exit_layer, float* logprob_out, int32_t* greedy_out) {
  if (!e || !prefix_ids || !prefix_offsets || !branch_ids || !branch_offsets || !branch_prefix || !logprob_out)
    return fail(LSK_ERR_INVALID, "null argument");
  const lsk_config& c = e->cfg;
  if (c.tp_size > 1)
    return fail(LSK_ERR_INVALID, "lsk_score_prefixed needs tp_size 1: tensor-parallel scoring is not supported");
  if (!e->pf_tc)
    return fail(LSK_ERR_INVALID, "lsk_score_prefixed needs the wgmma prompt pass, which this engine does not have");
  if (n_prefixes < 1) return fail(LSK_ERR_INVALID, "n_prefixes must be at least 1 (got %d)", n_prefixes);
  if (n_branches < 1) return fail(LSK_ERR_INVALID, "n_branches must be at least 1 (got %d)", n_branches);
  if (exit_layer > c.n_layers) return fail(LSK_ERR_INVALID, "exit_layer %d > n_layers %d", exit_layer, c.n_layers);
  auto check_parts = [&](const char* what, const int32_t* ids, const int32_t* off, int n) -> int {
    if (off[0] != 0) return fail(LSK_ERR_INVALID, "%s offsets[0] must be 0 (got %d)", what, off[0]);
    for (int j = 0; j < n; ++j) {
      if (off[j + 1] <= off[j])
        return fail(LSK_ERR_INVALID, "%s offsets are not increasing at %s %d (%d, %d): each needs at least 1 id", what,
                    what, j, off[j], off[j + 1]);
      for (int i = off[j]; i < off[j + 1]; ++i)
        if (ids[i] < 0 || ids[i] >= c.vocab) return fail(LSK_ERR_INVALID, "%s %d: token id %d out of range", what, j, ids[i]);
    }
    return LSK_OK;
  };
  TRY(check_parts("prefix", prefix_ids, prefix_offsets, n_prefixes));
  TRY(check_parts("branch", branch_ids, branch_offsets, n_branches));
  auto plen = [&](int p) { return prefix_offsets[p + 1] - prefix_offsets[p]; };
  auto blen = [&](int b) { return branch_offsets[b + 1] - branch_offsets[b]; };
  std::vector<ScorePrefix> pre(n_prefixes);   // each prefix with its branches, in input order
  for (int p = 0; p < n_prefixes; ++p) pre[p] = {prefix_ids + prefix_offsets[p], plen(p), {}};
  for (int b = 0; b < n_branches; ++b) {
    const int p = branch_prefix[b];
    if (p < 0 || p >= n_prefixes)
      return fail(LSK_ERR_INVALID, "branch %d: prefix index %d is outside [0, %d)", b, p, n_prefixes);
    if (plen(p) + blen(b) > c.max_ctx)
      return fail(LSK_ERR_CTX, "branch %d: prefix %d + branch = %d ids exceeds max_ctx %d", b, p, plen(p) + blen(b),
                  c.max_ctx);
    pre[p].br.push_back({branch_ids + branch_offsets[b], blen(b), branch_offsets[b]});
  }
  for (int p = 0; p < n_prefixes; ++p)
    if (pre[p].br.empty()) return fail(LSK_ERR_INVALID, "prefix %d has no branch", p);
  if (!lsk_weights_complete(e)) return fail(LSK_ERR_STATE, "weights not fully loaded");
  return score_packed(e, exit_layer <= 0 ? c.n_layers : exit_layer, pre, logprob_out, greedy_out);
}

// Teacher-forced scoring at several exits in one pass (score_sequence).
int lsk_score_exits(lsk_engine* e, const int32_t* ids, int32_t n, const int32_t* exits, int32_t n_exits,
                    const lsk_generation* sampling, float* logprob_out, int32_t* greedy_out, float* accept_out) {
  if (!e || !ids || !exits || !logprob_out) return fail(LSK_ERR_INVALID, "null argument");
  if (accept_out && !sampling) return fail(LSK_ERR_INVALID, "accept_out needs the sampling settings (sampling is NULL)");
  const lsk_config& c = e->cfg;
  if (c.tp_size > 1)
    return fail(LSK_ERR_INVALID, "lsk_score_exits needs tp_size 1: tensor-parallel scoring is not supported");
  if (n < 2) return fail(LSK_ERR_INVALID, "scoring needs at least 2 ids (got %d)", n);
  if (n > c.max_ctx) return fail(LSK_ERR_CTX, "sequence of %d ids exceeds max_ctx %d", n, c.max_ctx);
  if (n_exits < 1 || n_exits > LSK_MAX_EXITS)
    return fail(LSK_ERR_INVALID, "n_exits must be in [1, %d] (got %d)", LSK_MAX_EXITS, n_exits);
  for (int j = 0; j < n_exits; ++j) {
    if (exits[j] < 1 || exits[j] > c.n_layers)
      return fail(LSK_ERR_INVALID, "exits[%d] = %d is outside [1, n_layers %d]", j, exits[j], c.n_layers);
    if (j > 0 && exits[j] <= exits[j - 1])
      return fail(LSK_ERR_INVALID, "exits must be strictly increasing (exits[%d] = %d, exits[%d] = %d)", j - 1,
                  exits[j - 1], j, exits[j]);
  }
  for (int i = 0; i < n; ++i)
    if (ids[i] < 0 || ids[i] >= c.vocab) return fail(LSK_ERR_INVALID, "token id %d out of range", ids[i]);
  if (accept_out) {
    if (sampling->sample != 1 || !(sampling->temperature > 0.f))
      return fail(LSK_ERR_INVALID, "accept_out needs sampling settings with sample = 1 and temperature > 0");
    if (sampling->no_repeat_ngram_size != 0)
      return fail(LSK_ERR_INVALID, "accept_out does not model the n-gram ban: no_repeat_ngram_size must be 0");
    if (exits[n_exits - 1] != c.n_layers)
      return fail(LSK_ERR_INVALID, "accept_out needs the last exit at full depth (%d, got %d)", c.n_layers,
                  exits[n_exits - 1]);
  }
  if (!lsk_weights_complete(e)) return fail(LSK_ERR_STATE, "weights not fully loaded");
  return score_sequence(e, ids, n, exits, n_exits, sampling, logprob_out, greedy_out, accept_out);
}

int lsk_kv_len(const lsk_engine* e, int32_t* len_out) {
  if (!e || !len_out) return fail(LSK_ERR_INVALID, "null argument");
  *len_out = e->host_len;
  return LSK_OK;
}

int lsk_debug_set_page_table(lsk_engine* e, const int32_t* pages, int32_t n) {
  if (!e || !pages || n != e->n_pages) return fail(LSK_ERR_INVALID, "page table must have %d entries", e ? e->n_pages : 0);
  std::vector<char> seen(n, 0);
  for (int i = 0; i < n; ++i) {
    if (pages[i] < 0 || pages[i] >= n || seen[pages[i]]) return fail(LSK_ERR_INVALID, "page table is not a permutation");
    seen[pages[i]] = 1;
  }
  CU(cudaMemcpyAsync(e->page_table, pages, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  CU(cudaStreamSynchronize(e->stream));
  e->page_table_host.assign(pages, pages + n);
  return LSK_OK;
}

int lsk_debug_read(lsk_engine* e, int32_t what, int32_t layer, int64_t index, float* dst, int64_t n) {
  if (!e || !dst) return fail(LSK_ERR_INVALID, "null argument");
  CU(cudaStreamSynchronize(e->stream));
  if (what == LSK_DBG_HIDDEN) {
    if (n > (int64_t)kMaxRows * e->cfg.hidden) return fail(LSK_ERR_INVALID, "too many floats");
    CU(cudaMemcpy(dst, e->hidden, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return LSK_OK;
  }
  if (what == LSK_DBG_PROBS_DRAFT || what == LSK_DBG_PROBS_VERIFY) {
    const float* src = what == LSK_DBG_PROBS_DRAFT ? e->probs_d : e->probs_v;
    if (!src) return fail(LSK_ERR_STATE, "no sampling generation has run");
    if (n > (int64_t)kMaxRows * e->cfg.vocab) return fail(LSK_ERR_INVALID, "too many floats");
    CU(cudaMemcpy(dst, src, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return LSK_OK;
  }
  if (what == LSK_DBG_RESIDUAL) {
    if (!e->samp_scratch) return fail(LSK_ERR_STATE, "no sampling generation has run");
    if (n > (int64_t)e->cfg.vocab) return fail(LSK_ERR_INVALID, "too many floats");
    CU(cudaMemcpy(dst, e->samp_scratch, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return LSK_OK;
  }
  if (what == LSK_DBG_LOGITS) {
    if (!e->logits) return fail(LSK_ERR_STATE, "engine created without LSK_FLAG_KEEP_LOGITS");
    if (n > (int64_t)kMaxRows * e->vocab_l_pad) return fail(LSK_ERR_INVALID, "too many floats");
    CU(cudaMemcpy(dst, e->logits, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return LSK_OK;
  }
  if (what == LSK_DBG_ARGMAX) {
    // the engine's greedy choice per row of the last LM head: its candidates merged by the same
    // fixed-order reduction as the accept kernels (reduce_candidates / rank_best_kernel)
    if (!e->cur_cand_val || !e->cur_cand_idx) return fail(LSK_ERR_STATE, "no LM head has run");
    if (n < 2 || n % 2 || n > 2 * kMaxRows) return fail(LSK_ERR_INVALID, "n = 2 * rows (value, index), rows <= %d", kMaxRows);
    const int rows = (int)(n / 2);
    rank_best_kernel<<<1, 32 * kMaxRows, 0, e->stream>>>(cand_val_ptr(e), cand_idx_ptr(e), n_cand(e), rows,
                                                          e->rank_val, e->rank_idx);
    CU(cudaGetLastError());
    float val[kMaxRows];
    int idx[kMaxRows];
    CU(cudaMemcpyAsync(val, e->rank_val, (size_t)rows * 4, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaMemcpyAsync(idx, e->rank_idx, (size_t)rows * 4, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    for (int r = 0; r < rows; ++r) { dst[2 * r] = val[r]; dst[2 * r + 1] = (float)idx[r]; }
    return LSK_OK;
  }
  if (what == LSK_DBG_KROW || what == LSK_DBG_VROW) {
    // n = count * head_dim: `count` consecutive positions of one kv head, pos0 .. pos0 + count - 1
    const int hd = e->cfg.head_dim;
    if (layer < 0 || layer >= e->cfg.n_layers || n < hd || n % hd)
      return fail(LSK_ERR_INVALID, "bad layer / n (a multiple of head_dim floats: one row per position)");
    const int64_t head = index / e->cfg.max_ctx, pos0 = index % e->cfg.max_ctx, count = n / hd;
    if (head >= e->kv_heads_l) return fail(LSK_ERR_INVALID, "bad kv head");
    if (pos0 + count > e->cfg.max_ctx) return fail(LSK_ERR_INVALID, "rows %lld .. %lld cross max_ctx", (long long)pos0,
                                                   (long long)(pos0 + count - 1));
    std::vector<int> pt(e->n_pages);
    CU(cudaMemcpy(pt.data(), e->page_table, pt.size() * 4, cudaMemcpyDeviceToHost));
    const __nv_bfloat16* pool = (what == LSK_DBG_KROW ? e->kpool : e->vpool) + (size_t)layer * e->pool_layer_elems;
    // the token rows of one (page, kv head) block are contiguous; inside a row the 16-byte chunks
    // are swizzled (common.cuh: kv_elem_offset): one copy per page, then unswizzle row by row
    std::vector<__nv_bfloat16> tmp((size_t)kPageTokens * hd);
    for (int64_t p = pos0; p < pos0 + count;) {
      const int tok0 = (int)(p & 63);
      const int rows = (int)std::min<int64_t>(kPageTokens - tok0, pos0 + count - p);
      const __nv_bfloat16* src = pool + kv_elem_offset(hd, pt[p >> 6], e->kv_heads_l, (int)head, tok0, 0) -
                                 (size_t)(kv_chunk_swizzle(hd, tok0) * 8);
      CU(cudaMemcpy(tmp.data(), src, (size_t)rows * hd * 2, cudaMemcpyDeviceToHost));
      for (int r = 0; r < rows; ++r) {
        const int swz = kv_chunk_swizzle(hd, tok0 + r);
        float* d = dst + (size_t)(p - pos0 + r) * hd;
        for (int i = 0; i < hd; ++i) d[i] = __bfloat162float(tmp[(size_t)r * hd + (((i >> 3) ^ swz) << 3) + (i & 7)]);
      }
      p += rows;
    }
    return LSK_OK;
  }
  return fail(LSK_ERR_INVALID, "unknown debug selector %d", what);
}

// algorithmic bytes (SURVEY.md §8(d)), per GPU: packed weights streamed once per layer call,
// LM head once per head call, KV entries of the visible context once per layer call.
static double layer_weight_bytes(const lsk_engine* e) {
  const double h = e->cfg.hidden;
  return 2.0 * ((double)(e->q_rows + 2 * e->kv_rows) * h + h * e->q_rows + 3.0 * e->inter_l * h);
}
int lsk_round_bytes(const lsk_engine* e, int32_t d, int32_t ctx, double* out) {
  if (!e || !out) return fail(LSK_ERR_INVALID, "null argument");
  const int E = e->gen.exit_layer, L = e->cfg.n_layers;
  const double wl = layer_weight_bytes(e), wh = 2.0 * e->vocab_l * e->cfg.hidden;
  const double kv_tok = 2.0 * 2.0 * e->kv_rows;
  const double layer_calls = (double)(d + 1) * E + (L - E);
  *out = layer_calls * wl + (d + 1) * wh + layer_calls * ctx * kv_tok;
  return LSK_OK;
}
int lsk_ar_bytes(const lsk_engine* e, int32_t ctx, double* out) {
  if (!e || !out) return fail(LSK_ERR_INVALID, "null argument");
  const int nl = (e->gen.exit_layer > 0) ? e->gen.exit_layer : e->cfg.n_layers;
  *out = nl * (layer_weight_bytes(e) + ctx * 2.0 * 2.0 * e->kv_rows) + 2.0 * e->vocab_l * e->cfg.hidden;
  return LSK_OK;
}
int lsk_launch_count(const lsk_engine* e, int64_t* out) {
  if (!e || !out) return fail(LSK_ERR_INVALID, "null argument");
  *out = e->launches;
  return LSK_OK;
}
int lsk_last_device_ms(const lsk_engine* e, float* out) {
  if (!e || !out) return fail(LSK_ERR_INVALID, "null argument");
  *out = e->last_ms;
  return LSK_OK;
}

// Host-side schedule of one skinny GEMM (no GPU needed): what the launcher would do for
// y[m, n_rows] = x[m, K] . W^T with the given prologue / epilogue kinds on `sm_count` SMs.
int lsk_plan_gemm(int64_t n_rows, int64_t K, int32_t m, int32_t pro, int32_t epi, int32_t sm_count,
                  lsk_gemm_plan* out) {
  if (!out || n_rows % 16 || K % 32 || m < 1 || m > kMaxRows || sm_count < 1)
    return fail(LSK_ERR_INVALID, "bad plan query");
  const GemmPlan p = make_plan((int)n_rows, (int)K);
  const int NT = m <= 8 ? 1 : 2;
  const GemmSched sc = plan_sched(NT, m, pro, epi, p, sm_count);
  out->ok = sc.ok ? 1 : 0;
  out->nt = NT;
  out->tiles_per_pass = sc.tpp;
  out->n_chunks = sc.n_chunks;
  out->chunk_cols = sc.kc_sbs * 32;
  out->ring_stages = sc.n_stages;
  out->stage_bytes = kStageBytes;
  out->grid = sc.grid;
  out->block = kGemmThreads;
  out->smem_bytes = (int64_t)sc.smem;
  out->smem_limit = kSmemMax;
  out->n_tiles = p.n_tiles;
  return LSK_OK;
}

// Host-side launch plan of the attention kernel for `m` query rows (no GPU needed).
int lsk_plan_attention(int32_t head_dim, int32_t n_heads, int32_t n_kv_heads_local, int32_t m, int32_t sm_count,
                       lsk_attn_plan* out) {
  if (!out || (head_dim != 32 && head_dim != 64 && head_dim != 128) || n_heads < 1 || n_kv_heads_local < 1 ||
      n_heads % n_kv_heads_local || m < 1 || sm_count < 1)
    return fail(LSK_ERR_INVALID, "bad attention plan query");
  const int group = n_heads / n_kv_heads_local;
  const int splits = attn_default_splits(sm_count, n_kv_heads_local);
  const AttnLaunchPlan p = plan_attention_launch(head_dim, group, m, n_kv_heads_local, splits, kAttnMaxStages, sm_count);
  out->ok = (p.ok && attn_layout_smem(head_dim, group) <= (size_t)kSmemMax) ? 1 : 0;
  out->n_splits = splits;
  out->ring_stages = p.stages;
  out->grid = n_kv_heads_local * splits;
  out->block = kAttnThreads;
  out->row_blocks = (group * m + 15) / 16;
  out->kv_refetched_per_row_block = p.sp.reload_per_rb;
  out->smem_bytes = (int64_t)p.smem;
  out->smem_limit = kSmemMax;
  return LSK_OK;
}

// ---- stand-alone kernel entry points (unit tests / micro-benchmarks) ---------------------
int lsk_test_pack(const void* w, int64_t n, int64_t k, void* packed) {
  if (!w || !packed || n % 16 || k % 32) return fail(LSK_ERR_INVALID, "need n %% 16 == 0 and k %% 32 == 0");
  const int64_t pairs = n * (k / 2);
  int blocks = (int)((pairs + 255) / 256);
  if (blocks > 4096) blocks = 4096;
  pack_rows_kernel<<<blocks, 256>>>((const __nv_bfloat16*)w, k, 0, 0, n, k, (__nv_bfloat16*)packed, 0, MAP_PLAIN, k, 128);
  CU(cudaGetLastError());
  CU(cudaDeviceSynchronize());
  return LSK_OK;
}

// The launch plumbing of an engine for one stand-alone test call: the SM count and a stream for
// launches and zero fills.  The engine's destructor releases the stream, the events and every buffer
// on every return path.
static int test_engine(lsk_engine& t) {
  int dev = 0;
  CU(cudaGetDevice(&dev));
  CU(cudaDeviceGetAttribute(&t.sm_count, cudaDevAttrMultiProcessorCount, dev));
  CU(cudaStreamCreateWithFlags(&t.stream, cudaStreamNonBlocking));
  t.mem.stream = t.stream;
  return LSK_OK;
}

int lsk_test_gemm(const void* packed, int64_t n, int64_t k, const void* x, int32_t m, float* y,
                  int32_t iters, float* avg_ms) {
  if (!packed || !x || !y || n % 16 || k % 32 || m < 1 || m > kMaxRows) return fail(LSK_ERR_INVALID, "bad gemm test shape");
  lsk_engine tmp;   // only the launch plumbing is used
  TRY(test_engine(tmp));
  GemmPlan p = make_plan((int)n, (int)k);
  GemmArgs a{};
  a.W = (const uint4*)packed;
  a.M = m;
  a.x_bf16 = (const __nv_bfloat16*)x; a.xb_ld = (int)k;
  a.out_f32 = y; a.out_ld = (int)n;
  CU(cudaEventCreate(&tmp.ev0));
  CU(cudaEventCreate(&tmp.ev1));
  TRY((launch_gemm<PRO_BF16, EPI_STORE>(&tmp, p, a)));   // warm-up + result
  CU(cudaStreamSynchronize(tmp.stream));
  if (iters > 0) {
    CU(cudaEventRecord(tmp.ev0, tmp.stream));
    for (int i = 0; i < iters; ++i) TRY((launch_gemm<PRO_BF16, EPI_STORE>(&tmp, p, a)));
    CU(cudaEventRecord(tmp.ev1, tmp.stream));
    CU(cudaEventSynchronize(tmp.ev1));
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, tmp.ev0, tmp.ev1));
    if (avg_ms) *avg_ms = ms / iters;
  }
  return LSK_OK;
}

// natural K/V [kv_head][ctx][hd] -> the engine's paged pool layout (one layer)
__global__ void paginate_kv_kernel(const __nv_bfloat16* __restrict__ src, int n_kv, int ctx, int kHeadDim,
                                   const int* __restrict__ page_table, __nv_bfloat16* __restrict__ pool) {
  const int64_t total = (int64_t)n_kv * ctx * (kHeadDim / 8);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % (kHeadDim / 8));
    const int pos = (int)((i / (kHeadDim / 8)) % ctx);
    const int h = (int)(i / ((int64_t)(kHeadDim / 8) * ctx));
    const uint4 v = *reinterpret_cast<const uint4*>(src + ((size_t)h * ctx + pos) * kHeadDim + ch * 8);
    const int page = page_table[pos >> 6];
    *reinterpret_cast<uint4*>(pool + kv_elem_offset(kHeadDim, page, n_kv, h, pos & 63, ch * 8)) = v;
  }
}

// canonical operand rows [m][cols] (common.cuh: canon_offset) -> natural bf16 [m][cols]
__global__ void uncanon_rows_kernel(const unsigned char* __restrict__ src, int m, int cols,
                                    __nv_bfloat16* __restrict__ dst) {
  const int chunks = cols >> 3;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m * chunks; i += gridDim.x * blockDim.x) {
    const int row = i / chunks, k = (i % chunks) * 8;
    *reinterpret_cast<uint4*>(dst + (size_t)row * cols + k) = *reinterpret_cast<const uint4*>(src + canon_offset(row, k));
  }
}

// Stand-alone attention (unit test / micro-benchmark): m query rows at positions ctx-m .. ctx-1
// attend causally to keys 0 .. ctx-1.  q / out: [m][n_heads * head_dim] bf16; k / v: natural
// [n_kv_heads][ctx][head_dim] bf16 (k already rotated); page_perm (host, may be null) permutes the
// logical -> physical page map.  Same launch paths as the engine: m <= 16 rows are one decode block
// (base length ctx - m); 16 < m <= 128 rows are one prompt-pass chunk at c0 = ctx - m
// (launch_prompt_attention: base length 0, canonical output, unpacked here to [m][n_heads * head_dim]).
int lsk_test_attn(const void* q, const void* k, const void* v, int32_t n_heads, int32_t n_kv_heads,
                  int32_t head_dim, int32_t ctx, int32_t m, int32_t n_splits, const int32_t* page_perm, void* out,
                  int32_t iters, float* avg_ms) {
  const int kHeadDim = head_dim;
  if (head_dim != 32 && head_dim != 64 && head_dim != 128) return fail(LSK_ERR_INVALID, "head_dim %d unsupported", head_dim);
  if (!q || !k || !v || !out || n_heads < 1 || n_kv_heads < 1 || n_heads % n_kv_heads || ctx < m || m < 1 ||
      m > kPfTokens || n_splits < 1 || n_splits > 8)
    return fail(LSK_ERR_INVALID, "bad attention test shape");
  const bool prompt = m > kMaxRows;
  lsk_engine tmp;
  TRY(test_engine(tmp));
  tmp.n_splits = n_splits;
  TRY(alloc_attn_partials(&tmp, attn_bufs(n_kv_heads, n_heads / n_kv_heads, head_dim, n_splits, m)));
  const int n_pages = (ctx + kPageTokens - 1) / kPageTokens;
  const size_t pool_elems = (size_t)n_pages * n_kv_heads * kPageTokens * kHeadDim;
  std::vector<int> pth(n_pages);
  for (int i = 0; i < n_pages; ++i) pth[i] = page_perm ? page_perm[i] : i;
  for (int i = 0; i < n_pages; ++i)
    if (pth[i] < 0 || pth[i] >= n_pages) return fail(LSK_ERR_INVALID, "bad page permutation");
  __nv_bfloat16 *kp = nullptr, *vp = nullptr;
  int *pt = nullptr, *len = nullptr;
  unsigned char* canon = nullptr;
  TRY(tmp.mem.alloc(&kp, {pool_elems * 2, MEM_KV_POOL}, true));
  TRY(tmp.mem.alloc(&vp, {pool_elems * 2, MEM_KV_POOL}, true));
  TRY(tmp.mem.alloc(&pt, {(size_t)n_pages * 4, MEM_SCRATCH}));
  TRY(tmp.mem.alloc(&len, {4, MEM_SCRATCH}));
  const int base = prompt ? 0 : ctx - m;
  const int q_cols = n_heads * kHeadDim;
  if (prompt) TRY(tmp.mem.alloc(&canon, {(size_t)((q_cols + 63) / 64) * kCanonStageBytes, MEM_SCRATCH}, true));
  CU(cudaMemcpyAsync(pt, pth.data(), (size_t)n_pages * 4, cudaMemcpyHostToDevice, tmp.stream));
  CU(cudaMemcpyAsync(len, &base, 4, cudaMemcpyHostToDevice, tmp.stream));
  paginate_kv_kernel<<<tmp.sm_count * 4, 256, 0, tmp.stream>>>((const __nv_bfloat16*)k, n_kv_heads, ctx, head_dim, pt, kp);
  paginate_kv_kernel<<<tmp.sm_count * 4, 256, 0, tmp.stream>>>((const __nv_bfloat16*)v, n_kv_heads, ctx, head_dim, pt, vp);
  CU(cudaGetLastError());
  AttnArgs a{};
  a.q = (const __nv_bfloat16*)q; a.q_ld = q_cols;
  a.out = (__nv_bfloat16*)out; a.out_ld = q_cols;
  a.kpool = kp; a.vpool = vp; a.page_table = pt; a.base_len = len; a.pos_off = 0; a.M = m;
  a.group = n_heads / n_kv_heads; a.n_kv_heads = n_kv_heads; a.n_splits = n_splits;
  a.scale = 1.0f / sqrtf((float)kHeadDim);
  auto run = [&]() -> int {
    if (!prompt) return launch_attention(&tmp, a, head_dim);
    return launch_prompt_attention(&tmp, (const __nv_bfloat16*)q, q_cols, canon, kp, vp, pt, len, ctx - m, m,
                                   n_heads / n_kv_heads, n_kv_heads, head_dim);
  };
  TRY(run());
  if (prompt) {
    uncanon_rows_kernel<<<tmp.sm_count, 256, 0, tmp.stream>>>(canon, m, q_cols, (__nv_bfloat16*)out);
    CU(cudaGetLastError());
  }
  CU(cudaStreamSynchronize(tmp.stream));
  if (iters > 0) {
    CU(cudaEventCreate(&tmp.ev0));
    CU(cudaEventCreate(&tmp.ev1));
    CU(cudaEventRecord(tmp.ev0, tmp.stream));
    for (int i = 0; i < iters; ++i) TRY(run());
    CU(cudaEventRecord(tmp.ev1, tmp.stream));
    CU(cudaEventSynchronize(tmp.ev1));
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, tmp.ev0, tmp.ev1));
    if (avg_ms) *avg_ms = ms / iters;
  }
  return LSK_OK;
}

// Stand-alone attention of a batched round: attn_piece_kernel's sequence grid launched as
// enqueue_layer launches it for lsk_round_batch.  Sequence s has seq_rows query rows at positions
// ctx[s] - seq_rows .. ctx[s] - 1 (chunk rows s * seq_rows ..), its committed length in a DevState-strided
// array, and its keys k / v [n_seqs][n_kv_heads][slot_positions][head_dim] in logical pages
// [s * P, (s + 1) * P) of one pool, P = slot_positions / 64; page_perm (host, may be null) permutes the
// logical -> physical page map of all n_seqs * P pages.
int lsk_test_attn_seqs(const void* q, const void* k, const void* v, int32_t n_heads, int32_t n_kv_heads,
                       int32_t head_dim, int32_t n_seqs, int32_t seq_rows, const int32_t* ctx,
                       int32_t slot_positions, int32_t n_splits, const int32_t* page_perm, void* out) {
  if (head_dim != 32 && head_dim != 64 && head_dim != 128) return fail(LSK_ERR_INVALID, "head_dim %d unsupported", head_dim);
  if (!q || !k || !v || !out || !ctx || n_heads < 1 || n_kv_heads < 1 || n_heads % n_kv_heads || n_seqs < 1 ||
      seq_rows < 1 || n_seqs * seq_rows > kMaxRows || n_splits < 1 || n_splits > kMaxSplits)
    return fail(LSK_ERR_INVALID, "bad batched attention test shape");
  if (slot_positions < kPageTokens || slot_positions % kPageTokens)
    return fail(LSK_ERR_INVALID, "slot_positions %d is not a positive multiple of %d", slot_positions, kPageTokens);
  for (int s = 0; s < n_seqs; ++s)
    if (ctx[s] < seq_rows || ctx[s] > slot_positions)
      return fail(LSK_ERR_INVALID, "sequence %d: ctx %d outside [seq_rows %d, slot %d]", s, ctx[s], seq_rows, slot_positions);
  const int P = slot_positions / kPageTokens, n_pages = n_seqs * P;
  std::vector<int> pth(n_pages);
  std::vector<char> seen(n_pages, 0);
  for (int i = 0; i < n_pages; ++i) {
    pth[i] = page_perm ? page_perm[i] : i;
    if (pth[i] < 0 || pth[i] >= n_pages || seen[pth[i]]) return fail(LSK_ERR_INVALID, "bad page permutation");
    seen[pth[i]] = 1;
  }
  lsk_engine tmp;
  TRY(test_engine(tmp));
  tmp.n_splits = n_splits;
  const int group = n_heads / n_kv_heads, rows = n_seqs * seq_rows;
  TRY(alloc_attn_partials(&tmp, attn_bufs(n_kv_heads, group, head_dim, n_splits, rows)));
  TRY(tmp.mem.alloc(&tmp.batch_arrive, {(size_t)n_seqs * n_kv_heads * 4, MEM_SCRATCH}, true));
  // committed lengths DevState::len apart, the fields between them zero, as lsk_round_batch reads them
  const int len_stride = (int)(sizeof(DevState) / sizeof(int));
  std::vector<int> lenh((size_t)n_seqs * len_stride, 0);
  for (int s = 0; s < n_seqs; ++s) lenh[(size_t)s * len_stride] = ctx[s] - seq_rows;
  const size_t slot_elems = (size_t)n_kv_heads * slot_positions * head_dim;
  __nv_bfloat16 *kp = nullptr, *vp = nullptr;
  int *pt = nullptr, *len = nullptr;
  TRY(tmp.mem.alloc(&kp, {slot_elems * n_seqs * 2, MEM_KV_POOL}, true));
  TRY(tmp.mem.alloc(&vp, {slot_elems * n_seqs * 2, MEM_KV_POOL}, true));
  TRY(tmp.mem.alloc(&pt, {(size_t)n_pages * 4, MEM_SCRATCH}));
  TRY(tmp.mem.alloc(&len, {lenh.size() * 4, MEM_SCRATCH}));
  CU(cudaMemcpyAsync(pt, pth.data(), (size_t)n_pages * 4, cudaMemcpyHostToDevice, tmp.stream));
  CU(cudaMemcpyAsync(len, lenh.data(), lenh.size() * 4, cudaMemcpyHostToDevice, tmp.stream));
  for (int s = 0; s < n_seqs; ++s) {
    const size_t src = (size_t)s * slot_elems;
    paginate_kv_kernel<<<tmp.sm_count * 4, 256, 0, tmp.stream>>>((const __nv_bfloat16*)k + src, n_kv_heads,
                                                                  slot_positions, head_dim, pt + s * P, kp);
    paginate_kv_kernel<<<tmp.sm_count * 4, 256, 0, tmp.stream>>>((const __nv_bfloat16*)v + src, n_kv_heads,
                                                                  slot_positions, head_dim, pt + s * P, vp);
  }
  CU(cudaGetLastError());
  const int q_cols = n_heads * head_dim;
  AttnArgs a{};
  a.q = (const __nv_bfloat16*)q; a.q_ld = q_cols;
  a.out = (__nv_bfloat16*)out; a.out_ld = q_cols;
  a.kpool = kp; a.vpool = vp; a.page_table = pt; a.base_len = len; a.pos_off = 0; a.M = seq_rows;
  a.group = group; a.n_kv_heads = n_kv_heads; a.n_splits = n_splits;
  a.scale = 1.0f / sqrtf((float)head_dim);
  const AttnPieces pz{nullptr, (group * rows + 15) / 16 * 16, seq_rows, len_stride, P};
  TRY(launch_attention(&tmp, a, head_dim, &pz, n_seqs));
  CU(cudaStreamSynchronize(tmp.stream));
  return LSK_OK;
}

// wgmma LM head on caller-provided device buffers (unit test / micro-benchmark of lmhead_tc.cuh)
int lsk_test_lmhead_tc(const void* w, int64_t n, int64_t k, const float* x, const void* norm_w, float eps,
                       int32_t m, float* logits, float* best_val, int32_t* best_idx, int32_t iters,
                       float* avg_ms) {
  if (!w || !x || !norm_w || !best_val || !best_idx || n < 1 || k % kTcStageK || m < 1 || m > kMaxRows)
    return fail(LSK_ERR_INVALID, "bad wgmma LM-head test shape");
  int stages = kTcMaxStages;
  while (stages >= 3 && lmhead_tc_smem_bytes((int)k, stages) > (size_t)kSmemMax) --stages;
  if (stages < 3) return fail(LSK_ERR_INVALID, "hidden %lld does not fit the wgmma LM head", (long long)k);
  lsk_engine tmp;   // holds the buffers and events; the kernels run on the legacy default stream
  int dev = 0, sms = 0;
  CU(cudaGetDevice(&dev));
  CU(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int n_tiles = (int)((n + kTcTileRows - 1) / kTcTileRows);
  const int waves = (n_tiles + sms - 1) / sms;
  const int grid = (n_tiles + waves - 1) / waves;
  unsigned char* canon = nullptr;
  float* cval = nullptr;
  int* cidx = nullptr;
  TRY(tmp.mem.alloc(&canon, {(size_t)n_tiles * kTcTileRows * k * 2, MEM_LM_HEAD}));
  TRY(tmp.mem.alloc(&cval, {(size_t)grid * kMaxRows * 4, MEM_SCRATCH}));
  TRY(tmp.mem.alloc(&cidx, {(size_t)grid * kMaxRows * 4, MEM_SCRATCH}));
  pack_canonical_kernel<<<sms * 8, 256>>>((const __nv_bfloat16*)w, k, 0, n, k, reinterpret_cast<uint4*>(canon), n_tiles);
  CU(cudaGetLastError());
  CU(cudaFuncSetAttribute(lmhead_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemMax));
  LmHeadTcArgs t{};
  t.W = canon; t.n_tiles = n_tiles; t.K = (int)k; t.M = m; t.n_stages = stages;
  t.x_f32 = x; t.x_ld = (int)k; t.norm_w = (const __nv_bfloat16*)norm_w; t.eps = eps;
  t.logits = logits; t.logits_ld = (int)n; t.n_valid_rows = (int)n; t.vocab_off = 0;
  t.part_val = cval; t.part_idx = cidx;
  const size_t smem = lmhead_tc_smem_bytes((int)k, stages);
  CU(cudaEventCreate(&tmp.ev0));
  CU(cudaEventCreate(&tmp.ev1));
  lmhead_tc_kernel<<<grid, kTcThreads, smem>>>(t);
  CU(cudaGetLastError());
  rank_best_kernel<<<1, 256>>>(cval, cidx, grid, m, best_val, best_idx);
  CU(cudaGetLastError());
  CU(cudaDeviceSynchronize());
  if (iters > 0) {
    CU(cudaEventRecord(tmp.ev0));
    for (int i = 0; i < iters; ++i) lmhead_tc_kernel<<<grid, kTcThreads, smem>>>(t);
    CU(cudaEventRecord(tmp.ev1));
    CU(cudaEventSynchronize(tmp.ev1));
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, tmp.ev0, tmp.ev1));
    if (avg_ms) *avg_ms = ms / iters;
  }
  return LSK_OK;
}

// the scoring kernel alone (unit test): logits [rows][ld] fp32, the first `vocab` columns valid
int lsk_test_logprob(const float* logits, int32_t rows, int32_t vocab, int32_t ld, const int32_t* targets,
                     float* logprob, int32_t* greedy) {
  if (!logits || !targets || !logprob || rows < 1 || vocab < 1 || ld < vocab)
    return fail(LSK_ERR_INVALID, "bad log-probability test shape");
  logprob_rows_kernel<<<rows, kLogprobThreads>>>(logits, ld, vocab, (const int*)targets, logprob, (int*)greedy);
  CU(cudaGetLastError());
  CU(cudaDeviceSynchronize());
  return LSK_OK;
}

// the acceptance kernels alone (unit test): draft and full-depth logits [rows][ld] fp32, the first
// `vocab` columns valid; accept[r] = sum_v min of the two warped rows r
int lsk_test_accept(const float* logits_draft, const float* logits_verify, int32_t rows, int32_t vocab, int32_t ld,
                    const lsk_generation* sampling, float* accept) {
  if (!logits_draft || !logits_verify || !sampling || !accept || rows < 1 || vocab < 1 || ld < vocab)
    return fail(LSK_ERR_INVALID, "bad acceptance test shape");
  if (!(sampling->temperature > 0.f)) return fail(LSK_ERR_INVALID, "acceptance test needs temperature > 0");
  const WarpParams wp{sampling->temperature, sampling->top_k, sampling->top_p};
  DeviceMem mem;
  float* buf = nullptr;
  TRY(mem.alloc(&buf, {(size_t)2 * rows * vocab * 4, MEM_SCRATCH}));
  warp_rows_kernel<<<rows, kSampleThreads>>>(logits_draft, ld, vocab, wp, buf);
  accept_prob_kernel<<<rows, kSampleThreads>>>(logits_verify, ld, vocab, wp, buf, (size_t)0, 1,
                                               buf + (size_t)rows * vocab, accept, (size_t)0);
  CU(cudaGetLastError());
  CU(cudaDeviceSynchronize());
  return LSK_OK;
}

}  // extern "C"

static GenParams gen_params_of(const lsk_generation& g) {
  GenParams gp{};
  gp.n_eos = g.n_eos;
  for (int i = 0; i < g.n_eos; ++i) gp.eos[i] = g.eos_ids[i];
  gp.sample = 1;
  gp.temperature = g.temperature;
  gp.top_k = g.top_k;
  gp.top_p = g.top_p;
  gp.seed = g.seed;
  return gp;
}

extern "C" {

// the inverse-CDF draw alone (unit test): one CTA per u
int lsk_test_draw(const float* weights, int32_t vocab, const float* u, int32_t n, int32_t* picks) {
  if (!weights || !u || !picks || vocab < 1 || n < 1) return fail(LSK_ERR_INVALID, "bad draw test shape");
  draw_index_kernel<<<n, kSampleThreads>>>(weights, vocab, u, (int*)picks);
  CU(cudaGetLastError());
  CU(cudaDeviceSynchronize());
  return LSK_OK;
}

// the generation sampling kernel alone (unit test): step s of n_steps runs with step_count = step0 + s
int lsk_test_sample(const float* logits, int32_t rows, int32_t vocab, int32_t ld, const lsk_generation* sampling,
                    int32_t step0, int32_t n_steps, int32_t purpose, int32_t row_base, float* probs,
                    int32_t* tokens) {
  if (!logits || !sampling || !probs || !tokens || rows < 1 || vocab < 1 || ld < vocab || n_steps < 1 || step0 < 0)
    return fail(LSK_ERR_INVALID, "bad sampling test shape");
  if (!(sampling->temperature > 0.f)) return fail(LSK_ERR_INVALID, "sampling test needs temperature > 0");
  const GenParams gp = gen_params_of(*sampling);
  std::vector<DevState> states((size_t)n_steps);
  for (int s = 0; s < n_steps; ++s) {
    states[s] = DevState{};
    states[s].step_count = step0 + s;
  }
  DeviceMem mem;
  GenParams* gp_dev = nullptr;
  DevState* st_dev = nullptr;
  float* later = nullptr;                // the warped rows of steps > 0 (the same values again)
  TRY(mem.alloc(&gp_dev, {sizeof(GenParams), MEM_SCRATCH}));
  TRY(mem.alloc(&st_dev, {(size_t)n_steps * sizeof(DevState), MEM_SCRATCH}));
  if (n_steps > 1) TRY(mem.alloc(&later, {(size_t)rows * vocab * 4, MEM_SCRATCH}));
  CU(cudaMemcpy(gp_dev, &gp, sizeof(gp), cudaMemcpyHostToDevice));
  CU(cudaMemcpy(st_dev, states.data(), states.size() * sizeof(DevState), cudaMemcpyHostToDevice));
  for (int s = 0; s < n_steps; ++s)
    warp_and_sample_kernel<<<rows, kSampleThreads>>>(logits, ld, vocab, gp_dev, st_dev + s, s == 0 ? probs : later,
                                                     (int*)tokens + (size_t)s * rows, purpose, row_base);
  CU(cudaGetLastError());
  CU(cudaDeviceSynchronize());
  return LSK_OK;
}

// the sampled accept / resample kernel alone (unit test): every step starts from a fresh state
int lsk_test_accept_sample(const float* p_draft, const float* p_verify, int32_t vocab, int32_t d,
                           const int32_t* draft_ids, const int32_t* verified_ids, const lsk_generation* sampling,
                           int32_t kv_len0, int32_t step0, int32_t n_steps, lsk_round_out* out, float* residual) {
  if (!p_draft || !p_verify || !draft_ids || !verified_ids || !sampling || !out || !residual || vocab < 1 ||
      d < 1 || d > LSK_MAX_SPEC || n_steps < 1 || step0 < 0 || kv_len0 < 0 || sampling->n_eos < 0 ||
      sampling->n_eos > LSK_MAX_EOS)
    return fail(LSK_ERR_INVALID, "bad accept-sample test shape");
  for (size_t i = 0; i < (size_t)n_steps * d; ++i)
    if (draft_ids[i] < 0 || draft_ids[i] >= vocab) return fail(LSK_ERR_INVALID, "draft id outside the vocabulary");
  const GenParams gp = gen_params_of(*sampling);
  std::vector<DevState> states((size_t)n_steps);
  for (int s = 0; s < n_steps; ++s) {
    DevState& st = states[s];
    st = DevState{};
    st.len = kv_len0;
    st.step_count = step0 + s;
    for (int i = 0; i < d; ++i) st.tok[1 + i] = draft_ids[(size_t)s * d + i];
    for (int i = 0; i <= d; ++i) st.verified[i] = verified_ids[(size_t)s * (d + 1) + i];
  }
  DeviceMem mem;
  GenParams* gp_dev = nullptr;
  DevState* st_dev = nullptr;
  RoundResult* res_dev = nullptr;
  TRY(mem.alloc(&gp_dev, {sizeof(GenParams), MEM_SCRATCH}));
  TRY(mem.alloc(&st_dev, {(size_t)n_steps * sizeof(DevState), MEM_SCRATCH}));
  TRY(mem.alloc(&res_dev, {(size_t)n_steps * sizeof(RoundResult), MEM_SCRATCH}));
  CU(cudaMemcpy(gp_dev, &gp, sizeof(gp), cudaMemcpyHostToDevice));
  CU(cudaMemcpy(st_dev, states.data(), states.size() * sizeof(DevState), cudaMemcpyHostToDevice));
  CU(cudaMemset(res_dev, 0, (size_t)n_steps * sizeof(RoundResult)));
  for (int s = 0; s < n_steps; ++s)
    accept_sample_kernel<<<1, kSampleThreads>>>(p_draft, p_verify, vocab, d, st_dev + s, gp_dev, res_dev + s,
                                                residual, s + 1, (int*)nullptr, (const int*)nullptr);
  CU(cudaGetLastError());
  CU(cudaDeviceSynchronize());
  std::vector<RoundResult> res((size_t)n_steps);
  CU(cudaMemcpy(res.data(), res_dev, res.size() * sizeof(RoundResult), cudaMemcpyDeviceToHost));
  for (int s = 0; s < n_steps; ++s) {
    const RoundResult& r = res[s];
    lsk_round_out& o = out[s];
    o.n_drafted = r.n_drafted; o.n_matches = r.n_matches; o.n_emitted = r.n_emitted; o.kv_len = r.kv_len;
    for (int i = 0; i <= LSK_MAX_SPEC; ++i) {
      o.draft_ids[i] = r.draft_ids[i];
      o.emitted_ids[i] = r.emitted_ids[i];
      o.verified_ids[i] = r.verified_ids[i];
    }
  }
  return LSK_OK;
}

}  // extern "C"
