// common.cuh — device helpers shared by the sm_90a kernels of liblsk.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace lsk {

constexpr int kPageTokens = 64;    // tokens per KV page
constexpr int kMaxHeadDim = 128;   // head_dim in {32, 64, 128} (attention / RoPE epilogue are templated / parameterised)
constexpr int kMaxRows = 16;       // rows (tokens) one step can carry: D_max + 1

// ---------------------------------------------------------------------------------------
// programmatic dependent launch (PDL): a kernel may start while its predecessor drains;
// it must not touch the predecessor's outputs before pdl_wait().  Every kernel calls
// pdl_wait() exactly once so completion is transitive along the chain.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
}

// ---- mbarrier + TMA bulk copy (1-D cp.async.bulk, global -> shared, mbarrier completion)
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "LAB_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE;\n\t"
      "bra LAB_WAIT;\n\t"
      "DONE:\n\t}"
      ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                             uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}


// streaming 128-bit load of packed weights: read-only path, do not allocate in L1.
__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }

// D(16x8,f32) += A(16x16,bf16,row) * B(16x8,bf16,col)
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], uint32_t a0, uint32_t a1,
                                               uint32_t a2, uint32_t a3, uint32_t b0,
                                               uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 "
      "{%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* smem_ptr) {
  uint32_t addr = static_cast<uint32_t>(__cvta_generic_to_shared(smem_ptr));
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// arg-max with the "lowest index wins ties" rule used everywhere in the engine.
__device__ __forceinline__ bool better(float v, int i, float bv, int bi) {
  return (v > bv) || (v == bv && i < bi);
}

// ---------------------------------------------------------------------------------------
// KV pool layout: [layer][page][kv_head][64 tokens][head_dim] bf16.  Inside a token row the
// 16-byte chunks are XOR-swizzled so that a whole (page, kv head) block can be moved into shared
// memory by ONE TMA bulk copy and still be read conflict-free by the attention kernel's
// fragment loads / ldmatrix (8 rows x one 16-byte chunk per access phase): rows of >= 128 bytes
// (head_dim >= 64) use tok & 7, head_dim 32 (two rows per 128 bytes) uses (tok >> 1) & 3.
// Every reader and writer of the pool goes through these two functions.
// ---------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ int kv_chunk_swizzle(int hd, int tok) {
  return hd >= 64 ? (tok & 7) : ((tok >> 1) & 3);
}
__host__ __device__ __forceinline__ size_t kv_elem_offset(int hd, int page, int n_kv_heads, int head,
                                                         int tok, int d) {
  const int chunk = (d >> 3) ^ kv_chunk_swizzle(hd, tok);
  return ((size_t)(page * n_kv_heads + head) * kPageTokens + tok) * hd + chunk * 8 + (d & 7);
}

// ---------------------------------------------------------------------------------------
// K-major SWIZZLE_128B operand layout of the wgmma prefill GEMM (prefill_tc.cuh): stages of
// 128 rows x 64 k (16 KiB); a row's 64 k (128 bytes) are contiguous, rows 128 bytes apart, and
// inside every 8-row / 1 KiB atom the 16-byte chunks are XOR-swizzled with the row index — the
// layout a TMA tensor copy with CU_TENSOR_MAP_SWIZZLE_128B would produce, written here directly
// by the producing kernels so that plain 1-D bulk copies can move it (the swizzle keeps the tensor
// core's operand fetches free of shared-memory bank conflicts).
// Byte offset of element (row < 128, k):
// ---------------------------------------------------------------------------------------
constexpr int kCanonStageBytes = 128 * 64 * 2;
__host__ __device__ __forceinline__ size_t canon_offset(int row, int k) {
  const int s = k >> 6, c = (k >> 3) & 7;
  return (size_t)s * kCanonStageBytes + (size_t)row * 128 + ((c ^ (row & 7)) << 4) + (k & 7) * 2;
}

// Device-resident generation state (one per engine).  `tok[0]` is the pending input token,
// `tok[1 + i]` the i-th draft token of the current round.
struct DevState {
  int len;                    // committed KV length (= n_prompt + n_out - 1 once generating)
  int n_out;                  // tokens emitted so far (before EOS truncation)
  int step_count;             // rounds / AR steps executed (RNG stream position)
  int n_prompt;               // prompt length: hist[n_prompt + n_out] is where the next emitted token goes
  int tok[kMaxRows + 1];
  int verified[kMaxRows + 1];
  // adaptive rounds (lsk_round_adaptive): the threshold the host set for this round, the draft
  // confidences, and d_stop = the number of drafts the round keeps
  float min_conf;
  float conf[kMaxRows];
  int d_stop;
};

}  // namespace lsk
