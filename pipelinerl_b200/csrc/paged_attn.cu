// Hot path (1): paged-KV GQA attention for the decode step (one query token per sequence).
//
// Replaces the attention backend vLLM runs for the reference's sampler
// (FlashAttention / FlashInfer paged decode behind pipelinerl/async_llm.py:134).
// The KV read is what the step costs at long context: B * S * 2 * n_kv * 128 * 2 bytes
// per layer (57 344 B/token over 28 layers for Qwen2.5-7B), so the kernel is built to
// stream KV pages at HBM speed and touch every KV byte exactly once per step:
//   * one CTA per (sequence, kv head, context split); all R = n_q/n_kv query heads that
//     share the kv head are processed together (rows of one 16-row MMA tile);
//   * a producer warp TMA-stages whole pages (64 tokens x 128 d, K and V, 32 KB) into a
//     6-deep shared-memory ring (128-byte swizzle, mbarrier full/empty pipeline);
//   * 4 consumer warps each own 16 tokens of the page: S = Q K^T and O += P V on
//     mma.sync m16n8k16 (the work is ~7 FLOP per KV byte, far below any tensor roof:
//     tensor cores are used for issue efficiency, not throughput), online softmax in
//     fp32 (exp2 domain), ldmatrix with the matching XOR swizzle (conflict-free);
//   * per-split (m, l, O) partials are merged either by a small combine kernel (default) or by whichever split
//     CTA of the (sequence, kv head) finishes last (arrival ticket; prl_attn_set_fused_combine).
// KV cache layout (bf16): row = (((layer*2 + kv) * n_pages + page) * n_kv + kvh) * 64 + slot,
// 128 contiguous d per row — written by qkv_rope_cache_kernel (decode_ops.cu).
#include "prl_common.cuh"
#include "tc_ptx.cuh"
#include <math.h>

namespace prl {
namespace {

constexpr int kPage = 64;
constexpr int kD = 128;
constexpr int kStages = 6;
constexpr int kStageBytes = 4 * 8192;  // K lo/hi halves + V lo/hi halves, each 64 rows x 128 B
constexpr int kConsumers = 4;
constexpr int kThreads = (kConsumers + 1) * 32;
constexpr int kMaxPagesPerSplit = 1024;

struct AttnParams {
  const __nv_bfloat16* q;      // [B, n_q, 128]
  const int32_t* block_table;  // [B, max_blocks]
  const int32_t* seq_lens;     // [B]
  int max_blocks, n_q, n_kv, R;
  int64_t n_pages;
  int layer, n_splits;
  float scale_log2;
  float* o_part;               // [B, n_q, n_splits, 128]
  float* ml_part;              // [B, n_q, n_splits, 2]
  unsigned int* tickets;       // [B, n_kv] arrival counters (zero on entry, self-resetting); NULL = separate combine kernel
  __nv_bfloat16* out;          // [B, n_q*128]
};

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__global__ void __launch_bounds__(kThreads, 1)
paged_attn_decode_kernel(const __grid_constant__ CUtensorMap tm_kv, AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* base_ptr = smem_raw + (base - ptx::smem_u32(smem_raw));
  const uint32_t bar_base = base + kStages * kStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * (uint32_t)s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (uint32_t)(kStages + s); };
  int32_t* s_pages = reinterpret_cast<int32_t*>(base_ptr + kStages * kStageBytes + 8 * 2 * kStages);

  const int split = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_launch_dependents();
  pdl_wait();  // q, the current token's K/V and the scheduler state come from the preceding kernels
  const int seq_len = p.seq_lens[b];
  const int n_pages_b = (seq_len + kPage - 1) / kPage;
  const int per_split = (n_pages_b + p.n_splits - 1) / p.n_splits;
  const int p_begin = split * per_split;
  const int p_end = (p_begin + per_split < n_pages_b) ? p_begin + per_split : n_pages_b;
  const int n_it = p_end > p_begin ? p_end - p_begin : 0;
  const int R = p.R;

  // last-arriving split of a (sequence, kv head) merges all splits and writes the bf16 output: no combine launch
  auto finish = [&]() {
    if (p.tickets == nullptr) return;   // the stand-alone combine kernel merges the splits
    __shared__ unsigned int s_ticket;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_ticket = atomicAdd(&p.tickets[b * p.n_kv + kvh], 1u);
    __syncthreads();
    if (s_ticket != (unsigned)(p.n_splits - 1)) return;
    __threadfence();
    for (int i = threadIdx.x; i < R * kD; i += kThreads) {
      const int r = i / kD, d = i % kD;
      const int64_t head = (int64_t)b * p.n_q + kvh * R + r;
      float M = -INFINITY;
      for (int sp = 0; sp < p.n_splits; ++sp) M = fmaxf(M, __ldcg(&p.ml_part[(head * p.n_splits + sp) * 2]));
      float L = 0.f, O = 0.f;
      for (int sp = 0; sp < p.n_splits; ++sp) {
        const float ms = __ldcg(&p.ml_part[(head * p.n_splits + sp) * 2]);
        const float f = (ms == -INFINITY) ? 0.f : fast_exp2(ms - M);
        L += __ldcg(&p.ml_part[(head * p.n_splits + sp) * 2 + 1]) * f;
        O += __ldcg(&p.o_part[(head * p.n_splits + sp) * kD + d]) * f;
      }
      p.out[head * kD + d] = __float2bfloat16_rn(L > 0.f ? O / L : 0.f);
    }
    if (threadIdx.x == 0) p.tickets[b * p.n_kv + kvh] = 0u;  // re-arm for the next launch
  };

  if (n_it == 0) {  // empty split (short sequence): neutral partial
    for (int i = threadIdx.x; i < R * kD; i += kThreads) {
      const int r = i / kD, d = i % kD;
      const int64_t head = (int64_t)b * p.n_q + kvh * R + r;
      p.o_part[(head * p.n_splits + split) * kD + d] = 0.f;
      if (d == 0) {
        p.ml_part[(head * p.n_splits + split) * 2 + 0] = -INFINITY;
        p.ml_part[(head * p.n_splits + split) * 2 + 1] = 0.f;
      }
    }
    finish();
    return;
  }

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(full_bar(s), 1);
      ptx::mbar_init(empty_bar(s), kConsumers);
    }
    ptx::fence_barrier_init();
    ptx::prefetch_tensormap(&tm_kv);
  }
  for (int i = threadIdx.x; i < n_it; i += kThreads)
    s_pages[i] = p.block_table[(int64_t)b * p.max_blocks + p_begin + i];
  __syncthreads();

  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  float o[16][4];
#pragma unroll
  for (int i = 0; i < 16; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  const int g = lane >> 2, t = lane & 3;

  if (warp == kConsumers) {
    // ===== producer: TMA whole pages into the ring =====
    if (lane == 0) {
      for (int it = 0; it < n_it; ++it) {
        const int s = it % kStages;
        const uint32_t ph = (uint32_t)((it / kStages) & 1);
        ptx::mbar_wait(empty_bar(s), ph ^ 1u);
        ptx::mbar_arrive_expect_tx(full_bar(s), kStageBytes);
        const int page = s_pages[it];
        const int row_k = (int)(((((int64_t)p.layer * 2 + 0) * p.n_pages + page) * p.n_kv + kvh) * kPage);
        const int row_v = (int)(((((int64_t)p.layer * 2 + 1) * p.n_pages + page) * p.n_kv + kvh) * kPage);
        const uint32_t dst = base + (uint32_t)(s * kStageBytes);
        ptx::tma_load_2d(dst, &tm_kv, 0, row_k, full_bar(s), ptx::kEvictFirst);
        ptx::tma_load_2d(dst + 8192, &tm_kv, 64, row_k, full_bar(s), ptx::kEvictFirst);
        ptx::tma_load_2d(dst + 16384, &tm_kv, 0, row_v, full_bar(s), ptx::kEvictFirst);
        ptx::tma_load_2d(dst + 24576, &tm_kv, 64, row_v, full_bar(s), ptx::kEvictFirst);
      }
    }
  } else {
    // ===== consumers =====
    // Q fragments (A operand, rows = the R heads sharing this kv head, zero-padded to 16)
    uint32_t qa[8][4];
    {
      const __nv_bfloat16* qb = p.q + ((int64_t)b * p.n_q + kvh * R) * kD;
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        const int c = ks * 16 + 2 * t;
        qa[ks][0] = (g < R) ? *reinterpret_cast<const uint32_t*>(qb + g * kD + c) : 0u;
        qa[ks][1] = (g + 8 < R) ? *reinterpret_cast<const uint32_t*>(qb + (g + 8) * kD + c) : 0u;
        qa[ks][2] = (g < R) ? *reinterpret_cast<const uint32_t*>(qb + g * kD + c + 8) : 0u;
        qa[ks][3] = (g + 8 < R) ? *reinterpret_cast<const uint32_t*>(qb + (g + 8) * kD + c + 8) : 0u;
      }
    }
    const int mi = lane >> 3, lr = lane & 7;
    for (int it = 0; it < n_it; ++it) {
      const int s = it % kStages;
      const uint32_t ph = (uint32_t)((it / kStages) & 1);
      ptx::mbar_wait(full_bar(s), ph);
      const uint32_t kbase = base + (uint32_t)(s * kStageBytes);
      const uint32_t vbase = kbase + 16384;

      // ---- S = Q K^T over this warp's 16 tokens ----
      float sc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
      {
        const int row = warp * 16 + (mi >> 1) * 8 + lr;  // token row inside the page
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
          const int chunk = ks * 2 + (mi & 1);            // 16-byte chunk along d (0..15)
          const uint32_t addr = kbase + (uint32_t)((chunk >> 3) * 8192 + row * 128 + (((chunk & 7) ^ (row & 7)) << 4));
          uint32_t r0, r1, r2, r3;
          ldsm_x4(addr, r0, r1, r2, r3);
          mma_bf16(sc[0], qa[ks], r0, r1);
          mma_bf16(sc[1], qa[ks], r2, r3);
        }
      }
      // ---- scale, mask the tail of the last page, online softmax ----
      const int tok0 = (p_begin + it) * kPage + warp * 16;
      const bool tail = tok0 + 16 > seq_len;
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float v = sc[nt][e] * p.scale_log2;
          if (tail && (tok0 + nt * 8 + 2 * t + (e & 1)) >= seq_len) v = -INFINITY;
          sc[nt][e] = v;
        }
      uint32_t pa[4];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float mx = fmaxf(fmaxf(sc[0][2 * r], sc[0][2 * r + 1]), fmaxf(sc[1][2 * r], sc[1][2 * r + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m_run[r], mx);
        const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
        const float alpha = fast_exp2(m_run[r] - m_use);  // exp2(-inf) = 0 on the first tile
        const float p00 = fast_exp2(sc[0][2 * r] - m_use), p01 = fast_exp2(sc[0][2 * r + 1] - m_use);
        const float p10 = fast_exp2(sc[1][2 * r] - m_use), p11 = fast_exp2(sc[1][2 * r + 1] - m_use);
        l_run[r] = l_run[r] * alpha + (p00 + p01 + p10 + p11);
        m_run[r] = m_new;
#pragma unroll
        for (int i = 0; i < 16; ++i) { o[i][2 * r] *= alpha; o[i][2 * r + 1] *= alpha; }
        pa[r] = pack_bf16(p00, p01);      // a0 / a1: tokens 2t,2t+1 of the first 8
        pa[2 + r] = pack_bf16(p10, p11);  // a2 / a3: tokens 8+2t, 8+2t+1
      }
      // ---- O += P V ----
      {
        const int row = warp * 16 + (mi & 1) * 8 + lr;
#pragma unroll
        for (int dn = 0; dn < 8; ++dn) {
          const int chunk = dn * 2 + (mi >> 1);
          const uint32_t addr = vbase + (uint32_t)((chunk >> 3) * 8192 + row * 128 + (((chunk & 7) ^ (row & 7)) << 4));
          uint32_t r0, r1, r2, r3;
          ldsm_x4_t(addr, r0, r1, r2, r3);
          mma_bf16(o[2 * dn], pa, r0, r1);
          mma_bf16(o[2 * dn + 1], pa, r2, r3);
        }
      }
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(empty_bar(s));
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
      l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    }
  }

  // ---- merge the 4 consumer warps through shared memory (ring is drained) ----
  __syncthreads();
  float* s_o = reinterpret_cast<float*>(base_ptr);                 // [4][16][128]
  float* s_ml = s_o + kConsumers * 16 * kD;                        // [4][16][2]
  if (warp < kConsumers) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int rowi = g + 8 * r;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        float* dst = s_o + ((warp * 16 + rowi) * kD) + i * 8 + 2 * t;
        dst[0] = o[i][2 * r];
        dst[1] = o[i][2 * r + 1];
      }
      if (t == 0) {
        s_ml[(warp * 16 + rowi) * 2 + 0] = m_run[r];
        s_ml[(warp * 16 + rowi) * 2 + 1] = l_run[r];
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < R * kD; i += kThreads) {
    const int r = i / kD, d = i % kD;
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < kConsumers; ++w) M = fmaxf(M, s_ml[(w * 16 + r) * 2]);
    float L = 0.f, O = 0.f;
#pragma unroll
    for (int w = 0; w < kConsumers; ++w) {
      const float mw = s_ml[(w * 16 + r) * 2];
      const float f = (mw == -INFINITY) ? 0.f : fast_exp2(mw - M);
      L += s_ml[(w * 16 + r) * 2 + 1] * f;
      O += s_o[(w * 16 + r) * kD + d] * f;
    }
    const int64_t head = (int64_t)b * p.n_q + kvh * R + r;
    p.o_part[(head * p.n_splits + split) * kD + d] = O;
    if (d == 0) {
      p.ml_part[(head * p.n_splits + split) * 2 + 0] = M;
      p.ml_part[(head * p.n_splits + split) * 2 + 1] = L;
    }
  }
  finish();
}

// ---------------------------------------------------------------------------------------------
// Prefill: causal attention of a CHUNK of query tokens against the paged KV of their sequence
// (chunked prefill, conf/base.yaml:64,72: 1024-token chunks).  One CTA per (16-query tile, kv head,
// sequence); warp r owns query head kvh*R + r for those 16 tokens, so a KV page staged once by TMA
// serves all R heads x 16 queries (R*16 rows per page instead of R in decode) and no cross-warp
// merge is needed.  Same ring / swizzle / fragment layouts as the decode kernel.
// ---------------------------------------------------------------------------------------------
struct PrefillParams {
  const __nv_bfloat16* q;        // [rows, n_q, 128]
  __nv_bfloat16* out;            // [rows, n_q*128]
  const int32_t* block_table;    // [slots, max_blocks]
  const int32_t* seq_q_start;    // [n_seqs] first row of the sequence's chunk in q/out
  const int32_t* seq_q_len;      // [n_seqs] rows in the chunk
  const int32_t* seq_pos0;       // [n_seqs] position of the chunk's first token (= tokens already cached before it)
  const int32_t* seq_slot;       // [n_seqs] block-table row
  int max_blocks, n_q, n_kv, R;
  int64_t n_pages;
  int layer;
  float scale_log2;
};

constexpr int kPrefillMaxR = 8;

__global__ void __launch_bounds__((kPrefillMaxR + 1) * 32, 1)
paged_attn_prefill_kernel(const __grid_constant__ CUtensorMap tm_kv, PrefillParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = base + kStages * kStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * (uint32_t)s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (uint32_t)(kStages + s); };

  const int qtile = blockIdx.x, kvh = blockIdx.y, z = blockIdx.z;
  pdl_launch_dependents();
  pdl_wait();
  const int q_len = p.seq_q_len[z];
  const int t0 = qtile * 16;
  if (t0 >= q_len) return;
  const int row0 = p.seq_q_start[z] + t0;
  const int pos_first = p.seq_pos0[z] + t0;                 // position of query row 0 of this tile
  const int n_valid = (q_len - t0) < 16 ? (q_len - t0) : 16;
  const int kv_end = pos_first + n_valid;                   // keys [0, kv_end) are visible to the last row
  const int n_it = (kv_end + kPage - 1) / kPage;
  const int slot = p.seq_slot[z];
  const int R = p.R;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(full_bar(s), 1);
      ptx::mbar_init(empty_bar(s), (uint32_t)R);
    }
    ptx::fence_barrier_init();
    ptx::prefetch_tensormap(&tm_kv);
  }
  __syncthreads();

  if (warp == R) {
    if (lane == 0) {
      const int32_t* bt = p.block_table + (int64_t)slot * p.max_blocks;
      for (int it = 0; it < n_it; ++it) {
        const int s = it % kStages;
        const uint32_t ph = (uint32_t)((it / kStages) & 1);
        ptx::mbar_wait(empty_bar(s), ph ^ 1u);
        ptx::mbar_arrive_expect_tx(full_bar(s), kStageBytes);
        const int page = bt[it];
        const int row_k = (int)(((((int64_t)p.layer * 2 + 0) * p.n_pages + page) * p.n_kv + kvh) * kPage);
        const int row_v = (int)(((((int64_t)p.layer * 2 + 1) * p.n_pages + page) * p.n_kv + kvh) * kPage);
        const uint32_t dst = base + (uint32_t)(s * kStageBytes);
        // a sequence's KV is re-read by its other query tiles soon: keep it in L2
        ptx::tma_load_2d(dst, &tm_kv, 0, row_k, full_bar(s), ptx::kEvictLast);
        ptx::tma_load_2d(dst + 8192, &tm_kv, 64, row_k, full_bar(s), ptx::kEvictLast);
        ptx::tma_load_2d(dst + 16384, &tm_kv, 0, row_v, full_bar(s), ptx::kEvictLast);
        ptx::tma_load_2d(dst + 24576, &tm_kv, 64, row_v, full_bar(s), ptx::kEvictLast);
      }
    }
    return;
  }
  if (warp > R) return;

  const int g = lane >> 2, t = lane & 3;
  const int head = kvh * R + warp;
  uint32_t qa[8][4];
  {
    const __nv_bfloat16* q0 = p.q + ((int64_t)(row0 + g) * p.n_q + head) * kD;
    const __nv_bfloat16* q1 = p.q + ((int64_t)(row0 + g + 8) * p.n_q + head) * kD;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const int c = ks * 16 + 2 * t;
      qa[ks][0] = (g < n_valid) ? *reinterpret_cast<const uint32_t*>(q0 + c) : 0u;
      qa[ks][1] = (g + 8 < n_valid) ? *reinterpret_cast<const uint32_t*>(q1 + c) : 0u;
      qa[ks][2] = (g < n_valid) ? *reinterpret_cast<const uint32_t*>(q0 + c + 8) : 0u;
      qa[ks][3] = (g + 8 < n_valid) ? *reinterpret_cast<const uint32_t*>(q1 + c + 8) : 0u;
    }
  }
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  float o[16][4];
#pragma unroll
  for (int i = 0; i < 16; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  const int mi = lane >> 3, lr = lane & 7;

  for (int it = 0; it < n_it; ++it) {
    const int s = it % kStages;
    const uint32_t ph = (uint32_t)((it / kStages) & 1);
    ptx::mbar_wait(full_bar(s), ph);
    const uint32_t kbase = base + (uint32_t)(s * kStageBytes);
    const uint32_t vbase = kbase + 16384;

    float sc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { sc[i][0] = sc[i][1] = sc[i][2] = sc[i][3] = 0.f; }
#pragma unroll
    for (int np = 0; np < 4; ++np) {          // pairs of 8-token n-tiles
      const int row = np * 16 + (mi >> 1) * 8 + lr;
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        const int chunk = ks * 2 + (mi & 1);
        const uint32_t addr = kbase + (uint32_t)((chunk >> 3) * 8192 + row * 128 + (((chunk & 7) ^ (row & 7)) << 4));
        uint32_t r0, r1, r2, r3;
        ldsm_x4(addr, r0, r1, r2, r3);
        mma_bf16(sc[2 * np], qa[ks], r0, r1);
        mma_bf16(sc[2 * np + 1], qa[ks], r2, r3);
      }
    }
    // causal mask only on pages that reach past the first query of the tile
    const int key0 = it * kPage;
    const bool diag = key0 + kPage - 1 > pos_first;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v = sc[nt][e] * p.scale_log2;
        if (diag) {
          const int key = key0 + nt * 8 + 2 * t + (e & 1);
          const int qpos = pos_first + g + ((e >> 1) ? 8 : 0);
          if (key > qpos) v = -INFINITY;
        }
        sc[nt][e] = v;
      }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float mx = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) mx = fmaxf(mx, fmaxf(sc[nt][2 * r], sc[nt][2 * r + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[r], mx);
      const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
      const float alpha = fast_exp2(m_run[r] - m_use);
      float sum = 0.f;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        sc[nt][2 * r] = fast_exp2(sc[nt][2 * r] - m_use);
        sc[nt][2 * r + 1] = fast_exp2(sc[nt][2 * r + 1] - m_use);
        sum += sc[nt][2 * r] + sc[nt][2 * r + 1];
      }
      l_run[r] = l_run[r] * alpha + sum;
      m_run[r] = m_new;
#pragma unroll
      for (int i = 0; i < 16; ++i) { o[i][2 * r] *= alpha; o[i][2 * r + 1] *= alpha; }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {             // 16-token k-steps of P V
      uint32_t pa[4];
      pa[0] = pack_bf16(sc[2 * j][0], sc[2 * j][1]);
      pa[1] = pack_bf16(sc[2 * j][2], sc[2 * j][3]);
      pa[2] = pack_bf16(sc[2 * j + 1][0], sc[2 * j + 1][1]);
      pa[3] = pack_bf16(sc[2 * j + 1][2], sc[2 * j + 1][3]);
      const int row = j * 16 + (mi & 1) * 8 + lr;
#pragma unroll
      for (int dn = 0; dn < 8; ++dn) {
        const int chunk = dn * 2 + (mi >> 1);
        const uint32_t addr = vbase + (uint32_t)((chunk >> 3) * 8192 + row * 128 + (((chunk & 7) ^ (row & 7)) << 4));
        uint32_t r0, r1, r2, r3;
        ldsm_x4_t(addr, r0, r1, r2, r3);
        mma_bf16(o[2 * dn], pa, r0, r1);
        mma_bf16(o[2 * dn + 1], pa, r2, r3);
      }
    }
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(empty_bar(s));
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    const int rowi = g + 8 * r;
    if (rowi < n_valid) {
      const float inv = l_run[r] > 0.f ? 1.f / l_run[r] : 0.f;
      __nv_bfloat16* dst = p.out + ((int64_t)(row0 + rowi) * p.n_q + head) * kD;
#pragma unroll
      for (int i = 0; i < 16; ++i)
        *reinterpret_cast<uint32_t*>(dst + i * 8 + 2 * t) = pack_bf16(o[i][2 * r] * inv, o[i][2 * r + 1] * inv);
    }
  }
}

// stand-alone merge of the context splits (alternative to the in-kernel ticket merge; chosen at run time)
__global__ void __launch_bounds__(kD) attn_combine_kernel(const float* __restrict__ o_part,
                                                         const float* __restrict__ ml_part, int n_splits,
                                                         __nv_bfloat16* __restrict__ out) {
  const int64_t head = blockIdx.x;
  const int d = threadIdx.x;
  pdl_launch_dependents();
  pdl_wait();
  float M = -INFINITY;
  for (int s = 0; s < n_splits; ++s) M = fmaxf(M, ml_part[(head * n_splits + s) * 2]);
  float L = 0.f, O = 0.f;
  for (int s = 0; s < n_splits; ++s) {
    const float ms = ml_part[(head * n_splits + s) * 2];
    const float f = (ms == -INFINITY) ? 0.f : fast_exp2(ms - M);
    L += ml_part[(head * n_splits + s) * 2 + 1] * f;
    O += o_part[(head * n_splits + s) * kD + d] * f;
  }
  out[head * kD + d] = __float2bfloat16_rn(L > 0.f ? O / L : 0.f);
}

static int g_fused_combine = 0;

}  // namespace
}  // namespace prl

using namespace prl;

extern "C" int prl_attn_set_fused_combine(int32_t on) {
  g_fused_combine = on ? 1 : 0;
  return PRL_OK;
}

extern "C" int prl_paged_attn_splits(int32_t B, int32_t n_kv, int32_t max_seq_len) {
  const int pages = (max_seq_len + kPage - 1) / kPage;
  const int sms = num_sms();
  int splits = 1;
  // enough CTAs for >= 2 waves, at least 4 pages per CTA, never more pages than the smem page list holds
  while (B * n_kv * splits < 2 * sms && pages / (splits * 2) >= 4) splits *= 2;
  while ((pages + splits - 1) / splits > kMaxPagesPerSplit) splits *= 2;
  return splits;
}

extern "C" size_t prl_paged_attn_workspace_bytes(int32_t B, int32_t n_q, int32_t n_splits) {
  // partial O, (m, l) per split + one arrival counter per (sequence, kv head) (<= n_q of them)
  return (size_t)B * n_q * n_splits * (kD + 2) * sizeof(float) + (size_t)B * n_q * sizeof(unsigned int);
}

extern "C" int prl_paged_attn_decode(const void* q, const void* kv_cache, int64_t n_pages, int32_t n_layers,
                                     int32_t layer, const int32_t* block_table, int32_t max_blocks,
                                     const int32_t* seq_lens, int32_t B, int32_t n_q, int32_t n_kv, int32_t head_dim,
                                     int32_t page_size, int32_t n_splits, float sm_scale, void* out_bf16,
                                     void* workspace, size_t workspace_bytes, prl_stream_t stream_) {
  PRL_CHECK_ARG(q && kv_cache && block_table && seq_lens && out_bf16 && workspace, "prl_paged_attn_decode: NULL argument");
  PRL_CHECK_ARG(head_dim == kD && page_size == kPage, "prl_paged_attn_decode: head_dim must be 128 and page_size 64");
  PRL_CHECK_ARG(B >= 1 && n_kv >= 1 && n_q % n_kv == 0 && n_q / n_kv <= 16, "prl_paged_attn_decode: need n_q/n_kv <= 16");
  PRL_CHECK_ARG(n_splits >= 1 && layer >= 0 && layer < n_layers, "prl_paged_attn_decode: bad layer/splits");
  PRL_CHECK_ARG((max_blocks + n_splits - 1) / n_splits <= kMaxPagesPerSplit,
                "prl_paged_attn_decode: %d blocks / %d splits exceeds %d pages per CTA", max_blocks, n_splits,
                kMaxPagesPerSplit);
  PRL_CHECK_ARG(workspace_bytes >= prl_paged_attn_workspace_bytes(B, n_q, n_splits), "prl_paged_attn_decode: workspace too small");
  const int64_t total_rows = (int64_t)n_layers * 2 * n_pages * n_kv * kPage;
  PRL_CHECK_ARG(total_rows < (1ll << 31), "prl_paged_attn_decode: KV cache too large for 32-bit TMA row coordinates");
  CUtensorMap tm;
  int rc = make_tmap_2d_bf16(&tm, kv_cache, kD, (uint64_t)total_rows, kD * 2, 64, kPage);
  if (rc) return rc;
  AttnParams p;
  p.q = (const __nv_bfloat16*)q;
  p.block_table = block_table;
  p.seq_lens = seq_lens;
  p.max_blocks = max_blocks; p.n_q = n_q; p.n_kv = n_kv; p.R = n_q / n_kv;
  p.n_pages = n_pages; p.layer = layer; p.n_splits = n_splits;
  p.scale_log2 = sm_scale * 1.4426950408889634f;
  p.o_part = (float*)workspace;
  p.ml_part = p.o_part + (size_t)B * n_q * n_splits * kD;
  p.tickets = g_fused_combine ? reinterpret_cast<unsigned int*>(p.ml_part + (size_t)B * n_q * n_splits * 2) : nullptr;
  p.out = (__nv_bfloat16*)out_bf16;
  const int smem = kStages * kStageBytes + 1024 + 8 * 2 * kStages + 4 * kMaxPagesPerSplit + 16;
  static SmemAttr smem_attr = {};
  PRL_CUDA(ensure_smem(paged_attn_decode_kernel, smem, smem_attr));
  cudaStream_t stream = (cudaStream_t)stream_;
  dim3 grid((unsigned)n_splits, (unsigned)n_kv, (unsigned)B);
  PRL_CUDA(launch_pdl(paged_attn_decode_kernel, grid, dim3(kThreads), (size_t)smem, stream, tm, p));
  PRL_LAUNCH_CHECK();
  if (!g_fused_combine) {
    PRL_CUDA(launch_pdl(attn_combine_kernel, dim3((unsigned)(B * n_q)), dim3(kD), 0, stream, (const float*)p.o_part,
                        (const float*)p.ml_part, (int)n_splits, (__nv_bfloat16*)out_bf16));
    PRL_LAUNCH_CHECK();
  }
  return PRL_OK;
}

extern "C" int prl_paged_attn_prefill(const void* q, const void* kv_cache, int64_t n_pages, int32_t n_layers,
                                      int32_t layer, const int32_t* block_table, int32_t max_blocks,
                                      const int32_t* seq_q_start, const int32_t* seq_q_len, const int32_t* seq_pos0,
                                      const int32_t* seq_slot, int32_t n_seqs, int32_t max_q_len, int32_t n_q,
                                      int32_t n_kv, int32_t head_dim, int32_t page_size, float sm_scale,
                                      void* out_bf16, prl_stream_t stream_) {
  PRL_CHECK_ARG(q && kv_cache && block_table && seq_q_start && seq_q_len && seq_pos0 && seq_slot && out_bf16,
                "prl_paged_attn_prefill: NULL argument");
  PRL_CHECK_ARG(head_dim == kD && page_size == kPage, "prl_paged_attn_prefill: head_dim must be 128 and page_size 64");
  PRL_CHECK_ARG(n_seqs >= 1 && max_q_len >= 1 && n_kv >= 1 && n_q % n_kv == 0 && n_q / n_kv <= kPrefillMaxR,
                "prl_paged_attn_prefill: need n_q/n_kv <= %d", kPrefillMaxR);
  PRL_CHECK_ARG(layer >= 0 && layer < n_layers, "prl_paged_attn_prefill: bad layer");
  const int64_t total_rows = (int64_t)n_layers * 2 * n_pages * n_kv * kPage;
  PRL_CHECK_ARG(total_rows < (1ll << 31), "prl_paged_attn_prefill: KV cache too large for 32-bit TMA row coordinates");
  CUtensorMap tm;
  int rc = make_tmap_2d_bf16(&tm, kv_cache, kD, (uint64_t)total_rows, kD * 2, 64, kPage);
  if (rc) return rc;
  PrefillParams p;
  p.q = (const __nv_bfloat16*)q; p.out = (__nv_bfloat16*)out_bf16;
  p.block_table = block_table; p.seq_q_start = seq_q_start; p.seq_q_len = seq_q_len; p.seq_pos0 = seq_pos0;
  p.seq_slot = seq_slot; p.max_blocks = max_blocks; p.n_q = n_q; p.n_kv = n_kv; p.R = n_q / n_kv;
  p.n_pages = n_pages; p.layer = layer; p.scale_log2 = sm_scale * 1.4426950408889634f;
  const int smem = kStages * kStageBytes + 1024 + 8 * 2 * kStages + 16;
  static SmemAttr smem_attr = {};
  PRL_CUDA(ensure_smem(paged_attn_prefill_kernel, smem, smem_attr));
  dim3 grid((unsigned)((max_q_len + 15) / 16), (unsigned)n_kv, (unsigned)n_seqs);
  PRL_CUDA(launch_pdl(paged_attn_prefill_kernel, grid, dim3((p.R + 1) * 32), (size_t)smem, (cudaStream_t)stream_, tm, p));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}
