// wgmma chunked-prefill attention (hot path 1: the <= 1024-token prefill chunks vLLM interleaves with decode,
// conf/base.yaml:64,72; also prefix-shared prefill and reference-logprob scoring) and the learner's varlen forward.
//
// One CTA per (query tile, kv head, sequence).  A query tile packs nq = 128 / R consecutive query tokens x the R
// query heads of one GQA group into 128 rows (row = token * R + head), so every K/V page staged by TMA serves all R
// heads.  Two consumer warpgroups own 64 rows each; per 128-key step a warpgroup runs
//     S[64 x 128]  = Q K^T      wgmma, both operands K-major from shared memory (k = head dim), fp32 in registers
//     P            = exp2(S * scale - rowmax)   online softmax in registers (rows split over the 4 lanes of a quad)
//     O[64 x 128] += P V        wgmma with A = P straight from registers (bf16), B = V read AS STORED (MN-major)
// and rescales O in registers when the running maximum grows.  A TMA producer warp streams K/V pages through a
// 3-stage ring; the two warpgroups run independently, so one's softmax overlaps the other's tensor-core work.
//
// Two generations (prl_attn_set_fwd_generation / prl_attn_set_prefill_generation): 1 rescales O and the row sum at every
// step by exp2(m_old - m_new); 2 (default) keeps a per-row REFERENCE exponent and rescales only when the row maximum has
// grown by more than 2^8 since it was set -- P stays below 256 (exact range of bf16), and for trained or random scores the
// 64 multiplies per thread and step are skipped after the first steps of a row.
//
// Tensor-bound: 4 * 128 * S^2 / 2 FLOP per head (causal); K/V bytes are re-read from L2 by the other query tiles.
#include "prl_common.cuh"
#include "tc_ptx.cuh"

namespace prl {
namespace {

constexpr int kPageT = 64;
constexpr int kDT = 128;
constexpr int kKeys = 128;                 // keys per step = 2 pages
constexpr int kTile16K = 16384;            // one [128 rows x 128 B] operand tile
constexpr int kStageBytesT = 4 * kTile16K; // K lo/hi + V lo/hi
constexpr int kStagesT = 3;
constexpr int kThreadsT = 288;             // 2 consumer warpgroups + TMA producer warp
constexpr int kSmemT = 2 * kTile16K + kStagesT * kStageBytesT + 1024 + 8 * (2 * kStagesT + 1) + 16;
static_assert(kSmemT <= 232448, "attention forward exceeds the 227 KB shared-memory limit");

struct TcPrefillParams {
  __nv_bfloat16* out;            // [rows, n_q*128]
  const int32_t* block_table;    // [slots, max_blocks]
  const int32_t* seq_q_start;
  const int32_t* seq_q_len;
  const int32_t* seq_pos0;
  const int32_t* seq_slot;
  const int32_t* seq_kv_start;   // kContig only, may be NULL: row of the sequence's FIRST key in the K / V matrix when the queries
                                 // are a slice of the sequence (sequence-parallel learner; seq_pos0 = position of the first query)
  int max_blocks, n_q, n_kv, R, nq;
  int64_t n_pages;
  int layer;
  float scale_log2;
  // kContig (learner, packed row): K / V are columns of the same [T, qkv] matrix Q lives in -- no block table;
  // sequence z covers rows [seq_q_start[z], seq_q_start[z] + seq_q_len[z]) and its keys are those same rows
  int col_k, col_v;              // element column of K / V head 0
  float* lse;                    // [rows, n_q] log2-domain log-sum-exp of the scaled scores (may be NULL)
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

template <bool kContig, bool kLazyRescale>
__global__ void __launch_bounds__(kThreadsT, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_kv, TcPrefillParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t q_smem = base;                          // Q lo | Q hi
  const uint32_t kv_smem = base + 2 * kTile16K;          // kStagesT x (K lo | K hi | V lo | V hi)
  const uint32_t bar_base = kv_smem + kStagesT * kStageBytesT;
  auto full_bar = [&](int s) { return bar_base + 8u * (uint32_t)s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (uint32_t)(kStagesT + s); };
  const uint32_t q_bar = bar_base + 8u * (uint32_t)(2 * kStagesT);

  // packed training rows are long and causal: walk the query tiles heaviest-first
  const int qtile = kContig ? (int)(gridDim.x - 1 - blockIdx.x) : (int)blockIdx.x;
  const int kvh = blockIdx.y, z = blockIdx.z;
  const int q_len = p.seq_q_len[z];
  const int pos0 = (kContig && p.seq_pos0 == nullptr) ? 0 : p.seq_pos0[z];
  const int t0 = qtile * p.nq;
  if (t0 >= q_len) return;                               // uniform across the CTA, before any barrier
  const int row0 = p.seq_q_start[z] + t0;
  const int pos_first = pos0 + t0;
  const int n_valid = (q_len - t0) < p.nq ? (q_len - t0) : p.nq;
  const int kv_end = pos_first + n_valid;                // keys [0, kv_end) can be visible to this tile
  const int n_it = (kv_end + kKeys - 1) / kKeys;
  const int last_page = (kv_end - 1) / kPageT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 256) {
    for (int s = 0; s < kStagesT; ++s) {
      ptx::mbar_init(full_bar(s), 1);
      ptx::mbar_init(empty_bar(s), 2);   // one elected thread of each consumer warpgroup
    }
    ptx::mbar_init(q_bar, 1);
    ptx::fence_barrier_init();
    ptx::fence_proxy_async();
    ptx::prefetch_tensormap(&tm_q);
    ptx::prefetch_tensormap(&tm_kv);
  }
  __syncthreads();

  if (warp == 8) {
    // ===== TMA producer =====
    if (lane == 0) {
      ptx::mbar_arrive_expect_tx(q_bar, (uint32_t)(2 * 128 * p.R * p.nq));
      ptx::tma_load_3d(q_smem, &tm_q, 0, kvh * p.R, row0, q_bar, ptx::kEvictFirst);
      ptx::tma_load_3d(q_smem + kTile16K, &tm_q, 64, kvh * p.R, row0, q_bar, ptx::kEvictFirst);
      const int32_t* bt = kContig ? nullptr : p.block_table + (int64_t)p.seq_slot[z] * p.max_blocks;
      const int seq_row0 = (kContig && p.seq_kv_start != nullptr) ? p.seq_kv_start[z] : p.seq_q_start[z];
      for (int it = 0; it < n_it; ++it) {
        const int s = it % kStagesT;
        ptx::mbar_wait(empty_bar(s), (uint32_t)(((it / kStagesT) & 1) ^ 1));
        ptx::mbar_arrive_expect_tx(full_bar(s), (uint32_t)kStageBytesT);
#pragma unroll
        for (int kv = 0; kv < 2; ++kv) {
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            int pg = 2 * it + half;
            if (pg > last_page) pg = last_page;          // the tail step re-reads the last page; its keys are masked
            int row, c0;
            if (kContig) {                               // rows past the sequence / past T: masked keys (TMA zero-fills OOB)
              row = seq_row0 + pg * kPageT;
              c0 = (kv ? p.col_v : p.col_k) + kvh * kDT;
            } else {
              const int page = bt[pg];
              row = (int)(((((int64_t)p.layer * 2 + kv) * p.n_pages + page) * p.n_kv + kvh) * kPageT);
              c0 = 0;
            }
            const uint32_t dst = kv_smem + (uint32_t)(s * kStageBytesT + kv * 2 * kTile16K + half * 8192);
            ptx::tma_load_2d(dst, &tm_kv, c0, row, full_bar(s), ptx::kEvictLast);
            ptx::tma_load_2d(dst + kTile16K, &tm_kv, c0 + 64, row, full_bar(s), ptx::kEvictLast);
          }
        }
      }
    }
    return;
  }

  // ===== consumers: warpgroup g owns tile rows [64 g, 64 g + 64); this thread rows mr[0], mr[1] =====
  const int g = warp >> 2;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  int mr[2], qpos[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    mr[h] = g * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    qpos[h] = pos_first + mr[h] / p.R;
  }
  const int cq = 2 * (lane & 3);                         // first of this thread's two columns in each 8-column group
  float o[64];
#pragma unroll
  for (int e = 0; e < 64; ++e) o[e] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // m_run: the exponent P and l are relative to

  ptx::mbar_wait(q_bar, 0);
  for (int i = 0; i < n_it; ++i) {
    const int s = i % kStagesT;
    ptx::mbar_wait(full_bar(s), (uint32_t)((i / kStagesT) & 1));
    const uint32_t k_addr = kv_smem + (uint32_t)(s * kStageBytesT);
    const uint32_t v_addr = k_addr + 2 * kTile16K;
    float sv[64];
    ptx::wg_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint64_t a = ptx::make_kmajor_sw128_desc(q_smem + (uint32_t)((ks >> 2) * kTile16K + g * 8192)) + (uint64_t)(2 * (ks & 3));
      const uint64_t b = ptx::make_kmajor_sw128_desc(k_addr + (uint32_t)((ks >> 2) * kTile16K)) + (uint64_t)(2 * (ks & 3));
      ptx::wgmma_ss<0, 0>(sv, a, b, ks > 0 ? 1u : 0u);
    }
    ptx::wg_commit();
    ptx::wg_wait<0>();
    ptx::fence_acc(sv);
    const int key0 = i * kKeys;
    if (key0 + kKeys - 1 > pos_first) {                  // some (row, key) of this step is causally masked
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (key0 + 8 * j + cq + (e & 1) > qpos[e >> 1]) sv[4 * j + e] = -INFINITY;
    }
    float alpha[2], m_use[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 16; ++j) mx = fmaxf(mx, fmaxf(sv[4 * j + 2 * h], sv[4 * j + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx * p.scale_log2);   // scale > 0: max commutes with the scaling
      if (!kLazyRescale || m_new > m_run[h] + 8.f) {
        m_use[h] = (m_new == -INFINITY) ? 0.f : m_new;
        alpha[h] = ex2(m_run[h] - m_use[h]);              // 0 on the first step
        m_run[h] = m_new;
      } else {                                            // keep the reference: P <= 2^8
        m_use[h] = (m_run[h] == -INFINITY) ? 0.f : m_run[h];
        alpha[h] = 1.f;
      }
    }
    if (!kLazyRescale || alpha[0] != 1.f || alpha[1] != 1.f) {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        o[4 * j] *= alpha[0]; o[4 * j + 1] *= alpha[0];
        o[4 * j + 2] *= alpha[1]; o[4 * j + 3] *= alpha[1];
      }
    }
    float sum[2] = {0.f, 0.f};
    uint32_t pa[8][4];                                   // P as the A fragments of the 8 k16 steps of P V
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float p0 = ex2(fmaf(sv[4 * j], p.scale_log2, -m_use[0]));       // masked entries: exp2(-inf) = 0
      const float p1 = ex2(fmaf(sv[4 * j + 1], p.scale_log2, -m_use[0]));
      const float p2 = ex2(fmaf(sv[4 * j + 2], p.scale_log2, -m_use[1]));
      const float p3 = ex2(fmaf(sv[4 * j + 3], p.scale_log2, -m_use[1]));
      sum[0] += p0 + p1;
      sum[1] += p2 + p3;
      pa[j >> 1][(j & 1) * 2] = pack2(p0, p1);
      pa[j >> 1][(j & 1) * 2 + 1] = pack2(p2, p3);
    }
    l_run[0] = l_run[0] * alpha[0] + sum[0];             // this thread's share of the row sums
    l_run[1] = l_run[1] * alpha[1] + sum[1];
    ptx::fence_acc(o);
    ptx::wg_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
      ptx::wgmma_rs<1>(o, pa[kk], ptx::make_mnmajor_sw128_desc(v_addr, kTile16K) + (uint64_t)(128 * kk), 1u);
    ptx::wg_commit();
    ptx::wg_wait<0>();
    ptx::fence_acc(o);
    if (wg_leader) ptx::mbar_arrive(empty_bar(s));       // K and V of this stage are consumed
  }

  // ---- epilogue: normalise, write bf16 rows (and the log2-domain log-sum-exp the backward needs) ----
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int qi = mr[h] / p.R, r = mr[h] - qi * p.R;
    if (qi >= n_valid) continue;
    const float inv = l > 0.f ? 1.f / l : 0.f;
    if (kContig && p.lse != nullptr && (lane & 3) == 0)  // P = exp2(s * scale_log2 - lse) in the backward
      p.lse[(int64_t)(row0 + qi) * p.n_q + (kvh * p.R + r)] = m_run[h] + log2f(l);
    __nv_bfloat16* dst = p.out + ((int64_t)(row0 + qi) * p.n_q + (kvh * p.R + r)) * kDT + cq;
#pragma unroll
    for (int j = 0; j < 16; ++j)
      *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack2(o[4 * j + 2 * h] * inv, o[4 * j + 2 * h + 1] * inv);
  }
}

template <bool kContig>
cudaError_t launch_fwd(int generation, dim3 grid, const CUtensorMap& tq, const CUtensorMap& tkv, const TcPrefillParams& p,
                       cudaStream_t stream) {
  static SmemAttr smem_attr[2] = {};
  auto kernel = generation == 1 ? attn_fwd_kernel<kContig, false> : attn_fwd_kernel<kContig, true>;
  cudaError_t e = ensure_smem(kernel, kSmemT, smem_attr[generation == 1 ? 0 : 1]);
  if (e != cudaSuccess) return e;
  kernel<<<grid, kThreadsT, (size_t)kSmemT, stream>>>(tq, tkv, p);
  return cudaSuccess;
}

int g_fwd_generation = 2;       // prl_attn_varlen_fwd / _fwd_kv
int g_prefill_generation = 2;   // prl_paged_attn_prefill_tc

}  // namespace
}  // namespace prl

using namespace prl;

extern "C" int prl_attn_set_fwd_generation(int32_t gen) {
  PRL_CHECK_ARG(gen == 1 || gen == 2, "prl_attn_set_fwd_generation: 1 (rescale every step) or 2 (rescale past 2^8)");
  prl::g_fwd_generation = gen;
  return PRL_OK;
}

extern "C" int prl_attn_set_prefill_generation(int32_t gen) {
  PRL_CHECK_ARG(gen == 1 || gen == 2, "prl_attn_set_prefill_generation: 1 (rescale every step) or 2 (rescale past 2^8)");
  prl::g_prefill_generation = gen;
  return PRL_OK;
}

extern "C" int prl_paged_attn_prefill_tc(const void* q, int32_t q_rows, const void* kv_cache, int64_t n_pages,
                                         int32_t n_layers, int32_t layer, const int32_t* block_table,
                                         int32_t max_blocks, const int32_t* seq_q_start, const int32_t* seq_q_len,
                                         const int32_t* seq_pos0, const int32_t* seq_slot, int32_t n_seqs,
                                         int32_t max_q_len, int32_t n_q, int32_t n_kv, int32_t head_dim,
                                         int32_t page_size, float sm_scale, void* out_bf16, prl_stream_t stream_) {
  PRL_CHECK_ARG(q && kv_cache && block_table && seq_q_start && seq_q_len && seq_pos0 && seq_slot && out_bf16,
                "prl_paged_attn_prefill_tc: NULL argument");
  PRL_CHECK_ARG(head_dim == kDT && page_size == kPageT, "prl_paged_attn_prefill_tc: head_dim must be 128 and page_size 64");
  PRL_CHECK_ARG(q_rows >= 1 && n_seqs >= 1 && max_q_len >= 1 && n_kv >= 1 && n_q % n_kv == 0 && n_q / n_kv <= 128,
                "prl_paged_attn_prefill_tc: bad shape");
  PRL_CHECK_ARG(layer >= 0 && layer < n_layers, "prl_paged_attn_prefill_tc: bad layer");
  const int64_t total_rows = (int64_t)n_layers * 2 * n_pages * n_kv * kPageT;
  PRL_CHECK_ARG(total_rows < (1ll << 31), "prl_paged_attn_prefill_tc: KV cache too large for 32-bit TMA row coordinates");
  TcPrefillParams p;
  p.out = (__nv_bfloat16*)out_bf16;
  p.block_table = block_table; p.seq_q_start = seq_q_start; p.seq_q_len = seq_q_len; p.seq_pos0 = seq_pos0;
  p.seq_slot = seq_slot; p.seq_kv_start = nullptr; p.max_blocks = max_blocks; p.n_q = n_q; p.n_kv = n_kv; p.R = n_q / n_kv;
  p.nq = 128 / p.R;
  p.n_pages = n_pages; p.layer = layer; p.scale_log2 = sm_scale * 1.4426950408889634f;
  p.col_k = p.col_v = 0; p.lse = nullptr;
  CUtensorMap tq, tkv;
  int rc = make_tmap_2d_bf16(&tkv, kv_cache, kDT, (uint64_t)total_rows, kDT * 2, 64, kPageT);
  if (rc) return rc;
  rc = make_tmap_3d_bf16(&tq, q, kDT, (uint64_t)n_q, (uint64_t)q_rows, kDT * 2, (uint64_t)n_q * kDT * 2, 64, (uint32_t)p.R,
                         (uint32_t)p.nq);
  if (rc) return rc;
  dim3 grid((unsigned)((max_q_len + p.nq - 1) / p.nq), (unsigned)n_kv, (unsigned)n_seqs);
  PRL_CUDA(launch_fwd<false>(g_prefill_generation, grid, tq, tkv, p, (cudaStream_t)stream_));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}


// Learner forward (hot path 2): block-diagonal causal attention over ONE packed row, the varlen flash-attention call
// the reference makes through HF (pipelinerl/finetune/rl/__init__.py:204 with packed position_ids,
// conf/finetune/base.yaml:12-13,64).  qkv: [T, qkv_stride] bf16 = [q heads | k heads | v heads], q / k already roped.
// Same kernel as chunked prefill, K / V tiles streamed from the packed matrix instead of KV pages; also writes the
// log-sum-exp the backward needs.
extern "C" int prl_attn_varlen_fwd(const void* qkv, int64_t qkv_stride, int32_t T, const int32_t* seg_start,
                                   const int32_t* seg_len, int32_t n_seg, int32_t max_seg_len, int32_t n_q,
                                   int32_t n_kv, int32_t head_dim, float sm_scale, void* out_bf16, float* lse,
                                   prl_stream_t stream_) {
  PRL_CHECK_ARG(qkv && seg_start && seg_len && out_bf16, "prl_attn_varlen_fwd: NULL argument");
  PRL_CHECK_ARG(head_dim == kDT, "prl_attn_varlen_fwd: head_dim must be 128");
  PRL_CHECK_ARG(T >= 1 && n_seg >= 1 && max_seg_len >= 1 && n_kv >= 1 && n_q % n_kv == 0 && n_q / n_kv <= 64,
                "prl_attn_varlen_fwd: bad shape");
  PRL_CHECK_ARG(qkv_stride >= (int64_t)(n_q + 2 * n_kv) * kDT && qkv_stride % 8 == 0, "prl_attn_varlen_fwd: bad row stride");
  TcPrefillParams p;
  p.out = (__nv_bfloat16*)out_bf16;
  p.block_table = nullptr; p.seq_q_start = seg_start; p.seq_q_len = seg_len; p.seq_pos0 = nullptr; p.seq_slot = nullptr; p.seq_kv_start = nullptr;
  p.max_blocks = 0; p.n_q = n_q; p.n_kv = n_kv; p.R = n_q / n_kv; p.nq = 128 / p.R;
  p.n_pages = 0; p.layer = 0; p.scale_log2 = sm_scale * 1.4426950408889634f;
  p.col_k = n_q * kDT; p.col_v = (n_q + n_kv) * kDT; p.lse = lse;
  CUtensorMap tq, tkv;
  int rc = make_tmap_2d_bf16(&tkv, qkv, (uint64_t)(n_q + 2 * n_kv) * kDT, (uint64_t)T, (uint64_t)qkv_stride * 2, 64, kPageT);
  if (rc) return rc;
  rc = make_tmap_3d_bf16(&tq, qkv, kDT, (uint64_t)n_q, (uint64_t)T, kDT * 2, (uint64_t)qkv_stride * 2, 64, (uint32_t)p.R,
                         (uint32_t)p.nq);
  if (rc) return rc;
  dim3 grid((unsigned)((max_seg_len + p.nq - 1) / p.nq), (unsigned)n_kv, (unsigned)n_seg);
  PRL_CUDA(launch_fwd<true>(g_fwd_generation, grid, tq, tkv, p, (cudaStream_t)stream_));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

// Sequence-parallel form of prl_attn_varlen_fwd (the reference shards a packed row over `seq_parallel` ranks and runs
// ring attention, finetune_loop.py:507-517, finetune/types.py:145-180): the queries are the LOCAL slice q[Tq, q_stride]
// (query heads in the first n_q * 128 columns), the keys / values the all-gathered matrix kv[Tkv, kv_stride] =
// [k heads | v heads].  Local segment z: queries q rows [seg_q_start[z], + seg_q_len[z]), the first of them at position
// seg_pos0[z] of its sequence, whose first key is kv row seg_kv_start[z].
extern "C" int prl_attn_varlen_fwd_kv(const void* q, int64_t q_stride, int32_t Tq, const void* kv, int64_t kv_stride,
                                      int32_t Tkv, const int32_t* seg_q_start, const int32_t* seg_q_len,
                                      const int32_t* seg_pos0, const int32_t* seg_kv_start, int32_t n_seg,
                                      int32_t max_q_len, int32_t n_q, int32_t n_kv, int32_t head_dim, float sm_scale,
                                      void* out_bf16, float* lse, prl_stream_t stream_) {
  PRL_CHECK_ARG(q && kv && seg_q_start && seg_q_len && seg_pos0 && seg_kv_start && out_bf16, "prl_attn_varlen_fwd_kv: NULL argument");
  PRL_CHECK_ARG(head_dim == kDT, "prl_attn_varlen_fwd_kv: head_dim must be 128");
  PRL_CHECK_ARG(Tq >= 1 && Tkv >= 1 && n_seg >= 1 && max_q_len >= 1 && n_kv >= 1 && n_q % n_kv == 0 && n_q / n_kv <= 64,
                "prl_attn_varlen_fwd_kv: bad shape");
  PRL_CHECK_ARG(q_stride >= (int64_t)n_q * kDT && q_stride % 8 == 0 && kv_stride >= (int64_t)2 * n_kv * kDT && kv_stride % 8 == 0,
                "prl_attn_varlen_fwd_kv: bad row stride");
  TcPrefillParams p;
  p.out = (__nv_bfloat16*)out_bf16;
  p.block_table = nullptr; p.seq_q_start = seg_q_start; p.seq_q_len = seg_q_len; p.seq_pos0 = seg_pos0; p.seq_slot = nullptr;
  p.seq_kv_start = seg_kv_start;
  p.max_blocks = 0; p.n_q = n_q; p.n_kv = n_kv; p.R = n_q / n_kv; p.nq = 128 / p.R;
  p.n_pages = 0; p.layer = 0; p.scale_log2 = sm_scale * 1.4426950408889634f;
  p.col_k = 0; p.col_v = n_kv * kDT; p.lse = lse;
  CUtensorMap tq, tkv;
  int rc = make_tmap_2d_bf16(&tkv, kv, (uint64_t)(2 * n_kv) * kDT, (uint64_t)Tkv, (uint64_t)kv_stride * 2, 64, kPageT);
  if (rc) return rc;
  rc = make_tmap_3d_bf16(&tq, q, kDT, (uint64_t)n_q, (uint64_t)Tq, kDT * 2, (uint64_t)q_stride * 2, 64, (uint32_t)p.R, (uint32_t)p.nq);
  if (rc) return rc;
  dim3 grid((unsigned)((max_q_len + p.nq - 1) / p.nq), (unsigned)n_kv, (unsigned)n_seg);
  PRL_CUDA(launch_fwd<true>(g_fwd_generation, grid, tq, tkv, p, (cudaStream_t)stream_));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}
