// wgmma backward of the learner's block-diagonal causal attention over one packed row (hot path 2: what the
// reference gets from flash-attn varlen through HF, pipelinerl/finetune/rl/__init__.py:204 + backward
// finetune_loop.py:716-725; conf/finetune/base.yaml:12-13,64).  Forward: attn_tc.cu (prl_attn_varlen_fwd).
//
// Rows of every query tile pack the R query heads of one GQA group: row = token * R + head.  With that packing the
// contraction over query rows in dK = dS^T Q and dV = P^T dO sums over the R heads of the group inside the tensor core,
// in a fixed order -- no atomics, no cross-head reduction pass, bitwise reproducible.
//
//     P  = exp2(S * scale_log2 - lse)         S = Q K^T        (lse saved by the forward, log2 domain)
//     dP = dO V^T                              delta = rowsum(dO o O)
//     dS = P o (dP - delta)
//     dV = P^T dO        dK = scale * dS^T Q        dQ = scale * dS K
//
// Two kernels, each deterministic, each with two consumer warpgroups (fp32 accumulators in registers) fed by TMA:
//   * attn_bwd_dkdv_kernel  (K/V stationary): one CTA per (128-key tile, kv head, sequence), warpgroup g owns keys
//     [64 g, 64 g + 64); 64-row query sub-tiles (Q, dO) stream through a 3-slot TMA ring.  It works on the TRANSPOSED
//     scores, S^T = K Q^T and dP^T = V dO^T (all operands K-major), so P^T / dS^T are already the register A operands
//     of  dV += P^T dO  and  dK += dS^T Q, whose B operands dO / Q are read AS STORED (MN-major).
//   * attn_bwd_dq_kernel    (Q stationary): one CTA per 128-row query tile, 64-key K/V steps through a 4-slot ring,
//     S = Q K^T and dP = dO V^T from shared memory, then  dQ += dS K  with dS from registers and K read as stored;
//     a separate producer warp issues the TMA loads.
//
// Generations (prl_attn_set_bwd_generation) choose, per kernel, how P^T / dS^T (dK/dV kernel) and dS (dQ kernel) reach the
// tensor core: as the register A operand of wgmma (no round trip), or stored bf16 into a 128-byte-swizzled K-major
// shared-memory tile read by a shared-memory wgmma.  1 = shared memory in both, 2 (default) = registers in both,
// 3 = registers in dK/dV and shared memory in dQ, 4 = shared memory in dK/dV and registers in dQ.  All four give the same
// bits: the operand values and the MMA order are identical.
//
// Tensor-bound: per (query row, key) pair 4 + 3 products of the two kernels; 2 exp2.
#include "prl_common.cuh"
#include "tc_ptx.cuh"
namespace prl {
namespace {

constexpr int kD = 128;
constexpr int kT16 = 16384;   // [128 rows x 128 B] operand tile
constexpr int kT8 = 8192;     // [64 rows x 128 B]
constexpr int kThreadsB = 288;   // 2 consumer warpgroups + TMA producer warp

struct BwdParams {
  const float* lse;              // [T, n_q]
  const float* delta;            // [T, n_q]
  __nv_bfloat16* dqkv;           // [T, dqkv_stride]: dQ | dK | dV in the layout of qkv
  int64_t dqkv_stride;
  const int32_t* seg_start;
  const int32_t* seg_len;
  int n_q, n_kv, R;
  int nq;                        // query tokens per tile: 128 / R (dq kernel) or 64 / R (dkdv kernel)
  int col_k, col_v;              // element column of K / V head 0 inside a qkv row
  float scale_log2, sm_scale;
  // sequence-parallel form (NULL / dqkv values otherwise): the queries are a slice of their sequences
  const int32_t* seg_pos0;       // position of a segment's first LOCAL query inside its sequence
  const int32_t* seg_kv_start;   // row of the sequence's first key in the K / V matrix
  __nv_bfloat16* dkv;            // where dK / dV rows go: [kv rows, dkv_stride], columns dkv_col_k / dkv_col_v (+ head * 128)
  int64_t dkv_stride;
  int dkv_col_k, dkv_col_v;
};

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pk2(float a, float b) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}
// A warpgroup's m64 x 64 fp32 accumulator fragment (rows row0, row0 + 8 of this thread; columns 8 c + cq + {0, 1}) as bf16
// into a [64 rows x 128 B] K-major tile with the 128-byte swizzle a wgmma shared-memory descriptor reads (1024-B aligned base).
__device__ __forceinline__ void st_frag_sw128(uint8_t* tile, int row0, int cq, const float (&x)[32]) {
#pragma unroll
  for (int c = 0; c < 8; ++c)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + 8 * h;
      *reinterpret_cast<uint32_t*>(tile + row * 128 + (((c ^ (row & 7)) << 4) | (cq * 2))) = pk2(x[4 * c + 2 * h], x[4 * c + 2 * h + 1]);
    }
}
// generic-proxy stores of a warpgroup's operand tile -> visible to its wgmma (named barrier 2 + g: the 4 warps of group g)
__device__ __forceinline__ void wg_publish_smem(int g) {
  ptx::fence_proxy_async();
  asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory");
}

// =====================================================================================================
// delta[t, h] = sum_d dO[t, h, d] * O[t, h, d]      one warp per (token, head)
// =====================================================================================================
__global__ void attn_delta_kernel(const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ d_o,
                                  int64_t n_rows /* T * n_q */, float* __restrict__ delta) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n_rows) return;
  const int lane = threadIdx.x & 31;
  const uint2 a = ld_stream_u2(reinterpret_cast<const uint2*>(o + row * kD) + lane);
  const uint2 b = ld_stream_u2(reinterpret_cast<const uint2*>(d_o + row * kD) + lane);
  float s = bf16_bits_to_float(a.x & 0xFFFFu) * bf16_bits_to_float(b.x & 0xFFFFu);
  s = fmaf(bf16_bits_to_float(a.x >> 16), bf16_bits_to_float(b.x >> 16), s);
  s = fmaf(bf16_bits_to_float(a.y & 0xFFFFu), bf16_bits_to_float(b.y & 0xFFFFu), s);
  s = fmaf(bf16_bits_to_float(a.y >> 16), bf16_bits_to_float(b.y >> 16), s);
  s = warp_sum(s);
  if (lane == 0) delta[row] = s;
}

// =====================================================================================================
// dK, dV: K/V-stationary
// =====================================================================================================
constexpr int kQStages = 3;
constexpr int kQSlot = 4 * kT8;    // Q lo | Q hi | dO lo | dO hi   (64 query rows each)
constexpr int kKvBytes = 4 * kT16; // K lo | K hi | V lo | V hi      (128 keys each)
constexpr int kOpTiles = 2 * 2 * kT8;   // [warpgroup][P^T | dS^T] operand tiles of the shared-memory generations
constexpr int kSmemDkdv = 1024 + kKvBytes + kQStages * kQSlot + kOpTiles + 8 * (2 * kQStages + 1) + 16;
static_assert(kSmemDkdv <= 232448, "dkdv kernel exceeds the 227 KB shared-memory limit");

// dV and dK accumulators (128 registers) + S^T and dP^T (64) need more than the 168 registers a thread can have with 9
// warps on the SM (3 on one sub-partition): 8 warps, and thread 0 issues the TMA loads between its own MMAs
constexpr int kThreadsDkdv = 256;

template <bool kSmemOps>
__global__ void __launch_bounds__(kThreadsDkdv, 1)
attn_bwd_dkdv_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_do,
                     const __grid_constant__ CUtensorMap tm_kv, BwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* base_gen = smem_raw + (base - ptx::smem_u32(smem_raw));
  const uint32_t kv_smem = base;                         // K lo | K hi | V lo | V hi
  const uint32_t q_ring = base + kKvBytes;               // kQStages x (Q lo | Q hi | dO lo | dO hi)
  const uint32_t op_tiles = q_ring + kQStages * kQSlot;  // [warpgroup][P^T | dS^T], kSmemOps only
  const uint32_t bar_base = op_tiles + kOpTiles;
  auto full_bar = [&](int s) { return bar_base + 8u * (uint32_t)s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (uint32_t)(kQStages + s); };
  const uint32_t kv_bar = bar_base + 8u * (uint32_t)(2 * kQStages);

  const int kt = blockIdx.x, kvh = blockIdx.y, z = blockIdx.z;
  const int q_len = p.seg_len[z];
  const int pos0 = p.seg_pos0 ? p.seg_pos0[z] : 0;
  const int kv_len = pos0 + q_len;                       // keys [0, kv_len) of the sequence are visible to some local query
  const int key0 = kt * 128;
  if (key0 >= kv_len) return;                            // uniform across the CTA, before any barrier
  const int qrow0 = p.seg_start[z];                      // first local query row of the segment
  const int kvrow0 = p.seg_kv_start ? p.seg_kv_start[z] : qrow0;
  const int rows_used = p.R * p.nq;                      // query rows of a 64-row sub-tile that hold data
  const int t_first = key0 > pos0 ? key0 - pos0 : 0;     // first local query that sees a key of this tile
  const int j_first = t_first / p.nq;
  const int n_sub = (q_len + p.nq - 1) / p.nq - j_first;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // rows [rows_used, 64) of every Q / dO tile are never written by TMA: zero them once so that 0 * garbage cannot
  // reach dK / dV through the row contraction
  for (int i = threadIdx.x; i < kQStages * 4 * (64 - rows_used) * 8; i += blockDim.x) {
    const int per_tile = (64 - rows_used) * 8;
    const int tile = i / per_tile, w = i - tile * per_tile;
    *reinterpret_cast<uint4*>(base_gen + kKvBytes + tile * kT8 + rows_used * 128 + w * 16) = make_uint4(0, 0, 0, 0);
  }
  ptx::fence_proxy_async();
  auto load_q = [&](int j) {                             // sub-tile j -> slot j % kQStages
    const int s = j % kQStages;
    ptx::mbar_arrive_expect_tx(full_bar(s), (uint32_t)(4 * 128 * rows_used));
    const uint32_t dst = q_ring + (uint32_t)(s * kQSlot);
    const int t = qrow0 + (j_first + j) * p.nq;
    ptx::tma_load_3d(dst, &tm_q, 0, kvh * p.R, t, full_bar(s), ptx::kEvictLast);
    ptx::tma_load_3d(dst + kT8, &tm_q, 64, kvh * p.R, t, full_bar(s), ptx::kEvictLast);
    ptx::tma_load_3d(dst + 2 * kT8, &tm_do, 0, kvh * p.R, t, full_bar(s), ptx::kEvictLast);
    ptx::tma_load_3d(dst + 3 * kT8, &tm_do, 64, kvh * p.R, t, full_bar(s), ptx::kEvictLast);
  };
  if (threadIdx.x == 0) {
    for (int s = 0; s < kQStages; ++s) {
      ptx::mbar_init(full_bar(s), 1);
      ptx::mbar_init(empty_bar(s), 2);   // one elected thread of each consumer warpgroup
    }
    ptx::mbar_init(kv_bar, 1);
    ptx::fence_barrier_init();
    ptx::fence_proxy_async();
    ptx::mbar_arrive_expect_tx(kv_bar, (uint32_t)kKvBytes);
#pragma unroll
    for (int kv = 0; kv < 2; ++kv)
#pragma unroll
      for (int pg = 0; pg < 2; ++pg) {
        const int c0 = (kv ? p.col_v : p.col_k) + kvh * kD;
        const uint32_t dst = kv_smem + (uint32_t)(kv * 2 * kT16 + pg * kT8);
        ptx::tma_load_2d(dst, &tm_kv, c0, kvrow0 + key0 + 64 * pg, kv_bar, ptx::kEvictFirst);
        ptx::tma_load_2d(dst + kT16, &tm_kv, c0 + 64, kvrow0 + key0 + 64 * pg, kv_bar, ptx::kEvictFirst);
      }
    for (int j = 0; j < kQStages && j < n_sub; ++j) load_q(j);
  }
  __syncthreads();

  // ===== consumers: warpgroup g owns keys [64 g, 64 g + 64); this thread keys kr[0], kr[1] (tile-relative) =====
  const int g = warp >> 2;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  int kpos[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) kpos[h] = key0 + g * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
  const int cq = 2 * (lane & 3);
  float dv[64], dk[64];
#pragma unroll
  for (int e = 0; e < 64; ++e) { dv[e] = 0.f; dk[e] = 0.f; }

  ptx::mbar_wait(kv_bar, 0);
  for (int j = 0; j < n_sub; ++j) {
    const int s = j % kQStages;
    ptx::mbar_wait(full_bar(s), (uint32_t)((j / kQStages) & 1));
    const uint32_t q_addr = q_ring + (uint32_t)(s * kQSlot);
    const uint32_t do_addr = q_addr + 2 * kT8;
    float st[32], dpt[32];
    ptx::wg_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint64_t a = ptx::make_kmajor_sw128_desc(kv_smem + (uint32_t)((ks >> 2) * kT16 + g * kT8)) + (uint64_t)(2 * (ks & 3));
      const uint64_t b = ptx::make_kmajor_sw128_desc(q_addr + (uint32_t)((ks >> 2) * kT8)) + (uint64_t)(2 * (ks & 3));
      ptx::wgmma_ss<0, 0>(st, a, b, ks > 0 ? 1u : 0u);
    }
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint64_t a = ptx::make_kmajor_sw128_desc(kv_smem + (uint32_t)(2 * kT16 + (ks >> 2) * kT16 + g * kT8)) + (uint64_t)(2 * (ks & 3));
      const uint64_t b = ptx::make_kmajor_sw128_desc(do_addr + (uint32_t)((ks >> 2) * kT8)) + (uint64_t)(2 * (ks & 3));
      ptx::wgmma_ss<0, 0>(dpt, a, b, ks > 0 ? 1u : 0u);
    }
    ptx::wg_commit();
    ptx::wg_wait<0>();
    ptx::fence_acc(st);
    ptx::fence_acc(dpt);
    // columns = query rows of the sub-tile: this thread's 16 columns are 8 c + cq + {0, 1}
    const int tsub = (j_first + j) * p.nq;
    uint32_t pa[4][4], da[4][4];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 8 * c + cq + e;
        const int qi = col / p.R, hd = col - qi * p.R;
        const int t = tsub + qi;
        const bool ok = col < rows_used && t < q_len;
        float lse = INFINITY, dl = 0.f;
        if (ok) {
          const int64_t idx = (int64_t)(qrow0 + t) * p.n_q + kvh * p.R + hd;
          lse = __ldg(p.lse + idx);
          dl = __ldg(p.delta + idx);
        }
        const int qpos = pos0 + t;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = 4 * c + 2 * h + e;
          const float pv = (ok && kpos[h] <= qpos) ? ex2f(fmaf(st[r], p.scale_log2, -lse)) : 0.f;
          st[r] = pv;
          dpt[r] = pv * (dpt[r] - dl);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      pa[c >> 1][(c & 1) * 2] = pk2(st[4 * c], st[4 * c + 1]);
      pa[c >> 1][(c & 1) * 2 + 1] = pk2(st[4 * c + 2], st[4 * c + 3]);
      da[c >> 1][(c & 1) * 2] = pk2(dpt[4 * c], dpt[4 * c + 1]);
      da[c >> 1][(c & 1) * 2 + 1] = pk2(dpt[4 * c + 2], dpt[4 * c + 3]);
    }
    const uint32_t pt_tile = op_tiles + (uint32_t)(g * 2 * kT8), dst_tile = pt_tile + kT8;
    if constexpr (kSmemOps) {   // the previous sub-tile's wgmmas have completed: the tiles are free
      const int row0 = (warp & 3) * 16 + (lane >> 2);
      st_frag_sw128(base_gen + (pt_tile - base), row0, cq, st);
      st_frag_sw128(base_gen + (dst_tile - base), row0, cq, dpt);
      wg_publish_smem(g);
    }
    ptx::fence_acc(dv);
    ptx::fence_acc(dk);
    ptx::wg_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint64_t b = ptx::make_mnmajor_sw128_desc(do_addr, kT8) + (uint64_t)(128 * kk);
      if constexpr (kSmemOps) ptx::wgmma_ss<0, 1>(dv, ptx::make_kmajor_sw128_desc(pt_tile) + (uint64_t)(2 * kk), b, 1u);
      else ptx::wgmma_rs<1>(dv, pa[kk], b, 1u);
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint64_t b = ptx::make_mnmajor_sw128_desc(q_addr, kT8) + (uint64_t)(128 * kk);
      if constexpr (kSmemOps) ptx::wgmma_ss<0, 1>(dk, ptx::make_kmajor_sw128_desc(dst_tile) + (uint64_t)(2 * kk), b, 1u);
      else ptx::wgmma_rs<1>(dk, da[kk], b, 1u);
    }
    ptx::wg_commit();
    ptx::wg_wait<0>();
    ptx::fence_acc(dv);
    ptx::fence_acc(dk);
    if (wg_leader) ptx::mbar_arrive(empty_bar(s));
    if (threadIdx.x == 0 && j + kQStages < n_sub) {      // refill the slot once both warpgroups are done with it
      ptx::mbar_wait(empty_bar(s), (uint32_t)((j / kQStages) & 1));
      load_q(j + kQStages);
    }
  }

  // ---- epilogue: bf16 dK (scaled) and dV rows of the keys this sequence has ----
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (kpos[h] >= kv_len) continue;
    __nv_bfloat16* rowp = p.dkv + (int64_t)(kvrow0 + kpos[h]) * p.dkv_stride + kvh * kD + cq;
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      *reinterpret_cast<uint32_t*>(rowp + p.dkv_col_k + 8 * c) = pk2(dk[4 * c + 2 * h] * p.sm_scale, dk[4 * c + 2 * h + 1] * p.sm_scale);
      *reinterpret_cast<uint32_t*>(rowp + p.dkv_col_v + 8 * c) = pk2(dv[4 * c + 2 * h], dv[4 * c + 2 * h + 1]);
    }
  }
}

// =====================================================================================================
// dQ: Q-stationary
// =====================================================================================================
constexpr int kKvStagesQ = 4;
constexpr int kKvSlotQ = 4 * kT8;   // K lo | K hi | V lo | V hi   (64 keys each)
constexpr int kSmemDq = 1024 + 4 * kT16 + kKvStagesQ * kKvSlotQ + 2 * kT8 + 8 * (2 * kKvStagesQ + 1) + 16;   // + [warpgroup] dS tiles
static_assert(kSmemDq <= 232448, "dq kernel exceeds the 227 KB shared-memory limit");

template <bool kSmemOps>
__global__ void __launch_bounds__(kThreadsB, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_do,
                   const __grid_constant__ CUtensorMap tm_kv, BwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t q_smem = base;                          // Q lo | Q hi | dO lo | dO hi   (128 rows each)
  const uint32_t kv_ring = base + 4 * kT16;
  const uint32_t ds_tiles = kv_ring + kKvStagesQ * kKvSlotQ;   // [warpgroup] dS, kSmemOps only
  const uint32_t bar_base = ds_tiles + 2 * kT8;
  auto full_bar = [&](int s) { return bar_base + 8u * (uint32_t)s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (uint32_t)(kKvStagesQ + s); };
  const uint32_t q_bar = bar_base + 8u * (uint32_t)(2 * kKvStagesQ);

  const int qtile = (int)(gridDim.x - 1 - blockIdx.x);   // heaviest tiles first
  const int kvh = blockIdx.y, z = blockIdx.z;
  const int q_len = p.seg_len[z];
  const int pos0 = p.seg_pos0 ? p.seg_pos0[z] : 0;
  const int t0 = qtile * p.nq;
  if (t0 >= q_len) return;                               // uniform across the CTA, before any barrier
  const int row0 = p.seg_start[z] + t0;
  const int kvrow0 = p.seg_kv_start ? p.seg_kv_start[z] : p.seg_start[z];
  const int pos_first = pos0 + t0;
  const int n_valid = (q_len - t0) < p.nq ? (q_len - t0) : p.nq;
  const int kv_end = pos_first + n_valid;
  const int n_it = (kv_end + 63) / 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 256) {
    for (int s = 0; s < kKvStagesQ; ++s) {
      ptx::mbar_init(full_bar(s), 1);
      ptx::mbar_init(empty_bar(s), 2);
    }
    ptx::mbar_init(q_bar, 1);
    ptx::fence_barrier_init();
    ptx::fence_proxy_async();
  }
  __syncthreads();

  if (warp == 8) {
    // ===== TMA producer =====
    if (lane == 0) {
      ptx::mbar_arrive_expect_tx(q_bar, (uint32_t)(4 * 128 * p.R * p.nq));
      ptx::tma_load_3d(q_smem, &tm_q, 0, kvh * p.R, row0, q_bar, ptx::kEvictFirst);
      ptx::tma_load_3d(q_smem + kT16, &tm_q, 64, kvh * p.R, row0, q_bar, ptx::kEvictFirst);
      ptx::tma_load_3d(q_smem + 2 * kT16, &tm_do, 0, kvh * p.R, row0, q_bar, ptx::kEvictFirst);
      ptx::tma_load_3d(q_smem + 3 * kT16, &tm_do, 64, kvh * p.R, row0, q_bar, ptx::kEvictFirst);
      for (int it = 0; it < n_it; ++it) {
        const int s = it % kKvStagesQ;
        ptx::mbar_wait(empty_bar(s), (uint32_t)(((it / kKvStagesQ) & 1) ^ 1));
        ptx::mbar_arrive_expect_tx(full_bar(s), (uint32_t)kKvSlotQ);
        const uint32_t dst = kv_ring + (uint32_t)(s * kKvSlotQ);
        const int row = kvrow0 + 64 * it;                // rows past the sequence / past T: masked keys (TMA zero-fills OOB)
        ptx::tma_load_2d(dst, &tm_kv, p.col_k + kvh * kD, row, full_bar(s), ptx::kEvictLast);
        ptx::tma_load_2d(dst + kT8, &tm_kv, p.col_k + kvh * kD + 64, row, full_bar(s), ptx::kEvictLast);
        ptx::tma_load_2d(dst + 2 * kT8, &tm_kv, p.col_v + kvh * kD, row, full_bar(s), ptx::kEvictLast);
        ptx::tma_load_2d(dst + 3 * kT8, &tm_kv, p.col_v + kvh * kD + 64, row, full_bar(s), ptx::kEvictLast);
      }
    }
    return;
  }

  // ===== consumers: warpgroup g owns tile rows [64 g, 64 g + 64); this thread rows mr[0], mr[1] =====
  const int g = warp >> 2;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  int mr[2], qpos[2];
  float lse[2], dl[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    mr[h] = g * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    const int qi = mr[h] / p.R, hd = mr[h] - qi * p.R;
    qpos[h] = pos_first + qi;
    lse[h] = INFINITY;                                   // rows without a query: P = 0
    dl[h] = 0.f;
    if (qi < n_valid) {
      const int64_t idx = (int64_t)(row0 + qi) * p.n_q + kvh * p.R + hd;
      lse[h] = p.lse[idx];
      dl[h] = p.delta[idx];
    } else {
      qpos[h] = -1;
    }
  }
  const int cq = 2 * (lane & 3);
  float dq[64];
#pragma unroll
  for (int e = 0; e < 64; ++e) dq[e] = 0.f;

  ptx::mbar_wait(q_bar, 0);
  for (int i = 0; i < n_it; ++i) {
    const int s = i % kKvStagesQ;
    ptx::mbar_wait(full_bar(s), (uint32_t)((i / kKvStagesQ) & 1));
    const uint32_t k_addr = kv_ring + (uint32_t)(s * kKvSlotQ);
    const uint32_t v_addr = k_addr + 2 * kT8;
    float sv[32], dp[32];
    ptx::wg_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint64_t a = ptx::make_kmajor_sw128_desc(q_smem + (uint32_t)((ks >> 2) * kT16 + g * kT8)) + (uint64_t)(2 * (ks & 3));
      const uint64_t b = ptx::make_kmajor_sw128_desc(k_addr + (uint32_t)((ks >> 2) * kT8)) + (uint64_t)(2 * (ks & 3));
      ptx::wgmma_ss<0, 0>(sv, a, b, ks > 0 ? 1u : 0u);
    }
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint64_t a = ptx::make_kmajor_sw128_desc(q_smem + (uint32_t)(2 * kT16 + (ks >> 2) * kT16 + g * kT8)) + (uint64_t)(2 * (ks & 3));
      const uint64_t b = ptx::make_kmajor_sw128_desc(v_addr + (uint32_t)((ks >> 2) * kT8)) + (uint64_t)(2 * (ks & 3));
      ptx::wgmma_ss<0, 0>(dp, a, b, ks > 0 ? 1u : 0u);
    }
    ptx::wg_commit();
    ptx::wg_wait<0>();
    ptx::fence_acc(sv);
    ptx::fence_acc(dp);
    const int key0 = i * 64;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {   // dS in place of dP
        const int h = e >> 1;
        const int key = key0 + 8 * c + cq + (e & 1);
        const float pv = key <= qpos[h] ? ex2f(fmaf(sv[4 * c + e], p.scale_log2, -lse[h])) : 0.f;
        dp[4 * c + e] = pv * (dp[4 * c + e] - dl[h]);
      }
    }
    uint32_t da[4][4];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      da[c >> 1][(c & 1) * 2] = pk2(dp[4 * c], dp[4 * c + 1]);
      da[c >> 1][(c & 1) * 2 + 1] = pk2(dp[4 * c + 2], dp[4 * c + 3]);
    }
    const uint32_t ds_tile = ds_tiles + (uint32_t)(g * kT8);
    if constexpr (kSmemOps) {   // the previous step's wgmmas have completed: the tile is free
      st_frag_sw128(smem_raw + (ds_tile - ptx::smem_u32(smem_raw)), (warp & 3) * 16 + (lane >> 2), cq, dp);
      wg_publish_smem(g);
    }
    ptx::fence_acc(dq);
    ptx::wg_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint64_t b = ptx::make_mnmajor_sw128_desc(k_addr, kT8) + (uint64_t)(128 * kk);
      if constexpr (kSmemOps) ptx::wgmma_ss<0, 1>(dq, ptx::make_kmajor_sw128_desc(ds_tile) + (uint64_t)(2 * kk), b, 1u);
      else ptx::wgmma_rs<1>(dq, da[kk], b, 1u);
    }
    ptx::wg_commit();
    ptx::wg_wait<0>();
    ptx::fence_acc(dq);
    if (wg_leader) ptx::mbar_arrive(empty_bar(s));
  }

#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int qi = mr[h] / p.R, hd = mr[h] - qi * p.R;
    if (qi >= n_valid) continue;
    __nv_bfloat16* dst = p.dqkv + (int64_t)(row0 + qi) * p.dqkv_stride + (kvh * p.R + hd) * kD + cq;
#pragma unroll
    for (int c = 0; c < 16; ++c)
      *reinterpret_cast<uint32_t*>(dst + 8 * c) = pk2(dq[4 * c + 2 * h] * p.sm_scale, dq[4 * c + 2 * h + 1] * p.sm_scale);
  }
}

int g_bwd_generation = 2;

cudaError_t launch_dkdv(dim3 grid, const CUtensorMap& tq, const CUtensorMap& tdo, const CUtensorMap& tkv, const BwdParams& p,
                        cudaStream_t stream) {
  static SmemAttr attr[2] = {};
  const bool smem_ops = g_bwd_generation == 1 || g_bwd_generation == 4;
  auto kernel = smem_ops ? attn_bwd_dkdv_kernel<true> : attn_bwd_dkdv_kernel<false>;
  cudaError_t e = ensure_smem(kernel, kSmemDkdv, attr[smem_ops ? 1 : 0]);
  if (e != cudaSuccess) return e;
  kernel<<<grid, kThreadsDkdv, (size_t)kSmemDkdv, stream>>>(tq, tdo, tkv, p);
  return cudaSuccess;
}

cudaError_t launch_dq(dim3 grid, const CUtensorMap& tq, const CUtensorMap& tdo, const CUtensorMap& tkv, const BwdParams& p,
                      cudaStream_t stream) {
  static SmemAttr attr[2] = {};
  const bool smem_ops = g_bwd_generation == 1 || g_bwd_generation == 3;
  auto kernel = smem_ops ? attn_bwd_dq_kernel<true> : attn_bwd_dq_kernel<false>;
  cudaError_t e = ensure_smem(kernel, kSmemDq, attr[smem_ops ? 1 : 0]);
  if (e != cudaSuccess) return e;
  kernel<<<grid, kThreadsB, (size_t)kSmemDq, stream>>>(tq, tdo, tkv, p);
  return cudaSuccess;
}

}  // namespace
}  // namespace prl

using namespace prl;

extern "C" int prl_attn_set_bwd_generation(int32_t gen) {
  PRL_CHECK_ARG(gen >= 1 && gen <= 4, "prl_attn_set_bwd_generation: 1 (P / dS through shared memory), 2 (registers), "
                "3 (registers in dK/dV, shared memory in dQ) or 4 (shared memory in dK/dV, registers in dQ)");
  prl::g_bwd_generation = gen;
  return PRL_OK;
}

extern "C" size_t prl_attn_varlen_bwd_workspace_bytes(int32_t T, int32_t n_q) { return (size_t)T * (size_t)n_q * sizeof(float); }

// dqkv[T, dqkv_stride] <- gradients of the packed (roped) q | k | v given d_out; every row of every segment is written.
extern "C" int prl_attn_varlen_bwd(const void* qkv, int64_t qkv_stride, int32_t T, const int32_t* seg_start,
                                   const int32_t* seg_len, int32_t n_seg, int32_t max_seg_len, int32_t n_q,
                                   int32_t n_kv, int32_t head_dim, float sm_scale, const void* out_bf16,
                                   const void* d_out_bf16, const float* lse, void* dqkv, int64_t dqkv_stride,
                                   void* workspace, size_t workspace_bytes, prl_stream_t stream_) {
  PRL_CHECK_ARG(qkv && seg_start && seg_len && out_bf16 && d_out_bf16 && lse && dqkv && workspace,
                "prl_attn_varlen_bwd: NULL argument");
  PRL_CHECK_ARG(head_dim == kD, "prl_attn_varlen_bwd: head_dim must be 128");
  PRL_CHECK_ARG(T >= 1 && n_seg >= 1 && max_seg_len >= 1 && n_kv >= 1 && n_q % n_kv == 0 && n_q / n_kv <= 64,
                "prl_attn_varlen_bwd: bad shape (GQA group size must be <= 64)");
  const int64_t width = (int64_t)(n_q + 2 * n_kv) * kD;
  PRL_CHECK_ARG(qkv_stride >= width && qkv_stride % 8 == 0 && dqkv_stride >= width && dqkv_stride % 8 == 0,
                "prl_attn_varlen_bwd: bad row stride");
  PRL_CHECK_ARG(workspace_bytes >= prl_attn_varlen_bwd_workspace_bytes(T, n_q), "prl_attn_varlen_bwd: workspace too small");
  cudaStream_t stream = (cudaStream_t)stream_;
  float* delta = (float*)workspace;
  {
    const int64_t rows = (int64_t)T * n_q;
    attn_delta_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>((const __nv_bfloat16*)out_bf16,
                                                                     (const __nv_bfloat16*)d_out_bf16, rows, delta);
    PRL_LAUNCH_CHECK();
  }
  BwdParams p;
  p.lse = lse; p.delta = delta; p.dqkv = (__nv_bfloat16*)dqkv; p.dqkv_stride = dqkv_stride;
  p.seg_start = seg_start; p.seg_len = seg_len; p.n_q = n_q; p.n_kv = n_kv; p.R = n_q / n_kv;
  p.col_k = n_q * kD; p.col_v = (n_q + n_kv) * kD;
  p.scale_log2 = sm_scale * 1.4426950408889634f; p.sm_scale = sm_scale;
  p.seg_pos0 = nullptr; p.seg_kv_start = nullptr; p.dkv = (__nv_bfloat16*)dqkv; p.dkv_stride = dqkv_stride;
  p.dkv_col_k = p.col_k; p.dkv_col_v = p.col_v;
  CUtensorMap tkv, tq, tdo;
  int rc = make_tmap_2d_bf16(&tkv, qkv, (uint64_t)width, (uint64_t)T, (uint64_t)qkv_stride * 2, 64, 64);
  if (rc) return rc;
  {
    // ---- dK, dV ----
    p.nq = 64 / p.R;
    rc = make_tmap_3d_bf16(&tq, qkv, kD, (uint64_t)n_q, (uint64_t)T, kD * 2, (uint64_t)qkv_stride * 2, 64, (uint32_t)p.R, (uint32_t)p.nq);
    if (rc) return rc;
    rc = make_tmap_3d_bf16(&tdo, d_out_bf16, kD, (uint64_t)n_q, (uint64_t)T, kD * 2, (uint64_t)n_q * kD * 2, 64, (uint32_t)p.R, (uint32_t)p.nq);
    if (rc) return rc;
    dim3 grid((unsigned)((max_seg_len + 127) / 128), (unsigned)n_kv, (unsigned)n_seg);
    PRL_CUDA(launch_dkdv(grid, tq, tdo, tkv, p, stream));
    PRL_LAUNCH_CHECK();
  }
  {
    // ---- dQ ----
    p.nq = 128 / p.R;
    rc = make_tmap_3d_bf16(&tq, qkv, kD, (uint64_t)n_q, (uint64_t)T, kD * 2, (uint64_t)qkv_stride * 2, 64, (uint32_t)p.R, (uint32_t)p.nq);
    if (rc) return rc;
    rc = make_tmap_3d_bf16(&tdo, d_out_bf16, kD, (uint64_t)n_q, (uint64_t)T, kD * 2, (uint64_t)n_q * kD * 2, 64, (uint32_t)p.R, (uint32_t)p.nq);
    if (rc) return rc;
    dim3 grid((unsigned)((max_seg_len + p.nq - 1) / p.nq), (unsigned)n_kv, (unsigned)n_seg);
    PRL_CUDA(launch_dq(grid, tq, tdo, tkv, p, stream));
    PRL_LAUNCH_CHECK();
  }
  return PRL_OK;
}

// Sequence-parallel form of prl_attn_varlen_bwd (see prl_attn_varlen_fwd_kv for the segment description).  dq[Tq, dq_stride]
// receives the query-head gradients of the LOCAL queries; dkv[Tkv, dkv_stride] = [dK heads | dV heads] receives THIS RANK'S
// contribution to every key row (zero where no local query attends) -- the caller reduce-scatters it over the group.
extern "C" int prl_attn_varlen_bwd_kv(const void* q, int64_t q_stride, int32_t Tq, const void* kv, int64_t kv_stride,
                                      int32_t Tkv, const int32_t* seg_q_start, const int32_t* seg_q_len,
                                      const int32_t* seg_pos0, const int32_t* seg_kv_start, int32_t n_seg,
                                      int32_t max_q_len, int32_t max_kv_len, int32_t n_q, int32_t n_kv, int32_t head_dim,
                                      float sm_scale, const void* out_bf16, const void* d_out_bf16, const float* lse,
                                      void* dq, int64_t dq_stride, void* dkv, int64_t dkv_stride, void* workspace,
                                      size_t workspace_bytes, prl_stream_t stream_) {
  PRL_CHECK_ARG(q && kv && seg_q_start && seg_q_len && seg_pos0 && seg_kv_start && out_bf16 && d_out_bf16 && lse && dq && dkv && workspace,
                "prl_attn_varlen_bwd_kv: NULL argument");
  PRL_CHECK_ARG(head_dim == kD, "prl_attn_varlen_bwd_kv: head_dim must be 128");
  PRL_CHECK_ARG(Tq >= 1 && Tkv >= 1 && n_seg >= 1 && max_q_len >= 1 && max_kv_len >= max_q_len && n_kv >= 1 && n_q % n_kv == 0 &&
                n_q / n_kv <= 64, "prl_attn_varlen_bwd_kv: bad shape (GQA group size must be <= 64)");
  const int64_t kvw = (int64_t)2 * n_kv * kD;
  PRL_CHECK_ARG(q_stride >= (int64_t)n_q * kD && q_stride % 8 == 0 && dq_stride >= (int64_t)n_q * kD && dq_stride % 8 == 0 &&
                kv_stride >= kvw && kv_stride % 8 == 0 && dkv_stride >= kvw && dkv_stride % 8 == 0, "prl_attn_varlen_bwd_kv: bad row stride");
  PRL_CHECK_ARG(workspace_bytes >= prl_attn_varlen_bwd_workspace_bytes(Tq, n_q), "prl_attn_varlen_bwd_kv: workspace too small");
  cudaStream_t stream = (cudaStream_t)stream_;
  float* delta = (float*)workspace;
  {
    const int64_t rows = (int64_t)Tq * n_q;
    attn_delta_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>((const __nv_bfloat16*)out_bf16,
                                                                     (const __nv_bfloat16*)d_out_bf16, rows, delta);
    PRL_LAUNCH_CHECK();
  }
  PRL_CUDA(cudaMemset2DAsync(dkv, (size_t)dkv_stride * 2, 0, (size_t)kvw * 2, (size_t)Tkv, stream));
  BwdParams p;
  p.lse = lse; p.delta = delta; p.dqkv = (__nv_bfloat16*)dq; p.dqkv_stride = dq_stride;
  p.seg_start = seg_q_start; p.seg_len = seg_q_len; p.n_q = n_q; p.n_kv = n_kv; p.R = n_q / n_kv;
  p.col_k = 0; p.col_v = n_kv * kD;
  p.scale_log2 = sm_scale * 1.4426950408889634f; p.sm_scale = sm_scale;
  p.seg_pos0 = seg_pos0; p.seg_kv_start = seg_kv_start; p.dkv = (__nv_bfloat16*)dkv; p.dkv_stride = dkv_stride;
  p.dkv_col_k = 0; p.dkv_col_v = n_kv * kD;
  CUtensorMap tkv, tq, tdo;
  int rc = make_tmap_2d_bf16(&tkv, kv, (uint64_t)kvw, (uint64_t)Tkv, (uint64_t)kv_stride * 2, 64, 64);
  if (rc) return rc;
  {
    p.nq = 64 / p.R;
    rc = make_tmap_3d_bf16(&tq, q, kD, (uint64_t)n_q, (uint64_t)Tq, kD * 2, (uint64_t)q_stride * 2, 64, (uint32_t)p.R, (uint32_t)p.nq);
    if (rc) return rc;
    rc = make_tmap_3d_bf16(&tdo, d_out_bf16, kD, (uint64_t)n_q, (uint64_t)Tq, kD * 2, (uint64_t)n_q * kD * 2, 64, (uint32_t)p.R, (uint32_t)p.nq);
    if (rc) return rc;
    dim3 grid((unsigned)((max_kv_len + 127) / 128), (unsigned)n_kv, (unsigned)n_seg);
    PRL_CUDA(launch_dkdv(grid, tq, tdo, tkv, p, stream));
    PRL_LAUNCH_CHECK();
  }
  {
    p.nq = 128 / p.R;
    rc = make_tmap_3d_bf16(&tq, q, kD, (uint64_t)n_q, (uint64_t)Tq, kD * 2, (uint64_t)q_stride * 2, 64, (uint32_t)p.R, (uint32_t)p.nq);
    if (rc) return rc;
    rc = make_tmap_3d_bf16(&tdo, d_out_bf16, kD, (uint64_t)n_q, (uint64_t)Tq, kD * 2, (uint64_t)n_q * kD * 2, 64, (uint32_t)p.R, (uint32_t)p.nq);
    if (rc) return rc;
    dim3 grid((unsigned)((max_q_len + p.nq - 1) / p.nq), (unsigned)n_kv, (unsigned)n_seg);
    PRL_CUDA(launch_dq(grid, tq, tdo, tkv, p, stream));
    PRL_LAUNCH_CHECK();
  }
  return PRL_OK;
}

