// wgmma weight-streaming GEMM for the token step (hot path 1) and the output head.
//
//   Y[M_tok, N_out] = X[M_tok, K] * W[N_out, K]^T      (bf16 in, fp32 accumulate)
//
// replaces the cuBLAS GEMMs vLLM issues per decode step for Qwen2's qkv / o / gate_up /
// down projections (reached from pipelinerl/async_llm.py:134 through the vLLM engine) and
// the fp32 lm_head matmul of pipelinerl/vllm_quantization.py:266-278.
//
// Decode shapes are skinny (M_tok <= 64..256), so the kernel is laid out "swap-AB":
// the WEIGHT tile is the wgmma M operand (128 output features per CTA, 64 per consumer
// warpgroup), the tokens are the N operand (16..256), and D^T = W_tile * X^T accumulates in
// registers (row = output feature, column = token).  Every weight byte is read from HBM exactly
// once per step by TMA (EVICT_FIRST), the small activation tile is re-read from L2
// (EVICT_LAST); split-K fills the 132 SMs when N_out/128 < #SMs, with fp32 partials
// reduced by the consumer epilogue kernel (decode_ops.cu) in a fixed order.
//
// Warp roles (288 threads): warps 0..7 = two consumer warpgroups (wgmma, then the epilogue),
// warp 8 = TMA producer.  An optional second weight operand W_lo (bf16 residual of an fp32
// master) is accumulated into the same registers: fp32-equivalent head at the cost of a second
// bf16 stream (same bytes as an fp32 weight).
//
// HBM-bound: algorithmic bytes = 2*N*K (+2*N*K with W_lo) + 2*M*K + 4*split_k*M*N.
#include "prl_common.cuh"
#include "tc_ptx.cuh"

namespace prl {

int head_logprob_tn(const void* W, const void* W_lo, const void* X, int64_t M, int64_t V, int64_t K, float temperature,
                    const int64_t* targets, float* logprob_target, float* entropy, float* lse, void* workspace,
                    cudaStream_t stream);  // gemm_tn.cu

// ------------------------------------------------------------------------------------
// host: tensor maps
// ------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess || !p) {
      set_error("cuTensorMapEncodeTiled not available from the driver");
      return nullptr;
    }
    fn = (EncodeTiledFn)p;
  }
  return fn;
}

int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t inner_elems, uint64_t outer_rows,
                      uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return PRL_ERR_CUDA;
  if ((uintptr_t)base % 16 != 0 || row_stride_bytes % 16 != 0) {
    set_error("TMA operand must be 16-byte aligned (base %p, row stride %llu B)", base,
              (unsigned long long)row_stride_bytes);
    return PRL_ERR_INVALID;
  }
  cuuint64_t dims[2] = {inner_elems, outer_rows};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_rows};
  cuuint32_t elem_strides[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, elem_strides,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (inner %llu rows %llu stride %llu box %u x %u)", (int)r,
              (unsigned long long)inner_elems, (unsigned long long)outer_rows, (unsigned long long)row_stride_bytes,
              box_inner, box_rows);
    return PRL_ERR_CUDA;
  }
  return PRL_OK;
}

// 3-D bf16 tensor map (innermost dimension contiguous), 128-byte swizzle: box_inner * 2 bytes must be 128
int make_tmap_3d_bf16(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_bytes,
                      uint64_t stride2_bytes, uint32_t box0, uint32_t box1, uint32_t box2) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return PRL_ERR_CUDA;
  if ((uintptr_t)base % 16 != 0 || stride1_bytes % 16 != 0 || stride2_bytes % 16 != 0) {
    set_error("TMA operand must be 16-byte aligned (base %p, strides %llu / %llu B)", base,
              (unsigned long long)stride1_bytes, (unsigned long long)stride2_bytes);
    return PRL_ERR_INVALID;
  }
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {stride1_bytes, stride2_bytes};
  cuuint32_t box[3] = {box0, box1, box2};
  cuuint32_t elem_strides[3] = {1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, elem_strides,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled (3-D) failed with CUresult %d", (int)r);
    return PRL_ERR_CUDA;
  }
  return PRL_OK;
}

namespace {

constexpr int kBlockM = 128;  // output features per CTA (two wgmma M = 64 halves)
constexpr int kBlockK = 64;   // bf16 elements per stage row = 128 B = one swizzle atom
constexpr int kUmmaK = 16;
constexpr int kThreads = 288;
// Per-CTA tile ring at kNTile <= 64.  72 KB = 3 stages at the decode batch (kNTile = 64, 24 KB per stage) lets THREE CTAs
// share an SM (the kernel needs fewer than 75 registers per thread), so the token step's split plans (qkv 36 x 11 = 396,
// o and down 28 x 14 = 392, gate_up 296 CTAs) each run as one wave on 132 SMs instead of 1.1-1.5 waves with two CTAs
// per SM and a 96 KB ring.  The ring depth does not change any CTA's k-range: results are the same bits.
static int g_smem_budget = 72 * 1024;
static int g_tiled_weights = 0;  // weights stored as contiguous [N/128][K/64][128][64] tiles

struct HeadPart { float m, s, u, key, z; int idx; };  // per (vocab tile, token): online-softmax state + best sample

struct GemmParams {
  int64_t M, N, K;
  int kblocks;        // ceil(K / 64)
  int split_k;
  int has_lo;
  float* partials;    // [split_k, M, N]
  float* peer_partials;  // same layout in a tensor-parallel peer's memory (P2P stores), or NULL
  // fused head epilogue (logits never reach HBM): temperature, teacher-forcing targets, sampling
  int tiled;          // weight tile (n_tile, kb) is the contiguous 16 KB block number n_tile*kblocks + kb
  int head;
  float inv_temp;
  const int64_t* targets;   // [M] or NULL
  float* picked;            // [M] z of the target id (written by the CTA whose tile holds it)
  int greedy;
  unsigned long long seed;
  unsigned int step;
  HeadPart* head_part;      // [n_tiles, M]
  // SwiGLU epilogue of the token step's gate_up GEMM (split_k == 1): the CTA's 128 weight rows are 64 GATE rows
  // [64 t, 64 t + 64) and the 64 UP rows of the same features (I rows further down), and the epilogue writes
  // act[token, feature] = bf16(SiLU(gate) * up) -- the bits of the partial tile + silu_mul_kernel pair, without the pair
  int64_t swiglu_I;         // 0 = off
  __nv_bfloat16* act;       // [M, swiglu_I]
};

template <int kNTile>
struct SmemLayout {
  static constexpr int kABytes = kBlockM * kBlockK * 2;       // 16 KB
  static constexpr int kBBytes = kNTile * kBlockK * 2;
  static constexpr int kStageLd = kNTile + 1;                 // fp32 accumulator tile [128 features][kNTile + 1]: odd stride
  static constexpr int kEpiBytes = kBlockM * kStageLd * 4 + 4 * kNTile * (int)sizeof(HeadPart);
  static constexpr int stage_bytes(bool lo) { return kABytes * (lo ? 2 : 1) + kBBytes; }
  static int stages(bool lo) {
    int s = g_smem_budget / stage_bytes(lo);
    return s > 8 ? 8 : (s < 2 ? 2 : s);
  }
  // the epilogue reuses the drained tile ring for the accumulator tile (and the head statistics behind it)
  __host__ __device__ static int ring_bytes(int n_stages, bool lo) {
    const int r = n_stages * stage_bytes(lo);
    return r > kEpiBytes ? r : kEpiBytes;
  }
};

// Warp roles (288 threads): warps 0..7 = two consumer warpgroups (wgmma m64 x kNTile: warpgroup g owns weight rows
// [64 g, 64 g + 64) of the tile, fp32 accumulators in registers), warp 8 = TMA producer.
template <int kNTile, bool kHead>
__global__ void __launch_bounds__(kThreads, kNTile <= 64 ? 2 : 1)
gemm_swapab_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_wlo,
                   const __grid_constant__ CUtensorMap tm_x, GemmParams p, int n_stages) {
  using L = SmemLayout<kNTile>;
  extern __shared__ uint8_t smem_raw[];
  pdl_launch_dependents();  // let the next kernel start its own prologue / weight prefetch as early as possible
  const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - ptx::smem_u32(smem_raw));
  const bool lo = p.has_lo != 0;
  const int stage_bytes = L::stage_bytes(lo);
  // barriers live after the tile ring
  const uint32_t bar_base = smem_base + (uint32_t)L::ring_bytes(n_stages, lo);
  auto full_bar = [&](int s) { return bar_base + 8u * (uint32_t)s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (uint32_t)(n_stages + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // blockIdx.x enumerates (weight tile, token tile) with the token tile fastest, so the CTAs that share a
  // weight tile are co-scheduled and the tile is fetched from HBM once (prefill / training shapes, M > 256)
  const int m_tiles = (int)((p.M + kNTile - 1) / kNTile);
  const int n_tile = (int)blockIdx.x / m_tiles;
  const int n0 = n_tile * kBlockM;            // first output feature of this CTA
  const int split = blockIdx.y;
  const int m0 = ((int)blockIdx.x % m_tiles) * kNTile;  // first token of this CTA
  const int kb_begin = (int)(((int64_t)p.kblocks * split) / p.split_k);
  const int kb_end = (int)(((int64_t)p.kblocks * (split + 1)) / p.split_k);
  const int n_kb = kb_end - kb_begin;

  auto load_weights = [&](int i, int s) {
    const uint32_t a_dst = smem_base + (uint32_t)(s * stage_bytes);
    const int kcoord = (kb_begin + i) * kBlockK;
    const int wc0 = p.tiled ? 0 : kcoord;
    const int wc1 = p.tiled ? (n_tile * p.kblocks + kb_begin + i) * kBlockM : n0;
    if (p.swiglu_I) {   // tm_w boxes are 64 rows here: gate half, then up half of the same 64 features
      ptx::tma_load_2d(a_dst, &tm_w, wc0, n_tile * 64, full_bar(s), ptx::kEvictFirst);
      ptx::tma_load_2d(a_dst + L::kABytes / 2, &tm_w, wc0, (int)p.swiglu_I + n_tile * 64, full_bar(s), ptx::kEvictFirst);
    } else {
      ptx::tma_load_2d(a_dst, &tm_w, wc0, wc1, full_bar(s), ptx::kEvictFirst);
    }
    if (lo) ptx::tma_load_2d(a_dst + L::kABytes, &tm_wlo, wc0, wc1, full_bar(s), ptx::kEvictFirst);
  };

  // The producer thread arms the barriers and IMMEDIATELY fills the first ring pass with WEIGHT tiles: weights do not
  // depend on the preceding kernel (PDL lets this run under the predecessor's tail), so the first HBM round trip
  // overlaps the predecessor's tail and this CTA's prologue.
  const int pre = n_kb < n_stages ? n_kb : n_stages;
  if (threadIdx.x == 256) {
    for (int s = 0; s < n_stages; ++s) {
      ptx::mbar_init(full_bar(s), 1);
      ptx::mbar_init(empty_bar(s), 2);   // one elected thread of each consumer warpgroup
    }
    ptx::fence_barrier_init();
    ptx::fence_proxy_async();
    for (int i = 0; i < pre; ++i) {
      ptx::mbar_arrive_expect_tx(full_bar(i), (uint32_t)stage_bytes);
      load_weights(i, i);
    }
    ptx::prefetch_tensormap(&tm_x);
  }
  __syncthreads();

  if (warp == 8) {
    // ===== TMA producer =====  (first-pass weight tiles were issued before the CTA-wide sync)
    if (lane == 0) {
      pdl_wait();
      for (int i = 0; i < pre; ++i) {
        const uint32_t b_dst = smem_base + (uint32_t)(i * stage_bytes) + L::kABytes * (lo ? 2 : 1);
        ptx::tma_load_2d(b_dst, &tm_x, (kb_begin + i) * kBlockK, m0, full_bar(i), ptx::kEvictLast);
      }
      for (int i = pre; i < n_kb; ++i) {
        const int s = i % n_stages;
        const uint32_t ph = (uint32_t)((i / n_stages) & 1);
        ptx::mbar_wait(empty_bar(s), ph ^ 1u);
        ptx::mbar_arrive_expect_tx(full_bar(s), (uint32_t)stage_bytes);
        load_weights(i, s);
        const uint32_t b_dst = smem_base + (uint32_t)(s * stage_bytes) + L::kABytes * (lo ? 2 : 1);
        ptx::tma_load_2d(b_dst, &tm_x, (kb_begin + i) * kBlockK, m0, full_bar(s), ptx::kEvictLast);
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg = weight rows [64 wg, 64 wg + 64), all kNTile tokens =====
  const int wg = warp >> 2;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  float acc[kNTile / 2];
#pragma unroll
  for (int e = 0; e < kNTile / 2; ++e) acc[e] = 0.f;
  for (int i = 0; i < n_kb; ++i) {
    const int s = i % n_stages;
    ptx::mbar_wait(full_bar(s), (uint32_t)((i / n_stages) & 1));
    const uint32_t a_addr = smem_base + (uint32_t)(s * stage_bytes) + (uint32_t)(wg * 64 * 128);
    const uint32_t b_addr = smem_base + (uint32_t)(s * stage_bytes) + L::kABytes * (lo ? 2 : 1);
    const uint64_t a_desc = ptx::make_kmajor_sw128_desc(a_addr);
    const uint64_t b_desc = ptx::make_kmajor_sw128_desc(b_addr);
    ptx::fence_acc(acc);
    ptx::wg_fence();
#pragma unroll
    for (int k = 0; k < kBlockK / kUmmaK; ++k)
      ptx::wgmma_ss<0, 0>(acc, a_desc + (uint64_t)(2 * k), b_desc + (uint64_t)(2 * k), 1u);
    if (lo) {
      const uint64_t al_desc = ptx::make_kmajor_sw128_desc(a_addr + L::kABytes);
#pragma unroll
      for (int k = 0; k < kBlockK / kUmmaK; ++k)
        ptx::wgmma_ss<0, 0>(acc, al_desc + (uint64_t)(2 * k), b_desc + (uint64_t)(2 * k), 1u);
    }
    ptx::wg_commit();
    ptx::wg_wait<1>();                       // the previous stage's wgmmas are done: release that slot
    if (i > 0 && wg_leader) ptx::mbar_arrive(empty_bar((i - 1) % n_stages));
  }
  ptx::wg_wait<0>();
  ptx::fence_acc(acc);

  // ---- accumulators -> fp32 tile [feature][token] in the drained ring (every stage has been waited on) ----
  asm volatile("bar.sync 1, 256;" ::: "memory");   // both warpgroups are past their last shared-memory operand read
  float* stile = reinterpret_cast<float*>(smem_gen);
  {
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < kNTile / 8; ++j) {
      const int c = 8 * j + 2 * (lane & 3);
      stile[r0 * L::kStageLd + c] = acc[4 * j];
      stile[r0 * L::kStageLd + c + 1] = acc[4 * j + 1];
      stile[(r0 + 8) * L::kStageLd + c] = acc[4 * j + 2];
      stile[(r0 + 8) * L::kStageLd + c + 1] = acc[4 * j + 3];
    }
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");

  // ===== epilogue: thread = one output feature (lanes = 32 consecutive features), half of the tokens =====
  pdl_wait();  // the output buffers may still be read by the predecessor's consumer
  const int q = warp & 3;                    // feature quarter
  const int half = warp >> 2;                // token half
  const int fr = q * 32 + lane;              // tile row
  const int feat = n0 + fr;                  // output feature (vocab id) owned by this thread
  const int m_valid = (int)((p.M - m0) < kNTile ? (p.M - m0) : kNTile);
  const bool feat_ok = feat < p.N;
  constexpr int kHalfTok = kNTile / 2;
  const int tb = half * kHalfTok, te = tb + kHalfTok;
  const float* srow = stile + fr * L::kStageLd;
  if constexpr (!kHead) {
    if (p.swiglu_I) {
      // ---- SwiGLU: tile rows 0..63 = gate, 64..127 = up of features [64 t, 64 t + 64); columns = tokens ----
      if (q < 2) {
        const int64_t f = (int64_t)n_tile * 64 + fr;
        const float* urow = stile + (fr + 64) * L::kStageLd;
        for (int t = tb; t < te && t < m_valid; ++t) {
          const float gg = srow[t], uu = urow[t];
          p.act[(int64_t)(m0 + t) * p.swiglu_I + f] = __float2bfloat16_rn((gg / (1.f + __expf(-gg))) * uu);
        }
      }
    } else if (feat_ok) {
      // ---- fp32 partial tile: 32 lanes -> one 128-B row segment per token ----
      float* out = p.partials + ((int64_t)split * p.M + m0) * p.N + feat;
      // tensor-parallel row-parallel GEMM: the partial sums are ALSO stored straight into the peer GPU's reduction
      // buffer over NVLink, so the "all-reduce" is this epilogue plus the consumer's ordinary split reduction
      float* out_peer = p.peer_partials ? p.peer_partials + ((int64_t)split * p.M + m0) * p.N + feat : nullptr;
      for (int t = tb; t < te && t < m_valid; ++t) {
        out[(int64_t)t * p.N] = srow[t];
        if (out_peer) out_peer[(int64_t)t * p.N] = srow[t];
      }
    }
  } else {
    // ---- fused output head: per token, online-softmax statistics over this tile's 128 vocabulary rows,
    //      the target logit and the best Gumbel-perturbed logit; the logits themselves are never stored ----
    HeadPart* s_hp = reinterpret_cast<HeadPart*>(smem_gen + kBlockM * L::kStageLd * 4);  // [4][kNTile]
#pragma unroll 1
    for (int t = tb; t < te; ++t) {
      const int tok = m0 + t;
      const bool tok_ok = t < m_valid;
      const float z = feat_ok ? srow[t] * p.inv_temp : -INFINITY;
      const float m = warp_max(z);
      const float e = (z == -INFINITY) ? 0.f : __expf(z - m);
      const float ssum = warp_sum(e);
      const float usum = warp_sum(e > 0.f ? e * z : 0.f);
      float key = -INFINITY;
      if (feat_ok) key = p.greedy ? z : z + gumbel(p.seed, p.step, (uint32_t)tok, (uint32_t)feat);
      float bkey = key, bz = z;
      int bidx = feat_ok ? feat : 0x7fffffff;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float k2 = __shfl_xor_sync(0xffffffffu, bkey, o);
        const float z2 = __shfl_xor_sync(0xffffffffu, bz, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, bidx, o);
        if (k2 > bkey || (k2 == bkey && i2 < bidx)) { bkey = k2; bz = z2; bidx = i2; }
      }
      if (p.targets && tok_ok && feat_ok && p.targets[tok] == (int64_t)feat) p.picked[tok] = z;
      if (lane == 0) s_hp[q * kNTile + t] = HeadPart{m, ssum, usum, bkey, bz, bidx};
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");  // the consumer warps only
    for (int tkn = threadIdx.x; tkn < m_valid; tkn += 256) {
      HeadPart a = s_hp[tkn];
#pragma unroll
      for (int qq = 1; qq < 4; ++qq) {
        const HeadPart b = s_hp[qq * kNTile + tkn];
        const float mm = fmaxf(a.m, b.m);
        const float fa = (a.m == -INFINITY) ? 0.f : __expf(a.m - mm), fb = (b.m == -INFINITY) ? 0.f : __expf(b.m - mm);
        a.s = a.s * fa + b.s * fb;
        a.u = a.u * fa + b.u * fb;
        a.m = mm;
        if (b.key > a.key || (b.key == a.key && b.idx < a.idx)) { a.key = b.key; a.z = b.z; a.idx = b.idx; }
      }
      p.head_part[(int64_t)n_tile * p.M + m0 + tkn] = a;
    }
  }
}

// merge the per-tile head statistics of one token (fixed order -> deterministic)
__global__ void __launch_bounds__(128) head_combine_kernel(const HeadPart* __restrict__ part, int n_tiles, int64_t M,
                                                          const float* __restrict__ picked, int has_targets,
                                                          float* __restrict__ lp_target, float* __restrict__ entropy,
                                                          float* __restrict__ lse_out, int32_t* __restrict__ ids,
                                                          float* __restrict__ lp_sampled) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t tok = blockIdx.x;
  HeadPart a{-INFINITY, 0.f, 0.f, -INFINITY, 0.f, 0x7fffffff};
  auto merge = [](HeadPart& x, const HeadPart& y) {
    const float mm = fmaxf(x.m, y.m);
    const float fx = (x.m == -INFINITY) ? 0.f : __expf(x.m - mm), fy = (y.m == -INFINITY) ? 0.f : __expf(y.m - mm);
    x.s = x.s * fx + y.s * fy;
    x.u = x.u * fx + y.u * fy;
    x.m = mm;
    if (y.key > x.key || (y.key == x.key && y.idx < x.idx)) { x.key = y.key; x.z = y.z; x.idx = y.idx; }
  };
  for (int t = threadIdx.x; t < n_tiles; t += 128) merge(a, part[(int64_t)t * M + tok]);
  __shared__ HeadPart s_a[128];
  s_a[threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    HeadPart r = s_a[0];
    for (int i = 1; i < 128; ++i) merge(r, s_a[i]);
    const float lse = r.m + logf(r.s);
    if (lse_out) lse_out[tok] = lse;
    if (entropy) entropy[tok] = lse - r.u / r.s;
    if (lp_target && has_targets) lp_target[tok] = picked[tok] - lse;
    if (ids) ids[tok] = r.idx;
    if (lp_sampled) lp_sampled[tok] = r.z - lse;
  }
}

template <int kNTile>
int launch_gemm(const CUtensorMap& tw, const CUtensorMap& twl, const CUtensorMap& tx, const GemmParams& p,
                cudaStream_t stream) {
  using L = SmemLayout<kNTile>;
  const bool lo = p.has_lo != 0;
  int n_stages = L::stages(lo);
  if (kNTile >= 128) {  // compute-bound shapes (prefill / training): one CTA per SM with the deepest ring that fits
    n_stages = (200 * 1024) / L::stage_bytes(lo);
    if (n_stages > 8) n_stages = 8;
    if (n_stages < 2) n_stages = 2;
  }
  const int smem = L::ring_bytes(n_stages, lo) + 1024 /*align slack*/ + 8 * (2 * n_stages) + 16;
  auto kernel = p.head ? gemm_swapab_kernel<kNTile, true> : gemm_swapab_kernel<kNTile, false>;
  static SmemAttr smem_attr[2] = {};
  PRL_CUDA(ensure_smem(kernel, smem, smem_attr[p.head ? 1 : 0]));
  const int64_t feat_tiles = p.swiglu_I ? p.swiglu_I / 64 : (p.N + kBlockM - 1) / kBlockM;
  dim3 grid((unsigned)(feat_tiles * ((p.M + kNTile - 1) / kNTile)), (unsigned)p.split_k, 1);
  PRL_CUDA(launch_pdl(kernel, grid, dim3(kThreads), (size_t)smem, stream, tw, twl, tx, p, n_stages));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

// Weight tensor map.  Row-major: [N rows, K cols].  Tiled: the same bytes seen as [(N/128)*(K/64)*128 rows, 64 cols]
// — tile (n_tile, kb) is one contiguous 16 KB block, fetched by a single sequential TMA box.
int make_weight_tmap(CUtensorMap* out, const void* W, int64_t N, int64_t K, int tiled) {
  if (!tiled) return make_tmap_2d_bf16(out, W, (uint64_t)K, (uint64_t)N, (uint64_t)K * 2, kBlockK, kBlockM);
  if (N % kBlockM != 0 || K % kBlockK != 0) {
    set_error("tiled weights need N %% 128 == 0 and K %% 64 == 0 (N=%lld K=%lld)", (long long)N, (long long)K);
    return PRL_ERR_INVALID;
  }
  return make_tmap_2d_bf16(out, W, kBlockK, (uint64_t)(N / kBlockM) * (uint64_t)(K / kBlockK) * kBlockM, kBlockK * 2,
                           kBlockK, kBlockM);
}

int pick_ntile(int64_t M) {
  if (M <= 16) return 16;
  if (M <= 32) return 32;
  if (M <= 64) return 64;
  if (M <= 128) return 128;
  return 256;
}

}  // namespace
}  // namespace prl

using namespace prl;

extern "C" int prl_gemm_set_smem_budget_kb(int32_t kb) {
  PRL_CHECK_ARG(kb >= 48 && kb <= 220, "prl_gemm_set_smem_budget_kb: 48..220 KB");
  g_smem_budget = kb * 1024;
  return PRL_OK;
}

extern "C" int prl_gemm_set_tiled_weights(int32_t on) {
  g_tiled_weights = on ? 1 : 0;
  return PRL_OK;
}

extern "C" int prl_gemm_auto_split_k(int64_t M, int64_t N, int64_t K) {
  if (M <= 0 || N <= 0 || K <= 0) return 1;
  const int sms = num_sms();
  const int64_t tiles = ((N + kBlockM - 1) / kBlockM) * ((M + pick_ntile(M) - 1) / pick_ntile(M));
  const int kblocks = (int)((K + kBlockK - 1) / kBlockK);
  if (tiles >= sms) return 1;
  int best = 1;
  double best_eff = 0.0;
  for (int s = 1; s <= 16 && s <= kblocks; ++s) {
    if (kblocks / s < 4) break;  // keep at least 4 k-blocks per CTA so the pipeline fills
    const int64_t ctas = tiles * s;
    const int64_t waves = (ctas + sms - 1) / sms;
    const double eff = (double)ctas / (double)(waves * sms);
    if (eff > best_eff + 0.03) { best_eff = eff; best = s; }
  }
  return best;
}

static int gemm_splitk_impl(const void* W, const void* W_lo, const void* X, int64_t M, int64_t N, int64_t K,
                            int32_t split_k, float* partials, float* peer_partials, prl_stream_t stream_);

// Token-step gate_up GEMM with SiLU(gate) * up in its epilogue (sampler side, M <= 128 tokens, no split-K: 2 I / 128 tiles
// already fill the SMs): act[M, I] bf16 = the bits prl_gemm_bf16_splitk(split_k = 1) + prl_silu_mul produce, one launch and
// no [M, 2 I] fp32 tile in between.  W = gate_up_proj [2 I, K] as stored (gate rows first).
extern "C" int prl_gemm_swiglu_decode(const void* W, const void* X, int64_t M, int64_t I, int64_t K, void* act_bf16,
                                      prl_stream_t stream_) {
  PRL_CHECK_ARG(W && X && act_bf16, "prl_gemm_swiglu_decode: NULL argument");
  PRL_CHECK_ARG(M >= 1 && M <= 128 && I >= 64 && I % 64 == 0 && K >= 8 && K % 8 == 0,
                "prl_gemm_swiglu_decode: need 1 <= M <= 128, I %% 64 == 0, K %% 8 == 0 (M=%lld I=%lld K=%lld)", (long long)M,
                (long long)I, (long long)K);
  PRL_CHECK_ARG(!g_tiled_weights, "prl_gemm_swiglu_decode: not available with pre-tiled weights");
  const int nt = pick_ntile(M);
  GemmParams p = {};
  p.M = M; p.N = 2 * I; p.K = K; p.kblocks = (int)((K + kBlockK - 1) / kBlockK); p.split_k = 1;
  p.swiglu_I = I; p.act = (__nv_bfloat16*)act_bf16;
  CUtensorMap tw, tx;
  int rc = make_tmap_2d_bf16(&tw, W, (uint64_t)K, (uint64_t)(2 * I), (uint64_t)K * 2, kBlockK, 64);   // 64-row boxes
  if (rc) return rc;
  rc = make_tmap_2d_bf16(&tx, X, (uint64_t)K, (uint64_t)M, (uint64_t)K * 2, kBlockK, (uint32_t)nt);
  if (rc) return rc;
  cudaStream_t stream = (cudaStream_t)stream_;
  switch (nt) {
    case 16: return launch_gemm<16>(tw, tw, tx, p, stream);
    case 32: return launch_gemm<32>(tw, tw, tx, p, stream);
    case 64: return launch_gemm<64>(tw, tw, tx, p, stream);
    default: return launch_gemm<128>(tw, tw, tx, p, stream);
  }
}

extern "C" int prl_gemm_bf16_splitk(const void* W, const void* W_lo, const void* X, int64_t M, int64_t N, int64_t K,
                                    int32_t split_k, float* partials, prl_stream_t stream_) {
  return gemm_splitk_impl(W, W_lo, X, M, N, K, split_k, partials, nullptr, stream_);
}

extern "C" int prl_gemm_bf16_splitk_peer(const void* W, const void* X, int64_t M, int64_t N, int64_t K, int32_t split_k,
                                         float* partials, float* peer_partials, prl_stream_t stream_) {
  PRL_CHECK_ARG(peer_partials, "prl_gemm_bf16_splitk_peer: NULL peer buffer");
  return gemm_splitk_impl(W, nullptr, X, M, N, K, split_k, partials, peer_partials, stream_);
}

static int gemm_splitk_impl(const void* W, const void* W_lo, const void* X, int64_t M, int64_t N, int64_t K,
                            int32_t split_k, float* partials, float* peer_partials, prl_stream_t stream_) {
  PRL_CHECK_ARG(W && X && partials, "prl_gemm_bf16_splitk: NULL argument");
  PRL_CHECK_ARG(M >= 1 && N >= 1 && K >= 8 && K % 8 == 0, "prl_gemm_bf16_splitk: need M,N >= 1 and K %% 8 == 0 (M=%lld N=%lld K=%lld)",
                (long long)M, (long long)N, (long long)K);
  const int kblocks = (int)((K + kBlockK - 1) / kBlockK);
  if (split_k <= 0) split_k = prl_gemm_auto_split_k(M, N, K);
  PRL_CHECK_ARG(split_k <= kblocks, "prl_gemm_bf16_splitk: split_k %d > k-blocks %d", split_k, kblocks);
  const int nt = pick_ntile(M);
  GemmParams p = {};
  p.M = M; p.N = N; p.K = K; p.kblocks = kblocks; p.split_k = split_k; p.has_lo = W_lo ? 1 : 0; p.partials = partials;
  p.peer_partials = peer_partials;
  p.tiled = g_tiled_weights;
  CUtensorMap tw, twl, tx;
  int rc = make_weight_tmap(&tw, W, N, K, p.tiled);
  if (rc) return rc;
  rc = make_weight_tmap(&twl, W_lo ? W_lo : W, N, K, p.tiled);
  if (rc) return rc;
  rc = make_tmap_2d_bf16(&tx, X, (uint64_t)K, (uint64_t)M, (uint64_t)K * 2, kBlockK, (uint32_t)nt);
  if (rc) return rc;
  cudaStream_t stream = (cudaStream_t)stream_;
  switch (nt) {
    case 16: return launch_gemm<16>(tw, twl, tx, p, stream);
    case 32: return launch_gemm<32>(tw, twl, tx, p, stream);
    case 64: return launch_gemm<64>(tw, twl, tx, p, stream);
    case 128: return launch_gemm<128>(tw, twl, tx, p, stream);
    default: return launch_gemm<256>(tw, twl, tx, p, stream);
  }
}

extern "C" size_t prl_head_workspace_bytes(int64_t M, int64_t V) {
  const int64_t tiles = (V + kBlockM - 1) / kBlockM;
  return (size_t)(tiles * M) * sizeof(HeadPart) + (size_t)M * sizeof(float) + 64;
}

extern "C" int prl_head_logprob(const void* W, const void* W_lo, const void* X, int64_t M, int64_t V, int64_t K,
                                float temperature, const int64_t* targets, int32_t greedy, uint64_t seed, uint32_t step,
                                float* logprob_target, float* entropy, float* lse, int32_t* sampled_ids,
                                float* sampled_logprobs, void* workspace, size_t workspace_bytes,
                                prl_stream_t stream_) {
  PRL_CHECK_ARG(W && X && workspace, "prl_head_logprob: NULL argument");
  PRL_CHECK_ARG(M >= 1 && V >= 1 && K >= 8 && K % 8 == 0, "prl_head_logprob: need M,V >= 1 and K %% 8 == 0");
  PRL_CHECK_ARG(temperature > 0.f, "prl_head_logprob: temperature must be > 0");
  PRL_CHECK_ARG(!logprob_target || targets, "prl_head_logprob: logprob_target needs targets");
  PRL_CHECK_ARG(workspace_bytes >= prl_head_workspace_bytes(M, V), "prl_head_logprob: workspace too small");
  if (M > kBlockM && !sampled_ids && !sampled_logprobs && !g_tiled_weights) {
    // many tokens, statistics only (learner forward, reference-logprob scoring): 128 x 256 tiles, token-per-thread
    // epilogue (csrc/gemm_tn.cu)
    return head_logprob_tn(W, W_lo, X, M, V, K, temperature, targets, logprob_target, entropy, lse, workspace,
                           (cudaStream_t)stream_);
  }
  const int nt = pick_ntile(M);
  const int64_t tiles = (V + kBlockM - 1) / kBlockM;
  GemmParams p = {};
  p.M = M; p.N = V; p.K = K; p.kblocks = (int)((K + kBlockK - 1) / kBlockK); p.split_k = 1; p.has_lo = W_lo ? 1 : 0;
  p.head = 1; p.inv_temp = 1.f / temperature; p.targets = targets; p.greedy = greedy; p.seed = seed; p.step = step;
  p.head_part = (HeadPart*)workspace;
  p.picked = (float*)((char*)workspace + (size_t)(tiles * M) * sizeof(HeadPart));
  p.tiled = g_tiled_weights;
  CUtensorMap tw, twl, tx;
  int rc = make_weight_tmap(&tw, W, V, K, p.tiled);
  if (rc) return rc;
  rc = make_weight_tmap(&twl, W_lo ? W_lo : W, V, K, p.tiled);
  if (rc) return rc;
  rc = make_tmap_2d_bf16(&tx, X, (uint64_t)K, (uint64_t)M, (uint64_t)K * 2, kBlockK, (uint32_t)nt);
  if (rc) return rc;
  cudaStream_t stream = (cudaStream_t)stream_;
  switch (nt) {
    case 16: rc = launch_gemm<16>(tw, twl, tx, p, stream); break;
    case 32: rc = launch_gemm<32>(tw, twl, tx, p, stream); break;
    case 64: rc = launch_gemm<64>(tw, twl, tx, p, stream); break;
    case 128: rc = launch_gemm<128>(tw, twl, tx, p, stream); break;
    default: rc = launch_gemm<256>(tw, twl, tx, p, stream); break;
  }
  if (rc) return rc;
  PRL_CUDA(launch_pdl(head_combine_kernel, dim3((unsigned)M), dim3(128), 0, stream, (const HeadPart*)p.head_part,
                      (int)tiles, M, (const float*)p.picked, targets ? 1 : 0, logprob_target, entropy, lse, sampled_ids,
                      sampled_logprobs));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}
