// wgmma GEMM for the compute-bound shapes of the learner (hot path 2) and of prefill / scoring:
//
//   C[M, N] (=|+=) A[M, K] * B[N, K]^T  (+ bias[N]) (+ residual[M, N])     bf16 operands, fp32 accumulation
//
// replaces the cuBLAS GEMMs behind the HF Qwen2 forward/backward that rl_step drives
// (pipelinerl/finetune/rl/__init__.py:190-207 forward; finetune_loop.py:716-725 backward): with K-major ("TN")
// operands the same kernel serves
//   forward   Y  = X  * W^T            A = X [T, in],        B = W [out, in]
//   dgrad     dX = dY * W              A = dY [T, out],      B = W [out, in] read as stored (MN-major B)
//   wgrad     dW += dY^T * X           A = dY^T (MN-major),  B = X^T (MN-major)     (fp32 accumulate epilogue)
//
// One CTA owns a 128 x 256 output tile: a TMA producer warp stages A rows [128) and B rows [256) of the tile per 64-wide
// k-block (SWIZZLE_128B, 4-stage ring, 48 KB/stage), two consumer warpgroups each run wgmma m64n256k16 on 64 of the A
// rows with fp32 accumulators in registers.  After the mainloop the accumulators go through the drained ring to shared
// memory so that every epilogue thread owns ONE output row and half of its columns, and writes contiguous row segments
// (16-byte stores).  CTAs walk the tiles in an L2-friendly order (8 row-tiles x all column tiles per super-group).
//
// Tensor-core bound: flops = 2 M N K; algorithmic bytes = 2 (M K + N K) + out bytes.
#include "prl_common.cuh"
#include "tc_ptx.cuh"

namespace prl {
namespace {

constexpr int kTileM = 128;     // output rows per CTA (two wgmma M = 64 halves)
constexpr int kTileN = 256;     // output columns per CTA (wgmma N)
constexpr int kHalf = 128;      // operand rows per TMA box
constexpr int kBK = 64;         // bf16 per k-block row = one 128-B swizzle atom
constexpr int kStages = 4;
constexpr int kABytes = kTileM * kBK * 2;          // 16 KB
constexpr int kStageBytes = kABytes + kTileN * kBK * 2;  // 48 KB
constexpr int kMnChunkBytes = 64 * kBK * 2;        // one 64(MN) x 64(k) box of an MN-major operand: 8 KB
constexpr int kEpiLd = kTileN + 4;                 // fp32 accumulator tile [128][260] in the drained ring
static_assert(kTileM * kEpiLd * 4 <= kStages * kStageBytes, "epilogue tile must fit in the ring");
constexpr int kSmemTN = kStages * kStageBytes + 1024 + 8 * (2 * kStages) + 16;
constexpr int kThreadsTN = 288;
constexpr int kGroupM = 8;      // row tiles per raster super-group

struct TnParams {
  int64_t M, N, K;
  int kblocks;
  int k_wrap;        // k-blocks >= k_wrap read B from the SECOND tensor map and A from k-block (kb - k_wrap): C = A B^T + A B2^T
                     // in one accumulation (fp32-equivalent lm_head: B = bf16 hi part, B2 = bf16 lo residual)
  int m_tiles, n_tiles;
  int a_mn, b_mn;    // operand stored MN-major: A as [K, M] / B as [K, N] row-major (no transposed copy needed)
  void* C;
  int64_t ldc;
  int c_f32;         // 1: fp32 output, 0: bf16 output
  int accumulate;    // C += (fp32 only)
  const __nv_bfloat16* bias;      // [N] or NULL
  const __nv_bfloat16* residual;  // [M, ldr] or NULL
  int64_t ldr;
  float alpha;
  // SwiGLU epilogue (swiglu_I > 0): B = [gate rows | up rows] of gate_up_proj; the pair's two CTAs stage the gate rows and
  // the up rows of the SAME 128 features, so one accumulator row holds gate (columns 0..127) and up (128..255):
  //   act[row, f] = silu(gate) * up   is written from the epilogue (bf16), gate_up itself to C only when C != NULL
  int64_t swiglu_I;
  int swiglu_fp32;      // 1: SiLU(gate) * up of the fp32 ACCUMULATORS (the sampler's rounding points, decode_ops.cu silu_mul_kernel)
  __nv_bfloat16* act;      // [M, ld_act]
  int64_t ld_act;
  // head epilogue (kHead): logits never leave the SM
  const int64_t* targets;  // [M] or NULL
  float4* head_part;       // [n_tiles, M]: (max, sum exp, sum exp*z, target logit or -inf) of one 256-column vocabulary tile
  // head BACKWARD epilogue (kHead, dz != NULL): the logits tile is turned into d loss / d logits in registers and only its
  // bf16 value reaches HBM -- dz[row, col] = inv_T * (g_lp * ([col == target] - p) - g_ent * p * (log p + H))
  __nv_bfloat16* dz;       // [M, ld_dz]
  int64_t ld_dz;
  const float* bwd_lse;    // [M] natural-log logsumexp of the scaled logits (forward)
  const float* bwd_ent;    // [M] entropy (forward) or NULL
  const float* bwd_g_lp;   // [M] d loss / d logprob, or NULL (treated as 0)
  const float* bwd_g_ent;  // [M] d loss / d entropy, or NULL
  // SiLU * up BACKWARD epilogue (dgu != NULL; N = I, requires I % 32 == 0): this GEMM's output tile IS d act; the epilogue
  // reads gate / up of the forward and writes d gate | d up -- d act never reaches HBM
  const __nv_bfloat16* bwd_gu;   // [M, ld_gu] gate | up of the forward
  __nv_bfloat16* dgu;            // [M, ld_gu] d gate | d up
  int64_t ld_gu;
};

__device__ __forceinline__ void tile_coords(int t, const TnParams& p, int& tm, int& tn) {
  const int per_group = kGroupM * p.n_tiles;
  const int g = t / per_group;
  const int first_m = g * kGroupM;
  const int rows = (p.m_tiles - first_m) < kGroupM ? (p.m_tiles - first_m) : kGroupM;
  const int r = t - g * per_group;
  tm = first_m + r % rows;
  tn = r / rows;
}

// Warp roles (288 threads): warps 0..7 = two consumer warpgroups, warp 8 = TMA producer.
template <bool kHead, int kAmn, int kBmn>
__global__ void __launch_bounds__(kThreadsTN, 1)
gemm_tn_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
               const __grid_constant__ CUtensorMap tm_b2, TnParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + (uint32_t)(kStages * kStageBytes);
  auto full_bar = [&](int s) { return bar_base + 8u * (uint32_t)s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (uint32_t)(kStages + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int tm, tn;
  tile_coords((int)blockIdx.x, p, tm, tn);

  if (threadIdx.x == 256) {
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(full_bar(s), 1);
      ptx::mbar_init(empty_bar(s), 2);   // one elected thread of each consumer warpgroup
    }
    ptx::fence_barrier_init();
    ptx::fence_proxy_async();
    ptx::prefetch_tensormap(&tm_a);
    ptx::prefetch_tensormap(&tm_b);
  }
  __syncthreads();

  if (warp == 8) {
    // ===== TMA producer =====
    if (lane == 0) {
      const int a_row = tm * kTileM;
      // B rows of the tile in two 128-row halves; SwiGLU: the gate rows and the up rows of the SAME 128 features
      const int b_row0 = p.swiglu_I ? tn * kHalf : tn * kTileN;
      const int b_row1 = p.swiglu_I ? (int)p.swiglu_I + tn * kHalf : tn * kTileN + kHalf;
      for (int kb = 0; kb < p.kblocks; ++kb) {
        const int s = kb % kStages;
        ptx::mbar_wait(empty_bar(s), (uint32_t)(((kb / kStages) & 1) ^ 1));
        ptx::mbar_arrive_expect_tx(full_bar(s), (uint32_t)kStageBytes);
        const uint32_t a_dst = smem_base + (uint32_t)(s * kStageBytes);
        const uint32_t b_dst = a_dst + kABytes;
        const bool second = kb >= p.k_wrap;                 // hi + lo operand streams (K-major operands only)
        const int kk = (second ? kb - p.k_wrap : kb) * kBK;
        const CUtensorMap* tb = second ? &tm_b2 : &tm_b;
        if (!kAmn) {
          ptx::tma_load_2d(a_dst, &tm_a, kk, a_row, full_bar(s), ptx::kEvictNormal);
        } else {  // two 64(MN) x 64(k) boxes: inner coordinate = MN index, outer = k
          ptx::tma_load_2d(a_dst, &tm_a, a_row, kk, full_bar(s), ptx::kEvictNormal);
          ptx::tma_load_2d(a_dst + kMnChunkBytes, &tm_a, a_row + 64, kk, full_bar(s), ptx::kEvictNormal);
        }
        if (!kBmn) {
          ptx::tma_load_2d(b_dst, tb, kk, b_row0, full_bar(s), ptx::kEvictNormal);
          ptx::tma_load_2d(b_dst + kHalf * kBK * 2, tb, kk, b_row1, full_bar(s), ptx::kEvictNormal);
        } else {
          ptx::tma_load_2d(b_dst, tb, b_row0, kk, full_bar(s), ptx::kEvictNormal);
          ptx::tma_load_2d(b_dst + kMnChunkBytes, tb, b_row0 + 64, kk, full_bar(s), ptx::kEvictNormal);
          ptx::tma_load_2d(b_dst + 2 * kMnChunkBytes, tb, b_row1, kk, full_bar(s), ptx::kEvictNormal);
          ptx::tma_load_2d(b_dst + 3 * kMnChunkBytes, tb, b_row1 + 64, kk, full_bar(s), ptx::kEvictNormal);
        }
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg = tile rows [64 wg, 64 wg + 64) x all 256 columns =====
  const int wg = warp >> 2;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  constexpr uint64_t a_step = kAmn ? 128u : 2u, b_step = kBmn ? 128u : 2u;  // K += 16 in (addr >> 4) units
  float acc[kTileN / 2];
#pragma unroll
  for (int e = 0; e < kTileN / 2; ++e) acc[e] = 0.f;
  for (int kb = 0; kb < p.kblocks; ++kb) {
    const int s = kb % kStages;
    ptx::mbar_wait(full_bar(s), (uint32_t)((kb / kStages) & 1));
    const uint32_t a_addr = smem_base + (uint32_t)(s * kStageBytes) + (uint32_t)(wg * kMnChunkBytes);
    const uint32_t b_addr = smem_base + (uint32_t)(s * kStageBytes) + kABytes;
    const uint64_t a_desc = kAmn ? ptx::make_mnmajor_sw128_desc(a_addr, kMnChunkBytes) : ptx::make_kmajor_sw128_desc(a_addr);
    const uint64_t b_desc = kBmn ? ptx::make_mnmajor_sw128_desc(b_addr, kMnChunkBytes) : ptx::make_kmajor_sw128_desc(b_addr);
    ptx::fence_acc(acc);
    ptx::wg_fence();
#pragma unroll
    for (int k = 0; k < kBK / 16; ++k)
      ptx::wgmma_ss<kAmn, kBmn>(acc, a_desc + a_step * (uint64_t)k, b_desc + b_step * (uint64_t)k, 1u);
    ptx::wg_commit();
    ptx::wg_wait<1>();                       // the previous stage's wgmmas are done: release that slot
    if (kb > 0 && wg_leader) ptx::mbar_arrive(empty_bar((kb - 1) % kStages));
  }
  ptx::wg_wait<0>();
  ptx::fence_acc(acc);

  // ---- accumulators -> fp32 tile [128 rows][kEpiLd] in the drained ring ----
  asm volatile("bar.sync 1, 256;" ::: "memory");   // both warpgroups are past their last shared-memory operand read
  float* stile = reinterpret_cast<float*>(smem_raw + (smem_base - ptx::smem_u32(smem_raw)));
  {
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < kTileN / 8; ++j) {
      const int c = 8 * j + 2 * (lane & 3);
      *reinterpret_cast<float2*>(stile + r0 * kEpiLd + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(stile + (r0 + 8) * kEpiLd + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");

  // ===== epilogue: thread = one output row, columns [128 h, 128 h + 128) in 32-column chunks =====
  {
    const int lrow = threadIdx.x & 127;
    const int h = threadIdx.x >> 7;
    const float* srow = stile + lrow * kEpiLd;
    auto ld32 = [&](int c, uint32_t (&r)[32]) {
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        const float4 f = *reinterpret_cast<const float4*>(srow + c + j);
        r[j] = __float_as_uint(f.x); r[j + 1] = __float_as_uint(f.y); r[j + 2] = __float_as_uint(f.z); r[j + 3] = __float_as_uint(f.w);
      }
    };
    {
      const int64_t row = (int64_t)tm * kTileM + lrow;
      const int64_t col0 = (int64_t)tn * kTileN + h * kHalf;
      const bool row_ok = row < p.M;
      if constexpr (kHead) {
        // thread = one token; online softmax statistics over 128 vocabulary columns of the tile, all thread-local
        constexpr float kLog2e = 1.4426950408889634f;
        const int64_t tgt = (p.targets && row_ok) ? p.targets[row] : -1;
        if (p.dz != nullptr) {
          // ---- backward: logits -> d logits (same formula as tail_bwd_kernel, logprob_tail.cu), written as bf16 ----
          const float lse = row_ok ? p.bwd_lse[row] : 0.f;
          const float gl = (p.bwd_g_lp && row_ok) ? p.bwd_g_lp[row] : 0.f;
          const float ge = (p.bwd_g_ent && row_ok) ? p.bwd_g_ent[row] : 0.f;
          const float H = (p.bwd_g_ent && p.bwd_ent && row_ok) ? p.bwd_ent[row] : 0.f;
#pragma unroll 1
          for (int c0 = 0; c0 < kHalf; c0 += 32) {
            if (col0 + c0 >= p.N) break;
            if (!row_ok) continue;
            uint32_t r[32];
            ld32(h * kHalf + c0, r);
            const int64_t col = col0 + c0;
            const int n_ok = (int)((p.N - col) < 32 ? (p.N - col) : 32);
            __nv_bfloat16* dst = p.dz + row * p.ld_dz + col;
            const uint64_t rel = (uint64_t)(tgt - col);
            float g[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              const float lp = __uint_as_float(r[j]) * p.alpha - lse;
              const float pr = __expf(lp);
              float v = -gl * pr - ge * pr * (lp + H);
              if (rel == (uint64_t)j) v += gl;
              g[j] = v * p.alpha;
            }
            if (n_ok == 32) {
#pragma unroll
              for (int j = 0; j < 32; j += 8) {
                uint4 u;
                __nv_bfloat162* hb = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
                for (int e = 0; e < 4; ++e) hb[e] = __floats2bfloat162_rn(g[j + 2 * e], g[j + 2 * e + 1]);
                *reinterpret_cast<uint4*>(dst + j) = u;
              }
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if (j < n_ok) dst[j] = __float2bfloat16_rn(g[j]);
            }
          }
        } else {
        float m = -INFINITY, ssum = 0.f, usum = 0.f, zt = -INFINITY;
#pragma unroll 1
        for (int c0 = 0; c0 < kHalf; c0 += 32) {
          if (col0 + c0 >= p.N) break;
          uint32_t r[32];
          ld32(h * kHalf + c0, r);
          const int64_t col = col0 + c0;
          const int n_ok = (int)((p.N - col) < 32 ? (p.N - col) : 32);
          float z[32];
          float cm = -INFINITY;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            z[j] = (j < n_ok) ? __uint_as_float(r[j]) * p.alpha : -INFINITY;
            cm = fmaxf(cm, z[j]);
          }
          const float m2 = fmaxf(m, cm);
          const float sc = (m == -INFINITY) ? 0.f : exp2f((m - m2) * kLog2e);
          ssum *= sc;
          usum *= sc;
          m = m2;
          const float mb = m * kLog2e;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const float e = exp2f(fmaf(z[j], kLog2e, -mb));  // exp2(-inf) = 0 for the masked tail
            ssum += e;
            usum = fmaf(e, (j < n_ok) ? z[j] : 0.f, usum);
          }
          const uint64_t rel = (uint64_t)(tgt - col);
          if (rel < 32u) {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (rel == (uint64_t)j) zt = z[j];
          }
        }
        if (row_ok) p.head_part[(int64_t)(2 * tn + h) * p.M + row] = make_float4(m, ssum, usum, zt);
        }   // forward statistics
      } else if (p.swiglu_I) {
        // columns 0..127 of the tile = gate, 128..255 = up of features [tn * 128, tn * 128 + 128); thread half h takes
        // features [64 h, 64 h + 64)
        const int64_t f0 = (int64_t)tn * kHalf;
#pragma unroll 1
        for (int c0 = h * 64; c0 < h * 64 + 64; c0 += 32) {
          if (!row_ok) continue;
          uint32_t rg[32], ru[32];
          ld32(c0, rg);
          ld32(kHalf + c0, ru);
          __nv_bfloat16* ap = p.act + row * p.ld_act + f0 + c0;
          __nv_bfloat16* gp = p.C ? reinterpret_cast<__nv_bfloat16*>(p.C) + row * p.ldc + f0 + c0 : nullptr;
#pragma unroll
          for (int j = 0; j < 32; j += 8) {
            uint4 ua, ug, uu;
            __nv_bfloat162* ha = reinterpret_cast<__nv_bfloat162*>(&ua);
            __nv_bfloat162* hg = reinterpret_cast<__nv_bfloat162*>(&ug);
            __nv_bfloat162* hu = reinterpret_cast<__nv_bfloat162*>(&uu);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              // same rounding points as the two-kernel path: gate_up is rounded to bf16 first, SiLU * up is taken of the
              // ROUNDED values (prl_silu_mul_fwd reads the bf16 tensor), so fused and unfused results are bit-identical
              if (p.swiglu_fp32) {   // sampler prefill: identical bits to the fp32 GEMM output + silu_mul_kernel pair
                const float g0 = __uint_as_float(rg[j + 2 * e]), g1 = __uint_as_float(rg[j + 2 * e + 1]);
                const float u0 = __uint_as_float(ru[j + 2 * e]), u1 = __uint_as_float(ru[j + 2 * e + 1]);
                ha[e] = __floats2bfloat162_rn((g0 / (1.f + __expf(-g0))) * u0, (g1 / (1.f + __expf(-g1))) * u1);
                continue;
              }
              hg[e] = __floats2bfloat162_rn(__uint_as_float(rg[j + 2 * e]), __uint_as_float(rg[j + 2 * e + 1]));
              hu[e] = __floats2bfloat162_rn(__uint_as_float(ru[j + 2 * e]), __uint_as_float(ru[j + 2 * e + 1]));
              const float2 g = __bfloat1622float2(hg[e]), u = __bfloat1622float2(hu[e]);
              ha[e] = __floats2bfloat162_rn(g.x / (1.f + __expf(-g.x)) * u.x, g.y / (1.f + __expf(-g.y)) * u.y);
            }
            *reinterpret_cast<uint4*>(ap + j) = ua;
            if (gp) {
              *reinterpret_cast<uint4*>(gp + j) = ug;
              *reinterpret_cast<uint4*>(gp + p.swiglu_I + j) = uu;
            }
          }
        }
      } else {
#pragma unroll 1
      for (int c0 = 0; c0 < kHalf; c0 += 32) {
        if (col0 + c0 >= p.N) break;
        if (!row_ok) continue;
        uint32_t r[32];
        ld32(h * kHalf + c0, r);
        const int64_t col = col0 + c0;
        const bool full = (col + 32 <= p.N);
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]) * p.alpha;
        if (p.bias) {
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (full || col + j < p.N) v[j] += __bfloat162float(p.bias[col + j]);
        }
        if (p.residual) {
          const __nv_bfloat16* rp = p.residual + row * p.ldr + col;
          if (full && ((p.ldr & 7) == 0)) {
#pragma unroll
            for (int j = 0; j < 32; j += 8) {
              const uint4 u = *reinterpret_cast<const uint4*>(rp + j);
              const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float2 f = __bfloat1622float2(h[e]);
                v[j + 2 * e] += f.x;
                v[j + 2 * e + 1] += f.y;
              }
            }
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (col + j < p.N) v[j] += __bfloat162float(rp[j]);
          }
        }
        if (p.dgu != nullptr) {
          // d act tile -> (d gate, d up): same rounding points as the two-kernel path (d act rounded to bf16, then
          // silu_mul_bwd_kernel's arithmetic, learner_ops.cu), so fused and unfused results are bit-identical
          const __nv_bfloat16* gp = p.bwd_gu + row * p.ld_gu + col;
          __nv_bfloat16* dp = p.dgu + row * p.ld_gu + col;
#pragma unroll
          for (int j = 0; j < 32; j += 8) {
            const uint4 ug = *reinterpret_cast<const uint4*>(gp + j);
            const uint4 uu = *reinterpret_cast<const uint4*>(gp + p.N + j);
            const __nv_bfloat162* hg = reinterpret_cast<const __nv_bfloat162*>(&ug);
            const __nv_bfloat162* hu = reinterpret_cast<const __nv_bfloat162*>(&uu);
            uint4 og, ou;
            __nv_bfloat162* dg = reinterpret_cast<__nv_bfloat162*>(&og);
            __nv_bfloat162* du = reinterpret_cast<__nv_bfloat162*>(&ou);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float2 g = __bfloat1622float2(hg[e]), u = __bfloat1622float2(hu[e]);
              const float2 d = __bfloat1622float2(__floats2bfloat162_rn(v[j + 2 * e], v[j + 2 * e + 1]));
              const float s0 = 1.f / (1.f + __expf(-g.x)), s1 = 1.f / (1.f + __expf(-g.y));
              const float l0 = g.x * s0, l1 = g.y * s1;
              du[e] = __floats2bfloat162_rn(d.x * l0, d.y * l1);
              dg[e] = __floats2bfloat162_rn(d.x * u.x * (s0 + l0 * (1.f - s0)), d.y * u.y * (s1 + l1 * (1.f - s1)));
            }
            *reinterpret_cast<uint4*>(dp + j) = og;
            *reinterpret_cast<uint4*>(dp + p.N + j) = ou;
          }
          continue;
        }
        if (p.c_f32) {
          float* cp = reinterpret_cast<float*>(p.C) + row * p.ldc + col;
          if (full && ((p.ldc & 3) == 0)) {
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              float4 o = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
              if (p.accumulate) {
                const float4 old = *reinterpret_cast<const float4*>(cp + j);
                o.x += old.x; o.y += old.y; o.z += old.z; o.w += old.w;
              }
              *reinterpret_cast<float4*>(cp + j) = o;
            }
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (col + j < p.N) cp[j] = p.accumulate ? cp[j] + v[j] : v[j];
          }
        } else {
          __nv_bfloat16* cp = reinterpret_cast<__nv_bfloat16*>(p.C) + row * p.ldc + col;
          if (full && ((p.ldc & 7) == 0)) {
#pragma unroll
            for (int j = 0; j < 32; j += 8) {
              uint4 u;
              __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
              for (int e = 0; e < 4; ++e) h[e] = __floats2bfloat162_rn(v[j + 2 * e], v[j + 2 * e + 1]);
              *reinterpret_cast<uint4*>(cp + j) = u;
            }
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (col + j < p.N) cp[j] = __float2bfloat16(v[j]);
          }
        }
      }
      }  // !kHead
    }
  }
}

// one warp per token: merge the per-tile statistics in a fixed order (lane-strided tiles, then a shuffle tree)
__global__ void __launch_bounds__(128) head_tn_combine_kernel(const float4* __restrict__ part, int n_tiles, int64_t M,
                                                             int has_targets, float* __restrict__ lp_target,
                                                             float* __restrict__ entropy, float* __restrict__ lse_out) {
  const int64_t tok = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (tok >= M) return;
  float m = -INFINITY, s = 0.f, u = 0.f, zt = -INFINITY;
  auto merge = [&](float m2, float s2, float u2, float zt2) {
    const float mm = fmaxf(m, m2);
    const float f1 = (m == -INFINITY) ? 0.f : __expf(m - mm), f2 = (m2 == -INFINITY) ? 0.f : __expf(m2 - mm);
    s = s * f1 + s2 * f2;
    u = u * f1 + u2 * f2;
    m = mm;
    zt = fmaxf(zt, zt2);  // exactly one tile holds the target, the others carry -inf
  };
  for (int t = lane; t < n_tiles; t += 32) {
    const float4 v = part[(int64_t)t * M + tok];
    merge(v.x, v.y, v.z, v.w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    const float u2 = __shfl_xor_sync(0xffffffffu, u, o), z2 = __shfl_xor_sync(0xffffffffu, zt, o);
    merge(m2, s2, u2, z2);
  }
  if (lane == 0) {
    const float lse = m + logf(s);
    if (lse_out) lse_out[tok] = lse;
    if (entropy) entropy[tok] = lse - u / s;
    if (lp_target && has_targets) lp_target[tok] = zt - lse;
  }
}

// bf16 [R, C] -> [C, R]; 64 x 64 tiles through shared memory, 16-byte global accesses on both sides
__global__ void __launch_bounds__(256) transpose_bf16_kernel(const __nv_bfloat16* __restrict__ in, int64_t R, int64_t C,
                                                             int64_t ldi, __nv_bfloat16* __restrict__ out, int64_t ldo) {
  __shared__ __nv_bfloat16 tile[64][64 + 8];
  const int64_t r0 = (int64_t)blockIdx.y * 64, c0 = (int64_t)blockIdx.x * 64;
  const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;  // 8 x 32: each thread moves 8 bf16
  const bool vec_in = ((ldi & 7) == 0) && ((reinterpret_cast<uintptr_t>(in) & 15) == 0);
  const bool vec_out = ((ldo & 7) == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
#pragma unroll
  for (int rr = 0; rr < 64; rr += 32) {
    const int64_t r = r0 + rr + ty, c = c0 + tx * 8;
    if (r < R) {
      if (vec_in && c + 8 <= C) {
        const uint4 u = *reinterpret_cast<const uint4*>(in + r * ldi + c);
        const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(&u);
#pragma unroll
        for (int e = 0; e < 8; ++e) tile[rr + ty][tx * 8 + e] = h[e];
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (c + e < C) tile[rr + ty][tx * 8 + e] = in[r * ldi + c + e];
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int cc = 0; cc < 64; cc += 32) {
    const int64_t c = c0 + cc + ty, r = r0 + tx * 8;  // output row = input column
    if (c < C) {
      __nv_bfloat16 h[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) h[e] = tile[tx * 8 + e][cc + ty];
      if (vec_out && r + 8 <= R) {
        *reinterpret_cast<uint4*>(out + c * ldo + r) = *reinterpret_cast<const uint4*>(h);
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (r + e < R) out[c * ldo + r + e] = h[e];
      }
    }
  }
}

// one CTA per 128 x 256 output tile; the operand majorness is a compile-time property of the wgmma instruction
template <bool kHead, int kAmn, int kBmn>
int launch_tn_t(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tb2, const TnParams& p, cudaStream_t stream) {
  static SmemAttr smem_attr = {};
  PRL_CUDA(ensure_smem(gemm_tn_kernel<kHead, kAmn, kBmn>, kSmemTN, smem_attr));
  const int64_t tiles = (int64_t)p.m_tiles * p.n_tiles;
  PRL_CHECK_ARG(tiles < (1ll << 31), "prl_gemm_tn: too many output tiles");
  gemm_tn_kernel<kHead, kAmn, kBmn><<<dim3((unsigned)tiles), dim3(kThreadsTN), (size_t)kSmemTN, stream>>>(ta, tb, tb2, p);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

int launch_tn(bool head, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tb2, const TnParams& p,
              cudaStream_t stream) {
  if (head) return launch_tn_t<true, 0, 0>(ta, tb, tb2, p, stream);
  if (p.a_mn && p.b_mn) return launch_tn_t<false, 1, 1>(ta, tb, tb2, p, stream);
  if (p.a_mn) return launch_tn_t<false, 1, 0>(ta, tb, tb2, p, stream);
  if (p.b_mn) return launch_tn_t<false, 0, 1>(ta, tb, tb2, p, stream);
  return launch_tn_t<false, 0, 0>(ta, tb, tb2, p, stream);
}

}  // namespace
}  // namespace prl

using namespace prl;

extern "C" int prl_gemm_tn(const void* A, int64_t lda, const void* B, int64_t ldb, int64_t M, int64_t N, int64_t K,
                           void* C, int64_t ldc, int32_t c_is_f32, int32_t accumulate, const void* bias,
                           const void* residual, int64_t ldr, float alpha, prl_stream_t stream_) {
  return prl_gemm_ex(A, lda, 0, B, ldb, 0, M, N, K, C, ldc, c_is_f32, accumulate, bias, residual, ldr, alpha, stream_);
}

extern "C" int prl_gemm_ex(const void* A, int64_t lda, int32_t a_mn_major, const void* B, int64_t ldb,
                           int32_t b_mn_major, int64_t M, int64_t N, int64_t K, void* C, int64_t ldc, int32_t c_is_f32,
                           int32_t accumulate, const void* bias, const void* residual, int64_t ldr, float alpha,
                           prl_stream_t stream_) {
  PRL_CHECK_ARG(A && B && C, "prl_gemm_tn: NULL argument");
  PRL_CHECK_ARG(M >= 1 && N >= 1 && K >= 8, "prl_gemm_tn: need M, N >= 1 and K >= 8 (M=%lld N=%lld K=%lld)", (long long)M,
                (long long)N, (long long)K);
  PRL_CHECK_ARG(lda >= (a_mn_major ? M : K) && ldb >= (b_mn_major ? N : K) && lda % 8 == 0 && ldb % 8 == 0,
                "prl_gemm_tn: operand row strides must cover a row and be multiples of 8 elements (lda=%lld ldb=%lld K=%lld)",
                (long long)lda, (long long)ldb, (long long)K);
  PRL_CHECK_ARG(ldc >= N, "prl_gemm_tn: ldc %lld < N %lld", (long long)ldc, (long long)N);
  PRL_CHECK_ARG(!accumulate || c_is_f32, "prl_gemm_tn: accumulate needs an fp32 output");
  PRL_CHECK_ARG(!residual || ldr >= N, "prl_gemm_tn: ldr %lld < N %lld", (long long)ldr, (long long)N);
  TnParams p = {};
  p.M = M; p.N = N; p.K = K;
  p.kblocks = (int)((K + kBK - 1) / kBK);
  p.k_wrap = p.kblocks;
  p.m_tiles = (int)((M + kTileM - 1) / kTileM);
  p.n_tiles = (int)((N + kTileN - 1) / kTileN);
  p.C = C; p.ldc = ldc; p.c_f32 = c_is_f32; p.accumulate = accumulate;
  p.bias = (const __nv_bfloat16*)bias;
  p.residual = (const __nv_bfloat16*)residual;
  p.ldr = ldr;
  p.alpha = alpha;
  p.a_mn = a_mn_major ? 1 : 0;
  p.b_mn = b_mn_major ? 1 : 0;
  CUtensorMap ta, tb;
  int rc = a_mn_major ? make_tmap_2d_bf16(&ta, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda * 2, 64, kBK)
                      : make_tmap_2d_bf16(&ta, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda * 2, kBK, kHalf);
  if (rc) return rc;
  rc = b_mn_major ? make_tmap_2d_bf16(&tb, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb * 2, 64, kBK)
                  : make_tmap_2d_bf16(&tb, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb * 2, kBK, kHalf);
  if (rc) return rc;
  rc = launch_tn(false, ta, tb, tb, p, (cudaStream_t)stream_);
  if (rc) return rc;
  return PRL_OK;
}

// down_proj dgrad with the backward of SiLU(gate) * up in its epilogue: d gate_up[M, 2 I] from dY[M, H], W_down[H, I] (read as
// stored: MN-major B) and the forward's gate_up[M, 2 I]; d act = dY W_down is never written.  Bit-identical to
// prl_gemm_ex(dY, W_down, b_mn) -> prl_silu_mul_bwd.
extern "C" int prl_gemm_dgrad_swiglu(const void* dY, int64_t ldy, const void* W_down, int64_t ldw, int64_t M, int64_t I,
                                     int64_t H, const void* gate_up, void* d_gate_up, int64_t ld_gu, prl_stream_t stream_) {
  PRL_CHECK_ARG(dY && W_down && gate_up && d_gate_up, "prl_gemm_dgrad_swiglu: NULL argument");
  PRL_CHECK_ARG(M >= 1 && I >= 32 && I % 32 == 0 && H >= 8 && ldy >= H && ldy % 8 == 0 && ldw >= I && ldw % 8 == 0 &&
                ld_gu >= 2 * I && ld_gu % 8 == 0, "prl_gemm_dgrad_swiglu: bad shape (M=%lld I=%lld H=%lld)", (long long)M,
                (long long)I, (long long)H);
  TnParams p = {};
  p.M = M; p.N = I; p.K = H;
  p.kblocks = (int)((H + kBK - 1) / kBK);
  p.k_wrap = p.kblocks;
  p.m_tiles = (int)((M + kTileM - 1) / kTileM);
  p.n_tiles = (int)((I + kTileN - 1) / kTileN);
  p.alpha = 1.f;
  p.b_mn = 1;
  p.bwd_gu = (const __nv_bfloat16*)gate_up; p.dgu = (__nv_bfloat16*)d_gate_up; p.ld_gu = ld_gu;
  CUtensorMap ta, tb;
  int rc = make_tmap_2d_bf16(&ta, dY, (uint64_t)H, (uint64_t)M, (uint64_t)ldy * 2, kBK, kHalf);
  if (rc) return rc;
  rc = make_tmap_2d_bf16(&tb, W_down, (uint64_t)I, (uint64_t)H, (uint64_t)ldw * 2, 64, kBK);
  if (rc) return rc;
  rc = launch_tn(false, ta, tb, tb, p, (cudaStream_t)stream_);
  if (rc) return rc;
  return PRL_OK;
}

// gate_up GEMM with the SwiGLU activation in its epilogue: act[M, I] = silu(X Wg^T) * (X Wu^T), W = [Wg; Wu] ([2 I, K]).
// gate_up (bf16 [M, 2 I], may be NULL) is written as well when the backward will need it.
static int gemm_swiglu_impl(const void* X, int64_t ldx, const void* W, int64_t ldw, int64_t M, int64_t I, int64_t K,
                            void* act, int64_t ld_act, void* gate_up, int64_t ld_gu, int fp32_act, prl_stream_t stream_);

extern "C" int prl_gemm_swiglu(const void* X, int64_t ldx, const void* W, int64_t ldw, int64_t M, int64_t I, int64_t K,
                               void* act, int64_t ld_act, void* gate_up, int64_t ld_gu, prl_stream_t stream_) {
  return gemm_swiglu_impl(X, ldx, W, ldw, M, I, K, act, ld_act, gate_up, ld_gu, 0, stream_);
}

// Sampler form (chunked prefill / scoring): act = bf16(SiLU(gate) * up) taken of the fp32 accumulators -- the rounding points
// of the token step's GEMM + silu_mul_kernel pair, so a prompt prefilled in chunks and a prompt decoded token by token see
// the same MLP arithmetic; gate_up itself is never written.
extern "C" int prl_gemm_swiglu_f32(const void* X, int64_t ldx, const void* W, int64_t ldw, int64_t M, int64_t I, int64_t K,
                                   void* act, int64_t ld_act, prl_stream_t stream_) {
  return gemm_swiglu_impl(X, ldx, W, ldw, M, I, K, act, ld_act, nullptr, 0, 1, stream_);
}

static int gemm_swiglu_impl(const void* X, int64_t ldx, const void* W, int64_t ldw, int64_t M, int64_t I, int64_t K,
                            void* act, int64_t ld_act, void* gate_up, int64_t ld_gu, int fp32_act, prl_stream_t stream_) {
  PRL_CHECK_ARG(X && W && act, "prl_gemm_swiglu: NULL argument");
  PRL_CHECK_ARG(M >= 1 && I >= kHalf && I % kHalf == 0 && K >= 8, "prl_gemm_swiglu: need I %% 128 == 0 (M=%lld I=%lld K=%lld)",
                (long long)M, (long long)I, (long long)K);
  PRL_CHECK_ARG(ldx >= K && ldw >= K && ldx % 8 == 0 && ldw % 8 == 0 && ld_act >= I && ld_act % 8 == 0 &&
                    (!gate_up || (ld_gu >= 2 * I && ld_gu % 8 == 0)),
                "prl_gemm_swiglu: row strides must cover a row and be multiples of 8 elements");
  TnParams p = {};
  p.M = M; p.N = 2 * I; p.K = K;
  p.kblocks = (int)((K + kBK - 1) / kBK);
  p.k_wrap = p.kblocks;
  p.m_tiles = (int)((M + kTileM - 1) / kTileM);
  p.n_tiles = (int)(I / kHalf);
  p.C = gate_up; p.ldc = ld_gu; p.alpha = 1.f;
  p.swiglu_I = I; p.swiglu_fp32 = fp32_act; p.act = (__nv_bfloat16*)act; p.ld_act = ld_act;
  CUtensorMap ta, tb;
  int rc = make_tmap_2d_bf16(&ta, X, (uint64_t)K, (uint64_t)M, (uint64_t)ldx * 2, kBK, kHalf);
  if (rc) return rc;
  rc = make_tmap_2d_bf16(&tb, W, (uint64_t)K, (uint64_t)(2 * I), (uint64_t)ldw * 2, kBK, kHalf);
  if (rc) return rc;
  rc = launch_tn(false, ta, tb, tb, p, (cudaStream_t)stream_);
  if (rc) return rc;
  return PRL_OK;
}

namespace prl {
// fused output head for many tokens (M > 128): logprob of the target, entropy and logsumexp of softmax(X W^T / T)
// without storing logits.  Called by prl_head_logprob (gemm_tc.cu).  workspace: 2 ceil(V/256) * M float4 (one per
// 128-column half of a tile).
int head_logprob_tn(const void* W, const void* W_lo, const void* X, int64_t M, int64_t V, int64_t K, float temperature,
                    const int64_t* targets, float* logprob_target, float* entropy, float* lse, void* workspace,
                    cudaStream_t stream) {
  TnParams p = {};
  p.M = M; p.N = V; p.K = K;
  p.kblocks = (int)((K + kBK - 1) / kBK);
  p.k_wrap = p.kblocks;
  if (W_lo) p.kblocks *= 2;          // logits = X W_hi^T + X W_lo^T accumulated in the same registers
  p.m_tiles = (int)((M + kTileM - 1) / kTileM);
  p.n_tiles = (int)((V + kTileN - 1) / kTileN);
  p.alpha = 1.f / temperature;
  p.targets = targets;
  p.head_part = (float4*)workspace;
  CUtensorMap ta, tb, tb2;
  int rc = make_tmap_2d_bf16(&ta, X, (uint64_t)K, (uint64_t)M, (uint64_t)K * 2, kBK, kHalf);
  if (rc) return rc;
  rc = make_tmap_2d_bf16(&tb, W, (uint64_t)K, (uint64_t)V, (uint64_t)K * 2, kBK, kHalf);
  if (rc) return rc;
  rc = make_tmap_2d_bf16(&tb2, W_lo ? W_lo : W, (uint64_t)K, (uint64_t)V, (uint64_t)K * 2, kBK, kHalf);
  if (rc) return rc;
  rc = launch_tn(true, ta, tb, tb2, p, stream);
  if (rc) return rc;
  head_tn_combine_kernel<<<(unsigned)((M + 3) / 4), 128, 0, stream>>>((const float4*)workspace, 2 * p.n_tiles, M,
                                                                      targets ? 1 : 0, logprob_target, entropy, lse);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}
}  // namespace prl

// Backward of the fused output head without materialised logits: dz[M, ld_dz] (bf16) = d loss / d logits for every row, from
// ONE GEMM (X W_hi^T + X W_lo^T accumulated together, as the forward) whose epilogue applies
//   dz = inv_T * (g_lp * (onehot(target) - p) - g_ent * p * (log p + H)),   p = exp(z * inv_T - lse)
// in registers (reference: autograd through logits/T -> log_softmax / entropy, rl/__init__.py:207-233).  dz is the operand of
// the dX and dW GEMMs that follow; fp32 logits, fp32 d logits and the cast pass never exist.
extern "C" int prl_head_dlogits(const void* W, const void* W_lo, const void* X, int64_t M, int64_t V, int64_t K,
                                float temperature, const int64_t* targets, const float* lse, const float* entropy,
                                const float* g_logprobs, const float* g_entropy, void* dz_bf16, int64_t ld_dz,
                                prl_stream_t stream_) {
  using namespace prl;
  PRL_CHECK_ARG(W && X && targets && lse && dz_bf16, "prl_head_dlogits: NULL argument");
  PRL_CHECK_ARG(M >= 1 && V >= 1 && K >= 8 && K % 8 == 0 && ld_dz >= V && ld_dz % 8 == 0 && temperature > 0.f,
                "prl_head_dlogits: bad shape (M=%lld V=%lld K=%lld ld_dz=%lld)", (long long)M, (long long)V, (long long)K,
                (long long)ld_dz);
  PRL_CHECK_ARG(!g_entropy || entropy, "prl_head_dlogits: g_entropy needs the forward entropy");
  TnParams p = {};
  p.M = M; p.N = V; p.K = K;
  p.kblocks = (int)((K + kBK - 1) / kBK);
  p.k_wrap = p.kblocks;
  if (W_lo) p.kblocks *= 2;
  p.m_tiles = (int)((M + kTileM - 1) / kTileM);
  p.n_tiles = (int)((V + kTileN - 1) / kTileN);
  p.alpha = 1.f / temperature;
  p.targets = targets;
  p.dz = (__nv_bfloat16*)dz_bf16; p.ld_dz = ld_dz;
  p.bwd_lse = lse; p.bwd_ent = entropy; p.bwd_g_lp = g_logprobs; p.bwd_g_ent = g_entropy;
  CUtensorMap ta, tb, tb2;
  int rc = make_tmap_2d_bf16(&ta, X, (uint64_t)K, (uint64_t)M, (uint64_t)K * 2, kBK, kHalf);
  if (rc) return rc;
  rc = make_tmap_2d_bf16(&tb, W, (uint64_t)K, (uint64_t)V, (uint64_t)K * 2, kBK, kHalf);
  if (rc) return rc;
  rc = make_tmap_2d_bf16(&tb2, W_lo ? W_lo : W, (uint64_t)K, (uint64_t)V, (uint64_t)K * 2, kBK, kHalf);
  if (rc) return rc;
  rc = launch_tn(true, ta, tb, tb2, p, (cudaStream_t)stream_);
  if (rc) return rc;
  return PRL_OK;
}

extern "C" int prl_transpose_bf16(const void* in, int64_t rows, int64_t cols, int64_t ld_in, void* out, int64_t ld_out,
                                  prl_stream_t stream_) {
  PRL_CHECK_ARG(in && out, "prl_transpose_bf16: NULL argument");
  PRL_CHECK_ARG(rows >= 1 && cols >= 1 && ld_in >= cols && ld_out >= rows, "prl_transpose_bf16: bad shape / strides");
  dim3 grid((unsigned)((cols + 63) / 64), (unsigned)((rows + 63) / 64));
  PRL_CHECK_ARG(grid.y <= 65535, "prl_transpose_bf16: too many row tiles (%u)", grid.y);
  transpose_bf16_kernel<<<grid, 256, 0, (cudaStream_t)stream_>>>((const __nv_bfloat16*)in, rows, cols, ld_in,
                                                                 (__nv_bfloat16*)out, ld_out);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}
