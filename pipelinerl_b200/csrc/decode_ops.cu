// Hot path (1): the small fused kernels around the wgmma GEMMs of one token step.
//
// They replace, for the reference's sampler (vLLM behind pipelinerl/async_llm.py:134),
// vLLM's fused_add_rms_norm / rotary_embedding / reshape_and_cache_flash / silu_and_mul
// custom ops and the sampler + processed_logprobs path (conf/base.yaml:65).  Each one
// consumes the fp32 split-K partials of the preceding GEMM (summed in split order, so
// results are deterministic) and emits the bf16 operand of the next GEMM, i.e. the
// split-K reduction, bias, RoPE, KV-page write, residual add, RMSNorm and SiLU*mul are
// all "epilogue" work on L2-resident activations, never a separate pass over weights.
//
// Numerics contract (restated by oracle/decode_oracle.py): residual stream fp32,
// GEMM operands bf16, accumulation fp32, RoPE angles fp32, KV cache bf16.
#include "prl_common.cuh"
#include <math.h>

namespace prl {
namespace {

// Software prefetch ACROSS kernels through the 126 MB L2: a small epilogue kernel asks L2 to fetch the weights
// of an upcoming latency-bound GEMM (qkv / o_proj: 26-33 MB) while the long HBM-bound kernel in between
// (attention, gate_up, down) runs, so that GEMM then streams from L2 instead of paying DRAM latency cold.
// Lines are requested evict_last so the evict_first streams of the kernels in between do not displace them.
__device__ __forceinline__ void l2_prefetch_range(const void* ptr, size_t bytes, size_t tid, size_t nthreads) {
  if (!ptr) return;
  const char* base = static_cast<const char*>(ptr);
  const size_t n_lines = bytes >> 7;
  for (size_t i = tid; i < n_lines; i += nthreads)
    asm volatile("prefetch.global.L2::evict_last [%0];" ::"l"(base + (i << 7)));
}

__device__ __forceinline__ float block_sum(float v, float* s_red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  float t = 0.f;
  const int nw = (blockDim.x + 31) >> 5;
  for (int i = 0; i < nw; ++i) t += s_red[i];
  __syncthreads();
  return t;
}

// ---- embedding gather + RMSNorm ------------------------------------------------------
// h[b,:] = embed[token[b],:] ; x[b,:] = bf16(h * rsqrt(mean(h^2) + eps) * g)
__global__ void __launch_bounds__(256) embed_rmsnorm_kernel(const int32_t* __restrict__ tokens,
                                                           const __nv_bfloat16* __restrict__ embed,
                                                           const __nv_bfloat16* __restrict__ gamma, float eps, int H,
                                                           int vocab, float* __restrict__ h,
                                                           __nv_bfloat16* __restrict__ x) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_red[32];
  const int b = blockIdx.x;
  int tok = tokens[b];
  if (tok < 0 || tok >= vocab) tok = 0;
  const __nv_bfloat16* row = embed + (int64_t)tok * H;
  float ss = 0.f;
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    const float v = __bfloat162float(row[i]);
    h[(int64_t)b * H + i] = v;
    ss += v * v;
  }
  const float tot = block_sum(ss, s_red);
  const float r = rsqrtf(tot / (float)H + eps);
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    const float v = __bfloat162float(row[i]);
    x[(int64_t)b * H + i] = __float2bfloat16_rn(v * r * __bfloat162float(gamma[i]));
  }
}

// ---- split-K reduce + residual add + RMSNorm --------------------------------------------
// h[b,:] += sum_s part[s,b,:] ; x[b,:] = bf16(rmsnorm(h) * g)
// One block per token; each thread owns float4 column groups, issues the residual load and all
// n_split partial loads back to back (independent, L2-resident), so the kernel costs about one
// L2 round trip + one block reduction instead of a serial chain per element.
constexpr int kMaxSplitUnroll = 8;
__global__ void __launch_bounds__(1024) residual_rmsnorm_kernel(const float* __restrict__ part, int n_split, int B,
                                                               int H, const __nv_bfloat16* __restrict__ gamma,
                                                               float eps, float* __restrict__ h,
                                                               __nv_bfloat16* __restrict__ x, const void* pf_ptr,
                                                               size_t pf_bytes) {
  pdl_launch_dependents();
  l2_prefetch_range(pf_ptr, pf_bytes, (size_t)blockIdx.x * blockDim.x + threadIdx.x, (size_t)gridDim.x * blockDim.x);
  pdl_wait();
  extern __shared__ float s_row[];  // H floats (only used when a thread owns more than one group)
  __shared__ float s_red[32];
  const int b = blockIdx.x;
  const int H4 = H >> 2;
  float4* hrow = reinterpret_cast<float4*>(h + (int64_t)b * H);
  float ss = 0.f;
  float4 keep = make_float4(0.f, 0.f, 0.f, 0.f);
  const bool single = H4 <= (int)blockDim.x;
  for (int i = threadIdx.x; i < H4; i += blockDim.x) {
    float4 v = hrow[i];
    for (int s = 0; s < n_split; s += kMaxSplitUnroll) {
      float4 p[kMaxSplitUnroll];
#pragma unroll
      for (int u = 0; u < kMaxSplitUnroll; ++u)
        if (s + u < n_split) p[u] = reinterpret_cast<const float4*>(part + ((int64_t)(s + u) * B + b) * H)[i];
#pragma unroll
      for (int u = 0; u < kMaxSplitUnroll; ++u)
        if (s + u < n_split) { v.x += p[u].x; v.y += p[u].y; v.z += p[u].z; v.w += p[u].w; }
    }
    hrow[i] = v;
    if (single) keep = v; else reinterpret_cast<float4*>(s_row)[i] = v;
    ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  const float tot = block_sum(ss, s_red);
  const float r = rsqrtf(tot / (float)H + eps);
  for (int i = threadIdx.x; i < H4; i += blockDim.x) {
    const float4 v = single ? keep : reinterpret_cast<const float4*>(s_row)[i];
    const uint2 gw = reinterpret_cast<const uint2*>(gamma)[i];
    const float g0 = bf16_bits_to_float(gw.x & 0xffffu), g1 = bf16_bits_to_float(gw.x >> 16);
    const float g2 = bf16_bits_to_float(gw.y & 0xffffu), g3 = bf16_bits_to_float(gw.y >> 16);
    const uint32_t o0 = float_to_bf16_bits(v.x * r * g0), o1 = float_to_bf16_bits(v.y * r * g1);
    const uint32_t o2 = float_to_bf16_bits(v.z * r * g2), o3 = float_to_bf16_bits(v.w * r * g3);
    reinterpret_cast<uint2*>(x + (int64_t)b * H)[i] = make_uint2(o0 | (o1 << 16), o2 | (o3 << 16));
  }
}

// ---- split-K reduce + bias (+ per-head q/k RMSNorm) + RoPE + KV-page write ------------------------
// part [n_split, B, (n_q + 2 n_kv) * 128]; one block per (token, head), 64 threads = 64 rotation pairs.
// q -> q_out [B, n_q, 128] bf16 ; k, v -> cache rows ((layer*2 + kv) * n_pages + page) * n_kv * PAGE + kvh*PAGE + slot
// kNorm (Qwen3): every q and k head is RMS-normalised over its 128 values and scaled by the layer's gain (q_gamma for
// q heads, k_gamma for k heads) before the rotation, all in fp32; v heads are untouched.  Values are rounded to bf16
// once, after RoPE.  The kNorm = false instantiation is the Qwen2 step, unchanged.

// Sum of squares of one head's 128 values, held as pairs (x1, x2) by 64 consecutive threads (two whole warps): one
// butterfly per warp, then the two warp sums in order.  Both kernels below reduce in exactly this order, so they stay
// bit-identical.  Block-wide: every thread of the block must call it.
__device__ __forceinline__ float head_sumsq(float x1, float x2, float* s_ss) {
  float v = warp_sum(__fadd_rn(__fmul_rn(x1, x1), __fmul_rn(x2, x2)));
  const int warp = threadIdx.x >> 5;
  __syncthreads();  // s_ss may still be read from the previous head
  if ((threadIdx.x & 31) == 0) s_ss[warp] = v;
  __syncthreads();
  const int w0 = warp & ~1;
  return __fadd_rn(s_ss[w0], s_ss[w0 + 1]);
}

__device__ __forceinline__ float head_rstd(float ss, float eps) { return rsqrtf(__fmaf_rn(ss, 1.f / 128.f, eps)); }

template <bool kNorm>
__global__ void __launch_bounds__(64) qkv_rope_cache_kernel(const float* __restrict__ part, int n_split, int B,
                                                           const __nv_bfloat16* __restrict__ bias,
                                                           const __nv_bfloat16* __restrict__ q_gamma,
                                                           const __nv_bfloat16* __restrict__ k_gamma, float eps,
                                                           int n_q, int n_kv,
                                                           const int32_t* __restrict__ positions,
                                                           const int32_t* __restrict__ block_table, int max_blocks,
                                                           const int32_t* __restrict__ row_slot,
                                                           const float* __restrict__ inv_freq_tab,
                                                           __nv_bfloat16* __restrict__ q_out,
                                                           __nv_bfloat16* __restrict__ kv_cache, int64_t n_pages,
                                                           int layer, int page_size, const void* pf_ptr,
                                                           size_t pf_bytes) {
  pdl_launch_dependents();
  l2_prefetch_range(pf_ptr, pf_bytes, ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * blockDim.x + threadIdx.x,
                    (size_t)gridDim.x * gridDim.y * blockDim.x);
  pdl_wait();
  constexpr int D = 128;
  const int b = blockIdx.x, head = blockIdx.y, i = threadIdx.x;  // i in [0, 64)
  const int n_heads = n_q + 2 * n_kv;
  const int64_t ncol = (int64_t)n_heads * D;
  const int col = head * D + i;
  float x1 = 0.f, x2 = 0.f;
  for (int s = 0; s < n_split; ++s) {
    const float* p = part + ((int64_t)s * B + b) * ncol;
    x1 += p[col];
    x2 += p[col + 64];
  }
  if (bias) {
    x1 += __bfloat162float(bias[col]);
    x2 += __bfloat162float(bias[col + 64]);
  }
  const int pos = positions[b];
  const bool is_v = head >= n_q + n_kv;  // uniform over the block
  float o1 = x1, o2 = x2;
  if (!is_v) {
    if constexpr (kNorm) {
      __shared__ float s_ss[2];
      const float r = head_rstd(head_sumsq(x1, x2, s_ss), eps);
      const __nv_bfloat16* g = head < n_q ? q_gamma : k_gamma;
      x1 = x1 * r * __bfloat162float(g[i]);
      x2 = x2 * r * __bfloat162float(g[i + 64]);
    }
    // NeoX-style rotation of the pair (i, i + 64); inv_freq[i] = 1 / theta^(2i/128) is tabulated by the host
    // with the exact fp32 expression HF's rotary embedding uses, the angle is an fp32 product as there
    const float inv_freq = inv_freq_tab[i];
    float sn, cs;
    sincosf((float)pos * inv_freq, &sn, &cs);
    o1 = x1 * cs - x2 * sn;
    o2 = x2 * cs + x1 * sn;
  }
  if (head < n_q) {
    __nv_bfloat16* q = q_out + ((int64_t)b * n_q + head) * D;
    q[i] = __float2bfloat16_rn(o1);
    q[i + 64] = __float2bfloat16_rn(o2);
  } else {
    const int kv = is_v ? 1 : 0;
    const int kvh = is_v ? head - n_q - n_kv : head - n_q;
    const int slot_row = row_slot ? row_slot[b] : b;
    const int page = block_table[(int64_t)slot_row * max_blocks + pos / page_size];
    const int slot = pos % page_size;
    const int64_t row = (((int64_t)(layer * 2 + kv) * n_pages + page) * n_kv + kvh) * page_size + slot;
    __nv_bfloat16* dst = kv_cache + row * D;
    dst[i] = __float2bfloat16_rn(o1);
    dst[i + 64] = __float2bfloat16_rn(o2);
  }
}

// Same arithmetic, laid out for MANY rows (prefill chunks): one block walks whole token rows, the row's 64
// (cos, sin) pairs are computed once (the per-head kernel above recomputes them for each of the n_q + 2 n_kv heads)
// and every thread handles (head, pair) items with coalesced 4-byte loads.  Bitwise identical results.
// blockDim must be a multiple of 64, so that each head's 64 pairs are two whole warps of one pass (head_sumsq).
template <bool kNorm>
__global__ void __launch_bounds__(256) qkv_rope_cache_rows_kernel(const float* __restrict__ part, int n_split, int B,
                                                                const __nv_bfloat16* __restrict__ bias,
                                                                const __nv_bfloat16* __restrict__ q_gamma,
                                                                const __nv_bfloat16* __restrict__ k_gamma, float eps,
                                                                int n_q, int n_kv,
                                                                const int32_t* __restrict__ positions,
                                                                const int32_t* __restrict__ block_table, int max_blocks,
                                                                const int32_t* __restrict__ row_slot,
                                                                const float* __restrict__ inv_freq_tab,
                                                                __nv_bfloat16* __restrict__ q_out,
                                                                __nv_bfloat16* __restrict__ kv_cache, int64_t n_pages,
                                                                int layer, int page_size) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int D = 128;
  __shared__ float s_cs[64], s_sn[64];
  __shared__ float s_ss[kNorm ? 256 / 32 : 1];
  const int n_heads = n_q + 2 * n_kv;
  const int64_t ncol = (int64_t)n_heads * D;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    const int pos = positions[b];
    __syncthreads();
    if (threadIdx.x < 64) {
      float sn, cs;
      sincosf((float)pos * inv_freq_tab[threadIdx.x], &sn, &cs);
      s_cs[threadIdx.x] = cs;
      s_sn[threadIdx.x] = sn;
    }
    __syncthreads();
    const int slot_row = row_slot ? row_slot[b] : b;
    const int page = block_table[(int64_t)slot_row * max_blocks + pos / page_size];
    const int slot = pos % page_size;
    // every thread runs every pass (the norm's reduction is block-wide); threads past the last head only idle
    for (int w0 = 0; w0 < n_heads * 64; w0 += blockDim.x) {
      const int w = w0 + threadIdx.x;
      const bool live = w < n_heads * 64;
      const int head = w >> 6, i = w & 63;
      const int col = head * D + i;
      float x1 = 0.f, x2 = 0.f;
      if (live) {
        for (int s = 0; s < n_split; ++s) {
          const float* p = part + ((int64_t)s * B + b) * ncol;
          x1 += p[col];
          x2 += p[col + 64];
        }
        if (bias) {
          x1 += __bfloat162float(bias[col]);
          x2 += __bfloat162float(bias[col + 64]);
        }
      }
      const bool is_v = head >= n_q + n_kv;
      if constexpr (kNorm) {
        const float r = head_rstd(head_sumsq(x1, x2, s_ss), eps);
        if (live && !is_v) {
          const __nv_bfloat16* g = head < n_q ? q_gamma : k_gamma;
          x1 = x1 * r * __bfloat162float(g[i]);
          x2 = x2 * r * __bfloat162float(g[i + 64]);
        }
      }
      if (!live) continue;
      float o1 = x1, o2 = x2;
      if (!is_v) {
        const float cs = s_cs[i], sn = s_sn[i];
        o1 = x1 * cs - x2 * sn;
        o2 = x2 * cs + x1 * sn;
      }
      if (head < n_q) {
        __nv_bfloat16* q = q_out + ((int64_t)b * n_q + head) * D;
        q[i] = __float2bfloat16_rn(o1);
        q[i + 64] = __float2bfloat16_rn(o2);
      } else {
        const int kv = is_v ? 1 : 0;
        const int kvh = is_v ? head - n_q - n_kv : head - n_q;
        const int64_t row = (((int64_t)(layer * 2 + kv) * n_pages + page) * n_kv + kvh) * page_size + slot;
        __nv_bfloat16* dst = kv_cache + row * D;
        dst[i] = __float2bfloat16_rn(o1);
        dst[i + 64] = __float2bfloat16_rn(o2);
      }
    }
  }
}

// ---- split-K reduce + SiLU(gate) * up ------------------------------------------------------
// part [n_split, B, 2I] (gate columns first, as in the fused gate_up weight) -> act [B, I] bf16; 4 columns/thread
__global__ void __launch_bounds__(256) silu_mul_kernel(const float* __restrict__ part, int n_split, int B, int I,
                                                      __nv_bfloat16* __restrict__ act, const void* pf_ptr,
                                                      size_t pf_bytes) {
  pdl_launch_dependents();
  l2_prefetch_range(pf_ptr, pf_bytes, ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * blockDim.x + threadIdx.x,
                    (size_t)gridDim.x * gridDim.y * blockDim.x);
  pdl_wait();
  const int b = blockIdx.y;
  const int i4 = blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 * 4 >= I) return;
  float4 g = make_float4(0.f, 0.f, 0.f, 0.f), u = g;
  for (int s = 0; s < n_split; ++s) {
    const float* p = part + ((int64_t)s * B + b) * 2 * I;
    const float4 a = reinterpret_cast<const float4*>(p)[i4];
    const float4 c = reinterpret_cast<const float4*>(p + I)[i4];
    g.x += a.x; g.y += a.y; g.z += a.z; g.w += a.w;
    u.x += c.x; u.y += c.y; u.z += c.z; u.w += c.w;
  }
  auto f = [](float gg, float uu) { return (gg / (1.f + __expf(-gg))) * uu; };
  const uint32_t o0 = float_to_bf16_bits(f(g.x, u.x)), o1 = float_to_bf16_bits(f(g.y, u.y));
  const uint32_t o2 = float_to_bf16_bits(f(g.z, u.z)), o3 = float_to_bf16_bits(f(g.w, u.w));
  reinterpret_cast<uint2*>(act + (int64_t)b * I)[i4] = make_uint2(o0 | (o1 << 16), o2 | (o3 << 16));
}

// ---- sampler + in-kernel logprob capture ----------------------------------------------------
// logits [B, V] fp32 (split-K already 1 for the head).  Per token: z = logits / T;
// id = argmax(z + Gumbel noise) (== a sample from softmax(z)), or argmax(z) when greedy;
// logprob = z[id] - logsumexp(z)  (vLLM's processed_logprobs at top_p = 1, top_k = -1).
struct ArgMax { float v; int i; };
__device__ __forceinline__ ArgMax better(ArgMax a, ArgMax b) {
  // ties -> lowest index, like torch.argmax
  if (b.v > a.v || (b.v == a.v && b.i < a.i)) return b;
  return a;
}

constexpr int kSampleParts = 16;   // CTAs per row: 64 rows x 16 = 1024 CTAs keep every SM busy
constexpr int kSampleThreads = 256;
struct SamplePartial { float m, s, v, z; int i; int pad[3]; };  // z = logit/T of the best key (logprob without re-reading logits)

// phase 1: each CTA scans a contiguous 1/16 of the vocabulary of one row
__global__ void __launch_bounds__(kSampleThreads) sample_partial_kernel(const float* __restrict__ logits, int V,
                                                                       float inv_temp, int greedy, uint64_t seed,
                                                                       uint32_t step, int vocab_offset,
                                                                       SamplePartial* __restrict__ part,
                                                                       const float* __restrict__ inv_temp_rows,
                                                                       const uint8_t* __restrict__ greedy_rows) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, pi = blockIdx.y;
  // per-sequence sampling parameters (requests of different LLM handles share an engine: train T=1, eval greedy ...)
  if (inv_temp_rows != nullptr) inv_temp = inv_temp_rows[b];
  if (greedy_rows != nullptr) greedy = greedy_rows[b];
  const float* z = logits + (int64_t)b * V;
  const int per = (V + kSampleParts - 1) / kSampleParts;
  const int lo = pi * per, hi = (lo + per < V) ? lo + per : V;
  float m = -INFINITY, s = 0.f;
  ArgMax best{-INFINITY, 0x7fffffff};
  float best_z = 0.f;
  for (int i = lo + threadIdx.x; i < hi; i += kSampleThreads) {
    const float zi = z[i] * inv_temp;
    // a -inf logit (a min_tokens ban) adds nothing; guarded, as __expf(-inf - -inf) would be NaN
    if (zi > m) { s = s * __expf(m - zi) + 1.f; m = zi; } else if (zi != -INFINITY) { s += __expf(zi - m); }
    const int gid = vocab_offset + i;   // global vocabulary id (vocab-parallel head: this rank owns a slice)
    const float key = greedy ? zi : zi + gumbel(seed, step, (uint32_t)b, (uint32_t)gid);
    const ArgMax cand{key, gid};
    const ArgMax nb = better(best, cand);
    if (nb.i != best.i) best_z = zi;
    best = nb;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    const float mm = fmaxf(m, m2);
    s = (m == -INFINITY ? 0.f : s * __expf(m - mm)) + (m2 == -INFINITY ? 0.f : s2 * __expf(m2 - mm));
    m = mm;
    ArgMax o2{__shfl_xor_sync(0xffffffffu, best.v, o), __shfl_xor_sync(0xffffffffu, best.i, o)};
    const float z2 = __shfl_xor_sync(0xffffffffu, best_z, o);
    const ArgMax nb = better(best, o2);
    if (nb.i != best.i) best_z = z2;
    best = nb;
  }
  __shared__ float s_m[8], s_s[8], s_v[8], s_z[8];
  __shared__ int s_i[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { s_m[warp] = m; s_s[warp] = s; s_v[warp] = best.v; s_i[warp] = best.i; s_z[warp] = best_z; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float M = -INFINITY, S = 0.f, bz = 0.f;
    ArgMax bb{-INFINITY, 0x7fffffff};
    for (int w = 0; w < kSampleThreads / 32; ++w) {
      const float mm = fmaxf(M, s_m[w]);
      S = (M == -INFINITY ? 0.f : S * __expf(M - mm)) + (s_m[w] == -INFINITY ? 0.f : s_s[w] * __expf(s_m[w] - mm));
      M = mm;
      const ArgMax nb = better(bb, ArgMax{s_v[w], s_i[w]});
      if (nb.i != bb.i) bz = s_z[w];
      bb = nb;
    }
    SamplePartial out;
    out.m = M; out.s = S; out.v = bb.v; out.z = bz; out.i = bb.i; out.pad[0] = out.pad[1] = out.pad[2] = 0;
    part[b * kSampleParts + pi] = out;
  }
}

// phase 2: merge the partials of a row — 16 per vocabulary slice, `n_groups` slices ([group][B][16]; one group
// unless the head is vocab-parallel over tensor-parallel ranks) — in a fixed order; emit id and log-probability
__global__ void sample_finalize_kernel(int B, int n_groups, const SamplePartial* __restrict__ part,
                                       int32_t* __restrict__ out_ids, float* __restrict__ out_logprobs) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float M = -INFINITY, S = 0.f, bz = 0.f;
  ArgMax bb{-INFINITY, 0x7fffffff};
  for (int g = 0; g < n_groups; ++g)
    for (int k = 0; k < kSampleParts; ++k) {
      const SamplePartial q = part[((int64_t)g * B + b) * kSampleParts + k];
      const float mm = fmaxf(M, q.m);
      S = (M == -INFINITY ? 0.f : S * __expf(M - mm)) + (q.m == -INFINITY ? 0.f : q.s * __expf(q.m - mm));
      M = mm;
      const ArgMax nb = better(bb, ArgMax{q.v, q.i});
      if (nb.i != bb.i) bz = q.z;
      bb = nb;
    }
  out_ids[b] = bb.i;
  out_logprobs[b] = bz - (M + logf(S));
}

// ---- tensor-parallel synchronisation through peer memory (no NCCL on the token path) -----------------------------
// signal: after this rank's P2P stores (previous kernels of the stream) bump a counter in the PEER's memory.
__global__ void tp_signal_kernel(unsigned long long* peer_flag) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) {
    __threadfence_system();
    atomicAdd_system(peer_flag, 1ull);
  }
}
// wait: spin until the local counter (bumped by the peer) reaches epoch * per_step + k, i.e. the peer has issued
// its k-th signal of this token step.  `epoch` counts completed steps on this rank (tp_epoch_kernel).
__global__ void tp_wait_kernel(const unsigned long long* flag, const unsigned long long* epoch, int per_step, int k) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) {
    const unsigned long long want = (*epoch) * (unsigned long long)per_step + (unsigned long long)k;
    const long long t0 = clock64();
    while (true) {
      unsigned long long v;
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(flag) : "memory");
      if (v >= want) break;
      if (clock64() - t0 > 20000000000LL) asm volatile("trap;");  // ~10 s: the peer died
    }
  }
}
__global__ void tp_epoch_kernel(unsigned long long* epoch) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) *epoch += 1ull;
}

// ---- stop strings: vLLM's IncrementalDetokenizer.update + check_stop_strings, on bytes ------------------------------
// The detokenizer appends the token's text and looks for the first string, in request order, with an occurrence that
// ends inside the new text.  On bytes that is: the string whose KMP automaton completes a match while it consumes this
// token's bytes (a UTF-8 string can only match at character boundaries, and a character completes with its last
// byte).  Tokens up to min_tokens are fed, so a match may start inside them, but they never report (`checked` false).
// The automaton state of each (slot, string) is the length of the longest prefix of the string that ends the bytes fed
// so far; no text is kept.  Returns the index of the matching string, or -1.
__device__ __forceinline__ int match_stop_strings(const prl_stop_strings& st, int b, int id, bool core_stop,
                                                  bool checked) {
  const int ns = min(st.n_stop_str[b], st.max_stop_str);
  if (ns <= 0 || id < 0 || id >= st.vocab) return -1;
  const uint8_t flags = st.stop_str_flags[b];
  // include_stop_str_in_output=False: the eos / stop id that ended the request is not detokenized
  if (core_stop && !(flags & 1)) return -1;
  // skip_special_tokens=True: a special token's text is empty
  if ((flags & 2) && st.tok_special[id]) return -1;
  const uint8_t* bytes = st.tok_bytes + st.tok_offsets[id];
  const int nb = st.tok_offsets[id + 1] - st.tok_offsets[id];
  const int64_t row = (int64_t)b * st.max_stop_str;
  for (int j = 0; j < ns; ++j) {
    const uint8_t* s = st.stop_str + (row + j) * st.stop_str_stride;
    const int16_t* fail = st.stop_str_fail + (row + j) * st.stop_str_stride;
    const int len = st.stop_str_len[row + j];
    int q = st.stop_str_state[row + j];
    bool hit = false;
    for (int i = 0; i < nb; ++i) {
      const uint8_t c = bytes[i];
      while (q > 0 && s[q] != c) q = fail[q - 1];
      if (s[q] == c) ++q;
      if (q == len) {
        hit = true;
        q = fail[len - 1];
      }
    }
    st.stop_str_state[row + j] = q;
    if (hit && checked) return j;  // the slot finishes: the later strings' states are not needed any more
  }
  return -1;
}

// ---- advance the per-sequence state after a step (device-side, no host round trip) -------------
// Slot b just processed the token at position pos.  While the next position is still inside the
// prompt the sample is discarded and the next prompt token is fed (prefill-by-decode); afterwards
// the sampled id / logprob are appended to the slot's output ring and become the next input.
__global__ void advance_kernel(prl_engine_state st, prl_stop_strings ss) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= st.B) return;
  if (!st.active[b]) return;
  const int pos = st.positions[b];
  const int next = pos + 1;
  if (next < st.prompt_len[b]) {
    st.tokens[b] = st.prompt_buf[(int64_t)b * st.prompt_stride + next];
  } else {
    const int n = st.gen_count[b];
    const int id = st.sampled[b];
    st.out_ids[(int64_t)b * st.out_stride + n] = id;
    st.out_logprobs[(int64_t)b * st.out_stride + n] = st.sampled_logprobs[b];
    st.gen_count[b] = n + 1;
    st.tokens[b] = id;
    const bool ignore = st.ignore_eos || (st.ignore_eos_rows != nullptr && st.ignore_eos_rows[b]);
    // check_stop returns early while the slot holds fewer than min_tokens outputs (min_tokens <= max_new)
    const int min_tok = ss.min_tokens != nullptr ? ss.min_tokens[b] : 0;
    const bool core = n + 1 >= min_tok;
    const bool eos = core && (id == st.eos_id) && !ignore;
    // vLLM's check_stop order: the primary eos, then the slot's stop set, then the length cap, so a stop id drawn as
    // the last allowed token reports "stop"
    bool stop = eos;
    int reason = -1;
    if (core && !eos && st.stop_ids != nullptr) {
      const int32_t* row = st.stop_ids + (int64_t)b * st.stop_stride;
      const int m = min(st.n_stop[b], st.stop_stride);
      for (int j = 0; j < m; ++j) {
        if (row[j] == id) {
          stop = true;
          reason = id;
          break;
        }
      }
    }
    int match = -1;
    if (ss.tok_bytes != nullptr) match = match_stop_strings(ss, b, id, stop, n + 1 > min_tok);
    if (match >= 0) stop = true;  // OutputProcessor: a matched string makes it "stop", even over "length"
    if (stop || n + 1 >= st.max_new[b]) {
      st.finished[b] = stop ? 1 : 2;  // 1 = stop, 2 = length
      if (st.stop_reason != nullptr) st.stop_reason[b] = match >= 0 ? -1 : reason;
      if (ss.stop_str_match != nullptr) ss.stop_str_match[b] = match;
      st.active[b] = 0;
      st.seq_lens[b] = 0;            // the slot stops reading its KV
      st.positions[b] = 0;
      return;
    }
  }
  st.positions[b] = next;
  st.seq_lens[b] = next + 1;
}

// ---- min_tokens: -inf on the slot's stop ids while it holds fewer than min_tokens outputs ----------------------------
// One warp per row; a few ids per row.  Runs after the head GEMM, before the sampler reads the row.
__global__ void ban_min_tokens_kernel(float* __restrict__ logits, int B, int V, const int32_t* __restrict__ gen_count,
                                      const int32_t* __restrict__ min_tokens, const int32_t* __restrict__ ban_ids,
                                      int ban_stride, const int32_t* __restrict__ n_ban) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B || gen_count[b] >= min_tokens[b]) return;
  const int m = min(n_ban[b], ban_stride);
  for (int j = threadIdx.x & 31; j < m; j += 32) {
    const int id = ban_ids[(int64_t)b * ban_stride + j];
    if (id >= 0 && id < V) logits[(int64_t)b * V + id] = -INFINITY;
  }
}

// ---- penalties and min_p: vLLM's apply_penalties, then MinPLogitsProcessor after the temperature ---------------------
// One CTA per row; the row is streamed once for the penalties (logits, counts, prompt-mask words) and once more for
// min_p.  Each penalty step is its own fp32 rounding, as vLLM's three tensor ops are (no FMA contraction).  Counts and
// mask words are read through L2 (__ldcg): this CTA has just written them with plain stores and atomics.
constexpr int kPenThreads = 1024;

__device__ __forceinline__ float penalize(float l, int c, uint32_t prompt_word, int i, float r, float inv_r, float f,
                                          float pr) {
  if (c > 0 || ((prompt_word >> (i & 31)) & 1u)) l = __fmul_rn(l, l > 0.f ? inv_r : r);  // unmasked: vLLM's * 1.0
  l = __fsub_rn(l, __fmul_rn(f, (float)c));
  return __fsub_rn(l, __fmul_rn(pr, c > 0 ? 1.f : 0.f));
}

__device__ __forceinline__ float zmax4(float m, float4 l, float inv_temp) {
  return fmaxf(fmaxf(m, fmaxf(__fmul_rn(l.x, inv_temp), __fmul_rn(l.y, inv_temp))),
               fmaxf(__fmul_rn(l.z, inv_temp), __fmul_rn(l.w, inv_temp)));
}

__global__ void __launch_bounds__(kPenThreads) penalties_kernel(prl_penalties p) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, V = p.V;
  const float pr = p.presence[b], f = p.frequency[b], r = p.repetition[b];
  const float min_p = p.greedy[b] ? 0.f : p.min_p[b];   // vLLM resets min_p for greedy requests
  const bool pen = pr != 0.f || f != 0.f || r != 1.f;
  const bool use_min_p = min_p > 0.f;
  if (!pen && !use_min_p) return;
  float* row = p.logits + (int64_t)b * V;
  const float inv_temp = p.inv_temp[b];
  // 16-byte rows: four ids per load, so that one CTA keeps enough bytes in flight to stream its row
  const bool vec = (V & 3) == 0 && ((uintptr_t)p.logits & 15) == 0 && ((uintptr_t)p.counts & 15) == 0;
  float4* row4 = reinterpret_cast<float4*>(row);
  const int V4 = vec ? V >> 2 : 0;
  float m = -INFINITY;
  if (pen) {
    int32_t* cnt = p.counts + (int64_t)b * V;
    const int W = (V + 31) >> 5;
    uint32_t* mask = p.prompt_mask + (int64_t)b * W;
    int seen = p.seen[b];
    const int n_out = min(p.gen_count[b], p.out_stride);
    if (seen < 0) {                       // first launch for this request: fresh counts, its own prompt mask
      for (int i = threadIdx.x; i < V; i += kPenThreads) cnt[i] = 0;
      for (int i = threadIdx.x; i < W; i += kPenThreads) mask[i] = 0u;
      __syncthreads();
      const int32_t* prompt = p.prompt_buf + (int64_t)b * p.prompt_stride;
      const int n_prompt = min(p.prompt_len[b], p.prompt_stride);
      for (int i = threadIdx.x; i < n_prompt; i += kPenThreads) {
        const int id = prompt[i];
        if (id >= 0 && id < V) atomicOr(&mask[id >> 5], 1u << (id & 31));
      }
      seen = 0;
    }
    const int32_t* out = p.out_ids + (int64_t)b * p.out_stride;
    for (int i = seen + threadIdx.x; i < n_out; i += kPenThreads) {
      const int id = out[i];
      if (id >= 0 && id < V) atomicAdd(&cnt[id], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) p.seen[b] = max(seen, n_out);
    const float inv_r = __fdiv_rn(1.f, r);
    const int4* cnt4 = reinterpret_cast<const int4*>(cnt);
#pragma unroll 2
    for (int j = threadIdx.x; j < V4; j += kPenThreads) {
      float4 l = row4[j];
      const int4 c = __ldcg(cnt4 + j);
      const uint32_t w = __ldcg(mask + (j >> 3));
      const int i = j << 2;
      l.x = penalize(l.x, c.x, w, i, r, inv_r, f, pr);
      l.y = penalize(l.y, c.y, w, i + 1, r, inv_r, f, pr);
      l.z = penalize(l.z, c.z, w, i + 2, r, inv_r, f, pr);
      l.w = penalize(l.w, c.w, w, i + 3, r, inv_r, f, pr);
      row4[j] = l;
      m = zmax4(m, l, inv_temp);
    }
    for (int i = (V4 << 2) + threadIdx.x; i < V; i += kPenThreads) {
      const float l = penalize(row[i], __ldcg(cnt + i), __ldcg(mask + (i >> 5)), i, r, inv_r, f, pr);
      row[i] = l;
      m = fmaxf(m, __fmul_rn(l, inv_temp));
    }
  } else {
#pragma unroll 4
    for (int j = threadIdx.x; j < V4; j += kPenThreads) m = zmax4(m, row4[j], inv_temp);
    for (int i = (V4 << 2) + threadIdx.x; i < V; i += kPenThreads) m = fmaxf(m, __fmul_rn(row[i], inv_temp));
  }
  if (!use_min_p) return;
  // p_i < min_p * max p  <=>  exp(z_i - m) < min_p
  __shared__ float s_max[kPenThreads / 32];
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = m;
  __syncthreads();
  m = -INFINITY;
  for (int w = 0; w < kPenThreads / 32; ++w) m = fmaxf(m, s_max[w]);
  // each thread reads back the elements it wrote in pass 1 (same index mapping)
#pragma unroll 2
  for (int j = threadIdx.x; j < V4; j += kPenThreads) {
    float4 l = row4[j];
    if (expf(__fmul_rn(l.x, inv_temp) - m) < min_p) l.x = -INFINITY;
    if (expf(__fmul_rn(l.y, inv_temp) - m) < min_p) l.y = -INFINITY;
    if (expf(__fmul_rn(l.z, inv_temp) - m) < min_p) l.z = -INFINITY;
    if (expf(__fmul_rn(l.w, inv_temp) - m) < min_p) l.w = -INFINITY;
    row4[j] = l;
  }
  for (int i = (V4 << 2) + threadIdx.x; i < V; i += kPenThreads)
    if (expf(__fmul_rn(row[i], inv_temp) - m) < min_p) row[i] = -INFINITY;
}

}  // namespace
}  // namespace prl

using namespace prl;

extern "C" int prl_embed_rmsnorm(const int32_t* tokens, const void* embed, const void* gamma, float eps, int32_t B,
                                 int32_t H, int32_t vocab, float* h, void* x_bf16, prl_stream_t st) {
  PRL_CHECK_ARG(tokens && embed && gamma && h && x_bf16 && B >= 1 && H >= 1, "prl_embed_rmsnorm: bad argument");
  PRL_CUDA(launch_pdl(embed_rmsnorm_kernel, dim3(B), dim3(256), 0, (cudaStream_t)st, tokens, (const __nv_bfloat16*)embed,
                      (const __nv_bfloat16*)gamma, eps, (int)H, (int)vocab, h, (__nv_bfloat16*)x_bf16));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_residual_rmsnorm(const float* partials, int32_t n_split, int32_t B, int32_t H, const void* gamma,
                                    float eps, float* h, void* x_bf16, const void* l2_prefetch, size_t l2_prefetch_bytes,
                                    prl_stream_t st) {
  PRL_CHECK_ARG(partials && gamma && h && x_bf16 && B >= 1 && H >= 4 && n_split >= 0, "prl_residual_rmsnorm: bad argument");
  PRL_CHECK_ARG(H % 4 == 0, "prl_residual_rmsnorm: hidden size must be a multiple of 4 (got %d)", H);
  PRL_CHECK_ARG(H * 4 <= 96 * 1024, "prl_residual_rmsnorm: hidden size too large for the row buffer");
  static SmemAttr smem_attr = {};
  PRL_CUDA(ensure_smem(residual_rmsnorm_kernel, 96 * 1024, smem_attr));
  int threads = ((H / 4 + 31) / 32) * 32;
  if (threads > 1024) threads = 1024;
  const size_t smem = (H / 4 > threads) ? (size_t)H * 4 : 0;
  PRL_CUDA(launch_pdl(residual_rmsnorm_kernel, dim3(B), dim3(threads), smem, (cudaStream_t)st, partials, (int)n_split,
                      (int)B, (int)H, (const __nv_bfloat16*)gamma, eps, h, (__nv_bfloat16*)x_bf16, l2_prefetch,
                      l2_prefetch_bytes));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_qkv_norm_rope_cache(const float* partials, int32_t n_split, int32_t B, const void* bias,
                                       const void* q_gamma, const void* k_gamma, float eps, int32_t n_q, int32_t n_kv,
                                       int32_t head_dim, const int32_t* positions, const int32_t* block_table,
                                       int32_t max_blocks, const int32_t* row_slot, const float* inv_freq, void* q_out,
                                       void* kv_cache, int64_t n_pages, int32_t layer, int32_t page_size,
                                       const void* l2_prefetch, size_t l2_prefetch_bytes, prl_stream_t st) {
  PRL_CHECK_ARG(partials && positions && block_table && q_out && kv_cache && inv_freq, "prl_qkv_rope_cache: NULL argument");
  PRL_CHECK_ARG(head_dim == 128, "prl_qkv_rope_cache: head_dim must be 128 (got %d)", head_dim);
  PRL_CHECK_ARG(B >= 1 && n_q >= 1 && n_kv >= 1 && page_size >= 1 && max_blocks >= 1, "prl_qkv_rope_cache: bad shape");
  PRL_CHECK_ARG((q_gamma == nullptr) == (k_gamma == nullptr),
                "prl_qkv_norm_rope_cache: q_gamma and k_gamma must both be given (q/k norm) or both be NULL");
  const bool norm = q_gamma != nullptr;
  const __nv_bfloat16 *qg = (const __nv_bfloat16*)q_gamma, *kg = (const __nv_bfloat16*)k_gamma;
  if (B > 128) {  // prefill chunk: row-walking variant (same results, ~4x less time at 1024 rows)
    const unsigned blocks = (unsigned)(B < 132 * 8 ? B : 132 * 8);
    PRL_CUDA(launch_pdl(norm ? qkv_rope_cache_rows_kernel<true> : qkv_rope_cache_rows_kernel<false>, dim3(blocks),
                        dim3(256), 0, (cudaStream_t)st, partials, (int)n_split, (int)B, (const __nv_bfloat16*)bias, qg, kg,
                        eps, (int)n_q, (int)n_kv, positions, block_table, (int)max_blocks, row_slot, inv_freq,
                        (__nv_bfloat16*)q_out, (__nv_bfloat16*)kv_cache, n_pages, (int)layer, (int)page_size));
    PRL_LAUNCH_CHECK();
    return PRL_OK;
  }
  dim3 grid((unsigned)B, (unsigned)(n_q + 2 * n_kv));
  PRL_CUDA(launch_pdl(norm ? qkv_rope_cache_kernel<true> : qkv_rope_cache_kernel<false>, grid, dim3(64), 0,
                      (cudaStream_t)st, partials, (int)n_split, (int)B, (const __nv_bfloat16*)bias, qg, kg, eps, (int)n_q,
                      (int)n_kv, positions, block_table, (int)max_blocks, row_slot, inv_freq, (__nv_bfloat16*)q_out,
                      (__nv_bfloat16*)kv_cache, n_pages, (int)layer, (int)page_size, l2_prefetch, l2_prefetch_bytes));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_qkv_rope_cache(const float* partials, int32_t n_split, int32_t B, const void* bias, int32_t n_q,
                                  int32_t n_kv, int32_t head_dim, const int32_t* positions,
                                  const int32_t* block_table, int32_t max_blocks, const int32_t* row_slot,
                                  const float* inv_freq, void* q_out,
                                  void* kv_cache, int64_t n_pages, int32_t layer, int32_t page_size,
                                  const void* l2_prefetch, size_t l2_prefetch_bytes, prl_stream_t st) {
  return prl_qkv_norm_rope_cache(partials, n_split, B, bias, nullptr, nullptr, 0.f, n_q, n_kv, head_dim, positions,
                                 block_table, max_blocks, row_slot, inv_freq, q_out, kv_cache, n_pages, layer, page_size,
                                 l2_prefetch, l2_prefetch_bytes, st);
}

extern "C" int prl_silu_mul(const float* partials, int32_t n_split, int32_t B, int32_t I, void* act_bf16,
                            const void* l2_prefetch, size_t l2_prefetch_bytes, prl_stream_t st) {
  PRL_CHECK_ARG(partials && act_bf16 && B >= 1 && I >= 4 && n_split >= 1, "prl_silu_mul: bad argument");
  PRL_CHECK_ARG(I % 4 == 0, "prl_silu_mul: intermediate size must be a multiple of 4 (got %d)", I);
  dim3 grid((unsigned)((I / 4 + 255) / 256), (unsigned)B);
  PRL_CUDA(launch_pdl(silu_mul_kernel, grid, dim3(256), 0, (cudaStream_t)st, partials, (int)n_split, (int)B, (int)I,
                      (__nv_bfloat16*)act_bf16, l2_prefetch, l2_prefetch_bytes));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" size_t prl_sample_workspace_bytes(int32_t B) {
  return (size_t)(B < 1 ? 1 : B) * kSampleParts * sizeof(SamplePartial);
}

// phase 1 only: per-row partials of logits[:, vocab slice] into `partials` ([B][16]); ids are global (offset added)
extern "C" int prl_sample_partials(const float* logits, int32_t B, int32_t V, float temperature, int32_t greedy,
                                   uint64_t seed, uint32_t step, int32_t vocab_offset, void* partials,
                                   prl_stream_t st) {
  PRL_CHECK_ARG(logits && partials && B >= 1 && V >= 1, "prl_sample_partials: bad argument");
  PRL_CHECK_ARG(temperature > 0.f, "prl_sample_partials: temperature must be > 0 (use greedy=1 for argmax)");
  dim3 grid((unsigned)B, kSampleParts);
  PRL_CUDA(launch_pdl(sample_partial_kernel, grid, dim3(kSampleThreads), 0, (cudaStream_t)st, logits, (int)V,
                      1.f / temperature, (int)greedy, seed, step, (int)vocab_offset, (SamplePartial*)partials,
                      (const float*)nullptr, (const uint8_t*)nullptr));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_sample_logprob_rows(const float* logits, int32_t B, int32_t V, const float* inv_temperature_rows,
                                       const uint8_t* greedy_rows, uint64_t seed, uint32_t step, int32_t* out_ids,
                                       float* out_logprobs, void* workspace, size_t workspace_bytes, prl_stream_t st) {
  PRL_CHECK_ARG(logits && inv_temperature_rows && greedy_rows && out_ids && out_logprobs && B >= 1 && V >= 1,
                "prl_sample_logprob_rows: bad argument");
  PRL_CHECK_ARG(workspace && workspace_bytes >= prl_sample_workspace_bytes(B), "prl_sample_logprob_rows: workspace too small");
  dim3 grid((unsigned)B, kSampleParts);
  PRL_CUDA(launch_pdl(sample_partial_kernel, grid, dim3(kSampleThreads), 0, (cudaStream_t)st, logits, (int)V, 1.f, 0, seed,
                      step, 0, (SamplePartial*)workspace, inv_temperature_rows, greedy_rows));
  PRL_LAUNCH_CHECK();
  return prl_sample_finalize(workspace, B, 1, out_ids, out_logprobs, st);
}

// phase 2 only: merge n_groups x 16 partials per row ([group][B][16]) -> ids, logprobs
extern "C" int prl_sample_finalize(const void* partials, int32_t B, int32_t n_groups, int32_t* out_ids,
                                   float* out_logprobs, prl_stream_t st) {
  PRL_CHECK_ARG(partials && out_ids && out_logprobs && B >= 1 && n_groups >= 1, "prl_sample_finalize: bad argument");
  PRL_CUDA(launch_pdl(sample_finalize_kernel, dim3((B + 63) / 64), dim3(64), 0, (cudaStream_t)st, (int)B, (int)n_groups,
                      (const SamplePartial*)partials, out_ids, out_logprobs));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_sample_logprob(const float* logits, int32_t B, int32_t V, float temperature, int32_t greedy,
                                  uint64_t seed, uint32_t step, int32_t* out_ids, float* out_logprobs,
                                  void* workspace, size_t workspace_bytes, prl_stream_t st) {
  PRL_CHECK_ARG(workspace && workspace_bytes >= prl_sample_workspace_bytes(B), "prl_sample_logprob: workspace too small");
  int rc = prl_sample_partials(logits, B, V, temperature, greedy, seed, step, 0, workspace, st);
  if (rc) return rc;
  return prl_sample_finalize(workspace, B, 1, out_ids, out_logprobs, st);
}

extern "C" int prl_tp_signal(void* peer_flag, prl_stream_t st) {
  PRL_CHECK_ARG(peer_flag, "prl_tp_signal: NULL flag");
  PRL_CUDA(launch_pdl(tp_signal_kernel, dim3(1), dim3(32), 0, (cudaStream_t)st, (unsigned long long*)peer_flag));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}
extern "C" int prl_tp_wait(const void* flag, const void* epoch, int32_t signals_per_step, int32_t k, prl_stream_t st) {
  PRL_CHECK_ARG(flag && epoch && signals_per_step >= 1 && k >= 1 && k <= signals_per_step, "prl_tp_wait: bad argument");
  PRL_CUDA(launch_pdl(tp_wait_kernel, dim3(1), dim3(32), 0, (cudaStream_t)st, (const unsigned long long*)flag,
                      (const unsigned long long*)epoch, (int)signals_per_step, (int)k));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}
extern "C" int prl_tp_epoch(void* epoch, prl_stream_t st) {
  PRL_CHECK_ARG(epoch, "prl_tp_epoch: NULL counter");
  PRL_CUDA(launch_pdl(tp_epoch_kernel, dim3(1), dim3(32), 0, (cudaStream_t)st, (unsigned long long*)epoch));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_advance_state_strings(const prl_engine_state* state, const prl_stop_strings* strings,
                                         prl_stream_t st) {
  PRL_CHECK_ARG(state && state->B >= 1, "prl_advance_state: bad argument");
  PRL_CHECK_ARG(state->sampled && state->sampled_logprobs && state->tokens && state->positions && state->seq_lens &&
                    state->active && state->prompt_buf && state->prompt_len && state->out_ids &&
                    state->out_logprobs && state->gen_count && state->max_new && state->finished,
                "prl_advance_state: NULL field");
  PRL_CHECK_ARG(state->stop_ids == nullptr || (state->n_stop && state->stop_stride >= 1),
                "prl_advance_state: stop_ids needs n_stop and stop_stride >= 1");
  prl_stop_strings ss = {};
  if (strings != nullptr) ss = *strings;
  PRL_CHECK_ARG(ss.tok_bytes == nullptr ||
                    (ss.tok_offsets && ss.tok_special && ss.vocab >= 1 && ss.stop_str && ss.stop_str_fail &&
                     ss.stop_str_len && ss.n_stop_str && ss.stop_str_flags && ss.stop_str_state &&
                     ss.max_stop_str >= 1 && ss.stop_str_stride >= 1 && ss.stop_str_stride <= 32767),
                "prl_advance_state_strings: tok_bytes needs the token table, every stop-string field, max_stop_str >= 1 "
                "and 1 <= stop_str_stride <= 32767");
  PRL_CUDA(launch_pdl(advance_kernel, dim3((state->B + 127) / 128), dim3(128), 0, (cudaStream_t)st, *state, ss));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_advance_state(const prl_engine_state* state, prl_stream_t st) {
  return prl_advance_state_strings(state, nullptr, st);
}

extern "C" int prl_ban_min_tokens(float* logits, int32_t B, int32_t V, const int32_t* gen_count,
                                  const int32_t* min_tokens, const int32_t* ban_ids, int32_t ban_stride,
                                  const int32_t* n_ban, prl_stream_t st) {
  PRL_CHECK_ARG(logits && gen_count && min_tokens && ban_ids && n_ban, "prl_ban_min_tokens: NULL argument");
  PRL_CHECK_ARG(B >= 1 && V >= 1 && ban_stride >= 1, "prl_ban_min_tokens: bad shape (B=%d, V=%d, ban_stride=%d)", B, V,
                ban_stride);
  PRL_CUDA(launch_pdl(ban_min_tokens_kernel, dim3((B + 3) / 4), dim3(128), 0, (cudaStream_t)st, logits, (int)B, (int)V,
                      gen_count, min_tokens, ban_ids, (int)ban_stride, n_ban));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_apply_penalties(const prl_penalties* p, prl_stream_t st) {
  PRL_CHECK_ARG(p != nullptr, "prl_apply_penalties: NULL argument");
  PRL_CHECK_ARG(p->B >= 1 && p->V >= 1 && p->prompt_stride >= 1 && p->out_stride >= 1,
                "prl_apply_penalties: bad shape (B=%d, V=%d, prompt_stride=%d, out_stride=%d)", p->B, p->V,
                p->prompt_stride, p->out_stride);
  PRL_CHECK_ARG(p->logits && p->presence && p->frequency && p->repetition && p->min_p && p->inv_temp && p->greedy &&
                    p->prompt_buf && p->prompt_len && p->out_ids && p->gen_count && p->counts && p->prompt_mask &&
                    p->seen,
                "prl_apply_penalties: NULL field");
  PRL_CUDA(launch_pdl(penalties_kernel, dim3(p->B), dim3(kPenThreads), 0, (cudaStream_t)st, *p));
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}
