// Row-wise kernels of the learner body (hot path 2): everything between the GEMMs of the Qwen2 forward / backward
// that the reference runs as HF eager modules under autograd (pipelinerl/finetune/rl/__init__.py:190-207 reached
// through transformers' Qwen2RMSNorm / apply_rotary_pos_emb / Qwen2MLP; backward finetune_loop.py:716-725).
// All of them are HBM-bound: one pass over the activations, bf16 in / bf16 out, fp32 arithmetic, 16-byte accesses.
// Reductions over the token dimension (RMSNorm gain, qkv bias) are two-stage with a FIXED order: per-block partial
// rows in a workspace, then one pass that adds them into the fp32 gradient arena -> bitwise reproducible.
#include "prl_common.cuh"

namespace prl {
namespace {

constexpr int kRowThreads = 256;
constexpr int kMaxVec = 4;          // 8-element vectors per thread -> rows of up to 8192 elements
constexpr int kPartialBlocks = 528; // 4 per SM: grid of the persistent row kernels = rows of the partial workspace

struct Vec8 { float v[8]; };

__device__ __forceinline__ Vec8 load8(const __nv_bfloat16* p) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
  Vec8 r;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 f = __bfloat1622float2(h[e]);
    r.v[2 * e] = f.x;
    r.v[2 * e + 1] = f.y;
  }
  return r;
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const Vec8& r) {
  uint4 u;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int e = 0; e < 4; ++e) h[e] = __floats2bfloat162_rn(r.v[2 * e], r.v[2 * e + 1]);
  *reinterpret_cast<uint4*>(p) = u;
}

__device__ __forceinline__ float block_sum(float v, float* s_red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();  // s_red may still be read from the previous call
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < kRowThreads / 32; ++w) t += s_red[w];
  return t;
}

// y = bf16(x * rstd) * gamma  (the rounding order of HF's Qwen2RMSNorm); rstd kept for the backward
template <int kVec>
__global__ void __launch_bounds__(kRowThreads) rmsnorm_fwd_kernel(const __nv_bfloat16* __restrict__ x,
                                                                  const __nv_bfloat16* __restrict__ gamma, int64_t T,
                                                                  int H, float eps, __nv_bfloat16* __restrict__ y,
                                                                  float* __restrict__ rstd) {
  __shared__ float s_red[kRowThreads / 32];
  const int nvec = H >> 3;
  for (int64_t row = blockIdx.x; row < T; row += gridDim.x) {
    Vec8 xv[kVec];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      const int v = threadIdx.x + i * kRowThreads;
      if (v < nvec) {
        xv[i] = load8(x + row * H + v * 8);
#pragma unroll
        for (int e = 0; e < 8; ++e) ss += xv[i].v[e] * xv[i].v[e];
      }
    }
    const float r = rsqrtf(block_sum(ss, s_red) / (float)H + eps);
    if (threadIdx.x == 0) rstd[row] = r;
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      const int v = threadIdx.x + i * kRowThreads;
      if (v < nvec) {
        const Vec8 g = load8(gamma + v * 8);
        Vec8 o;
#pragma unroll
        for (int e = 0; e < 8; ++e) o.v[e] = __bfloat162float(__float2bfloat16(xv[i].v[e] * r)) * g.v[e];
        store8(y + row * H + v * 8, o);
      }
    }
  }
}

// dx = dres + rstd * (dy*gamma - xhat * mean(dy*gamma*xhat));  partial[block][c] = sum over this block's rows of dy*xhat
template <int kVec>
__global__ void __launch_bounds__(kRowThreads, kVec <= 2 ? 3 : 1) rmsnorm_bwd_kernel(const __nv_bfloat16* __restrict__ x,
                                                                  const __nv_bfloat16* __restrict__ gamma,
                                                                  const float* __restrict__ rstd,
                                                                  const __nv_bfloat16* __restrict__ dy,
                                                                  const __nv_bfloat16* __restrict__ dres, int64_t T, int H,
                                                                  __nv_bfloat16* __restrict__ dx,
                                                                  float* __restrict__ partial) {
  __shared__ float s_red[kRowThreads / 32];
  const int nvec = H >> 3;
  Vec8 gv[kVec], acc[kVec];
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int v = threadIdx.x + i * kRowThreads;
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[i].v[e] = 0.f;
    if (v < nvec) gv[i] = load8(gamma + v * 8);
  }
  for (int64_t row = blockIdx.x; row < T; row += gridDim.x) {
    const float r = rstd[row];
    Vec8 xh[kVec], dxh[kVec];
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      const int v = threadIdx.x + i * kRowThreads;
      if (v < nvec) {
        xh[i] = load8(x + row * H + v * 8);
        const Vec8 d = load8(dy + row * H + v * 8);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          xh[i].v[e] *= r;
          acc[i].v[e] += d.v[e] * xh[i].v[e];
          dxh[i].v[e] = d.v[e] * gv[i].v[e];
          dot += dxh[i].v[e] * xh[i].v[e];
        }
      }
    }
    const float m = block_sum(dot, s_red) / (float)H;
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      const int v = threadIdx.x + i * kRowThreads;
      if (v < nvec) {
        Vec8 o;
#pragma unroll
        for (int e = 0; e < 8; ++e) o.v[e] = r * (dxh[i].v[e] - xh[i].v[e] * m);
        if (dres) {
          const Vec8 dr = load8(dres + row * H + v * 8);
#pragma unroll
          for (int e = 0; e < 8; ++e) o.v[e] += dr.v[e];
        }
        store8(dx + row * H + v * 8, o);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int v = threadIdx.x + i * kRowThreads;
    if (v < nvec) {
      float* pp = partial + (int64_t)blockIdx.x * H + v * 8;
      *reinterpret_cast<float4*>(pp) = make_float4(acc[i].v[0], acc[i].v[1], acc[i].v[2], acc[i].v[3]);
      *reinterpret_cast<float4*>(pp + 4) = make_float4(acc[i].v[4], acc[i].v[5], acc[i].v[6], acc[i].v[7]);
    }
  }
}

template <int kVec>
__global__ void __launch_bounds__(kRowThreads) colsum_kernel(const __nv_bfloat16* __restrict__ x, int64_t ld, int64_t T,
                                                             int Cc, float* __restrict__ partial) {
  const int nvec = Cc >> 3;
  Vec8 acc[kVec];
#pragma unroll
  for (int i = 0; i < kVec; ++i)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[i].v[e] = 0.f;
  for (int64_t row = blockIdx.x; row < T; row += gridDim.x) {
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      const int v = threadIdx.x + i * kRowThreads;
      if (v < nvec) {
        const Vec8 d = load8(x + row * ld + v * 8);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[i].v[e] += d.v[e];
      }
    }
  }
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int v = threadIdx.x + i * kRowThreads;
    if (v < nvec) {
      float* pp = partial + (int64_t)blockIdx.x * Cc + v * 8;
      *reinterpret_cast<float4*>(pp) = make_float4(acc[i].v[0], acc[i].v[1], acc[i].v[2], acc[i].v[3]);
      *reinterpret_cast<float4*>(pp + 4) = make_float4(acc[i].v[4], acc[i].v[5], acc[i].v[6], acc[i].v[7]);
    }
  }
}

// out[c] += sum_b partial[b][c], b ascending
__global__ void __launch_bounds__(256) partial_reduce_kernel(const float* __restrict__ partial, int n_blocks, int Cc,
                                                             float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= Cc) return;
  float s = 0.f;
  for (int b = 0; b < n_blocks; ++b) s += partial[(int64_t)b * Cc + c];
  out[c] += s;
}

// in-place rotation of the first n_heads heads of each row: (x1, x2) -> (x1 cos - s x2 sin, x2 cos + s x1 sin)
__global__ void rope_kernel(__nv_bfloat16* __restrict__ x, int64_t ld, int64_t T, int n_heads, int head_dim,
                            const int32_t* __restrict__ pos, const float* __restrict__ inv_freq, float sign) {
  extern __shared__ float s_cs[];  // [half] cos, [half] sin
  const int half = head_dim >> 1;
  const int per_head = half >> 3;  // threads per head (8 pairs each)
  for (int64_t row = blockIdx.x; row < T; row += gridDim.x) {
    __syncthreads();
    for (int i = threadIdx.x; i < half; i += blockDim.x) {
      float sn, cs;
      sincosf((float)pos[row] * inv_freq[i], &sn, &cs);
      s_cs[i] = cs;
      s_cs[half + i] = sn * sign;
    }
    __syncthreads();
    for (int w = threadIdx.x; w < n_heads * per_head; w += blockDim.x) {
      const int head = w / per_head, i0 = (w % per_head) * 8;
      __nv_bfloat16* p = x + row * ld + (int64_t)head * head_dim + i0;
      const Vec8 a = load8(p), b = load8(p + half);
      Vec8 oa, ob;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float cs = s_cs[i0 + e], sn = s_cs[half + i0 + e];
        oa.v[e] = a.v[e] * cs - b.v[e] * sn;
        ob.v[e] = b.v[e] * cs + a.v[e] * sn;
      }
      store8(p, oa);
      store8(p + half, ob);
    }
  }
}

// ---- Qwen3: per-head RMSNorm of q and k, then RoPE (forward), and the backward of the pair ---------------------------
// qkv [T, ld] bf16 in place; heads [0, n_q) are q, [n_q, n_q + n_kv) are k (v heads are not touched).  One block per
// row (grid-stride), one warp per head: lane l owns the rotation pairs (2l, 2l + 64) and (2l + 1, 2l + 65).  Per head,
// in fp32: y = x * rstd * gamma with rstd = rsqrt(mean(x^2) + eps), then the rotation, rounded to bf16 once.
constexpr int kQkThreads = 256;

__device__ __forceinline__ void load_pair4(const __nv_bfloat16* p, int lane, float (&v)[4]) {
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p + 2 * lane));
  const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p + 64 + 2 * lane));
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}
__device__ __forceinline__ void store_pair4(__nv_bfloat16* p, int lane, const float (&v)[4]) {
  *reinterpret_cast<__nv_bfloat162*>(p + 2 * lane) = __floats2bfloat162_rn(v[0], v[1]);
  *reinterpret_cast<__nv_bfloat162*>(p + 64 + 2 * lane) = __floats2bfloat162_rn(v[2], v[3]);
}

// x_pre [T, (n_q + n_kv) * 128] (nullable): the pre-norm q | k columns, kept for the backward; rstd [T, n_q + n_kv]
__global__ void __launch_bounds__(kQkThreads) qk_norm_rope_fwd_kernel(__nv_bfloat16* __restrict__ x, int64_t ld,
                                                                      int64_t T, int n_q, int n_kv,
                                                                      const __nv_bfloat16* __restrict__ q_gamma,
                                                                      const __nv_bfloat16* __restrict__ k_gamma, float eps,
                                                                      const int32_t* __restrict__ pos,
                                                                      const float* __restrict__ inv_freq,
                                                                      __nv_bfloat16* __restrict__ x_pre,
                                                                      float* __restrict__ rstd) {
  __shared__ float s_cs[64], s_sn[64];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  const int nh = n_q + n_kv;
  float gq[4], gk[4];
  load_pair4(q_gamma, lane, gq);
  load_pair4(k_gamma, lane, gk);
  for (int64_t row = blockIdx.x; row < T; row += gridDim.x) {
    __syncthreads();
    if (threadIdx.x < 64) {
      float sn, cs;
      sincosf((float)pos[row] * inv_freq[threadIdx.x], &sn, &cs);
      s_cs[threadIdx.x] = cs;
      s_sn[threadIdx.x] = sn;
    }
    __syncthreads();
    const float c0 = s_cs[2 * lane], c1 = s_cs[2 * lane + 1], s0 = s_sn[2 * lane], s1 = s_sn[2 * lane + 1];
    for (int head = warp; head < nh; head += n_warps) {
      __nv_bfloat16* p = x + row * ld + (int64_t)head * 128;
      float v[4];
      load_pair4(p, lane, v);
      if (x_pre) {
        __nv_bfloat16* q = x_pre + (row * nh + head) * 128;
        *reinterpret_cast<__nv_bfloat162*>(q + 2 * lane) = *reinterpret_cast<const __nv_bfloat162*>(p + 2 * lane);
        *reinterpret_cast<__nv_bfloat162*>(q + 64 + 2 * lane) = *reinterpret_cast<const __nv_bfloat162*>(p + 64 + 2 * lane);
      }
      const float ss = warp_sum(v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3]);
      const float r = rsqrtf(ss * (1.f / 128.f) + eps);
      if (rstd && lane == 0) rstd[row * nh + head] = r;
      const bool is_q = head < n_q;
      float y[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) y[e] = v[e] * r * (is_q ? gq[e] : gk[e]);
      float o[4];
      o[0] = y[0] * c0 - y[2] * s0;
      o[2] = y[2] * c0 + y[0] * s0;
      o[1] = y[1] * c1 - y[3] * s1;
      o[3] = y[3] * c1 + y[1] * s1;
      store_pair4(p, lane, o);
    }
  }
}

// dx (the gradient of the roped q | k columns of dqkv, in place) -> inverse rotation -> RMSNorm backward:
//   dx = rstd * (g * dy - xhat * mean(xhat * g * dy)),  dgamma += sum over rows and heads of dy * xhat (q and k apart)
// partial[block][256] = this block's gain sums (q: [0, 128), k: [128, 256)), summed over its warps in a fixed order.
__global__ void __launch_bounds__(kQkThreads) qk_norm_rope_bwd_kernel(__nv_bfloat16* __restrict__ dx, int64_t ld,
                                                                      int64_t T, int n_q, int n_kv,
                                                                      const __nv_bfloat16* __restrict__ q_gamma,
                                                                      const __nv_bfloat16* __restrict__ k_gamma,
                                                                      const int32_t* __restrict__ pos,
                                                                      const float* __restrict__ inv_freq,
                                                                      const __nv_bfloat16* __restrict__ x_pre,
                                                                      const float* __restrict__ rstd,
                                                                      float* __restrict__ partial) {
  __shared__ float s_cs[64], s_sn[64];
  __shared__ float s_acc[kQkThreads / 32][256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  const int nh = n_q + n_kv;
  float gq[4], gk[4], aq[4] = {0.f, 0.f, 0.f, 0.f}, ak[4] = {0.f, 0.f, 0.f, 0.f};
  load_pair4(q_gamma, lane, gq);
  load_pair4(k_gamma, lane, gk);
  for (int64_t row = blockIdx.x; row < T; row += gridDim.x) {
    __syncthreads();
    if (threadIdx.x < 64) {
      float sn, cs;
      sincosf((float)pos[row] * inv_freq[threadIdx.x], &sn, &cs);
      s_cs[threadIdx.x] = cs;
      s_sn[threadIdx.x] = sn;
    }
    __syncthreads();
    const float c0 = s_cs[2 * lane], c1 = s_cs[2 * lane + 1], s0 = s_sn[2 * lane], s1 = s_sn[2 * lane + 1];
    for (int head = warp; head < nh; head += n_warps) {
      __nv_bfloat16* p = dx + row * ld + (int64_t)head * 128;
      float d[4], xv[4];
      load_pair4(p, lane, d);
      load_pair4(x_pre + (row * nh + head) * 128, lane, xv);
      float dy[4];  // the transpose of the rotation
      dy[0] = d[0] * c0 + d[2] * s0;
      dy[2] = d[2] * c0 - d[0] * s0;
      dy[1] = d[1] * c1 + d[3] * s1;
      dy[3] = d[3] * c1 - d[1] * s1;
      const float r = rstd[row * nh + head];
      const bool is_q = head < n_q;
      float xh[4], gd[4], dot = 0.f;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        xh[e] = xv[e] * r;
        gd[e] = (is_q ? gq[e] : gk[e]) * dy[e];
        dot += xh[e] * gd[e];
      }
      const float m = warp_sum(dot) * (1.f / 128.f);
      float o[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) o[e] = r * (gd[e] - xh[e] * m);
      store_pair4(p, lane, o);
      if (is_q) {
#pragma unroll
        for (int e = 0; e < 4; ++e) aq[e] += dy[e] * xh[e];
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) ak[e] += dy[e] * xh[e];
      }
    }
  }
  const int idx[4] = {2 * lane, 2 * lane + 1, 64 + 2 * lane, 65 + 2 * lane};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    s_acc[warp][idx[e]] = aq[e];
    s_acc[warp][128 + idx[e]] = ak[e];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 256; c += blockDim.x) {
    float t = 0.f;
    for (int w = 0; w < n_warps; ++w) t += s_acc[w][c];
    partial[(int64_t)blockIdx.x * 256 + c] = t;
  }
}

// dq_gamma[c] += sum_b partial[b][c], dk_gamma[c] += sum_b partial[b][128 + c], b ascending
__global__ void __launch_bounds__(256) qk_gain_reduce_kernel(const float* __restrict__ partial, int n_blocks,
                                                             float* __restrict__ dq_gamma, float* __restrict__ dk_gamma) {
  const int c = threadIdx.x;
  float s = 0.f;
  for (int b = 0; b < n_blocks; ++b) s += partial[(int64_t)b * 256 + c];
  if (c < 128) dq_gamma[c] += s; else dk_gamma[c - 128] += s;
}

__global__ void __launch_bounds__(256) silu_mul_fwd_kernel(const __nv_bfloat16* __restrict__ gu, int64_t T, int I,
                                                           __nv_bfloat16* __restrict__ act) {
  const int64_t nvec = T * (I >> 3);
  const int per_row = I >> 3;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = v / per_row;
    const int c = (int)(v % per_row) * 8;
    const Vec8 g = load8(gu + row * 2 * I + c), u = load8(gu + row * 2 * I + I + c);
    Vec8 o;
#pragma unroll
    for (int e = 0; e < 8; ++e) o.v[e] = g.v[e] / (1.f + __expf(-g.v[e])) * u.v[e];
    store8(act + row * I + c, o);
  }
}

__global__ void __launch_bounds__(256) silu_mul_bwd_kernel(const __nv_bfloat16* __restrict__ gu,
                                                           const __nv_bfloat16* __restrict__ dact, int64_t T, int I,
                                                           __nv_bfloat16* __restrict__ dgu) {
  const int64_t nvec = T * (I >> 3);
  const int per_row = I >> 3;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = v / per_row;
    const int c = (int)(v % per_row) * 8;
    const Vec8 g = load8(gu + row * 2 * I + c), u = load8(gu + row * 2 * I + I + c), d = load8(dact + row * I + c);
    Vec8 dg, du;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float s = 1.f / (1.f + __expf(-g.v[e]));
      const float silu = g.v[e] * s;
      du.v[e] = d.v[e] * silu;
      dg.v[e] = d.v[e] * u.v[e] * (s + silu * (1.f - s));
    }
    store8(dgu + row * 2 * I + c, dg);
    store8(dgu + row * 2 * I + I + c, du);
  }
}

__global__ void __launch_bounds__(256) embed_gather_kernel(const __nv_bfloat16* __restrict__ table,
                                                           const int64_t* __restrict__ ids, int64_t T, int H,
                                                           __nv_bfloat16* __restrict__ out) {
  const int nvec = H >> 3;
  for (int64_t row = blockIdx.x; row < T; row += gridDim.x) {
    const int64_t id = ids[row];
    for (int v = threadIdx.x; v < nvec; v += blockDim.x)
      *reinterpret_cast<uint4*>(out + row * H + v * 8) = *reinterpret_cast<const uint4*>(table + id * H + v * 8);
  }
}

__global__ void __launch_bounds__(256) embed_scatter_kernel(float* __restrict__ dtable, const int64_t* __restrict__ ids,
                                                            const __nv_bfloat16* __restrict__ dh, int64_t T, int H) {
  const int nvec = H >> 3;
  for (int64_t row = blockIdx.x; row < T; row += gridDim.x) {
    const int64_t id = ids[row];
    for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
      const Vec8 d = load8(dh + row * H + v * 8);
#pragma unroll
      for (int e = 0; e < 8; ++e) atomicAdd(dtable + id * H + v * 8 + e, d.v[e]);
    }
  }
}

int row_grid(int64_t T) { return (int)(T < kPartialBlocks ? T : kPartialBlocks); }

}  // namespace
}  // namespace prl

using namespace prl;

extern "C" size_t prl_rowops_workspace_bytes(int64_t cols) { return (size_t)kPartialBlocks * (size_t)cols * sizeof(float); }

#define PRL_ROW_ARGS(name, H)                                                                                       \
  PRL_CHECK_ARG((H) >= 8 && (H) % 8 == 0 && (H) <= kRowThreads * kMaxVec * 8, name ": row length must be a multiple " \
                "of 8 in [8, 8192] (got %lld)", (long long)(H))

extern "C" int prl_rmsnorm_fwd(const void* x, const void* gamma, int64_t T, int64_t H, float eps, void* y, float* rstd,
                               prl_stream_t stream) {
  PRL_CHECK_ARG(x && gamma && y && rstd && T >= 1, "prl_rmsnorm_fwd: bad argument");
  PRL_ROW_ARGS("prl_rmsnorm_fwd", H);
  const unsigned grid = (unsigned)(T < 4 * kPartialBlocks ? T : 4 * kPartialBlocks);
#define PRL_FWD(V) rmsnorm_fwd_kernel<V><<<grid, kRowThreads, 0, (cudaStream_t)stream>>>( \
      (const __nv_bfloat16*)x, (const __nv_bfloat16*)gamma, T, (int)H, eps, (__nv_bfloat16*)y, rstd)
  if (H <= 2048) PRL_FWD(1); else if (H <= 4096) PRL_FWD(2); else PRL_FWD(4);
#undef PRL_FWD
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_rmsnorm_bwd(const void* x, const void* gamma, const float* rstd, const void* dy, const void* dres,
                               int64_t T, int64_t H, void* dx, float* dgamma, void* workspace, size_t workspace_bytes,
                               prl_stream_t stream) {
  PRL_CHECK_ARG(x && gamma && rstd && dy && dx && dgamma && workspace && T >= 1, "prl_rmsnorm_bwd: bad argument");
  PRL_ROW_ARGS("prl_rmsnorm_bwd", H);
  PRL_CHECK_ARG(workspace_bytes >= prl_rowops_workspace_bytes(H), "prl_rmsnorm_bwd: workspace too small");
  const int g = row_grid(T);
#define PRL_BWD(V) rmsnorm_bwd_kernel<V><<<g, kRowThreads, 0, (cudaStream_t)stream>>>( \
      (const __nv_bfloat16*)x, (const __nv_bfloat16*)gamma, rstd, (const __nv_bfloat16*)dy, (const __nv_bfloat16*)dres, T, \
      (int)H, (__nv_bfloat16*)dx, (float*)workspace)
  if (H <= 2048) PRL_BWD(1); else if (H <= 4096) PRL_BWD(2); else PRL_BWD(4);
#undef PRL_BWD
  PRL_LAUNCH_CHECK();
  partial_reduce_kernel<<<(unsigned)((H + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const float*)workspace, g, (int)H,
                                                                                       dgamma);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_colsum_bf16(const void* x, int64_t ld, int64_t T, int64_t cols, float* out, void* workspace,
                               size_t workspace_bytes, prl_stream_t stream) {
  PRL_CHECK_ARG(x && out && workspace && T >= 1 && ld >= cols && ld % 8 == 0, "prl_colsum_bf16: bad argument");
  PRL_ROW_ARGS("prl_colsum_bf16", cols);
  PRL_CHECK_ARG(workspace_bytes >= prl_rowops_workspace_bytes(cols), "prl_colsum_bf16: workspace too small");
  const int g = row_grid(T);
#define PRL_CS(V) colsum_kernel<V><<<g, kRowThreads, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, ld, T, (int)cols, \
                                                                            (float*)workspace)
  if (cols <= 2048) PRL_CS(1); else if (cols <= 4096) PRL_CS(2); else PRL_CS(4);
#undef PRL_CS
  PRL_LAUNCH_CHECK();
  partial_reduce_kernel<<<(unsigned)((cols + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const float*)workspace, g,
                                                                                          (int)cols, out);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_rope_inplace(void* x, int64_t ld, int64_t T, int32_t n_heads, int32_t head_dim, const int32_t* pos,
                                const float* inv_freq, float sign, prl_stream_t stream) {
  PRL_CHECK_ARG(x && pos && inv_freq && T >= 1 && n_heads >= 1, "prl_rope_inplace: bad argument");
  PRL_CHECK_ARG(head_dim >= 16 && head_dim % 16 == 0 && head_dim <= 512 && ld % 8 == 0 && ld >= (int64_t)n_heads * head_dim,
                "prl_rope_inplace: head_dim must be a multiple of 16 and ld a multiple of 8 covering the rotated heads");
  int threads = n_heads * (head_dim / 16);
  threads = threads > 256 ? 256 : ((threads + 31) / 32 * 32);
  rope_kernel<<<(unsigned)(T < 8 * kPartialBlocks ? T : 8 * kPartialBlocks), threads, (size_t)head_dim * sizeof(float),
                (cudaStream_t)stream>>>((__nv_bfloat16*)x, ld, T, n_heads, head_dim, pos, inv_freq, sign);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_qk_norm_rope_fwd(void* qkv, int64_t ld, int64_t T, int32_t n_q, int32_t n_kv, int32_t head_dim,
                                    const void* q_gamma, const void* k_gamma, float eps, const int32_t* pos,
                                    const float* inv_freq, void* qk_pre, float* rstd, prl_stream_t stream) {
  PRL_CHECK_ARG(qkv && q_gamma && k_gamma && pos && inv_freq && T >= 1 && n_q >= 1 && n_kv >= 1,
                "prl_qk_norm_rope_fwd: bad argument");
  PRL_CHECK_ARG(head_dim == 128, "prl_qk_norm_rope_fwd: head_dim must be 128 (got %d)", head_dim);
  PRL_CHECK_ARG(ld % 8 == 0 && ld >= (int64_t)(n_q + n_kv) * 128, "prl_qk_norm_rope_fwd: ld must be a multiple of 8 "
                "covering the q | k heads");
  PRL_CHECK_ARG((qk_pre == nullptr) == (rstd == nullptr), "prl_qk_norm_rope_fwd: qk_pre and rstd go together");
  qk_norm_rope_fwd_kernel<<<(unsigned)(T < 4 * kPartialBlocks ? T : 4 * kPartialBlocks), kQkThreads, 0,
                            (cudaStream_t)stream>>>((__nv_bfloat16*)qkv, ld, T, (int)n_q, (int)n_kv,
                                                    (const __nv_bfloat16*)q_gamma, (const __nv_bfloat16*)k_gamma, eps, pos,
                                                    inv_freq, (__nv_bfloat16*)qk_pre, rstd);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_qk_norm_rope_bwd(void* dqkv, int64_t ld, int64_t T, int32_t n_q, int32_t n_kv, int32_t head_dim,
                                    const void* q_gamma, const void* k_gamma, const int32_t* pos, const float* inv_freq,
                                    const void* qk_pre, const float* rstd, float* dq_gamma, float* dk_gamma,
                                    void* workspace, size_t workspace_bytes, prl_stream_t stream) {
  PRL_CHECK_ARG(dqkv && q_gamma && k_gamma && pos && inv_freq && qk_pre && rstd && dq_gamma && dk_gamma && workspace &&
                    T >= 1 && n_q >= 1 && n_kv >= 1,
                "prl_qk_norm_rope_bwd: bad argument");
  PRL_CHECK_ARG(head_dim == 128, "prl_qk_norm_rope_bwd: head_dim must be 128 (got %d)", head_dim);
  PRL_CHECK_ARG(ld % 8 == 0 && ld >= (int64_t)(n_q + n_kv) * 128, "prl_qk_norm_rope_bwd: ld must be a multiple of 8 "
                "covering the q | k heads");
  PRL_CHECK_ARG(workspace_bytes >= prl_rowops_workspace_bytes(256), "prl_qk_norm_rope_bwd: workspace too small");
  const int g = row_grid(T);
  qk_norm_rope_bwd_kernel<<<g, kQkThreads, 0, (cudaStream_t)stream>>>(
      (__nv_bfloat16*)dqkv, ld, T, (int)n_q, (int)n_kv, (const __nv_bfloat16*)q_gamma, (const __nv_bfloat16*)k_gamma, pos,
      inv_freq, (const __nv_bfloat16*)qk_pre, rstd, (float*)workspace);
  PRL_LAUNCH_CHECK();
  qk_gain_reduce_kernel<<<1, 256, 0, (cudaStream_t)stream>>>((const float*)workspace, g, dq_gamma, dk_gamma);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_silu_mul_fwd(const void* gate_up, int64_t T, int64_t I, void* act, prl_stream_t stream) {
  PRL_CHECK_ARG(gate_up && act && T >= 1 && I >= 8 && I % 8 == 0, "prl_silu_mul_fwd: bad argument (I %% 8 == 0)");
  const int64_t blocks = (T * (I / 8) + 255) / 256;
  silu_mul_fwd_kernel<<<(unsigned)(blocks < 132 * 16 ? blocks : 132 * 16), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)gate_up, T, (int)I, (__nv_bfloat16*)act);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_silu_mul_bwd(const void* gate_up, const void* dact, int64_t T, int64_t I, void* dgate_up,
                                prl_stream_t stream) {
  PRL_CHECK_ARG(gate_up && dact && dgate_up && T >= 1 && I >= 8 && I % 8 == 0, "prl_silu_mul_bwd: bad argument");
  const int64_t blocks = (T * (I / 8) + 255) / 256;
  silu_mul_bwd_kernel<<<(unsigned)(blocks < 132 * 16 ? blocks : 132 * 16), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)gate_up, (const __nv_bfloat16*)dact, T, (int)I, (__nv_bfloat16*)dgate_up);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_embed_gather(const void* table, const int64_t* ids, int64_t T, int64_t H, void* out,
                                prl_stream_t stream) {
  PRL_CHECK_ARG(table && ids && out && T >= 1 && H >= 8 && H % 8 == 0, "prl_embed_gather: bad argument");
  embed_gather_kernel<<<(unsigned)(T < 4096 ? T : 4096), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)table, ids, T,
                                                                                         (int)H, (__nv_bfloat16*)out);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_embed_scatter_add(float* dtable, const int64_t* ids, const void* dh, int64_t T, int64_t H,
                                     prl_stream_t stream) {
  PRL_CHECK_ARG(dtable && ids && dh && T >= 1 && H >= 8 && H % 8 == 0, "prl_embed_scatter_add: bad argument");
  embed_scatter_kernel<<<(unsigned)(T < 4096 ? T : 4096), 256, 0, (cudaStream_t)stream>>>(dtable, ids,
                                                                                          (const __nv_bfloat16*)dh, T, (int)H);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}
