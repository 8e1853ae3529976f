// Hot path (2c): fused AdamW over a flat parameter arena.
//
// Replaces, in one read-modify-write pass over the optimizer state:
//   torch.optim.AdamW built by pipelinerl/finetune/optim.py:8-29 (decay groups:
//   names containing "bias" / "LayerNorm.weight" get weight_decay 0),
//   clip_grad_norm_ at finetune_loop.py:739 and the fp32->bf16 re-cast that the
//   DeepSpeed bf16 optimizer performs at finetune_loop.py:727-736.
//
// Two launches, no host sync: (1) sum-of-squares partials of the (scaled)
// gradient, (2) the update; every block of (2) re-reduces the few hundred
// partials in a fixed order, so the clip coefficient is deterministic.
//
// HBM-bound: 14 B/param read (g bf16 2, master 4, m 4, v 4) + 14 B/param
// written (master 4, m 4, v 4, bf16 2) = 28 B/param (+2 with the bf16 "lo"
// residual that makes the output head fp32-equivalent).
#include "prl_common.cuh"
#include <math.h>

namespace prl {
namespace {

constexpr int kThreads = 256;
constexpr int kVec = 4;                         // elements per thread per iteration
constexpr int kChunk = kThreads * kVec * 4;     // 4096 elements per block iteration
constexpr int kMaxNormBlocks = 132 * 8;

struct AdamWorkspace {
  double partial[kMaxNormBlocks];
  int n_partials;
};

template <bool kBf16>
__device__ __forceinline__ void load_grad4(const void* g, int64_t i, float scale, float out[4]) {
  if (kBf16) {
    const uint2 raw = ld_stream_u2(reinterpret_cast<const uint2*>(static_cast<const __nv_bfloat16*>(g) + i));
    out[0] = bf16_bits_to_float(raw.x & 0xffffu) * scale;
    out[1] = bf16_bits_to_float(raw.x >> 16) * scale;
    out[2] = bf16_bits_to_float(raw.y & 0xffffu) * scale;
    out[3] = bf16_bits_to_float(raw.y >> 16) * scale;
  } else {
    const float4 raw = ld_stream_f4(reinterpret_cast<const float4*>(static_cast<const float*>(g) + i));
    out[0] = raw.x * scale; out[1] = raw.y * scale; out[2] = raw.z * scale; out[3] = raw.w * scale;
  }
}
template <bool kBf16>
__device__ __forceinline__ float load_grad1(const void* g, int64_t i, float scale) {
  if (kBf16) return __bfloat162float(static_cast<const __nv_bfloat16*>(g)[i]) * scale;
  return static_cast<const float*>(g)[i] * scale;
}

template <bool kBf16>
__global__ void __launch_bounds__(kThreads) grad_sumsq_kernel(const void* __restrict__ g, int64_t n, float scale,
                                                             AdamWorkspace* ws) {
  double acc = 0.0;
  const int64_t n4 = n / 4;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n4; v += (int64_t)gridDim.x * blockDim.x) {
    float x[4];
    load_grad4<kBf16>(g, v * 4, scale, x);
    float s = x[0] * x[0];
    s = fmaf(x[1], x[1], s); s = fmaf(x[2], x[2], s); s = fmaf(x[3], x[3], s);
    acc += (double)s;
  }
  if (blockIdx.x == 0) {
    for (int64_t i = n4 * 4 + threadIdx.x; i < n; i += blockDim.x) {
      const float x = load_grad1<kBf16>(g, i, scale);
      acc += (double)x * (double)x;
    }
  }
  __shared__ double s_w[kThreads / kWarp];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int i = 0; i < kThreads / kWarp; ++i) t += s_w[i];
    ws->partial[blockIdx.x] = t;
    if (blockIdx.x == 0) ws->n_partials = gridDim.x;
  }
}

struct UpdateConsts {
  float lr, beta1, beta2, eps;
  float weight_decay;     // decay FACTOR 1 - lr*wd (1 for no-decay tensors)
  float step_size;        // lr / (1 - beta1^t)
  float bc2_sqrt;         // sqrt(1 - beta2^t)
  // torch evaluates these scalars in double precision before the fp32 tensor op; 1.f - 0.999f would be
  // off by 4.7e-5 relative
  float one_minus_beta1, one_minus_beta2;
  float max_grad_norm, grad_scale;
};

__device__ __forceinline__ void adam_elem(float g, float& p, float& m, float& v, const UpdateConsts& k, float wd /* decay factor */) {
  // same operation order as torch.optim.adamw (_single_tensor_adam)
  p = p * wd;                                  // wd = 1 - lr * weight_decay, evaluated in double on the host
  m = m + (g - m) * k.one_minus_beta1;         // lerp_(grad, 1 - beta1)
  v = v * k.beta2 + k.one_minus_beta2 * g * g; // mul_(beta2).addcmul_(g, g, 1 - beta2)
  const float denom = sqrtf(v) / k.bc2_sqrt + k.eps;
  p = p - k.step_size * (m / denom);
}

template <bool kBf16>
__global__ void __launch_bounds__(kThreads) adamw_kernel(prl_adamw_args a, UpdateConsts k, const AdamWorkspace* ws,
                                                         float* __restrict__ grad_norm_out, int n_norm_blocks) {
  // global grad norm: fixed-order re-reduction of the partials (identical in every block)
  __shared__ float s_clip;
  __shared__ double s_red[kThreads / kWarp];
  {
    double t = 0;
    for (int i = threadIdx.x; i < n_norm_blocks; i += blockDim.x) t += ws->partial[i];
    t = warp_sum(t);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = t;
    __syncthreads();
    if (threadIdx.x == 0) {
      double tot = 0;
      for (int i = 0; i < kThreads / kWarp; ++i) tot += s_red[i];
      const float norm = (float)sqrt(tot);
      float clip = 1.f;
      if (k.max_grad_norm > 0.f) {
        // torch.nn.utils.clip_grad_norm_: clip_coef = max_norm / (total_norm + 1e-6), clamped to 1
        clip = fminf(k.max_grad_norm / (norm + 1e-6f), 1.f);
      }
      s_clip = clip;
      if (blockIdx.x == 0 && grad_norm_out) *grad_norm_out = norm;
    }
    __syncthreads();
  }
  const float gscale = k.grad_scale * s_clip;

  __shared__ int s_tensor;
  const int64_t n_chunks = (a.n + kChunk - 1) / kChunk;
  for (int64_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const int64_t base = c * kChunk;
    const int64_t end = (base + kChunk < a.n) ? base + kChunk : a.n;
    // decay group lookup: binary search for the tensor containing `base`
    if (threadIdx.x == 0) {
      int lo = 0, hi = a.n_tensors;  // invariant: offsets[lo] <= base < offsets[hi]
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (a.tensor_offsets[mid] <= base) lo = mid; else hi = mid;
      }
      s_tensor = lo;
    }
    __syncthreads();
    int tix = s_tensor;
    int64_t t_end = a.tensor_offsets[tix + 1];
    __syncthreads();

#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int64_t i = base + ((int64_t)it * kThreads + threadIdx.x) * kVec;
      if (i >= end) break;
      while (i >= t_end) { ++tix; t_end = a.tensor_offsets[tix + 1]; }
      const bool fast = (i + kVec <= end) && (i + kVec <= t_end) && ((i & 3) == 0);
      if (fast) {
        float g[4];
        load_grad4<kBf16>(a.grad, i, gscale, g);
        float4 p = *reinterpret_cast<const float4*>(a.master + i);
        float4 m = *reinterpret_cast<const float4*>(a.exp_avg + i);
        float4 v = *reinterpret_cast<const float4*>(a.exp_avg_sq + i);
        const float wd = a.tensor_no_decay[tix] ? 1.f : k.weight_decay;
        adam_elem(g[0], p.x, m.x, v.x, k, wd);
        adam_elem(g[1], p.y, m.y, v.y, k, wd);
        adam_elem(g[2], p.z, m.z, v.z, k, wd);
        adam_elem(g[3], p.w, m.w, v.w, k, wd);
        *reinterpret_cast<float4*>(a.master + i) = p;
        *reinterpret_cast<float4*>(a.exp_avg + i) = m;
        *reinterpret_cast<float4*>(a.exp_avg_sq + i) = v;
        if (a.param_bf16) {
          const uint32_t b0 = float_to_bf16_bits(p.x), b1 = float_to_bf16_bits(p.y);
          const uint32_t b2 = float_to_bf16_bits(p.z), b3 = float_to_bf16_bits(p.w);
          st_stream_u2(reinterpret_cast<uint2*>(static_cast<__nv_bfloat16*>(a.param_bf16) + i),
                       make_uint2(b0 | (b1 << 16), b2 | (b3 << 16)));
          if (a.param_bf16_lo) {
            const uint32_t l0 = float_to_bf16_bits(p.x - bf16_bits_to_float(b0));
            const uint32_t l1 = float_to_bf16_bits(p.y - bf16_bits_to_float(b1));
            const uint32_t l2 = float_to_bf16_bits(p.z - bf16_bits_to_float(b2));
            const uint32_t l3 = float_to_bf16_bits(p.w - bf16_bits_to_float(b3));
            st_stream_u2(reinterpret_cast<uint2*>(static_cast<__nv_bfloat16*>(a.param_bf16_lo) + i),
                         make_uint2(l0 | (l1 << 16), l2 | (l3 << 16)));
          }
        }
      } else {
        int tj = tix;
        int64_t tj_end = t_end;
        for (int64_t j = i; j < i + kVec && j < end; ++j) {
          while (j >= tj_end) { ++tj; tj_end = a.tensor_offsets[tj + 1]; }
          const float g = load_grad1<kBf16>(a.grad, j, gscale);
          float p = a.master[j], m = a.exp_avg[j], v = a.exp_avg_sq[j];
          adam_elem(g, p, m, v, k, a.tensor_no_decay[tj] ? 1.f : k.weight_decay);
          a.master[j] = p; a.exp_avg[j] = m; a.exp_avg_sq[j] = v;
          if (a.param_bf16) {
            const __nv_bfloat16 hi = __float2bfloat16_rn(p);
            static_cast<__nv_bfloat16*>(a.param_bf16)[j] = hi;
            if (a.param_bf16_lo)
              static_cast<__nv_bfloat16*>(a.param_bf16_lo)[j] = __float2bfloat16_rn(p - __bfloat162float(hi));
          }
        }
      }
    }
  }
}


// =====================================================================================================
// Learner data parallelism as ONE fused exchange step over NVLink peer memory (SURVEY §8e, row a7):
//   reduce-scatter(grad) -> clip -> AdamW on this rank's 1/Ng shard -> all-gather(bf16 params)
// Every rank maps every other rank's full gradient arena and bf16 parameter arena (CUDA IPC).  Kernel A
// (shard_reduce) sums the Ng gradients of this rank's shard straight out of peer memory (P2P loads) into an
// fp32 scratch and leaves its partial sum of squares in every rank's norm table; kernel B (shard_update)
// applies clip + AdamW to the shard (fp32 master / m / v exist ONLY for the shard: optimizer state is sharded
// Ng ways) and stores the re-cast bf16 parameters into every rank's parameter arena (P2P stores).
// Replaces the DDP/ZeRO gradient all-reduce + per-rank full AdamW of the reference
// (finetune_loop.py:716-755, conf/deepspeed/*.json); no NCCL on the data path, host barriers only between phases.
// =====================================================================================================
constexpr int kMaxPeers = 8;

struct ShardParams {
  int64_t n, lo, hi;
  float* master; float* exp_avg; float* exp_avg_sq;     // shard-local, index i - lo
  const void* grads[kMaxPeers];
  void* shadows[kMaxPeers];
  int n_peers, rank, grad_is_bf16;
  float* gsum;                                          // [hi - lo]
  double* norm_tables[kMaxPeers];                       // norm_tables[p][r] = rank r's partial, stored in rank p's memory
  const int64_t* tensor_offsets; const uint8_t* tensor_no_decay; int n_tensors;
  float grad_scale;
};

template <bool kBf16>
__global__ void __launch_bounds__(kThreads) shard_reduce_kernel(ShardParams a, AdamWorkspace* ws) {
  double acc = 0.0;
  const int64_t n4 = (a.hi - a.lo) / 4;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < n4; v += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = a.lo + v * 4;
    float s[4] = {0.f, 0.f, 0.f, 0.f};
    for (int p = 0; p < a.n_peers; ++p) {   // fixed peer order on every rank -> bitwise identical sums everywhere
      float g[4];
      load_grad4<kBf16>(a.grads[p], i, a.grad_scale, g);
      s[0] += g[0]; s[1] += g[1]; s[2] += g[2]; s[3] += g[3];
    }
    *reinterpret_cast<float4*>(a.gsum + v * 4) = make_float4(s[0], s[1], s[2], s[3]);
    acc += (double)(s[0] * s[0] + s[1] * s[1] + s[2] * s[2] + s[3] * s[3]);
  }
  __shared__ double s_w[kThreads / kWarp];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int i = 0; i < kThreads / kWarp; ++i) t += s_w[i];
    ws->partial[blockIdx.x] = t;
  }
}

__global__ void shard_norm_publish_kernel(ShardParams a, const AdamWorkspace* ws, int n_blocks) {
  __shared__ double s_red[kThreads / kWarp];
  double t = 0;
  for (int i = threadIdx.x; i < n_blocks; i += blockDim.x) t += ws->partial[i];
  t = warp_sum(t);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0;
    for (int i = 0; i < kThreads / kWarp; ++i) tot += s_red[i];
    for (int p = 0; p < a.n_peers; ++p) a.norm_tables[p][a.rank] = tot;   // P2P store into every rank's table
    __threadfence_system();
  }
}

__global__ void __launch_bounds__(kThreads) shard_update_kernel(ShardParams a, UpdateConsts k, const double* norm_table,
                                                                float* __restrict__ grad_norm_out) {
  __shared__ float s_clip;
  __shared__ int s_tensor;
  if (threadIdx.x == 0) {
    double tot = 0;
    for (int r = 0; r < a.n_peers; ++r) tot += norm_table[r];
    const float norm = (float)sqrt(tot);
    s_clip = (k.max_grad_norm > 0.f) ? fminf(k.max_grad_norm / (norm + 1e-6f), 1.f) : 1.f;
    if (blockIdx.x == 0 && grad_norm_out) *grad_norm_out = norm;
  }
  __syncthreads();
  const float clip = s_clip;
  const int64_t n_chunks = (a.hi - a.lo + kChunk - 1) / kChunk;
  for (int64_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const int64_t base = a.lo + c * kChunk;
    const int64_t end = (base + kChunk < a.hi) ? base + kChunk : a.hi;
    if (threadIdx.x == 0) {
      int lo = 0, hi = a.n_tensors;
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (a.tensor_offsets[mid] <= base) lo = mid; else hi = mid;
      }
      s_tensor = lo;
    }
    __syncthreads();
    int tix = s_tensor;
    int64_t t_end = a.tensor_offsets[tix + 1];
    __syncthreads();
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int64_t i = base + ((int64_t)it * kThreads + threadIdx.x) * kVec;
      if (i >= end) break;
      // shard bounds and tensor starts are multiples of 64 elements (arena alignment), so a 4-vector never straddles
      while (i >= t_end) { ++tix; t_end = a.tensor_offsets[tix + 1]; }
      const int64_t j = i - a.lo;
      const float4 g = *reinterpret_cast<const float4*>(a.gsum + j);
      float4 p = *reinterpret_cast<const float4*>(a.master + j);
      float4 m = *reinterpret_cast<const float4*>(a.exp_avg + j);
      float4 v = *reinterpret_cast<const float4*>(a.exp_avg_sq + j);
      const float wd = a.tensor_no_decay[tix] ? 1.f : k.weight_decay;
      adam_elem(g.x * clip, p.x, m.x, v.x, k, wd);
      adam_elem(g.y * clip, p.y, m.y, v.y, k, wd);
      adam_elem(g.z * clip, p.z, m.z, v.z, k, wd);
      adam_elem(g.w * clip, p.w, m.w, v.w, k, wd);
      *reinterpret_cast<float4*>(a.master + j) = p;
      *reinterpret_cast<float4*>(a.exp_avg + j) = m;
      *reinterpret_cast<float4*>(a.exp_avg_sq + j) = v;
      const uint32_t b0 = float_to_bf16_bits(p.x), b1 = float_to_bf16_bits(p.y);
      const uint32_t b2 = float_to_bf16_bits(p.z), b3 = float_to_bf16_bits(p.w);
      const uint2 packed = make_uint2(b0 | (b1 << 16), b2 | (b3 << 16));
      for (int q = 0; q < a.n_peers; ++q)   // all-gather: every rank's bf16 parameter arena receives this shard
        *reinterpret_cast<uint2*>(static_cast<__nv_bfloat16*>(a.shadows[q]) + i) = packed;
    }
  }
}

}  // namespace
}  // namespace prl

using namespace prl;

extern "C" size_t prl_adamw_workspace_bytes(void) { return sizeof(AdamWorkspace); }

extern "C" int prl_adamw_step(const prl_adamw_args* a, float* grad_norm_out, void* workspace,
                              size_t workspace_bytes, prl_stream_t stream_) {
  PRL_CHECK_ARG(a && workspace, "prl_adamw_step: NULL argument");
  PRL_CHECK_ARG(workspace_bytes >= sizeof(AdamWorkspace), "prl_adamw_step: workspace too small");
  PRL_CHECK_ARG(a->n >= 0, "prl_adamw_step: n < 0");
  if (a->n == 0) return PRL_OK;
  PRL_CHECK_ARG(a->master && a->exp_avg && a->exp_avg_sq && a->grad, "prl_adamw_step: NULL state pointer");
  PRL_CHECK_ARG(a->n_tensors >= 1 && a->tensor_offsets && a->tensor_no_decay, "prl_adamw_step: missing tensor table");
  PRL_CHECK_ARG(a->step >= 1, "prl_adamw_step: step is 1-based");
  PRL_CHECK_ARG(((uintptr_t)a->master % 16 == 0) && ((uintptr_t)a->exp_avg % 16 == 0) &&
                    ((uintptr_t)a->exp_avg_sq % 16 == 0) && ((uintptr_t)a->grad % 16 == 0) &&
                    (!a->param_bf16 || (uintptr_t)a->param_bf16 % 8 == 0) &&
                    (!a->param_bf16_lo || (uintptr_t)a->param_bf16_lo % 8 == 0),
                "prl_adamw_step: arena pointers must be 16-byte aligned");
  cudaStream_t stream = (cudaStream_t)stream_;
  AdamWorkspace* ws = (AdamWorkspace*)workspace;

  const float gs = a->grad_scale == 0.f ? 1.f : a->grad_scale;
  int norm_blocks = (int)((a->n / 4 + kThreads - 1) / kThreads);
  if (norm_blocks < 1) norm_blocks = 1;
  const int cap = num_sms() * 8 < kMaxNormBlocks ? num_sms() * 8 : kMaxNormBlocks;
  if (norm_blocks > cap) norm_blocks = cap;
  if (a->grad_is_bf16) grad_sumsq_kernel<true><<<norm_blocks, kThreads, 0, stream>>>(a->grad, a->n, gs, ws);
  else grad_sumsq_kernel<false><<<norm_blocks, kThreads, 0, stream>>>(a->grad, a->n, gs, ws);
  PRL_LAUNCH_CHECK();

  UpdateConsts k;
  k.lr = (float)a->lr; k.beta1 = (float)a->beta1; k.beta2 = (float)a->beta2; k.eps = (float)a->eps;
  k.weight_decay = (float)(1.0 - a->lr * a->weight_decay);  // decay FACTOR
  k.one_minus_beta1 = (float)(1.0 - a->beta1);
  k.one_minus_beta2 = (float)(1.0 - a->beta2);
  const double bc1 = 1.0 - pow(a->beta1, (double)a->step);
  const double bc2 = 1.0 - pow(a->beta2, (double)a->step);
  k.step_size = (float)(a->lr / bc1);
  k.bc2_sqrt = (float)sqrt(bc2);
  k.max_grad_norm = a->max_grad_norm;
  k.grad_scale = gs;

  const int64_t n_chunks = (a->n + kChunk - 1) / kChunk;
  int blocks = (int)(n_chunks < (int64_t)num_sms() * 8 ? n_chunks : (int64_t)num_sms() * 8);
  if (a->grad_is_bf16) adamw_kernel<true><<<blocks, kThreads, 0, stream>>>(*a, k, ws, grad_norm_out, norm_blocks);
  else adamw_kernel<false><<<blocks, kThreads, 0, stream>>>(*a, k, ws, grad_norm_out, norm_blocks);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

// ---- sharded exchange step (see the block comment above shard_reduce_kernel) -----------------------------------
static int fill_shard_params(const prl_adamw_shard_args* a, ShardParams* sp) {
  PRL_CHECK_ARG(a, "prl_adamw_sharded: NULL args");
  PRL_CHECK_ARG(a->n_peers >= 1 && a->n_peers <= kMaxPeers && a->rank >= 0 && a->rank < a->n_peers,
                "prl_adamw_sharded: need 1..8 peers and a valid rank");
  PRL_CHECK_ARG(a->shard_begin >= 0 && a->shard_end >= a->shard_begin && a->shard_end <= a->n &&
                    a->shard_begin % 64 == 0 && (a->shard_end % 64 == 0 || a->shard_end == a->n),
                "prl_adamw_sharded: shard bounds must be 64-element aligned");
  PRL_CHECK_ARG(a->master && a->exp_avg && a->exp_avg_sq && a->gsum_scratch && a->tensor_offsets && a->tensor_no_decay,
                "prl_adamw_sharded: NULL state pointer");
  sp->n = a->n; sp->lo = a->shard_begin; sp->hi = a->shard_end;
  sp->master = a->master; sp->exp_avg = a->exp_avg; sp->exp_avg_sq = a->exp_avg_sq;
  sp->n_peers = a->n_peers; sp->rank = a->rank; sp->grad_is_bf16 = a->grad_is_bf16;
  sp->gsum = a->gsum_scratch;
  for (int p = 0; p < a->n_peers; ++p) {
    PRL_CHECK_ARG(a->grads[p] && a->shadows[p] && a->norm_tables[p], "prl_adamw_sharded: NULL peer pointer %d", p);
    sp->grads[p] = a->grads[p]; sp->shadows[p] = a->shadows[p]; sp->norm_tables[p] = a->norm_tables[p];
  }
  sp->tensor_offsets = a->tensor_offsets; sp->tensor_no_decay = a->tensor_no_decay; sp->n_tensors = a->n_tensors;
  sp->grad_scale = a->grad_scale == 0.f ? 1.f : a->grad_scale;
  return PRL_OK;
}

extern "C" int prl_adamw_sharded_reduce(const prl_adamw_shard_args* a, void* workspace, size_t workspace_bytes,
                                        prl_stream_t stream_) {
  ShardParams sp;
  int rc = fill_shard_params(a, &sp);
  if (rc) return rc;
  PRL_CHECK_ARG(workspace && workspace_bytes >= sizeof(AdamWorkspace), "prl_adamw_sharded_reduce: workspace too small");
  cudaStream_t stream = (cudaStream_t)stream_;
  AdamWorkspace* ws = (AdamWorkspace*)workspace;
  const int64_t n4 = (sp.hi - sp.lo) / 4;
  int blocks = (int)((n4 + kThreads - 1) / kThreads);
  if (blocks < 1) blocks = 1;
  const int cap = num_sms() * 8 < kMaxNormBlocks ? num_sms() * 8 : kMaxNormBlocks;
  if (blocks > cap) blocks = cap;
  if (sp.grad_is_bf16) shard_reduce_kernel<true><<<blocks, kThreads, 0, stream>>>(sp, ws);
  else shard_reduce_kernel<false><<<blocks, kThreads, 0, stream>>>(sp, ws);
  PRL_LAUNCH_CHECK();
  shard_norm_publish_kernel<<<1, kThreads, 0, stream>>>(sp, ws, blocks);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

extern "C" int prl_adamw_sharded_update(const prl_adamw_shard_args* a, float* grad_norm_out, prl_stream_t stream_) {
  ShardParams sp;
  int rc = fill_shard_params(a, &sp);
  if (rc) return rc;
  PRL_CHECK_ARG(a->step >= 1, "prl_adamw_sharded_update: step is 1-based");
  UpdateConsts k;
  k.lr = (float)a->lr; k.beta1 = (float)a->beta1; k.beta2 = (float)a->beta2; k.eps = (float)a->eps;
  k.weight_decay = (float)(1.0 - a->lr * a->weight_decay);
  k.one_minus_beta1 = (float)(1.0 - a->beta1);
  k.one_minus_beta2 = (float)(1.0 - a->beta2);
  const double bc1 = 1.0 - pow(a->beta1, (double)a->step);
  const double bc2 = 1.0 - pow(a->beta2, (double)a->step);
  k.step_size = (float)(a->lr / bc1);
  k.bc2_sqrt = (float)sqrt(bc2);
  k.max_grad_norm = a->max_grad_norm;
  k.grad_scale = 1.f;
  const int64_t n_chunks = (sp.hi - sp.lo + kChunk - 1) / kChunk;
  if (n_chunks == 0) return PRL_OK;
  int blocks = (int)(n_chunks < (int64_t)num_sms() * 8 ? n_chunks : (int64_t)num_sms() * 8);
  shard_update_kernel<<<blocks, kThreads, 0, (cudaStream_t)stream_>>>(sp, k, a->norm_tables[a->rank], grad_norm_out);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}


// ---- bf16 residual of an fp32 master tensor: lo = bf16(master - float(bf16(master))) -------------------------------------
// The lm_head is computed in fp32 on both sides of the reference (vllm_quantization.py:266-278, finetune/checkpoints.py:44-105).
// Here the head weight travels as TWO bf16 operand streams, hi = bf16(master) (the ordinary bf16 parameter) and this
// residual; hi + lo carries 16 mantissa bits, the tensor core accumulates both in fp32.  Written into up to 8 destinations
// (every data-parallel learner's arena tail, over NVLink peer memory), 16-byte stores.
namespace prl { namespace {
struct ResidualDsts { __nv_bfloat16* p[8]; };
__global__ void __launch_bounds__(256) bf16_residual_kernel(const float* __restrict__ master, int64_t n, ResidualDsts d, int n_dst) {
  const int64_t i8 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i8 >= n) return;
  if (i8 + 8 <= n) {
    const float4 a = ld_stream_f4(reinterpret_cast<const float4*>(master + i8));
    const float4 b = ld_stream_f4(reinterpret_cast<const float4*>(master + i8 + 4));
    const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    uint32_t w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float h0 = __bfloat162float(__float2bfloat16_rn(v[2 * k])), h1 = __bfloat162float(__float2bfloat16_rn(v[2 * k + 1]));
      w[k] = float_to_bf16_bits(v[2 * k] - h0) | (float_to_bf16_bits(v[2 * k + 1] - h1) << 16);
    }
    for (int t = 0; t < n_dst; ++t) st_stream_u4(reinterpret_cast<uint4*>(d.p[t] + i8), make_uint4(w[0], w[1], w[2], w[3]));
  } else {
    for (int64_t i = i8; i < n; ++i) {
      const float h = __bfloat162float(__float2bfloat16_rn(master[i]));
      for (int t = 0; t < n_dst; ++t) d.p[t][i] = __float2bfloat16_rn(master[i] - h);
    }
  }
}
} }

extern "C" int prl_bf16_residual(const float* master, int64_t n, void* const* lo_dsts, int32_t n_dst, prl_stream_t stream_) {
  PRL_CHECK_ARG(master && lo_dsts && n >= 1 && n_dst >= 1 && n_dst <= 8, "prl_bf16_residual: bad argument");
  PRL_CHECK_ARG((uintptr_t)master % 16 == 0, "prl_bf16_residual: master must be 16-byte aligned");
  prl::ResidualDsts d = {};
  for (int t = 0; t < n_dst; ++t) {
    PRL_CHECK_ARG(lo_dsts[t] && (uintptr_t)lo_dsts[t] % 16 == 0, "prl_bf16_residual: destinations must be 16-byte aligned");
    d.p[t] = (__nv_bfloat16*)lo_dsts[t];
  }
  const int64_t threads = (n + 7) / 8;
  prl::bf16_residual_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(master, n, d, (int)n_dst);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}
