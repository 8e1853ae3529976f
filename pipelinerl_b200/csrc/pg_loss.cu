// Hot path (2a): policy-gradient loss tail, forward + backward + all statistics
// in one streaming pass over the packed row.
//
// Replaces pipelinerl/finetune/rl/__init__.py:237-439 (everything rl_step does
// after new_logprobs/entropy exist) and rl/utils.py:71-92 (sum_sum).  In the
// reference sum_sum() is a Python loop over segments but mathematically a plain
// masked sum, so the only place the segment structure matters is GSPO
// (rl/__init__.py:310-350, rl/utils.py:106-208), handled by a per-segment
// pre-pass.
//
// HBM-bound: algorithmic traffic is 44 B/token read (new_lp 4, entropy 4,
// labels 8, 7 fp32 columns) + 4 B/token written (dL/dlogprob).
#include "prl_common.cuh"
#include <math.h>

namespace prl {
namespace {

constexpr int kThreads = 256;

// sum accumulators
enum {
  A_LOSS = 0, A_REWARD, A_ENTROPY, A_OLD, A_NEW, A_REF, A_ADV, A_KL, A_KL_NO, A_ABS_LR,
  A_RATIO, A_RATIO_SUM, A_RATIO_SQ, A_RATIO_REF_NEW, A_RATIO_REF_OLD, A_CLAMP_REF_NEW,
  A_CLAMP_NEW_OLD, A_TOKEN_WEIGHT, A_COUNT, A_NSEQ, A_NSUM
};
// max / min accumulators
enum { M_REWARD = 0, M_ADV, M_KL, M_TW, M_NMM };

struct Partial {
  double sum[A_NSUM];
  float mx[M_NMM];
  float mn[M_NMM];
  int flags;
  int pad;
};

struct SegSums {  // GSPO per-segment accumulators (doubles: order-insensitive to ~1e-16)
  double lrn_sum, adv_sum, tok_count, weight_sum;
};

struct Workspace {
  unsigned int ticket;
  unsigned int pad[3];
};

__device__ __forceinline__ float token_weight(const prl_pg_config& c, float group_tokens, float overflow) {
  float w = c.group_normalization ? (1.0f / group_tokens) : (1.0f / c.batch_size);
  if (c.overlong_filtering) w = w * (1.0f - overflow);
  return w;
}

// ---- GSPO pre-pass: per-segment masked sums (rl/utils.py:106-208) ----------
__global__ void __launch_bounds__(kThreads) gspo_segment_kernel(prl_pg_batch b, prl_pg_config c, SegSums* seg) {
  const int64_t n = b.T - 1;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    if (b.labels[t + 1] == -100) continue;
    const int64_t s = b.segment_ids[t + 1];
    if (s < 0 || s >= b.n_segments) continue;
    const float lr = b.new_logprobs[t] - b.old_logprobs[t + 1];
    const float w = token_weight(c, b.group_tokens[t + 1], b.overflow[t + 1]);
    atomicAdd(&seg[s].lrn_sum, (double)lr);
    atomicAdd(&seg[s].adv_sum, (double)b.advantages[t + 1]);
    atomicAdd(&seg[s].tok_count, 1.0);
    atomicAdd(&seg[s].weight_sum, (double)w);
  }
}

struct SegTerm { float grad_coef; float indicator; };

// per-segment GSPO quantities (rl/__init__.py:320-346)
__device__ __forceinline__ void gspo_segment_terms(const SegSums& ss, const prl_pg_config& c, float& loss_term,
                                                   float& grad_coef, float& indicator) {
  const float cnt = (float)ss.tok_count;
  const float cnt_c = fmaxf(cnt, 1e-6f);
  const float wsum = (float)ss.weight_sum;
  const float gr = expf((float)ss.lrn_sum / cnt_c);
  const float ga = (float)ss.adv_sum / cnt_c;
  const bool valid = (cnt > 0.f) && (wsum > 0.f);
  const float lo = 1.f - c.epsilon_low, hi = 1.f + c.epsilon_high;
  const float gr_c = fminf(fmaxf(gr, lo), hi);
  const float s1 = gr * ga, s2 = gr_c * ga;
  const bool clipped = (gr_c != gr);
  indicator = (clipped && valid) ? 1.f : 0.f;
  loss_term = valid ? fminf(s1, s2) * wsum : 0.f;
  // d min(s1,s2)/d gr: inside the clip range both branches carry gradient (tie: halves add up);
  // outside only the unclipped branch when it is the smaller one.
  float dmin = 0.f;
  if (!clipped) dmin = ga;
  else if (s1 < s2) dmin = ga;
  else if (s1 == s2) dmin = 0.5f * ga;
  // d gr / d lrn_sum = gr / cnt_c ; loss = -sum(min * wsum)
  grad_coef = valid ? (-wsum * dmin * gr / cnt_c) : 0.f;
}

// ---- main pass ---------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) pg_loss_kernel(prl_pg_batch b, prl_pg_config c, float* __restrict__ loss_out,
                                                          float* __restrict__ dlp, float* __restrict__ dent,
                                                          double* __restrict__ stats, int* __restrict__ nonfinite,
                                                          Workspace* ws, Partial* partials, const SegSums* seg,
                                                          const double* __restrict__ seg_local_count) {
  const int64_t n = b.T - 1;
  float acc[A_NSUM];
  float mx[M_NMM], mn[M_NMM];
#pragma unroll
  for (int i = 0; i < A_NSUM; ++i) acc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < M_NMM; ++i) { mx[i] = -INFINITY; mn[i] = INFINITY; }
  int flags = 0;
  const bool gspo = (c.policy_loss == PRL_LOSS_GSPO);
  const float lo = 1.f - c.epsilon_low, hi = 1.f + c.epsilon_high;
  const float cv = c.clamp_log_ratio_ref_new_value;

  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const bool m = (b.labels[t + 1] != -100);
    if (b.position_ids && b.position_ids[t + 1] == 0) acc[A_NSEQ] += 1.f;
    const float new_lp = b.new_logprobs[t];
    // the reference asserts finiteness over ALL positions, masked or not (:213, :263, :291)
    if (!isfinite(new_lp)) flags |= 1;
    const float ref_lp = b.ref_logprobs[t + 1];
    const float lr_ref_new = ref_lp - new_lp;
    if (!isfinite(lr_ref_new)) flags |= 2;
    const float lr_c = fminf(fmaxf(lr_ref_new, -cv), cv);
    const float kl = expf(lr_c) - lr_c - 1.f;
    if (!isfinite(kl)) flags |= 4;
    float g = 0.f, ge = 0.f;
    if (m) {
      const float old_lp = b.old_logprobs[t + 1];
      const float adv = b.advantages[t + 1];
      const float rew = b.rewards[t + 1];
      const float nl = b.num_labels[t + 1];
      const float ent = b.entropy ? b.entropy[t] : 0.f;
      const float w = token_weight(c, b.group_tokens[t + 1], b.overflow[t + 1]);
      const float lr = new_lp - old_lp;
      float ratio = expf(lr);
      const float kl_no = ratio - lr - 1.f;
      float lpw = c.use_advantages ? adv : rew;
      if (c.relu_log_p_weights) lpw = fmaxf(lpw, 0.f);
      const bool kl_in = fabsf(lr_ref_new) <= cv;  // clamp() passes gradient on the closed interval
      const float dkl = kl_in ? -(expf(lr_c) - 1.f) : 0.f;  // d approx_kl / d new_lp

      float policy = 0.f, dpol = 0.f, ind = 0.f;
      if (c.policy_loss == PRL_LOSS_PPO) {
        const float rc = fminf(fmaxf(ratio, lo), hi);
        const float s1 = ratio * lpw, s2 = rc * lpw;
        policy = fminf(s1, s2);
        const bool clipped = (rc != ratio);
        ind = clipped ? 1.f : 0.f;
        if (!clipped) dpol = lpw * ratio;             // tie: both halves carry ratio*lpw/2
        else if (s1 < s2) dpol = lpw * ratio;
        else if (s1 == s2) dpol = 0.5f * lpw * ratio;  // only reachable with lpw == 0
      } else if (c.policy_loss == PRL_LOSS_REINFORCE) {
        ind = (ratio > hi) ? 1.f : 0.f;
        ratio = fminf(fmaxf(ratio, 0.f), hi);          // the stats below see the clamped ratio (:308)
        policy = new_lp * lpw * ratio;
        dpol = lpw * ratio;                            // ratio is detached
      } else {  // GSPO: sequence-level objective; token loss comes from the segment terms
        const int64_t s = b.segment_ids[t + 1];
        if (s >= 0 && s < b.n_segments) {
          float lt, gc, si;
          gspo_segment_terms(seg[s], c, lt, gc, si);
          ind = si;
          g = b.sentinel ? 0.f : gc;
        }
      }
      if (!gspo) {
        const float tok = policy - c.kl_coef * kl + (c.use_entropy_loss ? c.entropy_bonus_coef * ent : 0.f);
        acc[A_LOSS] += tok * w;
        g = -w * (dpol - c.kl_coef * dkl);
        ge = c.use_entropy_loss ? (-w * c.entropy_bonus_coef) : 0.f;
      }
      const float inv = 1.f / nl;
      acc[A_REWARD] += rew * inv;
      acc[A_ENTROPY] += ent * inv;
      acc[A_OLD] += old_lp * inv;
      acc[A_NEW] += new_lp * inv;
      acc[A_REF] += ref_lp * inv;
      acc[A_ADV] += adv * inv;
      acc[A_KL] += kl * inv;
      acc[A_KL_NO] += kl_no * inv;
      acc[A_ABS_LR] += fabsf(lr) * inv;
      acc[A_RATIO] += ratio * inv;
      acc[A_RATIO_SUM] += ratio;
      acc[A_RATIO_SQ] += ratio * ratio;
      acc[A_RATIO_REF_NEW] += expf(lr_ref_new) * inv;
      acc[A_RATIO_REF_OLD] += expf(ref_lp - old_lp) * inv;
      acc[A_CLAMP_REF_NEW] += ((fabsf(lr_ref_new) > cv) ? 1.f : 0.f) * inv;
      acc[A_CLAMP_NEW_OLD] += ind * inv;
      acc[A_TOKEN_WEIGHT] += w * inv;
      acc[A_COUNT] += 1.f;
      mx[M_REWARD] = fmaxf(mx[M_REWARD], rew); mn[M_REWARD] = fminf(mn[M_REWARD], rew);
      mx[M_ADV] = fmaxf(mx[M_ADV], adv);       mn[M_ADV] = fminf(mn[M_ADV], adv);
      mx[M_KL] = fmaxf(mx[M_KL], kl);          mn[M_KL] = fminf(mn[M_KL], kl);
      mx[M_TW] = fmaxf(mx[M_TW], w);           mn[M_TW] = fminf(mn[M_TW], w);
    }
    if (dlp) dlp[t] = g;
    if (dent) dent[t] = ge;
  }

  // block reduction -> partials[blockIdx]
  __shared__ double s_sum[kThreads / kWarp][A_NSUM];
  __shared__ float s_mx[kThreads / kWarp][M_NMM], s_mn[kThreads / kWarp][M_NMM];
  __shared__ int s_flags[kThreads / kWarp];
  __shared__ bool s_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < A_NSUM; ++i) {
    const double v = warp_sum((double)acc[i]);
    if (lane == 0) s_sum[warp][i] = v;
  }
#pragma unroll
  for (int i = 0; i < M_NMM; ++i) {
    const float a = warp_max(mx[i]), z = warp_min(mn[i]);
    if (lane == 0) { s_mx[warp][i] = a; s_mn[warp][i] = z; }
  }
  flags = __reduce_or_sync(0xffffffffu, flags);
  if (lane == 0) s_flags[warp] = flags;
  __syncthreads();
  if (threadIdx.x < A_NSUM) {
    double v = 0;
    for (int w2 = 0; w2 < kThreads / kWarp; ++w2) v += s_sum[w2][threadIdx.x];
    partials[blockIdx.x].sum[threadIdx.x] = v;
  } else if (threadIdx.x >= 32 && threadIdx.x < 32 + M_NMM) {
    const int i = threadIdx.x - 32;
    float a = -INFINITY, z = INFINITY;
    for (int w2 = 0; w2 < kThreads / kWarp; ++w2) { a = fmaxf(a, s_mx[w2][i]); z = fminf(z, s_mn[w2][i]); }
    partials[blockIdx.x].mx[i] = a;
    partials[blockIdx.x].mn[i] = z;
  } else if (threadIdx.x == 64) {
    int f = 0;
    for (int w2 = 0; w2 < kThreads / kWarp; ++w2) f |= s_flags[w2];
    partials[blockIdx.x].flags = f;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(&ws->ticket, 1u);
    s_last = (prev == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();

  // ---- final, deterministic reduction by the last block ----------------------
  __shared__ double f_sum[A_NSUM];
  __shared__ float f_mx[M_NMM], f_mn[M_NMM];
  __shared__ int f_flags;
  __shared__ double f_gspo;
  if (threadIdx.x < A_NSUM) {
    double v = 0;
    for (unsigned int i = 0; i < gridDim.x; ++i) v += partials[i].sum[threadIdx.x];
    f_sum[threadIdx.x] = v;
  } else if (threadIdx.x >= 32 && threadIdx.x < 32 + M_NMM) {
    const int k = threadIdx.x - 32;
    float a = -INFINITY, z = INFINITY;
    for (unsigned int i = 0; i < gridDim.x; ++i) { a = fmaxf(a, partials[i].mx[k]); z = fminf(z, partials[i].mn[k]); }
    f_mx[k] = a; f_mn[k] = z;
  } else if (threadIdx.x == 64) {
    int f = 0;
    for (unsigned int i = 0; i < gridDim.x; ++i) f |= partials[i].flags;
    f_flags = f;
  } else if (threadIdx.x == 96) {
    double tot = 0;
    if (gspo && !b.sentinel) {
      for (int s = 0; s < b.n_segments; ++s) {
        float lt, gc, si;
        gspo_segment_terms(seg[s], c, lt, gc, si);
        // sequence parallelism: `seg` holds the sums over ALL ranks; this rank reports the share of a segment's loss that
        // its own tokens carry, so that the ranks' losses add up to the loss of the whole row
        double share = 1.0;
        if (seg_local_count != nullptr) share = seg[s].tok_count > 0 ? seg_local_count[s] / seg[s].tok_count : 0.0;
        tot += (double)lt * share;
      }
    }
    f_gspo = tot;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const double total = gspo ? f_gspo : f_sum[A_LOSS];
    const float loss = (float)(-total);
    int f = f_flags;
    if (!isfinite(loss)) f |= 8;
    *loss_out = loss;
    *nonfinite = f;
    stats[PRL_STAT_LOSS] = loss; stats[PRL_STAT_MAX_LOSS] = loss; stats[PRL_STAT_MIN_LOSS] = loss;
    stats[PRL_STAT_REWARD] = f_sum[A_REWARD];
    stats[PRL_STAT_MAX_REWARD] = f_mx[M_REWARD]; stats[PRL_STAT_MIN_REWARD] = f_mn[M_REWARD];
    stats[PRL_STAT_ENTROPY] = f_sum[A_ENTROPY];
    stats[PRL_STAT_OLD_LOGPROBS] = f_sum[A_OLD];
    stats[PRL_STAT_NEW_LOGPROBS] = f_sum[A_NEW];
    stats[PRL_STAT_REF_LOGPROBS] = f_sum[A_REF];
    stats[PRL_STAT_ADVANTAGE] = f_sum[A_ADV];
    stats[PRL_STAT_MAX_ADVANTAGE] = f_mx[M_ADV]; stats[PRL_STAT_MIN_ADVANTAGE] = f_mn[M_ADV];
    stats[PRL_STAT_KL] = f_sum[A_KL];
    stats[PRL_STAT_KL_NEW_OLD] = f_sum[A_KL_NO];
    stats[PRL_STAT_MEAN_ABS_LOG_RATIO_NEW_OLD] = f_sum[A_ABS_LR];
    stats[PRL_STAT_MAX_KL] = f_mx[M_KL]; stats[PRL_STAT_MIN_KL] = f_mn[M_KL];
    stats[PRL_STAT_RATIO_NEW_OLD] = f_sum[A_RATIO];
    stats[PRL_STAT_RATIO_NEW_OLD_SUM] = f_sum[A_RATIO_SUM];
    stats[PRL_STAT_RATIO_NEW_OLD_SQUARED_SUM] = f_sum[A_RATIO_SQ];
    stats[PRL_STAT_RATIO_REF_NEW] = f_sum[A_RATIO_REF_NEW];
    stats[PRL_STAT_RATIO_REF_OLD] = f_sum[A_RATIO_REF_OLD];
    stats[PRL_STAT_CLAMP_LOG_RATIO_REF_NEW_INDICATOR] = f_sum[A_CLAMP_REF_NEW];
    stats[PRL_STAT_CLAMP_LOG_RATIO_NEW_OLD_INDICATOR] = f_sum[A_CLAMP_NEW_OLD];
    stats[PRL_STAT_TOKEN_WEIGHT] = f_sum[A_TOKEN_WEIGHT];
    stats[PRL_STAT_MAX_TOKEN_WEIGHT] = f_mx[M_TW]; stats[PRL_STAT_MIN_TOKEN_WEIGHT] = f_mn[M_TW];
    const double n_seq = b.position_ids ? 1.0 + f_sum[A_NSEQ] : (double)b.num_sequences;
    stats[PRL_STAT_KL_COEF] = n_seq * (double)c.kl_coef;
    stats[PRL_STAT_ENTROPY_BONUS_COEF] = n_seq * (double)c.entropy_bonus_coef;
    stats[PRL_STAT_NUM_OUTPUT_TOKENS_SUM] = f_sum[A_COUNT];
    stats[PRL_STAT_INPUT_SIZE] = (double)b.T;
    ws->ticket = 0;  // re-arm for the next call on this workspace
  }
}

constexpr int kMaxBlocks = 132 * 8;

}  // namespace
}  // namespace prl

using namespace prl;

extern "C" size_t prl_pg_workspace_bytes(int32_t max_segments) {
  if (max_segments < 0) max_segments = 0;
  return sizeof(Workspace) + sizeof(Partial) * (size_t)kMaxBlocks + sizeof(SegSums) * (size_t)max_segments;
}

extern "C" int prl_pg_loss_fwd_bwd(const prl_pg_batch* batch, const prl_pg_config* cfg, float* loss,
                                   float* dloss_dlogprob, float* dloss_dentropy, double* stats,
                                   int32_t* nonfinite, void* workspace, size_t workspace_bytes,
                                   prl_stream_t stream_) {
  PRL_CHECK_ARG(batch && cfg && loss && stats && nonfinite && workspace, "prl_pg_loss_fwd_bwd: NULL argument");
  PRL_CHECK_ARG(batch->T >= 1, "prl_pg_loss_fwd_bwd: T must be >= 1 (got %lld)", (long long)batch->T);
  PRL_CHECK_ARG(batch->T == 1 || (batch->new_logprobs && batch->labels && batch->rewards && batch->advantages &&
                                  batch->ref_logprobs && batch->old_logprobs && batch->group_tokens &&
                                  batch->num_labels && batch->overflow),
                "prl_pg_loss_fwd_bwd: NULL column pointer");
  PRL_CHECK_ARG(cfg->policy_loss >= PRL_LOSS_PPO && cfg->policy_loss <= PRL_LOSS_GSPO,
                "prl_pg_loss_fwd_bwd: unknown policy_loss %d", cfg->policy_loss);
  const bool gspo = cfg->policy_loss == PRL_LOSS_GSPO;
  const int nseg = gspo ? batch->n_segments : 0;
  if (gspo) {
    PRL_CHECK_ARG(batch->segment_ids != nullptr, "GSPO loss requires packed sequences with segments");
    PRL_CHECK_ARG(batch->n_segments >= 0, "prl_pg_loss_fwd_bwd: n_segments < 0");
  }
  PRL_CHECK_ARG(cfg->group_normalization || cfg->batch_size > 0.f,
                "prl_pg_loss_fwd_bwd: batch_size must be > 0 unless group_normalization");
  PRL_CHECK_ARG(workspace_bytes >= prl_pg_workspace_bytes(nseg), "prl_pg_loss_fwd_bwd: workspace too small");
  cudaStream_t stream = (cudaStream_t)stream_;

  Workspace* ws = (Workspace*)workspace;
  Partial* partials = (Partial*)((char*)workspace + sizeof(Workspace));
  SegSums* seg = (SegSums*)((char*)partials + sizeof(Partial) * (size_t)kMaxBlocks);

  const int64_t n = batch->T - 1;
  int blocks = (int)((n + kThreads - 1) / kThreads);
  if (blocks < 1) blocks = 1;
  const int cap = num_sms() * 8 < kMaxBlocks ? num_sms() * 8 : kMaxBlocks;
  if (blocks > cap) blocks = cap;

  // the ticket must be zero on entry; a memset node is cheaper than trusting the caller
  PRL_CUDA(cudaMemsetAsync(ws, 0, sizeof(Workspace), stream));
  if (gspo && nseg > 0) {
    PRL_CUDA(cudaMemsetAsync(seg, 0, sizeof(SegSums) * (size_t)nseg, stream));
    if (n > 0) {
      gspo_segment_kernel<<<blocks, kThreads, 0, stream>>>(*batch, *cfg, seg);
      PRL_LAUNCH_CHECK();
    }
  }
  pg_loss_kernel<<<blocks, kThreads, 0, stream>>>(*batch, *cfg, loss, dloss_dlogprob, dloss_dentropy, stats,
                                                 nonfinite, ws, partials, seg, nullptr);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}

// ---- GSPO under sequence parallelism (reference rl/utils.py:194-206: the per-segment sums are all-reduced over the group) ----
// Step 1: this rank's per-segment sums of its slice, seg_sums[n_segments][4] = (sum log-ratio, sum advantage, token count,
// sum token weight) as doubles.  The caller all-reduces (SUM) the array over the group and keeps a copy of column 2.
extern "C" int prl_pg_gspo_segment_sums(const prl_pg_batch* batch, const prl_pg_config* cfg, double* seg_sums,
                                        prl_stream_t stream_) {
  PRL_CHECK_ARG(batch && cfg && seg_sums, "prl_pg_gspo_segment_sums: NULL argument");
  PRL_CHECK_ARG(cfg->policy_loss == PRL_LOSS_GSPO && batch->segment_ids != nullptr && batch->n_segments >= 1,
                "prl_pg_gspo_segment_sums: needs the GSPO loss, segment_ids and n_segments >= 1");
  static_assert(sizeof(SegSums) == 4 * sizeof(double), "SegSums is the 4-double row the ABI documents");
  cudaStream_t stream = (cudaStream_t)stream_;
  PRL_CUDA(cudaMemsetAsync(seg_sums, 0, sizeof(SegSums) * (size_t)batch->n_segments, stream));
  const int64_t n = batch->T - 1;
  if (n > 0) {
    int blocks = (int)((n + kThreads - 1) / kThreads);
    const int cap = num_sms() * 8 < kMaxBlocks ? num_sms() * 8 : kMaxBlocks;
    if (blocks > cap) blocks = cap;
    gspo_segment_kernel<<<blocks, kThreads, 0, stream>>>(*batch, *cfg, (SegSums*)seg_sums);
    PRL_LAUNCH_CHECK();
  }
  return PRL_OK;
}

// Step 2: prl_pg_loss_fwd_bwd with the segment sums GIVEN (the group's totals) instead of computed; `seg_local_count`
// (this rank's token counts, [n_segments] doubles) scales each segment's loss term to this rank's share.
extern "C" int prl_pg_loss_fwd_bwd_seg(const prl_pg_batch* batch, const prl_pg_config* cfg, float* loss,
                                       float* dloss_dlogprob, float* dloss_dentropy, double* stats, int32_t* nonfinite,
                                       void* workspace, size_t workspace_bytes, const double* seg_sums,
                                       const double* seg_local_count, prl_stream_t stream_) {
  PRL_CHECK_ARG(batch && cfg && loss && stats && nonfinite && workspace && seg_sums, "prl_pg_loss_fwd_bwd_seg: NULL argument");
  PRL_CHECK_ARG(cfg->policy_loss == PRL_LOSS_GSPO && batch->segment_ids != nullptr && batch->n_segments >= 1,
                "prl_pg_loss_fwd_bwd_seg: needs the GSPO loss, segment_ids and n_segments >= 1");
  PRL_CHECK_ARG(batch->T >= 1, "prl_pg_loss_fwd_bwd_seg: T must be >= 1");
  PRL_CHECK_ARG(cfg->group_normalization || cfg->batch_size > 0.f, "prl_pg_loss_fwd_bwd_seg: batch_size must be > 0 unless group_normalization");
  PRL_CHECK_ARG(workspace_bytes >= prl_pg_workspace_bytes(0), "prl_pg_loss_fwd_bwd_seg: workspace too small");
  cudaStream_t stream = (cudaStream_t)stream_;
  Workspace* ws = (Workspace*)workspace;
  Partial* partials = (Partial*)((char*)workspace + sizeof(Workspace));
  const int64_t n = batch->T - 1;
  int blocks = (int)((n + kThreads - 1) / kThreads);
  if (blocks < 1) blocks = 1;
  const int cap = num_sms() * 8 < kMaxBlocks ? num_sms() * 8 : kMaxBlocks;
  if (blocks > cap) blocks = cap;
  PRL_CUDA(cudaMemsetAsync(ws, 0, sizeof(Workspace), stream));
  pg_loss_kernel<<<blocks, kThreads, 0, stream>>>(*batch, *cfg, loss, dloss_dlogprob, dloss_dentropy, stats, nonfinite, ws,
                                                 partials, (const SegSums*)seg_sums, seg_local_count);
  PRL_LAUNCH_CHECK();
  return PRL_OK;
}
