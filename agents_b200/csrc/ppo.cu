// PPO update math (kernel family iii-c): fused clipped-surrogate / value / entropy losses with
// their gradients, advantage normalisation, streaming normalisers, Normal log-prob / sampling.
//
// Restates, per (b,t) element of a [B,T] batch:
//   policy_gradient_loss        agents/ppo/ppo_agent.py:1329-1512
//   value_estimation_loss       agents/ppo/ppo_agent.py:1203-1327
//   entropy_regularization_loss agents/ppo/ppo_agent.py:1159-1201
//   common.aggregate_losses     utils/common.py:1400-1476  (mean over T, sum over B / global B)
//   _normalize_advantages       agents/ppo/ppo_agent.py:100-110 (tf.nn.moments + batch_norm)
//   compute_return_and_advantage / make_trajectory_mask  ppo_agent.py:617-719, ppo_utils.py:35-59
//   StreamingTensorNormalizer   utils/tensor_normalizer.py:134-205,288-470 (Chan merge + Kahan)
// Everything is HBM-bound element-wise work: one thread per (b,t), reductions in two fixed-order
// stages (deterministic).
#include <math.h>

#include "common.cuh"

namespace b200rl {

constexpr float kLog2Pi = 1.8378770664093453f;
constexpr int kStepLastP = 2;
constexpr int kRedBlocks = 2 * kNumSMs;

struct PpoArgs {
  const float* loc; const float* scale; int64_t ld_ls;      // current policy Normal(loc, scale)
  const float* action;                                       // [N, A]
  const float* old_logp; const float* adv; const float* ret; // [N]
  const float* v; const float* v_old; const float* w;        // [N]
  int64_t N, A, T;
  float global_batch, clip_eps, value_clip, vf_coef, ent_coef, logp_clip;
  float* dloc; float* dscale; int64_t ld_g;                  // gradients, same column layout
  float* dv;                                                 // [N]
  float* partial;                                            // [kRedBlocks, 4]
  // KL penalty (ppo_agent.py:1514-1630): behaviour policy Normal(old_loc, old_scale); the
  // scalar d(kl_penalty)/d(mean_kl) sits in kl_terms[2] (b200rl_ppo_kl_terms)
  const float* old_loc; const float* old_scale; int64_t ld_old;
  const float* kl_terms; float kl_grad_scale;
};

// KL(Normal(mu_a, s_a) || Normal(mu_b, s_b)) per dimension, TFP's closed form
// (tfp.distributions.normal._kl_normal_normal): 0.5*((mu_a - mu_b)/s_b)^2 + 0.5*expm1(2d) - d,
// d = log s_a - log s_b.
__device__ __forceinline__ float kl_normal(float mu_a, float s_a, float mu_b, float s_b) {
  const float d = logf(s_a) - logf(s_b);
  const float z = mu_a / s_b - mu_b / s_b;
  return 0.5f * z * z + 0.5f * expm1f(2.f * d) - d;
}

__global__ void __launch_bounds__(256) ppo_loss_kernel(const PpoArgs a) {
  pdl_prologue();
  __shared__ float red[32];
  float s_pg = 0.f, s_ve = 0.f, s_ent = 0.f, s_clip = 0.f;
  const float denom = (float)a.T * a.global_batch;  // mean over T, then sum over B / global B
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < a.N; n += stride) {
    const float w = a.w[n];
    // log-prob and entropy of the diagonal Normal (summed over action dims, common.py:682-755)
    float logp = 0.f, ent = 0.f;
    for (int64_t k = 0; k < a.A; ++k) {
      const float mu = a.loc[n * a.ld_ls + k], sg = a.scale[n * a.ld_ls + k];
      const float z = (a.action[n * a.A + k] - mu) / sg;
      const float lsg = logf(sg);
      logp += -0.5f * z * z - lsg - 0.5f * kLog2Pi;
      ent += 0.5f + 0.5f * kLog2Pi + lsg;
    }
    float lp = logp, dlp = 1.f;
    if (a.logp_clip > 0.f) {  // ppo_agent.py:1364-1368
      lp = fminf(fmaxf(logp, -a.logp_clip), a.logp_clip);
      dlp = (logp < -a.logp_clip || logp > a.logp_clip) ? 0.f : 1.f;
    }
    const float A_hat = a.adv[n];
    const float ratio = expf(lp - a.old_logp[n]);                              // :1374
    const float lo = 1.f - a.clip_eps, hi = 1.f + a.clip_eps;
    const float ratio_c = fminf(fmaxf(ratio, lo), hi);                         // :1375-1379
    const float obj = ratio * A_hat, obj_c = ratio_c * A_hat;
    float pg, dobj_dratio;
    if (a.clip_eps > 0.f) {
      pg = -fminf(obj, obj_c);                                                 // :1391-1397
      if (obj <= obj_c) dobj_dratio = A_hat;
      else dobj_dratio = (ratio < lo || ratio > hi) ? 0.f : A_hat;
      s_clip += (fabsf(ratio - 1.f) > a.clip_eps) ? 1.f : 0.f;                 // :1407-1417
    } else {
      pg = -obj;
      dobj_dratio = A_hat;
    }
    s_pg += pg * w;
    // value loss
    const float R = a.ret[n], v = a.v[n];
    float err = (R - v) * (R - v);                                             // :1262
    float derr_dv = -2.f * (R - v);
    if (a.value_clip > 0.f) {                                                  // :1264-1279
      const float vo = a.v_old[n];
      const float dvv = v - vo;
      const float vc = vo + fminf(fmaxf(dvv, -a.value_clip), a.value_clip);
      const float err_c = (R - vc) * (R - vc);
      if (err_c > err) {
        err = err_c;
        derr_dv = (dvv < -a.value_clip || dvv > a.value_clip) ? 0.f : -2.f * (R - vc);
      }
    }
    s_ve += err * w;
    s_ent += -ent * w;
    // gradients of total = pg + vf_coef*ve + ent_coef*ent_loss
    const float g_logp = -dobj_dratio * ratio * dlp * w / denom;   // dL_pg / dlogp
    const float g_ent = -a.ent_coef * w / denom;                   // dL_ent / d(entropy)
    // d(kl_penalty)/d(kl_n) = (2 c max(mean_kl - cutoff, 0) + beta) * w_n / N_global
    const float g_kl = a.kl_terms ? a.kl_terms[2] * a.kl_grad_scale * w : 0.f;
    for (int64_t k = 0; k < a.A; ++k) {
      const float mu = a.loc[n * a.ld_ls + k], sg = a.scale[n * a.ld_ls + k];
      const float d = a.action[n * a.A + k] - mu;
      const float inv = 1.f / sg;
      float gl = g_logp * d * inv * inv;
      float gs = g_logp * (d * d * inv * inv * inv - inv) + g_ent * inv;
      if (a.kl_terms) {   // KL(old || new) w.r.t. the new (mu, sigma)
        const float mo = a.old_loc[n * a.ld_old + k], so = a.old_scale[n * a.ld_old + k];
        const float dm = mo - mu;
        gl += g_kl * (-dm * inv * inv);
        gs += g_kl * (inv - (dm * dm + so * so) * inv * inv * inv);
      }
      a.dloc[n * a.ld_g + k] = gl;
      a.dscale[n * a.ld_g + k] = gs;
    }
    a.dv[n] = a.vf_coef * derr_dv * w / denom;
  }
  const float t_pg = block_sum(s_pg, red);
  const float t_ve = block_sum(s_ve, red);
  const float t_ent = block_sum(s_ent, red);
  const float t_clip = block_sum(s_clip, red);
  if (threadIdx.x == 0) {
    float* p = a.partial + (int64_t)blockIdx.x * 4;
    p[0] = t_pg; p[1] = t_ve; p[2] = t_ent; p[3] = t_clip;
  }
}

// losses[0..5] = {policy_gradient, value_estimation, entropy_regularization, clip_fraction,
//                 total (without l2), kl_penalty}
__global__ void __launch_bounds__(512) ppo_loss_final_kernel(const float* __restrict__ partial,
                                                             int nblocks, float denom, float n,
                                                             float vf_coef, float ent_coef,
                                                             const float* __restrict__ kl_terms,
                                                             float* __restrict__ losses,
                                                             int32_t* nan_flag) {
  pdl_prologue();
  __shared__ float red[32];
  float v[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float s = (threadIdx.x < nblocks) ? partial[threadIdx.x * 4 + j] : 0.f;
    v[j] = block_sum(s, red);
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float pg = v[0] / denom, ve = vf_coef * v[1] / denom, en = ent_coef * v[2] / denom;
    losses[0] = pg;
    losses[1] = ve;
    losses[2] = en;
    losses[3] = v[3] / n;
    const float kl = kl_terms ? kl_terms[0] + kl_terms[1] : 0.f;   // kl_penalty_loss (:1628-1630)
    losses[5] = kl;
    losses[4] = pg + ve + en + kl;
    if (nan_flag && !isfinite(losses[4])) *nan_flag = 1;
  }
}

__global__ void normal_logp_kernel(const float* __restrict__ loc, const float* __restrict__ scale,
                                   int64_t ld, const float* __restrict__ action, int64_t N,
                                   int64_t A, float* __restrict__ out) {
  pdl_prologue();
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float logp = 0.f;
  for (int64_t k = 0; k < A; ++k) {
    const float sg = scale[n * ld + k];
    const float z = (action[n * A + k] - loc[n * ld + k]) / sg;
    logp += -0.5f * z * z - logf(sg) - 0.5f * kLog2Pi;
  }
  out[n] = logp;
}

// action = clip(loc + scale * z), z = philox_normal of element n*A+k;
// rng_call: uint64[2] {call, ticket}.
__global__ void normal_sample_kernel(const float* __restrict__ loc,
                                     const float* __restrict__ scale, int64_t ld, int64_t N,
                                     int64_t A, const float* __restrict__ amin,
                                     const float* __restrict__ amax, uint64_t seed,
                                     uint64_t* rng_call, float* __restrict__ out) {
  pdl_prologue();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N * A) {
    const int64_t n = i / A, k = i - n * A;
    const float z = philox_normal((uint64_t)i, rng_call[0], seed);
    float v = loc[n * ld + k] + scale[n * ld + k] * z;
    if (amin) v = fminf(fmaxf(v, amin[k]), amax[k]);
    out[i] = v;
  }
  next_rng_call(rng_call);
}

// NormalProjectionNetwork head (networks/normal_projection_network.py): loc = tanh-squash of
// the mean layer to the action spec, scale = softplus(bias) broadcast over the batch.
__global__ void normal_proj_fwd_kernel(const float* __restrict__ m_raw,
                                       const float* __restrict__ s_raw,
                                       const float* __restrict__ amin,
                                       const float* __restrict__ amax, int64_t N, int64_t A,
                                       float* __restrict__ loc, float* __restrict__ scale) {
  pdl_prologue();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * A) return;
  const int64_t k = i % A;
  const float mean_scale = 0.5f * (amax[k] - amin[k]), mean_shift = 0.5f * (amax[k] + amin[k]);
  loc[i] = mean_shift + mean_scale * tanhf(m_raw[i]);
  const float s = s_raw[k];
  scale[i] = s > 20.f ? s : log1pf(expf(s));  // tf.nn.softplus
}
// dm_raw = dloc * mean_scale * (1 - tanh^2); ds_part = dscale * sigmoid(s_raw) (column-summed by
// the caller with b200rl_colsum).
__global__ void normal_proj_bwd_kernel(const float* __restrict__ m_raw,
                                       const float* __restrict__ s_raw,
                                       const float* __restrict__ amin,
                                       const float* __restrict__ amax,
                                       const float* __restrict__ dloc,
                                       const float* __restrict__ dscale, int64_t N, int64_t A,
                                       float* __restrict__ dm_raw, float* __restrict__ ds_part) {
  pdl_prologue();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * A) return;
  const int64_t k = i % A;
  const float mean_scale = 0.5f * (amax[k] - amin[k]);
  const float t = tanhf(m_raw[i]);
  dm_raw[i] = dloc[i] * mean_scale * (1.f - t * t);
  ds_part[i] = dscale[i] / (1.f + expf(-s_raw[k]));
}

// ---- column moments: mean then sum of squared differences (tf.nn.moments / normalizer) --------
__global__ void __launch_bounds__(256) colsum_rows_kernel(const float* __restrict__ x,
                                                          const float* __restrict__ center,
                                                          int squared, int64_t rows, int64_t cols,
                                                          float* __restrict__ part) {
  pdl_prologue();
  // grid = (cols, nblk): block (c, j) sums rows j, j+nblk, ... of column c
  __shared__ float red[32];
  const int64_t c = blockIdx.x;
  const float ctr = center ? center[c] : 0.f;
  float s = 0.f;
  for (int64_t r = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; r < rows;
       r += (int64_t)gridDim.y * blockDim.x) {
    const float v = x[r * cols + c] - ctr;
    s += squared ? v * v : v;
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) part[c * gridDim.y + blockIdx.y] = s;
}
__global__ void colsum_rows_final_kernel(const float* __restrict__ part, int nblk, int64_t cols,
                                         float scale, float* __restrict__ out) {
  pdl_prologue();
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  float s = 0.f;
  for (int j = 0; j < nblk; ++j) s += part[c * nblk + j];
  out[c] = s * scale;
}

// out = x*inv + (-mean*inv), inv = rsqrt(var + eps)  (tf.nn.batch_normalization), optional clip.
// var = m2[c] / count[c] when count != NULL else m2[c] is the variance itself.
__global__ void normalize_kernel(const float* __restrict__ x, float* __restrict__ out,
                                 int64_t rows, int64_t cols, const float* __restrict__ mean,
                                 const float* __restrict__ m2, const float* __restrict__ count,
                                 float eps, float clip) {
  pdl_prologue();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int64_t c = i % cols;
  const float var = count ? m2[c] / count[c] : m2[c];
  const float inv = rsqrtf(var + eps);
  const float mu = mean ? mean[c] : 0.f;
  float v = __fadd_rn(__fmul_rn(x[i], inv), __fmul_rn(-mu, inv));
  if (clip > 0.f) v = fminf(fmaxf(v, -clip), clip);
  out[i] = v;
}

// parallel_variance_calculation + kahan_summation (utils/tensor_normalizer.py:397-470)
__global__ void normalizer_update_kernel(float* __restrict__ count, float* __restrict__ avg,
                                         float* __restrict__ m2, float* __restrict__ carry,
                                         const float* __restrict__ avg_a,
                                         const float* __restrict__ m2_a, float n_a, int64_t cols) {
  pdl_prologue();
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  const float n_b = count[c], avg_b = avg[c], m2_b = m2[c], m2_b_c = carry[c];
  const float n_ab = n_a + n_b;
  const float delta = avg_b - avg_a[c];
  const float s_delta = delta * n_b / n_ab;
  const float avg_ab = avg_a[c] + s_delta;
  const float value = m2_a[c] + (delta * n_a * s_delta);
  const float y = value - m2_b_c;
  const float t = m2_b + y;
  carry[c] = (t - m2_b) - y;
  m2[c] = t;
  count[c] = n_ab;
  avg[c] = avg_ab;
}

// disc_eff = gamma * discount * (next_step_type != LAST)   (ppo_agent.py:632-660)
__global__ void ppo_discounts_kernel(const float* __restrict__ discount,
                                     const int32_t* __restrict__ next_step_type, float gamma,
                                     int64_t n, float* __restrict__ out) {
  pdl_prologue();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float mask = next_step_type[i] == kStepLastP ? 0.f : 1.f;
  out[i] = __fmul_rn(__fmul_rn(discount[i], gamma), mask);
}

// weights = [weights *] (step_type != LAST) & !(return == 0 & advantage == 0)
__global__ void ppo_weights_kernel(const int32_t* __restrict__ step_type,
                                   const float* __restrict__ ret, const float* __restrict__ adv,
                                   const float* __restrict__ weights, int64_t n,
                                   float* __restrict__ out) {
  pdl_prologue();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool valid = step_type[i] != kStepLastP && !(ret[i] == 0.f && adv[i] == 0.f);
  out[i] = valid ? (weights ? weights[i] : 1.f) : 0.f;
}


// sum_n w_n * KL(old_n || new_n) in two fixed-order stages (kl_penalty_loss :1613-1617); the
// weighted per-element values are optionally kept (update_adaptive_kl_beta, debug).
__global__ void __launch_bounds__(256) ppo_kl_partial_kernel(
    const float* __restrict__ loc, const float* __restrict__ scale, int64_t ld,
    const float* __restrict__ old_loc, const float* __restrict__ old_scale, int64_t ld_old,
    const float* __restrict__ w, int64_t N, int64_t A, float* __restrict__ out_kl,
    float* __restrict__ partial) {
  pdl_prologue();
  __shared__ float red[32];
  float s = 0.f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < N; n += stride) {
    float kl = 0.f;
    for (int64_t k = 0; k < A; ++k)
      kl += kl_normal(old_loc[n * ld_old + k], old_scale[n * ld_old + k], loc[n * ld + k],
                      scale[n * ld + k]);
    kl *= w ? w[n] : 1.f;
    if (out_kl) out_kl[n] = kl;
    s += kl;
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}
__global__ void __launch_bounds__(512) ppo_kl_final_kernel(const float* __restrict__ partial,
                                                           int nblocks, float scale,
                                                           float* __restrict__ out) {
  pdl_prologue();
  __shared__ float red[32];
  float s = (threadIdx.x < nblocks) ? partial[threadIdx.x] : 0.f;
  s = block_sum(s, red);
  if (threadIdx.x == 0) *out = s * scale;
}

// terms[3] = {kl_cutoff_loss (:1514-1539), adaptive_kl_loss (:1541-1558),
//             d(kl_cutoff_loss + adaptive_kl_loss)/d(mean_kl)}
__global__ void ppo_kl_terms_kernel(const float* __restrict__ mean_kl,
                                    const float* __restrict__ beta, float cutoff,
                                    float cutoff_coef, int use_cutoff,
                                    float* __restrict__ terms) {
  pdl_prologue();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const float m = *mean_kl;
  float cut = 0.f, dcut = 0.f;
  if (use_cutoff) {
    const float over = fmaxf(m - cutoff, 0.f);
    cut = cutoff_coef * over * over;
    dcut = 2.f * cutoff_coef * over;
  }
  const float b = beta ? *beta : 0.f;
  terms[0] = cut;
  terms[1] = b * m;
  terms[2] = dcut + b;
}

// update_adaptive_kl_beta (:1632-1675): x1.5 above target*(1+tol), /1.5 below target*(1-tol),
// clipped to [10e-16, 10e16].
__global__ void ppo_kl_beta_update_kernel(const float* __restrict__ mean_kl,
                                          float* __restrict__ beta, float target, float tol) {
  pdl_prologue();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const float m = *mean_kl;
  float f = 1.f;
  if (m < target * (1.f - tol)) f = 1.f / 1.5f;
  else if (m > target * (1.f + tol)) f = 1.5f;
  *beta = fminf(fmaxf(*beta * f, 10e-16f), 10e16f);
}

// ---- Categorical policy (discrete actions): CategoricalProjectionNetwork logits [N, A] --------
// A row of logits is handled by a group of G lanes (B200RL_GROUP_ROWS, common.cuh); G follows
// from A (lane_group): one thread per row for narrow rows, 8 or 32 lanes with shuffle reductions
// for wide ones, so a row is read with coalesced loads.  row_softmax_stats / clamp_action live in
// common.cuh (shared with reinforce.cu).

struct PpoCatArgs {
  const float* logits; int64_t ld;                           // current policy Categorical(logits)
  const int32_t* action;                                     // [N]
  const float* old_logp; const float* adv; const float* ret; // [N]
  const float* v; const float* v_old; const float* w;        // [N]
  int64_t N, A, T;
  float global_batch, clip_eps, value_clip, vf_coef, ent_coef, logp_clip;
  float* dlogits; int64_t ld_g;
  float* dv;
  float* partial;                                            // [kCatRedBlocks, 4]
  int32_t* nan_flag;
  // KL penalty: behaviour policy Categorical(old_logits); d(kl_penalty)/d(mean_kl) in kl_terms[2]
  const float* old_logits; int64_t ld_old;
  const float* kl_terms; float kl_grad_scale;
};

// The categorical twin of ppo_loss_kernel: same surrogate / value / entropy terms and the same
// 4-partial layout for ppo_loss_final_kernel.  dL/dz_j = g_logp (1[j=a] - p_j)
// + g_ent (-p_j (log p_j + H)) + g_kl (p_j - q_j), q = softmax(old_logits).
template <int G>
__global__ void __launch_bounds__(256) ppo_loss_cat_kernel(const PpoCatArgs a) {
  pdl_prologue();
  __shared__ float red[32];
  float s_pg = 0.f, s_ve = 0.f, s_ent = 0.f, s_clip = 0.f;
  const float denom = (float)a.T * a.global_batch;
  B200RL_GROUP_ROWS(G, a.N) {
    const bool valid = n < a.N;
    const int64_t r = valid ? n : n0;
    const float* z = a.logits + r * a.ld;
    const int act = clamp_action(a.action[r], a.A, valid ? a.nan_flag : nullptr);
    float m, s, t;
    row_softmax_stats<G>(z, a.A, lane, m, s, t);
    const float log_s = logf(s);
    const float ent = log_s - t / s;
    const float logp = (z[act] - m) - log_s;
    float lp = logp, dlp = 1.f;
    if (a.logp_clip > 0.f) {
      lp = fminf(fmaxf(logp, -a.logp_clip), a.logp_clip);
      dlp = (logp < -a.logp_clip || logp > a.logp_clip) ? 0.f : 1.f;
    }
    const float w = a.w[r];
    const float A_hat = a.adv[r];
    const float ratio = expf(lp - a.old_logp[r]);
    const float lo = 1.f - a.clip_eps, hi = 1.f + a.clip_eps;
    const float ratio_c = fminf(fmaxf(ratio, lo), hi);
    const float obj = ratio * A_hat, obj_c = ratio_c * A_hat;
    float pg, dobj_dratio, clipped = 0.f;
    if (a.clip_eps > 0.f) {
      pg = -fminf(obj, obj_c);
      if (obj <= obj_c) dobj_dratio = A_hat;
      else dobj_dratio = (ratio < lo || ratio > hi) ? 0.f : A_hat;
      clipped = (fabsf(ratio - 1.f) > a.clip_eps) ? 1.f : 0.f;
    } else {
      pg = -obj;
      dobj_dratio = A_hat;
    }
    const float R = a.ret[r], v = a.v[r];
    float err = (R - v) * (R - v);
    float derr_dv = -2.f * (R - v);
    if (a.value_clip > 0.f) {
      const float vo = a.v_old[r];
      const float dvv = v - vo;
      const float vc = vo + fminf(fmaxf(dvv, -a.value_clip), a.value_clip);
      const float err_c = (R - vc) * (R - vc);
      if (err_c > err) {
        err = err_c;
        derr_dv = (dvv < -a.value_clip || dvv > a.value_clip) ? 0.f : -2.f * (R - vc);
      }
    }
    if (valid && lane == 0) {
      s_pg += pg * w;
      s_ve += err * w;
      s_ent += -ent * w;
      s_clip += clipped;
      a.dv[r] = a.vf_coef * derr_dv * w / denom;
    }
    const float g_logp = -dobj_dratio * ratio * dlp * w / denom;
    const float g_ent = -a.ent_coef * w / denom;
    float g_kl = 0.f, mo = 0.f, lso = 0.f;
    const float* zo = nullptr;
    if (a.kl_terms) {
      g_kl = a.kl_terms[2] * a.kl_grad_scale * w;
      zo = a.old_logits + r * a.ld_old;
      float so, to;
      row_softmax_stats<G>(zo, a.A, lane, mo, so, to);
      lso = logf(so);
    }
    if (valid) {
      for (int64_t j = lane; j < a.A; j += G) {
        const float lpj = (z[j] - m) - log_s;
        const float p = expf(lpj);
        float g = g_logp * ((j == act ? 1.f : 0.f) - p) + g_ent * (-p * (lpj + ent));
        if (zo) g += g_kl * (p - expf((zo[j] - mo) - lso));
        a.dlogits[r * a.ld_g + j] = g;
      }
    }
  }
  const float t_pg = block_sum(s_pg, red);
  const float t_ve = block_sum(s_ve, red);
  const float t_ent = block_sum(s_ent, red);
  const float t_clip = block_sum(s_clip, red);
  if (threadIdx.x == 0) {
    float* p = a.partial + (int64_t)blockIdx.x * 4;
    p[0] = t_pg; p[1] = t_ve; p[2] = t_ent; p[3] = t_clip;
  }
}

template <int G>
__global__ void __launch_bounds__(256) categorical_logp_kernel(const float* __restrict__ logits,
                                                               int64_t ld,
                                                               const int32_t* __restrict__ action,
                                                               int64_t N, int64_t A,
                                                               float* __restrict__ out,
                                                               int32_t* nan_flag) {
  pdl_prologue();
  B200RL_GROUP_ROWS(G, N) {
    const bool valid = n < N;
    const int64_t r = valid ? n : n0;
    const float* z = logits + r * ld;
    const int act = clamp_action(action[r], A, valid ? nan_flag : nullptr);
    float m, s, t;
    row_softmax_stats<G>(z, A, lane, m, s, t);
    if (valid && lane == 0) out[r] = (z[act] - m) - logf(s);
  }
}

// sum_n w_n * KL(Categorical(old)_n || Categorical(new)_n), KL = sum_j q_j (log q_j - log p_j)
// (tfp _kl_categorical_categorical), two fixed-order stages like ppo_kl_partial_kernel.
template <int G>
__global__ void __launch_bounds__(256) ppo_kl_cat_partial_kernel(
    const float* __restrict__ logits, int64_t ld, const float* __restrict__ old_logits,
    int64_t ld_old, const float* __restrict__ w, int64_t N, int64_t A, float* __restrict__ out_kl,
    float* __restrict__ partial) {
  pdl_prologue();
  __shared__ float red[32];
  float acc = 0.f;
  B200RL_GROUP_ROWS(G, N) {
    const bool valid = n < N;
    const int64_t r = valid ? n : n0;
    const float* z = logits + r * ld;
    const float* zo = old_logits + r * ld_old;
    float m, s, t, mo, so, to;
    row_softmax_stats<G>(z, A, lane, m, s, t);
    row_softmax_stats<G>(zo, A, lane, mo, so, to);
    const float ls = logf(s), lso = logf(so);
    float kl = 0.f;
    for (int64_t j = lane; j < A; j += G) {
      const float lq = (zo[j] - mo) - lso;
      const float q = expf(lq);
      kl += q > 0.f ? q * (lq - ((z[j] - m) - ls)) : 0.f;
    }
    kl = grp_sum<G>(kl);
    kl *= w ? w[r] : 1.f;
    if (valid && lane == 0) {
      if (out_kl) out_kl[r] = kl;
      acc += kl;
    }
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = acc;
}

// Collect-policy draw, one thread per row: u = uniform_f32(philox(counter=(n, call), key=seed).x);
// action = smallest k with u < cdf_k, cdf the fp32 running sum in index order of
// exp(z - max) / sum exp(z - max); A-1 if there is none.  rng_call: uint64[2] {call, ticket}.
__global__ void categorical_sample_kernel(const float* __restrict__ logits, int64_t ld, int64_t N,
                                          int64_t A, uint64_t seed, uint64_t* rng_call,
                                          int32_t* __restrict__ out) {
  pdl_prologue();
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n < N) {
    const float* z = logits + n * ld;
    float m = z[0];
    for (int64_t k = 1; k < A; ++k) m = fmaxf(m, z[k]);
    float s = 0.f;
    for (int64_t k = 0; k < A; ++k) s += expf(z[k] - m);
    const float u = uniform_f32(philox4x32_10((uint64_t)n, rng_call[0], seed).x);
    int32_t pick = (int32_t)(A - 1);
    float cdf = 0.f;
    for (int64_t k = 0; k < A; ++k) {
      cdf += expf(z[k] - m) / s;
      if (u < cdf) { pick = (int32_t)k; break; }
    }
    out[n] = pick;
  }
  next_rng_call(rng_call);
}

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_ppo_loss(const float* loc, const float* scale, int64_t ld_ls, const float* action,
                    const float* old_logp, const float* adv, const float* ret, const float* v,
                    const float* v_old, const float* w, int64_t N, int64_t A, int64_t T,
                    float global_batch, float clip_eps, float value_clip, float vf_coef,
                    float ent_coef, float logp_clip, float* losses, float* dloc, float* dscale,
                    int64_t ld_g, float* dv, int32_t* nan_flag, const b200rl_ppo_kl_t* kl,
                    void* workspace, int64_t ws_bytes, void* stream) {
  B200RL_CHECK_ARG(loc && scale && action && old_logp && adv && ret && v && w && losses && dloc &&
                       dscale && dv,
                   "ppo_loss: NULL argument");
  B200RL_CHECK_ARG(N >= 1 && A >= 1 && T >= 1 && global_batch > 0.f, "ppo_loss: bad sizes");
  B200RL_CHECK_ARG(value_clip <= 0.f || v_old, "old_value_predictions is None but needed for value clipping.");
  B200RL_CHECK_ARG(workspace && ws_bytes >= (int64_t)(kRedBlocks * 4 * sizeof(float)),
                   "ppo_loss: workspace too small");
  B200RL_CHECK_ARG(ld_ls >= A && ld_g >= A, "ppo_loss: leading dimension < A");
  cudaStream_t st = (cudaStream_t)stream;
  PpoArgs a{loc, scale, ld_ls, action, old_logp, adv, ret, v, v_old, w, N, A, T, global_batch,
            clip_eps, value_clip, vf_coef, ent_coef, logp_clip, dloc, dscale, ld_g, dv,
            (float*)workspace, nullptr, nullptr, 0, nullptr, 0.f};
  if (kl != nullptr) {
    B200RL_CHECK_ARG(kl->old_loc && kl->old_scale && kl->terms && kl->ld_old >= A,
                     "ppo_loss: incomplete KL-penalty arguments");
    a.old_loc = kl->old_loc; a.old_scale = kl->old_scale; a.ld_old = kl->ld_old;
    a.kl_terms = kl->terms; a.kl_grad_scale = kl->grad_scale;
  }
  int nb = (int)((N + 255) / 256);
  if (nb > kRedBlocks) nb = kRedBlocks;
  B200RL_LAUNCH(ppo_loss_kernel, nb, 256, 0, st, a);
  B200RL_CHECK_LAUNCH("ppo_loss");
  B200RL_LAUNCH(ppo_loss_final_kernel, 1, 512, 0, st, (const float*)workspace, nb, (float)T * global_batch, (float)N, vf_coef, ent_coef, a.kl_terms, losses, nan_flag);
  B200RL_CHECK_LAUNCH("ppo_loss_final");
  return B200RL_OK;
}

int b200rl_ppo_kl(const float* loc, const float* scale, int64_t ld, const float* old_loc,
                  const float* old_scale, int64_t ld_old, const float* w, int64_t N, int64_t A,
                  float out_scale, float* out_kl, float* out_sum, void* workspace,
                  int64_t ws_bytes, void* stream) {
  B200RL_CHECK_ARG(loc && scale && old_loc && old_scale && out_sum, "ppo_kl: NULL argument");
  B200RL_CHECK_ARG(N >= 1 && A >= 1 && ld >= A && ld_old >= A, "ppo_kl: bad sizes");
  B200RL_CHECK_ARG(workspace && ws_bytes >= (int64_t)(kRedBlocks * sizeof(float)),
                   "ppo_kl: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  int nb = (int)((N + 255) / 256);
  if (nb > kRedBlocks) nb = kRedBlocks;
  B200RL_LAUNCH(ppo_kl_partial_kernel, nb, 256, 0, st, loc, scale, ld, old_loc, old_scale, ld_old, w, N, A, out_kl, (float*)workspace);
  B200RL_CHECK_LAUNCH("ppo_kl_partial");
  B200RL_LAUNCH(ppo_kl_final_kernel, 1, 512, 0, st, (const float*)workspace, nb, out_scale, out_sum);
  B200RL_CHECK_LAUNCH("ppo_kl_final");
  return B200RL_OK;
}

int b200rl_ppo_kl_terms(const float* mean_kl_dev, const float* beta_dev, float kl_cutoff_factor,
                        float adaptive_kl_target, float kl_cutoff_coef, float* terms_dev,
                        void* stream) {
  B200RL_CHECK_ARG(mean_kl_dev && terms_dev, "ppo_kl_terms: NULL argument");
  B200RL_LAUNCH(ppo_kl_terms_kernel, 1, 32, 0, (cudaStream_t)stream, mean_kl_dev, beta_dev, kl_cutoff_factor * adaptive_kl_target, kl_cutoff_coef, kl_cutoff_factor > 0.f ? 1 : 0, terms_dev);
  B200RL_CHECK_LAUNCH("ppo_kl_terms");
  return B200RL_OK;
}

int b200rl_ppo_kl_beta_update(const float* mean_kl_dev, float* beta_dev, float adaptive_kl_target,
                              float adaptive_kl_tolerance, void* stream) {
  B200RL_CHECK_ARG(mean_kl_dev && beta_dev, "ppo_kl_beta_update: NULL argument");
  B200RL_LAUNCH(ppo_kl_beta_update_kernel, 1, 32, 0, (cudaStream_t)stream, mean_kl_dev, beta_dev, adaptive_kl_target, adaptive_kl_tolerance);
  B200RL_CHECK_LAUNCH("ppo_kl_beta_update");
  return B200RL_OK;
}

int b200rl_normal_logp(const float* loc, const float* scale, int64_t ld, const float* action,
                       int64_t N, int64_t A, float* out, void* stream) {
  B200RL_CHECK_ARG(loc && scale && action && out && N >= 0 && A >= 1 && ld >= A,
                   "normal_logp: bad argument");
  if (N == 0) return B200RL_OK;
  B200RL_LAUNCH(normal_logp_kernel, blocks_of_256(N), 256, 0, (cudaStream_t)stream, loc, scale, ld, action, N, A, out);
  B200RL_CHECK_LAUNCH("normal_logp");
  return B200RL_OK;
}

int b200rl_normal_sample(const float* loc, const float* scale, int64_t ld, int64_t N, int64_t A,
                         const float* amin, const float* amax, uint64_t seed,
                         uint64_t* rng_call_dev, float* out, void* stream) {
  B200RL_CHECK_ARG(loc && scale && out && rng_call_dev && N >= 1 && A >= 1 && ld >= A,
                   "normal_sample: bad argument");
  B200RL_CHECK_ARG((amin == nullptr) == (amax == nullptr), "normal_sample: amin/amax mismatch");
  B200RL_LAUNCH(normal_sample_kernel, blocks_of_256(N * A), 256, 0, (cudaStream_t)stream, loc, scale, ld, N, A, amin, amax, seed, rng_call_dev, out);
  B200RL_CHECK_LAUNCH("normal_sample");
  return B200RL_OK;
}

}  // extern "C"

// The categorical kernels fill the GPU up to the 512 partials one 512-thread final kernel reduces
// (about 4 CTAs of 256 per SM; the continuous kernels keep kRedBlocks).
constexpr int kCatRedBlocks = 512;

extern "C" {

int b200rl_ppo_loss_categorical(const float* logits, int64_t ld, const int32_t* action,
                                const float* old_logp, const float* adv, const float* ret,
                                const float* v, const float* v_old, const float* w, int64_t N,
                                int64_t A, int64_t T, float global_batch, float clip_eps,
                                float value_clip, float vf_coef, float ent_coef, float logp_clip,
                                float* losses, float* dlogits, int64_t ld_g, float* dv,
                                int32_t* nan_flag, const b200rl_ppo_kl_logits_t* kl,
                                void* workspace, int64_t ws_bytes, void* stream) {
  B200RL_CHECK_ARG(logits && action && old_logp && adv && ret && v && w && losses && dlogits && dv,
                   "ppo_loss_categorical: NULL argument");
  B200RL_CHECK_ARG(N >= 1 && A >= 1 && T >= 1 && global_batch > 0.f,
                   "ppo_loss_categorical: bad sizes");
  B200RL_CHECK_ARG(value_clip <= 0.f || v_old, "old_value_predictions is None but needed for value clipping.");
  B200RL_CHECK_ARG(workspace && ws_bytes >= (int64_t)(kCatRedBlocks * 4 * sizeof(float)),
                   "ppo_loss_categorical: workspace too small");
  B200RL_CHECK_ARG(ld >= A && ld_g >= A, "ppo_loss_categorical: leading dimension < A");
  cudaStream_t st = (cudaStream_t)stream;
  PpoCatArgs a{logits, ld, action, old_logp, adv, ret, v, v_old, w, N, A, T, global_batch,
               clip_eps, value_clip, vf_coef, ent_coef, logp_clip, dlogits, ld_g, dv,
               (float*)workspace, nan_flag, nullptr, 0, nullptr, 0.f};
  if (kl != nullptr) {
    B200RL_CHECK_ARG(kl->old_logits && kl->terms && kl->ld_old >= A,
                     "ppo_loss_categorical: incomplete KL-penalty arguments");
    a.old_logits = kl->old_logits; a.ld_old = kl->ld_old;
    a.kl_terms = kl->terms; a.kl_grad_scale = kl->grad_scale;
  }
  const int G = lane_group(A);
  const unsigned nb = group_blocks(N, G, kCatRedBlocks);
  if (G == 1) B200RL_LAUNCH(ppo_loss_cat_kernel<1>, nb, 256, 0, st, a);
  else if (G == 8) B200RL_LAUNCH(ppo_loss_cat_kernel<8>, nb, 256, 0, st, a);
  else B200RL_LAUNCH(ppo_loss_cat_kernel<32>, nb, 256, 0, st, a);
  B200RL_CHECK_LAUNCH("ppo_loss_categorical");
  B200RL_LAUNCH(ppo_loss_final_kernel, 1, 512, 0, st, (const float*)workspace, (int)nb, (float)T * global_batch, (float)N, vf_coef, ent_coef, a.kl_terms, losses, nan_flag);
  B200RL_CHECK_LAUNCH("ppo_loss_final");
  return B200RL_OK;
}

int b200rl_categorical_logp(const float* logits, int64_t ld, const int32_t* action, int64_t N,
                            int64_t A, float* out, int32_t* nan_flag, void* stream) {
  B200RL_CHECK_ARG(logits && action && out && N >= 0 && A >= 1 && ld >= A,
                   "categorical_logp: bad argument");
  if (N == 0) return B200RL_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int G = lane_group(A);
  const unsigned nb = group_blocks(N, G, 1 << 30);
  if (G == 1) B200RL_LAUNCH(categorical_logp_kernel<1>, nb, 256, 0, st, logits, ld, action, N, A, out, nan_flag);
  else if (G == 8) B200RL_LAUNCH(categorical_logp_kernel<8>, nb, 256, 0, st, logits, ld, action, N, A, out, nan_flag);
  else B200RL_LAUNCH(categorical_logp_kernel<32>, nb, 256, 0, st, logits, ld, action, N, A, out, nan_flag);
  B200RL_CHECK_LAUNCH("categorical_logp");
  return B200RL_OK;
}

int b200rl_ppo_kl_categorical(const float* logits, int64_t ld, const float* old_logits,
                              int64_t ld_old, const float* w, int64_t N, int64_t A,
                              float out_scale, float* out_kl, float* out_sum, void* workspace,
                              int64_t ws_bytes, void* stream) {
  B200RL_CHECK_ARG(logits && old_logits && out_sum, "ppo_kl_categorical: NULL argument");
  B200RL_CHECK_ARG(N >= 1 && A >= 1 && ld >= A && ld_old >= A, "ppo_kl_categorical: bad sizes");
  B200RL_CHECK_ARG(workspace && ws_bytes >= (int64_t)(kCatRedBlocks * sizeof(float)),
                   "ppo_kl_categorical: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int G = lane_group(A);
  const unsigned nb = group_blocks(N, G, kCatRedBlocks);
  float* part = (float*)workspace;
  if (G == 1) B200RL_LAUNCH(ppo_kl_cat_partial_kernel<1>, nb, 256, 0, st, logits, ld, old_logits, ld_old, w, N, A, out_kl, part);
  else if (G == 8) B200RL_LAUNCH(ppo_kl_cat_partial_kernel<8>, nb, 256, 0, st, logits, ld, old_logits, ld_old, w, N, A, out_kl, part);
  else B200RL_LAUNCH(ppo_kl_cat_partial_kernel<32>, nb, 256, 0, st, logits, ld, old_logits, ld_old, w, N, A, out_kl, part);
  B200RL_CHECK_LAUNCH("ppo_kl_categorical_partial");
  B200RL_LAUNCH(ppo_kl_final_kernel, 1, 512, 0, st, (const float*)workspace, (int)nb, out_scale, out_sum);
  B200RL_CHECK_LAUNCH("ppo_kl_final");
  return B200RL_OK;
}

int b200rl_categorical_sample(const float* logits, int64_t ld, int64_t N, int64_t A,
                              uint64_t seed, uint64_t* rng_call_dev, int32_t* out, void* stream) {
  B200RL_CHECK_ARG(logits && out && rng_call_dev && N >= 1 && A >= 1 && ld >= A,
                   "categorical_sample: bad argument");
  B200RL_LAUNCH(categorical_sample_kernel, blocks_of_256(N), 256, 0, (cudaStream_t)stream, logits, ld, N, A, seed, rng_call_dev, out);
  B200RL_CHECK_LAUNCH("categorical_sample");
  return B200RL_OK;
}

int b200rl_normal_proj_fwd(const float* m_raw, const float* s_raw, const float* amin,
                           const float* amax, int64_t N, int64_t A, float* loc, float* scale,
                           void* stream) {
  B200RL_CHECK_ARG(m_raw && s_raw && amin && amax && loc && scale && N >= 1 && A >= 1,
                   "normal_proj_fwd: bad argument");
  B200RL_LAUNCH(normal_proj_fwd_kernel, blocks_of_256(N * A), 256, 0, (cudaStream_t)stream, m_raw, s_raw, amin, amax, N, A, loc, scale);
  B200RL_CHECK_LAUNCH("normal_proj_fwd");
  return B200RL_OK;
}

int b200rl_normal_proj_bwd(const float* m_raw, const float* s_raw, const float* amin,
                           const float* amax, const float* dloc, const float* dscale, int64_t N,
                           int64_t A, float* dm_raw, float* ds_part, void* stream) {
  B200RL_CHECK_ARG(m_raw && s_raw && amin && amax && dloc && dscale && dm_raw && ds_part &&
                       N >= 1 && A >= 1,
                   "normal_proj_bwd: bad argument");
  B200RL_LAUNCH(normal_proj_bwd_kernel, blocks_of_256(N * A), 256, 0, (cudaStream_t)stream, m_raw, s_raw, amin, amax, dloc, dscale, N, A, dm_raw, ds_part);
  B200RL_CHECK_LAUNCH("normal_proj_bwd");
  return B200RL_OK;
}

/* Column sums of x[rows, cols] (optionally of (x - center)^2), scaled: out[c] = scale * sum. */
int b200rl_colsum(const float* x, const float* center, int squared, int64_t rows, int64_t cols,
                  float scale, float* out, void* workspace, int64_t ws_bytes, void* stream) {
  B200RL_CHECK_ARG(x && out && rows >= 1 && cols >= 1, "colsum: bad argument");
  int nblk = (int)((rows + 255) / 256);
  const int cap = cols >= 64 ? 8 : 128;
  if (nblk > cap) nblk = cap;
  B200RL_CHECK_ARG(cols <= 65535 * 1ll, "colsum: too many columns");
  B200RL_CHECK_ARG(workspace && ws_bytes >= (int64_t)(cols * nblk * sizeof(float)),
                   "colsum: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid((unsigned)cols, (unsigned)nblk);
  B200RL_LAUNCH(colsum_rows_kernel, grid, 256, 0, st, x, center, squared, rows, cols, (float*)workspace);
  B200RL_CHECK_LAUNCH("colsum_rows");
  B200RL_LAUNCH(colsum_rows_final_kernel, blocks_of_256(cols), 256, 0, st, (const float*)workspace, nblk, cols, scale, out);
  B200RL_CHECK_LAUNCH("colsum_rows_final");
  return B200RL_OK;
}

int b200rl_normalize(const float* x, float* out, int64_t rows, int64_t cols, const float* mean,
                     const float* m2, const float* count, float eps, float clip, void* stream) {
  B200RL_CHECK_ARG(x && out && m2 && rows >= 1 && cols >= 1, "normalize: bad argument");
  B200RL_LAUNCH(normalize_kernel, blocks_of_256(rows * cols), 256, 0, (cudaStream_t)stream, x, out, rows, cols, mean, m2, count, eps, clip);
  B200RL_CHECK_LAUNCH("normalize");
  return B200RL_OK;
}

int b200rl_normalizer_update(float* count, float* avg, float* m2, float* carry,
                             const float* avg_a, const float* m2_a, float n_a, int64_t cols,
                             void* stream) {
  B200RL_CHECK_ARG(count && avg && m2 && carry && avg_a && m2_a && cols >= 1,
                   "normalizer_update: bad argument");
  B200RL_LAUNCH(normalizer_update_kernel, blocks_of_256(cols), 256, 0, (cudaStream_t)stream, count, avg, m2, carry, avg_a, m2_a, n_a, cols);
  B200RL_CHECK_LAUNCH("normalizer_update");
  return B200RL_OK;
}

int b200rl_ppo_discounts(const float* discount, const int32_t* next_step_type, float gamma,
                         int64_t n, float* out, void* stream) {
  B200RL_CHECK_ARG(discount && next_step_type && out && n >= 1, "ppo_discounts: bad argument");
  B200RL_LAUNCH(ppo_discounts_kernel, blocks_of_256(n), 256, 0, (cudaStream_t)stream, discount, next_step_type, gamma, n, out);
  B200RL_CHECK_LAUNCH("ppo_discounts");
  return B200RL_OK;
}

int b200rl_ppo_weights(const int32_t* step_type, const float* ret, const float* adv,
                       const float* weights, int64_t n, float* out, void* stream) {
  B200RL_CHECK_ARG(step_type && ret && adv && out && n >= 1, "ppo_weights: bad argument");
  B200RL_LAUNCH(ppo_weights_kernel, blocks_of_256(n), 256, 0, (cudaStream_t)stream, step_type, ret, adv, weights, n, out);
  B200RL_CHECK_LAUNCH("ppo_weights");
  return B200RL_OK;
}

}  // extern "C"
