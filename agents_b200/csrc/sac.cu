// SAC update math (kernel family iii-d): reparameterised tanh-Normal sampling with log-prob,
// twin-Q TD target / critic loss, actor loss, alpha loss — each forward and backward fused.
//
// Restates agents/sac/sac_agent.py: _actions_and_log_probs :537-557, critic_loss :559-643,
// actor_loss :645-694, alpha_loss :696-739; agents/sac/tanh_normal_projection_network.py:112-143
// (loc, std = exp(log_std)); distributions/utils.py:40-160 SquashToSpecNormal and
// distributions/tanh_bijector_stable.py:68-82 (log|d tanh| = 2 (log 2 - u - softplus(-2u))).
// All reductions are single-block, fixed-order (B <= a few thousand rows).
#include <math.h>

#include "common.cuh"

namespace b200rl {

// head [N, 2A] = (loc | log_std).  u = loc + exp(log_std) * eps;  a = shift + half * tanh(u);
// log_pi = sum_k [ -0.5 eps^2 - log_std - 0.5 log(2 pi) - log(half) - 2 (log2 - u - softplus(-2u)) ]
__global__ void sac_sample_kernel(const float* __restrict__ head, int64_t N, int64_t A,
                                  const float* __restrict__ amin, const float* __restrict__ amax,
                                  const float* __restrict__ eps_in, uint64_t seed,
                                  uint64_t* rng_call, float* __restrict__ action, int64_t ld_a,
                                  float* __restrict__ logp, float* __restrict__ u_out,
                                  float* __restrict__ eps_out) {
  pdl_prologue();
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n < N) {
    float lp = 0.f;
    for (int64_t k = 0; k < A; ++k) {
      const float e = eps_in ? eps_in[n * A + k]
                             : philox_normal((uint64_t)(n * A + k), rng_call[0], seed);
      const float loc = head[n * 2 * A + k], ls = head[n * 2 * A + A + k];
      const float u = loc + expf(ls) * e;
      const float half = 0.5f * (amax[k] - amin[k]), shift = 0.5f * (amax[k] + amin[k]);
      action[n * ld_a + k] = shift + half * tanhf(u);
      lp += -0.5f * e * e - ls - 0.5f * kLog2PiS - logf(half) -
            2.f * (kLog2 - u - softplus_f(-2.f * u));
      if (u_out) u_out[n * A + k] = u;
      if (eps_out) eps_out[n * A + k] = e;
    }
    logp[n] = lp;
  }
  if (!eps_in) next_rng_call(rng_call);
}

// Given dL/da (sum of up to two [N, ld] views) and dL/dlogp, write dL/dhead [N, 2A].
__global__ void sac_sample_bwd_kernel(const float* __restrict__ head,
                                      const float* __restrict__ u_saved,
                                      const float* __restrict__ eps_saved,
                                      const float* __restrict__ amin,
                                      const float* __restrict__ amax,
                                      const float* __restrict__ da1, const float* __restrict__ da2,
                                      int64_t ld_da, const float* __restrict__ dlogp, int64_t N,
                                      int64_t A, float* __restrict__ dhead) {
  pdl_prologue();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * A) return;
  const int64_t n = i / A, k = i - n * A;
  const float u = u_saved[i], e = eps_saved[i];
  const float std = expf(head[n * 2 * A + A + k]);
  const float half = 0.5f * (amax[k] - amin[k]);
  const float t = tanhf(u);
  float da = da1 ? da1[n * ld_da + k] : 0.f;
  if (da2) da += da2[n * ld_da + k];
  const float g = dlogp[n];
  // d a / d u = half (1 - t^2);  d logp / d u = 2 t (from -log|d tanh|), d logp / d log_std = -1
  const float du = da * half * (1.f - t * t) + g * 2.f * t;
  dhead[n * 2 * A + k] = du;
  dhead[n * 2 * A + A + k] = du * std * e - g;
}

__global__ void __launch_bounds__(256) sac_critic_loss_kernel(
    const float* __restrict__ q1, const float* __restrict__ q2, const float* __restrict__ tq1,
    const float* __restrict__ tq2, const float* __restrict__ next_logp,
    const float* __restrict__ reward, const float* __restrict__ discount,
    const float* __restrict__ weights, const float* __restrict__ log_alpha, int64_t B,
    float gamma, float reward_scale, float loss_weight, float global_batch,
    float* __restrict__ loss, float* __restrict__ dq1, float* __restrict__ dq2,
    float* __restrict__ td_targets, int32_t* nan_flag) {
  pdl_prologue();
  __shared__ float red[32];
  const float alpha = expf(log_alpha[0]);
  float s = 0.f;
  for (int64_t b = threadIdx.x; b < B; b += blockDim.x) {
    const float tq = fminf(tq1[b], tq2[b]) - alpha * next_logp[b];            // :603-606
    const float y = reward_scale * reward[b] + gamma * discount[b] * tq;      // :608-611
    if (td_targets) td_targets[b] = y;
    const float e1 = y - q1[b], e2 = y - q2[b];
    const float w = weights ? weights[b] : 1.f;
    const float l = e1 * e1 + e2 * e2;                                        // :621-623
    s += (weights && w == 0.f) ? 0.f : l * w;
    const float c = loss_weight * w / global_batch;
    dq1[b] = -2.f * e1 * c;
    dq2[b] = -2.f * e2 * c;
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float out = loss_weight * s / global_batch;
    loss[0] = out;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
  }
}

__global__ void __launch_bounds__(256) sac_actor_loss_kernel(
    const float* __restrict__ q1, const float* __restrict__ q2, const float* __restrict__ logp,
    const float* __restrict__ weights, const float* __restrict__ log_alpha, int64_t B,
    float loss_weight, float global_batch, float* __restrict__ loss, float* __restrict__ dlogp,
    float* __restrict__ dq1, float* __restrict__ dq2, int32_t* nan_flag) {
  pdl_prologue();
  __shared__ float red[32];
  const float alpha = expf(log_alpha[0]);
  float s = 0.f;
  for (int64_t b = threadIdx.x; b < B; b += blockDim.x) {
    const float a = q1[b], c = q2[b];
    const float qmin = fminf(a, c);                                            // :676
    const float w = weights ? weights[b] : 1.f;
    const float l = alpha * logp[b] - qmin;                                    // :677
    s += (weights && w == 0.f) ? 0.f : l * w;
    const float k = loss_weight * w / global_batch;
    dlogp[b] = alpha * k;
    const bool first = a <= c;  // tf.minimum routes the gradient to x where x <= y
    dq1[b] = first ? -k : 0.f;
    dq2[b] = first ? 0.f : -k;
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float out = loss_weight * s / global_batch;
    loss[0] = out;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
  }
}

__global__ void __launch_bounds__(256) sac_alpha_loss_kernel(
    const float* __restrict__ logp, const float* __restrict__ weights,
    const float* __restrict__ log_alpha, int64_t B, float target_entropy, int use_log_alpha,
    float loss_weight, float global_batch, float* __restrict__ loss,
    float* __restrict__ dlog_alpha, int32_t* nan_flag) {
  pdl_prologue();
  __shared__ float red[32];
  float s = 0.f;
  for (int64_t b = threadIdx.x; b < B; b += blockDim.x) {
    const float w = weights ? weights[b] : 1.f;
    const float diff = -logp[b] - target_entropy;                              // :720
    s += (weights && w == 0.f) ? 0.f : diff * w;
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float la = log_alpha[0];
    const float coef = use_log_alpha ? la : expf(la);                          // :721-724
    const float dcoef = use_log_alpha ? 1.f : expf(la);
    const float out = loss_weight * coef * s / global_batch;
    loss[0] = out;
    dlog_alpha[0] = loss_weight * dcoef * s / global_batch;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
  }
}

__global__ void concat2_kernel(const float* __restrict__ a, int64_t lda, int64_t da,
                               const float* __restrict__ b, int64_t ldb, int64_t db, int64_t N,
                               float* __restrict__ out) {
  pdl_prologue();
  const int64_t w = da + db;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * w) return;
  const int64_t n = i / w, k = i - n * w;
  out[i] = k < da ? a[n * lda + k] : b[n * ldb + (k - da)];
}

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_sac_sample(const float* head, int64_t N, int64_t A, const float* amin,
                      const float* amax, const float* eps_in, uint64_t seed,
                      uint64_t* rng_call_dev, float* action, int64_t ld_action, float* logp,
                      float* u_out, float* eps_out, void* stream) {
  B200RL_CHECK_ARG(head && amin && amax && action && logp && N >= 1 && A >= 1 && ld_action >= A,
                   "sac_sample: bad argument");
  B200RL_CHECK_ARG(eps_in || rng_call_dev, "sac_sample: need eps or rng_call_dev");
  B200RL_LAUNCH(sac_sample_kernel, blocks_of_256(N), 256, 0, (cudaStream_t)stream, head, N, A, amin, amax, eps_in, seed, rng_call_dev, action, ld_action, logp, u_out, eps_out);
  B200RL_CHECK_LAUNCH("sac_sample");
  return B200RL_OK;
}

int b200rl_sac_sample_bwd(const float* head, const float* u_saved, const float* eps_saved,
                          const float* amin, const float* amax, const float* da1,
                          const float* da2, int64_t ld_da, const float* dlogp, int64_t N,
                          int64_t A, float* dhead, void* stream) {
  B200RL_CHECK_ARG(head && u_saved && eps_saved && amin && amax && dlogp && dhead && N >= 1 &&
                       A >= 1,
                   "sac_sample_bwd: bad argument");
  B200RL_LAUNCH(sac_sample_bwd_kernel, blocks_of_256(N * A), 256, 0, (cudaStream_t)stream, head, u_saved, eps_saved, amin, amax, da1, da2, ld_da, dlogp, N, A, dhead);
  B200RL_CHECK_LAUNCH("sac_sample_bwd");
  return B200RL_OK;
}

int b200rl_sac_critic_loss(const float* q1, const float* q2, const float* tq1, const float* tq2,
                           const float* next_logp, const float* reward, const float* discount,
                           const float* weights, const float* log_alpha_dev, int64_t B,
                           float gamma, float reward_scale, float loss_weight,
                           float global_batch, float* loss, float* dq1, float* dq2,
                           float* td_targets, int32_t* nan_flag, void* stream) {
  B200RL_CHECK_ARG(q1 && q2 && tq1 && tq2 && next_logp && reward && discount && log_alpha_dev &&
                       loss && dq1 && dq2 && B >= 1 && global_batch > 0.f,
                   "sac_critic_loss: bad argument");
  B200RL_LAUNCH(sac_critic_loss_kernel, 1, 256, 0, (cudaStream_t)stream, q1, q2, tq1, tq2, next_logp, reward, discount, weights, log_alpha_dev, B, gamma, reward_scale, loss_weight, global_batch, loss, dq1, dq2, td_targets, nan_flag);
  B200RL_CHECK_LAUNCH("sac_critic_loss");
  return B200RL_OK;
}

int b200rl_sac_actor_loss(const float* q1, const float* q2, const float* logp,
                          const float* weights, const float* log_alpha_dev, int64_t B,
                          float loss_weight, float global_batch, float* loss, float* dlogp,
                          float* dq1, float* dq2, int32_t* nan_flag, void* stream) {
  B200RL_CHECK_ARG(q1 && q2 && logp && log_alpha_dev && loss && dlogp && dq1 && dq2 && B >= 1 &&
                       global_batch > 0.f,
                   "sac_actor_loss: bad argument");
  B200RL_LAUNCH(sac_actor_loss_kernel, 1, 256, 0, (cudaStream_t)stream, q1, q2, logp, weights, log_alpha_dev, B, loss_weight, global_batch, loss, dlogp, dq1, dq2, nan_flag);
  B200RL_CHECK_LAUNCH("sac_actor_loss");
  return B200RL_OK;
}

int b200rl_sac_alpha_loss(const float* logp, const float* weights, const float* log_alpha_dev,
                          int64_t B, float target_entropy, int use_log_alpha, float loss_weight,
                          float global_batch, float* loss, float* dlog_alpha, int32_t* nan_flag,
                          void* stream) {
  B200RL_CHECK_ARG(logp && log_alpha_dev && loss && dlog_alpha && B >= 1 && global_batch > 0.f,
                   "sac_alpha_loss: bad argument");
  B200RL_LAUNCH(sac_alpha_loss_kernel, 1, 256, 0, (cudaStream_t)stream, logp, weights, log_alpha_dev, B, target_entropy, use_log_alpha, loss_weight, global_batch, loss, dlog_alpha, nan_flag);
  B200RL_CHECK_LAUNCH("sac_alpha_loss");
  return B200RL_OK;
}

int b200rl_concat2(const float* a, int64_t lda, int64_t da, const float* b, int64_t ldb,
                   int64_t db, int64_t N, float* out, void* stream) {
  B200RL_CHECK_ARG(a && b && out && N >= 1 && da >= 1 && db >= 1 && lda >= da && ldb >= db,
                   "concat2: bad argument");
  B200RL_LAUNCH(concat2_kernel, blocks_of_256(N * (da + db)), 256, 0, (cudaStream_t)stream, a, lda, da, b, ldb, db, N, out);
  B200RL_CHECK_LAUNCH("concat2");
  return B200RL_OK;
}

}  // extern "C"
