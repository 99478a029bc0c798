// TD3 update math: scale-to-spec with target-policy smoothing, twin-critic TD loss, and the
// deterministic actor loss with its backward through scale_to_spec.
//
// Restates agents/td3/td3_agent.py: critic_loss (target smoothing, min of the target critics,
// TD target, td_errors_loss_fn on both critics, mean over the batch) and actor_loss
// (-Q1(s, pi(s)) aggregated over the batch); agents/ddpg/actor_network.py + utils/common.py
// scale_to_spec (means + magnitudes * tanh output).  The loss reductions run in one block with a
// fixed order and no float atomics, so eager runs and graph replays give the same bits.
#include <math.h>

#include "common.cuh"

namespace b200rl {

// out[n, k] = mean_k + mag_k * y[n, k]  (+ clip(std * z, +-noise_clip))  (clamped to the spec).
// z ~ N(0,1) comes from noise_in [N, A] or from philox_normal on element n*A+k of the call
// rng_call[0]; rng_call: uint64[2] {call, ticket}, advanced only when the device draws.
// y and out may alias (the agent rewrites the action columns of a critic input in place), so
// neither is __restrict__.
__global__ void td3_scale_to_spec_kernel(const float* y, int64_t ld_y, int64_t N,
                                         int64_t A, const float* __restrict__ amin,
                                         const float* __restrict__ amax, float noise_std,
                                         float noise_clip, const float* __restrict__ noise_in,
                                         uint64_t seed, uint64_t* rng_call, int clamp,
                                         float* out, int64_t ld_out) {
  pdl_prologue();
  const bool draw = noise_std > 0.f && noise_in == nullptr;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N * A) {
    const int64_t n = i / A, k = i - n * A;
    const float lo = amin[k], hi = amax[k];
    float v = 0.5f * (hi + lo) + 0.5f * (hi - lo) * y[n * ld_y + k];
    if (noise_std > 0.f) {
      const float z = noise_in ? noise_in[i] : philox_normal((uint64_t)i, rng_call[0], seed);
      v += fminf(fmaxf(noise_std * z, -noise_clip), noise_clip);
    }
    if (clamp) v = fminf(fmaxf(v, lo), hi);
    out[n * ld_out + k] = v;
  }
  if (draw) next_rng_call(rng_call);
}

// y = reward_scale r + gamma d min(tq1, tq2);  loss = sum_b w_b (l(y, q1) + l(y, q2)) / B;
// dq_i = w_b / B * dl(y, q_i)/dq_i, l = td_elem_loss of e = y - q.
__global__ void __launch_bounds__(1024) td3_critic_loss_kernel(
    const float* __restrict__ q1, const float* __restrict__ q2, const float* __restrict__ tq1,
    const float* __restrict__ tq2, const float* __restrict__ reward,
    const float* __restrict__ discount, const float* __restrict__ weights, int64_t B,
    float gamma, float reward_scale, int loss_kind, float* __restrict__ loss,
    float* __restrict__ dq1, float* __restrict__ dq2, float* __restrict__ td_targets,
    int32_t* nan_flag) {
  pdl_prologue();
  __shared__ float red[32];
  const float inv_b = 1.f / (float)B;
  float s = 0.f;
  for (int64_t b = threadIdx.x; b < B; b += blockDim.x) {
    const float y = reward_scale * reward[b] + gamma * discount[b] * fminf(tq1[b], tq2[b]);
    if (td_targets) td_targets[b] = y;
    const float e1 = y - q1[b], e2 = y - q2[b];
    float l2, l, g1, g2;
    td_elem_loss(e2, loss_kind, l2, g2);
    td_elem_loss(e1, loss_kind, l, g1, l2);                 // l = l(e1) + l(e2)
    const float w = weights ? weights[b] : 1.f;
    s += l * w;
    const float c = w * inv_b;
    dq1[b] = g1 * c;
    dq2[b] = g2 * c;
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float out = s / (float)B;
    loss[0] = out;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
  }
}

// loss = sum_b w_b (-q_b) / B;  dq_b = -w_b / B.
__global__ void __launch_bounds__(1024) td3_actor_loss_kernel(
    const float* __restrict__ q, const float* __restrict__ weights, int64_t B,
    float* __restrict__ loss, float* __restrict__ dq, int32_t* nan_flag) {
  pdl_prologue();
  __shared__ float red[32];
  const float inv_b = 1.f / (float)B;
  float s = 0.f;
  for (int64_t b = threadIdx.x; b < B; b += blockDim.x) {
    const float w = weights ? weights[b] : 1.f;
    s += -q[b] * w;
    dq[b] = -w * inv_b;
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float out = s / (float)B;
    loss[0] = out;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
  }
}

// dL/dy[n, k] = mag_k * dL/da[n, k]: the backward of scale_to_spec; the tanh derivative of the
// action layer is applied by the layer's own backward.
__global__ void td3_actor_bwd_kernel(const float* __restrict__ da, int64_t ld_da,
                                     const float* __restrict__ amin,
                                     const float* __restrict__ amax, int64_t N, int64_t A,
                                     float* __restrict__ dy) {
  pdl_prologue();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * A) return;
  const int64_t n = i / A, k = i - n * A;
  dy[i] = 0.5f * (amax[k] - amin[k]) * da[n * ld_da + k];
}

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_td3_scale_to_spec(const float* y, int64_t ld_y, int64_t N, int64_t A,
                             const float* amin, const float* amax, float noise_std,
                             float noise_clip, const float* noise_in, uint64_t seed,
                             uint64_t* rng_call_dev, int clamp, float* out, int64_t ld_out,
                             void* stream) {
  B200RL_CHECK_ARG(y && amin && amax && out && N >= 1 && A >= 1 && ld_y >= A && ld_out >= A,
                   "td3_scale_to_spec: bad argument");
  B200RL_CHECK_ARG(noise_std >= 0.f && noise_clip >= 0.f, "td3_scale_to_spec: negative noise");
  B200RL_CHECK_ARG(noise_std == 0.f || noise_in || rng_call_dev,
                   "td3_scale_to_spec: noise needs noise_in or rng_call_dev");
  B200RL_LAUNCH(td3_scale_to_spec_kernel, blocks_of_256(N * A), 256, 0, (cudaStream_t)stream, y, ld_y, N, A, amin, amax, noise_std, noise_clip, noise_in, seed, rng_call_dev, clamp, out, ld_out);
  B200RL_CHECK_LAUNCH("td3_scale_to_spec");
  return B200RL_OK;
}

int b200rl_td3_critic_loss(const float* q1, const float* q2, const float* tq1, const float* tq2,
                           const float* reward, const float* discount, const float* weights,
                           int64_t B, float gamma, float reward_scale, int loss_kind,
                           float* loss, float* dq1, float* dq2, float* td_targets,
                           int32_t* nan_flag, void* stream) {
  B200RL_CHECK_ARG(q1 && q2 && tq1 && tq2 && reward && discount && loss && dq1 && dq2 && B >= 1,
                   "td3_critic_loss: bad argument");
  B200RL_CHECK_ARG(loss_kind == B200RL_LOSS_HUBER || loss_kind == B200RL_LOSS_SQUARED,
                   "td3_critic_loss: unknown loss kind");
  B200RL_LAUNCH(td3_critic_loss_kernel, 1, reduce_threads(B), 0, (cudaStream_t)stream, q1, q2, tq1, tq2, reward, discount, weights, B, gamma, reward_scale, loss_kind, loss, dq1, dq2, td_targets, nan_flag);
  B200RL_CHECK_LAUNCH("td3_critic_loss");
  return B200RL_OK;
}

int b200rl_td3_actor_loss(const float* q, const float* weights, int64_t B, float* loss,
                          float* dq, int32_t* nan_flag, void* stream) {
  B200RL_CHECK_ARG(q && loss && dq && B >= 1, "td3_actor_loss: bad argument");
  B200RL_LAUNCH(td3_actor_loss_kernel, 1, reduce_threads(B), 0, (cudaStream_t)stream, q, weights, B, loss, dq, nan_flag);
  B200RL_CHECK_LAUNCH("td3_actor_loss");
  return B200RL_OK;
}

int b200rl_td3_actor_bwd(const float* da, int64_t ld_da, const float* amin, const float* amax,
                         int64_t N, int64_t A, float* dy, void* stream) {
  B200RL_CHECK_ARG(da && amin && amax && dy && N >= 1 && A >= 1 && ld_da >= A,
                   "td3_actor_bwd: bad argument");
  B200RL_LAUNCH(td3_actor_bwd_kernel, blocks_of_256(N * A), 256, 0, (cudaStream_t)stream, da, ld_da, amin, amax, N, A, dy);
  B200RL_CHECK_LAUNCH("td3_actor_bwd");
  return B200RL_OK;
}

}  // extern "C"
