// DDPG update math: the single-critic TD loss, the clipped-dQ/da actor loss with its backward
// through scale_to_spec, and the Ornstein-Uhlenbeck exploration noise of OUNoisePolicy.
//
// Restates agents/ddpg/ddpg_agent.py: critic_loss (y = reward_scale r + gamma d Q'(s', a'),
// td_errors_loss_fn, mean over the batch) and actor_loss (element_wise_squared_loss(
// stop_gradient(a + clip(dqda)), a), mean over the batch); policies/ou_noise_policy.py with
// utils/common.py OUProcess (x <- (1 - damping) x + N(0, stddev), added to every row).  The loss
// reductions run in one block with a fixed order and no float atomics, so eager runs and graph
// replays give the same bits.  ddpg_seq_{critic,actor}_loss are the same two losses over the
// [B, T-1] transitions of recurrent sequences (multi-CTA, partials added by the last CTA).
#include <math.h>

#include "common.cuh"

namespace b200rl {

// y = reward_scale r + gamma d tq;  loss = sum_b w_b l(y, q_b) / B;  dq_b = w_b / B * dl/dq_b,
// l = td_elem_loss of e = y - q.
__global__ void __launch_bounds__(1024) ddpg_critic_loss_kernel(
    const float* __restrict__ q, const float* __restrict__ tq, const float* __restrict__ reward,
    const float* __restrict__ discount, const float* __restrict__ weights, int64_t B,
    float gamma, float reward_scale, int loss_kind, float* __restrict__ loss,
    float* __restrict__ dq, float* __restrict__ td_targets, int32_t* nan_flag) {
  pdl_prologue();
  __shared__ float red[32];
  const float inv_b = 1.f / (float)B;
  float s = 0.f;
  for (int64_t b = threadIdx.x; b < B; b += blockDim.x) {
    const float y = reward_scale * reward[b] + gamma * discount[b] * tq[b];
    if (td_targets) td_targets[b] = y;
    const float e = y - q[b];
    float l, g;
    td_elem_loss(e, loss_kind, l, g);
    const float w = weights ? weights[b] : 1.f;
    s += l * w;
    dq[b] = g * (w * inv_b);
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float out = s / (float)B;
    loss[0] = out;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
  }
}

// c = clip(dqda, +-clip_value) (c = dqda when !clip);  loss = sum_b w_b sum_k c_bk^2 / (B A);
// dy[b, k] = mag_k * (-2 w_b c_bk / (B A)): dL/da with no gradient through c, times the
// scale_to_spec derivative, i.e. the gradient w.r.t. the actor's tanh output.
__global__ void __launch_bounds__(1024) ddpg_actor_loss_kernel(
    const float* __restrict__ dqda, int64_t ld, const float* __restrict__ weights, int64_t B,
    int64_t A, int clip, float clip_value, const float* __restrict__ amin,
    const float* __restrict__ amax, float* __restrict__ loss, float* __restrict__ dy,
    int32_t* nan_flag) {
  pdl_prologue();
  __shared__ float red[32];
  const float inv_n = 1.f / ((float)B * (float)A);
  float s = 0.f;
  for (int64_t i = threadIdx.x; i < B * A; i += blockDim.x) {
    const int64_t b = i / A, k = i - b * A;
    float c = dqda[b * ld + k];
    if (clip) c = fminf(fmaxf(c, -clip_value), clip_value);
    const float w = weights ? weights[b] : 1.f;
    s += c * c * w;
    dy[i] = 0.5f * (amax[k] - amin[k]) * (-2.f * w * c * inv_n);
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float out = s * inv_n;
    loss[0] = out;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
  }
}

// The OU step of component k: (1 - damping) x_k + stddev z_k, with z_k = noise_in[k] or
// philox_normal on element k of the call rng_call[0].  Every thread that needs x_new[k] computes
// it from the unchanged x_old, so every block sees the same value.
__device__ __forceinline__ float ou_step(const float* state, int64_t k, float rho, float stddev,
                                         const float* noise_in, uint64_t seed, uint64_t call) {
  const float z = noise_in ? noise_in[k] : philox_normal((uint64_t)k, call, seed);
  return __fmaf_rn(rho, state[k], stddev * z);
}

// out[n, k] = loc[n, k] + x_new[k] (clamped to [amin, amax] when amin), one OU step per launch.
// rng_call: uint64[2] {call, ticket}.  The state is stored only by the block that takes the last
// ticket, after every other block has read x_old; the call counter advances there too, and only
// when the device draws.
__global__ void ou_noise_kernel(const float* __restrict__ loc, int64_t ld_loc, int64_t N,
                                int64_t A, float* state, float rho, float stddev,
                                const float* __restrict__ noise_in, uint64_t seed,
                                uint64_t* rng_call, const float* __restrict__ amin,
                                const float* __restrict__ amax, float* __restrict__ out,
                                int64_t ld_out) {
  pdl_prologue();
  __shared__ bool last;
  const uint64_t call = rng_call[0];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N * A) {
    const int64_t n = i / A, k = i - n * A;
    float v = loc[n * ld_loc + k] + ou_step(state, k, rho, stddev, noise_in, seed, call);
    if (amin) v = fminf(fmaxf(v, amin[k]), amax[k]);
    out[n * ld_out + k] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) last = last_block_ticket((uint32_t*)(rng_call + 1));
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int64_t k = threadIdx.x; k < A; k += blockDim.x)
    state[k] = ou_step(state, k, rho, stddev, noise_in, seed, call);
  __syncthreads();
  if (threadIdx.x == 0) {
    if (!noise_in) rng_call[0] = call + 1;
    __threadfence();
  }
}

// ---- recurrent DDPG: the same two losses over the [B, T-1] transitions of a sequence ------------
// Row r = b*(T-1) + t of q / tq / dq (and of dqda / dy) is transition t of sequence b.  G lanes per
// batch row: lane l takes the row's elements l, l + G, ... in order, the G lane sums meet in a fixed
// shuffle tree, every block stores one partial, and the block that takes the last ticket adds the
// partials in index order.  Every sum has a fixed order for a given shape, so repeated launches and
// graph replays give the same bits.  With T-1 = 1, dq and dy are the feed-forward kernels' bits.

// y = reward_scale r[b, t] + gamma d[b, t] tq[r];  td_loss_b = sum_t l(y - q[r]);
// loss = sum_b w_b td_loss_b / B;  dq[r] = w_b / B * dl/dq.  No LAST mask (ddpg_agent.py's TODO).
template <int G>
__global__ void __launch_bounds__(256) ddpg_seq_critic_loss_kernel(
    const float* __restrict__ q, const float* __restrict__ tq, const float* __restrict__ reward,
    const float* __restrict__ discount, int64_t ld, int64_t st, const float* __restrict__ weights,
    int64_t w_stride, int64_t B, int64_t Tm, float gamma, float reward_scale, int loss_kind,
    float* __restrict__ loss, float* __restrict__ dq, int32_t* nan_flag, float* partials,
    uint32_t* ticket) {
  pdl_prologue();
  __shared__ float red[32];
  __shared__ bool last;
  const float inv_b = 1.f / (float)B;
  float partial = 0.f;
  B200RL_GROUP_ROWS(G, B) {
    const bool live = n < B;
    const int64_t b = live ? n : n0;
    const float w = weights ? weights[b * w_stride] : 1.f;
    double s = 0.0;   // a lane may sum ~1000 steps: accumulate in double, round once
    for (int64_t t = lane; t < Tm; t += G) {
      const int64_t r = b * Tm + t;
      const float y = reward_scale * reward[b * ld + t * st] + gamma * discount[b * ld + t * st] *
                                                                   tq[r];
      float l, g;
      td_elem_loss(y - q[r], loss_kind, l, g);
      s += l;
      if (live) dq[r] = g * (w * inv_b);
    }
    const float row = grp_sum<G>((float)s);
    if (live && lane == 0) partial += row * w;
  }
  const float total = seq_loss_total(partial, partials, ticket, red, &last);
  if (last && threadIdx.x == 0) {
    const float out = total / (float)B;
    loss[0] = out;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
  }
}

// c = clip(dqda[r, k]) (c = dqda when !clip);  loss = sum_b w_b sum_{t,k} c^2 / (B A);
// dy[r, k] = mag_k * (-2 w_b c / (B A)).  Lanes stride over the (T-1)*A elements of row b.
template <int G>
__global__ void __launch_bounds__(256) ddpg_seq_actor_loss_kernel(
    const float* __restrict__ dqda, int64_t ld, const float* __restrict__ weights,
    int64_t w_stride, int64_t B, int64_t Tm, int64_t A, int clip, float clip_value,
    const float* __restrict__ amin, const float* __restrict__ amax, float* __restrict__ loss,
    float* __restrict__ dy, int32_t* nan_flag, float* partials, uint32_t* ticket) {
  pdl_prologue();
  __shared__ float red[32];
  __shared__ bool last;
  const float inv_n = 1.f / ((float)B * (float)A);
  const int64_t W = Tm * A;
  float partial = 0.f;
  B200RL_GROUP_ROWS(G, B) {
    const bool live = n < B;
    const int64_t b = live ? n : n0;
    const float w = weights ? weights[b * w_stride] : 1.f;
    double s = 0.0;   // a lane may sum ~1000 (t, k) terms: accumulate in double, round once
#pragma unroll 1
    for (int64_t j = lane; j < W; j += G) {
      const int64_t t = j / A, k = j - t * A, r = b * Tm + t;
      float c = dqda[r * ld + k];
      if (clip) c = fminf(fmaxf(c, -clip_value), clip_value);
      s += c * c * w;
      if (live) dy[r * A + k] = 0.5f * (amax[k] - amin[k]) * (-2.f * w * c * inv_n);
    }
    const float row = grp_sum<G>((float)s);
    if (live && lane == 0) partial += row;
  }
  const float total = seq_loss_total(partial, partials, ticket, red, &last);
  if (last && threadIdx.x == 0) {
    const float out = total * inv_n;
    loss[0] = out;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
  }
}

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_ddpg_critic_loss(const float* q, const float* tq, const float* reward,
                            const float* discount, const float* weights, int64_t B, float gamma,
                            float reward_scale, int loss_kind, float* loss, float* dq,
                            float* td_targets, int32_t* nan_flag, void* stream) {
  B200RL_CHECK_ARG(q && tq && reward && discount && loss && dq && B >= 1,
                   "ddpg_critic_loss: bad argument");
  B200RL_CHECK_ARG(loss_kind == B200RL_LOSS_HUBER || loss_kind == B200RL_LOSS_SQUARED,
                   "ddpg_critic_loss: unknown loss kind");
  B200RL_LAUNCH(ddpg_critic_loss_kernel, 1, reduce_threads(B), 0, (cudaStream_t)stream, q, tq, reward, discount, weights, B, gamma, reward_scale, loss_kind, loss, dq, td_targets, nan_flag);
  B200RL_CHECK_LAUNCH("ddpg_critic_loss");
  return B200RL_OK;
}

int b200rl_ddpg_actor_loss(const float* dqda, int64_t ld_dqda, const float* weights, int64_t B,
                           int64_t A, int clip, float dqda_clipping, const float* amin,
                           const float* amax, float* loss, float* dy, int32_t* nan_flag,
                           void* stream) {
  B200RL_CHECK_ARG(dqda && amin && amax && loss && dy && B >= 1 && A >= 1 && ld_dqda >= A,
                   "ddpg_actor_loss: bad argument");
  B200RL_CHECK_ARG(!clip || dqda_clipping >= 0.f, "ddpg_actor_loss: negative dqda_clipping");
  B200RL_LAUNCH(ddpg_actor_loss_kernel, 1, reduce_threads(B * A), 0, (cudaStream_t)stream, dqda, ld_dqda, weights, B, A, clip, dqda_clipping, amin, amax, loss, dy, nan_flag);
  B200RL_CHECK_LAUNCH("ddpg_actor_loss");
  return B200RL_OK;
}

int b200rl_ddpg_seq_critic_loss(const float* q, const float* tq, const float* reward,
                                const float* discount, int64_t ld, int64_t stride,
                                const float* weights, int64_t weight_stride, int64_t B, int64_t T,
                                float gamma, float reward_scale, int loss_kind, float* loss,
                                float* dq, int32_t* nan_flag, float* partials, uint32_t* ticket,
                                void* stream) {
  B200RL_CHECK_ARG(q && tq && reward && discount && loss && dq && partials && ticket,
                   "ddpg_seq_critic_loss: NULL argument");
  B200RL_CHECK_ARG(B >= 1, "ddpg_seq_critic_loss: B=%lld", (long long)B);
  B200RL_CHECK_ARG(T >= 2, "Trajectory frame count must be at least 2, but saw %lld", (long long)T);
  B200RL_CHECK_ARG(loss_kind == B200RL_LOSS_HUBER || loss_kind == B200RL_LOSS_SQUARED,
                   "ddpg_seq_critic_loss: unknown loss kind %d", loss_kind);
  B200RL_CHECK_ARG(ld >= 0 && stride >= 0 && weight_stride >= 0,
                   "ddpg_seq_critic_loss: strides must be >= 0");
  const int64_t Tm = T - 1;
  const int G = lane_group(Tm);
  const unsigned blocks = group_blocks(B, G, B200RL_DDPG_SEQ_MAX_BLOCKS);
  cudaStream_t st = (cudaStream_t)stream;
#define B200RL_DDPG_SEQ_CRITIC(GG)                                                                \
  B200RL_LAUNCH(ddpg_seq_critic_loss_kernel<GG>, blocks, 256, 0, st, q, tq, reward, discount, ld, \
                stride, weights, weight_stride, B, Tm, gamma, reward_scale, loss_kind, loss, dq,  \
                nan_flag, partials, ticket)
  if (G == 1)
    B200RL_DDPG_SEQ_CRITIC(1);
  else if (G == 8)
    B200RL_DDPG_SEQ_CRITIC(8);
  else
    B200RL_DDPG_SEQ_CRITIC(32);
#undef B200RL_DDPG_SEQ_CRITIC
  B200RL_CHECK_LAUNCH("ddpg_seq_critic_loss");
  return B200RL_OK;
}

int b200rl_ddpg_seq_actor_loss(const float* dqda, int64_t ld_dqda, const float* weights,
                               int64_t weight_stride, int64_t B, int64_t T, int64_t A, int clip,
                               float dqda_clipping, const float* amin, const float* amax,
                               float* loss, float* dy, int32_t* nan_flag, float* partials,
                               uint32_t* ticket, void* stream) {
  B200RL_CHECK_ARG(dqda && amin && amax && loss && dy && partials && ticket,
                   "ddpg_seq_actor_loss: NULL argument");
  B200RL_CHECK_ARG(B >= 1 && A >= 1 && ld_dqda >= A && weight_stride >= 0,
                   "ddpg_seq_actor_loss: B=%lld A=%lld ld=%lld", (long long)B, (long long)A,
                   (long long)ld_dqda);
  B200RL_CHECK_ARG(T >= 2, "Trajectory frame count must be at least 2, but saw %lld", (long long)T);
  B200RL_CHECK_ARG(!clip || dqda_clipping >= 0.f, "ddpg_seq_actor_loss: negative dqda_clipping");
  const int64_t Tm = T - 1;
  const int G = lane_group(Tm * A);
  const unsigned blocks = group_blocks(B, G, B200RL_DDPG_SEQ_MAX_BLOCKS);
  cudaStream_t st = (cudaStream_t)stream;
#define B200RL_DDPG_SEQ_ACTOR(GG)                                                                 \
  B200RL_LAUNCH(ddpg_seq_actor_loss_kernel<GG>, blocks, 256, 0, st, dqda, ld_dqda, weights,       \
                weight_stride, B, Tm, A, clip, dqda_clipping, amin, amax, loss, dy, nan_flag,     \
                partials, ticket)
  if (G == 1)
    B200RL_DDPG_SEQ_ACTOR(1);
  else if (G == 8)
    B200RL_DDPG_SEQ_ACTOR(8);
  else
    B200RL_DDPG_SEQ_ACTOR(32);
#undef B200RL_DDPG_SEQ_ACTOR
  B200RL_CHECK_LAUNCH("ddpg_seq_actor_loss");
  return B200RL_OK;
}

int b200rl_ou_noise(const float* loc, int64_t ld_loc, int64_t N, int64_t A, float* state,
                    float damping, float stddev, const float* noise_in, uint64_t seed,
                    uint64_t* rng_call_dev, const float* amin, const float* amax, float* out,
                    int64_t ld_out, void* stream) {
  B200RL_CHECK_ARG(loc && state && rng_call_dev && out && N >= 1 && A >= 1 && ld_loc >= A &&
                       ld_out >= A,
                   "ou_noise: bad argument");
  B200RL_CHECK_ARG((amin == nullptr) == (amax == nullptr), "ou_noise: amin/amax mismatch");
  B200RL_CHECK_ARG(stddev >= 0.f, "ou_noise: negative stddev");
  B200RL_LAUNCH(ou_noise_kernel, (unsigned)((N * A + 255) / 256), 256, 0, (cudaStream_t)stream, loc, ld_loc, N, A, state, 1.f - damping, stddev, noise_in, seed, rng_call_dev, amin, amax, out, ld_out);
  B200RL_CHECK_LAUNCH("ou_noise");
  return B200RL_OK;
}

}  // extern "C"
