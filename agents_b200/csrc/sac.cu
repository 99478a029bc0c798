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

// ---- recurrent SAC: the three losses over the [B, T-1] transitions of a sequence ---------------
// Row r = b*(T-1) + t of q1 / q2 / tq1 / tq2 / logp and of the gradients is transition t of
// sequence b.  G lanes per batch row take its steps l, l + G, ... in order and accumulate in
// double; the G lane sums meet in a fixed shuffle tree, the row sum is weighted once, and
// seq_loss_total adds the block partials in index order.  Every sum has a fixed order for a given
// shape, so repeated launches and graph replays give the same bits.  With T-1 = 1 the per-row
// gradients are the feed-forward kernels' bits.  A row of weight 0 adds exactly 0.

// tq = min(tq1, tq2) - alpha next_logp;  y = reward_scale r[b, t] + gamma d[b, t] tq;
// loss = loss_weight sum_b w_b sum_t [(y - q1)^2 + (y - q2)^2] / B;  dq_i = -2 (y - q_i) c with
// c = loss_weight w_b / B.  No LAST mask (as sac_agent.py with AsTransition).
template <int G>
__global__ void __launch_bounds__(256) sac_seq_critic_loss_kernel(
    const float* __restrict__ q1, const float* __restrict__ q2, const float* __restrict__ tq1,
    const float* __restrict__ tq2, const float* __restrict__ next_logp,
    const float* __restrict__ reward, const float* __restrict__ discount, int64_t ld, int64_t st,
    const float* __restrict__ weights, int64_t w_stride, const float* __restrict__ log_alpha,
    int64_t B, int64_t Tm, float gamma, float reward_scale, float loss_weight,
    float* __restrict__ loss, float* __restrict__ dq1, float* __restrict__ dq2, int32_t* nan_flag,
    float* partials, uint32_t* ticket) {
  pdl_prologue();
  __shared__ float red[32];
  __shared__ bool last;
  const float alpha = expf(log_alpha[0]);
  const float global_batch = (float)B;
  float partial = 0.f;
  B200RL_GROUP_ROWS(G, B) {
    const bool live = n < B;
    const int64_t b = live ? n : n0;
    const float w = weights ? weights[b * w_stride] : 1.f;
    const float c = loss_weight * w / global_batch;
    double s = 0.0;   // a lane may sum ~1000 steps: accumulate in double, round once
    for (int64_t t = lane; t < Tm; t += G) {
      const int64_t r = b * Tm + t;
      const float tq = fminf(tq1[r], tq2[r]) - alpha * next_logp[r];
      const float y = reward_scale * reward[b * ld + t * st] + gamma * discount[b * ld + t * st] *
                                                                   tq;
      const float e1 = y - q1[r], e2 = y - q2[r];
      s += e1 * e1 + e2 * e2;
      if (live) {
        dq1[r] = -2.f * e1 * c;
        dq2[r] = -2.f * e2 * c;
      }
    }
    const float row = grp_sum<G>((float)s);
    if (live && lane == 0) partial += (weights && w == 0.f) ? 0.f : row * w;
  }
  const float total = seq_loss_total(partial, partials, ticket, red, &last);
  if (last && threadIdx.x == 0) {
    const float out = loss_weight * total / global_batch;
    loss[0] = out;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
  }
}

// loss = loss_weight sum_b w_b sum_t (alpha logp - min(q1, q2)) / B;  with k = loss_weight w_b / B:
// dlogp = alpha k, and -k to q1 where q1 <= q2 (tf.minimum's gradient routing), else to q2.
template <int G>
__global__ void __launch_bounds__(256) sac_seq_actor_loss_kernel(
    const float* __restrict__ q1, const float* __restrict__ q2, const float* __restrict__ logp,
    const float* __restrict__ weights, int64_t w_stride, const float* __restrict__ log_alpha,
    int64_t B, int64_t Tm, float loss_weight, float* __restrict__ loss,
    float* __restrict__ dlogp, float* __restrict__ dq1, float* __restrict__ dq2,
    int32_t* nan_flag, float* partials, uint32_t* ticket) {
  pdl_prologue();
  __shared__ float red[32];
  __shared__ bool last;
  const float alpha = expf(log_alpha[0]);
  const float global_batch = (float)B;
  float partial = 0.f;
  B200RL_GROUP_ROWS(G, B) {
    const bool live = n < B;
    const int64_t b = live ? n : n0;
    const float w = weights ? weights[b * w_stride] : 1.f;
    const float k = loss_weight * w / global_batch;
    double s = 0.0;
    for (int64_t t = lane; t < Tm; t += G) {
      const int64_t r = b * Tm + t;
      const float a = q1[r], c = q2[r];
      s += alpha * logp[r] - fminf(a, c);
      if (live) {
        const bool first = a <= c;
        dlogp[r] = alpha * k;
        dq1[r] = first ? -k : 0.f;
        dq2[r] = first ? 0.f : -k;
      }
    }
    const float row = grp_sum<G>((float)s);
    if (live && lane == 0) partial += (weights && w == 0.f) ? 0.f : row * w;
  }
  const float total = seq_loss_total(partial, partials, ticket, red, &last);
  if (last && threadIdx.x == 0) {
    const float out = loss_weight * total / global_batch;
    loss[0] = out;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
  }
}

// S = sum_b w_b sum_t (-logp - target_entropy);  loss = loss_weight coef S / B and
// dlog_alpha = loss_weight dcoef S / B, coef = log_alpha (dcoef 1) or alpha (dcoef alpha).
template <int G>
__global__ void __launch_bounds__(256) sac_seq_alpha_loss_kernel(
    const float* __restrict__ logp, const float* __restrict__ weights, int64_t w_stride,
    const float* __restrict__ log_alpha, int64_t B, int64_t Tm, float target_entropy,
    int use_log_alpha, float loss_weight, float* __restrict__ loss,
    float* __restrict__ dlog_alpha, int32_t* nan_flag, float* partials, uint32_t* ticket) {
  pdl_prologue();
  __shared__ float red[32];
  __shared__ bool last;
  float partial = 0.f;
  B200RL_GROUP_ROWS(G, B) {
    const bool live = n < B;
    const int64_t b = live ? n : n0;
    const float w = weights ? weights[b * w_stride] : 1.f;
    double s = 0.0;
    for (int64_t t = lane; t < Tm; t += G) s += -logp[b * Tm + t] - target_entropy;
    const float row = grp_sum<G>((float)s);
    if (live && lane == 0) partial += (weights && w == 0.f) ? 0.f : row * w;
  }
  const float total = seq_loss_total(partial, partials, ticket, red, &last);
  if (last && threadIdx.x == 0) {
    const float la = log_alpha[0];
    const float coef = use_log_alpha ? la : expf(la);
    const float dcoef = use_log_alpha ? 1.f : expf(la);
    const float out = loss_weight * coef * total / (float)B;
    loss[0] = out;
    dlog_alpha[0] = loss_weight * dcoef * total / (float)B;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
  }
}

}  // namespace b200rl

namespace {

// Lanes per row, grid and argument checks shared by the three sequence-loss entry points.
int sac_seq_shape(const char* name, int64_t B, int64_t T, int64_t weight_stride, int* G,
                  unsigned* blocks) {
  B200RL_CHECK_ARG(B >= 1, "%s: B=%lld", name, (long long)B);
  B200RL_CHECK_ARG(T >= 2, "Trajectory frame count must be at least 2, but saw %lld", (long long)T);
  B200RL_CHECK_ARG(weight_stride >= 0, "%s: weight_stride must be >= 0", name);
  *G = b200rl::lane_group(T - 1);
  *blocks = b200rl::group_blocks(B, *G, B200RL_SAC_SEQ_MAX_BLOCKS);
  return B200RL_OK;
}

}  // namespace

// G is one of 1, 8, 32 (lane_group); the launch picks the matching instantiation.
#define B200RL_SAC_SEQ_LAUNCH(kernel, G, blocks, st, ...)         \
  do {                                                            \
    if ((G) == 1)                                                 \
      B200RL_LAUNCH(kernel<1>, blocks, 256, 0, st, __VA_ARGS__);  \
    else if ((G) == 8)                                            \
      B200RL_LAUNCH(kernel<8>, blocks, 256, 0, st, __VA_ARGS__);  \
    else                                                          \
      B200RL_LAUNCH(kernel<32>, blocks, 256, 0, st, __VA_ARGS__); \
  } while (0)

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

int b200rl_sac_seq_critic_loss(const float* q1, const float* q2, const float* tq1,
                               const float* tq2, const float* next_logp, const float* reward,
                               const float* discount, int64_t ld, int64_t stride,
                               const float* weights, int64_t weight_stride,
                               const float* log_alpha_dev, int64_t B, int64_t T, float gamma,
                               float reward_scale, float loss_weight, float* loss, float* dq1,
                               float* dq2, int32_t* nan_flag, float* partials, uint32_t* ticket,
                               void* stream) {
  B200RL_CHECK_ARG(q1 && q2 && tq1 && tq2 && next_logp && reward && discount && log_alpha_dev &&
                       loss && dq1 && dq2 && partials && ticket,
                   "sac_seq_critic_loss: NULL argument");
  B200RL_CHECK_ARG(ld >= 0 && stride >= 0, "sac_seq_critic_loss: strides must be >= 0");
  int G;
  unsigned blocks;
  const int rc = sac_seq_shape("sac_seq_critic_loss", B, T, weight_stride, &G, &blocks);
  if (rc != B200RL_OK) return rc;
  B200RL_SAC_SEQ_LAUNCH(sac_seq_critic_loss_kernel, G, blocks, (cudaStream_t)stream, q1, q2, tq1,
                        tq2, next_logp, reward, discount, ld, stride, weights, weight_stride,
                        log_alpha_dev, B, T - 1, gamma, reward_scale, loss_weight, loss, dq1, dq2,
                        nan_flag, partials, ticket);
  B200RL_CHECK_LAUNCH("sac_seq_critic_loss");
  return B200RL_OK;
}

int b200rl_sac_seq_actor_loss(const float* q1, const float* q2, const float* logp,
                              const float* weights, int64_t weight_stride,
                              const float* log_alpha_dev, int64_t B, int64_t T, float loss_weight,
                              float* loss, float* dlogp, float* dq1, float* dq2, int32_t* nan_flag,
                              float* partials, uint32_t* ticket, void* stream) {
  B200RL_CHECK_ARG(q1 && q2 && logp && log_alpha_dev && loss && dlogp && dq1 && dq2 && partials &&
                       ticket,
                   "sac_seq_actor_loss: NULL argument");
  int G;
  unsigned blocks;
  const int rc = sac_seq_shape("sac_seq_actor_loss", B, T, weight_stride, &G, &blocks);
  if (rc != B200RL_OK) return rc;
  B200RL_SAC_SEQ_LAUNCH(sac_seq_actor_loss_kernel, G, blocks, (cudaStream_t)stream, q1, q2, logp,
                        weights, weight_stride, log_alpha_dev, B, T - 1, loss_weight, loss, dlogp,
                        dq1, dq2, nan_flag, partials, ticket);
  B200RL_CHECK_LAUNCH("sac_seq_actor_loss");
  return B200RL_OK;
}

int b200rl_sac_seq_alpha_loss(const float* logp, const float* weights, int64_t weight_stride,
                              const float* log_alpha_dev, int64_t B, int64_t T,
                              float target_entropy, int use_log_alpha, float loss_weight,
                              float* loss, float* dlog_alpha, int32_t* nan_flag, float* partials,
                              uint32_t* ticket, void* stream) {
  B200RL_CHECK_ARG(logp && log_alpha_dev && loss && dlog_alpha && partials && ticket,
                   "sac_seq_alpha_loss: NULL argument");
  int G;
  unsigned blocks;
  const int rc = sac_seq_shape("sac_seq_alpha_loss", B, T, weight_stride, &G, &blocks);
  if (rc != B200RL_OK) return rc;
  B200RL_SAC_SEQ_LAUNCH(sac_seq_alpha_loss_kernel, G, blocks, (cudaStream_t)stream, logp, weights,
                        weight_stride, log_alpha_dev, B, T - 1, target_entropy, use_log_alpha,
                        loss_weight, loss, dlog_alpha, nan_flag, partials, ticket);
  B200RL_CHECK_LAUNCH("sac_seq_alpha_loss");
  return B200RL_OK;
}

}  // extern "C"
