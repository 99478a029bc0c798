// CQL-SAC (kernel family iii-d): the conservative term of the critic step, its candidate actions,
// the optional reward noise and the behavioural-cloning (BC) actor term.
//
// Restates agents/cql/cql_sac_agent.py: _cql_loss :534-679, actor_loss :681-750 (BC branch),
// _get_cql_alpha :752-765, the Lagrange step of _train :336-348, reward noise :832-839;
// distributions/tanh_bijector_stable.py:58-82 (inverse tanh with the +-0.99999997 clip).
//
// Critic joint-input rows (one forward / backward per critic covers all of them):
//   [0, B)             (s_b, a_data_b)
//   [B, B+BN)          (s_b, a ~ pi(.|s_b))     row B + b*N + j
//   [B+BN, B+2BN)      (s_b, a ~ U[min, max))   row B + BN + b*N + j
// (nest_utils.tile_batch order: the N candidates of state b are consecutive.)
// Reductions are fixed-order (per-block partials, one single-CTA finish), so results repeat bit
// for bit.
#include <math.h>

#include "common.cuh"

namespace b200rl {

constexpr int kCqlRedBlocks = 256;

// Tiles the observation into every candidate row, fills the uniform candidates' actions
// (tf.random.uniform(minval, maxval) = minval + u * (maxval - minval), u in [0, 1)) and tiles the
// actor head [B, 2A] -> [BN, 2A] for b200rl_sac_sample.  The policy candidates' action columns are
// left to b200rl_sac_sample.
__global__ void cql_candidates_kernel(const float* __restrict__ obs, int64_t ld_obs, int64_t B,
                                      int64_t N, int64_t D, int64_t A,
                                      const float* __restrict__ amin,
                                      const float* __restrict__ amax,
                                      const float* __restrict__ u_in, uint64_t seed,
                                      uint64_t* rng_call, const float* __restrict__ head,
                                      float* __restrict__ x, float* __restrict__ head_tiled) {
  pdl_prologue();
  const int64_t W = D + A, BN = B * N;
  const int64_t n_x = 2 * BN * W, n_h = BN * 2 * A;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_x) {
    const int64_t r = i / W, c = i - r * W;
    const int64_t b = (r < BN ? r : r - BN) / N;
    float* dst = x + (B + r) * W + c;
    if (c < D) {
      *dst = obs[b * ld_obs + c];
    } else if (r >= BN) {                                                       // :607-612
      const int64_t k = c - D, e = (r - BN) * A + k;
      const float u = u_in ? u_in[e]
                           : uniform_f32(philox4x32_10((uint64_t)e, rng_call[0], seed).x);
      *dst = __fadd_rn(amin[k], __fmul_rn(u, amax[k] - amin[k]));
    }
  } else if (i < n_x + n_h) {
    const int64_t t = i - n_x;
    const int64_t r = t / (2 * A), c = t - r * 2 * A;
    head_tiled[t] = head[(r / N) * 2 * A + c];
  }
  if (!u_in) next_rng_call(rng_call);
}

// reward + tf.random.normal(shape, 0, reward_noise_variance): the "variance" is the stddev
// (:832-839).  Nothing is added while stddev_dev[0] <= 0.
__global__ void cql_reward_noise_kernel(const float* __restrict__ reward, int64_t B,
                                        const float* __restrict__ stddev,
                                        const float* __restrict__ z_in, uint64_t seed,
                                        uint64_t* rng_call, float* __restrict__ out) {
  pdl_prologue();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B) {
    const float s = stddev[0];
    const float z = z_in ? z_in[i] : philox_normal((uint64_t)i, rng_call[0], seed);
    out[i] = s > 0.f ? __fadd_rn(reward[i], __fmul_rn(z, s)) : reward[i];
  }
  if (!z_in) next_rng_call(rng_call);
}

// _get_cql_alpha (:752-765): exp(clip_by_value(log_cql_alpha, lo, hi)) with Lagrange, else the
// (user-changeable) device scalar.
__device__ __forceinline__ float cql_alpha_value(const float* cql_alpha, const float* log_cql_alpha,
                                                 float lo, float hi) {
  return log_cql_alpha ? expf(fmaxf(fminf(log_cql_alpha[0], hi), lo)) : cql_alpha[0];
}

struct CqlLossArgs {
  const float* q1; const float* q2;        // [B + 2BN] critic outputs on the joint rows
  const float* logp;                       // [BN] log-probs of the policy candidates
  int64_t B, N;
  float uniform_logp, temperature;
  const float* cql_alpha; const float* log_cql_alpha; float clip_lo, clip_hi;
  int bc_debug;
  float* dq1; float* dq2;                  // [B + 2BN]; rows [0, B) hold the TD gradient
  float* partial;                          // [kCqlRedBlocks]
};

// Candidate j of state b for one critic: tau * Q - log density (:598-637).
__device__ __forceinline__ float cql_logit(const CqlLossArgs& a, const float* q, int64_t b,
                                           int64_t j, int64_t& row) {
  const int64_t BN = a.B * a.N;
  if (j < a.N) {
    row = a.B + b * a.N + j;
    return q[row] * a.temperature - a.logp[b * a.N + j];
  }
  row = a.B + BN + b * a.N + (j - a.N);
  return q[row] * a.temperature - a.uniform_logp;
}

// Per state b and critic i: lse_i = logsumexp_j(logit_ij) / tau over the 2N candidates
// (max-subtracted), d lse_i / d Q_ij = softmax_j.  cql_loss = sum_b [(lse_1 - q1_b) + (lse_2 - q2_b)]
// / (2B) (:651-675), so dQ_candidate = cql_alpha / (2B) * softmax and the data rows get
// -cql_alpha / (2B), added to the TD gradient (overwriting it with bc_debug_mode, :289-292).
// A state is handled by G lanes (G from 2N, as the categorical PPO kernels pick it from A).
template <int G>
__global__ void __launch_bounds__(256) cql_loss_rows_kernel(const CqlLossArgs a) {
  pdl_prologue();
  __shared__ float red[32];
  const float g = cql_alpha_value(a.cql_alpha, a.log_cql_alpha, a.clip_lo, a.clip_hi) /
                  (2.f * (float)a.B);
  const int64_t M = 2 * a.N;
  float acc = 0.f;
  B200RL_GROUP_ROWS(G, a.B) {
    const bool valid = n < a.B;
    const int64_t b = valid ? n : n0;
    float term = 0.f;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const float* q = c ? a.q2 : a.q1;
      float* dq = c ? a.dq2 : a.dq1;
      int64_t row;
      float m = -INFINITY;
      for (int64_t j = lane; j < M; j += G) m = fmaxf(m, cql_logit(a, q, b, j, row));
      m = grp_max<G>(m);
      float s = 0.f;
      for (int64_t j = lane; j < M; j += G) s += expf(cql_logit(a, q, b, j, row) - m);
      s = grp_sum<G>(s);
      term += (m + logf(s)) / a.temperature - q[b];
      if (valid) {
        const float gs = g / s;
        for (int64_t j = lane; j < M; j += G) {
          const float e = expf(cql_logit(a, q, b, j, row) - m);
          dq[row] = gs * e;
        }
      }
    }
    if (valid && lane == 0) {
      acc += term;
      a.dq1[b] = a.bc_debug ? -g : a.dq1[b] - g;
      a.dq2[b] = a.bc_debug ? -g : a.dq2[b] - g;
    }
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) a.partial[blockIdx.x] = acc;
}

// out[0] cql_loss, out[1] cql_alpha, out[2] the critic loss the critic gradient is taken of
// (critic_loss + cql_alpha * cql_loss, or cql_alpha * cql_loss with bc_debug_mode), out[3]
// cql_alpha_loss = -cql_alpha * (cql_loss - cql_tau) with Lagrange (else 0) and its gradient
// w.r.t. log_cql_alpha, which clip_by_value passes inside [lo, hi] (bounds included).
__global__ void __launch_bounds__(256) cql_loss_final_kernel(
    const float* __restrict__ partial, int nb, int64_t B, const float* __restrict__ cql_alpha,
    const float* __restrict__ log_cql_alpha, float lo, float hi, float cql_tau, int bc_debug,
    const float* __restrict__ critic_loss, float* __restrict__ out,
    float* __restrict__ dlog_cql_alpha, int32_t* nan_flag) {
  pdl_prologue();
  __shared__ float red[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) s += partial[i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float cql = s / (2.f * (float)B);
    const float alpha = cql_alpha_value(cql_alpha, log_cql_alpha, lo, hi);
    out[0] = cql;
    out[1] = alpha;
    out[2] = bc_debug ? cql * alpha : critic_loss[0] + cql * alpha;
    float closs = 0.f;
    if (log_cql_alpha) {
      const float la = log_cql_alpha[0];
      closs = -alpha * (cql - cql_tau);
      dlog_cql_alpha[0] = (la >= lo && la <= hi) ? closs : 0.f;
    }
    out[3] = closs;
    if (nan_flag && !(isfinite(cql) && isfinite(closs))) *nan_flag = 1;
  }
}

// log pi(a | s) of the tanh-squashed Normal for one action dimension, with
// z = (atanh(clip(y)) - loc) / std, y = (a - shift) / half (SquashToSpecNormal.log_prob).  As in
// the reference, only |y| <= 1 is clipped: an action outside the spec gives NaN (the nan flag).
__device__ __forceinline__ float bc_logp_dim(float loc, float ls, float a, float lo, float hi,
                                             float& z) {
  const float half = 0.5f * (hi - lo), shift = 0.5f * (hi + lo);
  float y = (a - shift) / half;
  if (fabsf(y) <= 1.f) y = fminf(fmaxf(y, -0.99999997f), 0.99999997f);
  const float u = atanhf(y);
  z = (u - loc) / expf(ls);
  return -0.5f * z * z - ls - 0.5f * kLog2PiS - logf(half) -
         2.f * (kLog2 - u - softplus_f(-2.f * u));
}

// BC branch of actor_loss (:712-718) while train_step < num_bc_steps: per example
// exp(log_alpha) * log pi(a~|s) - log pi(a_data|s); the critics get no gradient.  Past the BC
// phase SAC's loss and gradients are left as they are.
__global__ void __launch_bounds__(256) cql_bc_actor_loss_kernel(
    const float* __restrict__ head, const float* __restrict__ action, int64_t ld_a,
    const float* __restrict__ amin, const float* __restrict__ amax, const float* __restrict__ logp,
    const float* __restrict__ weights, const float* __restrict__ log_alpha,
    const int64_t* __restrict__ train_step, int64_t num_bc_steps, int64_t B, int64_t A,
    float loss_weight, float global_batch, float* __restrict__ loss, float* __restrict__ dq1,
    float* __restrict__ dq2, int32_t* nan_flag) {
  pdl_prologue();
  if (train_step[0] >= num_bc_steps) return;
  __shared__ float red[32];
  const float alpha = expf(log_alpha[0]);
  float s = 0.f;
  for (int64_t b = threadIdx.x; b < B; b += blockDim.x) {
    float lp = 0.f, z;
    for (int64_t k = 0; k < A; ++k)
      lp += bc_logp_dim(head[b * 2 * A + k], head[b * 2 * A + A + k], action[b * ld_a + k],
                        amin[k], amax[k], z);
    const float w = weights ? weights[b] : 1.f;
    const float l = alpha * logp[b] - lp;
    s += (weights && w == 0.f) ? 0.f : l * w;
    dq1[b] = 0.f;
    dq2[b] = 0.f;
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float out = loss_weight * s / global_batch;
    loss[0] = out;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
  }
}

// Adds d(-loss_weight * w * log pi(a_data|s) / global_batch)/dhead to the dhead sac_sample_bwd
// wrote: d log pi / d loc = z / std, d log pi / d log_std = z^2 - 1.
__global__ void cql_bc_actor_bwd_kernel(const float* __restrict__ head,
                                        const float* __restrict__ action, int64_t ld_a,
                                        const float* __restrict__ amin,
                                        const float* __restrict__ amax,
                                        const float* __restrict__ weights,
                                        const int64_t* __restrict__ train_step,
                                        int64_t num_bc_steps, int64_t B, int64_t A,
                                        float loss_weight, float global_batch,
                                        float* __restrict__ dhead) {
  pdl_prologue();
  if (train_step[0] >= num_bc_steps) return;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * A) return;
  const int64_t b = i / A, k = i - b * A;
  const float ls = head[b * 2 * A + A + k];
  float z;
  bc_logp_dim(head[b * 2 * A + k], ls, action[b * ld_a + k], amin[k], amax[k], z);
  const float c = loss_weight * (weights ? weights[b] : 1.f) / global_batch;
  dhead[b * 2 * A + k] -= c * (z / expf(ls));
  dhead[b * 2 * A + A + k] -= c * (z * z - 1.f);
}

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_cql_candidates(const float* obs, int64_t ld_obs, int64_t B, int64_t N, int64_t D,
                          int64_t A, const float* amin, const float* amax, const float* u_in,
                          uint64_t seed, uint64_t* rng_call_dev, const float* head, float* x,
                          float* head_tiled, void* stream) {
  B200RL_CHECK_ARG(obs && amin && amax && head && x && head_tiled && B >= 1 && N >= 1 && D >= 1 &&
                       A >= 1 && ld_obs >= D,
                   "cql_candidates: bad argument");
  B200RL_CHECK_ARG(u_in || rng_call_dev, "cql_candidates: need u_in or rng_call_dev");
  const int64_t n = 2 * B * N * (D + A) + B * N * 2 * A;
  B200RL_LAUNCH(cql_candidates_kernel, blocks_of_256(n), 256, 0, (cudaStream_t)stream, obs, ld_obs, B, N, D, A, amin, amax, u_in, seed, rng_call_dev, head, x, head_tiled);
  B200RL_CHECK_LAUNCH("cql_candidates");
  return B200RL_OK;
}

int b200rl_cql_reward_noise(const float* reward, int64_t B, const float* stddev_dev,
                            const float* z_in, uint64_t seed, uint64_t* rng_call_dev, float* out,
                            void* stream) {
  B200RL_CHECK_ARG(reward && stddev_dev && out && B >= 1, "cql_reward_noise: bad argument");
  B200RL_CHECK_ARG(z_in || rng_call_dev, "cql_reward_noise: need z_in or rng_call_dev");
  B200RL_LAUNCH(cql_reward_noise_kernel, blocks_of_256(B), 256, 0, (cudaStream_t)stream, reward, B, stddev_dev, z_in, seed, rng_call_dev, out);
  B200RL_CHECK_LAUNCH("cql_reward_noise");
  return B200RL_OK;
}

int b200rl_cql_loss(const float* q1, const float* q2, const float* logp, int64_t B, int64_t N,
                    float uniform_logp, float temperature, const float* cql_alpha_dev,
                    const float* log_cql_alpha_dev, float clip_lo, float clip_hi, float cql_tau,
                    int bc_debug, const float* critic_loss, float* dq1, float* dq2, float* out,
                    float* dlog_cql_alpha, int32_t* nan_flag, void* workspace, int64_t ws_bytes,
                    void* stream) {
  B200RL_CHECK_ARG(q1 && q2 && logp && critic_loss && dq1 && dq2 && out && B >= 1 && N >= 1 &&
                       temperature > 0.f,
                   "cql_loss: bad argument");
  B200RL_CHECK_ARG(cql_alpha_dev || log_cql_alpha_dev, "cql_loss: need cql_alpha or log_cql_alpha");
  B200RL_CHECK_ARG(!log_cql_alpha_dev || dlog_cql_alpha, "cql_loss: Lagrange needs dlog_cql_alpha");
  B200RL_CHECK_ARG(workspace && ws_bytes >= (int64_t)(kCqlRedBlocks * sizeof(float)),
                   "cql_loss: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  CqlLossArgs a;
  a.q1 = q1; a.q2 = q2; a.logp = logp; a.B = B; a.N = N;
  a.uniform_logp = uniform_logp; a.temperature = temperature;
  a.cql_alpha = cql_alpha_dev; a.log_cql_alpha = log_cql_alpha_dev;
  a.clip_lo = clip_lo; a.clip_hi = clip_hi; a.bc_debug = bc_debug;
  a.dq1 = dq1; a.dq2 = dq2; a.partial = (float*)workspace;
  const int G = lane_group(2 * N);
  const unsigned nb = group_blocks(B, G, kCqlRedBlocks);
  if (G == 1) B200RL_LAUNCH(cql_loss_rows_kernel<1>, nb, 256, 0, st, a);
  else if (G == 8) B200RL_LAUNCH(cql_loss_rows_kernel<8>, nb, 256, 0, st, a);
  else B200RL_LAUNCH(cql_loss_rows_kernel<32>, nb, 256, 0, st, a);
  B200RL_CHECK_LAUNCH("cql_loss_rows");
  B200RL_LAUNCH(cql_loss_final_kernel, 1, 256, 0, st, (const float*)workspace, (int)nb, B, cql_alpha_dev, log_cql_alpha_dev, clip_lo, clip_hi, cql_tau, bc_debug, critic_loss, out, dlog_cql_alpha, nan_flag);
  B200RL_CHECK_LAUNCH("cql_loss_final");
  return B200RL_OK;
}

int b200rl_cql_bc_actor_loss(const float* head, const float* action, int64_t ld_action,
                             const float* amin, const float* amax, const float* logp,
                             const float* weights, const float* log_alpha_dev,
                             const int64_t* train_step_dev, int64_t num_bc_steps, int64_t B,
                             int64_t A, float loss_weight, float global_batch, float* loss,
                             float* dq1, float* dq2, int32_t* nan_flag, void* stream) {
  B200RL_CHECK_ARG(head && action && amin && amax && logp && log_alpha_dev && train_step_dev &&
                       loss && dq1 && dq2 && B >= 1 && A >= 1 && ld_action >= A &&
                       global_batch > 0.f,
                   "cql_bc_actor_loss: bad argument");
  B200RL_LAUNCH(cql_bc_actor_loss_kernel, 1, 256, 0, (cudaStream_t)stream, head, action, ld_action, amin, amax, logp, weights, log_alpha_dev, train_step_dev, num_bc_steps, B, A, loss_weight, global_batch, loss, dq1, dq2, nan_flag);
  B200RL_CHECK_LAUNCH("cql_bc_actor_loss");
  return B200RL_OK;
}

int b200rl_cql_bc_actor_bwd(const float* head, const float* action, int64_t ld_action,
                            const float* amin, const float* amax, const float* weights,
                            const int64_t* train_step_dev, int64_t num_bc_steps, int64_t B,
                            int64_t A, float loss_weight, float global_batch, float* dhead,
                            void* stream) {
  B200RL_CHECK_ARG(head && action && amin && amax && train_step_dev && dhead && B >= 1 &&
                       A >= 1 && ld_action >= A && global_batch > 0.f,
                   "cql_bc_actor_bwd: bad argument");
  B200RL_LAUNCH(cql_bc_actor_bwd_kernel, blocks_of_256(B * A), 256, 0, (cudaStream_t)stream, head, action, ld_action, amin, amax, weights, train_step_dev, num_bc_steps, B, A, loss_weight, global_batch, dhead);
  B200RL_CHECK_LAUNCH("cql_bc_actor_bwd");
  return B200RL_OK;
}

}  // extern "C"
