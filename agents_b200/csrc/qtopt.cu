// QT-Opt: the cross-entropy-method (CEM) action search of CEMPolicy, the QT-Opt TD loss and the
// continuous epsilon-greedy / uniform draw of EpsilonGreedyPolicy and RandomTFPolicy.
//
// Restates policies/qtopt_cem_policy.py (actor_func :232-399, _score :416-465), the
// GaussianActionsSampler of policies/samplers/qtopt_cem_actions_sampler_continuous.py
// (sample_batch_and_clip, refit_distribution_to with tf.nn.moments), agents/qtopt/qtopt_agent.py
// (_loss :588-698) and, for float action specs, policies/epsilon_greedy_policy.py with
// tensor_spec.sample_spec_nest.
//
// One search over B states with N samples, M elites and I iterations is one cem_sample launch,
// then I x (critic forward over the B*N rows + one cem_refit launch).  The samples live only in
// the action columns of the critic's [B*N, W] joint-stack input; rows follow tile_batch order
// (sample n of state b is row b*N + n), and draw (row, k) uses Philox element row*A + k.
#include <limits.h>
#include <math.h>

#include "common.cuh"

namespace b200rl {

constexpr int kCemWarps = 4;               // states per cem_refit block
// shared words per warp (elite indices, mean, var) within the default 48 KB per block
constexpr int kCemSmemWords = 3072;
constexpr uint64_t kUniformTag = 0x51544F50554E4946ull;

__device__ __forceinline__ float cem_draw(float mean, float var, float minimal_var, float lo,
                                          float hi, const float* z_in, int64_t e, uint64_t call,
                                          uint64_t seed) {
  const float z = z_in ? z_in[e] : philox_normal((uint64_t)e, call, seed);
  const float a = mean + sqrtf(fmaxf(var, minimal_var)) * z;
  return fminf(fmaxf(a, lo), hi);
}

// x[r, c] for r < B*N, c < C + A: the source row r / N for c < C (the observation, or h_obs with
// an observation branch), a clipped N(mean, max(var, minimal_var)) draw for the action column
// c - C.  ld_mean = ld_var = 0 broadcasts one [A] initial distribution to every state.
__global__ void cem_sample_kernel(const float* __restrict__ src, int64_t ld_src, int64_t B,
                                  int64_t N, int64_t C, int64_t A, const float* __restrict__ mean,
                                  int64_t ld_mean, const float* __restrict__ var, int64_t ld_var,
                                  float minimal_var, const float* __restrict__ amin,
                                  const float* __restrict__ amax, const float* __restrict__ z_in,
                                  uint64_t seed, uint64_t* rng_call, float* __restrict__ x,
                                  int64_t ld_x) {
  pdl_prologue();
  const int64_t W = C + A;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t call = z_in ? 0 : rng_call[0];
  if (i < B * N * W) {
    const int64_t r = i / W, c = i - r * W, b = r / N;
    if (c < C) {
      x[r * ld_x + c] = src[b * ld_src + c];
    } else {
      const int64_t k = c - C;
      x[r * ld_x + c] = cem_draw(mean[b * ld_mean + k], var[b * ld_var + k], minimal_var, amin[k],
                                 amax[k], z_in, r * A + k, call, seed);
    }
  }
  if (!z_in) next_rng_call(rng_call);
}

// (v, i) ranks before (w, j): larger score first, the lower index on a tie (tf.nn.top_k).  NaN
// scores rank as -inf.
__device__ __forceinline__ bool ranks_before(float v, int i, float w, int j) {
  return v > w || (v == w && i < j);
}

// One warp per state b.  Elite j is the best sample ranked after elite j - 1, found by one warp
// scan of the N scores per elite (no per-state storage but the M indices).  mean and var are
// refitted over the elites in rank order (tf.nn.moments: the mean first, then the mean of squared
// deviations, both divided by M).  Unless `last`, the next N samples are drawn into the action
// columns; on the last iteration the best sample and its score are written instead.  With
// elite_idx [B, M] the selection is skipped and those samples (clamped to [0, N)) are refitted.
__global__ void __launch_bounds__(kCemWarps * 32) cem_refit_kernel(
    const float* __restrict__ scores, const int32_t* __restrict__ elite_idx, float* x, int64_t ld_x,
    int64_t col, int64_t B, int64_t N, int64_t M, int64_t A, float minimal_var,
    const float* __restrict__ amin, const float* __restrict__ amax, int last,
    const float* __restrict__ z_in, uint64_t seed, uint64_t* rng_call, float* __restrict__ mean,
    float* __restrict__ var, float* __restrict__ best_action, float* __restrict__ best_score) {
  pdl_prologue();
  extern __shared__ unsigned char cem_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t per_warp = M + 2 * A;                    // 4-byte words
  int32_t* idx = (int32_t*)cem_smem + warp * per_warp;
  float* smean = (float*)(idx + M);
  float* svar = smean + A;
  const bool draw = !last;
  const uint64_t call = (draw && !z_in) ? rng_call[0] : 0;
  const int64_t b = (int64_t)blockIdx.x * kCemWarps + warp;
  if (b < B) {
    const int64_t r0 = b * N;
    if (elite_idx) {
      for (int64_t j = lane; j < M; j += 32) {
        const int32_t e = elite_idx[b * M + j];
        idx[j] = e < 0 ? 0 : (e >= N ? (int32_t)(N - 1) : e);
      }
    } else {
      float pv = INFINITY;
      int pi = -1;
      for (int64_t j = 0; j < M; ++j) {
        float bv = -INFINITY;
        int bi = INT_MAX;
        for (int64_t n = lane; n < N; n += 32) {
          float v = scores[r0 + n];
          if (isnan(v)) v = -INFINITY;
          if (ranks_before(pv, pi, v, (int)n) && ranks_before(v, (int)n, bv, bi)) {
            bv = v;
            bi = (int)n;
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
          const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
          if (ranks_before(ov, oi, bv, bi)) {
            bv = ov;
            bi = oi;
          }
        }
        if (lane == 0) idx[j] = bi;
        pv = bv;
        pi = bi;
      }
    }
    __syncwarp();
    const float fm = (float)M;
    for (int64_t k = lane; k < A; k += 32) {
      float s = 0.f;
      for (int64_t j = 0; j < M; ++j) s += x[(r0 + idx[j]) * ld_x + col + k];
      const float mu = s / fm;
      float q = 0.f;
      for (int64_t j = 0; j < M; ++j) {
        const float d = x[(r0 + idx[j]) * ld_x + col + k] - mu;
        q += d * d;
      }
      const float v = q / fm;
      smean[k] = mu;
      svar[k] = v;
      mean[b * A + k] = mu;
      var[b * A + k] = v;
      if (last && best_action) best_action[b * A + k] = x[(r0 + idx[0]) * ld_x + col + k];
    }
    if (last && best_score && lane == 0) best_score[b] = scores[r0 + idx[0]];
    __syncwarp();                                        // every elite is read before a redraw
    if (draw) {
      for (int64_t t = lane; t < N * A; t += 32) {
        const int64_t n = t / A, k = t - n * A, r = r0 + n;
        x[r * ld_x + col + k] = cem_draw(smean[k], svar[k], minimal_var, amin[k], amax[k], z_in,
                                         r * A + k, call, seed);
      }
    }
  }
  if (draw && !z_in) next_rng_call(rng_call);
}

// next_q = min(tq1, tq2) (tq1 alone when tq2 is NULL); y = reward_scale r + gamma d next_q;
// m = step_type != LAST; td_error = m (y - q); td_loss = m l(y, q);
// loss = sum_b w_b td_loss_b / B; dq = m w_b / B dl/dq.  One block, fixed order.
__global__ void __launch_bounds__(1024) qtopt_td_loss_kernel(
    const float* __restrict__ q, const float* __restrict__ tq1, const float* __restrict__ tq2,
    const float* __restrict__ reward, const float* __restrict__ discount,
    const int32_t* __restrict__ step_type, int64_t step_stride, const float* __restrict__ weights,
    int64_t B, float gamma, float reward_scale, int loss_kind, float* __restrict__ loss,
    float* __restrict__ td_loss, float* __restrict__ td_error, float* __restrict__ dq,
    int32_t* nan_flag) {
  pdl_prologue();
  __shared__ float red[32];
  const float inv_b = 1.f / (float)B;
  float s = 0.f;
  for (int64_t b = threadIdx.x; b < B; b += blockDim.x) {
    const float nq = tq2 ? fminf(tq2[b], tq1[b]) : tq1[b];
    const float y = reward_scale * reward[b] + gamma * discount[b] * nq;
    const float m = step_type[b * step_stride] == 2 ? 0.f : 1.f;
    const float e = y - q[b];
    float l, g;
    td_elem_loss(e, loss_kind, l, g);
    const float w = weights ? weights[b] : 1.f;
    td_error[b] = m * e;
    td_loss[b] = m * l;
    s += m * l * w;
    dq[b] = m * g * (w * inv_b);
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float out = s / (float)B;
    loss[0] = out;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
  }
}

// Row n of action [N, A] is replaced, where u_n < epsilon, by lo + u (hi - lo) per column
// (tf.random.uniform over the bounded spec).  u_n = uniform(Philox(n, call, seed).x); the column
// draws use element n*A + k under a second key.  epsilon >= 1 replaces every row.
__global__ void epsilon_uniform_kernel(float* __restrict__ action, int64_t ld, int64_t N,
                                       int64_t A, float epsilon, const float* __restrict__ amin,
                                       const float* __restrict__ amax, uint64_t seed,
                                       uint64_t* rng_call) {
  pdl_prologue();
  const uint64_t call = rng_call[0];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N * A) {
    const int64_t n = i / A, k = i - n * A;
    const float u = uniform_f32(philox4x32_10((uint64_t)n, call, seed).x);
    if (u < epsilon) {
      const float v = uniform_f32(philox4x32_10((uint64_t)i, call, seed ^ kUniformTag).x);
      action[n * ld + k] = __fadd_rn(amin[k], __fmul_rn(v, amax[k] - amin[k]));
    }
  }
  next_rng_call(rng_call);
}

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_cem_sample(const float* src, int64_t ld_src, int64_t B, int64_t N, int64_t C,
                      int64_t A, const float* mean, int64_t ld_mean, const float* var,
                      int64_t ld_var, float minimal_var, const float* amin, const float* amax,
                      const float* z_in, uint64_t seed, uint64_t* rng_call_dev, float* x,
                      int64_t ld_x, void* stream) {
  B200RL_CHECK_ARG(mean && var && amin && amax && x && B >= 1 && N >= 1 && C >= 0 && A >= 1 &&
                       ld_mean >= 0 && ld_var >= 0 && ld_x >= C + A && (C == 0 || src) &&
                       ld_src >= C,
                   "cem_sample: bad argument");
  B200RL_CHECK_ARG(z_in || rng_call_dev, "cem_sample: need z_in or rng_call_dev");
  B200RL_CHECK_ARG(minimal_var >= 0.f, "cem_sample: negative minimal_var");
  B200RL_LAUNCH(cem_sample_kernel, blocks_of_256(B * N * (C + A)), 256, 0, (cudaStream_t)stream, src, ld_src, B, N, C, A, mean, ld_mean, var, ld_var, minimal_var, amin, amax, z_in, seed, rng_call_dev, x, ld_x);
  B200RL_CHECK_LAUNCH("cem_sample");
  return B200RL_OK;
}

int b200rl_cem_refit(const float* scores, const int32_t* elite_idx, float* x, int64_t ld_x,
                     int64_t col, int64_t B, int64_t N, int64_t M, int64_t A, float minimal_var,
                     const float* amin, const float* amax, int last, const float* z_in,
                     uint64_t seed, uint64_t* rng_call_dev, float* mean, float* var,
                     float* best_action, float* best_score, void* stream) {
  B200RL_CHECK_ARG(x && mean && var && B >= 1 && N >= 1 && A >= 1 && col >= 0 &&
                       ld_x >= col + A && N <= INT_MAX,
                   "cem_refit: bad argument");
  B200RL_CHECK_ARG(M >= 1 && M <= N && M + 2 * A <= kCemSmemWords,
                   "cem_refit: need 1 <= M <= N and M + 2A <= %d (M=%lld N=%lld A=%lld)",
                   kCemSmemWords, (long long)M, (long long)N, (long long)A);
  B200RL_CHECK_ARG(scores || elite_idx, "cem_refit: need scores or elite_idx");
  B200RL_CHECK_ARG(last || (amin && amax && (z_in || rng_call_dev)),
                   "cem_refit: drawing needs amin, amax and z_in or rng_call_dev");
  B200RL_CHECK_ARG(!(last && best_score && !scores), "cem_refit: best_score needs scores");
  B200RL_CHECK_ARG(minimal_var >= 0.f, "cem_refit: negative minimal_var");
  const size_t smem = (size_t)kCemWarps * (size_t)(M + 2 * A) * 4;
  B200RL_LAUNCH(cem_refit_kernel, (unsigned)((B + kCemWarps - 1) / kCemWarps), kCemWarps * 32, smem, (cudaStream_t)stream, scores, elite_idx, x, ld_x, col, B, N, M, A, minimal_var, amin, amax, last, z_in, seed, rng_call_dev, mean, var, best_action, best_score);
  B200RL_CHECK_LAUNCH("cem_refit");
  return B200RL_OK;
}

int b200rl_qtopt_td_loss(const float* q, const float* tq1, const float* tq2, const float* reward,
                         const float* discount, const int32_t* step_type, int64_t step_stride,
                         const float* weights, int64_t B, float gamma, float reward_scale,
                         int loss_kind, float* loss, float* td_loss, float* td_error, float* dq,
                         int32_t* nan_flag, void* stream) {
  B200RL_CHECK_ARG(q && tq1 && reward && discount && step_type && loss && td_loss && td_error &&
                       dq && B >= 1 && step_stride >= 1,
                   "qtopt_td_loss: bad argument");
  B200RL_CHECK_ARG(loss_kind == B200RL_LOSS_HUBER || loss_kind == B200RL_LOSS_SQUARED,
                   "qtopt_td_loss: unknown loss kind");
  B200RL_LAUNCH(qtopt_td_loss_kernel, 1, reduce_threads(B), 0, (cudaStream_t)stream, q, tq1, tq2, reward, discount, step_type, step_stride, weights, B, gamma, reward_scale, loss_kind, loss, td_loss, td_error, dq, nan_flag);
  B200RL_CHECK_LAUNCH("qtopt_td_loss");
  return B200RL_OK;
}

int b200rl_epsilon_uniform(float* action, int64_t ld, int64_t N, int64_t A, float epsilon,
                           const float* amin, const float* amax, uint64_t seed,
                           uint64_t* rng_call_dev, void* stream) {
  B200RL_CHECK_ARG(action && amin && amax && rng_call_dev && N >= 1 && A >= 1 && ld >= A,
                   "epsilon_uniform: bad argument");
  B200RL_LAUNCH(epsilon_uniform_kernel, blocks_of_256(N * A), 256, 0, (cudaStream_t)stream, action, ld, N, A, epsilon, amin, amax, seed, rng_call_dev);
  B200RL_CHECK_LAUNCH("epsilon_uniform");
  return B200RL_OK;
}

}  // extern "C"
