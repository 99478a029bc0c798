// Behavioral-cloning losses: sparse softmax cross-entropy over logits (discrete actions) and the
// mean squared error of a predicted action (continuous actions), with their gradients and the
// aggregation of agents/behavioral_cloning/behavioral_cloning_agent.py.
//
// Both restate common.aggregate_losses with tf.math.multiply_no_nan: loss = sum_n w_n pe_n / N
// over the N = B (or B*T) rows, where a row with w_n = 0 adds exactly 0 and gets an all-zero
// gradient even when its loss is inf or NaN.  The per-example loss pe_n is written unweighted.
// A row of A columns is handled by a group of G lanes (lane_group, common.cuh); each block writes
// one partial sum and one 512-thread block reduces the partials in a fixed order, so eager runs
// and graph replays give the same bits.
#include <math.h>

#include "common.cuh"

namespace b200rl {

constexpr int kBcRedBlocks = 512;

// w_n = weights[n / w_div] (w_div = 1: per row, T: per batch entry, N: a scalar); NULL: 1.
__device__ __forceinline__ float bc_weight(const float* __restrict__ weights, int64_t w_div,
                                           int64_t n) {
  return weights ? weights[n / w_div] : 1.f;
}

// pe_n = log sum_j exp(z_j) - z_label, label = action[n * a_stride] - minimum.
// dlogits[n, j] = w_n / N (softmax_j - [j = label]).  A label outside [0, A) sets nan_flag and
// pe_n = NaN; its gradient row is computed against the clamped label.
template <int G>
__global__ void __launch_bounds__(256) bc_discrete_kernel(
    const float* __restrict__ logits, int64_t ld, const int32_t* __restrict__ action,
    int64_t a_stride, int32_t minimum, const float* __restrict__ weights, int64_t w_div,
    int64_t N, int64_t A, float* __restrict__ per_example, float* __restrict__ dlogits,
    int64_t ld_g, float* __restrict__ partial, int32_t* nan_flag) {
  pdl_prologue();
  __shared__ float red[32];
  const float inv_n = 1.f / (float)N;
  float acc = 0.f;
  B200RL_GROUP_ROWS(G, N) {
    const bool valid = n < N;
    const int64_t r = valid ? n : n0;
    const float* z = logits + r * ld;
    const int32_t raw = action[r * a_stride] - minimum;
    const bool bad = raw < 0 || raw >= A;
    const int label = clamp_action(raw, A, valid ? nan_flag : nullptr);
    float m, s, t;
    row_softmax_stats<G>(z, A, lane, m, s, t);
    const float log_s = logf(s);
    const float pe = bad ? NAN : log_s - (z[label] - m);
    const float w = bc_weight(weights, w_div, r);
    if (valid) {
      if (lane == 0) {
        per_example[r] = pe;
        acc += w == 0.f ? 0.f : w * pe;
      }
      const float g = w * inv_n;
      for (int64_t j = lane; j < A; j += G) {
        const float p = expf((z[j] - m) - log_s);
        dlogits[r * ld_g + j] = w == 0.f ? 0.f : g * (p - (j == label ? 1.f : 0.f));
      }
    }
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = acc;
}

// pe_n = mean_k (a_nk - t_nk)^2.
// Deterministic (scale == NULL): a = scale_to_spec(y) = 0.5 (max + min) + 0.5 (max - min) y, and
//   dpred = mag_k * 2 w_n (a - t) / (N A), the gradient w.r.t. the tanh output y.
// Normal: a = loc + scale * z with z = noise_in[n * A + k], or Philox + Box-Muller on element
//   n * A + k of the call rng_call[0] (normal_sample_kernel's stream, not clipped);
//   dpred = dloc = 2 w_n (a - t) / (N A), dscale = dloc * z.
template <int G>
__global__ void __launch_bounds__(256) bc_continuous_kernel(
    const float* __restrict__ pred, const float* __restrict__ scale, int64_t ld,
    const float* __restrict__ target, int64_t ld_t, const float* __restrict__ amin,
    const float* __restrict__ amax, const float* __restrict__ noise_in, uint64_t seed,
    const uint64_t* __restrict__ rng_call, const float* __restrict__ weights, int64_t w_div,
    int64_t N, int64_t A, float* __restrict__ per_example, float* __restrict__ dpred,
    float* __restrict__ dscale, int64_t ld_g, float* __restrict__ partial) {
  pdl_prologue();
  __shared__ float red[32];
  const uint64_t call = (scale && !noise_in) ? rng_call[0] : 0;
  const float inv_a = 1.f / (float)A;
  const float inv_na = 1.f / ((float)N * (float)A);
  float acc = 0.f;
  B200RL_GROUP_ROWS(G, N) {
    const bool valid = n < N;
    const int64_t r = valid ? n : n0;
    const float w = bc_weight(weights, w_div, r);
    const float g = 2.f * w * inv_na;
    float se = 0.f;
    for (int64_t k = lane; k < A; k += G) {
      const float p = pred[r * ld + k];
      float a, z = 0.f, dmul;
      if (scale) {
        z = noise_in ? noise_in[r * A + k] : philox_normal((uint64_t)(r * A + k), call, seed);
        a = p + scale[r * ld + k] * z;
        dmul = 1.f;
      } else {
        const float lo = amin[k], hi = amax[k];
        a = 0.5f * (hi + lo) + 0.5f * (hi - lo) * p;
        dmul = 0.5f * (hi - lo);
      }
      const float d = a - target[r * ld_t + k];
      se += d * d;
      if (valid) {
        const float gd = w == 0.f ? 0.f : g * d;
        dpred[r * ld_g + k] = dmul * gd;
        if (scale) dscale[r * ld_g + k] = gd * z;
      }
    }
    se = grp_sum<G>(se);
    if (valid && lane == 0) {
      const float pe = se * inv_a;
      per_example[r] = pe;
      acc += w == 0.f ? 0.f : w * pe;
    }
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = acc;
}

// loss[0] = sum of the partials / N, in a fixed order.  With advance_rng the Philox call counter
// moves on after every partial block has read it.
__global__ void __launch_bounds__(512) bc_loss_final_kernel(const float* __restrict__ partial,
                                                            int nblocks, float n,
                                                            float* __restrict__ loss,
                                                            int32_t* nan_flag,
                                                            uint64_t* rng_call) {
  pdl_prologue();
  __shared__ float red[32];
  const float s = block_sum(threadIdx.x < nblocks ? partial[threadIdx.x] : 0.f, red);
  if (threadIdx.x == 0) {
    const float out = s / n;
    loss[0] = out;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
    if (rng_call) rng_call[0] = rng_call[0] + 1;
  }
}

}  // namespace b200rl

using namespace b200rl;

static bool bc_weight_layout_ok(const float* weights, int64_t w_div, int64_t N) {
  return weights == nullptr || (w_div >= 1 && N % w_div == 0);
}

extern "C" {

int b200rl_bc_discrete_loss(const float* logits, int64_t ld, const int32_t* action,
                            int64_t action_stride, int32_t minimum, const float* weights,
                            int64_t w_div, int64_t N, int64_t A, float* loss, float* per_example,
                            float* dlogits, int64_t ld_g, int32_t* nan_flag, void* workspace,
                            int64_t ws_bytes, void* stream) {
  B200RL_CHECK_ARG(logits && action && loss && per_example && dlogits,
                   "bc_discrete_loss: NULL argument");
  B200RL_CHECK_ARG(N >= 1 && A >= 1 && ld >= A && ld_g >= A && action_stride >= 1,
                   "bc_discrete_loss: bad sizes");
  B200RL_CHECK_ARG(bc_weight_layout_ok(weights, w_div, N), "bc_discrete_loss: bad weight layout");
  B200RL_CHECK_ARG(workspace && ws_bytes >= (int64_t)(kBcRedBlocks * sizeof(float)),
                   "bc_discrete_loss: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  float* part = (float*)workspace;
  const int G = lane_group(A);
  const unsigned nb = group_blocks(N, G, kBcRedBlocks);
  if (G == 1) B200RL_LAUNCH(bc_discrete_kernel<1>, nb, 256, 0, st, logits, ld, action, action_stride, minimum, weights, w_div, N, A, per_example, dlogits, ld_g, part, nan_flag);
  else if (G == 8) B200RL_LAUNCH(bc_discrete_kernel<8>, nb, 256, 0, st, logits, ld, action, action_stride, minimum, weights, w_div, N, A, per_example, dlogits, ld_g, part, nan_flag);
  else B200RL_LAUNCH(bc_discrete_kernel<32>, nb, 256, 0, st, logits, ld, action, action_stride, minimum, weights, w_div, N, A, per_example, dlogits, ld_g, part, nan_flag);
  B200RL_CHECK_LAUNCH("bc_discrete_loss");
  B200RL_LAUNCH(bc_loss_final_kernel, 1, 512, 0, st, (const float*)part, (int)nb, (float)N, loss, nan_flag, (uint64_t*)nullptr);
  B200RL_CHECK_LAUNCH("bc_loss_final");
  return B200RL_OK;
}

int b200rl_bc_continuous_loss(const float* pred, const float* scale, int64_t ld,
                              const float* target, int64_t ld_t, const float* amin,
                              const float* amax, const float* noise_in, uint64_t seed,
                              uint64_t* rng_call_dev, int advance_rng, const float* weights,
                              int64_t w_div, int64_t N, int64_t A, float* loss,
                              float* per_example, float* dpred, float* dscale, int64_t ld_g,
                              int32_t* nan_flag, void* workspace, int64_t ws_bytes,
                              void* stream) {
  B200RL_CHECK_ARG(pred && target && loss && per_example && dpred,
                   "bc_continuous_loss: NULL argument");
  B200RL_CHECK_ARG(N >= 1 && A >= 1 && ld >= A && ld_t >= A && ld_g >= A,
                   "bc_continuous_loss: bad sizes");
  if (scale) {
    B200RL_CHECK_ARG(dscale, "bc_continuous_loss: a Normal prediction needs dscale");
    B200RL_CHECK_ARG(noise_in || rng_call_dev, "bc_continuous_loss: need noise_in or rng_call_dev");
  } else {
    B200RL_CHECK_ARG(amin && amax, "bc_continuous_loss: a deterministic prediction needs amin/amax");
  }
  B200RL_CHECK_ARG(!advance_rng || (scale && rng_call_dev && !noise_in),
                   "bc_continuous_loss: advance_rng needs device draws");
  B200RL_CHECK_ARG(bc_weight_layout_ok(weights, w_div, N),
                   "bc_continuous_loss: bad weight layout");
  B200RL_CHECK_ARG(workspace && ws_bytes >= (int64_t)(kBcRedBlocks * sizeof(float)),
                   "bc_continuous_loss: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  float* part = (float*)workspace;
  const int G = lane_group(A);
  const unsigned nb = group_blocks(N, G, kBcRedBlocks);
  if (G == 1) B200RL_LAUNCH(bc_continuous_kernel<1>, nb, 256, 0, st, pred, scale, ld, target, ld_t, amin, amax, noise_in, seed, (const uint64_t*)rng_call_dev, weights, w_div, N, A, per_example, dpred, dscale, ld_g, part);
  else if (G == 8) B200RL_LAUNCH(bc_continuous_kernel<8>, nb, 256, 0, st, pred, scale, ld, target, ld_t, amin, amax, noise_in, seed, (const uint64_t*)rng_call_dev, weights, w_div, N, A, per_example, dpred, dscale, ld_g, part);
  else B200RL_LAUNCH(bc_continuous_kernel<32>, nb, 256, 0, st, pred, scale, ld, target, ld_t, amin, amax, noise_in, seed, (const uint64_t*)rng_call_dev, weights, w_div, N, A, per_example, dpred, dscale, ld_g, part);
  B200RL_CHECK_LAUNCH("bc_continuous_loss");
  B200RL_LAUNCH(bc_loss_final_kernel, 1, 512, 0, st, (const float*)part, (int)nb, (float)N, loss, nan_flag, advance_rng ? rng_call_dev : (uint64_t*)nullptr);
  B200RL_CHECK_LAUNCH("bc_loss_final");
  return B200RL_OK;
}

}  // extern "C"
