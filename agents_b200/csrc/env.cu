// Batched environment step + action selection, HBM-resident (kernel family i).
//
// The reference steps Python environments through tf.numpy_function
// (environments/tf_py_environment.py:275-326) once per loop iteration of
// drivers/dynamic_step_driver.py:117-174; here the whole batch of environments is a set of
// device arrays advanced by one launch, and the epsilon-greedy choice
// (policies/epsilon_greedy_policy.py:120-145) is one more.
#include <math.h>

#include "common.cuh"

namespace b200rl {

constexpr int kFirst = 0, kMid = 1, kLast = 2;   // trajectories/time_step.py:113-121
constexpr uint64_t kStateDomain = 1ull << 62;    // Philox element index domain for per-env draws

// rng_call layout: uint64[2] = {call index, ticket (low 32 bits used)}.
__global__ void __launch_bounds__(256) eps_greedy_kernel(const float* __restrict__ q,
                                                         const int32_t* __restrict__ mask,
                                                         int64_t B, int64_t A, float eps,
                                                         uint64_t seed, uint64_t* rng_call,
                                                         const float* __restrict__ u_in,
                                                         const int32_t* __restrict__ rand_in,
                                                         int32_t* __restrict__ out) {
  pdl_prologue();
  const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) {
    // greedy: Categorical(logits).mode() == first argmax; masked logits -> dtype.min
    int best = 0;
    float bv = 0.f;
    int allowed = 0;
    for (int a = 0; a < A; ++a) {
      const bool ok = !mask || mask[b * A + a] != 0;
      allowed += ok ? 1 : 0;
      const float v = ok ? q[b * A + a] : -3.4028234663852886e38f;
      if (a == 0 || v > bv) { bv = v; best = a; }
    }
    float u;
    int rnd;
    if (u_in) {
      u = u_in[b];
      rnd = rand_in[b];
    } else {
      const Philox4 r = philox4x32_10((uint64_t)b, rng_call[0], seed);
      u = uniform_f32(r.x);
      if (!mask) {
        rnd = (int)(r.y % (uint32_t)A);
      } else {
        int kth = allowed > 0 ? (int)(r.y % (uint32_t)allowed) : 0;
        rnd = 0;
        for (int a = 0; a < A; ++a)
          if (mask[b * A + a] != 0) {
            if (kth == 0) { rnd = a; break; }
            --kth;
          }
      }
    }
    out[b] = (u >= eps) ? best : rnd;  // tf.where(rng >= epsilon, greedy, random)
  }
  if (!u_in) next_rng_call(rng_call);
}

// grid = (chunks, B).  Each thread fills 16 B of observation from one Philox block.
__global__ void __launch_bounds__(256) env_random_step_kernel(
    int32_t* __restrict__ step_type, int32_t* __restrict__ out_step_type, void* __restrict__ obs,
    int64_t obs_elems, int obs_is_u8, float* __restrict__ reward, float* __restrict__ discount,
    int64_t B, float p_term, uint64_t seed, uint64_t* rng_call) {
  pdl_prologue();
  const int64_t b = blockIdx.y;
  const uint64_t call = rng_call[0];
  const int64_t vec_per_env = obs_is_u8 ? (obs_elems + 15) / 16 : (obs_elems + 3) / 4;
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < vec_per_env) {
    const Philox4 r = philox4x32_10((uint64_t)(b * vec_per_env + j), call, seed);
    if (obs_is_u8) {
      uint8_t* o = (uint8_t*)obs + b * obs_elems + j * 16;
      const uint32_t w[4] = {r.x, r.y, r.z, r.w};
      if (j * 16 + 16 <= obs_elems && (obs_elems % 16) == 0) {
        *reinterpret_cast<uint4*>(o) = make_uint4(w[0], w[1], w[2], w[3]);
      } else {
        for (int i = 0; i < 16 && j * 16 + i < obs_elems; ++i)
          o[i] = (uint8_t)(w[i >> 2] >> (8 * (i & 3)));
      }
    } else {
      float* o = (float*)obs + b * obs_elems + j * 4;
      const uint32_t w[4] = {r.x, r.y, r.z, r.w};
      for (int i = 0; i < 4 && j * 4 + i < obs_elems; ++i)
        o[i] = (float)(w[i] >> 8) * (1.0f / 8388608.0f) - 1.0f;  // U[-1,1)
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const Philox4 r = philox4x32_10(kStateDomain + (uint64_t)b, call, seed);
    const int32_t st = step_type[b];
    int32_t nst;
    if (st == kLast) {  // auto-reset: ts.restart (time_step.py:135-195)
      nst = kFirst;
      reward[b] = 0.f;
      discount[b] = 1.f;
    } else {
      reward[b] = uniform_f32(r.x);
      const bool term = uniform_f32(r.y) < p_term;
      nst = term ? kLast : kMid;  // ts.termination / ts.transition
      discount[b] = term ? 0.f : 1.f;
    }
    step_type[b] = nst;
    if (out_step_type) out_step_type[b] = nst;
  }
  next_rng_call(rng_call);
}

__global__ void __launch_bounds__(256) env_cartpole_step_kernel(
    float* __restrict__ state, int32_t* __restrict__ steps, int32_t* __restrict__ step_type,
    const int32_t* __restrict__ action, float* __restrict__ obs, float* __restrict__ reward,
    float* __restrict__ discount, int64_t B, int32_t max_steps, uint64_t seed,
    uint64_t* rng_call) {
  pdl_prologue();
  const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) {
    float x = state[b * 4 + 0], xd = state[b * 4 + 1], th = state[b * 4 + 2], thd = state[b * 4 + 3];
    const int32_t st = step_type[b];
    if (st == kLast) {
      const Philox4 r = philox4x32_10((uint64_t)b, rng_call[0], seed);
      x = uniform_f32(r.x) * 0.1f - 0.05f;
      xd = uniform_f32(r.y) * 0.1f - 0.05f;
      th = uniform_f32(r.z) * 0.1f - 0.05f;
      thd = uniform_f32(r.w) * 0.1f - 0.05f;
      steps[b] = 0;
      step_type[b] = kFirst;
      reward[b] = 0.f;
      discount[b] = 1.f;
    } else {
      const float gravity = 9.8f, masspole = 0.1f, total_mass = 1.1f, length = 0.5f;
      const float polemass_length = 0.05f, force_mag = 10.f, tau = 0.02f;
      const float force = action[b] == 1 ? force_mag : -force_mag;
      const float c = cosf(th), s = sinf(th);
      const float temp = (force + polemass_length * thd * thd * s) / total_mass;
      const float thacc =
          (gravity * s - c * temp) / (length * (4.0f / 3.0f - masspole * c * c / total_mass));
      const float xacc = temp - polemass_length * thacc * c / total_mass;
      x = x + tau * xd;
      xd = xd + tau * xacc;
      th = th + tau * thd;
      thd = thd + tau * thacc;
      const int32_t n = steps[b] + 1;
      steps[b] = n;
      const bool fell = x < -2.4f || x > 2.4f || th < -0.20943951f || th > 0.20943951f;
      const bool trunc = n >= max_steps;
      reward[b] = 1.f;
      step_type[b] = (fell || trunc) ? kLast : kMid;
      discount[b] = fell ? 0.f : 1.f;  // truncation keeps discount (environments/wrappers.py TimeLimit)
    }
    state[b * 4 + 0] = x; state[b * 4 + 1] = xd; state[b * 4 + 2] = th; state[b * 4 + 3] = thd;
    obs[b * 4 + 0] = x; obs[b * 4 + 1] = xd; obs[b * 4 + 2] = th; obs[b * 4 + 3] = thd;
  }
  next_rng_call(rng_call);
}

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_epsilon_greedy(const float* q, const int32_t* mask, int64_t B, int64_t A, float eps,
                          uint64_t seed, uint64_t* rng_call_dev, const float* u_dev,
                          const int32_t* rand_dev, int32_t* out_action, void* stream) {
  B200RL_CHECK_ARG(q && out_action && B >= 1 && A >= 1, "epsilon_greedy: bad argument");
  B200RL_CHECK_ARG((u_dev == nullptr) == (rand_dev == nullptr),
                   "epsilon_greedy: u and rand must both be given or both NULL");
  B200RL_CHECK_ARG(u_dev || rng_call_dev, "epsilon_greedy: need rng_call_dev");
  B200RL_LAUNCH(eps_greedy_kernel, (unsigned)((B + 255) / 256), 256, 0, (cudaStream_t)stream, q, mask, B, A, eps, seed, rng_call_dev, u_dev, rand_dev, out_action);
  B200RL_CHECK_LAUNCH("epsilon_greedy");
  return B200RL_OK;
}

int b200rl_env_random_step(int32_t* step_type, int32_t* out_step_type, void* obs,
                           int64_t obs_elems, int obs_is_u8, float* reward, float* discount,
                           int64_t B, float p_term, uint64_t seed, uint64_t* rng_call_dev,
                           void* stream) {
  B200RL_CHECK_ARG(step_type && obs && reward && discount && rng_call_dev && B >= 1 &&
                       obs_elems >= 1,
                   "env_random_step: bad argument");
  B200RL_CHECK_ARG(B <= 65535, "env_random_step: B too large for grid.y");
  const int64_t vec = obs_is_u8 ? (obs_elems + 15) / 16 : (obs_elems + 3) / 4;
  dim3 grid((unsigned)((vec + 255) / 256), (unsigned)B);
  B200RL_LAUNCH(env_random_step_kernel, grid, 256, 0, (cudaStream_t)stream, step_type, out_step_type, obs, obs_elems, obs_is_u8, reward, discount, B, p_term, seed, rng_call_dev);
  B200RL_CHECK_LAUNCH("env_random_step");
  return B200RL_OK;
}

int b200rl_env_cartpole_step(float* state, int32_t* steps, int32_t* step_type,
                             const int32_t* action, float* obs, float* reward, float* discount,
                             int64_t B, int32_t max_steps, uint64_t seed,
                             uint64_t* rng_call_dev, void* stream) {
  B200RL_CHECK_ARG(state && steps && step_type && action && obs && reward && discount &&
                       rng_call_dev && B >= 1,
                   "env_cartpole_step: bad argument");
  B200RL_LAUNCH(env_cartpole_step_kernel, (unsigned)((B + 255) / 256), 256, 0, (cudaStream_t)stream, state, steps, step_type, action, obs, reward, discount, B, max_steps, seed, rng_call_dev);
  B200RL_CHECK_LAUNCH("env_cartpole_step");
  return B200RL_OK;
}

}  // extern "C"
