// Categorical DQN (C51, Bellemare et al. 2017) loss epilogue, forward and backward fused, and the
// expected-Q reduction of the categorical policies (kernel family iii-b).
//
// Restates, per row of a [B] batch (agents/categorical_dqn/categorical_dqn_agent.py):
//   _next_q_distribution            :520-556 softmax over the atoms of every action, expected Q
//                                   (common.convert_q_logits_to_values), greedy action of the
//                                   target policy (masked actions at -inf,
//                                   policies/categorical_q_policy.py:170-190), its distribution
//   target support                  :377-398 (one step) / :400-432 (n step, discounted_return
//                                   with final value 0 and reduce_prod of the discounts)
//   project_distribution            :562-731 in its clipped-quotient form (N^2 terms per row)
//   softmax_cross_entropy_with_logits_v2 of the chosen action's logits :440-461
//   aggregate_losses                :463-466 mean over global_batch, no sample weights
// and writes dLoss/dlogits so no autograd tape is needed for the epilogue.
//
// Stages (fixed-order reductions only, so a graph replay equals the eager call bit for bit):
//   1. c51_rows_kernel   one warp per row: per-row loss into the workspace, dq row.
//   2. c51_mean_kernel   one block sums the per-row losses in index order, / global_batch.
#include <math.h>

#include "common.cuh"

namespace b200rl {

namespace {

constexpr int kC51MaxAtoms = 1024;
constexpr int kC51MaxBlocks = 4 * kNumSMs;

// Warps (rows) per block: three [N] float arrays per warp in shared memory, at most 36 KB per
// block.  Spreading B = 256 rows over 128 blocks of 2 warps instead of 32 blocks of 8 measured
// no faster on H100s (18.4 against 18.8 us per call in separate runs, within their spread).
int c51_warps(int64_t N) {
  int64_t w = 3072 / N;
  return (int)(w < 1 ? 1 : (w > 8 ? 8 : w));
}

__global__ void __launch_bounds__(256) c51_rows_kernel(
    const float* __restrict__ q, const float* __restrict__ next_q,
    const int32_t* __restrict__ next_mask, const int32_t* __restrict__ actions,
    int64_t action_stride, const float* __restrict__ reward, const float* __restrict__ discount,
    const float* __restrict__ z, const float* __restrict__ z_sel, int64_t B, int64_t A, int64_t N,
    int64_t T, float gamma,
    float reward_scale, float global_batch, float* __restrict__ row_loss, float* __restrict__ dq,
    int32_t* __restrict__ nan_flag) {
  pdl_prologue();
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int wpb = blockDim.x >> 5;
  float* tz = smem + (int64_t)wid * 3 * N;   // clipped target support of this warp's row
  float* pj = tz + N;                        // target probabilities of the greedy action
  float* mp = pj + N;                        // projected target distribution m
  const float z0 = z[0], zl = z[N - 1];
  const float dz = z[1] - z[0];              // delta_z = target_support[1] - target_support[0] (:607-609)
  const int64_t AN = A * N;
  for (int64_t b = (int64_t)blockIdx.x * wpb + wid; b < B; b += (int64_t)gridDim.x * wpb) {
    // ---- shifted support --------------------------------------------------------------------
    const float* rw = reward + b * T;
    const float* dc = discount + b * T;
    float R, D;
    const bool one_step = (T == 2);
    if (one_step) {
      R = __fmul_rn(reward_scale, rw[0]);            // reward_term (:388-394)
      D = dc[0];                                     // gamma * (discount * z) below (:378-398)
    } else {
      R = 0.f;                                       // discounted_return, final_value 0 (:409-415)
      for (int64_t t = T - 2; t >= 0; --t)
        R = __fadd_rn(__fmul_rn(reward_scale, rw[t]), __fmul_rn(__fmul_rn(gamma, dc[t]), R));
      D = 1.f;                                       // reduce_prod(gamma * discount) (:420)
      for (int64_t t = 0; t < T - 1; ++t) D = __fmul_rn(D, __fmul_rn(gamma, dc[t]));
    }
    // ---- greedy action of the target policy at s_n (its own support z_sel) --------------------
    const float* nq = next_q + b * AN;
    int best = 0;
    float best_v = 0.f, best_m = 0.f, best_s = 1.f;
    for (int64_t a = 0; a < A; ++a) {
      const float* l = nq + a * N;
      float m, s, t_;
      row_softmax_stats<32>(l, N, lane, m, s, t_);
      float qa = 0.f;
      for (int64_t j = lane; j < N; j += 32) qa += __fmul_rn(z_sel[j], expf(l[j] - m) / s);
      qa = grp_sum<32>(qa);
      if (next_mask && next_mask[b * A + a] == 0) qa = -INFINITY;   // :184-187
      if (a == 0 || qa > best_v) {                                  // first argmax (mode)
        best_v = qa; best = (int)a; best_m = m; best_s = s;
      }
    }
    const float* lb = nq + (int64_t)best * N;
    for (int64_t j = lane; j < N; j += 32) {
      const float t = one_step ? __fadd_rn(R, __fmul_rn(gamma, __fmul_rn(D, z[j])))
                               : __fadd_rn(R, __fmul_rn(D, z[j]));
      tz[j] = fminf(fmaxf(t, z0), zl);               // clip_by_value(supports, v_min, v_max) (:660)
      pj[j] = expf(lb[j] - best_m) / best_s;
    }
    __syncwarp();
    // ---- chosen action's logits -------------------------------------------------------------
    const int32_t act = clamp_action(actions[b * action_stride], A, lane == 0 ? nan_flag : nullptr);
    const float* l = q + b * AN + (int64_t)act * N;
    float m, s, t_;
    row_softmax_stats<32>(l, N, lane, m, s, t_);
    const float log_s = logf(s);
    // ---- projection + cross entropy -----------------------------------------------------------
    float loss_p = 0.f, msum = 0.f;
    for (int64_t i = lane; i < N; i += 32) {
      const float zi = z[i];
      float mi = 0.f;
      for (int64_t j = 0; j < N; ++j) {
        const float quot = 1.f - fabsf(tz[j] - zi) / dz;              // :697-698
        mi = fmaf(fminf(fmaxf(quot, 0.f), 1.f), pj[j], mi);          // :710-729
      }
      loss_p += mi * (log_s - (l[i] - m));           // m_i * (logsumexp(l) - l_i)
      msum += mi;
      mp[i] = mi;
    }
    loss_p = grp_sum<32>(loss_p);
    msum = grp_sum<32>(msum);
    __syncwarp();
    // ---- dLoss/dlogits: (softmax(l) * sum(m) - m) / global_batch on the chosen action ---------
    float* dr = dq + b * AN;
    for (int64_t k = lane; k < AN; k += 32) {
      const int64_t i = k - (int64_t)act * N;
      float g = 0.f;
      if (i >= 0 && i < N) g = (expf(l[i] - m) / s * msum - mp[i]) / global_batch;
      dr[k] = g;
    }
    if (lane == 0) row_loss[b] = loss_p;
    __syncwarp();                                    // tz / pj / mp are rewritten by the next row
  }
}

__global__ void __launch_bounds__(256) c51_mean_kernel(const float* __restrict__ row_loss,
                                                       int64_t B, float global_batch,
                                                       float* __restrict__ loss,
                                                       int32_t* __restrict__ nan_flag) {
  pdl_prologue();
  __shared__ float red[32];
  float p = 0.f;
  for (int64_t b = threadIdx.x; b < B; b += blockDim.x) p += row_loss[b];
  const float total = block_sum(p, red);
  if (threadIdx.x == 0) {
    const float out = total / global_batch;
    loss[0] = out;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
  }
}

// q[r] = sum_j z_j softmax(logits[r])_j over rows r of [B*A, N] (common.convert_q_logits_to_values).
template <int G>
__global__ void __launch_bounds__(256) c51_q_values_kernel(const float* __restrict__ logits,
                                                           const float* __restrict__ z,
                                                           int64_t rows, int64_t N,
                                                           float* __restrict__ q) {
  pdl_prologue();
  B200RL_GROUP_ROWS(G, rows) {
    const bool valid = n < rows;
    const float* l = logits + (valid ? n : n0) * N;
    float m, s, t_;
    row_softmax_stats<G>(l, N, lane, m, s, t_);
    float v = 0.f;
    for (int64_t j = lane; j < N; j += G) v += __fmul_rn(z[j], expf(l[j] - m) / s);
    v = grp_sum<G>(v);
    if (valid && lane == 0) q[n] = v;
  }
}

}  // namespace

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_c51_loss(const float* q, const float* next_q, const int32_t* next_mask,
                    const int32_t* actions, int64_t action_stride, const float* reward,
                    const float* discount, const float* support,
                    const float* select_support, int64_t B, int64_t A, int64_t N,
                    int64_t T, float gamma, float reward_scale, float global_batch, float* loss,
                    float* dq, int32_t* nan_flag, void* workspace, int64_t ws_bytes,
                    void* stream) {
  B200RL_CHECK_ARG(q && next_q && actions && reward && discount && support && loss && dq,
                   "c51_loss: NULL argument");
  B200RL_CHECK_ARG(B >= 1 && A >= 1, "c51_loss: B=%lld A=%lld", (long long)B, (long long)A);
  B200RL_CHECK_ARG(N >= 2 && N <= kC51MaxAtoms, "c51_loss: num_atoms must be in [2, %d], got %lld",
                   kC51MaxAtoms, (long long)N);
  B200RL_CHECK_ARG(T >= 2, "Trajectory frame count must be at least 2, but saw %lld", (long long)T);
  B200RL_CHECK_ARG(global_batch > 0.f, "c51_loss: global_batch must be > 0");
  B200RL_CHECK_ARG(action_stride >= 1, "c51_loss: action_stride must be >= 1");
  B200RL_CHECK_ARG(workspace && ws_bytes >= 4 * B, "c51_loss: workspace needs 4*B bytes");
  cudaStream_t st = (cudaStream_t)stream;
  const int wpb = c51_warps(N);
  int64_t nb = (B + wpb - 1) / wpb;
  if (nb > kC51MaxBlocks) nb = kC51MaxBlocks;
  float* rows = (float*)workspace;
  B200RL_LAUNCH(c51_rows_kernel, (unsigned)nb, 32 * wpb, (size_t)wpb * 3 * N * sizeof(float), st, q, next_q, next_mask, actions, action_stride, reward, discount, support, select_support ? select_support : support, B, A, N, T, gamma, reward_scale, global_batch, rows, dq, nan_flag);
  B200RL_CHECK_LAUNCH("c51_loss");
  B200RL_LAUNCH(c51_mean_kernel, 1, 256, 0, st, (const float*)rows, B, global_batch, loss, nan_flag);
  B200RL_CHECK_LAUNCH("c51_loss_mean");
  return B200RL_OK;
}

int b200rl_c51_q_values(const float* logits, const float* support, int64_t B, int64_t A,
                        int64_t N, float* q, void* stream) {
  B200RL_CHECK_ARG(logits && support && q, "c51_q_values: NULL argument");
  B200RL_CHECK_ARG(B >= 1 && A >= 1 && N >= 1, "c51_q_values: B=%lld A=%lld N=%lld",
                   (long long)B, (long long)A, (long long)N);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t rows = B * A;
  const int G = N <= 64 ? 8 : 32;
  int64_t nb = (rows * G + 255) / 256;
  if (nb > kC51MaxBlocks) nb = kC51MaxBlocks;
  if (G == 8) B200RL_LAUNCH(c51_q_values_kernel<8>, (unsigned)nb, 256, 0, st, logits, support, rows, N, q);
  else B200RL_LAUNCH(c51_q_values_kernel<32>, (unsigned)nb, 256, 0, st, logits, support, rows, N, q);
  B200RL_CHECK_LAUNCH("c51_q_values");
  return B200RL_OK;
}

}  // extern "C"
