// DQN / DDQN loss epilogue, forward and backward fused (kernel family iii-b).
//
// Restates, as one launch over [B] rows:
//   to_n_step_transition          trajectories/trajectory.py:815-832
//   index_with_actions            utils/common.py:367-411
//   GreedyPolicy(QPolicy) argmax  policies/greedy_policy.py:70-89, q_policy.py:150-194
//   compute_td_targets            agents/dqn/dqn_agent.py:75-78
//   huber / squared element loss  utils/common.py:1199-1208
//   valid_mask, aggregate_losses  agents/dqn/dqn_agent.py:514-538, utils/common.py:1400-1476
// and additionally writes dLoss/dq so no autograd tape is needed for the epilogue.
//
// dqn_seq_td_loss is the same epilogue over the [B, T-1] transitions of a recurrent Q network's
// sequence (trajectory.to_transition, dqn_agent.py:514-523): one TD element per (b, t), the LAST
// mask of step t, and td_loss summed over time before the weights and the mean.
#include <math.h>

#include "common.cuh"

namespace b200rl {

constexpr int kStepLast = 2;  // trajectories/time_step.py:113-121

// Greedy action of a selector row (first max wins, like tf.argmax); masked actions read dtype.min.
__device__ __forceinline__ int64_t dqn_greedy(const float* __restrict__ sel,
                                              const int32_t* __restrict__ mask, int64_t A) {
  int64_t best = 0;
  float best_v = -INFINITY;
  bool any = false;
  for (int64_t a = 0; a < A; ++a) {
    float v = sel[a];
    if (mask && mask[a] == 0) v = -3.4028234663852886e38f;  // dtype.min
    if (!any || v > best_v) {
      best_v = v;
      best = a;
      any = true;
    }
  }
  return best;
}

// Element loss l and dl/dq of the TD error e (tf.compat.v1.losses.huber_loss's
// 0.5 * min(|e|, 1)^2 + (|e| - min(|e|, 1)), or e^2).  This rounding is DQN's own: td_elem_loss
// (common.cuh) rounds differently for |e| > 1.
__device__ __forceinline__ void dqn_elem_loss(float e, int loss_kind, float& l, float& dl_dq) {
  if (loss_kind == B200RL_LOSS_HUBER) {
    const float ae = fabsf(e);
    const float quad = fminf(ae, 1.f);
    const float lin = __fsub_rn(ae, quad);
    l = __fadd_rn(__fmul_rn(0.5f, __fmul_rn(quad, quad)), lin);
    dl_dq = -fmaxf(-1.f, fminf(1.f, e));
  } else {
    l = __fmul_rn(e, e);
    dl_dq = -2.f * e;
  }
}

__global__ void __launch_bounds__(256) dqn_td_loss_kernel(
    const float* __restrict__ q, const float* __restrict__ next_q_tgt,
    const float* __restrict__ next_q_sel, const int32_t* __restrict__ next_mask,
    const int32_t* __restrict__ actions, const int32_t* __restrict__ step_type0,
    const float* __restrict__ traj_reward, const float* __restrict__ traj_discount,
    const float* __restrict__ weights, int64_t action_stride, int64_t step_stride, int64_t B,
    int64_t A, int64_t T, float gamma,
    float gamma_pow, float reward_scale, int loss_kind, float global_batch,
    float* __restrict__ loss, float* __restrict__ td_loss, float* __restrict__ td_error,
    float* __restrict__ dq, int32_t* __restrict__ nan_flag) {
  pdl_prologue();
  __shared__ float red[32];
  float partial = 0.f;
  const int64_t n = T - 1;
  for (int64_t b = threadIdx.x; b < B; b += blockDim.x) {
    // n-step reward / discount (foldr order)
    float R = 0.f, D = 1.f;
    for (int64_t t = n - 1; t >= 0; --t)
      R = __fadd_rn(__fmul_rn(R, __fmul_rn(gamma, traj_discount[b * T + t])),
                    traj_reward[b * T + t]);
    for (int64_t t = 0; t < n; ++t) D = __fmul_rn(D, traj_discount[b * T + t]);
    D = __fmul_rn(gamma_pow, D);
    // greedy action of the selector network at s_n (first max wins, like tf.argmax)
    int64_t best = 0;
    float best_v = -INFINITY;
    bool any = false;
    for (int64_t a = 0; a < A; ++a) {
      float v = next_q_sel[b * A + a];
      if (next_mask && next_mask[b * A + a] == 0) v = -3.4028234663852886e38f;  // dtype.min
      if (!any || v > best_v) {
        best_v = v;
        best = a;
        any = true;
      }
    }
    const float nq = next_q_tgt[b * A + best];
    int32_t act = actions[b * action_stride];
    act = act < 0 ? 0 : (act >= A ? (int32_t)A - 1 : act);   // out-of-spec actions must not index past q
    const float qsa = q[b * A + act];
    const float rew = __fmul_rn(reward_scale, R);
    const float disc = __fmul_rn(gamma, D);
    const float target = __fadd_rn(rew, __fmul_rn(disc, nq));
    const float e = __fsub_rn(target, qsa);
    float l, dl_dq;  // element loss and its derivative w.r.t. q
    dqn_elem_loss(e, loss_kind, l, dl_dq);
    const float valid = (step_type0[b * step_stride] == kStepLast) ? 0.f : 1.f;
    const float tl = __fmul_rn(valid, l);
    td_loss[b] = tl;
    td_error[b] = __fmul_rn(valid, e);
    float w = 1.f;
    float wl = tl;
    if (weights) {
      w = weights[b];
      wl = (w == 0.f) ? 0.f : __fmul_rn(tl, w);  // multiply_no_nan
    }
    partial += wl;
    for (int64_t a = 0; a < A; ++a) dq[b * A + a] = 0.f;
    dq[b * A + act] = valid * w * dl_dq / global_batch;
  }
  const float total = block_sum(partial, red);
  if (threadIdx.x == 0) {
    const float out = total / global_batch;
    loss[0] = out;
    if (nan_flag && !isfinite(out)) *nan_flag = 1;
  }
}

struct DqnSeqArgs {
  const float* q;            // [B*(T-1), A] online Q over time_steps
  const float* next_q_tgt;   // [B*(T-1), A] target Q over next_time_steps
  const float* next_q_sel;   // [B*(T-1), A] the table whose argmax picks the bootstrap action
  const int32_t* next_mask;  // [B*(T-1), A] or NULL
  const int32_t* actions;    // element (b, t) at actions[b * act_ld + t * act_st]
  const int32_t* step_type;  // element (b, t) at step_type[b * st_ld + t * st_st]
  const float* reward;       // [B, T]
  const float* discount;     // [B, T]
  const float* weights;      // weights[b * w_stride] or NULL
  int64_t act_ld, act_st, st_ld, st_st, w_stride, B, A, T;
  float gamma, reward_scale, global_batch;
  int loss_kind;
  float *loss, *td_loss, *td_error, *dq;
  int32_t* nan_flag;
  float* partials;           // one per block
  uint32_t* ticket;
};

// G lanes per batch row: lane l takes the steps t = l, l + G, ... of row b in order, the G lane sums
// meet in a fixed shuffle tree, and every block stores one partial of its rows' weighted td_loss.
// The block that takes the last ticket adds the partials in index order.  Every sum has a fixed
// order for a given shape, so repeated launches and graph replays give the same bits.
template <int G>
__global__ void __launch_bounds__(256) dqn_seq_td_loss_kernel(const DqnSeqArgs p) {
  pdl_prologue();
  __shared__ float red[32];
  __shared__ bool last;
  const int64_t Tm = p.T - 1, A = p.A;
  float partial = 0.f;
  B200RL_GROUP_ROWS(G, p.B) {
    const bool live = n < p.B;
    const int64_t b = live ? n : n0;
    const float w = p.weights ? p.weights[b * p.w_stride] : 1.f;
    float s = 0.f;
    for (int64_t t = lane; t < Tm; t += G) {
      const int64_t r = b * Tm + t;
      const int64_t best = dqn_greedy(p.next_q_sel + r * A, p.next_mask ? p.next_mask + r * A
                                                                        : nullptr, A);
      const float nq = p.next_q_tgt[r * A + best];
      const int32_t act = clamp_action(p.actions[b * p.act_ld + t * p.act_st], A,
                                       live ? p.nan_flag : nullptr);
      const float qsa = p.q[r * A + act];
      const float rew = __fmul_rn(p.reward_scale, p.reward[b * p.T + t]);
      const float disc = __fmul_rn(p.gamma, p.discount[b * p.T + t]);
      const float e = __fsub_rn(__fadd_rn(rew, __fmul_rn(disc, nq)), qsa);
      float l, dl_dq;
      dqn_elem_loss(e, p.loss_kind, l, dl_dq);
      const float valid = (p.step_type[b * p.st_ld + t * p.st_st] == kStepLast) ? 0.f : 1.f;
      s += __fmul_rn(valid, l);
      if (live) {
        p.td_error[r] = __fmul_rn(valid, e);
        for (int64_t a = 0; a < A; ++a) p.dq[r * A + a] = 0.f;
        p.dq[r * A + act] = valid * w * dl_dq / p.global_batch;
      }
    }
    s = grp_sum<G>(s);
    if (live && lane == 0) {
      p.td_loss[b] = s;
      partial += (w == 0.f) ? 0.f : __fmul_rn(s, w);  // multiply_no_nan
    }
  }
  const float total = block_sum(partial, red);
  if (threadIdx.x == 0) {
    p.partials[blockIdx.x] = total;
    last = last_block_ticket(p.ticket);
  }
  __syncthreads();
  if (!last) return;
  float s = 0.f;
  for (unsigned i = threadIdx.x; i < gridDim.x; i += blockDim.x) s += __ldcg(p.partials + i);
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float out = s / p.global_batch;
    p.loss[0] = out;
    if (p.nan_flag && !isfinite(out)) *p.nan_flag = 1;
  }
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_dqn_td_loss(const float* q, const float* next_q_tgt,
                                  const float* next_q_sel, const int32_t* next_mask,
                                  const int32_t* actions, const int32_t* step_type0,
                                  const float* traj_reward, const float* traj_discount,
                                  const float* weights, int64_t action_stride,
                                  int64_t step_stride, int64_t B, int64_t A, int64_t T,
                                  double gamma, double reward_scale, int loss_kind,
                                  float global_batch, float* loss, float* td_loss,
                                  float* td_error, float* dq, int32_t* nan_flag, void* stream) {
  B200RL_CHECK_ARG(q && next_q_tgt && next_q_sel && actions && step_type0 && traj_reward &&
                       traj_discount && loss && td_loss && td_error && dq,
                   "dqn_td_loss: NULL argument");
  B200RL_CHECK_ARG(B >= 1 && A >= 1, "dqn_td_loss: B=%lld A=%lld", (long long)B, (long long)A);
  B200RL_CHECK_ARG(T >= 2, "Trajectory frame count must be at least 2, but saw %lld", (long long)T);
  B200RL_CHECK_ARG(loss_kind == B200RL_LOSS_HUBER || loss_kind == B200RL_LOSS_SQUARED,
                   "dqn_td_loss: unknown loss kind %d", loss_kind);
  B200RL_CHECK_ARG(global_batch > 0.f, "dqn_td_loss: global_batch must be > 0");
  B200RL_CHECK_ARG(action_stride >= 1 && step_stride >= 1, "dqn_td_loss: strides must be >= 1");
  B200RL_LAUNCH(dqn_td_loss_kernel, 1, 256, 0, (cudaStream_t)stream, q, next_q_tgt, next_q_sel, next_mask, actions, step_type0, traj_reward, traj_discount, weights, action_stride, step_stride, B, A, T, (float)gamma, (float)pow(gamma, (double)(T - 2)), (float)reward_scale, loss_kind, global_batch, loss, td_loss, td_error, dq, nan_flag);
  B200RL_CHECK_LAUNCH("dqn_td_loss");
  return B200RL_OK;
}

extern "C" int b200rl_dqn_seq_td_loss(
    const float* q, const float* next_q_tgt, const float* next_q_sel, const int32_t* next_mask,
    const int32_t* actions, int64_t action_ld, int64_t action_stride, const int32_t* step_type,
    int64_t step_ld, int64_t step_stride, const float* reward, const float* discount,
    const float* weights, int64_t weight_stride, int64_t B, int64_t A, int64_t T, double gamma,
    double reward_scale, int loss_kind, float global_batch, float* loss, float* td_loss,
    float* td_error, float* dq, int32_t* nan_flag, float* partials, uint32_t* ticket,
    void* stream) {
  B200RL_CHECK_ARG(q && next_q_tgt && next_q_sel && actions && step_type && reward && discount &&
                       loss && td_loss && td_error && dq && partials && ticket,
                   "dqn_seq_td_loss: NULL argument");
  B200RL_CHECK_ARG(B >= 1 && A >= 1, "dqn_seq_td_loss: B=%lld A=%lld", (long long)B,
                   (long long)A);
  B200RL_CHECK_ARG(T >= 2, "Trajectory frame count must be at least 2, but saw %lld", (long long)T);
  B200RL_CHECK_ARG(loss_kind == B200RL_LOSS_HUBER || loss_kind == B200RL_LOSS_SQUARED,
                   "dqn_seq_td_loss: unknown loss kind %d", loss_kind);
  B200RL_CHECK_ARG(global_batch > 0.f, "dqn_seq_td_loss: global_batch must be > 0");
  B200RL_CHECK_ARG(action_ld >= 0 && action_stride >= 0 && step_ld >= 0 && step_stride >= 0 &&
                       weight_stride >= 0,
                   "dqn_seq_td_loss: strides must be >= 0");
  DqnSeqArgs p;
  p.q = q; p.next_q_tgt = next_q_tgt; p.next_q_sel = next_q_sel; p.next_mask = next_mask;
  p.actions = actions; p.step_type = step_type; p.reward = reward; p.discount = discount;
  p.weights = weights;
  p.act_ld = action_ld; p.act_st = action_stride; p.st_ld = step_ld; p.st_st = step_stride;
  p.w_stride = weight_stride; p.B = B; p.A = A; p.T = T;
  p.gamma = (float)gamma; p.reward_scale = (float)reward_scale; p.global_batch = global_batch;
  p.loss_kind = loss_kind;
  p.loss = loss; p.td_loss = td_loss; p.td_error = td_error; p.dq = dq; p.nan_flag = nan_flag;
  p.partials = partials; p.ticket = ticket;
  const int G = lane_group(T - 1);
  const unsigned blocks = group_blocks(B, G, B200RL_DQN_SEQ_MAX_BLOCKS);
  cudaStream_t st = (cudaStream_t)stream;
  if (G == 1)
    B200RL_LAUNCH(dqn_seq_td_loss_kernel<1>, blocks, 256, 0, st, p);
  else if (G == 8)
    B200RL_LAUNCH(dqn_seq_td_loss_kernel<8>, blocks, 256, 0, st, p);
  else
    B200RL_LAUNCH(dqn_seq_td_loss_kernel<32>, blocks, 256, 0, st, p);
  B200RL_CHECK_LAUNCH("dqn_seq_td_loss");
  return B200RL_OK;
}
