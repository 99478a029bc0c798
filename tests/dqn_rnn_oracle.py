"""numpy restatement of the recurrent DqnAgent / DdqnAgent loss and train step (TEST
INFRASTRUCTURE), on oracle.lstm.RnnNet networks.

Follows agents/dqn/dqn_agent.py with a stateful q_network: AsTransition(squeeze_time_dim=False)
(trajectory.to_transition) :286-291, _loss :494-538 (valid mask of time_steps, td_loss summed
over time, aggregate_losses), the target updater :385-409 and _train :412-449.  Each transition's
element loss is oracle.dqn.dqn_loss at n = 1, so the rounding is the feed-forward oracle's.
"""
import copy

import numpy as np
import torch

from oracle import dqn as odqn
from oracle import optim

f32 = np.float32


def dqn_seq_loss(q, next_q_target, next_q_select, actions, step_type, reward, discount,
                 gamma=1.0, reward_scale=1.0, loss_fn='huber', weights=None, next_mask=None,
                 global_batch=None):
  """TD loss over [B, T-1] transitions.  q / next_q_* / next_mask: [B*(T-1), A] rows (row
  b*(T-1) + t); actions, step_type, reward, discount: [B, T-1] (the [:, :-1] columns).
  Returns dict(loss, td_loss [B], td_error [B, T-1], dq [B*(T-1), A])."""
  B, Tm = np.asarray(actions).shape
  N = B * Tm
  w = None if weights is None else np.broadcast_to(np.asarray(weights, f32), (B,)).copy()
  gb = f32(global_batch if global_batch is not None else B)
  # one n = 1 transition per row: reward / discount columns [r_t, unused]
  traj_r = np.stack([np.asarray(reward, f32).reshape(N), np.zeros(N, f32)], 1)
  traj_d = np.stack([np.asarray(discount, f32).reshape(N), np.ones(N, f32)], 1)
  el = odqn.dqn_loss(q, next_q_target, next_q_select, np.asarray(actions).reshape(N),
                     np.asarray(step_type).reshape(N), traj_r, traj_d, gamma, reward_scale,
                     loss_fn, weights=None if w is None else np.repeat(w, Tm),
                     next_mask=next_mask, global_batch=gb)
  td_loss = el['td_loss'].reshape(B, Tm).sum(1, dtype=f32)                   # :519-523
  per_example = td_loss if w is None else np.where(w == 0, f32(0), td_loss * w).astype(f32)
  loss = f32(np.sum(per_example, dtype=f32) / gb)
  return dict(loss=loss, td_loss=td_loss, td_error=el['td_error'].reshape(B, Tm), dq=el['dq'])


def seq_loss_float64(q, next_t, next_sel, actions, step_type, reward, discount, gamma, scale,
                     kind, weights, mask):
  """float64 torch autograd of the reference formula (clamped actions) from float32 inputs;
  returns (loss, td_loss [B], td_error [B, T-1], dq [B*(T-1), A]) as float64 numpy."""
  B, Tm = actions.shape
  N, A = q.shape
  q = torch.tensor(q, dtype=torch.float64, requires_grad=True)
  sel = torch.tensor(next_sel, dtype=torch.float64)
  if mask is not None:
    sel = torch.where(torch.as_tensor(np.asarray(mask)) != 0, sel,
                      torch.tensor(float(np.finfo(f32).min), dtype=torch.float64))
  best = torch.argmax(sel, 1)      # first max
  nq = torch.tensor(next_t, dtype=torch.float64)[torch.arange(N), best]
  qa = q[torch.arange(N), torch.as_tensor(np.clip(actions.reshape(N), 0, A - 1), dtype=torch.int64)]
  y = scale * torch.tensor(reward.reshape(N), dtype=torch.float64) + \
      gamma * torch.tensor(discount.reshape(N), dtype=torch.float64) * nq
  e = y - qa
  l = torch.where(e.abs() <= 1, 0.5 * e * e, e.abs() - 0.5) if kind == 'huber' else e * e
  valid = torch.as_tensor(step_type.reshape(N) != 2, dtype=torch.float64)
  td_loss = (valid * l).reshape(B, Tm).sum(1)
  w = torch.ones(B, dtype=torch.float64) if weights is None else \
      torch.as_tensor(np.broadcast_to(np.asarray(weights, np.float64), (B,)).copy())
  loss = (td_loss * w).sum() / B
  dq, = torch.autograd.grad(loss, q)
  return (float(loss.detach()), td_loss.detach().numpy(), (valid * e).reshape(B, Tm).detach().numpy(),
          dq.numpy())


class RecurrentDqnOracle(object):
  """One-replica recurrent DQN / DDQN learner.  exp: dict of [B, T, ...] arrays with keys
  step_type, next_step_type, observation, action, reward, discount and optionally mask
  ([B, T, A] action mask of the observations).  l2: [(index into q_net.params(), coef)]."""

  def __init__(self, q_net, optimizer, gamma=1.0, reward_scale=1.0, loss_fn='huber',
               target_update_tau=1.0, target_update_period=1, gradient_clipping=None,
               ddqn=False, l2=()):
    self.q_net = q_net
    self.target_net = copy.deepcopy(q_net)
    self.optimizer = optimizer
    self.gamma, self.reward_scale, self.loss_fn = gamma, reward_scale, loss_fn
    self.gradient_clipping = gradient_clipping
    self.ddqn = ddqn
    self.l2 = list(l2)
    self.train_step_counter = 0
    self._update_target = optim.Periodically(
        lambda: optim.soft_variables_update(self.q_net.params(), self.target_net.params(),
                                            target_update_tau), target_update_period)

  def loss(self, exp, weights=None):
    st = np.asarray(exp['step_type'])
    B, T = st.shape
    N = B * (T - 1)
    obs = np.asarray(exp['observation'], f32)
    x0 = obs[:, :-1].reshape(N, -1)
    x1 = obs[:, 1:].reshape(N, -1)
    st0, st1 = st[:, :-1], np.asarray(exp['next_step_type'])[:, :-1]
    self.target_net.step_type = st1
    next_t = self.target_net.forward(x1)
    next_sel = next_t
    if self.ddqn:
      self.q_net.step_type = st1
      next_sel = self.q_net.forward(x1)
    self.q_net.step_type = st0
    q, tape = self.q_net.forward(x0, keep=True)
    mask = exp.get('mask')
    next_mask = None if mask is None else np.asarray(mask)[:, 1:].reshape(N, -1)
    out = dqn_seq_loss(q, next_t, next_sel, np.asarray(exp['action'])[:, :-1], st0,
                       np.asarray(exp['reward'])[:, :-1], np.asarray(exp['discount'])[:, :-1],
                       self.gamma, self.reward_scale, self.loss_fn, weights, next_mask)
    params = self.q_net.params()
    reg = f32(0)
    for i, coef in self.l2:
      reg = f32(reg + f32(coef) * np.sum(params[i] * params[i], dtype=f32))
    out['loss'] = f32(out['loss'] + reg)
    out['tape'] = tape
    return out

  def train(self, exp, weights=None):
    out = self.loss(exp, weights)
    grads = self.q_net.backward(out['tape'], out['dq'])
    params = self.q_net.params()
    for i, coef in self.l2:
      grads[i] = (grads[i] + f32(2 * coef) * params[i]).astype(f32)
    if self.gradient_clipping is not None:
      grads = [optim.clip_by_norm(g, self.gradient_clipping) for g in grads]
    self.optimizer.apply(params, grads)
    self.train_step_counter += 1
    self._update_target()
    out['grads'] = grads
    return out


def reference_smoke_case():
  """The data of the reference's testLossRNNSmokeTest (dqn_agent_test.py:357-414): B = 2, T = 3,
  observations (1, 2), (5, 6), (9, 10) and (3, 4), (7, 8), (11, 12), FIRST then MID, actions
  (0, 1), rewards (10, 20), discounts (0.7, 0.8); one keras LSTM(2) with 0.5 kernels and the
  default bias (unit forget bias).  Returns (exp, [W, U, b])."""
  obs = np.array([[[1, 2], [5, 6], [9, 10]], [[3, 4], [7, 8], [11, 12]]], f32)
  exp = dict(observation=obs,
             step_type=np.array([[0, 1, 1]] * 2, np.int32),
             next_step_type=np.ones((2, 3), np.int32),
             action=np.array([[0] * 3, [1] * 3], np.int32),
             reward=np.array([[10] * 3, [20] * 3], f32),
             discount=np.array([[0.7] * 3, [0.8] * 3], f32))
  b = np.zeros(8, f32)
  b[2:4] = 1.0
  return exp, [np.full((2, 8), 0.5, f32), np.full((2, 8), 0.5, f32), b]


REFERENCE_SMOKE_LOSS = 28.722265   # at gamma 1.0 (the reference _loss's own default)
