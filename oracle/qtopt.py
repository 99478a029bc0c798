"""numpy restatement of QtOptAgent's train step and of CEMPolicy's search (TEST INFRASTRUCTURE).

Follows agents/qtopt/qtopt_agent.py: _train / _loss (n-step reduction of reward and discount as
trajectory.to_n_step_transition; a' = CEM search on the TARGET network at s'; next_q =
min(Q_delayed, Q_delayed_2) at (s', a') with enable_td3, else Q_target(s', a'); y = reward_scale r
+ gamma d next_q; td_loss = ~is_last(s) * l(y, Q(s, a)); loss = sum_b w_b td_loss_b / B;
clip_gradient_norms per variable; optimiser step; counter += 1; _update_both: delayed_2 <- delayed,
delayed <- target, target <- q, each on its own Periodically), policies/qtopt_cem_policy.py
actor_func (variance floor, sample, score, tf.nn.top_k, refit; the action is the best sample of the
last iteration) and the continuous GaussianActionsSampler (clip to the spec; tf.nn.moments: the
mean first, then the mean of squared deviations, both / M).  Moments are summed in rank order in
float32, as the kernel does.  The N(0, 1) draws z [I, B, N, A] are supplied by the caller.
"""
import copy

import numpy as np

from oracle import optim
from oracle.td3 import HUBER, SQUARED, Critic, element_loss  # noqa: F401

f32 = np.float32


def top_k(scores, m):
  """[B, m] indices of the m largest scores per row, larger first, the lower index on a tie."""
  return np.argsort(-np.asarray(scores, f32), axis=1, kind='stable')[:, :m]


def moments(x):
  """(mean, var) over axis 1 of x [B, M, A]: float32 sums in order, each divided by M."""
  M = x.shape[1]
  s = np.zeros((x.shape[0], x.shape[2]), f32)
  for j in range(M):
    s = (s + x[:, j]).astype(f32)
  mean = (s / f32(M)).astype(f32)
  q = np.zeros_like(s)
  for j in range(M):
    d = (x[:, j] - mean).astype(f32)
    q = (q + d * d).astype(f32)
  return mean, (q / f32(M)).astype(f32)


def sample(mean, var, z, minimal_var, amin, amax):
  """clip(mean + sqrt(max(var, minimal_var)) z, amin, amax) for mean, var [B, A], z [B, N, A]."""
  sd = np.sqrt(np.maximum(var, f32(minimal_var))).astype(f32)
  return np.clip((mean[:, None] + sd[:, None] * z).astype(f32), amin, amax).astype(f32)


def cem_search(score_fn, B, init_mean, init_var, z, num_elites, minimal_var, amin, amax):
  """(best_action [B, A], best_score [B]); score_fn maps actions [B*N, A] (tile_batch order) to
  scores [B*N]."""
  A = z.shape[-1]
  mean = np.broadcast_to(np.asarray(init_mean, f32), (B, A)).astype(f32)
  var = np.broadcast_to(np.asarray(init_var, f32), (B, A)).astype(f32)
  rows = np.arange(B)[:, None]
  for zi in z:
    a = sample(mean, var, zi, minimal_var, amin, amax)
    N = a.shape[1]
    s = np.asarray(score_fn(a.reshape(B * N, A)), f32).reshape(B, N)
    idx = top_k(s, num_elites)
    elites = a[rows, idx]
    mean, var = moments(elites)
  return elites[:, 0], s[rows[:, 0], idx[:, 0]]


def nstep_reduce(reward, discount, gamma):
  """(reward, discount) [B] of [B, n+1] frames, as b200rl_nstep_reduce."""
  n = reward.shape[1] - 1
  acc = np.zeros(reward.shape[0], f32)
  for t in range(n - 1, -1, -1):
    acc = (acc * (f32(gamma) * discount[:, t]).astype(f32) + reward[:, t]).astype(f32)
  prod = np.ones(reward.shape[0], f32)
  for t in range(n):
    prod = (prod * discount[:, t]).astype(f32)
  return acc, (f32(gamma ** (n - 1)) * prod).astype(f32)


class QtOptOracle(object):
  """critic: a Critic (oracle.td3); the target and both delayed networks start as copies."""

  def __init__(self, critic, amin, amax, init_mean, init_var, opt=None, num_samples=32,
               num_elites=4, num_iter=3, minimal_var=1e-4, gamma=1.0, reward_scale=1.0, tau=1.0,
               target_update_period=1, enable_td3=True, delayed_target_update_period=5,
               loss=HUBER, gradient_clipping=None):
    self.q = critic
    self.target = copy.deepcopy(critic)
    self.delayed = copy.deepcopy(critic) if enable_td3 else None
    self.delayed_2 = copy.deepcopy(critic) if enable_td3 else None
    self.amin, self.amax = np.asarray(amin, f32), np.asarray(amax, f32)
    self.init_mean, self.init_var = init_mean, init_var
    self.opt = opt
    self.N, self.M, self.I, self.minimal_var = num_samples, num_elites, num_iter, minimal_var
    self.gamma, self.reward_scale, self.loss_kind = gamma, reward_scale, loss
    self.enable_td3, self.clip = enable_td3, gradient_clipping
    self.train_step_counter = 0
    upd = lambda src, dst, t: (lambda: optim.soft_variables_update(src.params(), dst.params(), t))
    self._updates = [optim.Periodically(upd(self.q, self.target, tau), target_update_period)]
    if enable_td3:
      self._updates = [
          optim.Periodically(upd(self.delayed, self.delayed_2, 1.0), delayed_target_update_period),
          optim.Periodically(upd(self.target, self.delayed, 1.0), delayed_target_update_period),
      ] + self._updates

  def search(self, net, obs, z):
    B = obs.shape[0]
    tiled = np.repeat(obs, self.N, axis=0)
    return cem_search(lambda a: net.forward(tiled, a), B, self.init_mean, self.init_var, z,
                      self.M, self.minimal_var, self.amin, self.amax)

  def loss_and_grads(self, exp, z, weights=None):
    """exp: [B, n+1, ...] arrays (observation, action, reward, discount, step_type)."""
    obs, obs2 = exp['observation'][:, 0], exp['observation'][:, -1]
    act = exp['action'][:, 0]
    r, d = nstep_reduce(exp['reward'], exp['discount'], self.gamma)
    B = obs.shape[0]
    a2, best = self.search(self.target, obs2, z)
    if self.enable_td3:
      nq = np.minimum(self.delayed_2.forward(obs2, a2), self.delayed.forward(obs2, a2))
    else:
      nq = best
    y = (f32(self.reward_scale) * r + (f32(self.gamma) * d).astype(f32) * nq).astype(f32)
    m = (exp['step_type'][:, 0] != 2).astype(f32)
    q, tape = self.q.forward(obs, act, keep=True)
    l, g = element_loss(y, q, self.loss_kind)
    w = np.ones(B, f32) if weights is None else np.asarray(weights, f32)
    td_loss = (m * l).astype(f32)
    loss = f32(np.sum(td_loss * w, dtype=f32) / f32(B))
    dq = (m * g * (w / f32(B))).astype(f32)
    grads = self.q.backward(tape, dq)[0]
    return dict(loss=loss, td_loss=td_loss, td_error=(m * (y - q)).astype(f32), y=y,
                next_action=a2), grads

  def train(self, exp, z, weights=None):
    out, grads = self.loss_and_grads(exp, z, weights)
    if self.clip is not None:
      grads = [optim.clip_by_norm(g, self.clip) for g in grads]
    self.opt.apply(self.q.params(), grads)
    self.train_step_counter += 1
    for u in self._updates:
      u()
    return out
