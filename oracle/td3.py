"""numpy restatement of Td3Agent's losses and train step (TEST INFRASTRUCTURE).

Follows agents/td3/td3_agent.py: _train (critic step; actor loss against the UPDATED critic 1;
actor gradients applied only when train_step_counter % actor_update_period == 0, counter taken
before its increment; counter += 1; Periodically soft update of both target critics and the
target actor), critic_loss (target smoothing a' = target_actor(s') + clip(N(0, sigma), +-c), not
clipped to the spec; y = reward_scale r + gamma d min(Q'1, Q'2); mean_b(w_b (l(y,Q1) + l(y,Q2)))),
actor_loss (sum_b(w_b * -Q1(s, pi(s))) / B), _apply_gradients (clip_gradient_norms per variable);
agents/ddpg/actor_network.py (Dense stack, Dense(A, tanh), scale_to_spec) and
agents/ddpg/critic_network.py (observation branch, concat(h_obs, action), joint stack, Dense(1)).
The target-smoothing draws z ~ N(0, 1) are supplied by the caller.
"""
import copy

import numpy as np

from oracle import nn
from oracle import optim

f32 = np.float32
HUBER, SQUARED = 'huber', 'squared'


def scale_to_spec(y, amin, amax):
  """means + magnitudes * y (utils/common.py scale_to_spec)."""
  return (f32(0.5) * (amax + amin) + f32(0.5) * (amax - amin) * y).astype(f32)


def element_loss(y, q, kind):
  """(l(y, q), dl/dq) with l the Huber (delta 1) or the squared TD error."""
  e = (y - q).astype(f32)
  if kind == HUBER:
    a = np.abs(e)
    return (np.where(a <= 1, f32(0.5) * e * e, a - f32(0.5)).astype(f32),
            (-np.clip(e, -1, 1)).astype(f32))
  if kind == SQUARED:
    return (e * e).astype(f32), (f32(-2) * e).astype(f32)
  raise ValueError(kind)


def critic_loss(q1, q2, tq1, tq2, reward, discount, kind=HUBER, gamma=1.0, reward_scale=1.0,
                weights=None):
  """Returns (loss, dq1, dq2, td_targets)."""
  B = q1.shape[0]
  y = (f32(reward_scale) * reward + f32(gamma) * discount * np.minimum(tq1, tq2)).astype(f32)
  l1, g1 = element_loss(y, q1, kind)
  l2, g2 = element_loss(y, q2, kind)
  w = np.ones(B, f32) if weights is None else np.asarray(weights, f32)
  loss = f32(np.sum((l1 + l2) * w, dtype=f32) / f32(B))
  c = (w / f32(B)).astype(f32)
  return loss, (g1 * c).astype(f32), (g2 * c).astype(f32), y


def actor_loss(q, weights=None):
  """Returns (loss, dq)."""
  B = q.shape[0]
  w = np.ones(B, f32) if weights is None else np.asarray(weights, f32)
  return f32(np.sum(-q * w, dtype=f32) / f32(B)), (-w / f32(B)).astype(f32)


def dense_backward(seq, tape, dy):
  """Parameter gradients (aligned with seq.params()) and the input gradient of a Dense stack."""
  grads = []
  for i in range(len(seq.layers) - 1, -1, -1):
    l = seq.layers[i]
    xin, y = tape[i]
    dz = nn.act_bwd(y, dy, l.get('act'))
    dy, dw, db = nn.dense_bwd(xin, l['w'], dz)
    grads = [dw] + ([db] if l.get('b') is not None else []) + grads
  return grads, dy


class Critic(object):
  """obs: Sequential of the observation branch (or None); joint: Sequential ending in Dense(1)."""

  def __init__(self, joint, obs=None):
    self.joint, self.obs = joint, obs

  def params(self):
    return (self.obs.params() if self.obs else []) + self.joint.params()

  def forward(self, observation, action, keep=False):
    h, otape = (self.obs.forward(observation, keep=True) if self.obs else (observation, None))
    x = np.concatenate([h, action], axis=1).astype(f32)
    q, jtape = self.joint.forward(x, keep=True)
    return (q[:, 0], (otape, jtape)) if keep else q[:, 0]

  def backward(self, tape, dq):
    """Returns (parameter gradients, dQ/d concat(h_obs, action))."""
    otape, jtape = tape
    grads, dx = dense_backward(self.joint, jtape, dq[:, None].astype(f32))
    if self.obs:
      hd = self.obs.layers[-1]['w'].shape[1]
      ograds, _ = dense_backward(self.obs, otape, dx[:, :hd])
      grads = ograds + grads
    return grads, dx

  def action_column(self, obs_dim):
    return self.obs.layers[-1]['w'].shape[1] if self.obs else obs_dim


class Td3Oracle(object):
  """actor: Sequential ending in Dense(A, tanh) (amin/amax None: an unbounded actor, no
  scale_to_spec); critics: Critic."""

  def __init__(self, actor, critic1, critic2, amin, amax, actor_opt=None, critic_opt=None,
               gamma=0.99, reward_scale=1.0, tau=0.005, target_update_period=1,
               actor_update_period=1, loss=HUBER, target_policy_noise=0.2,
               target_policy_noise_clip=0.5, gradient_clipping=None):
    self.actor, self.c1, self.c2 = actor, critic1, critic2
    self.ta, self.t1, self.t2 = copy.deepcopy(actor), copy.deepcopy(critic1), copy.deepcopy(critic2)
    self.amin = None if amin is None else np.asarray(amin, f32)
    self.amax = None if amax is None else np.asarray(amax, f32)
    self.actor_opt, self.critic_opt = actor_opt, critic_opt
    self.gamma, self.reward_scale, self.loss = gamma, reward_scale, loss
    self.sigma, self.noise_clip = f32(target_policy_noise), f32(target_policy_noise_clip)
    self.clip = gradient_clipping
    self.actor_update_period = actor_update_period
    self.train_step_counter = 0
    self.actor_updates = 0
    self._update_target = optim.Periodically(
        lambda: optim.soft_variables_update(
            self.c1.params() + self.c2.params() + self.actor.params(),
            self.t1.params() + self.t2.params() + self.ta.params(), tau), target_update_period)

  def _scale(self, y):
    return y if self.amin is None else scale_to_spec(y, self.amin, self.amax)

  def _clip(self, grads):
    return grads if self.clip is None else [optim.clip_by_norm(g, self.clip) for g in grads]

  def target_actions(self, obs2, z=None):
    a2 = self._scale(self.ta.forward(obs2))
    if z is not None and self.sigma > 0:      # not clipped to the action spec (reference quirk)
      a2 = (a2 + np.clip(self.sigma * z, -self.noise_clip, self.noise_clip)).astype(f32)
    return a2

  def critic_grads(self, obs, act, reward, discount, obs2, z=None, weights=None):
    a2 = self.target_actions(obs2, z)
    tq1, tq2 = self.t1.forward(obs2, a2), self.t2.forward(obs2, a2)
    q1, tape1 = self.c1.forward(obs, act, keep=True)
    q2, tape2 = self.c2.forward(obs, act, keep=True)
    loss, dq1, dq2, _ = critic_loss(q1, q2, tq1, tq2, reward, discount, self.loss, self.gamma,
                                    self.reward_scale, weights)
    return loss, self.c1.backward(tape1, dq1)[0] + self.c2.backward(tape2, dq2)[0]

  def actor_grads(self, obs, weights=None):
    y, atape = self.actor.forward(obs, keep=True)
    q, ctape = self.c1.forward(obs, self._scale(y), keep=True)
    loss, dq = actor_loss(q, weights)
    _, dx = self.c1.backward(ctape, dq)
    col = self.c1.action_column(obs.shape[1])
    da = dx[:, col:col + y.shape[1]]
    dy = da if self.amin is None else (f32(0.5) * (self.amax - self.amin) * da).astype(f32)
    grads, _ = dense_backward(self.actor, atape, dy)
    return loss, grads

  def train(self, exp, target_noise=None, weights=None):
    """exp: [B, 2, ...] arrays (observation, action, reward, discount); target_noise: z [B, A]."""
    obs, obs2 = exp['observation'][:, 0], exp['observation'][:, 1]
    act, r, d = exp['action'][:, 0], exp['reward'][:, 0], exp['discount'][:, 0]
    closs, cgrads = self.critic_grads(obs, act, r, d, obs2, target_noise, weights)
    self.critic_opt.apply(self.c1.params() + self.c2.params(), self._clip(cgrads))
    aloss, agrads = self.actor_grads(obs, weights)
    if self.train_step_counter % self.actor_update_period == 0:
      self.actor_opt.apply(self.actor.params(), self._clip(agrads))
      self.actor_updates += 1
    self.train_step_counter += 1
    self._update_target()
    return dict(loss=f32(aloss + closs), actor_loss=aloss, critic_loss=closs)
