"""numpy restatement of DdpgAgent's losses and train step and of the OU noise (TEST
INFRASTRUCTURE).

Follows agents/ddpg/ddpg_agent.py: _train (critic step; actor loss against the UPDATED critic;
counter += 1; Periodically soft update of the target critic and the target actor), critic_loss
(a' = target_actor(s') with no noise and no clip; y = reward_scale r + gamma d Q'(s', a');
mean_b(w_b l(y, Q))), actor_loss (dqda = dQ/da of sum(Q); c = clip(dqda, +-dqda_clipping);
element_wise_squared_loss(stop_gradient(a + c), a) = c^2; weighted mean over the batch), and
_apply_gradients (clip_gradient_norms per variable); policies/ou_noise_policy.py with
utils/common.py OUProcess.  The two choices the agent documents are encoded here:
  * dqda_clipping=0 clips dQ/da to [0, 0], as the reference code does (its docstring says "no
    clipping"), so the actor gradient is zero;
  * the weights multiply each row of the [B, A] actor loss (w_b per batch entry); the reference
    broadcasts [B, A] * [B], which is [B, B] when A = 1 and an error for most other shapes.
The actor loss is the exact c^2, not the reference's float32 ((a + c) - a)^2.  The OU draws
z ~ N(0, 1) are supplied by the caller.
"""
import copy

import numpy as np

from oracle import optim
from oracle.td3 import HUBER, SQUARED, Critic, dense_backward, element_loss, scale_to_spec  # noqa: F401

f32 = np.float32


def critic_loss(q, tq, reward, discount, kind=HUBER, gamma=1.0, reward_scale=1.0, weights=None):
  """Returns (loss, dq, td_targets)."""
  B = q.shape[0]
  y = (f32(reward_scale) * reward + f32(gamma) * discount * tq).astype(f32)
  l, g = element_loss(y, q, kind)
  w = np.ones(B, f32) if weights is None else np.asarray(weights, f32)
  loss = f32(np.sum(l * w, dtype=f32) / f32(B))
  return loss, (g * (w / f32(B))).astype(f32), y


def actor_loss(dqda, dqda_clipping=None, weights=None):
  """dqda [B, A] = dQ/da; returns (loss, dloss/da)."""
  B, A = dqda.shape
  c = dqda if dqda_clipping is None else np.clip(dqda, -f32(dqda_clipping), f32(dqda_clipping))
  c = c.astype(f32)
  w = (np.ones(B, f32) if weights is None else np.asarray(weights, f32))[:, None]
  inv = f32(1) / (f32(B) * f32(A))
  return f32(np.sum(c * c * w, dtype=f32) * inv), (f32(-2) * w * c * inv).astype(f32)


def ou_step(x, z, damping, stddev):
  """x <- (1 - damping) x + stddev z (common.OUProcess.__call__ with N(0, stddev) = stddev z)."""
  return (f32(1 - f32(damping)) * x + f32(stddev) * z).astype(f32)


def ou_actions(loc, xs, amin=None, amax=None):
  """The same OU state x [A] added to every row of loc [N, A], clipped to the spec when given."""
  out = (loc + xs[None, :]).astype(f32)
  return out if amin is None else np.clip(out, amin, amax).astype(f32)


class DdpgOracle(object):
  """actor: Sequential ending in Dense(A, tanh) (amin/amax None: an unbounded actor, no
  scale_to_spec); critic: Critic."""

  def __init__(self, actor, critic, amin, amax, actor_opt=None, critic_opt=None, gamma=1.0,
               reward_scale=1.0, tau=1.0, target_update_period=1, loss=HUBER, dqda_clipping=None,
               gradient_clipping=None):
    self.actor, self.critic = actor, critic
    self.ta, self.tc = copy.deepcopy(actor), copy.deepcopy(critic)
    self.amin = None if amin is None else np.asarray(amin, f32)
    self.amax = None if amax is None else np.asarray(amax, f32)
    self.actor_opt, self.critic_opt = actor_opt, critic_opt
    self.gamma, self.reward_scale, self.loss = gamma, reward_scale, loss
    self.dqda_clipping = dqda_clipping
    self.clip = gradient_clipping
    self.train_step_counter = 0
    self._update_target = optim.Periodically(
        lambda: optim.soft_variables_update(self.critic.params() + self.actor.params(),
                                            self.tc.params() + self.ta.params(), tau),
        target_update_period)

  def _scale(self, y):
    return y if self.amin is None else scale_to_spec(y, self.amin, self.amax)

  def _clip(self, grads):
    return grads if self.clip is None else [optim.clip_by_norm(g, self.clip) for g in grads]

  def critic_grads(self, obs, act, reward, discount, obs2, weights=None):
    a2 = self._scale(self.ta.forward(obs2))
    tq = self.tc.forward(obs2, a2)
    q, tape = self.critic.forward(obs, act, keep=True)
    loss, dq, _ = critic_loss(q, tq, reward, discount, self.loss, self.gamma, self.reward_scale,
                              weights)
    return loss, self.critic.backward(tape, dq)[0]

  def dqda(self, obs, a):
    """dQ(s_b, a_b)/da_b of sum(Q), per sample."""
    _, ctape = self.critic.forward(obs, a, keep=True)
    _, dx = self.critic.backward(ctape, np.ones(obs.shape[0], f32))
    col = self.critic.action_column(obs.shape[1])
    return dx[:, col:col + a.shape[1]]

  def actor_grads(self, obs, weights=None):
    y, atape = self.actor.forward(obs, keep=True)
    loss, da = actor_loss(self.dqda(obs, self._scale(y)), self.dqda_clipping, weights)
    dy = da if self.amin is None else (f32(0.5) * (self.amax - self.amin) * da).astype(f32)
    grads, _ = dense_backward(self.actor, atape, dy)
    return loss, grads

  def train(self, exp, weights=None):
    """exp: [B, 2, ...] arrays (observation, action, reward, discount)."""
    obs, obs2 = exp['observation'][:, 0], exp['observation'][:, 1]
    act, r, d = exp['action'][:, 0], exp['reward'][:, 0], exp['discount'][:, 0]
    closs, cgrads = self.critic_grads(obs, act, r, d, obs2, weights)
    self.critic_opt.apply(self.critic.params(), self._clip(cgrads))
    aloss, agrads = self.actor_grads(obs, weights)
    self.actor_opt.apply(self.actor.params(), self._clip(agrads))
    self.train_step_counter += 1
    self._update_target()
    return dict(loss=f32(aloss + closs), actor_loss=aloss, critic_loss=closs)
