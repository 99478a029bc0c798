"""numpy restatement of the recurrent SacAgent losses and train step (TEST INFRASTRUCTURE), on
oracle.sac's tanh-Normal sample, oracle.lstm's LSTM and dense stacks and ddpg_rnn_oracle's
recurrent critic.

Follows agents/sac/sac_agent.py with stateful networks (data_converter.AsTransition(
squeeze_time_dim=False)): transition t of a [B, T] sequence is row b*(T-1) + t.  The actor's a'
and the target critics run over obs[:, 1:] with next_step_type[:, :-1]; the online critics and the
actor-step and alpha-step samples over obs[:, :-1] with step_type[:, :-1]; all from the zero state.
  critic_loss: cw sum_b w_b sum_t [(y - q1)^2 + (y - q2)^2] / B,
               y = rs r + gamma d (min(tq1, tq2) - alpha log pi');
  actor_loss:  aw sum_b w_b sum_t (alpha log pi - min(q1, q2)) / B, dQ/da through each critic's
               recurrence, the min's gradient on q1 where q1 <= q2;
  alpha_loss:  alw coef sum_b w_b sum_t (-log pi - H) / B, coef = log alpha or alpha;
  _train:      critic step, actor step against the updated critics, alpha step against the updated
               actor, counter += 1, Periodically soft update of both target critics.
A row of weight 0 adds exactly 0 to every loss.
"""
import copy

import numpy as np

from oracle import optim
from oracle import sac as osac
import ddpg_rnn_oracle

f32 = np.float32
RnnCritic = ddpg_rnn_oracle.RnnCritic


def _rows(per_step, B, weights):
  """sum_b w_b sum_t per_step / B, with rows of weight 0 adding exactly 0."""
  w = np.broadcast_to(np.asarray(1.0 if weights is None else weights, f32), (B,))
  row = np.asarray(per_step, f32).reshape(B, -1).sum(1, dtype=f32)
  return f32(np.sum(np.where(w == 0, f32(0), row * w), dtype=f32) / f32(B)), w


def seq_critic_loss(q1, q2, tq1, tq2, next_logp, reward, discount, log_alpha, gamma=1.0,
                    reward_scale=1.0, weights=None, loss_weight=1.0):
  """q*, tq*, next_logp [B*(T-1)]; reward, discount [B, T-1].  Returns (loss, dq1, dq2)."""
  B, Tm = np.asarray(reward).shape
  tq = np.minimum(tq1, tq2) - np.exp(f32(log_alpha)) * next_logp
  y = (f32(reward_scale) * np.asarray(reward, f32).reshape(-1) +
       f32(gamma) * np.asarray(discount, f32).reshape(-1) * tq).astype(f32)
  e1, e2 = y - q1, y - q2
  loss, w = _rows(e1 * e1 + e2 * e2, B, weights)
  c = np.repeat(f32(loss_weight) * w / f32(B), Tm).astype(f32)
  return f32(loss_weight * loss), (-2 * e1 * c).astype(f32), (-2 * e2 * c).astype(f32)


def seq_actor_loss(q1, q2, logp, log_alpha, B, weights=None, loss_weight=1.0):
  """Returns (loss, dlogp, dq1, dq2), each gradient [B*(T-1)]."""
  alpha = np.exp(f32(log_alpha))
  loss, w = _rows(alpha * logp - np.minimum(q1, q2), B, weights)
  k = np.repeat(f32(loss_weight) * w / f32(B), q1.shape[0] // B).astype(f32)
  first = q1 <= q2
  return (f32(loss_weight * loss), (alpha * k).astype(f32), np.where(first, -k, 0).astype(f32),
          np.where(first, 0, -k).astype(f32))


def seq_alpha_loss(logp, log_alpha, B, target_entropy, use_log_alpha=True, weights=None,
                   loss_weight=1.0):
  """Returns (loss, dloss/dlog_alpha)."""
  s, _ = _rows(-logp - f32(target_entropy), B, weights)
  la = f32(log_alpha)
  coef, dcoef = (la, f32(1)) if use_log_alpha else (np.exp(la), np.exp(la))
  return f32(loss_weight * coef * s), f32(loss_weight * dcoef * s)


def sample_bwd(head, u, eps, amin, amax, da, dlogp):
  """dLoss/dhead [N, 2A] from dLoss/da [N, A] and dLoss/dlogp [N] (oracle.sac's chain)."""
  A = head.shape[1] // 2
  half = (amax - amin) / 2
  t = np.tanh(u)
  du = da * half * (1 - t * t) + dlogp[:, None] * 2 * t
  return np.concatenate([du, du * np.exp(head[:, A:]) * eps - dlogp[:, None]], 1).astype(f32)


class RecurrentSacOracle(object):
  """actor: oracle.lstm.RnnNet whose post stack ends in a linear Dense(2A); critics: RnnCritic.
  exp: dict of [B, T, ...] arrays (observation, action, reward, discount, step_type,
  next_step_type); eps_*: [B, T-1, A] draws."""

  def __init__(self, actor, critic1, critic2, amin, amax, actor_opt, critic_opt, alpha_opt,
               gamma=1.0, reward_scale=1.0, tau=1.0, period=1, target_entropy=None,
               initial_log_alpha=0.0, critic_loss_weight=0.5, actor_loss_weight=1.0,
               alpha_loss_weight=1.0, use_log_alpha=True):
    self.actor, self.c1, self.c2 = actor, critic1, critic2
    self.t1, self.t2 = copy.deepcopy(critic1), copy.deepcopy(critic2)
    self.amin, self.amax = np.asarray(amin, f32), np.asarray(amax, f32)
    A = self.amin.shape[0]
    self.target_entropy = f32(-A / 2.0 if target_entropy is None else target_entropy)
    self.log_alpha = np.array([initial_log_alpha], f32)
    self.actor_opt, self.critic_opt, self.alpha_opt = actor_opt, critic_opt, alpha_opt
    self.gamma, self.reward_scale = gamma, reward_scale
    self.cw, self.aw, self.alw = critic_loss_weight, actor_loss_weight, alpha_loss_weight
    self.use_log_alpha = use_log_alpha
    self.train_step_counter = 0
    self._update_target = optim.Periodically(
        lambda: optim.soft_variables_update(self.c1.params() + self.c2.params(),
                                            self.t1.params() + self.t2.params(), tau), period)

  windows = staticmethod(ddpg_rnn_oracle.RecurrentDdpgOracle.windows)

  def _sample(self, x, st, eps, keep=False):
    self.actor.step_type = st
    head, tape = self.actor.forward(x, keep=True)
    a, logp, u = osac.sample_and_log_prob(head, eps.reshape(head.shape[0], -1), self.amin,
                                          self.amax)
    return (a, logp, (head, tape, u)) if keep else (a, logp)

  def _q(self, net, x, a, st, keep=False):
    net.step_type = st
    return net.forward(x, a, keep=keep)

  def critic_grads(self, w, eps, weights=None):
    """(loss, grads of c1 + c2)."""
    a2, logp2 = self._sample(w['x1'], w['st1'], eps)
    tq1, tq2 = self._q(self.t1, w['x1'], a2, w['st1']), self._q(self.t2, w['x1'], a2, w['st1'])
    q1, tape1 = self._q(self.c1, w['x0'], w['act'], w['st0'], keep=True)
    q2, tape2 = self._q(self.c2, w['x0'], w['act'], w['st0'], keep=True)
    loss, dq1, dq2 = seq_critic_loss(q1, q2, tq1, tq2, logp2, w['r'], w['d'], self.log_alpha[0],
                                     self.gamma, self.reward_scale, weights, self.cw)
    return loss, self.c1.backward(tape1, dq1)[0] + self.c2.backward(tape2, dq2)[0]

  def actor_grads(self, w, eps, weights=None):
    """(loss, actor grads, dQ1/da + dQ2/da [N, A])."""
    eps = eps.reshape(w['x0'].shape[0], -1).astype(f32)
    a, logp, (head, atape, u) = self._sample(w['x0'], w['st0'], eps, keep=True)
    q1, t1 = self._q(self.c1, w['x0'], a, w['st0'], keep=True)
    q2, t2 = self._q(self.c2, w['x0'], a, w['st0'], keep=True)
    loss, dlogp, dq1, dq2 = seq_actor_loss(q1, q2, logp, self.log_alpha[0], w['B'], weights,
                                           self.aw)
    da = self.c1.backward(t1, dq1)[1] + self.c2.backward(t2, dq2)[1]
    dhead = sample_bwd(head, u, eps, self.amin, self.amax, da, dlogp)
    self.actor.step_type = w['st0']
    return loss, [np.asarray(g, f32) for g in self.actor.backward(atape, dhead)], da

  def alpha_grad(self, w, eps, weights=None):
    _, logp3 = self._sample(w['x0'], w['st0'], eps)
    return seq_alpha_loss(logp3, self.log_alpha[0], w['B'], self.target_entropy,
                          self.use_log_alpha, weights, self.alw)

  def train(self, exp, eps_next, eps_actor, eps_alpha, weights=None):
    w = self.windows(exp)
    closs, cgrads = self.critic_grads(w, eps_next, weights)
    self.critic_opt.apply(self.c1.params() + self.c2.params(), cgrads)
    aloss, agrads, _ = self.actor_grads(w, eps_actor, weights)
    self.actor_opt.apply(self.actor.params(), agrads)
    alloss, dla = self.alpha_grad(w, eps_alpha, weights)
    self.alpha_opt.apply([self.log_alpha], [np.array([dla], f32)])
    self.train_step_counter += 1
    self._update_target()
    return dict(loss=f32(closs + aloss + alloss), critic_loss=closs, actor_loss=aloss,
                alpha_loss=alloss, critic_grads=cgrads, actor_grads=agrads, dlog_alpha=dla)
