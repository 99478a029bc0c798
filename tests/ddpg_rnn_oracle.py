"""numpy restatement of the recurrent DdpgAgent losses and train step (TEST INFRASTRUCTURE), on
oracle.lstm's LSTM and dense stacks.

Follows agents/ddpg/ddpg_agent.py with stateful networks (data_converter.AsTransition(
squeeze_time_dim=False), trajectory.to_transition): transition t of a [B, T] sequence is
(obs[:, t], step_type[:, t], action[:, t], reward[:, t], discount[:, t], obs[:, t+1] with
next_step_type[:, t]).  The online actor and critic run over obs[:, :-1] with step_type[:, :-1],
the targets over obs[:, 1:] with next_step_type[:, :-1], all from the zero state.
  critic_loss: sum over time of the element loss (no LAST mask), times w_b, mean over B;
  actor_loss:  dqda = d(sum of all Q)/da through the critic's recurrence, c = clip(dqda),
               sum_b w_b sum_{t,k} c^2 / (B A);
  _train:      critic step, actor step against the updated critic, counter += 1, Periodically
               soft update of the target critic and actor.
"""
import copy

import numpy as np

from oracle import ddpg as oddpg
from oracle import lstm as olstm
from oracle import optim

f32 = np.float32


def seq_critic_loss(q, tq, reward, discount, kind=oddpg.HUBER, gamma=1.0, reward_scale=1.0,
                    weights=None):
  """q, tq [B*(T-1)]; reward, discount [B, T-1].  Returns (loss, td_loss [B], dq [B*(T-1)])."""
  B, Tm = np.asarray(reward).shape
  y = (f32(reward_scale) * np.asarray(reward, f32).reshape(-1) +
       f32(gamma) * np.asarray(discount, f32).reshape(-1) * tq).astype(f32)
  l, g = oddpg.element_loss(y, q, kind)
  w = np.broadcast_to(np.asarray(1.0 if weights is None else weights, f32), (B,))
  td_loss = l.reshape(B, Tm).sum(1, dtype=f32)
  loss = f32(np.sum(td_loss * w, dtype=f32) / f32(B))
  return loss, td_loss, (g * np.repeat(w / f32(B), Tm)).astype(f32)


def seq_actor_loss(dqda, B, dqda_clipping=None, weights=None):
  """dqda [B*(T-1), A]; returns (loss, dloss/da [B*(T-1), A])."""
  N, A = dqda.shape
  c = dqda if dqda_clipping is None else np.clip(dqda, -f32(dqda_clipping), f32(dqda_clipping))
  c = c.astype(f32)
  w = np.repeat(np.broadcast_to(np.asarray(1.0 if weights is None else weights, f32), (B,)),
                N // B)[:, None]
  inv = f32(1) / (f32(B) * f32(A))
  return f32(np.sum(c * c * w, dtype=f32) * inv), (f32(-2) * w * c * inv).astype(f32)


class RnnCritic(object):
  """Observation / action dense branches -> concat -> joint dense stack -> stacked LSTM -> output
  dense stack ending in Dense(1).  Layers are {'w', 'b', 'act'}; cells [W, U, b].  `step_type`
  [B, T] must be set before each forward; rows are the B*T steps in batch-major order."""

  def __init__(self, obs, act, joint, cells, post):
    self.obs, self.act, self.joint, self.post = obs, act, joint, post
    self.cells = [list(c) for c in cells]
    self.step_type = None

  def params(self):
    dense = lambda ls: [p for l in ls for p in (l['w'], l['b'])]   # noqa: E731
    return (dense(self.obs) + dense(self.act) + dense(self.joint) +
            [p for c in self.cells for p in c] + dense(self.post))

  def forward(self, obs, act, keep=False):
    B, T = self.step_type.shape
    h, otape = olstm._dense_stack_fwd(self.obs, obs)
    a, atape = olstm._dense_stack_fwd(self.act, act)
    x, jtape = olstm._dense_stack_fwd(self.joint, np.concatenate([h, a], 1).astype(f32))
    hs, _, caches = olstm.stacked_forward(x.reshape(B, T, -1), self.cells, self.step_type)
    q, ptape = olstm._dense_stack_fwd(self.post, hs.reshape(B * T, -1).astype(f32))
    q = q.reshape(-1)
    return (q, (otape, atape, jtape, caches, ptape, h.shape[1])) if keep else q

  def backward(self, tape, dq):
    """Returns (grads aligned with params(), dLoss/d(action) [B*T, A])."""
    otape, atape, jtape, caches, ptape, hw = tape
    B, T = self.step_type.shape
    dh, gpost = olstm._dense_stack_bwd(self.post, ptape, np.asarray(dq, f32).reshape(-1, 1))
    dx, cgrads = olstm.stacked_backward(caches, dh.reshape(B, T, -1))
    dcat, gjoint = olstm._dense_stack_bwd(self.joint, jtape, dx.reshape(B * T, -1).astype(f32))
    _, gobs = olstm._dense_stack_bwd(self.obs, otape, dcat[:, :hw])
    da, gact = olstm._dense_stack_bwd(self.act, atape, dcat[:, hw:])
    grads = gobs + gact + gjoint + [g for cg in cgrads for g in cg] + gpost
    return [np.asarray(g, f32) for g in grads], np.asarray(da, f32)


class RecurrentDdpgOracle(object):
  """actor: oracle.lstm.RnnNet whose post stack ends in Dense(A, tanh); critic: RnnCritic.
  exp: dict of [B, T, ...] arrays (observation, action, reward, discount, step_type,
  next_step_type)."""

  def __init__(self, actor, critic, amin, amax, actor_opt, critic_opt, gamma=1.0,
               reward_scale=1.0, tau=1.0, target_update_period=1, loss=oddpg.HUBER,
               dqda_clipping=None, gradient_clipping=None):
    self.actor, self.critic = actor, critic
    self.ta, self.tc = copy.deepcopy(actor), copy.deepcopy(critic)
    self.amin, self.amax = np.asarray(amin, f32), np.asarray(amax, f32)
    self.actor_opt, self.critic_opt = actor_opt, critic_opt
    self.gamma, self.reward_scale, self.loss = gamma, reward_scale, loss
    self.dqda_clipping, self.clip = dqda_clipping, gradient_clipping
    self.train_step_counter = 0
    self._update_target = optim.Periodically(
        lambda: optim.soft_variables_update(self.critic.params() + self.actor.params(),
                                            self.tc.params() + self.ta.params(), tau),
        target_update_period)

  def _clip(self, grads):
    return grads if self.clip is None else [optim.clip_by_norm(g, self.clip) for g in grads]

  @staticmethod
  def windows(exp):
    obs = np.asarray(exp['observation'], f32)
    B, T = obs.shape[:2]
    st = np.asarray(exp['step_type'])
    return dict(B=B, T=T, x0=obs[:, :-1].reshape(B * (T - 1), -1),
                x1=obs[:, 1:].reshape(B * (T - 1), -1), st0=st[:, :-1],
                st1=np.asarray(exp['next_step_type'])[:, :-1],
                act=np.asarray(exp['action'], f32)[:, :-1].reshape(B * (T - 1), -1),
                r=np.asarray(exp['reward'], f32)[:, :-1], d=np.asarray(exp['discount'], f32)[:, :-1])

  def critic_grads(self, w, weights=None):
    self.ta.step_type = self.tc.step_type = w['st1']
    a2 = oddpg.scale_to_spec(self.ta.forward(w['x1']), self.amin, self.amax)
    tq = self.tc.forward(w['x1'], a2)
    self.critic.step_type = w['st0']
    q, tape = self.critic.forward(w['x0'], w['act'], keep=True)
    loss, _, dq = seq_critic_loss(q, tq, w['r'], w['d'], self.loss, self.gamma,
                                  self.reward_scale, weights)
    return loss, self.critic.backward(tape, dq)[0], dq

  def dqda(self, w, a):
    self.critic.step_type = w['st0']
    _, tape = self.critic.forward(w['x0'], a, keep=True)
    return self.critic.backward(tape, np.ones(a.shape[0], f32))[1]

  def actor_grads(self, w, weights=None):
    self.actor.step_type = w['st0']
    y, atape = self.actor.forward(w['x0'], keep=True)
    dqda = self.dqda(w, oddpg.scale_to_spec(y, self.amin, self.amax))
    loss, da = seq_actor_loss(dqda, w['B'], self.dqda_clipping, weights)
    dy = (f32(0.5) * (self.amax - self.amin) * da).astype(f32)
    self.actor.step_type = w['st0']
    return loss, [np.asarray(g, f32) for g in self.actor.backward(atape, dy)], dqda

  def train(self, exp, weights=None):
    w = self.windows(exp)
    closs, cgrads, _ = self.critic_grads(w, weights)
    cgrads = self._clip(cgrads)
    self.critic_opt.apply(self.critic.params(), cgrads)
    aloss, agrads, _ = self.actor_grads(w, weights)
    agrads = self._clip(agrads)
    self.actor_opt.apply(self.actor.params(), agrads)
    self.train_step_counter += 1
    self._update_target()
    return dict(loss=f32(aloss + closs), actor_loss=aloss, critic_loss=closs,
                critic_grads=cgrads, actor_grads=agrads)
