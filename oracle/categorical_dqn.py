"""numpy restatement of CategoricalDqnAgent's loss and train step (TEST INFRASTRUCTURE).

Follows agents/categorical_dqn/categorical_dqn_agent.py: the support :192-196 (tf.linspace),
_loss :271-518, _next_q_distribution :520-556, project_distribution :562-731;
policies/categorical_q_policy.py:139-145 (np.linspace support) and :174-190 (expected Q, masked
actions at -inf, greedy = first argmax); utils/common.py convert_q_logits_to_values and
aggregate_losses :1400-1476; tf.nn.softmax_cross_entropy_with_logits_v2.
"""
import copy

import numpy as np

from oracle import optim
from oracle import value_ops

f32 = np.float32


def tf_linspace(start, stop, num):
  """tf.linspace in float32 (the agent's support, :196): start, start + i * delta, stop with
  delta = (stop - start) / (num - 1), every operation rounded to float32."""
  start, stop = f32(start), f32(stop)
  delta = f32(stop - start) / f32(num - 1)
  mid = (start + (np.arange(1, num - 1).astype(f32) * delta).astype(f32)).astype(f32)
  return np.concatenate([[start], mid, [stop]]).astype(f32)


def policy_support(min_q_value, max_q_value, num_atoms):
  """np.linspace(..., dtype=float32) (the policy's support, categorical_q_policy.py:141-144)."""
  return np.linspace(min_q_value, max_q_value, num_atoms, dtype=np.float32)


def softmax(logits):
  logits = np.asarray(logits, dtype=f32)
  e = np.exp(logits - logits.max(axis=-1, keepdims=True)).astype(f32)
  return (e / e.sum(axis=-1, keepdims=True, dtype=f32)).astype(f32)


def convert_q_logits_to_values(logits, support):
  """common.convert_q_logits_to_values: sum_j support_j softmax(logits)_j over the last axis."""
  return np.sum(softmax(logits) * np.asarray(support, dtype=f32), axis=-1, dtype=f32)


def greedy_action(q_values, mask=None):
  """categorical_q_policy.py:184-190 + greedy_policy: masked actions at -inf, first argmax."""
  q = np.asarray(q_values, dtype=f32)
  if mask is not None:
    q = np.where(np.asarray(mask).astype(bool), q, f32(-np.inf))
  return np.argmax(q, axis=-1)


def project_distribution(supports, weights, target_support):
  """project_distribution (:562-731), clipped-quotient form: [B, N] (supports, weights) onto the
  equally spaced target_support [N]."""
  supports = np.asarray(supports, dtype=f32)
  weights = np.asarray(weights, dtype=f32)
  target_support = np.asarray(target_support, dtype=f32)
  delta_z = f32(target_support[1] - target_support[0])                     # :607-609
  v_min, v_max = target_support[0], target_support[-1]                     # :651
  clipped = np.clip(supports, v_min, v_max)[:, None, :]                    # :660
  numerator = np.abs(clipped - target_support[None, :, None]).astype(f32)  # :697
  quotient = (f32(1) - (numerator / delta_z).astype(f32)).astype(f32)      # :698
  clipped_quotient = np.clip(quotient, f32(0), f32(1))                     # :710
  return np.sum(clipped_quotient * weights[:, None, :], axis=2, dtype=f32)  # :726-729


def target_support(reward, discount, support, gamma=1.0, reward_scale=1.0):
  """Bellman-shifted support [B, N] and (returns, final discount) of :377-432."""
  reward = np.asarray(reward, dtype=f32)
  discount = np.asarray(discount, dtype=f32)
  support = np.asarray(support, dtype=f32)
  if reward.shape[1] == 2:                                                 # n_step_update == 1
    d, r = discount[:, 0:1], reward[:, 0:1]
    next_value_term = (d * support[None]).astype(f32)                      # :384-386
    reward_term = (f32(reward_scale) * r).astype(f32)                      # :392-394
    ts_ = (reward_term + (f32(gamma) * next_value_term).astype(f32)).astype(f32)
    return ts_, r[:, 0] * f32(reward_scale), (f32(gamma) * d[:, 0]).astype(f32)
  rewards = (f32(reward_scale) * reward[:, :-1]).astype(f32)               # :403
  discounts = (f32(gamma) * discount[:, :-1]).astype(f32)                  # :404
  returns = value_ops.discounted_return(rewards, discounts, time_major=False,
                                        provide_all_returns=False)         # :409-415
  final = np.ones(discounts.shape[0], dtype=f32)
  for t in range(discounts.shape[1]):                                      # reduce_prod (:420)
    final = (final * discounts[:, t]).astype(f32)
  ts_ = (returns[:, None] + (final[:, None] * support[None]).astype(f32)).astype(f32)
  return ts_, returns, final


def c51_loss(q_logits, next_logits, actions, reward, discount, support, gamma=1.0,
             reward_scale=1.0, next_mask=None, select_support=None, global_batch=None,
             reg_loss=None):
  """Everything after the network evaluations in CategoricalDqnAgent._loss.

  q_logits / next_logits [B, A, N]; reward / discount [B, T].  `select_support` is the support of
  the target greedy policy (np.linspace, default `support`).  Sample weights do not enter: the
  reference never passes them to aggregate_losses (:463-466).  Returns dict(loss, per_example,
  dlogits [B, A, N] = dLoss/dq_logits, target [B, N], returns, final_discount, best).
  """
  q_logits = np.asarray(q_logits, dtype=f32)
  next_logits = np.asarray(next_logits, dtype=f32)
  support = np.asarray(support, dtype=f32)
  B, A, N = q_logits.shape
  sel = support if select_support is None else np.asarray(select_support, dtype=f32)
  next_q = convert_q_logits_to_values(next_logits, sel)                   # :541-544
  best = greedy_action(next_q, next_mask)                                  # :548-550
  next_p = softmax(next_logits)[np.arange(B), best]                        # :556
  ts_, returns, final = target_support(reward, discount, support, gamma, reward_scale)
  target = project_distribution(ts_, next_p, support)                      # :434-438
  acts = np.asarray(actions, dtype=np.int64)
  logits = q_logits[np.arange(B), acts]                                    # :441-444
  mx = logits.max(axis=1, keepdims=True)
  sh = (logits - mx).astype(f32)
  lse = np.log(np.sum(np.exp(sh), axis=1, keepdims=True, dtype=f32)).astype(f32)
  per_example = np.sum(target * (lse - sh), axis=1, dtype=f32)             # :459-461
  gb = f32(global_batch if global_batch is not None else B)
  loss = f32(np.sum(per_example, dtype=f32) / gb)                          # aggregate_losses
  total = loss if reg_loss is None else f32(loss + f32(reg_loss))
  p = np.exp(sh - lse).astype(f32)
  dlogits = np.zeros_like(q_logits)
  dlogits[np.arange(B), acts] = ((p * target.sum(axis=1, keepdims=True, dtype=f32) - target) /
                                 gb).astype(f32)
  return dict(loss=total, weighted=loss, per_example=per_example, dlogits=dlogits, target=target,
              returns=returns, final_discount=final, best=best)


class CategoricalDqnOracle(object):
  """One-replica CategoricalDqnAgent learner on numpy Sequentials (oracle/nn.py).

  Dense layer dicts may carry an 'l2' coefficient: coef * sum(w^2) joins the loss and
  2 * coef * w the gradient, as Keras kernel regularisers do through aggregate_losses.
  """

  def __init__(self, q_net, optimizer, num_atoms, min_q_value=-10.0, max_q_value=10.0, gamma=1.0,
               reward_scale=1.0, target_update_tau=1.0, target_update_period=1,
               gradient_clipping=None):
    self.q_net = q_net
    self.target_net = copy.deepcopy(q_net)
    self.optimizer = optimizer
    self.num_atoms = num_atoms
    self.support = tf_linspace(min_q_value, max_q_value, num_atoms)
    self.select_support = policy_support(min_q_value, max_q_value, num_atoms)
    self.gamma, self.reward_scale = gamma, reward_scale
    self.gradient_clipping = gradient_clipping
    self.train_step_counter = 0
    self._update_target = optim.Periodically(
        lambda: optim.soft_variables_update(self.q_net.params(), self.target_net.params(),
                                            target_update_tau), target_update_period)

  def _reg(self):
    reg, pairs = f32(0), []
    for l in self.q_net.layers:
      coef = l.get('l2', 0.0)
      if coef:
        reg = f32(reg + f32(coef) * np.sum(l['w'] * l['w'], dtype=f32))
        pairs.append((l['w'], coef))
    return reg, pairs

  def loss(self, exp, keep=False):
    """exp: dict of [B, T, ...] arrays with keys observation, action, reward, discount and
    optionally mask ([B, T, A] action constraint)."""
    obs0, obsn = exp['observation'][:, 0], exp['observation'][:, -1]
    q, tape = self.q_net.forward(obs0, keep=True)
    nxt = self.target_net.forward(obsn)
    B = q.shape[0]
    A = q.shape[1] // self.num_atoms
    mask = exp.get('mask')
    reg, _ = self._reg()
    out = c51_loss(q.reshape(B, A, self.num_atoms), nxt.reshape(B, A, self.num_atoms),
                   exp['action'][:, 0], exp['reward'], exp['discount'], self.support, self.gamma,
                   self.reward_scale, next_mask=None if mask is None else mask[:, -1],
                   select_support=self.select_support, reg_loss=reg)
    if keep:
      out['tape'] = tape
    return out

  def train(self, exp):
    out = self.loss(exp, keep=True)
    B = out['dlogits'].shape[0]
    grads = self.q_net.backward(out['tape'], out['dlogits'].reshape(B, -1))
    _, pairs = self._reg()
    params = self.q_net.params()
    for w, coef in pairs:
      i = next(k for k, p in enumerate(params) if p is w)
      grads[i] = (grads[i] + f32(2.0 * coef) * w).astype(f32)
    if self.gradient_clipping is not None:
      grads = [optim.clip_by_norm(g, self.gradient_clipping) for g in grads]
    out['grads'] = [g.copy() for g in grads]
    self.optimizer.apply(params, grads)
    self.train_step_counter += 1
    self._update_target()
    return out
