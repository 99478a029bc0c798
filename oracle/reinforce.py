"""numpy restatement of ReinforceAgent update math (TEST INFRASTRUCTURE).

Follows agents/reinforce/reinforce_agent.py: _standard_normalize :48-61, _entropy_loss :64-80,
_train :255-311 (returns, one optimiser over actor + value, per-variable clipping), total_loss
:313-440 (num_episodes, valid mask, advantages), policy_gradient_loss :442-506,
entropy_regularization_loss :508-534, value_estimation_loss :536-567.
is_last reads next_step_type, is_boundary reads step_type (trajectories/trajectory.py:91-99).

The backward is written out by hand (tests/test_oracle_reinforce.py checks it against float64
autograd).  value_preds are not stop-gradient inside the advantages, so with a baseline the
policy-gradient loss also trains the value network.  With g_i = d(pg)/d(adv_n_i),
D = sigma + eps and S = sum_i g_i (adv_i - mean):
  d(pg)/d(adv_j) = (g_j - mean(g)) / D - (adv_j - mean) S / (N sigma D^2)      (normalised)
  d(pg)/d(V_j)   = -d(pg)/d(adv_j)
where sigma = 0 the second term is defined as 0 (the reference produces 0 * inf = NaN there).
The Normal / Categorical formulas come from oracle.ppo and oracle.ppo_discrete.
"""
import numpy as np

from oracle import optim
from oracle import ppo
from oracle import ppo_discrete
from oracle import value_ops

f32 = np.float32
STEP_FIRST, STEP_MID, STEP_LAST = 0, 1, 2
EPS = f32(np.finfo(np.float32).eps)
NO_EPISODE_MESSAGE = ('No complete episode found. REINFORCE requires full episodes to compute '
                      'losses.')


def compute_returns(reward, discount, next_step_type, gamma):
  """discounted_return of reward with (next_step_type != LAST) * discount * gamma, batch-major,
  final value 0 (:262-269)."""
  mask = (np.asarray(next_step_type) != STEP_LAST).astype(f32)
  disc = (mask * np.asarray(discount, f32) * f32(gamma)).astype(f32)
  return value_ops.discounted_return(reward, disc, time_major=False)


def valid_mask(next_step_type):
  """1 where some t' >= t of the row has is_last (reverse cumsum > 0, :344-346)."""
  is_last = (np.asarray(next_step_type) == STEP_LAST).astype(f32)
  return (np.cumsum(is_last[:, ::-1], axis=1)[:, ::-1] > 0).astype(f32)


def num_episodes(next_step_type):
  return f32(np.sum(np.asarray(next_step_type) == STEP_LAST))


def standard_normalize(x):
  """(x - mean) / (sqrt(var) + eps), population moments over every entry (:48-61)."""
  x = np.asarray(x, f32)
  mean = np.mean(x, dtype=f32)
  var = np.mean((x - mean) ** 2, dtype=f32)
  return ((x - mean) / (np.sqrt(var) + EPS)).astype(f32)


def policy_gradient_loss(logp, is_boundary, adv, num_eps, weights=None):
  """-sum(logp * ~is_boundary * adv * weights) / num_episodes (:442-506)."""
  t = np.asarray(logp, f32) * (1 - np.asarray(is_boundary, f32)) * np.asarray(adv, f32)
  if weights is not None:
    t = t * np.asarray(weights, f32)
  return f32(-np.sum(t, dtype=f32) / f32(num_eps))


def entropy_regularization_loss(entropy, weights, coef):
  """coef * mean(-H * weights) over all entries; 0 when coef is falsy (:64-80, :508-534)."""
  if not coef:
    return f32(0)
  e = -np.asarray(entropy, f32)
  if weights is not None:
    e = e * np.asarray(weights, f32)
  return f32(np.mean(e, dtype=f32) * f32(coef))


def value_estimation_loss(value_preds, returns, num_eps, weights, coef):
  """coef * sum((returns - V)^2 * weights) / num_episodes (:536-567)."""
  err = (np.asarray(returns, f32) - np.asarray(value_preds, f32)) ** 2
  if weights is not None:
    err = err * np.asarray(weights, f32)
  return f32(np.sum(err, dtype=f32) * f32(coef) / f32(num_eps))


def loss_and_grads(logp, ent, returns, value, step_type, next_step_type, weights=None,
                   use_advantage=True, normalize=True, entropy_coef=None, value_coef=0.2):
  """The loss terms of total_loss (without regularisation) and their gradients w.r.t. log pi,
  the entropy H and the value predictions.  Every array is [B, T]; value may be None."""
  B, T = np.shape(returns)
  N = f32(B * T)
  ret = np.asarray(returns, f32)
  ne = num_episodes(next_step_type)
  if ne == 0:
    raise ValueError(NO_EPISODE_MESSAGE)
  w = valid_mask(next_step_type)
  if weights is not None:
    w = (np.asarray(weights, f32) * w).astype(f32)
  c = ((np.asarray(step_type) != STEP_LAST) * w).astype(f32)
  use_adv = use_advantage and value is not None
  adv = (ret - value).astype(f32) if use_adv else ret
  mean = np.mean(adv, dtype=f32)
  sigma = np.sqrt(np.mean((adv - mean) ** 2, dtype=f32))
  D = f32(sigma + EPS)
  adv_n = ((adv - mean) / D).astype(f32) if normalize else adv
  pg = policy_gradient_loss(logp, np.asarray(step_type) == STEP_LAST, adv_n, ne, w)
  en = entropy_regularization_loss(ent, w, entropy_coef)
  ve = value_estimation_loss(value, ret, ne, w, value_coef) if value is not None else f32(0)
  g_logp = (-c * adv_n / ne).astype(f32)
  g_ent = (-f32(entropy_coef) * w / N).astype(f32) if entropy_coef else np.zeros_like(w)
  dv = None
  if value is not None:
    dv = (f32(value_coef) * 2 * (value - ret) * w / ne).astype(f32)
    if use_adv:
      g = (-c * np.asarray(logp, f32) / ne).astype(f32)      # d(pg) / d(adv_n)
      if normalize:
        S = np.sum(g * (adv - mean), dtype=f32)
        coef = S / (N * sigma * D * D) if sigma > 0 else f32(0)
        dadv = (g - np.mean(g, dtype=f32)) / D - (adv - mean) * coef
      else:
        dadv = g
      dv = (dv - dadv).astype(f32)
  return dict(policy_gradient_loss=pg, entropy_regularization_loss=en, value_estimation_loss=ve,
              num_episodes=ne, total=f32(pg + en + ve)), (g_logp, g_ent, dv)


def normal_param_grads(loc, scale, action, g_logp, g_ent):
  """(dloc, dscale) [N, A] of g_logp * log N(a; loc, scale) + g_ent * H, log pi / H summed over A."""
  d = action - loc
  inv = 1.0 / scale
  dloc = (g_logp[:, None] * d * inv * inv).astype(f32)
  dscale = (g_logp[:, None] * (d * d * inv ** 3 - inv) + g_ent[:, None] * inv).astype(f32)
  return dloc, dscale


def l2_terms(net):
  """(loss, grads aligned with net.params()) of the layers' `l2` kernel regularisers."""
  loss, grads = f32(0), []
  for l in net.layers:
    if l['kind'] not in ('conv', 'dense'):
      continue
    coef = f32(l.get('l2', 0.0))
    loss = f32(loss + coef * np.sum(l['w'] * l['w'], dtype=f32))
    grads.append((2 * coef * l['w']).astype(f32))
    if l.get('b') is not None:
      grads.append(np.zeros_like(l['b']))
  return loss, grads


class ReinforceOracle(object):
  """ReinforceAgent train step on numpy nets.

  actor: oracle.nn.Sequential ending in a linear Dense(A).  Normal head (discrete=False): loc =
  shift + half_range * tanh(m_raw), scale = softplus(std_bias) (as oracle.ppo.PPOOracle).
  Categorical head (discrete=True): the Dense output is the logits.  value: Sequential ending in
  Dense(1), or None.  Layer dicts may carry an 'l2' kernel-regulariser coefficient.
  Experience dicts hold [B, T] step_type / next_step_type / reward / discount, [B, T, ...]
  observation and action ([B, T, A] float, or [B, T] int for discrete)."""

  def __init__(self, actor, value, optimizer, std_bias=None, amin=None, amax=None,
               discrete=False, value_estimation_loss_coef=0.2, use_advantage_loss=True,
               gamma=1.0, normalize_returns=True, gradient_clipping=None,
               entropy_regularization=None):
    self.actor, self.value, self.opt, self.discrete = actor, value, optimizer, discrete
    if not discrete:
      self.std_bias = np.asarray(std_bias, f32)
      self.amin, self.amax = np.asarray(amin, f32), np.asarray(amax, f32)
    self.value_coef = value_estimation_loss_coef
    self.use_advantage = use_advantage_loss
    self.gamma, self.normalize = gamma, normalize_returns
    self.gradient_clipping = gradient_clipping
    self.entropy_coef = entropy_regularization
    self.train_step_counter = 0

  def params(self):
    p = self.actor.params()
    if not self.discrete:
      p = p + [self.std_bias]
    return p + (self.value.params() if self.value is not None else [])

  def dist(self, obs):
    out, tape = self.actor.forward(obs, keep=True)
    if self.discrete:
      return out, tape
    half, shift = (self.amax - self.amin) / 2, (self.amax + self.amin) / 2
    loc = (shift + half * np.tanh(out)).astype(f32)
    scale = np.broadcast_to(ppo.softplus(self.std_bias), loc.shape).astype(f32)
    return (loc, scale, out), tape

  def loss_and_grads(self, exp, weights=None):
    B, T = exp['reward'].shape
    N = B * T
    ret = compute_returns(exp['reward'], exp['discount'], exp['next_step_type'], self.gamma)
    obs = exp['observation'].reshape((N,) + exp['observation'].shape[2:])
    params, atape = self.dist(obs)
    if self.discrete:
      action = exp['action'].reshape(N)
      logp = ppo_discrete.categorical_log_prob(params, action)
      ent = ppo_discrete.categorical_entropy(params)
    else:
      loc, scale, m_raw = params
      action = exp['action'].reshape(N, -1)
      logp = ppo.normal_log_prob(loc, scale, action)
      ent = ppo.normal_entropy(scale)
    v = vtape = None
    if self.value is not None:
      v, vtape = self.value.forward(obs, keep=True)
      v = v[:, 0].reshape(B, T)
    info, (g_logp, g_ent, dv) = loss_and_grads(
        logp.reshape(B, T), ent.reshape(B, T), ret, v, exp['step_type'], exp['next_step_type'],
        weights, self.use_advantage, self.normalize, self.entropy_coef, self.value_coef)
    g_logp, g_ent = g_logp.reshape(N), g_ent.reshape(N)
    if self.discrete:
      dlogits = ppo_discrete.categorical_loss_grad(params, action, g_logp, g_ent)
      grads = self.actor.backward(atape, dlogits)
    else:
      dloc, dscale = normal_param_grads(loc, scale, action, g_logp, g_ent)
      half = (self.amax - self.amin) / 2
      dm_raw = (dloc * half * (1 - np.tanh(m_raw) ** 2)).astype(f32)
      sig = 1.0 / (1.0 + np.exp(-self.std_bias))
      grads = self.actor.backward(atape, dm_raw) + [(dscale * sig).sum(axis=0).astype(f32)]
    areg, agrads = l2_terms(self.actor)
    k = len(agrads)
    grads[:k] = [(g + r).astype(f32) for g, r in zip(grads[:k], agrads)]
    vreg = f32(0)
    if self.value is not None:
      vreg, vgrads = l2_terms(self.value)
      vg = self.value.backward(vtape, dv.reshape(N, 1))
      grads = grads + [(g + r).astype(f32) for g, r in zip(vg, vgrads)]
    info['policy_network_regularization_loss'] = areg
    info['value_network_regularization_loss'] = vreg
    info['loss'] = f32(info['total'] + areg + vreg)
    return info, grads

  def train(self, exp, weights=None):
    """_train (:255-311): one step; per-variable clipping (eager_utils.clip_gradient_norms)."""
    info, grads = self.loss_and_grads(exp, weights)
    if self.gradient_clipping:
      grads = [optim.clip_by_norm(g, self.gradient_clipping) for g in grads]
    self.opt.apply(self.params(), grads)
    self.train_step_counter += 1
    return info
