"""numpy restatement of PPO with a Categorical policy (TEST INFRASTRUCTURE).

PPOAgent covers discrete actions with a Categorical over logits (agents/ppo/ppo_agent.py:48;
networks/actor_distribution_network.py:157-158 selects CategoricalProjectionNetwork,
categorical_projection_network.py:88-95).  The distribution formulas are TFP's:
  log_prob(a) = log_softmax(z)[a]  (max-subtracted),  entropy = -sum_j p_j log p_j,
  KL(q || p) = sum_j q_j (log q_j - log p_j)  (`_kl_categorical_categorical`).
The backward w.r.t. the logits is written out by hand (tests/test_oracle_ppo_discrete.py checks it
against torch autograd):
  d logp / dz_j = 1[j=a] - p_j,  dH / dz_j = -p_j (log p_j + H),  dKL(q||p) / dz_j = p_j - q_j.
Everything that does not depend on the distribution (returns, GAE, masks, advantage
normalisation, value loss, normalisers, optimiser) is oracle.ppo's.

`categorical_sample` restates the collect draw of b200rl_categorical_sample over oracle.philox:
u = uniform_f32(philox(counter=(n, call), key=seed).x); the action is the smallest k with
u < cdf_k, cdf the fp32 running sum in index order of exp(z - max) / sum exp(z - max); A-1 if none.
"""
import numpy as np

from oracle import optim
from oracle import philox
from oracle import ppo

f32 = np.float32


def log_softmax(logits):
  z = np.asarray(logits, f32)
  d = (z - z.max(axis=-1, keepdims=True)).astype(f32)
  return (d - np.log(np.exp(d).sum(axis=-1, keepdims=True, dtype=f32))).astype(f32)


def categorical_log_prob(logits, action):
  lp = log_softmax(logits)
  return np.take_along_axis(lp, np.asarray(action, np.int64)[..., None], axis=-1)[..., 0]


def categorical_entropy(logits):
  lp = log_softmax(logits)
  return (-(np.exp(lp) * lp).sum(axis=-1, dtype=f32)).astype(f32)


def categorical_kl(logits_a, logits_b):
  """KL(Categorical(logits_a) || Categorical(logits_b)) per row."""
  la, lb = log_softmax(logits_a), log_softmax(logits_b)
  return (np.exp(la) * (la - lb)).sum(axis=-1, dtype=f32).astype(f32)


def categorical_loss_grad(logits, action, g_logp, g_ent, g_kl=None, old_logits=None):
  """dL/dlogits for per-row scalar weights g_logp (d L / d logp), g_ent (d L / d entropy) and
  g_kl (d L / d KL(old || new))."""
  lp = log_softmax(logits)
  p = np.exp(lp).astype(f32)
  ent = (-(p * lp).sum(axis=-1, dtype=f32)).astype(f32)
  onehot = np.zeros_like(p)
  onehot[np.arange(p.shape[0]), np.asarray(action, np.int64)] = 1
  g = g_logp[:, None] * (onehot - p) + g_ent[:, None] * (-p * (lp + ent[:, None]))
  if g_kl is not None:
    q = np.exp(log_softmax(old_logits))
    g = g + g_kl[:, None] * (p - q)
  return g.astype(f32)


def categorical_cdf(logits):
  """The [N, A] fp32 running cdf, in index order, of exp(z - max) / sum exp(z - max)."""
  z = np.asarray(logits, f32)
  e = np.exp(z - z.max(axis=1, keepdims=True)).astype(f32)
  s = np.zeros(z.shape[0], f32)
  for k in range(z.shape[1]):               # index-order fp32 sums, as the kernel does
    s = (s + e[:, k]).astype(f32)
  cdf = np.zeros_like(e)
  c = np.zeros(z.shape[0], f32)
  for k in range(z.shape[1]):
    c = (c + (e[:, k] / s).astype(f32)).astype(f32)
    cdf[:, k] = c
  return cdf


def categorical_sample(logits, seed, call):
  """(int32 [N] draws, the uniforms u) of the collect policy for Philox call index `call`."""
  cdf = categorical_cdf(logits)
  n, a = cdf.shape
  u = philox.uniform_f32(philox.philox(np.arange(n, dtype=np.uint64), call, seed)[0])
  hit = u[:, None] < cdf
  out = np.where(hit.any(axis=1), hit.argmax(axis=1), a - 1).astype(np.int32)
  return out, u


class CategoricalPPOOracle(ppo.PPOOracle):
  """PPOOracle with a Categorical actor: `actor` is an oracle.nn.Sequential (an optional
  cast_scale / conv / flatten front, then dense layers) ending in the linear logits layer.
  Experience dicts carry integer `action` [B, T] and behaviour `logits` [B, T, A]."""

  def __init__(self, actor, value, optimizer, **kw):
    super().__init__(actor, np.zeros(0, f32), value, np.zeros(0, f32), np.zeros(0, f32),
                     optimizer, **kw)

  def dist(self, obs, keep=False):
    logits, tape = self.actor.forward(obs, keep=True)
    return (logits, tape) if keep else logits

  def params(self):
    return self.actor.params() + self.value.params()

  def _flat_obs(self, exp):
    B, T = exp['reward'].shape
    obs = exp['observation']
    return obs.reshape((B * T,) + obs.shape[2:])

  def preprocess(self, exp):
    B, T = exp['reward'].shape
    vp = self.value.forward(self.norm_obs(self._flat_obs(exp))).reshape(B, T)
    reward = exp['reward'][:, :-1]
    if self.reward_normalizer is not None:
      reward = self.reward_normalizer.normalize(reward, center_mean=False,
                                                clip_value=self.reward_norm_clipping)
    ret, adv = ppo.compute_return_and_advantage(reward, exp['discount'][:, :-1],
                                                exp['next_step_type'][:, :-1], vp, self.gamma,
                                                self.lam, self.use_gae, self.use_td)
    pad = np.zeros((B, 1), f32)
    return vp, np.concatenate([ret, pad], 1), np.concatenate([adv, pad], 1)

  def loss_and_grads(self, obs, action, old_logp, ret, adv_n, v_old, w, B, T, global_batch=None,
                     old_logits=None):
    N = B * T
    gb = f32(global_batch or B)
    denom = f32(T) * gb
    logits, atape = self.dist(obs, keep=True)
    v, vtape = self.value.forward(obs, keep=True)
    v = v[:, 0]
    logp = categorical_log_prob(logits, action)
    ent = categorical_entropy(logits)
    sh = (B, T)
    pg, clip_frac = ppo.policy_gradient_loss(logp.reshape(sh), old_logp.reshape(sh),
                                             adv_n.reshape(sh), w.reshape(sh), self.clip_eps,
                                             self.logp_clip, gb)
    ve = ppo.value_estimation_loss(v.reshape(sh), ret.reshape(sh), w.reshape(sh), self.vf_coef,
                                   self.value_clip, None if v_old is None else v_old.reshape(sh),
                                   gb)
    en = ppo.entropy_regularization_loss(ent.reshape(sh), w.reshape(sh), self.ent_coef, gb)
    use_kl = not (self.initial_beta == 0 and self.kl_cutoff_factor == 0)
    klp, g_kl = f32(0), None
    if use_kl:
      kl = (categorical_kl(old_logits, logits) * w).astype(f32)
      klp = f32(ppo.kl_cutoff_loss(kl, self.kl_cutoff_factor, self.kl_target, self.kl_cutoff_coef)
                + ppo.adaptive_kl_loss(kl, self.beta))
      mean_kl = np.mean(kl, dtype=f32)
      dmean = f32(0)
      if self.kl_cutoff_factor > 0:
        dmean += f32(2 * self.kl_cutoff_coef) * np.maximum(
            mean_kl - f32(self.kl_cutoff_factor * self.kl_target), f32(0))
      if self.beta is not None:
        dmean += f32(self.beta)
      g_kl = (dmean * w / f32(N)).astype(f32)
    total = f32(pg + ve + en + klp)
    # ---- backward: the surrogate and value terms exactly as oracle.ppo, then the logits
    lp, dlp = logp, np.ones(N, f32)
    if self.logp_clip > 0:
      dlp = ((logp >= -self.logp_clip) & (logp <= self.logp_clip)).astype(f32)
      lp = np.clip(logp, -self.logp_clip, self.logp_clip)
    ratio = np.exp(lp - old_logp)
    lo, hi = 1 - self.clip_eps, 1 + self.clip_eps
    ratio_c = np.clip(ratio, lo, hi)
    if self.clip_eps > 0:
      unclipped_is_min = ratio * adv_n <= ratio_c * adv_n
      inside = (ratio >= lo) & (ratio <= hi)
      dobj = np.where(unclipped_is_min, adv_n, np.where(inside, adv_n, 0.0))
    else:
      dobj = adv_n
    g_logp = (-dobj * ratio * dlp * w / denom).astype(f32)
    g_ent = (-f32(self.ent_coef) * w / denom).astype(f32)
    dlogits = categorical_loss_grad(logits, action, g_logp, g_ent, g_kl, old_logits)
    err = (ret - v) ** 2
    derr = -2 * (ret - v)
    if self.value_clip > 0:
      dv_ = v - v_old
      vc = v_old + np.clip(dv_, -self.value_clip, self.value_clip)
      err_c = (ret - vc) ** 2
      use_c = err_c > err
      derr = np.where(use_c, np.where(np.abs(dv_) <= self.value_clip, -2 * (ret - vc), 0.0), derr)
    dv = (f32(self.vf_coef) * derr * w / denom).astype(f32)
    grads = self.actor.backward(atape, dlogits) + self.value.backward(vtape, dv[:, None])
    info = dict(loss=total, pg=pg, ve=ve, ent=en, clip_fraction=clip_frac, kl=klp)
    return info, grads, dlogits, dv

  def train(self, exp, weights=None, preprocessed=False, update_normalizers=True):
    B, T = exp['reward'].shape
    if preprocessed:
      vp, ret, adv = (np.asarray(exp[k], f32) for k in ('value_prediction', 'return', 'advantage'))
    else:
      vp, ret, adv = self.preprocess(exp)
    mask = ppo.make_trajectory_mask(exp['step_type'], ret, adv)
    w = mask if weights is None else (np.asarray(weights, f32) * mask).astype(f32)
    action = np.asarray(exp['action']).reshape(B * T).astype(np.int64)
    A = exp['logits'].shape[-1]
    old_logits = np.asarray(exp['logits'], f32).reshape(B * T, A)
    old_logp = categorical_log_prob(old_logits, action)
    adv_n = ppo.normalize_advantages(adv)
    raw_obs = self._flat_obs(exp)
    obs = self.norm_obs(raw_obs)
    infos = []
    for _ in range(self.num_epochs):
      info, grads, _, _ = self.loss_and_grads(obs, action, old_logp, ret.reshape(-1),
                                              adv_n.reshape(-1), vp.reshape(-1), w.reshape(-1),
                                              B, T, old_logits=old_logits)
      if self.gradient_clipping:
        grads, _ = optim.clip_by_global_norm(grads, self.gradient_clipping)
      self.opt.apply(self.params(), grads)
      self.train_step_counter += 1
      infos.append(info)
    if self.initial_beta > 0:
      kl = (categorical_kl(old_logits, self.dist(obs)) * w.reshape(-1)).astype(f32)
      self.beta = ppo.update_adaptive_kl_beta(self.beta, kl, self.kl_target, self.kl_tol)
    if update_normalizers:
      if self.obs_normalizer is not None:
        self.obs_normalizer.update(raw_obs)
      if self.reward_normalizer is not None:
        self.reward_normalizer.update(exp['reward'])
    return infos
