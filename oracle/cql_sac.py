"""numpy restatement of CqlSacAgent losses and train step (TEST INFRASTRUCTURE).

Follows agents/cql/cql_sac_agent.py: _train :241-392 (critic step with TD + cql_alpha * cql_loss,
actor step (BC while train_step < num_bc_steps), alpha step, Lagrange step on log_cql_alpha,
train_step += 1, target update), _cql_loss :534-679, actor_loss :681-750, _get_cql_alpha
:752-765, _critic_loss_with_optional_entropy_term :767-876; distributions/tanh_bijector_stable.py
:58-66 (inverse tanh clipped to +-0.99999997).  Reuses oracle/sac.py for the SAC pieces.
Every draw is supplied by the caller (the reference's streams are unpinned, DESIGN.md §2).
"""
import numpy as np

from oracle import optim
from oracle import sac as osac

f32 = np.float32
TANH_CLIP = f32(0.99999997)      # 0.99999994 in float32


def uniform_log_prob(amin, amax, action_dim):
  """:624-631 on the bounds as stored: reduce_sum(-log(max - min)) * action_shape[0]."""
  lo, hi = np.asarray(amin, f32), np.asarray(amax, f32)
  return f32(np.sum(-np.log(hi - lo), dtype=f32) * f32(action_dim))


def uniform_actions(u, amin, amax):
  """tf.random.uniform(minval, maxval) from draws u in [0, 1): minval + u * (maxval - minval)."""
  lo = np.broadcast_to(np.asarray(amin, f32), u.shape[1:])
  hi = np.broadcast_to(np.asarray(amax, f32), u.shape[1:])
  return (lo + (u * (hi - lo)).astype(f32)).astype(f32)


def cql_loss(q1, q2, q1_pi, q2_pi, logp_pi, q1_unif, q2_unif, uniform_logp, temperature=1.0):
  """:598-675.  q1, q2 [B] at the dataset actions; q*_pi, logp_pi, q*_unif [B, N].

  Returns (cql_loss, grads) with grads[name] = d cql_loss / d that input (hand-written:
  d lse / d Q_j = softmax_j, d / d q_data = -1 / (2B))."""
  tau = f32(temperature)
  B, N = q1_pi.shape
  terms, grads = [], {}
  for name, q, qp, qu in (('1', q1, q1_pi, q1_unif), ('2', q2, q2_pi, q2_unif)):
    z = np.concatenate([qp * tau - logp_pi, qu * tau - f32(uniform_logp)], axis=1).astype(f32)
    m = z.max(axis=1, keepdims=True)
    e = np.exp(z - m).astype(f32)
    s = e.sum(axis=1, keepdims=True, dtype=f32)
    lse = ((m[:, 0] + np.log(s[:, 0])) / tau).astype(f32)
    terms.append((lse - q).astype(f32))
    p = (e / s).astype(f32)
    grads['q' + name] = np.full(B, -1.0 / (2 * B), f32)
    grads['q' + name + '_pi'] = (p[:, :N] / (2 * B)).astype(f32)
    grads['q' + name + '_unif'] = (p[:, N:] / (2 * B)).astype(f32)
  return f32(np.mean(terms[0] + terms[1], dtype=f32) / f32(2)), grads


def squashed_log_prob(head, action, amin, amax):
  """log pi(action) of the tanh-squashed Normal with head [B, 2A] = (loc | log_std), and its
  gradient w.r.t. the head (the action is data).  Returns (logp [B], dlogp_dhead [B, 2A])."""
  A = head.shape[1] // 2
  loc, ls = head[:, :A], head[:, A:]
  half, shift = (amax - amin) / 2, (amax + amin) / 2
  y = ((action - shift) / half).astype(f32)
  y = np.where(np.abs(y) <= 1, np.clip(y, -TANH_CLIP, TANH_CLIP), y).astype(f32)
  u = np.arctanh(y).astype(f32)
  std = np.exp(ls).astype(f32)
  z = ((u - loc) / std).astype(f32)
  logp = np.sum(-0.5 * z * z - ls - 0.5 * osac.LOG2PI - np.log(half)
                - 2.0 * (osac.LOG2 - u - osac.softplus(-2.0 * u)), axis=1).astype(f32)
  return logp, np.concatenate([z / std, z * z - 1], axis=1).astype(f32)


def critic_loss(q1, q2, tq1, tq2, next_logp, reward, discount, log_alpha, include_entropy_term,
                gamma=1.0, reward_scale=1.0, noise_std=0.0, z_reward=None, weights=None):
  """:815-870: SAC's critic loss, the entropy term only if include_entropy_term, and reward noise
  reward + noise_std * z added before reward_scale.  Returns (loss, td_targets)."""
  if not include_entropy_term:
    next_logp = np.zeros_like(next_logp)
  if noise_std > 0:
    reward = (reward + (z_reward * f32(noise_std)).astype(f32)).astype(f32)
  return osac.critic_loss(q1, q2, tq1, tq2, next_logp, reward, discount, log_alpha, gamma,
                          reward_scale, weights)


def bc_actor_loss(logp, logp_data, log_alpha, weights=None, global_batch=None):
  """:712-718: exp(log_alpha) * log pi(a~|s) - log pi(a_data|s)."""
  per = (np.exp(f32(log_alpha)) * logp - logp_data).astype(f32)
  return osac._agg(per, weights, global_batch)


def lagrange_step(log_cql_alpha, cql_loss_value, cql_tau, clipping=None):
  """:336-348 with _get_cql_alpha: returns (cql_alpha, cql_alpha_loss, d loss / d log_cql_alpha);
  clip_by_value passes the gradient inside [lo, hi], bounds included."""
  la = f32(log_cql_alpha)
  lo, hi = clipping if clipping is not None else (-np.inf, np.inf)
  alpha = f32(np.exp(max(min(la, f32(hi)), f32(lo))))
  loss = f32(-alpha * (f32(cql_loss_value) - f32(cql_tau)))
  return alpha, loss, (loss if lo <= la <= hi else f32(0))


class CqlSacOracle(osac.SacOracle):
  """SacOracle plus the CQL critic term, BC actor phase and Lagrange cql_alpha.

  `cql_alpha` may be reassigned between steps (the reference's tf.Variable)."""

  def __init__(self, actor, critic1, critic2, amin, amax, actor_opt, critic_opt, alpha_opt,
               cql_alpha, num_cql_samples, include_critic_entropy_term=False,
               use_lagrange_cql_alpha=False, cql_alpha_learning_rate=1e-4, cql_tau=10.0,
               reward_noise_variance=0.0, num_bc_steps=0, log_cql_alpha_clipping=None,
               softmax_temperature=1.0, bc_debug_mode=False, uniform_logp=None, **sac_kw):
    super().__init__(actor, critic1, critic2, amin, amax, actor_opt, critic_opt, alpha_opt,
                     **sac_kw)
    A = self.amin.shape[0]
    self.cql_alpha = f32(cql_alpha)
    self.lagrange = use_lagrange_cql_alpha
    self.log_cql_alpha = np.array([np.log(f32(cql_alpha))], f32)
    self.cql_alpha_opt = optim.AdamTF(cql_alpha_learning_rate, eps=1e-7)
    self.cql_tau, self.clipping = cql_tau, log_cql_alpha_clipping
    self.N = num_cql_samples
    self.entropy_term = include_critic_entropy_term
    self.noise_std = f32(reward_noise_variance)
    self.num_bc_steps, self.temperature, self.bc_debug = num_bc_steps, softmax_temperature, bc_debug_mode
    self.uniform_logp = (uniform_log_prob(self.amin, self.amax, A) if uniform_logp is None
                         else f32(uniform_logp))

  def _alpha_now(self):
    if self.lagrange:
      return lagrange_step(self.log_cql_alpha[0], 0.0, 0.0, self.clipping)[0]
    return f32(self.cql_alpha)

  def train(self, exp, eps_next, eps_actor, eps_alpha, eps_cql, u_cql, z_reward=None,
            weights=None):
    obs, obs2 = exp['observation'][:, 0], exp['observation'][:, 1]
    act = exp['action'][:, 0]
    r, d = exp['reward'][:, 0], exp['discount'][:, 0]
    B, N = r.shape[0], self.N
    la = float(self.log_alpha[0])
    w = np.ones(B, f32) if weights is None else np.asarray(weights, f32)
    # ---- critic step (:269-299)
    a2, logp2, _ = osac.sample_and_log_prob(self.actor.forward(obs2), eps_next, self.amin, self.amax)
    tq1, tq2 = self._q(self.t1, obs2, a2), self._q(self.t2, obs2, a2)
    head = self.actor.forward(obs)
    a_pi, logp_pi, _ = osac.sample_and_log_prob(np.repeat(head, N, axis=0), eps_cql, self.amin,
                                                self.amax)
    a_unif = uniform_actions(u_cql, self.amin, self.amax)
    obs_t = np.repeat(obs, N, axis=0)
    x = np.concatenate([np.concatenate([obs, act], 1), np.concatenate([obs_t, a_pi], 1),
                        np.concatenate([obs_t, a_unif], 1)], axis=0).astype(f32)
    q1, tape1 = self.c1.forward(x, keep=True)
    q2, tape2 = self.c2.forward(x, keep=True)
    q1, q2 = q1[:, 0], q2[:, 0]
    closs, y = critic_loss(q1[:B], q2[:B], tq1, tq2, logp2, r, d, la, self.entropy_term,
                           self.gamma, self.reward_scale, self.noise_std, z_reward, weights)
    closs = f32(self.cw * closs)
    cql_alpha = self._alpha_now()
    split = lambda q: (q[:B], q[B:B + B * N].reshape(B, N), q[B + B * N:].reshape(B, N))
    (q1d, q1p, q1u), (q2d, q2p, q2u) = split(q1), split(q2)
    cql, g = cql_loss(q1d, q2d, q1p, q2p, logp_pi.reshape(B, N), q1u, q2u, self.uniform_logp,
                      self.temperature)
    td = f32(0) if self.bc_debug else f32(1)
    g1 = np.concatenate([td * (-2 * (y - q1d) * self.cw * w / B) + cql_alpha * g['q1'],
                         cql_alpha * g['q1_pi'].reshape(-1), cql_alpha * g['q1_unif'].reshape(-1)])
    g2 = np.concatenate([td * (-2 * (y - q2d) * self.cw * w / B) + cql_alpha * g['q2'],
                         cql_alpha * g['q2_pi'].reshape(-1), cql_alpha * g['q2_unif'].reshape(-1)])
    grads = (self.c1.backward(tape1, g1.astype(f32)[:, None]) +
             self.c2.backward(tape2, g2.astype(f32)[:, None]))
    self.critic_opt.apply(self.c1.params() + self.c2.params(), grads)
    critic_total = f32(cql * cql_alpha) if self.bc_debug else f32(closs + cql * cql_alpha)
    # ---- actor step with the updated critics (:301-314, actor_loss :681-750)
    head, atape = self.actor.forward(obs, keep=True)
    A = head.shape[1] // 2
    a, logp, u = osac.sample_and_log_prob(head, eps_actor, self.amin, self.amax)
    qa1, t1 = self._q(self.c1, obs, a, keep=True)
    qa2, t2 = self._q(self.c2, obs, a, keep=True)
    k = (self.aw * w / B).astype(f32)
    bc = self.train_step_counter < self.num_bc_steps
    if bc:
      logp_data, dlogp_data = squashed_log_prob(head, act, self.amin, self.amax)
      aloss = f32(self.aw * bc_actor_loss(logp, logp_data, la, weights))
      da = np.zeros_like(a)
    else:
      aloss = f32(self.aw * osac.actor_loss(qa1, qa2, logp, la, weights))
      first = qa1 <= qa2
      dq1 = np.where(first, -k, 0).astype(f32)[:, None]
      dq2 = np.where(first, 0, -k).astype(f32)[:, None]
      da = osac._input_grad(self.c1, t1, dq1)[:, -A:] + osac._input_grad(self.c2, t2, dq2)[:, -A:]
    gl = (np.exp(f32(la)) * k).astype(f32)
    half = (self.amax - self.amin) / 2
    t = np.tanh(u)
    du = da * half * (1 - t * t) + gl[:, None] * 2 * t
    std = np.exp(head[:, A:])
    dhead = np.concatenate([du, du * std * eps_actor - gl[:, None]], axis=1).astype(f32)
    if bc:
      dhead = (dhead - k[:, None] * dlogp_data).astype(f32)
    self.actor_opt.apply(self.actor.params(), self.actor.backward(atape, dhead))
    # ---- alpha step with the updated actor (:316-325)
    _, logp3, _ = osac.sample_and_log_prob(self.actor.forward(obs), eps_alpha, self.amin, self.amax)
    alloss = f32(self.alw * osac.alpha_loss(logp3, la, self.target_entropy, True, weights))
    dla = f32(self.alw * np.sum(np.where(w == 0, 0, (-logp3 - self.target_entropy) * w), dtype=f32) / B)
    self.alpha_opt.apply([self.log_alpha], [np.array([dla], f32)])
    # ---- Lagrange step (:336-348)
    cql_alpha_loss = f32(0)
    if self.lagrange:
      _, cql_alpha_loss, dlca = lagrange_step(self.log_cql_alpha[0], cql, self.cql_tau, self.clipping)
      self.cql_alpha_opt.apply([self.log_cql_alpha], [np.array([dlca], f32)])
    self.train_step_counter += 1
    self._update_target()
    return dict(loss=f32(critic_total + aloss + alloss), critic_loss=closs, actor_loss=aloss,
                alpha_loss=alloss, cql_loss=cql, cql_alpha=cql_alpha, cql_alpha_loss=cql_alpha_loss)
