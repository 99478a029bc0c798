"""Conservative Q-learning on the SAC path (offline RL) on libb200rl.

Drop-in for `tf_agents.agents.cql.cql_sac_agent.CqlSacAgent` (reference
agents/cql/cql_sac_agent.py:55-876), a SacAgent whose critic loss adds the CQL(H) term
(Kumar et al. 2020, eq. 4) and whose actor clones the dataset actions for the first
`num_bc_steps` train steps.  `train` follows the reference order (_train :241-392): critic step
(TD + cql_alpha * cql_loss) -> actor step (BC or SAC) -> alpha step -> Lagrange step on
log_cql_alpha -> train_step += 1 -> target update.

Critic step: the B dataset rows and the 2BN candidate rows (N policy samples of the pre-update
actor and N uniform actions per state) are stacked into ONE critic joint input, so each critic
runs one forward and one backward, as in SacAgent.  csrc/cql.cu writes the candidate rows
(b200rl_cql_candidates; the policy actions come from b200rl_sac_sample over the BN tiled heads,
written straight into the joint input), the TD part is SAC's fused critic loss on rows [0, B), and
b200rl_cql_loss completes dQ of every row.  The BC branch reads the device train_step counter, so
a captured graph crosses the BC boundary; with num_bc_steps == 0 its kernels are not enqueued and
the actor step is SacAgent's.

`cql_alpha` may be a float or a 0-d float32 CUDA tensor the user changes between steps (the
reference's tf.Variable); the kernels read it on every call and graph replay.  `random_seed`
seeds the Philox streams, like SacAgent(seed=).

Extension (keyword-only): `train(..., noise=(eps_next, eps_actor, eps_alpha, eps_cql, u_cql,
z_reward))` supplies every draw ("oracle mode"): the three SAC N(0,1) draws [B, A], the CQL policy
draws [B*N, A], the uniform draws in [0, 1) [B*N, A] and the reward noise N(0,1) [B] (None when
reward_noise_variance is 0).
"""
import collections
import math

import numpy as np
import torch

from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.agents import tf_agent
from agents_b200.agents.sac import sac_agent
from agents_b200.utils import nest

CqlSacLossInfo = collections.namedtuple(
    'CqlSacLossInfo',
    ('critic_loss', 'actor_loss', 'alpha_loss', 'cql_loss', 'cql_alpha', 'cql_alpha_loss'))
_CQL_SEED_TAGS = (0x43514C5F504F4C49, 0x43514C5F554E4946, 0x43514C5F52455744)   # pi, uniform, reward
_WS_FLOATS = 256          # b200rl_cql_loss workspace (kCqlRedBlocks partials)


def uniform_log_prob(action_spec):
    """`reduce_sum(-log(max - min)) * action_shape[0]` on the bounds as stored (:624-631): scalar
    bounds give -A log(range), per-dimension bounds -A sum_k log(range_k)."""
    spec = nest.flatten(action_spec)[0]
    lo = np.asarray(spec.minimum, np.float32)
    hi = np.asarray(spec.maximum, np.float32)
    return float(np.sum(-np.log(hi - lo), dtype=np.float32) * np.float32(spec.shape[0]))


def _rows(t):
    """(tensor, row stride) of a [N, K] view whose rows are contiguous."""
    if t.dim() != 2 or t.stride(1) != 1:
      t = t.contiguous()
    return t, t.stride(0)


class CqlSacAgent(sac_agent.SacAgent):
  """A CQL-SAC agent based on the SAC agent."""

  def __init__(self, time_step_spec, action_spec, critic_network, actor_network, actor_optimizer,
               critic_optimizer, alpha_optimizer, cql_alpha, num_cql_samples,
               include_critic_entropy_term, use_lagrange_cql_alpha, cql_alpha_learning_rate=1e-4,
               cql_tau=10.0, random_seed=None, reward_noise_variance=0.0, num_bc_steps=0,
               actor_loss_weight=1.0, critic_loss_weight=0.5, alpha_loss_weight=1.0,
               actor_policy_ctor=None, critic_network_2=None, target_critic_network=None,
               target_critic_network_2=None, target_update_tau=1.0, target_update_period=1,
               td_errors_loss_fn=None, gamma=1.0, reward_scale_factor=1.0, initial_log_alpha=0.0,
               use_log_alpha_in_alpha_loss=True, target_entropy=None, gradient_clipping=None,
               log_cql_alpha_clipping=None, softmax_temperature=1.0, bc_debug_mode=False,
               debug_summaries=False, summarize_grads_and_vars=False, train_step_counter=None,
               name=None):
    for net in (critic_network, actor_network, critic_network_2, target_critic_network,
                target_critic_network_2):
      if net is not None and getattr(net, 'state_spec', ()):
        raise NotImplementedError('CqlSacAgent supports feed-forward networks only: recurrent '
                                  'CQL-SAC is not implemented.')
    if int(num_cql_samples) < 1:
      raise ValueError('num_cql_samples must be >= 1.')
    if float(softmax_temperature) <= 0:
      raise ValueError('softmax_temperature must be > 0.')
    seed = 0 if random_seed is None else int(random_seed)
    super().__init__(
        time_step_spec, action_spec, critic_network=critic_network, actor_network=actor_network,
        actor_optimizer=actor_optimizer, critic_optimizer=critic_optimizer,
        alpha_optimizer=alpha_optimizer, actor_loss_weight=actor_loss_weight,
        critic_loss_weight=critic_loss_weight, alpha_loss_weight=alpha_loss_weight,
        actor_policy_ctor=actor_policy_ctor, critic_network_2=critic_network_2,
        target_critic_network=target_critic_network,
        target_critic_network_2=target_critic_network_2, target_update_tau=target_update_tau,
        target_update_period=target_update_period, td_errors_loss_fn=td_errors_loss_fn,
        gamma=gamma, reward_scale_factor=reward_scale_factor, initial_log_alpha=initial_log_alpha,
        use_log_alpha_in_alpha_loss=use_log_alpha_in_alpha_loss, target_entropy=target_entropy,
        gradient_clipping=gradient_clipping, debug_summaries=debug_summaries,
        summarize_grads_and_vars=summarize_grads_and_vars, train_step_counter=train_step_counter,
        name=name, seed=seed)
    dev = self._log_alpha.device
    self._use_lagrange_cql_alpha = bool(use_lagrange_cql_alpha)
    self._cql_alpha = None
    self._log_cql_alpha = None
    if self._use_lagrange_cql_alpha:
      # a padded 4-float buffer (like _log_alpha) stepped by its own Keras Adam (:207-213)
      self._log_cql_alpha = torch.zeros(4, dtype=torch.float32, device=dev)
      self._log_cql_alpha[0] = math.log(float(cql_alpha))
      self._dlog_cql_alpha = torch.zeros(4, dtype=torch.float32, device=dev)
      self._cql_alpha_optimizer = optimizers.Adam(cql_alpha_learning_rate)
    else:
      self._dlog_cql_alpha = None
      self._cql_alpha = self._device_scalar(cql_alpha, 'cql_alpha')
    self._cql_tau = float(cql_tau)
    lo, hi = log_cql_alpha_clipping if log_cql_alpha_clipping is not None else (-math.inf, math.inf)
    self._log_cql_alpha_clipping = (float(lo), float(hi))
    self._num_cql_samples = int(num_cql_samples)
    self._include_critic_entropy_term = bool(include_critic_entropy_term)
    self._reward_noise_std = None
    if isinstance(reward_noise_variance, torch.Tensor) or float(reward_noise_variance) > 0:
      self._reward_noise_std = self._device_scalar(reward_noise_variance, 'reward_noise_variance')
    self._num_bc_steps = int(num_bc_steps)
    self._softmax_temperature = float(softmax_temperature)
    self._bc_debug_mode = bool(bc_debug_mode)
    self._uniform_logp = uniform_log_prob(action_spec)
    self._cql_seeds = [(seed ^ t) & 0xFFFFFFFFFFFFFFFF for t in _CQL_SEED_TAGS]
    self._cql_rngs = [torch.zeros(2, dtype=torch.int64, device=dev) for _ in _CQL_SEED_TAGS]
    self._cql_ws = torch.zeros(_WS_FLOATS, dtype=torch.float32, device=dev)

  def _device_scalar(self, value, what):
    if isinstance(value, torch.Tensor):
      if value.dim() != 0 or value.dtype != torch.float32 or value.device != self._log_alpha.device:
        raise ValueError(f'{what} as a tensor must be a 0-d float32 tensor on the agent device.')
      return value
    return torch.tensor(float(value), dtype=torch.float32, device=self._log_alpha.device)

  @property
  def cql_alpha(self):
    """The CQL weight the next critic step uses (a device scalar)."""
    if self._use_lagrange_cql_alpha:
      lo, hi = self._log_cql_alpha_clipping
      return torch.exp(torch.clamp(self._log_cql_alpha[0], lo, hi))
    return self._cql_alpha

  def _train(self, experience, weights=None, noise=None):
    if self.replicas > 1:
      raise NotImplementedError('CqlSacAgent trains on one replica: the reference takes the CQL '
                                'term over the local batch and SUM-reduces the Lagrange gradient, '
                                'which the data-parallel path does not reproduce.')
    b = self._batch(experience, weights)
    n_next = n_actor = n_alpha = None
    n_cql = (None, None, None)
    if noise is not None:
      n_next, n_actor, n_alpha, *n_cql = noise
    closs, out = self._cql_critic_step(b, n_next, *n_cql)
    aloss = self._actor_step(b, n_actor)
    alloss = self._alpha_step(b, n_alpha)
    if self._use_lagrange_cql_alpha:                                          # :336-348
      self._cql_alpha_optimizer.apply_flat(self._log_cql_alpha, self._dlog_cql_alpha)
    self._bump_train_step(1)
    self._update_target()
    total = out[2] + aloss + alloss                                            # :381
    return tf_agent.LossInfo(total.reshape(()), CqlSacLossInfo(
        closs.reshape(()), aloss.reshape(()), alloss.reshape(()), out[0], out[1], out[3]))

  def _cql_critic_step(self, b, n_next, eps_cql, u_cql, z_reward):
    """:269-299: the gradient of critic_loss_weight * TD + cql_alpha * cql_loss (only the CQL
    term in bc_debug_mode) over one joint input of B + 2BN rows per critic."""
    c1, c2 = self._critic_network_1, self._critic_network_2
    actor = self._actor_network
    B, N, D, A = b.B, self._num_cql_samples, c1.obs_dim, c1.act_dim
    W, BN = D + A, b.B * self._num_cql_samples
    st = _lib.stream()
    dev = b.reward.device
    f32 = lambda t: None if t is None else torch.as_tensor(t, dtype=torch.float32,
                                                           device=dev).contiguous()
    tq1, tq2, logp2 = self._next_targets(b, n_next)
    if not self._include_critic_entropy_term:                                 # :828-829
      logp2 = torch.zeros(B, dtype=torch.float32, device=dev)
    reward = b.reward
    if self._reward_noise_std is not None:                                    # :832-839
      reward = self._new(B)
      _lib.call('b200rl_cql_reward_noise', _lib.ptr(b.reward), B, _lib.ptr(self._reward_noise_std),
                _lib.ptr(f32(z_reward)), self._cql_seeds[2], _lib.ptr(self._cql_rngs[2]),
                _lib.ptr(reward), st)
    x = self._new(B + 2 * BN, W)
    c1.joint_input(b.obs, b.action, out=x)
    obs, ld_obs = _rows(b.obs)
    head, _ = actor(b.obs)                                   # the pre-update actor at s (:570-576)
    head_t, cand_logp = self._new(BN, 2 * A), self._new(BN)
    _lib.call('b200rl_cql_candidates', _lib.dptr(obs), ld_obs, B, N, D, A,
              _lib.ptr(actor.action_min), _lib.ptr(actor.action_max), _lib.ptr(f32(u_cql)),
              self._cql_seeds[1], _lib.ptr(self._cql_rngs[1]), _lib.ptr(head), _lib.ptr(x),
              _lib.ptr(head_t), st)
    _lib.call('b200rl_sac_sample', _lib.ptr(head_t), BN, A, _lib.ptr(actor.action_min),
              _lib.ptr(actor.action_max), _lib.ptr(f32(eps_cql)), self._cql_seeds[0],
              _lib.ptr(self._cql_rngs[0]), x.data_ptr() + 4 * (B * W + D), W,
              _lib.ptr(cand_logp), None, None, st)
    q1, tape1 = c1.forward_train_joint(x)
    q2, tape2 = c2.forward_train_joint(x)
    closs, dq1, dq2 = self._new(1), self._new(B + 2 * BN, 1), self._new(B + 2 * BN, 1)
    _lib.call('b200rl_sac_critic_loss', _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(tq1), _lib.ptr(tq2),
              _lib.ptr(logp2), _lib.ptr(reward), _lib.ptr(b.discount), _lib.ptr(b.weights),
              _lib.ptr(self._log_alpha), B, float(self._gamma), float(self._reward_scale_factor),
              float(self._critic_loss_weight), b.gb, _lib.ptr(closs), _lib.ptr(dq1), _lib.ptr(dq2),
              None, _lib.ptr(self._nan_flag), st)
    out = self._new(4)
    lo, hi = self._log_cql_alpha_clipping
    _lib.call('b200rl_cql_loss', _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(cand_logp), B, N,
              self._uniform_logp, self._softmax_temperature, _lib.ptr(self._cql_alpha),
              _lib.ptr(self._log_cql_alpha), lo, hi, self._cql_tau, int(self._bc_debug_mode),
              _lib.ptr(closs), _lib.ptr(dq1), _lib.ptr(dq2), _lib.ptr(out),
              _lib.ptr(self._dlog_cql_alpha), _lib.ptr(self._nan_flag), _lib.ptr(self._cql_ws),
              4 * self._cql_ws.numel(), st)
    self._apply_critic_grads(tape1, dq1, tape2, dq2)
    return closs, out

  def _actor_loss_hook(self, b, head, logp, aloss, dqa1, dqa2):
    """BC branch of actor_loss (:712-718) while train_step < num_bc_steps."""
    if self._num_bc_steps <= 0:
      return
    actor = self._actor_network
    action, ld = _rows(b.action)
    _lib.call('b200rl_cql_bc_actor_loss', _lib.ptr(head), _lib.dptr(action), ld,
              _lib.ptr(actor.action_min), _lib.ptr(actor.action_max), _lib.ptr(logp),
              _lib.ptr(b.weights), _lib.ptr(self._log_alpha), _lib.ptr(self.train_step_counter),
              self._num_bc_steps, b.B, actor.num_actions, float(self._actor_loss_weight), b.gb,
              _lib.ptr(aloss), _lib.ptr(dqa1), _lib.ptr(dqa2), _lib.ptr(self._nan_flag),
              _lib.stream())

  def _actor_dhead_hook(self, b, head, dhead):
    if self._num_bc_steps <= 0:
      return
    actor = self._actor_network
    action, ld = _rows(b.action)
    _lib.call('b200rl_cql_bc_actor_bwd', _lib.ptr(head), _lib.dptr(action), ld,
              _lib.ptr(actor.action_min), _lib.ptr(actor.action_max), _lib.ptr(b.weights),
              _lib.ptr(self.train_step_counter), self._num_bc_steps, b.B, actor.num_actions,
              float(self._actor_loss_weight), b.gb, _lib.ptr(dhead), _lib.stream())

  def check_numerics(self):
    if int(self._nan_flag.item()) != 0:
      raise FloatingPointError('Critic/actor/alpha/CQL/CQL-alpha loss is inf or nan.')
