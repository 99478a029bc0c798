"""Soft Actor-Critic agent on libb200rl.

Drop-in for `tf_agents.agents.sac.sac_agent.SacAgent` (reference agents/sac/sac_agent.py:61-739)
for the configuration of examples/sac/haarnoja18/sac_train_eval.py: twin critics on
concat(observation, action), tanh-Normal actor, learned temperature, three optimisers,
Polyak target critics.  `train(experience[B, 2, ...])` follows the reference order exactly
(:314-410): critic step -> actor step against the UPDATED critics -> alpha step against the
UPDATED actor -> train_step += 1 -> target update; each of the three policy samples is an
independent reparameterised draw.

Device work per step (csrc/sac.cu, nn.cu, optim.cu): actor forward at s' + fused tanh-Normal
sample/log-prob, 2 target-critic forwards, 2 critic forwards, fused twin-Q TD target + loss +
dQ, 2 critic backwards, Adam; actor forward at s + sample, 2 critic forwards, fused actor loss,
2 critic input-gradient backwards, fused sample backward, actor backward, Adam; actor forward +
sample, fused alpha loss, Adam; fused Polyak over both critics.

Extension (keyword-only): `train(..., noise=(eps_next, eps_actor, eps_alpha))` supplies the
three N(0,1) draws ("oracle mode") so parity tests are independent of the RNG stream.
"""
import collections

import torch

from agents_b200 import _lib
from agents_b200.agents import tf_agent
from agents_b200.networks import network as network_lib
from agents_b200.policies import tf_policy
from agents_b200.trajectories import policy_step
from agents_b200.trajectories import trajectory
from agents_b200.utils import common
from agents_b200.utils import nest

SacLossInfo = collections.namedtuple('SacLossInfo', ('critic_loss', 'actor_loss', 'alpha_loss'))
_Batch = collections.namedtuple('_Batch', ('obs', 'obs2', 'action', 'reward', 'discount', 'weights',
                                           'B', 'gb'))
_SAC_SEED_TAG = 0x5341435F53414D50


class SacPolicy(tf_policy.TFPolicy):
  """ActorPolicy over the tanh-Normal actor: sampled (collect) or mode (greedy) actions."""

  def __init__(self, time_step_spec, action_spec, actor_network, training=False, seed=0,
               greedy=False):
    super().__init__(time_step_spec, action_spec)
    self._actor = actor_network
    self._greedy = greedy
    self._seed = (int(seed) ^ _SAC_SEED_TAG) & 0xFFFFFFFFFFFFFFFF
    self._rng = None

  def variables(self):
    return self._actor.variables

  def sample(self, observation, noise=None, keep=False):
    """Returns (action [N, A], logp [N], ctx) with ctx = (head, tape, u, eps) when keep."""
    a_dim = self._actor.num_actions
    if keep:
      head, tape = self._actor.forward_train(observation)
    else:
      (head, _), tape = self._actor(observation), None
    n = head.shape[0]
    dev = head.device
    if self._rng is None or self._rng.device != dev:
      self._rng = torch.zeros(2, dtype=torch.int64, device=dev)
    action = torch.empty((n, a_dim), dtype=torch.float32, device=dev)
    logp = torch.empty(n, dtype=torch.float32, device=dev)
    u = torch.empty((n, a_dim), dtype=torch.float32, device=dev) if keep else None
    eps = torch.empty((n, a_dim), dtype=torch.float32, device=dev) if keep else None
    if noise is not None:
      noise = torch.as_tensor(noise, dtype=torch.float32, device=dev).contiguous()
    _lib.call('b200rl_sac_sample', _lib.ptr(head), n, a_dim, _lib.ptr(self._actor.action_min),
              _lib.ptr(self._actor.action_max), _lib.ptr(noise), self._seed, _lib.ptr(self._rng),
              _lib.ptr(action), a_dim, _lib.ptr(logp), _lib.ptr(u), _lib.ptr(eps), _lib.stream())
    return action, logp, (head, tape, u, eps)

  def _action(self, time_step, policy_state, seed):
    noise = None
    if self._greedy:  # mode of the squashed Normal: tanh(loc)
      n = time_step.step_type.shape[0]
      noise = torch.zeros((n, self._actor.num_actions), dtype=torch.float32,
                          device=time_step.step_type.device)
    action, _, _ = self.sample(time_step.observation, noise=noise)
    return policy_step.PolicyStep(action, policy_state, ())


class SacAgent(tf_agent.TFAgent):
  """A SAC agent (Haarnoja et al. 2018)."""

  def __init__(self, time_step_spec, action_spec, critic_network, actor_network, actor_optimizer,
               critic_optimizer, alpha_optimizer, actor_loss_weight=1.0, critic_loss_weight=0.5,
               alpha_loss_weight=1.0, actor_policy_ctor=None, critic_network_2=None,
               target_critic_network=None, target_critic_network_2=None, target_update_tau=1.0,
               target_update_period=1, td_errors_loss_fn=None, gamma=1.0, reward_scale_factor=1.0,
               initial_log_alpha=0.0, use_log_alpha_in_alpha_loss=True, target_entropy=None,
               gradient_clipping=None, debug_summaries=False, summarize_grads_and_vars=False,
               train_step_counter=None, name=None, seed=0):
    for net in (critic_network, actor_network, critic_network_2, target_critic_network,
                target_critic_network_2):
      if net is not None and getattr(net, 'state_spec', ()):
        raise NotImplementedError('SacAgent supports feed-forward networks only: a recurrent '
                                  'network needs sequence training.')
    flat_action_spec = nest.flatten(action_spec)
    if len(flat_action_spec) != 1:
      raise NotImplementedError('Only a single continuous action tensor is supported.')
    if td_errors_loss_fn is not None and td_errors_loss_fn is not common.element_wise_squared_loss:
      raise ValueError('td_errors_loss_fn must be the squared difference (the reference default, '
                       'sac_agent.py:101) to run inside the fused CUDA epilogue.')
    if gradient_clipping is not None:
      raise NotImplementedError('gradient_clipping is not supported by this SacAgent.')
    self._critic_network_1 = critic_network
    critic_network.create_variables()
    self._critic_network_2 = critic_network_2 or critic_network.copy(name='CriticNetwork2')
    self._critic_network_2.create_variables()
    if critic_network_2 is None:
      # an independent initialisation, like the reference's `critic_network.copy()` + re-init
      self._critic_network_2.set_seed((critic_network._seed or 0) + 1)
      self._critic_network_2._built = False
      self._critic_network_2.create_variables()
    self._target_critic_network_1 = target_critic_network or critic_network.copy(
        name='TargetCriticNetwork1')
    self._target_critic_network_2 = target_critic_network_2 or self._critic_network_2.copy(
        name='TargetCriticNetwork2')
    self._target_critic_network_1.create_variables()
    self._target_critic_network_2.create_variables()
    self._actor_network = actor_network
    actor_network.create_variables(time_step_spec.observation)
    device = actor_network.device
    self._critic_params, self._critic_grads = network_lib.allocate_jointly(
        [self._critic_network_1, self._critic_network_2])
    self._target_params, _ = network_lib.allocate_jointly(
        [self._target_critic_network_1, self._target_critic_network_2])
    self._log_alpha = torch.zeros(4, dtype=torch.float32, device=device)
    self._log_alpha[0] = float(initial_log_alpha)
    self._dlog_alpha = torch.zeros(4, dtype=torch.float32, device=device)
    self._use_log_alpha_in_alpha_loss = use_log_alpha_in_alpha_loss
    a_dim = int(flat_action_spec[0].shape[0]) if flat_action_spec[0].shape else 1
    self._target_entropy = (-a_dim / 2.0) if target_entropy is None else float(target_entropy)
    self._actor_optimizer, self._critic_optimizer, self._alpha_optimizer = (
        actor_optimizer, critic_optimizer, alpha_optimizer)
    self._actor_loss_weight, self._critic_loss_weight, self._alpha_loss_weight = (
        actor_loss_weight, critic_loss_weight, alpha_loss_weight)
    self._gamma, self._reward_scale_factor = gamma, reward_scale_factor
    self._target_update_tau, self._target_update_period = target_update_tau, target_update_period
    self._update_target = common.Periodically(
        lambda period, ctr: common.soft_variables_update(self._critic_params, self._target_params,
                                                         target_update_tau, period=period,
                                                         counter=ctr),
        target_update_period, 'update_targets', device=device)
    policy = SacPolicy(time_step_spec, action_spec, actor_network, greedy=True)
    collect_policy = SacPolicy(time_step_spec, action_spec, actor_network, seed=seed)
    self._train_policy = SacPolicy(time_step_spec, action_spec, actor_network, seed=seed + 1)
    super(SacAgent, self).__init__(
        time_step_spec, action_spec, policy=policy, collect_policy=collect_policy,
        train_sequence_length=2, debug_summaries=debug_summaries,
        summarize_grads_and_vars=summarize_grads_and_vars, train_step_counter=train_step_counter,
        device=device)
    self._nan_flag = torch.zeros(1, dtype=torch.int32, device=device)
    self.replicas = 1
    self._grad_sync = None

  @property
  def log_alpha(self):
    return self._log_alpha[0]

  def _initialize(self):
    """Copies the critics into the target critics (sac_agent.py:298-312)."""
    common.soft_variables_update(self._critic_params, self._target_params, tau=1.0)

  def _train(self, experience, weights=None, noise=None):
    b = self._batch(experience, weights)
    n_next = n_actor = n_alpha = None
    if noise is not None:
      n_next, n_actor, n_alpha = noise
    closs = self._critic_step(b, n_next)
    aloss = self._actor_step(b, n_actor)
    alloss = self._alpha_step(b, n_alpha)
    self._bump_train_step(1)
    self._update_target()
    total = closs + aloss + alloss
    return tf_agent.LossInfo(total.reshape(()), SacLossInfo(closs.reshape(()), aloss.reshape(()),
                                                            alloss.reshape(())))

  def _batch(self, experience, weights):
    """The [B, 2, ...] experience as the step tensors the three updates read."""
    if not isinstance(experience, trajectory.Trajectory):
      raise TypeError('Input type not supported: {}'.format(type(experience)))
    tf_agent.validate_trajectory(experience, self.training_data_spec, 2)
    obs_all = nest.flatten(experience.observation)[0]
    obs, obs2 = obs_all[:, 0].float(), obs_all[:, 1].float()
    action = nest.flatten(experience.action)[0][:, 0].float()
    reward = experience.reward[:, 0].float().contiguous()
    discount = experience.discount[:, 0].float().contiguous()
    B = reward.shape[0]
    if weights is not None:
      weights = torch.as_tensor(weights, dtype=torch.float32,
                                device=reward.device).expand(B).contiguous()
    return _Batch(obs=obs, obs2=obs2, action=action, reward=reward, discount=discount,
                  weights=weights, B=B, gb=float(B * self.replicas))

  def _new(self, *shape):
    return torch.empty(shape, dtype=torch.float32, device=self._log_alpha.device)

  def _next_targets(self, b, noise):
    """a' ~ pi(.|s'), log pi(a'|s') and the two target-critic values at (s', a')."""
    a2, logp2, _ = self._train_policy.sample(b.obs2, noise=noise)
    tq1, _ = self._target_critic_network_1((b.obs2, a2))
    tq2, _ = self._target_critic_network_2((b.obs2, a2))
    return tq1, tq2, logp2

  def _apply_critic_grads(self, tape1, dq1, tape2, dq2):
    self._critic_network_1.backward(tape1, dq1)
    self._critic_network_2.backward(tape2, dq2)
    if self._grad_sync is not None:
      self._grad_sync(self._critic_grads)
    self._critic_optimizer.apply_flat(self._critic_params, self._critic_grads)

  def _critic_step(self, b, noise):
    """sac_agent.py:341-362, critic_loss :559-643."""
    c1, c2 = self._critic_network_1, self._critic_network_2
    tq1, tq2, logp2 = self._next_targets(b, noise)
    x = c1.joint_input(b.obs, b.action)
    q1, tape1 = c1.forward_train_joint(x)
    q2, tape2 = c2.forward_train_joint(x)
    B = b.B
    closs, dq1, dq2 = self._new(1), self._new(B, 1), self._new(B, 1)
    _lib.call('b200rl_sac_critic_loss', _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(tq1), _lib.ptr(tq2),
              _lib.ptr(logp2), _lib.ptr(b.reward), _lib.ptr(b.discount), _lib.ptr(b.weights),
              _lib.ptr(self._log_alpha), B, float(self._gamma), float(self._reward_scale_factor),
              float(self._critic_loss_weight), b.gb, _lib.ptr(closs), _lib.ptr(dq1), _lib.ptr(dq2),
              None, _lib.ptr(self._nan_flag), _lib.stream())
    self._apply_critic_grads(tape1, dq1, tape2, dq2)
    return closs

  def _actor_loss_hook(self, b, head, logp, aloss, dqa1, dqa2):
    """Runs after the SAC actor loss, before the critics' input gradients (CqlSacAgent: BC)."""

  def _actor_dhead_hook(self, b, head, dhead):
    """Runs after dL/dhead is written, before the actor backward (CqlSacAgent: BC)."""

  def _actor_step(self, b, noise):
    """Against the updated critics (:364-377, actor_loss :645-694)."""
    c1, c2 = self._critic_network_1, self._critic_network_2
    a_dim, o_dim = c1.act_dim, c1.obs_dim
    B, st = b.B, _lib.stream()
    a, logp, (head, atape, u, eps) = self._train_policy.sample(b.obs, noise=noise, keep=True)
    xa = c1.joint_input(b.obs, a)
    qa1, t1 = c1.forward_train_joint(xa)
    qa2, t2 = c2.forward_train_joint(xa)
    aloss, dlogp, dqa1, dqa2 = self._new(1), self._new(B), self._new(B, 1), self._new(B, 1)
    _lib.call('b200rl_sac_actor_loss', _lib.ptr(qa1), _lib.ptr(qa2), _lib.ptr(logp),
              _lib.ptr(b.weights), _lib.ptr(self._log_alpha), B, float(self._actor_loss_weight),
              b.gb, _lib.ptr(aloss), _lib.ptr(dlogp), _lib.ptr(dqa1), _lib.ptr(dqa2),
              _lib.ptr(self._nan_flag), st)
    self._actor_loss_hook(b, head, logp, aloss, dqa1, dqa2)
    _, dx1 = c1.backward(t1, dqa1, need_input_grad=True, need_param_grads=False)
    _, dx2 = c2.backward(t2, dqa2, need_input_grad=True, need_param_grads=False)
    dhead = self._new(B, 2 * a_dim)
    _lib.call('b200rl_sac_sample_bwd', _lib.ptr(head), _lib.ptr(u), _lib.ptr(eps),
              _lib.ptr(self._actor_network.action_min), _lib.ptr(self._actor_network.action_max),
              dx1.data_ptr() + 4 * o_dim, dx2.data_ptr() + 4 * o_dim, o_dim + a_dim,
              _lib.ptr(dlogp), B, a_dim, _lib.ptr(dhead), st)
    self._actor_dhead_hook(b, head, dhead)
    agrads = self._actor_network.backward(atape, dhead)
    if self._grad_sync is not None:
      self._grad_sync(agrads)
    self._actor_optimizer.apply_flat(self._actor_network.flat_params, agrads)
    return aloss

  def _alpha_step(self, b, noise):
    """Against the updated actor (:379-390, alpha_loss :696-739)."""
    _, logp3, _ = self._train_policy.sample(b.obs, noise=noise)
    alloss = self._new(1)
    _lib.call('b200rl_sac_alpha_loss', _lib.ptr(logp3), _lib.ptr(b.weights),
              _lib.ptr(self._log_alpha), b.B, float(self._target_entropy),
              int(self._use_log_alpha_in_alpha_loss), float(self._alpha_loss_weight), b.gb,
              _lib.ptr(alloss), _lib.ptr(self._dlog_alpha), _lib.ptr(self._nan_flag),
              _lib.stream())
    if self._grad_sync is not None:
      self._grad_sync(self._dlog_alpha)
    self._alpha_optimizer.apply_flat(self._log_alpha, self._dlog_alpha)
    return alloss

  def check_numerics(self):
    if int(self._nan_flag.item()) != 0:
      raise FloatingPointError('Critic/actor/alpha loss is inf or nan.')
