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

Recurrent SAC: with a tanh-Normal ActorDistributionRnnNetwork actor
(continuous_projection_net=TanhNormalProjectionNetwork) and CriticRnnNetwork critics the agent
trains on whole [B, T] sequences, T >= 2 (train_sequence_length None;
data_converter.AsTransition(squeeze_time_dim=False)).  Transition t < T-1 of sequence b is row
b*(T-1) + t.  Every network runs from the zero state with a reset at FIRST: the actor's a' and the
target critics over observation[:, 1:] with next_step_type[:, :-1]; the online critics and the
actor's actor-step and alpha-step samples over observation[:, :-1] with step_type[:, :-1].
  * Each loss sums over time, then applies the weights, then takes the mean over B; there is no
    LAST mask, as in the reference.
  * The actor loss's dQ/da comes through each critic's full BPTT (a_t moves every later Q), with
    input gradients only: the critics' own gradients are not touched.
  * The noise draws of `train(..., noise=...)` are [B, T-1, A].
Device work per recurrent step (csrc/sac.cu, lstm.cu, nn.cu, optim.cu): actor sequence forward +
sample over observation[:, 1:], 2 target-critic sequence forwards, 2 critic sequence forwards,
b200rl_sac_seq_critic_loss (reward and discount read in place from the [B, T] experience), 2
critic BPTT backwards, Adam; actor sequence forward + sample, 2 critic sequence forwards,
b200rl_sac_seq_actor_loss, 2 input-gradient-only critic BPTTs, sample backward, actor BPTT, Adam;
actor sequence forward + sample, b200rl_sac_seq_alpha_loss, Adam; one Polyak launch.
Data-parallel recurrent training raises.
"""
import collections

import torch

from agents_b200 import _lib
from agents_b200.agents import tf_agent
from agents_b200.agents.ddpg import ddpg_agent
from agents_b200.networks import actor_distribution_rnn_network
from agents_b200.networks import critic_rnn_network
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


def _check_recurrent(actor_network, critics):
  """True for a tanh-Normal ActorDistributionRnnNetwork actor with CriticRnnNetwork critics, False
  for feed-forward networks only; any other stateful combination raises NotImplementedError."""
  nets = [actor_network] + [c for c in critics if c is not None]
  if not any(getattr(n, 'state_spec', ()) for n in nets):
    return False
  if not (isinstance(actor_network, actor_distribution_rnn_network.ActorDistributionRnnNetwork)
          and actor_network.tanh_normal and
          all(isinstance(c, critic_rnn_network.CriticRnnNetwork) for c in nets[1:])):
    raise NotImplementedError(
        'SacAgent supports feed-forward networks, or a recurrent ActorDistributionRnnNetwork '
        'actor with continuous_projection_net=TanhNormalProjectionNetwork and CriticRnnNetwork '
        'critics; got {}.'.format(', '.join(type(n).__name__ for n in nets)))
  return True


class SacPolicy(tf_policy.TFPolicy):
  """ActorPolicy over the tanh-Normal actor: sampled (collect) or mode (greedy) actions.

  A recurrent actor (ActorDistributionRnnNetwork with the tanh-Normal head) makes the policy
  stateful: `policy_state_spec` is the actor's `state_spec`, and each call runs one [B, 1] step
  from the given state (the zero state where step_type is FIRST) and returns the new state."""

  def __init__(self, time_step_spec, action_spec, actor_network, training=False, seed=0,
               greedy=False):
    super().__init__(time_step_spec, action_spec,
                     policy_state_spec=getattr(actor_network, 'state_spec', ()))
    self._actor = actor_network
    self._greedy = greedy
    self._seed = (int(seed) ^ _SAC_SEED_TAG) & 0xFFFFFFFFFFFFFFFF
    self._rng = None

  def variables(self):
    return self._actor.variables

  def get_initial_state(self, batch_size=None):
    if not self._policy_state_spec:
      return ()
    return self._actor.get_initial_state(batch_size)

  def sample(self, observation, noise=None, keep=False, step_type=None):
    """Returns (action [N, A], logp [N], ctx) with ctx = (head, tape, u, eps) when keep.  A
    recurrent actor takes observation [B, T, ...] with step_type [B, T] and runs from the zero
    state; N = B*T in batch-major order."""
    if self._policy_state_spec:
      if keep:
        head, tape = self._actor.forward_train(observation, step_type)
      else:
        (head, _), tape = self._actor.distribution_params(observation, step_type), None
    elif keep:
      head, tape = self._actor.forward_train(observation)
    else:
      (head, _), tape = self._actor(observation), None
    action, logp, u, eps = self._draw(head, noise, keep)
    return action, logp, (head, tape, u, eps)

  def _draw(self, head, noise, keep):
    """(action, logp, u, eps) from the [N, 2A] head; u and eps (kept for the backward) are None
    unless keep."""
    a_dim = self._actor.num_actions
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
    return action, logp, u, eps

  def _action(self, time_step, policy_state, seed):
    noise = None
    if self._greedy:  # mode of the squashed Normal: tanh(loc)
      n = time_step.step_type.shape[0]
      noise = torch.zeros((n, self._actor.num_actions), dtype=torch.float32,
                          device=time_step.step_type.device)
    if not self._policy_state_spec:
      action, _, _ = self.sample(time_step.observation, noise=noise)
      return policy_step.PolicyStep(action, policy_state, ())
    if len(nest.flatten(policy_state)) != len(nest.flatten(self._policy_state_spec)):
      raise ValueError('This SacPolicy is stateful (its actor is recurrent): pass the policy_state '
                       'from get_initial_state(batch_size) or from the previous action().')
    head, state = self._actor.distribution_params(time_step.observation, time_step.step_type,
                                                  policy_state)
    action, _, _, _ = self._draw(head, noise, keep=False)
    return policy_step.PolicyStep(action, state, ())


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
    self._recurrent = _check_recurrent(actor_network, (
        critic_network, critic_network_2, target_critic_network, target_critic_network_2))
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
        train_sequence_length=None if self._recurrent else 2, debug_summaries=debug_summaries,
        summarize_grads_and_vars=summarize_grads_and_vars, train_step_counter=train_step_counter,
        device=device)
    self._nan_flag = torch.zeros(1, dtype=torch.int32, device=device)
    self.replicas = 1
    self._grad_sync = None
    if self._recurrent:   # b200rl_sac_seq_*_loss scratch: block partials and a last-block ticket
      self._seq_partials = torch.empty(_lib.SAC_SEQ_MAX_BLOCKS, dtype=torch.float32, device=device)
      self._seq_ticket = torch.zeros(1, dtype=torch.int32, device=device)

  @property
  def log_alpha(self):
    return self._log_alpha[0]

  def _initialize(self):
    """Copies the critics into the target critics (sac_agent.py:298-312)."""
    common.soft_variables_update(self._critic_params, self._target_params, tau=1.0)

  def _train(self, experience, weights=None, noise=None):
    n_next = n_actor = n_alpha = None
    if noise is not None:
      n_next, n_actor, n_alpha = noise
    if self._recurrent:
      if self.replicas != 1 or self._grad_sync is not None:
        raise NotImplementedError('Recurrent SacAgent does not support data-parallel training.')
      b = self._seq_batch(experience, weights)
      closs = self._seq_critic_step(b, n_next)
      aloss = self._seq_actor_step(b, n_actor)
      alloss = self._seq_alpha_step(b, n_alpha)
    else:
      b = self._batch(experience, weights)
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

  # ---- recurrent SAC -----------------------------------------------------------------------
  # DDPG's unpacking of the [B, T] experience into the [B, T-1] windows of the transitions
  _seq_batch = ddpg_agent.DdpgAgent._seq_batch

  def _seq_scratch(self):
    return _lib.ptr(self._nan_flag), _lib.ptr(self._seq_partials), _lib.ptr(self._seq_ticket)

  def _seq_critic_step(self, b, noise):
    """The [B, T-1] critic loss against the target critics over observation[:, 1:]; both critics'
    BPTT gradients, one optimiser step."""
    c1, c2 = self._critic_network_1, self._critic_network_2
    a2, logp2, _ = self._train_policy.sample(b.obs2, noise=noise, step_type=b.step_type2)
    tq1, _ = self._target_critic_network_1((b.obs2, a2), b.step_type2)
    tq2, _ = self._target_critic_network_2((b.obs2, a2), b.step_type2)
    q1, tape1 = c1.forward_train((b.obs, b.action), b.step_type)
    q2, tape2 = c2.forward_train((b.obs, b.action), b.step_type)
    n = b.B * (b.T - 1)
    closs, dq1, dq2 = self._new(1), self._new(n), self._new(n)
    _lib.call('b200rl_sac_seq_critic_loss', _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(tq1),
              _lib.ptr(tq2), _lib.ptr(logp2), _lib.dptr(b.reward), _lib.dptr(b.discount),
              b.reward.stride(0), b.reward.stride(1), _lib.ptr(b.weights), b.w_stride,
              _lib.ptr(self._log_alpha), b.B, b.T, float(self._gamma),
              float(self._reward_scale_factor), float(self._critic_loss_weight), _lib.ptr(closs),
              _lib.ptr(dq1), _lib.ptr(dq2), *self._seq_scratch(), _lib.stream())
    self._apply_critic_grads(tape1, dq1, tape2, dq2)
    return closs

  def _seq_actor_step(self, b, noise):
    """The [B, T-1] actor loss against the updated critics: dQ/da of each critic through its
    BPTT (input gradients only), the sample backward, the actor BPTT, one optimiser step."""
    c1, c2, actor = self._critic_network_1, self._critic_network_2, self._actor_network
    n, st = b.B * (b.T - 1), _lib.stream()
    a, logp, (head, atape, u, eps) = self._train_policy.sample(b.obs, noise=noise, keep=True,
                                                                step_type=b.step_type)
    qa1, t1 = c1.forward_train((b.obs, a), b.step_type)
    qa2, t2 = c2.forward_train((b.obs, a), b.step_type)
    aloss, dlogp, dqa1, dqa2 = self._new(1), self._new(n), self._new(n), self._new(n)
    _lib.call('b200rl_sac_seq_actor_loss', _lib.ptr(qa1), _lib.ptr(qa2), _lib.ptr(logp),
              _lib.ptr(b.weights), b.w_stride, _lib.ptr(self._log_alpha), b.B, b.T,
              float(self._actor_loss_weight), _lib.ptr(aloss), _lib.ptr(dlogp), _lib.ptr(dqa1),
              _lib.ptr(dqa2), *self._seq_scratch(), st)
    da1, da2 = c1.action_gradient(t1, dqa1), c2.action_gradient(t2, dqa2)
    if da1.stride() != da2.stride() or da1.stride(1) != 1:   # sample_bwd takes one row stride
      da1, da2 = da1.contiguous(), da2.contiguous()
    dhead = self._new(n, 2 * actor.num_actions)
    _lib.call('b200rl_sac_sample_bwd', _lib.ptr(head), _lib.ptr(u), _lib.ptr(eps),
              _lib.ptr(actor.action_min), _lib.ptr(actor.action_max), _lib.dptr(da1),
              _lib.dptr(da2), da1.stride(0), _lib.ptr(dlogp), n, actor.num_actions,
              _lib.ptr(dhead), st)
    agrads = actor.backward(atape, dhead)
    self._actor_optimizer.apply_flat(actor.flat_params, agrads)
    return aloss

  def _seq_alpha_step(self, b, noise):
    """The [B, T-1] alpha loss against the updated actor, one optimiser step."""
    _, logp3, _ = self._train_policy.sample(b.obs, noise=noise, step_type=b.step_type)
    alloss = self._new(1)
    _lib.call('b200rl_sac_seq_alpha_loss', _lib.ptr(logp3), _lib.ptr(b.weights), b.w_stride,
              _lib.ptr(self._log_alpha), b.B, b.T, float(self._target_entropy),
              int(self._use_log_alpha_in_alpha_loss), float(self._alpha_loss_weight),
              _lib.ptr(alloss), _lib.ptr(self._dlog_alpha), *self._seq_scratch(), _lib.stream())
    self._alpha_optimizer.apply_flat(self._log_alpha, self._dlog_alpha)
    return alloss

  def check_numerics(self):
    if int(self._nan_flag.item()) != 0:
      raise FloatingPointError('Critic/actor/alpha loss is inf or nan.')
