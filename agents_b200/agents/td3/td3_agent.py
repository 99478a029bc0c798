"""Twin Delayed DDPG (TD3) agent on libb200rl.

Drop-in for `tf_agents.agents.td3.td3_agent.Td3Agent` (Fujimoto et al. 2018) for the
configuration of the reference's examples/td3: a deterministic ActorNetwork, twin critics on
(observation, action), target networks for all three, a delayed actor update.
`train(experience[B, 2, ...])` follows the reference order:
  critic step -> actor loss against the UPDATED critic 1 -> actor gradients applied only when
  train_step_counter % actor_update_period == 0 (the counter before its increment) ->
  train_step_counter += 1 -> Periodically(target_update_period) soft update of both target
  critics and the target actor with target_update_tau.
The actor loss is computed and returned on every step, also when it is not applied.  With
actor_update_period > 1 the actor optimiser must take a device gate (AdamOptimizer.apply_flat's
`gate`).

Target smoothing: a' = target_actor(s') + clip(N(0, target_policy_noise), +-noise_clip), and, as
in the reference, a' is NOT clipped to the action spec.  y = reward_scale r + gamma d min(Q'1, Q'2).
Critic loss mean_b(w_b (l(y, Q1) + l(y, Q2))), divided by the batch size (not by the sum of the
weights); l is `common.element_wise_huber_loss` (the default, delta 1) or
`common.element_wise_squared_loss`.  The reference example passes
`tf.compat.v1.losses.huber_loss`, which with weights=None gives the same value as the
element-wise Huber default.  Actor loss sum_b(w_b * -Q1(s, pi(s))) / B.

Device work per step (csrc/td3.cu, nn.cu, optim.cu): target-actor forward + scale/smoothing
written into the target critics' joint-stack input, 2 target-critic forwards, 2 critic forwards,
fused twin TD loss + dQ, 2 critic backwards, [per-variable clip], Adam; actor forward +
scale_to_spec into critic 1's joint-stack input, critic 1 forward, fused actor loss, critic 1
input-gradient backward, scale_to_spec backward, actor backward, [clip], Adam gated on the device
train-step counter; counter += 1; one Polyak launch over the joint [critic 1 | critic 2 | actor]
buffer.  The actor backward also runs on steps whose update the gate skips, so the step is one
fixed graph.  The joint-stack input is concat(observation, action), shared by joint-only twin
critics, or concat(h_obs, action) per critic with an observation branch (CriticNetwork
`stack_input`).

Extension (keyword-only): `train(..., noise=(target_noise,))` supplies the N(0, 1) draws z [B, A]
of the target smoothing (the added noise is clip(target_policy_noise * z, +-noise_clip)), so
parity tests are independent of the RNG stream ("oracle mode").
"""
import collections

import torch

from agents_b200 import _lib
from agents_b200.agents import tf_agent
from agents_b200.networks import network as network_lib
from agents_b200.policies import actor_policy
from agents_b200.policies import gaussian_policy
from agents_b200.trajectories import trajectory
from agents_b200.utils import common
from agents_b200.utils import nest

Td3Info = collections.namedtuple('Td3Info', ('actor_loss', 'critic_loss'))
_Batch = collections.namedtuple('_Batch', ('obs', 'obs2', 'action', 'reward', 'discount',
                                           'weights', 'B'))
_TD3_SEED_TAG = 0x5444335F534D4F4F


def _loss_kind(fn):
  if fn is None or fn is common.element_wise_huber_loss:
    return _lib.LOSS_HUBER
  if fn is common.element_wise_squared_loss:
    return _lib.LOSS_SQUARED
  raise ValueError('td_errors_loss_fn must be common.element_wise_huber_loss (the default) or '
                   'common.element_wise_squared_loss to run inside the fused CUDA loss.')


def _segments(nets, device):
  """Per-variable offsets over the nets' consecutive flat buffers (for clip_by_norm_segments)."""
  offs, base = [0], 0
  for n in nets:
    offs += [base + o for o in n.param_offsets[1:]]
    base += n.flat_params.numel()
  return torch.tensor(offs, dtype=torch.int64, device=device)


class Td3Agent(tf_agent.TFAgent):
  """A TD3 agent."""

  def __init__(self, time_step_spec, action_spec, actor_network, critic_network, actor_optimizer,
               critic_optimizer, exploration_noise_std=0.1, critic_network_2=None,
               target_actor_network=None, target_critic_network=None,
               target_critic_network_2=None, target_update_tau=1.0, target_update_period=1,
               actor_update_period=1, td_errors_loss_fn=None, gamma=1.0, reward_scale_factor=1.0,
               target_policy_noise=0.2, target_policy_noise_clip=0.5, gradient_clipping=None,
               debug_summaries=False, summarize_grads_and_vars=False, train_step_counter=None,
               name=None, seed=0):
    if len(nest.flatten(action_spec)) != 1:
      raise NotImplementedError('Only a single continuous action tensor is supported.')
    if getattr(actor_network, 'state_spec', ()) or getattr(critic_network, 'state_spec', ()):
      raise NotImplementedError('Td3Agent supports stateless (non-RNN) networks only.')
    if int(actor_update_period) < 1:
      raise ValueError('actor_update_period must be >= 1.')
    self._loss_kind = _loss_kind(td_errors_loss_fn)
    self._actor_network = actor_network
    actor_network.create_variables(time_step_spec.observation)
    self._target_actor_network = target_actor_network or actor_network.copy(
        name='TargetActorNetwork')
    self._target_actor_network.create_variables(time_step_spec.observation)
    self._critic_network_1 = critic_network
    critic_network.create_variables()
    self._critic_network_2 = critic_network_2 or critic_network.copy(name='CriticNetwork2')
    self._critic_network_2.create_variables()
    if critic_network_2 is None:
      # an independent initialisation, like the reference's `critic_network.copy()`
      self._critic_network_2.set_seed((critic_network._seed or 0) + 1)
      self._critic_network_2._built = False
      self._critic_network_2.create_variables()
      target_critic_network_2 = None
    self._target_critic_network_1 = target_critic_network or critic_network.copy(
        name='TargetCriticNetwork1')
    self._target_critic_network_2 = target_critic_network_2 or self._critic_network_2.copy(
        name='TargetCriticNetwork2')
    self._target_critic_network_1.create_variables()
    self._target_critic_network_2.create_variables()
    device = actor_network.device
    online = [self._critic_network_1, self._critic_network_2, actor_network]
    targets = [self._target_critic_network_1, self._target_critic_network_2,
               self._target_actor_network]
    # [critic 1 | critic 2 | actor]: the critic optimiser steps the first two, the actor
    # optimiser the third, and one Polyak launch covers all three.  One launch matters: the
    # Periodically counter advances on every b200rl_soft_update call.
    self._online_params, online_grads = network_lib.allocate_jointly(online)
    self._target_params, _ = network_lib.allocate_jointly(targets)
    nc = self._critic_network_1.flat_params.numel() + self._critic_network_2.flat_params.numel()
    self._critic_params, self._critic_grads = self._online_params[:nc], online_grads[:nc]
    self._actor_optimizer, self._critic_optimizer = actor_optimizer, critic_optimizer
    self._exploration_noise_std = exploration_noise_std
    self._target_update_tau, self._target_update_period = target_update_tau, target_update_period
    self._actor_update_period = int(actor_update_period)
    self._gamma, self._reward_scale_factor = gamma, reward_scale_factor
    self._target_policy_noise = float(target_policy_noise)
    self._target_policy_noise_clip = float(target_policy_noise_clip)
    self._gradient_clipping = gradient_clipping
    self._critic_segments = self._actor_segments = None
    if gradient_clipping is not None:
      self._critic_segments = _segments(online[:2], device)
      self._actor_segments = _segments(online[2:], device)
    self._update_target = common.Periodically(
        lambda period, ctr: common.soft_variables_update(self._online_params, self._target_params,
                                                         target_update_tau, period=period,
                                                         counter=ctr),
        target_update_period, 'update_targets', device=device)
    self._seed = (int(seed) ^ _TD3_SEED_TAG) & 0xFFFFFFFFFFFFFFFF
    self._target_noise_rng = torch.zeros(2, dtype=torch.int64, device=device)
    policy = actor_policy.ActorPolicy(time_step_spec, action_spec, actor_network, clip=True)
    collect_policy = gaussian_policy.GaussianPolicy(
        actor_policy.ActorPolicy(time_step_spec, action_spec, actor_network, clip=False),
        scale=exploration_noise_std, clip=True, seed=seed)
    super(Td3Agent, self).__init__(
        time_step_spec, action_spec, policy=policy, collect_policy=collect_policy,
        train_sequence_length=2, debug_summaries=debug_summaries,
        summarize_grads_and_vars=summarize_grads_and_vars, train_step_counter=train_step_counter,
        device=device)
    self._nan_flag = torch.zeros(1, dtype=torch.int32, device=device)
    self.replicas = 1
    self._grad_sync = None

  def _initialize(self):
    """Hard-copies both critics and the actor into their targets (td3_agent.py _initialize)."""
    common.soft_variables_update(self._online_params, self._target_params, tau=1.0)

  def _train(self, experience, weights=None, noise=None):
    if self.replicas != 1 or self._grad_sync is not None:
      raise NotImplementedError('Td3Agent does not support data-parallel training.')
    b = self._batch(experience, weights)
    target_noise = None if noise is None else noise[0]
    closs = self._critic_step(b, target_noise)
    aloss = self._actor_step(b)
    self._bump_train_step(1)
    self._update_target()
    total = aloss + closs
    return tf_agent.LossInfo(total.reshape(()), Td3Info(aloss.reshape(()), closs.reshape(())))

  def _batch(self, experience, weights):
    """The [B, 2, ...] experience as the step tensors the two updates read."""
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
                  weights=weights, B=B)

  def _new(self, *shape):
    return torch.empty(shape, dtype=torch.float32, device=self._nan_flag.device)

  def _clip(self, grads, segments):
    if segments is not None:     # eager_utils.clip_gradient_norms: tf.clip_by_norm per variable
      _lib.call('b200rl_clip_by_norm_segments', _lib.ptr(grads), _lib.ptr(segments),
                segments.numel() - 1, float(self._gradient_clipping), _lib.stream())

  @staticmethod
  def _stack_inputs(critics, obs, action):
    """[(x, obs_tape)] joint-stack inputs of `critics` at (obs, action): joint-only critics share
    one concat(obs, action) buffer, critics with an observation branch each take
    concat(h_obs, action)."""
    if not any(c.has_observation_branch for c in critics):
      x = critics[0].joint_input(obs, action)
      return [(x, None)] * len(critics)
    return [c.stack_input(obs, action, keep=True) for c in critics]

  def _critic_step(self, b, target_noise):
    """critic_loss with target smoothing; both critics' gradients, one optimiser step."""
    c1, c2 = self._critic_network_1, self._critic_network_2
    targets = [self._target_critic_network_1, self._target_critic_network_2]
    ta = self._target_actor_network
    y2 = ta.tanh_output(b.obs2)
    # a' = target_actor(s') + clipped noise.  Not clamped to the action spec: the reference adds
    # the noise after scale_to_spec and does not clip the sum.  Joint-only target critics read a'
    # from one shared [obs | a'] buffer, written over y' in place; with an observation branch a'
    # is drawn once and each target critic concatenates it to its own h_obs.
    smooth = dict(noise_std=self._target_policy_noise, noise_clip=self._target_policy_noise_clip,
                  noise=target_noise, seed=self._seed, rng=self._target_noise_rng)
    if any(c.has_observation_branch for c in targets):
      ins = self._stack_inputs(targets, b.obs2, ta.scale_to_spec(y2, **smooth))
    else:
      ins = self._stack_inputs(targets, b.obs2, y2)
      a2 = ins[0][0][:, c1.obs_dim:]
      ta.scale_to_spec(a2, out=a2, **smooth)
    tq1 = targets[0].forward_stack(*ins[0])[0]
    tq2 = targets[1].forward_stack(*ins[1])[0]
    (x1, o1), (x2, o2) = self._stack_inputs([c1, c2], b.obs, b.action)
    q1, tape1 = c1.forward_stack(x1, o1, keep=True)
    q2, tape2 = c2.forward_stack(x2, o2, keep=True)
    B = b.B
    closs, dq1, dq2 = self._new(1), self._new(B, 1), self._new(B, 1)
    _lib.call('b200rl_td3_critic_loss', _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(tq1), _lib.ptr(tq2),
              _lib.ptr(b.reward), _lib.ptr(b.discount), _lib.ptr(b.weights), B,
              float(self._gamma), float(self._reward_scale_factor), self._loss_kind,
              _lib.ptr(closs), _lib.ptr(dq1), _lib.ptr(dq2), None, _lib.ptr(self._nan_flag),
              _lib.stream())
    c1.backward(tape1, dq1)
    c2.backward(tape2, dq2)
    self._clip(self._critic_grads, self._critic_segments)
    self._critic_optimizer.apply_flat(self._critic_params, self._critic_grads)
    return closs

  def _actor_step(self, b):
    """actor_loss against the updated critic 1; the update is gated on the device counter."""
    actor, c1 = self._actor_network, self._critic_network_1
    A, B, st = actor.num_actions, b.B, _lib.stream()
    y, atape = actor.forward_train(b.obs)
    xa, otape = c1.stack_input(b.obs, y, keep=True)
    col = c1.action_column
    a = xa[:, col:col + A]
    actor.scale_to_spec(a, out=a)
    qa, tape = c1.forward_stack(xa, otape, keep=True)
    aloss, dqa = self._new(1), self._new(B, 1)
    _lib.call('b200rl_td3_actor_loss', _lib.ptr(qa), _lib.ptr(b.weights), B, _lib.ptr(aloss),
              _lib.ptr(dqa), _lib.ptr(self._nan_flag), st)
    _, dx = c1.backward(tape, dqa, need_input_grad=True, need_param_grads=False)
    dy = self._new(B, A)
    _lib.call('b200rl_td3_actor_bwd', _lib.ptr(dx) + 4 * col, dx.stride(0),
              _lib.ptr(actor.action_min), _lib.ptr(actor.action_max), B, A, _lib.ptr(dy), st)
    agrads = actor.backward(atape, dy)
    self._clip(agrads, self._actor_segments)
    if self._actor_update_period == 1:
      self._actor_optimizer.apply_flat(actor.flat_params, agrads)
    else:
      self._actor_optimizer.apply_flat(actor.flat_params, agrads,
                                       gate=(self.train_step_counter, self._actor_update_period))
    return aloss

  def check_numerics(self):
    if int(self._nan_flag.item()) != 0:
      raise FloatingPointError('Critic or actor loss is inf or nan.')
