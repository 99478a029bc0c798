"""Deep Deterministic Policy Gradient (DDPG) agent on libb200rl.

Drop-in for `tf_agents.agents.ddpg.ddpg_agent.DdpgAgent` (Lillicrap et al. 2016) for the
configuration of the reference's examples/v2/train_eval.py: a deterministic ActorNetwork, one
critic on (observation, action), target networks for both, and an OUNoisePolicy collect policy.
`train(experience[B, 2, ...])` follows the reference order:
  critic step -> actor step against the UPDATED critic -> train_step_counter += 1 ->
  Periodically(target_update_period) soft update of the target critic and the target actor with
  target_update_tau.
The actor is updated on every step.

Critic: a' = target_actor(s') (scale_to_spec of the tanh output, no noise, no clip);
y = reward_scale r + gamma d Q'(s', a'); critic loss mean_b(w_b l(y, Q(s, a))), divided by the
batch size; l is `common.element_wise_huber_loss` (the default, delta 1) or
`common.element_wise_squared_loss`, anything else raises ValueError.
Actor: a = actor(s), dqda[b, k] = dQ(s_b, a_b)/da_b[k] (the gradient of sum(Q), per sample),
c = clip(dqda, +-dqda_clipping) (c = dqda when dqda_clipping is None), and the loss is
element_wise_squared_loss(stop_gradient(a + c), a) averaged over the batch and the action:
sum_b w_b sum_k c_bk^2 / (B A), with gradient -2 w_b c_bk / (B A) w.r.t. a and none through c.
  * dqda_clipping=0 clips dQ/da to [0, 0], as the reference code does (its docstring says "no
    clipping"), so the actor gradient is zero and the actor only moves through Adam's momentum.
  * Departure: the weights multiply each row of the [B, A] actor loss, the documented intent
    ("per-batch-entry importance weights").  The reference multiplies a [B, A] loss by [B]
    weights, which TF broadcasts to [B, B] when A = 1 and rejects for most other shapes.  A
    scalar weight gives the same result both ways.
  * The loss is computed as the exact c^2; the reference's float32 ((a + c) - a)^2 rounds the
    sum first, which differs in the last bits of c when |a| >> |c|.

Device work per step (csrc/ddpg.cu, td3.cu, nn.cu, optim.cu): target-actor forward +
scale_to_spec written in place into the target critic's joint-stack input, target-critic forward,
critic forward, fused TD loss + dQ, critic backward, [per-variable clip], Adam; actor forward +
scale_to_spec into the critic's joint-stack input, critic forward, critic input-gradient backward
of sum(Q) (no parameter gradients), fused actor loss + dL/d(tanh output), actor backward, [clip],
Adam; counter += 1; one Polyak launch over the joint [critic | actor] buffer.

Recurrent DDPG: with an ActorRnnNetwork and a CriticRnnNetwork the agent trains on whole [B, T]
sequences, T >= 2 (train_sequence_length None; data_converter.AsTransition(squeeze_time_dim=False)).
Transition t < T-1 is (observation[:, t], step_type[:, t], action[:, t], reward[:, t],
discount[:, t], observation[:, t+1] with next_step_type[:, t]).  Every network runs from the zero
state with a reset at FIRST: the online actor and critic over observation[:, :-1] with
step_type[:, :-1], the target actor and critic over observation[:, 1:] with next_step_type[:, :-1].
So the target recurrence starts one step later than the online one, as in the reference.
  * Critic loss: the element loss of y - Q over the [B, T-1] transitions, summed over time, times
    the weights, mean over B (the divisor is B).  There is no LAST / boundary mask: the reference
    has a TODO there instead, and this matches it.
  * Actor loss: dqda[b, t] = d(sum of all Q)/da[b, t], through the critic's LSTM (a_t also moves
    every later Q), so it comes from a BPTT through the critic; the loss sum_b w_b sum_{t,k} c^2 /
    (B A) as above.
Device work per recurrent step (csrc/ddpg.cu, lstm.cu, td3.cu, nn.cu, optim.cu): target-actor
sequence forward + scale_to_spec, target-critic sequence forward, critic sequence forward,
b200rl_ddpg_seq_critic_loss (TD targets, element loss, time sum, weights, mean and dq in one
launch; reward and discount read in place from the [B, T] experience), critic BPTT backward,
[clip], Adam; actor sequence forward + scale_to_spec, critic sequence forward, critic input-gradient
BPTT of sum(Q) (no parameter-gradient GEMMs), b200rl_ddpg_seq_actor_loss, actor BPTT backward,
[clip], Adam; counter += 1; one Polyak launch.  Data-parallel recurrent training raises.
"""
import collections

import torch

from agents_b200 import _lib
from agents_b200.agents import tf_agent
from agents_b200.agents.td3 import td3_agent
from agents_b200.networks import actor_rnn_network
from agents_b200.networks import critic_rnn_network
from agents_b200.networks import network as network_lib
from agents_b200.policies import actor_policy
from agents_b200.policies import ou_noise_policy
from agents_b200.trajectories import trajectory
from agents_b200.utils import common
from agents_b200.utils import nest

DdpgInfo = collections.namedtuple('DdpgInfo', ('actor_loss', 'critic_loss'))
_SeqBatch = collections.namedtuple(
    '_SeqBatch', ('obs', 'step_type', 'obs2', 'step_type2', 'action', 'reward', 'discount',
                  'weights', 'w_stride', 'B', 'T'))


def _check_recurrent(actor_network, critic_network):
  """True for the recurrent pair (ActorRnnNetwork, CriticRnnNetwork), False for two feed-forward
  networks; any other stateful combination raises NotImplementedError."""
  stateful = [bool(getattr(n, 'state_spec', ())) for n in (actor_network, critic_network)]
  if not any(stateful):
    return False
  if not all(stateful):
    raise NotImplementedError(
        'DdpgAgent needs both networks recurrent or both feed-forward: got a {} actor and a {} '
        'critic.'.format(*('recurrent' if f else 'feed-forward' for f in stateful)))
  if not (isinstance(actor_network, actor_rnn_network.ActorRnnNetwork) and
          isinstance(critic_network, critic_rnn_network.CriticRnnNetwork)):
    raise NotImplementedError(
        'DdpgAgent trains stateful networks only as an ActorRnnNetwork actor with a '
        'CriticRnnNetwork critic; got {} and {}.'.format(type(actor_network).__name__,
                                                          type(critic_network).__name__))
  return True


class DdpgAgent(tf_agent.TFAgent):
  """A DDPG agent."""

  def __init__(self, time_step_spec, action_spec, actor_network, critic_network,
               actor_optimizer=None, critic_optimizer=None, ou_stddev=1.0, ou_damping=1.0,
               target_actor_network=None, target_critic_network=None, target_update_tau=1.0,
               target_update_period=1, dqda_clipping=None, td_errors_loss_fn=None, gamma=1.0,
               reward_scale_factor=1.0, gradient_clipping=None, debug_summaries=False,
               summarize_grads_and_vars=False, train_step_counter=None, name=None, seed=0):
    if len(nest.flatten(action_spec)) != 1:
      raise NotImplementedError('Only a single continuous action tensor is supported.')
    self._recurrent = _check_recurrent(actor_network, critic_network)
    self._loss_kind = td3_agent._loss_kind(td_errors_loss_fn)
    self._actor_network = actor_network
    actor_network.create_variables(time_step_spec.observation)
    self._target_actor_network = target_actor_network or actor_network.copy(
        name='TargetActorNetwork')
    self._target_actor_network.create_variables(time_step_spec.observation)
    self._critic_network = critic_network
    critic_network.create_variables()
    self._target_critic_network = target_critic_network or critic_network.copy(
        name='TargetCriticNetwork')
    self._target_critic_network.create_variables()
    device = actor_network.device
    online = [critic_network, actor_network]
    # [critic | actor]: each optimiser steps its own slice, one Polyak launch covers both (the
    # Periodically counter advances on every b200rl_soft_update call)
    self._online_params, online_grads = network_lib.allocate_jointly(online)
    self._target_params, _ = network_lib.allocate_jointly(
        [self._target_critic_network, self._target_actor_network])
    nc = critic_network.flat_params.numel()
    self._critic_params, self._critic_grads = self._online_params[:nc], online_grads[:nc]
    self._actor_optimizer, self._critic_optimizer = actor_optimizer, critic_optimizer
    self._ou_stddev, self._ou_damping = ou_stddev, ou_damping
    self._target_update_tau, self._target_update_period = target_update_tau, target_update_period
    if dqda_clipping is not None and float(dqda_clipping) < 0:
      raise ValueError('dqda_clipping must be >= 0 or None.')
    self._dqda_clipping = dqda_clipping
    self._gamma, self._reward_scale_factor = gamma, reward_scale_factor
    self._gradient_clipping = gradient_clipping
    self._critic_segments = self._actor_segments = None
    if gradient_clipping is not None:
      self._critic_segments = td3_agent._segments(online[:1], device)
      self._actor_segments = td3_agent._segments(online[1:], device)
    self._update_target = common.Periodically(
        lambda period, ctr: common.soft_variables_update(self._online_params, self._target_params,
                                                         target_update_tau, period=period,
                                                         counter=ctr),
        target_update_period, 'update_targets', device=device)
    policy = actor_policy.ActorPolicy(time_step_spec, action_spec, actor_network, clip=True)
    collect_policy = ou_noise_policy.OUNoisePolicy(
        actor_policy.ActorPolicy(time_step_spec, action_spec, actor_network, clip=False),
        ou_stddev=ou_stddev, ou_damping=ou_damping, clip=True, seed=seed)
    super(DdpgAgent, self).__init__(
        time_step_spec, action_spec, policy=policy, collect_policy=collect_policy,
        train_sequence_length=None if self._recurrent else 2, debug_summaries=debug_summaries,
        summarize_grads_and_vars=summarize_grads_and_vars, train_step_counter=train_step_counter,
        device=device)
    self._nan_flag = torch.zeros(1, dtype=torch.int32, device=device)
    self._ones = None
    self.replicas = 1
    self._grad_sync = None
    if self._recurrent:   # b200rl_ddpg_seq_*_loss scratch: block partials and a last-block ticket
      self._seq_partials = torch.empty(_lib.DDPG_SEQ_MAX_BLOCKS, dtype=torch.float32,
                                       device=device)
      self._seq_ticket = torch.zeros(1, dtype=torch.int32, device=device)

  # TD3's experience unpacking, buffer allocation and per-variable gradient clipping
  _batch = td3_agent.Td3Agent._batch
  _new = td3_agent.Td3Agent._new
  _clip = td3_agent.Td3Agent._clip

  def _initialize(self):
    """Hard-copies the critic and the actor into their targets (ddpg_agent.py _initialize)."""
    common.soft_variables_update(self._online_params, self._target_params, tau=1.0)

  def _train(self, experience, weights=None):
    if self.replicas != 1 or self._grad_sync is not None:
      raise NotImplementedError('DdpgAgent does not support data-parallel training.')
    if self._actor_optimizer is None or self._critic_optimizer is None:
      raise ValueError('Optimizer is undefined.')
    if self._recurrent:
      b = self._seq_batch(experience, weights)
      closs = self._seq_critic_step(b)
      aloss = self._seq_actor_step(b)
    else:
      b = self._batch(experience, weights)
      closs = self._critic_step(b)
      aloss = self._actor_step(b)
    self._bump_train_step(1)
    self._update_target()
    total = aloss + closs
    return tf_agent.LossInfo(total.reshape(()), DdpgInfo(aloss.reshape(()), closs.reshape(())))

  def _critic_input(self, critic, actor, obs, keep):
    """(x, obs_tape): the critic's joint-stack input at (obs, actor(obs)), the action written in
    place over the actor's tanh output by scale_to_spec (no noise, no clamp)."""
    if keep:
      y, atape = actor.forward_train(obs)
    else:
      y, atape = actor.tanh_output(obs), None
    x, otape = critic.stack_input(obs, y, keep=keep)
    col = critic.action_column
    a = x[:, col:col + actor.num_actions]
    actor.scale_to_spec(a, out=a)
    return x, otape, atape

  def _critic_step(self, b):
    """critic_loss against Q'(s', target_actor(s')); critic gradients, one optimiser step."""
    c, tc = self._critic_network, self._target_critic_network
    x2, o2, _ = self._critic_input(tc, self._target_actor_network, b.obs2, keep=False)
    tq = tc.forward_stack(x2, o2)[0]
    x, otape = c.stack_input(b.obs, b.action, keep=True)
    q, tape = c.forward_stack(x, otape, keep=True)
    closs, dq = self._new(1), self._new(b.B, 1)
    _lib.call('b200rl_ddpg_critic_loss', _lib.ptr(q), _lib.ptr(tq), _lib.ptr(b.reward),
              _lib.ptr(b.discount), _lib.ptr(b.weights), b.B, float(self._gamma),
              float(self._reward_scale_factor), self._loss_kind, _lib.ptr(closs), _lib.ptr(dq),
              None, _lib.ptr(self._nan_flag), _lib.stream())
    c.backward(tape, dq)
    self._clip(self._critic_grads, self._critic_segments)
    self._critic_optimizer.apply_flat(self._critic_params, self._critic_grads)
    return closs

  def _ones_like_q(self, B):
    if self._ones is None or self._ones.shape[0] != B:
      self._ones = torch.ones(B, 1, dtype=torch.float32, device=self._nan_flag.device)
    return self._ones

  def _actor_step(self, b):
    """actor_loss against the updated critic: dQ/da of sum(Q), clipped, regressed onto."""
    actor, c = self._actor_network, self._critic_network
    A, B = actor.num_actions, b.B
    x, otape, atape = self._critic_input(c, actor, b.obs, keep=True)
    _, tape = c.forward_stack(x, otape, keep=True)
    _, dx = c.backward(tape, self._ones_like_q(B), need_input_grad=True, need_param_grads=False)
    clip = self._dqda_clipping is not None
    aloss, dy = self._new(1), self._new(B, A)
    _lib.call('b200rl_ddpg_actor_loss', _lib.ptr(dx) + 4 * c.action_column, dx.stride(0),
              _lib.ptr(b.weights), B, A, int(clip), float(self._dqda_clipping) if clip else 0.0,
              _lib.ptr(actor.action_min), _lib.ptr(actor.action_max), _lib.ptr(aloss),
              _lib.ptr(dy), _lib.ptr(self._nan_flag), _lib.stream())
    agrads = actor.backward(atape, dy)
    self._clip(agrads, self._actor_segments)
    self._actor_optimizer.apply_flat(actor.flat_params, agrads)
    return aloss

  # ---- recurrent DDPG ----------------------------------------------------------------------
  def _seq_batch(self, experience, weights):
    """The [B, T] experience as the [B, T-1] windows the recurrent updates read."""
    if not isinstance(experience, trajectory.Trajectory):
      raise TypeError('Input type not supported: {}'.format(type(experience)))
    tf_agent.validate_trajectory(experience, self.training_data_spec, None)
    obs_all = nest.flatten(experience.observation)[0]
    B, T = obs_all.shape[0], obs_all.shape[1]
    if T < 2:
      raise ValueError('Trajectory frame count must be at least 2, but saw {}'.format(T))
    reward, discount = experience.reward.float(), experience.discount.float()
    if reward.stride() != discount.stride():
      reward, discount = reward.contiguous(), discount.contiguous()
    w_stride = 0
    if weights is not None:
      weights = torch.as_tensor(weights, dtype=torch.float32, device=reward.device)
      if weights.numel() > 1:
        weights, w_stride = weights.reshape(B).contiguous(), 1
      else:
        weights = weights.reshape(1)
    return _SeqBatch(obs=obs_all[:, :-1].float(), step_type=experience.step_type[:, :-1],
                     obs2=obs_all[:, 1:].float(), step_type2=experience.next_step_type[:, :-1],
                     action=nest.flatten(experience.action)[0][:, :-1].float(), reward=reward,
                     discount=discount, weights=weights, w_stride=w_stride, B=B, T=T)

  def _seq_critic_step(self, b):
    """The [B, T-1] critic loss against the target networks over observation[:, 1:]; critic
    BPTT gradients, one optimiser step."""
    c, tc, ta = self._critic_network, self._target_critic_network, self._target_actor_network
    y2, _ = ta.tanh_output(b.obs2, b.step_type2)
    ta.scale_to_spec(y2, out=y2)
    tq, _ = tc((b.obs2, y2), b.step_type2)
    q, tape = c.forward_train((b.obs, b.action), b.step_type)
    closs, dq = self._new(1), self._new(b.B * (b.T - 1))
    _lib.call('b200rl_ddpg_seq_critic_loss', _lib.ptr(q), _lib.ptr(tq), _lib.dptr(b.reward),
              _lib.dptr(b.discount), b.reward.stride(0), b.reward.stride(1), _lib.ptr(b.weights),
              b.w_stride, b.B, b.T, float(self._gamma), float(self._reward_scale_factor),
              self._loss_kind, _lib.ptr(closs), _lib.ptr(dq), _lib.ptr(self._nan_flag),
              _lib.ptr(self._seq_partials), _lib.ptr(self._seq_ticket), _lib.stream())
    c.backward(tape, dq)
    self._clip(self._critic_grads, self._critic_segments)
    self._critic_optimizer.apply_flat(self._critic_params, self._critic_grads)
    return closs

  def _seq_actor_step(self, b):
    """The [B, T-1] actor loss against the updated critic: dQ/da of sum(Q) through the critic's
    BPTT (input gradients only), clipped, regressed onto."""
    actor, c = self._actor_network, self._critic_network
    A, n = actor.num_actions, b.B * (b.T - 1)
    y, atape = actor.forward_train(b.obs, b.step_type)
    a = actor.scale_to_spec(y)
    _, tape = c.forward_train((b.obs, a), b.step_type)
    dqda = c.action_gradient(tape, self._ones_like_q(n))
    clip = self._dqda_clipping is not None
    aloss, dy = self._new(1), self._new(n, A)
    _lib.call('b200rl_ddpg_seq_actor_loss', _lib.dptr(dqda), dqda.stride(0), _lib.ptr(b.weights),
              b.w_stride, b.B, b.T, A, int(clip), float(self._dqda_clipping) if clip else 0.0,
              _lib.ptr(actor.action_min), _lib.ptr(actor.action_max), _lib.ptr(aloss),
              _lib.ptr(dy), _lib.ptr(self._nan_flag), _lib.ptr(self._seq_partials),
              _lib.ptr(self._seq_ticket), _lib.stream())
    agrads = actor.backward(atape, dy)
    self._clip(agrads, self._actor_segments)
    self._actor_optimizer.apply_flat(actor.flat_params, agrads)
    return aloss

  def check_numerics(self):
    if int(self._nan_flag.item()) != 0:
      raise FloatingPointError('Critic or actor loss is inf or nan.')
