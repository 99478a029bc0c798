"""Behavioral cloning (BC) agent on libb200rl.

Drop-in for `tf_agents.agents.behavioral_cloning.behavioral_cloning_agent.BehavioralCloningAgent`:
supervised learning of the actions in the experience from the observations, with the reference's
two default losses, each one fused kernel in csrc/behavioral_cloning.cu:
  * one scalar discrete action: tf.nn.sparse_softmax_cross_entropy_with_logits(labels=action -
    minimum, logits) over the logits of a QNetwork, a Sequential ending in a Dense layer of
    A = maximum - minimum + 1 units, or the Categorical head of an ActorDistributionNetwork;
  * one continuous action: tf.losses.mse(action, prediction), the mean over the action axis, where
    the prediction is the scale_to_spec output of an ActorNetwork, or the reparameterised sample
    loc + scale z of the Normal head of an ActorDistributionNetwork (the reference's
    `bc_output.sample()`, not clipped).
The per-example losses are aggregated as common.aggregate_losses does with multiply_no_nan:
sum_n w_n pe_n / N over the N = B (or B*T) rows, plus the network's L2 regularisation losses.
`weights` may be a scalar, [B] (broadcast over T) or [B, T].

`train(experience, weights)` runs: forward with its tape -> loss kernel -> L2 terms -> backward ->
[per-variable clip_by_norm] -> optimiser step -> train_step += 1.  It does not synchronise with the
host, and its launches capture into one CUDA graph.  `loss()` is the same math without the tape or
the update.

Normal draws: z for element n*A + k comes from Philox with the agent's {call, ticket} counter
(b200rl_normal_sample's stream).  `train()` advances the counter after its draws; `loss()` draws
with the current counter and leaves it alone, so two `loss()` calls on the same experience agree,
as the reference test of loss stability expects.  Extension (keyword-only): `train(...,
noise=z)` / `loss(..., noise=z)` supply z [N, A] instead, and the counter does not move.

Not supported, each raising with a message: a custom `loss_fn` (NotImplementedError: a Python loss
cannot run inside the fused kernel), RNN cloning networks, TanhNormalActorNetwork, other network
types for the action kind, and more than one replica.  Departure: continuous actions of rank > 1
raise NotImplementedError; the reference accepts them.
"""
import collections

import numpy as np
import torch

from agents_b200 import _lib
from agents_b200.agents import tf_agent
from agents_b200.agents.td3 import td3_agent
from agents_b200.networks import actor_distribution_network as adn
from agents_b200.networks import tanh_normal_projection_network
from agents_b200.policies import actor_policy
from agents_b200.policies import q_policy
from agents_b200.trajectories import trajectory
from agents_b200.utils import nest
from agents_b200.utils import workspace

_BC_SEED_TAG = 0x42435F4E4F524D4C

LOGITS, DETERMINISTIC, NORMAL = 'logits', 'deterministic', 'normal'


class BehavioralCloningLossInfo(collections.namedtuple('BehavioralCloningLossInfo', ('loss',))):
  """Stores a per-batch-entry loss value."""


class BehavioralCloningAgent(tf_agent.TFAgent):
  """A behavioral cloning agent."""

  def __init__(self, time_step_spec, action_spec, cloning_network, optimizer, num_outer_dims=1,
               epsilon_greedy=0.1, loss_fn=None, gradient_clipping=None, debug_summaries=False,
               summarize_grads_and_vars=False, train_step_counter=None, name=None, seed=0):
    flat = nest.flatten(action_spec)
    if not flat:
      raise ValueError('The `action_spec` must contain at least one action.')
    single_discrete_scalar = (len(flat) == 1 and len(flat[0].shape) == 0 and
                              not flat[0].dtype.is_floating_point)
    single_continuous = len(flat) == 1 and flat[0].dtype.is_floating_point
    if not loss_fn and not single_discrete_scalar and not single_continuous:
      raise ValueError('A `loss_fn` must be provided unless there is a single, scalar discrete '
                       'action or a single (scalar or non-scalar) continuous action.')
    if loss_fn is not None:
      raise NotImplementedError('BehavioralCloningAgent supports its default losses only: a '
                                'Python `loss_fn` cannot run inside the fused CUDA loss kernel.')
    if num_outer_dims not in (1, 2):
      raise ValueError('num_outer_dims must be 1 or 2.')
    if getattr(cloning_network, 'state_spec', ()):
      raise NotImplementedError('BehavioralCloningAgent supports stateless (non-RNN) cloning '
                                'networks only.')
    if isinstance(cloning_network, tanh_normal_projection_network.TanhNormalActorNetwork):
      raise NotImplementedError('A TanhNormalActorNetwork cannot be cloned: its sample has no '
                                'fused MSE loss here; use an ActorNetwork or an '
                                'ActorDistributionNetwork.')
    spec = flat[0]
    if single_continuous and len(spec.shape) > 1:
      raise NotImplementedError('BehavioralCloningAgent supports continuous actions of rank 0 '
                                f'or 1, got shape {tuple(spec.shape)}.')
    self._cloning_network = cloning_network
    self._optimizer = optimizer
    self._gradient_clipping = gradient_clipping
    self._num_outer_dims = int(num_outer_dims)
    is_adn = isinstance(cloning_network, adn.ActorDistributionNetwork)
    out_spec = cloning_network.create_variables(time_step_spec.observation)
    if single_continuous:
      if getattr(cloning_network, 'deterministic', False):
        self._kind = DETERMINISTIC
      elif is_adn and not cloning_network.discrete:
        self._kind = NORMAL
      else:
        raise NotImplementedError('For a continuous action the cloning network must be an '
                                  'ActorNetwork or an ActorDistributionNetwork with a Normal head.')
      self._num_actions = cloning_network.num_actions
    else:
      self._minimum = int(np.asarray(spec.minimum).reshape(()))
      self._num_actions = int(np.asarray(spec.maximum).reshape(())) - self._minimum + 1
      if is_adn and not cloning_network.discrete:
        raise NotImplementedError('A discrete action needs logits: a QNetwork, a Sequential '
                                  'ending in a Dense layer or a Categorical '
                                  'ActorDistributionNetwork.')
      if getattr(cloning_network, 'deterministic', False) or \
          tuple(out_spec.shape) != (self._num_actions,):
        raise NotImplementedError(
            'For a discrete action the cloning network must emit {} logits; saw output spec '
            '{}.'.format(self._num_actions, tuple(out_spec.shape)))
      self._kind = LOGITS
    device = cloning_network.device
    if self._kind == LOGITS:
      base = q_policy.QPolicy(time_step_spec, action_spec, q_network=cloning_network)
      policy = q_policy.GreedyPolicy(base)
      collect_policy = q_policy.EpsilonGreedyPolicy(base, epsilon=epsilon_greedy, seed=seed)
    else:
      collect_policy = actor_policy.ActorPolicy(time_step_spec, action_spec, cloning_network,
                                                clip=True, seed=seed)
      policy = actor_policy.ActorPolicy(time_step_spec, action_spec, cloning_network, clip=True,
                                        collect=False, seed=seed)
    super(BehavioralCloningAgent, self).__init__(
        time_step_spec, action_spec, policy, collect_policy, train_sequence_length=None,
        num_outer_dims=num_outer_dims, debug_summaries=debug_summaries,
        summarize_grads_and_vars=summarize_grads_and_vars, train_step_counter=train_step_counter,
        device=device)
    self._seed = (int(seed) ^ _BC_SEED_TAG) & 0xFFFFFFFFFFFFFFFF
    self._sample_rng = torch.zeros(2, dtype=torch.int64, device=device)
    self._nan_flag = torch.zeros(1, dtype=torch.int32, device=device)
    self._segments = None
    if gradient_clipping is not None:
      self._segments = td3_agent._segments([cloning_network], device)
    self.replicas = 1
    self._grad_sync = None

  @property
  def cloning_network(self):
    return self._cloning_network

  def _initialize(self):
    pass

  # ---- loss / train -------------------------------------------------------------------------
  def _flatten(self, experience, weights):
    """(observation [N, ...], action, outer shape, weights [numel], w_div) of the experience."""
    if not isinstance(experience, trajectory.Trajectory):
      raise TypeError('Input type not supported: {}'.format(type(experience)))
    tf_agent.validate_trajectory(experience, self.training_data_spec, None,
                                 num_outer_dims=self._num_outer_dims)
    obs = nest.flatten(experience.observation)[0]
    action = nest.flatten(experience.action)[0]
    k = self._num_outer_dims
    outer = tuple(obs.shape[:k])
    n = int(np.prod(outer))
    obs = obs.reshape((n,) + tuple(obs.shape[k:]))
    w_div = 1
    if weights is not None:
      weights = torch.as_tensor(weights, dtype=torch.float32, device=obs.device)
      if weights.numel() == 1:
        w_div = n
      elif tuple(weights.shape) == outer[:1] and k == 2:
        w_div = outer[1]
      elif tuple(weights.shape) != outer:
        raise ValueError('weights must be a scalar, [B] or [B, T] = {}; got shape {}.'.format(
            list(outer), list(weights.shape)))
      weights = weights.reshape(-1).contiguous()
    return obs, action, outer, n, weights, w_div

  def _new(self, *shape):
    return torch.empty(shape, dtype=torch.float32, device=self._nan_flag.device)

  def _forward_loss(self, experience, weights, keep_tape, noise=None, advance=False):
    """(loss [1], per_example [N], gradient w.r.t. the network output, tape, outer shape)."""
    net, A = self._cloning_network, self._num_actions
    obs, action, outer, n, weights, w_div = self._flatten(experience, weights)
    loss, pe = self._new(1), self._new(n)
    ws, nb = workspace.get(obs.device, 4 * 512)
    if self._kind == LOGITS:
      logits, tape = net.forward_train(obs) if keep_tape else (net(obs)[0], None)
      act = action.reshape(n)
      if act.dtype != torch.int32:
        act = act.to(torch.int32)
      act = act.contiguous()
      grad = self._new(n, A)
      _lib.call('b200rl_bc_discrete_loss', _lib.ptr(logits), logits.stride(0), _lib.ptr(act), 1,
                self._minimum, _lib.ptr(weights), w_div, n, A, _lib.ptr(loss), _lib.ptr(pe),
                _lib.ptr(grad), A, _lib.ptr(self._nan_flag), _lib.ptr(ws), nb, _lib.stream())
    else:
      target = action.reshape(n, A).float().contiguous()
      if self._kind == DETERMINISTIC:
        pred, tape = net.forward_train(obs) if keep_tape else (net.tanh_output(obs), None)
        scale = dscale = None
      else:
        if keep_tape:
          (pred, scale), tape = net.forward_train(obs)
        else:
          (pred, scale), tape = net.distribution_params(obs), None
        dscale = self._new(n, A)
      if noise is not None:
        noise = torch.as_tensor(noise, dtype=torch.float32, device=obs.device).reshape(n, A)
        noise = noise.contiguous()
      dpred = self._new(n, A)
      _lib.call('b200rl_bc_continuous_loss', _lib.ptr(pred), _lib.ptr(scale), A, _lib.ptr(target),
                A, _lib.ptr(net.action_min) if scale is None else None,
                _lib.ptr(net.action_max) if scale is None else None, _lib.ptr(noise), self._seed,
                _lib.ptr(self._sample_rng), int(advance and scale is not None and noise is None),
                _lib.ptr(weights), w_div, n, A, _lib.ptr(loss), _lib.ptr(pe), _lib.ptr(dpred),
                _lib.ptr(dscale), A, _lib.ptr(self._nan_flag), _lib.ptr(ws), nb, _lib.stream())
      grad = dpred if scale is None else (dpred, dscale)
    # regularisation losses (common.aggregate_losses, scale_regularization_loss)
    for coef, w in net.losses:
      _lib.call('b200rl_l2_sum', _lib.ptr(w), w.numel(), float(coef), _lib.ptr(loss),
                _lib.stream())
    return loss, pe, grad, tape, outer

  def _check_replicas(self):
    if self.replicas != 1 or self._grad_sync is not None:
      raise NotImplementedError('BehavioralCloningAgent does not support data-parallel training.')

  def _loss(self, experience, weights=None, training=False, noise=None):
    self._check_replicas()
    loss, pe, _, _, outer = self._forward_loss(experience, weights, keep_tape=False, noise=noise)
    return tf_agent.LossInfo(loss.reshape(()), BehavioralCloningLossInfo(pe.reshape(outer)))

  def _train(self, experience, weights=None, noise=None):
    self._check_replicas()
    if self._optimizer is None:
      raise ValueError('Optimizer is undefined.')
    net = self._cloning_network
    loss, pe, grad, tape, outer = self._forward_loss(experience, weights, keep_tape=True,
                                                     noise=noise, advance=True)
    grads = net.backward(tape, grad)
    for coef, w in net.losses:   # d/dw coef*sum(w^2) = 2*coef*w
      off = w.data_ptr() - net.flat_params.data_ptr()
      g = grads[off // 4: off // 4 + w.numel()]
      _lib.call('b200rl_add_scaled', _lib.ptr(g), _lib.ptr(w), w.numel(), 2.0 * float(coef),
                _lib.stream())
    if self._segments is not None:   # eager_utils.clip_gradient_norms: tf.clip_by_norm per variable
      _lib.call('b200rl_clip_by_norm_segments', _lib.ptr(grads), _lib.ptr(self._segments),
                self._segments.numel() - 1, float(self._gradient_clipping), _lib.stream())
    self._optimizer.apply_flat(net.flat_params, grads)
    self._bump_train_step(1)
    return tf_agent.LossInfo(loss.reshape(()), BehavioralCloningLossInfo(pe.reshape(outer)))

  def check_numerics(self):
    """Raises if any loss so far was inf/nan or a label was outside the action spec; syncs."""
    if int(self._nan_flag.item()) != 0:
      raise FloatingPointError('Behavioral cloning loss is inf or nan, or an action label is '
                               'outside the action spec.')
