"""REINFORCE agent on libb200rl.

Drop-in for `tf_agents.agents.reinforce.reinforce_agent.ReinforceAgent`
(agents/reinforce/reinforce_agent.py:120-567): Monte-Carlo policy gradient (Williams 1992) over
whole episodes, with an optional state-value baseline (Sutton & Barto 2018, 13.4), return /
advantage normalisation and an entropy bonus.  The actor is an ActorDistributionNetwork: a Normal
head for continuous actions or a Categorical head for discrete ones.

Device work of `train(experience[B, T])` (csrc/ppo.cu, scans.cu, reinforce.cu, nn.cu, optim.cu):
  gamma*discount*(next_step_type != LAST) -> returns scan -> actor (+ value) forward ->
  b200rl_reinforce_loss (episode masks, num_episodes, normalisation moments, losses, gradients of
  the distribution parameters and of V) -> backward -> L2 terms -> per-variable clipping ->
  one Adam step over actor + value -> train_step += 1.

Kept from the reference: value_preds are not stop-gradient inside the advantages (:284-292,
:355-364), so with a baseline the policy-gradient loss also trains the value network.
Departure: where the advantages have zero spread the reference's value gradient through the
normalisation is 0 * inf = NaN; here that term is 0.

An experience without a complete episode aborts the reference's train step (:328-336).  Eagerly,
`train` reads one flag word after the loss launch and raises ValueError with the reference's
message before the optimiser runs.  Inside a captured graph there is no host read: the loss kernel
zeroes every gradient (so the Adam step only advances its moments) and raises a flag bit that
`check_numerics()` reports.
"""
import collections
import ctypes

import torch

from agents_b200 import _lib
from agents_b200.agents import tf_agent
from agents_b200.networks import network as network_lib
from agents_b200.policies import actor_policy
from agents_b200.trajectories import trajectory
from agents_b200.utils import nest
from agents_b200.utils import workspace

ReinforceAgentLossInfo = collections.namedtuple('ReinforceAgentLossInfo', (
    'policy_gradient_loss', 'policy_network_regularization_loss', 'entropy_regularization_loss',
    'value_estimation_loss', 'value_network_regularization_loss'))

NO_EPISODE_MESSAGE = ('No complete episode found. REINFORCE requires full episodes to compute '
                      'losses.')
_FLAG_NONFINITE, _FLAG_NO_EPISODE = 1, 2
_STEP_MID, _STEP_LAST = 1, 2


class ReinforceAgent(tf_agent.TFAgent):
  """A REINFORCE agent, optionally with a learned state-value baseline."""

  def __init__(self, time_step_spec, action_spec, actor_network, optimizer, value_network=None,
               value_estimation_loss_coef=0.2, advantage_fn=None, use_advantage_loss=True,
               gamma=1.0, normalize_returns=True, gradient_clipping=None, debug_summaries=False,
               summarize_grads_and_vars=False, entropy_regularization=None,
               train_step_counter=None, name=None, seed=0):
    if advantage_fn is not None:
      raise NotImplementedError(
          'ReinforceAgent does not take a custom advantage_fn: the loss kernel differentiates '
          'advantages = returns - value_preds (or returns) itself. Use use_advantage_loss.')
    for label, net in (('actor_network', actor_network), ('value_network', value_network)):
      if net is not None and getattr(net, 'state_spec', ()):
        raise NotImplementedError(f'ReinforceAgent supports stateless networks only; {label} '
                                  'has a state (RNN actors are not supported).')
    if not hasattr(actor_network, 'distribution_params'):
      raise TypeError('actor_network must emit distribution parameters '
                      '(an ActorDistributionNetwork).')
    self._actor_network = actor_network
    self._value_network = value_network
    actor_network.create_variables(time_step_spec.observation)
    nets = [actor_network]
    if value_network is not None:
      value_network.create_variables(time_step_spec.observation)
      nets.append(value_network)
    self._flat_params, self._flat_grads = network_lib.allocate_jointly(nets)
    # per-variable offsets in the joint buffer (eager_utils.clip_gradient_norms clips each one)
    offs, base = [0], 0
    for net in nets:
      offs.extend(base + o for o in net.param_offsets[1:])
      base += net.flat_params.numel()
    self._clip_offsets_host = offs
    self._clip_offsets = None
    device = actor_network.device
    self._optimizer = optimizer
    self._gamma = float(gamma)
    self._normalize_returns = bool(normalize_returns)
    self._gradient_clipping = gradient_clipping
    self._entropy_regularization = entropy_regularization
    self._value_estimation_loss_coef = float(value_estimation_loss_coef)
    self._baseline = value_network is not None
    self._use_advantage = bool(use_advantage_loss) and self._baseline
    collect_policy = actor_policy.ActorPolicy(time_step_spec, action_spec, actor_network,
                                              clip=True, collect=True, seed=seed)
    policy = actor_policy.ActorPolicy(time_step_spec, action_spec, actor_network, clip=True,
                                      collect=False, seed=seed)
    super(ReinforceAgent, self).__init__(
        time_step_spec, action_spec, policy, collect_policy, train_sequence_length=None,
        debug_summaries=debug_summaries, summarize_grads_and_vars=summarize_grads_and_vars,
        train_step_counter=train_step_counter, device=device)
    self._flag = torch.zeros(1, dtype=torch.int32, device=device)
    self._num_episodes = torch.zeros(1, dtype=torch.float32, device=device)
    self.replicas = 1
    self._grad_sync = None

  @property
  def actor_network(self):
    return self._actor_network

  @property
  def value_network(self):
    return self._value_network

  def _initialize(self):
    pass

  # ---- the loss kernel ---------------------------------------------------------------------------
  def _entropy_coef(self):
    return float(self._entropy_regularization) if self._entropy_regularization else 0.0

  def _launch(self, params, action, returns, value, step_type, next_step_type, weights, B, T,
              use_advantage, normalize, entropy_coef, value_coef):
    """b200rl_reinforce_loss over [B, T] rows; params are (loc, scale) [N, A] or logits [N, A].
    Returns (losses[6], dparams, dvalue)."""
    dev = returns.device
    N = B * T
    if isinstance(params, tuple):
      p0, p1 = params
      A = p0.shape[1]
      d0, d1 = torch.empty_like(p0), torch.empty_like(p1)
      dparams = (d0, d1)
    else:
      p0, p1 = params, None
      A = p0.shape[1]
      d0, d1 = torch.empty_like(p0), None
      dparams = d0
    losses = torch.empty(6, dtype=torch.float32, device=dev)
    dv = torch.empty(N, dtype=torch.float32, device=dev) if value is not None else None
    ws, nb = workspace.get(dev, 4 * (4096 + (B + 3) // 4 * 4 + N))
    _lib.call('b200rl_reinforce_loss', _lib.ptr(p0), _lib.ptr(p1), A, _lib.ptr(action), A,
              _lib.ptr(returns), _lib.ptr(value), _lib.ptr(step_type), _lib.ptr(next_step_type),
              _lib.ptr(weights), B, T, int(use_advantage), int(normalize), float(entropy_coef),
              float(value_coef), _lib.ptr(losses), _lib.ptr(d0), _lib.ptr(d1), A, _lib.ptr(dv),
              _lib.ptr(self._num_episodes), _lib.ptr(self._flag), _lib.ptr(ws), nb, _lib.stream())
    return losses, dparams, dv

  def _actions(self, action, N, A):
    if self._actor_network.discrete:
      return action.reshape(N).to(torch.int32).contiguous()
    return action.float().reshape(N, A).contiguous()

  def _forward_loss(self, experience, returns, weights, keep_tape):
    if not isinstance(experience, trajectory.Trajectory):
      raise TypeError('Input type not supported: {}'.format(type(experience)))
    tf_agent.validate_trajectory(experience, self.training_data_spec, None)
    obs = nest.flatten(experience.observation)[0]
    B, T = obs.shape[0], obs.shape[1]
    N = B * T
    obs = obs.reshape((N,) + tuple(obs.shape[2:])).contiguous()
    dev = obs.device
    if keep_tape:
      params, actx = self._actor_network.forward_train(obs)
    else:
      params, actx = self._actor_network.distribution_params(obs), None
    v = vtape = None
    if self._baseline:
      if keep_tape:
        v, vtape = self._value_network.forward_train(obs)
      else:
        v, _ = self._value_network(obs)
      v = v.reshape(N).contiguous()
    if weights is not None:
      weights = torch.as_tensor(weights, dtype=torch.float32, device=dev).expand(B, T).contiguous()
    A = self._actor_network.num_actions
    losses, dparams, dv = self._launch(
        params, self._actions(experience.action, N, A), returns.float().contiguous(), v,
        experience.step_type.to(torch.int32).contiguous(),
        experience.next_step_type.to(torch.int32).contiguous(), weights, B, T,
        self._use_advantage, self._normalize_returns, self._entropy_coef(),
        self._value_estimation_loss_coef)
    self._regularization_losses(losses)
    return losses, (actx, dparams, vtape, dv)

  def _regularization_losses(self, losses):
    """The networks' L2 kernel regularisers (Network.losses, tf.nn.scale_regularization_loss on
    one replica) into losses[1] (actor) / losses[4] (value) and the total losses[5]."""
    for net, slot in ((self._actor_network, 1), (self._value_network, 4)):
      if net is None:
        continue
      for coef, w in net.losses:
        for dst in (slot, 5):
          _lib.call('b200rl_l2_sum', _lib.ptr(w), w.numel(), float(coef),
                    losses.data_ptr() + 4 * dst, _lib.stream())

  def _returns(self, experience):
    """discounted_return(reward, (next_step_type != LAST) * discount * gamma), batch-major, final
    value 0 (:262-269)."""
    reward = experience.reward.float().contiguous()
    B, T = reward.shape
    disc = torch.empty((B, T), dtype=torch.float32, device=reward.device)
    _lib.call('b200rl_ppo_discounts', _lib.ptr(experience.discount.float().contiguous()),
              _lib.ptr(experience.next_step_type.to(torch.int32).contiguous()), self._gamma,
              B * T, _lib.ptr(disc), _lib.stream())
    returns = torch.empty((B, T), dtype=torch.float32, device=reward.device)
    _lib.call('b200rl_discounted_return', _lib.ptr(reward), _lib.ptr(disc), None,
              _lib.ptr(returns), B, T, 0, 1, _lib.stream())
    return returns

  @staticmethod
  def _loss_info(losses):
    extra = ReinforceAgentLossInfo(
        policy_gradient_loss=losses[0], policy_network_regularization_loss=losses[1],
        entropy_regularization_loss=losses[2], value_estimation_loss=losses[3],
        value_network_regularization_loss=losses[4])
    return tf_agent.LossInfo(losses[5], extra)

  # ---- train (:255-311) --------------------------------------------------------------------------
  def _train(self, experience, weights=None):
    if self.replicas > 1:
      raise NotImplementedError('ReinforceAgent trains on one replica: the normalisation moments '
                                'and num_episodes would have to be reduced across replicas.')
    if self._optimizer is None:
      raise ValueError('Optimizer is undefined.')
    returns = self._returns(experience)
    losses, (actx, dparams, vtape, dv) = self._forward_loss(experience, returns, weights,
                                                            keep_tape=True)
    if not torch.cuda.is_current_stream_capturing():
      flag = int(self._flag.item())           # the one host read of an eager step
      if flag & _FLAG_NO_EPISODE:
        self._flag.fill_(flag & ~_FLAG_NO_EPISODE)
        raise ValueError(NO_EPISODE_MESSAGE)
    self._actor_network.backward(actx, dparams)
    if self._baseline:
      self._value_network.backward(vtape, dv.reshape(-1, 1))
    self._regularization_grads()
    if self._gradient_clipping:                  # eager_utils.clip_gradient_norms, per variable
      if self._clip_offsets is None:
        self._clip_offsets = torch.tensor(self._clip_offsets_host, dtype=torch.int64,
                                          device=self._flat_grads.device)
      _lib.call('b200rl_clip_by_norm_segments', _lib.ptr(self._flat_grads),
                _lib.ptr(self._clip_offsets), len(self._clip_offsets_host) - 1,
                float(self._gradient_clipping), _lib.stream())
    self._optimizer.apply_flat(self._flat_params, self._flat_grads)
    self._bump_train_step(1)
    return self._loss_info(losses)

  def _regularization_grads(self):
    """d(coef * sum(kernel^2)) = 2 * coef * kernel, added after the backward passes (which
    overwrite the gradient buffer)."""
    for net in (self._actor_network, self._value_network):
      if net is None:
        continue
      for coef, w in net.losses:
        off = (w.data_ptr() - self._flat_params.data_ptr()) // 4
        g = self._flat_grads[off:off + w.numel()]
        _lib.call('b200rl_add_scaled', _lib.ptr(g), _lib.ptr(w), w.numel(), 2.0 * float(coef),
                  _lib.stream())

  def _loss(self, experience, weights=None, training=False):
    return self.total_loss(experience, self._returns(experience), weights, training)

  # ---- public losses (:313-567) ------------------------------------------------------------------
  def total_loss(self, experience, returns, weights, training=False):
    """LossInfo(total, ReinforceAgentLossInfo) of [B, T] experience and returns (:313-440).
    Launches the fused kernel without a backward or an update; a batch without a complete
    episode sets the flag that check_numerics() reports."""
    losses, _ = self._forward_loss(experience, returns, weights, keep_tape=False)
    return self._loss_info(losses)

  def _params_rows(self, actions_distribution):
    flat = lambda t: t.float().reshape(-1, t.shape[-1]).contiguous()
    if isinstance(actions_distribution, (tuple, list)):
      return tuple(flat(t) for t in actions_distribution)
    return flat(actions_distribution)

  def _rows_launch(self, params, actions, step_type, returns, weights, value, entropy_coef,
                   value_coef):
    """One [1, N] launch in which every row ends an episode (next_step_type = LAST), so the kernel
    divides by N and applies no validity mask."""
    p0 = params[0] if isinstance(params, tuple) else params
    N, A = p0.shape
    dev = p0.device
    if isinstance(params, tuple):
      actions = actions.float().reshape(N, A).contiguous()
    else:
      actions = actions.reshape(N).to(torch.int32).contiguous()
    f = lambda t: None if t is None else torch.as_tensor(
        t, dtype=torch.float32, device=dev).expand(N).contiguous()
    nst = torch.full((N,), _STEP_LAST, dtype=torch.int32, device=dev)
    losses, _, _ = self._launch(params, actions, f(returns), f(value), step_type, nst, f(weights),
                                1, N, False, False, entropy_coef, value_coef)
    return losses, N

  def policy_gradient_loss(self, actions_distribution, actions, is_boundary, returns,
                           num_episodes, weights=None):
    """-sum(log pi(a) * ~is_boundary * returns * weights) / num_episodes (:442-506).
    actions_distribution: (loc, scale) [N, A] tensors, or [N, A] logits."""
    params = self._params_rows(actions_distribution)
    dev = (params[0] if isinstance(params, tuple) else params).device
    bnd = torch.as_tensor(is_boundary, device=dev).reshape(-1).bool()
    step_type = torch.where(bnd, _STEP_LAST, _STEP_MID).to(torch.int32).contiguous()
    losses, N = self._rows_launch(params, torch.as_tensor(actions, device=dev), step_type,
                                  returns, weights, None, 0.0, 0.0)
    return losses[0] * (float(N) / torch.as_tensor(num_episodes, dtype=torch.float32, device=dev))

  def entropy_regularization_loss(self, actions_distribution, weights=None):
    """entropy_regularization * mean(-H * weights); 0 without entropy regularisation (:508-534)."""
    params = self._params_rows(actions_distribution)
    p0 = params[0] if isinstance(params, tuple) else params
    if not self._entropy_regularization:
      return torch.zeros((), dtype=torch.float32, device=p0.device)
    N = p0.shape[0]
    zeros_a = torch.zeros((N, p0.shape[1]) if isinstance(params, tuple) else (N,),
                          device=p0.device)
    step_type = torch.full((N,), _STEP_MID, dtype=torch.int32, device=p0.device)
    losses, _ = self._rows_launch(params, zeros_a, step_type, 0.0, weights, None,
                                  self._entropy_coef(), 0.0)
    return losses[2]

  def value_estimation_loss(self, value_preds, returns, num_episodes, weights=None):
    """value_estimation_loss_coef * sum((returns - V)^2 * weights) / num_episodes (:536-567)."""
    v = torch.as_tensor(value_preds, dtype=torch.float32).reshape(-1)
    dev, N = v.device, v.numel()
    logits = torch.zeros((N, 1), dtype=torch.float32, device=dev)    # log pi = 0, H = 0
    step_type = torch.full((N,), _STEP_MID, dtype=torch.int32, device=dev)
    losses, _ = self._rows_launch(logits, torch.zeros(N, dtype=torch.int32, device=dev),
                                  step_type, returns, weights, v,
                                  0.0, self._value_estimation_loss_coef)
    return losses[3] * (float(N) / torch.as_tensor(num_episodes, dtype=torch.float32, device=dev))

  def check_numerics(self):
    """Raises if a loss so far was inf / nan, an action was out of range, or a batch held no
    complete episode (the captured-graph form of the eager ValueError); syncs the stream."""
    flag = int(self._flag.item())
    if flag & _FLAG_NO_EPISODE:
      raise FloatingPointError(NO_EPISODE_MESSAGE)
    if flag & _FLAG_NONFINITE:
      raise FloatingPointError('Loss is inf or nan')
