"""QT-Opt agent on libb200rl.

Drop-in for `tf_agents.agents.qtopt.qtopt_agent.QtOptAgent` (Kalashnikov et al. 2018) with a
stateless CriticNetwork Q(s, a) and the continuous GaussianActionsSampler.  There is no actor:
`policy` is CEMPolicy(target_q_network), a cross-entropy-method search for argmax_a Q(s, a), and
`collect_policy` is EpsilonGreedyPolicy(policy), which replaces a row with a uniform action with
probability epsilon_greedy.  `train(experience[B, n_step_update + 1, ...])` follows the reference:
  n-step reduction of reward and discount (b200rl_nstep_reduce) ->
  a' = CEM search on the TARGET network at s' ->
  next_q = min(Q_delayed(s', a'), Q_delayed_2(s', a')) with enable_td3, else Q_target(s', a') ->
  y = reward_scale r + gamma d next_q; td_loss = m l(y, Q(s, a)) with m = ~is_last(s) ->
  loss = sum_b w_b td_loss_b / B + regularisation -> backward -> [per-variable clip] ->
  optimiser step -> train_step_counter += 1 ->
  delayed_2 <- delayed, then delayed <- target (tau 1, delayed_target_update_period each), then
  target <- q (target_update_tau, target_update_period), each on its own Periodically counter;
  in this order delayed_2 receives the delayed weights from before the step's update.
l is `common.element_wise_huber_loss` (the default) or `common.element_wise_squared_loss`;
anything else raises ValueError.  Without enable_td3 next_q is the search's own best score, the
target network's value at a' (the reference evaluates the same network at the same action again).

Device work per step (csrc/qtopt.cu, scans.cu, nn.cu, optim.cu): nstep_reduce; [observation
branch of the target on B rows]; cem_sample; num_iter_cem x (target joint-stack forward over the
B*N rows + cem_refit); [two delayed forwards at (s', a')]; the online forward; fused TD loss + dQ;
backward; [clip]; optimiser; counter; one to three Polyak launches.

Not supported (raise): in_graph_bellman_update=False, RNN Q-networks, auxiliary_loss_fns,
emit_log_probability, nested or discrete action specs, more than one replica.

Extension (keyword-only): `train(..., noise=(z,))` supplies the N(0, 1) draws z
[num_iter_cem, B, num_samples_cem, A] of the target-side search ("noise mode" of the parity tests).
"""
import collections

import torch

from agents_b200 import _lib
from agents_b200.agents import tf_agent
from agents_b200.agents.td3 import td3_agent
from agents_b200.policies import epsilon_greedy_policy
from agents_b200.policies import qtopt_cem_policy
from agents_b200.trajectories import trajectory
from agents_b200.utils import common
from agents_b200.utils import nest


class QtOptLossInfo(collections.namedtuple('QtOptLossInfo', ('td_loss', 'td_error'))):
  """Per-example masked TD loss (unweighted) and TD error (qtopt_agent.py:53-74)."""


class QtOptAgent(tf_agent.TFAgent):
  """A QT-Opt agent."""

  def __init__(self, time_step_spec, action_spec, q_network, optimizer, actions_sampler,
               epsilon_greedy=0.1, n_step_update=1, emit_log_probability=False,
               in_graph_bellman_update=True, init_mean_cem=None, init_var_cem=None,
               num_samples_cem=32, num_elites_cem=4, num_iter_cem=3, target_q_network=None,
               target_update_tau=1.0, target_update_period=1, enable_td3=True,
               target_q_network_delayed=None, target_q_network_delayed_2=None,
               delayed_target_update_period=5, td_errors_loss_fn=None, auxiliary_loss_fns=None,
               gamma=1.0, reward_scale_factor=1.0, gradient_clipping=None, debug_summaries=False,
               summarize_grads_and_vars=False, train_step_counter=None, info_spec=None, name=None,
               seed=0):
    if not in_graph_bellman_update:
      raise NotImplementedError('in_graph_bellman_update=False (target_q stored in replay) is not '
                                'supported.')
    if getattr(q_network, 'state_spec', ()):
      raise NotImplementedError('QtOptAgent supports stateless (non-RNN) Q-networks only.')
    if auxiliary_loss_fns:
      raise NotImplementedError('auxiliary_loss_fns are not supported.')
    if emit_log_probability:
      raise NotImplementedError('emit_log_probability is not supported.')
    flat = nest.flatten(action_spec)
    if len(flat) != 1 or not flat[0].dtype.is_floating_point or len(flat[0].shape) != 1:
      raise ValueError('QtOptAgent supports one rank-1 bounded float action, got {}.'.format(
          action_spec))
    if init_mean_cem is None or init_var_cem is None:
      raise ValueError('init_mean_cem and init_var_cem are required.')
    if int(n_step_update) < 1:
      raise ValueError('n_step_update must be >= 1.')
    if not enable_td3 and (target_q_network_delayed or target_q_network_delayed_2):
      raise ValueError('enable_td3 is set to False but target_q_network_delayed or '
                       'target_q_network_delayed_2 is passed.')
    self._loss_kind = td3_agent._loss_kind(td_errors_loss_fn)
    self._sampler = actions_sampler
    self._q_network = q_network
    q_network.create_variables()
    self._target_q_network = self._copy(q_network, target_q_network, 'TargetQNetwork')
    self._enable_td3 = bool(enable_td3)
    self._target_q_network_delayed = self._target_q_network_delayed_2 = None
    device = q_network.device
    if self._enable_td3:
      self._target_q_network_delayed = self._copy(q_network, target_q_network_delayed,
                                                  'TargetQNetworkDelayed')
      self._target_q_network_delayed_2 = self._copy(q_network, target_q_network_delayed_2,
                                                    'TargetQNetworkDelayed2')
      self._target_updater_delayed_2 = common.Periodically(
          lambda period, ctr: common.soft_variables_update(
              self._target_q_network_delayed, self._target_q_network_delayed_2, 1.0,
              period=period, counter=ctr),
          delayed_target_update_period, 'periodic_update_targets_delayed', device=device)
      self._target_updater_delayed = common.Periodically(
          lambda period, ctr: common.soft_variables_update(
              self._target_q_network, self._target_q_network_delayed, 1.0, period=period,
              counter=ctr),
          delayed_target_update_period, 'periodic_update_targets_delayed', device=device)
    # the target <- q updater keeps the name the other agents use, so its counter is checkpointed
    # the same way
    self._update_target = common.Periodically(
        lambda period, ctr: common.soft_variables_update(
            self._q_network, self._target_q_network, target_update_tau, period=period,
            counter=ctr),
        target_update_period, 'periodic_update_targets', device=device)
    self._epsilon_greedy = epsilon_greedy
    self._n_step_update = int(n_step_update)
    self._optimizer = optimizer
    self._gamma, self._reward_scale_factor = gamma, reward_scale_factor
    self._gradient_clipping = gradient_clipping
    self._clip_offsets = None
    policy = qtopt_cem_policy.CEMPolicy(
        time_step_spec, action_spec, q_network=self._target_q_network, sampler=actions_sampler,
        init_mean=init_mean_cem, init_var=init_var_cem, num_samples=num_samples_cem,
        num_elites=num_elites_cem, num_iterations=num_iter_cem, training=False, seed=seed)
    collect_policy = epsilon_greedy_policy.EpsilonGreedyPolicy(policy, epsilon=epsilon_greedy,
                                                               seed=seed)
    super(QtOptAgent, self).__init__(
        time_step_spec, action_spec, policy, collect_policy,
        train_sequence_length=self._n_step_update + 1, debug_summaries=debug_summaries,
        summarize_grads_and_vars=summarize_grads_and_vars, train_step_counter=train_step_counter,
        device=device)
    self._nan_flag = torch.zeros(1, dtype=torch.int32, device=device)
    self.replicas = 1
    self._grad_sync = None

  @staticmethod
  def _copy(q_network, net, name):
    if net is None:
      net = q_network.copy(name=name)
    elif net is q_network:
      raise ValueError('Shared variables found in q_network and {}.'.format(name))
    net.create_variables()
    return net

  @property
  def policy_q_network(self):
    return self._target_q_network

  @property
  def enable_td3(self):
    return self._enable_td3

  def _initialize(self):
    """Hard-copies q into the target and both delayed networks (qtopt_agent.py:416-431)."""
    common.soft_variables_update(self._q_network, self._target_q_network, tau=1.0)
    if self._enable_td3:
      common.soft_variables_update(self._q_network, self._target_q_network_delayed, tau=1.0)
      common.soft_variables_update(self._q_network, self._target_q_network_delayed_2, tau=1.0)

  def _update_both(self):
    """qtopt_agent.py:433-436: delayed_2 <- delayed, delayed <- target, target <- q."""
    self._target_updater_delayed_2()
    self._target_updater_delayed()
    self._update_target()

  def _train(self, experience, weights=None, noise=None):
    if self.replicas != 1 or self._grad_sync is not None:
      raise NotImplementedError('QtOptAgent does not support data-parallel training.')
    if self._optimizer is None:
      raise ValueError('Optimizer is undefined.')
    loss, td_loss, td_error, dq, tape, reg = self._forward_loss(
        experience, weights, None if noise is None else noise[0])
    net = self._q_network
    grads = net.backward(tape, dq)
    for coef, w in reg:                      # d/dw coef*sum(w^2) = 2*coef*w
      off = w.data_ptr() - net.flat_params.data_ptr()
      _lib.call('b200rl_add_scaled', _lib.ptr(grads[off // 4: off // 4 + w.numel()]),
                _lib.ptr(w), w.numel(), 2.0 * float(coef), _lib.stream())
    if self._gradient_clipping is not None:  # eager_utils.clip_gradient_norms, per variable
      if self._clip_offsets is None:
        self._clip_offsets = torch.tensor(net.param_offsets, dtype=torch.int64,
                                          device=grads.device)
      _lib.call('b200rl_clip_by_norm_segments', _lib.ptr(grads), _lib.ptr(self._clip_offsets),
                len(net.param_offsets) - 1, float(self._gradient_clipping), _lib.stream())
    self._optimizer.apply_flat(net.flat_params, grads)
    self._bump_train_step(1)
    if self._enable_td3:
      self._update_both()
    else:
      self._update_target()
    return tf_agent.LossInfo(loss.reshape(()), QtOptLossInfo(td_loss=td_loss, td_error=td_error))

  def _loss(self, experience, weights=None, training=False, noise=None):
    """QT-Opt loss without an update (qtopt_agent.py:588-698)."""
    loss, td_loss, td_error, _, _, _ = self._forward_loss(
        experience, weights, None if noise is None else noise[0], keep=False)
    return tf_agent.LossInfo(loss.reshape(()), QtOptLossInfo(td_loss=td_loss, td_error=td_error))

  def _next_q(self, obs2, z):
    """Q of the next state at the target network's CEM action (qtopt_agent.py:712-748)."""
    a2, best = self._policy.search(obs2, z=z)
    if not self._enable_td3:
      return best, None
    d1, d2 = self._target_q_network_delayed, self._target_q_network_delayed_2
    ins = td3_agent.Td3Agent._stack_inputs([d1, d2], obs2, a2)
    return d1.forward_stack(*ins[0])[0], d2.forward_stack(*ins[1])[0]

  def _forward_loss(self, experience, weights, z, keep=True):
    if not isinstance(experience, trajectory.Trajectory):
      raise TypeError('Input type not supported: {}'.format(type(experience)))
    tf_agent.validate_trajectory(experience, self.training_data_spec,
                                 self._train_sequence_length)
    tr = trajectory.to_n_step_transition(experience, self._gamma)
    obs = nest.flatten(tr.time_step.observation)[0].float()
    obs2 = nest.flatten(tr.next_time_step.observation)[0].float()
    action = nest.flatten(tr.action_step.action)[0].float()
    B = obs.shape[0]
    tq1, tq2 = self._next_q(obs2, z)
    net = self._q_network
    x, otape = net.stack_input(obs, action, keep=keep)
    q, tape = net.forward_stack(x, otape, keep=keep)
    dev = q.device
    step = tr.time_step.step_type
    if step.dtype != torch.int32:
      step = step.to(torch.int32)
    step = step.contiguous()
    if weights is not None:
      weights = torch.as_tensor(weights, dtype=torch.float32, device=dev)
      weights = weights.expand(B).contiguous() if weights.dim() == 0 else weights.contiguous()
    loss = torch.empty(1, dtype=torch.float32, device=dev)
    td_loss = torch.empty(B, dtype=torch.float32, device=dev)
    td_error = torch.empty(B, dtype=torch.float32, device=dev)
    dq = torch.empty((B, 1), dtype=torch.float32, device=dev)
    _lib.call('b200rl_qtopt_td_loss', _lib.ptr(q), _lib.ptr(tq1), _lib.ptr(tq2),
              _lib.ptr(tr.next_time_step.reward), _lib.ptr(tr.next_time_step.discount),
              _lib.ptr(step), 1, _lib.ptr(weights), B, float(self._gamma),
              float(self._reward_scale_factor), self._loss_kind, _lib.ptr(loss),
              _lib.ptr(td_loss), _lib.ptr(td_error), _lib.ptr(dq), _lib.ptr(self._nan_flag),
              _lib.stream())
    reg = net.losses                         # common.aggregate_losses regularization_loss
    for coef, w in reg:
      _lib.call('b200rl_l2_sum', _lib.ptr(w), w.numel(), float(coef), _lib.ptr(loss),
                _lib.stream())
    return loss, td_loss, td_error, dq, tape, reg

  def check_numerics(self):
    if int(self._nan_flag.item()) != 0:
      raise FloatingPointError('Loss is inf or nan')
