"""DQN / Double-DQN agents on libb200rl.

Drop-in for `tf_agents.agents.dqn.dqn_agent.{DqnAgent, DdqnAgent}` (reference
agents/dqn/dqn_agent.py:82-700): same constructor arguments, `train(experience, weights)`
returning `LossInfo(loss, DqnLossInfo(td_loss, td_error))`, `policy` / `collect_policy`,
`train_sequence_length = n_step_update + 1`.

Device work per train step (all libb200rl, csrc/{nn,dqn,optim}.cu):
  Q(s_0) forward (activations kept), target Q(s_n) forward [, online Q(s_n) for DDQN]
  -> fused n-step / TD-target / Huber / mask / mean + dLoss/dq     (b200rl_dqn_td_loss)
  -> backward through the Q network                                   (dense/conv bwd)
  -> [per-variable clip_by_norm] -> fused optimiser step -> train_step += 1
  -> Periodically-gated Polyak/hard target update                     (b200rl_soft_update)
The reference evaluates the target network twice (:622 and inside the greedy policy :634);
both evaluations are identical, so it is evaluated once here.

With a recurrent q_network (QRnnNetwork, any LSTMEncodingNetwork) the agent trains on whole
[B, T] sequences, T >= 2 (train_sequence_length None, dqn_agent.py:264-299): transition t of a
sequence is (observation[:, t], action[:, t], reward[:, t], discount[:, t], observation[:, t+1])
(trajectory.to_transition).  The online network runs over observation[:, :-1] with
step_type[:, :-1], the target (and, for DDQN / D3QN, the online selector) over observation[:, 1:]
with next_step_type[:, :-1], each from the zero state; b200rl_dqn_seq_td_loss then forms the
[B, T-1] TD loss, sums it over time and aggregates it, and LSTMEncodingNetwork.backward runs BPTT.
"""
import collections

import torch

from agents_b200 import _lib
from agents_b200.agents import tf_agent
from agents_b200.policies import q_policy
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory
from agents_b200.utils import common
from agents_b200.utils import nest
from agents_b200.utils import workspace


class DqnLossInfo(collections.namedtuple('DqnLossInfo', ('td_loss', 'td_error'))):
  """Per-example TD loss and unweighted TD error (dqn_agent.py:53-72)."""


def compute_td_targets(next_q_values, rewards, discounts):
  """dqn_agent.py:75-78 (host composition; the train path uses the fused kernel)."""
  return (rewards + discounts * next_q_values).detach()


def _loss_kind(fn):
  if fn is None or fn is common.element_wise_huber_loss:
    return _lib.LOSS_HUBER
  if fn is common.element_wise_squared_loss:
    return _lib.LOSS_SQUARED
  raise ValueError('td_errors_loss_fn must be common.element_wise_huber_loss or '
                   'common.element_wise_squared_loss (custom Python losses cannot run inside '
                   'the fused CUDA epilogue).')


class DqnAgent(tf_agent.TFAgent):
  """A DQN agent (Mnih et al. 2015) with n-step updates."""

  _DOUBLE_Q = False          # select the bootstrap action with the online network
  _SELECT_UNMASKED = False   # D3qn: raw argmax over the selector's output (no action constraints)
  _FUSED_TD_LOSS = True      # False: td_errors_loss_fn is accepted but not used (CategoricalDqnAgent)
  # data-parallel runs all-reduce the gradient in buckets of at least this many bytes, overlapped
  # with the rest of the backward pass
  _bucket_bytes = 1 << 20

  def __init__(self, time_step_spec, action_spec, q_network, optimizer,
               observation_and_action_constraint_splitter=None, epsilon_greedy=0.1,
               n_step_update=1, boltzmann_temperature=None, emit_log_probability=False,
               target_q_network=None, target_update_tau=1.0, target_update_period=1,
               td_errors_loss_fn=None, gamma=1.0, reward_scale_factor=1.0,
               gradient_clipping=None, debug_summaries=False, summarize_grads_and_vars=False,
               train_step_counter=None, training_data_spec=None, name=None, seed=0):
    self._check_action_spec(action_spec)
    if epsilon_greedy is not None and boltzmann_temperature is not None:
      raise ValueError(
          'Configured both epsilon_greedy value {} and temperature {}, '
          'however only one of them can be used for exploration.'.format(
              epsilon_greedy, boltzmann_temperature))
    if boltzmann_temperature is not None:
      raise NotImplementedError('BoltzmannPolicy is outside the hot path (SURVEY.md §2.1).')
    self._splitter = observation_and_action_constraint_splitter
    self._q_network = q_network
    net_observation_spec = time_step_spec.observation
    if self._splitter is not None:
      net_observation_spec, _ = self._splitter(net_observation_spec)
    self._recurrent = bool(q_network.state_spec)
    if self._recurrent and n_step_update != 1:
      raise NotImplementedError(
          'DqnAgent does not currently support n-step updates with stateful '
          'networks (i.e., RNNs), but n_step_update = {}'.format(n_step_update))
    out = q_network.create_variables(net_observation_spec)
    if self._recurrent and tuple(out.shape) != (self._num_actions,):
      # e.g. a bare LSTMEncodingNetwork: an encoder, not a recurrent Q network
      raise NotImplementedError(
          'DqnAgent trains feed-forward Q networks and recurrent Q networks that emit ({},) Q '
          'values per step (QRnnNetwork); this stateful q_network emits {}.'.format(
              self._num_actions, tuple(out.shape)))
    if target_q_network is not None:
      target_q_network.create_variables(net_observation_spec)
      if target_q_network is q_network:
        raise ValueError('Shared variables found in q_network and target_q_network.')
      self._target_q_network = target_q_network
    else:
      self._target_q_network = q_network.copy(name='TargetQNetwork')
    device = q_network.device
    self._check_network_output(self._q_network, 'q_network')
    self._check_network_output(self._target_q_network, 'target_q_network')
    self._epsilon_greedy = epsilon_greedy
    self._n_step_update = n_step_update
    self._optimizer = optimizer
    self._td_errors_loss_fn = td_errors_loss_fn or common.element_wise_huber_loss
    self._loss_kind = _loss_kind(self._td_errors_loss_fn) if self._FUSED_TD_LOSS else None
    self._gamma = gamma
    self._reward_scale_factor = reward_scale_factor
    self._gradient_clipping = gradient_clipping
    self._target_update_tau = target_update_tau
    self._target_update_period = target_update_period
    self._update_target = self._get_target_updater(target_update_tau, target_update_period,
                                                   device)
    self._seed = seed
    policy, collect_policy = self._setup_policy(time_step_spec, action_spec)
    train_sequence_length = None if self._recurrent else n_step_update + 1
    super(DqnAgent, self).__init__(
        time_step_spec, action_spec, policy, collect_policy,
        train_sequence_length=train_sequence_length, debug_summaries=debug_summaries,
        summarize_grads_and_vars=summarize_grads_and_vars,
        train_step_counter=train_step_counter, training_data_spec=training_data_spec,
        device=device)
    self._nan_flag = torch.zeros(1, dtype=torch.int32, device=device)
    self._side_stream = torch.cuda.Stream(device=device)
    self._clip_offsets = None
    self.replicas = 1           # set by train.Learner for data-parallel runs
    self._grad_sync = None      # callable(flat_grads) installed by train.Learner
    self._comm_stream = torch.cuda.Stream(device=device)
    if self._recurrent:   # b200rl_dqn_seq_td_loss scratch: block partials and a last-block ticket
      self._seq_partials = torch.empty(_lib.DQN_SEQ_MAX_BLOCKS, dtype=torch.float32, device=device)
      self._seq_ticket = torch.zeros(1, dtype=torch.int32, device=device)

  # ---- construction helpers -----------------------------------------------------------------
  def _check_action_spec(self, action_spec):
    flat = nest.flatten(action_spec)
    if len(flat) > 1 or len(flat[0].shape) > 0:
      raise ValueError('Only scalar actions are supported now, but action spec is: {}'.format(
          action_spec))
    spec = flat[0]
    if spec.minimum != 0:
      raise ValueError('Action specs should have minimum of 0, but saw: {0}'.format(spec))
    self._num_actions = int(spec.maximum - spec.minimum + 1)

  def _check_network_output(self, net, label):
    out = net.create_variables()
    if tuple(out.shape) != (self._num_actions,):
      raise ValueError('Expected {} to emit a floating point tensor with inner dims ({},); but '
                       'saw network output spec: {}'.format(label, self._num_actions, out))

  def _setup_policy(self, time_step_spec, action_spec):
    policy = q_policy.QPolicy(time_step_spec, action_spec, q_network=self._q_network,
                              observation_and_action_constraint_splitter=self._splitter)
    collect_policy = q_policy.EpsilonGreedyPolicy(policy, epsilon=self._epsilon_greedy,
                                                  seed=self._seed)
    greedy = q_policy.GreedyPolicy(policy)
    self._target_policy = q_policy.QPolicy(
        time_step_spec, action_spec, q_network=self._target_q_network,
        observation_and_action_constraint_splitter=self._splitter)
    return greedy, collect_policy

  def _initialize(self):
    common.soft_variables_update(self._q_network, self._target_q_network, tau=1.0)

  def _get_target_updater(self, tau=1.0, period=1, device='cuda'):
    """Periodic soft update of the target network (dqn_agent.py:385-409)."""
    def update(period_, counter):
      common.soft_variables_update(self._q_network, self._target_q_network, tau,
                                   period=period_, counter=counter)
    return common.Periodically(update, period, 'periodic_update_targets', device=device)

  # ---- loss / train -------------------------------------------------------------------------
  def _split_obs(self, obs):
    if self._splitter is None:
      return obs, None
    return self._splitter(obs)

  def _prepare(self, experience):
    if not isinstance(experience, trajectory.Trajectory):
      raise TypeError('Input type not supported: {}'.format(type(experience)))
    tf_agent.validate_trajectory(experience, self.training_data_spec,
                                 self._train_sequence_length)
    return experience

  def _forward_loss(self, experience, weights, keep_tape):
    exp = self._prepare(experience)
    B, T = exp.discount.shape[0], exp.discount.shape[1]
    if self._recurrent:
      if self.replicas > 1:
        raise NotImplementedError('DqnAgent with a recurrent network trains on one replica.')
      if T < 2:
        raise ValueError('Trajectory frame count must be at least 2, but saw {}'.format(T))
      # [B, T-1] sequences: the online net sees time_steps, the target side next_time_steps
      obs0, _ = self._split_obs(nest.map_structure(lambda t: t[:, :-1], exp.observation))
      obsn, next_mask = self._split_obs(nest.map_structure(lambda t: t[:, 1:], exp.observation))
      if next_mask is not None:
        next_mask = next_mask.reshape(B * (T - 1), self._num_actions)
      online_args = (obs0, exp.step_type[:, :-1])
      target_args = (obsn, exp.next_step_type[:, :-1])
    else:
      obs0, _ = self._split_obs(nest.map_structure(lambda t: t[:, 0], exp.observation))
      obsn, next_mask = self._split_obs(nest.map_structure(lambda t: t[:, T - 1], exp.observation))
      online_args, target_args = (obs0,), (obsn,)
    # The target-side forwards do not depend on the online forward: inside a captured graph fork
    # them onto a side stream and join before the TD kernel (eager launches are host-bound, the
    # fork only pays inside a graph).
    main = torch.cuda.current_stream()
    side = self._side_stream if torch.cuda.is_current_stream_capturing() else None
    if side is not None:
      side.wait_stream(main)
    with torch.cuda.stream(side if side is not None else main), \
        workspace.slot(1 if side is not None else 0):
      next_t, _ = self._target_q_network(*target_args)
      if isinstance(next_t, tuple):                # dueling nets may emit (q, ...) (:723-726)
        next_t = next_t[0]
      next_sel = next_t
      if self._DOUBLE_Q:
        next_sel, _ = self._q_network(*target_args)  # DdqnAgent (dqn_agent.py:686-688)
        if isinstance(next_sel, tuple):            # D3qnAgent reads element 1 (:730)
          next_sel = next_sel[1] if self._SELECT_UNMASKED else next_sel[0]
    if self._SELECT_UNMASKED:
      next_mask = None                             # tf.math.argmax on the raw values (:731)
    if keep_tape:
      q, tape = self._q_network.forward_train(*online_args)
    else:
      (q, _), tape = self._q_network(*online_args), None
    if side is not None:
      main.wait_stream(side)
    else:
      workspace.mirror(q.device, 1)   # size the side-stream scratch for a later capture
    if self._recurrent:
      rows = (B * (T - 1), self._num_actions)
      return self._td_seq(exp, B, T, q.reshape(rows), next_t.reshape(rows),
                          next_sel.reshape(rows), next_mask, weights, tape)
    return self._td(exp, B, T, q, next_t, next_sel, next_mask, weights, tape)

  def _td(self, exp, B, T, q, next_t, next_sel, next_mask, weights, tape):
    """TD targets, element-wise loss and dLoss/dq from the three Q tables (one kernel)."""
    dev = q.device
    # [:, 0] columns of the [B, T] tensors are read in place (no gather/cast launches)
    actions, a_stride = self._column0(exp.action)
    step0, s_stride = self._column0(exp.step_type)
    rew = exp.reward.float().contiguous()
    disc = exp.discount.float().contiguous()
    if weights is not None:
      weights = torch.as_tensor(weights, dtype=torch.float32, device=dev)
      weights = weights.expand(B).contiguous() if weights.dim() == 0 else weights.contiguous()
    if next_mask is not None:
      next_mask = next_mask.to(torch.int32).contiguous()
    loss = torch.empty(1, dtype=torch.float32, device=dev)
    td_loss = torch.empty(B, dtype=torch.float32, device=dev)
    td_error = torch.empty(B, dtype=torch.float32, device=dev)
    dq = torch.empty((B, self._num_actions), dtype=torch.float32, device=dev)
    _lib.call('b200rl_dqn_td_loss', _lib.ptr(q), _lib.ptr(next_t), _lib.ptr(next_sel),
              _lib.ptr(next_mask), _lib.dptr(actions), _lib.dptr(step0), _lib.ptr(rew),
              _lib.ptr(disc), _lib.ptr(weights), a_stride, s_stride, B, self._num_actions, T,
              float(self._gamma),
              float(self._reward_scale_factor), self._loss_kind, float(B * self.replicas),
              _lib.ptr(loss), _lib.ptr(td_loss), _lib.ptr(td_error), _lib.ptr(dq),
              _lib.ptr(self._nan_flag), _lib.stream())
    return loss, td_loss, td_error, dq, tape, self._add_reg_loss(loss)

  def _td_seq(self, exp, B, T, q, next_t, next_sel, next_mask, weights, tape):
    """The [B, T-1] sequence TD loss and dLoss/dq from the three [B*(T-1), A] tables (one kernel);
    td_loss is [B] (summed over time) and td_error [B, T-1]."""
    dev = q.device
    actions, a_ld, a_st = self._int32_bt(exp.action)
    steps, s_ld, s_st = self._int32_bt(exp.step_type)
    rew = exp.reward.float().contiguous()
    disc = exp.discount.float().contiguous()
    w_stride = 0
    if weights is not None:
      weights = torch.as_tensor(weights, dtype=torch.float32, device=dev)
      if weights.numel() > 1:
        weights, w_stride = weights.reshape(B).contiguous(), 1
    if next_mask is not None:
      next_mask = next_mask.to(torch.int32).contiguous()
    loss = torch.empty(1, dtype=torch.float32, device=dev)
    td_loss = torch.empty(B, dtype=torch.float32, device=dev)
    td_error = torch.empty((B, T - 1), dtype=torch.float32, device=dev)
    dq = torch.empty_like(q)
    _lib.call('b200rl_dqn_seq_td_loss', _lib.ptr(q), _lib.ptr(next_t), _lib.ptr(next_sel),
              _lib.ptr(next_mask), _lib.dptr(actions), a_ld, a_st,
              _lib.dptr(steps), s_ld, s_st, _lib.ptr(rew), _lib.ptr(disc), _lib.ptr(weights),
              w_stride, B, self._num_actions, T, float(self._gamma),
              float(self._reward_scale_factor), self._loss_kind, float(B), _lib.ptr(loss),
              _lib.ptr(td_loss), _lib.ptr(td_error), _lib.ptr(dq), _lib.ptr(self._nan_flag),
              _lib.ptr(self._seq_partials), _lib.ptr(self._seq_ticket), _lib.stream())
    return loss, td_loss, td_error, dq, tape, self._add_reg_loss(loss)

  def _add_reg_loss(self, loss):
    """Adds the regularisation losses to `loss` (common.aggregate_losses :1470-1475)."""
    reg = self._q_network.losses
    for coef, w in reg:
      _lib.call('b200rl_l2_sum', _lib.ptr(w), w.numel(), float(coef) / self.replicas,
                _lib.ptr(loss), _lib.stream())
    return reg

  @staticmethod
  def _column0(t):
    """(tensor, element stride) such that element b of column 0 of `t` [B, T] is
    tensor.data_ptr()[b * stride]; int32 storage is used as is, other dtypes are cast once."""
    col = t[:, 0]
    if col.dtype != torch.int32:
      return col.to(torch.int32).contiguous(), 1
    return col, (col.stride(0) if col.numel() > 1 else 1)

  @staticmethod
  def _int32_bt(t):
    """(tensor, row stride, time stride) of an int [B, T] tensor: element (b, t) is
    tensor.data_ptr()[b * row + t * time]; int32 storage is read in place, other dtypes are cast
    once."""
    if t.dtype != torch.int32:
      t = t.to(torch.int32).contiguous()
    return t, t.stride(0), t.stride(1)

  def _loss(self, experience, td_errors_loss_fn=None, gamma=None, reward_scale_factor=None,
            weights=None, training=False):
    """DQN loss (dqn_agent.py:462-579)."""
    loss, td_loss, td_error, _, _, _ = self._forward_loss(experience, weights, keep_tape=False)
    return tf_agent.LossInfo(loss.reshape(()), DqnLossInfo(td_loss=td_loss, td_error=td_error))

  def _train(self, experience, weights=None):
    """One gradient step (dqn_agent.py:412-449)."""
    loss, td_loss, td_error, dq, tape, reg = self._forward_loss(experience, weights,
                                                                keep_tape=True)
    net = self._q_network
    # Data-parallel runs: start the all-reduce of the gradient tail (the fc layers come out of
    # the backward pass first and hold 95 % of the bytes of the Atari net) on a communication
    # stream as soon as it is complete, and reduce the small head after the last conv gradient.
    bucketed = self._grad_sync is not None and not reg
    hook = None
    if bucketed:
      total = net.flat_grads.numel()
      state = {'lo': total, 'sent': total}
      comm = self._comm_stream

      def hook(lo, hi):
        state['lo'] = min(state['lo'], lo)
        if (state['sent'] - state['lo']) * 4 >= self._bucket_bytes:
          cur = torch.cuda.current_stream()
          comm.wait_stream(cur)
          with torch.cuda.stream(comm):
            self._grad_sync(net.flat_grads[state['lo']:state['sent']])
          state['sent'] = state['lo']
    # (the recurrent backward takes no hook: bucketed is False on its one replica)
    grads = net.backward(tape, dq, grad_hook=hook) if bucketed else net.backward(tape, dq)
    if bucketed:
      main = torch.cuda.current_stream()
      if state['sent'] > 0:
        self._comm_stream.wait_stream(main)
        with torch.cuda.stream(self._comm_stream):
          self._grad_sync(grads[0:state['sent']])
      main.wait_stream(self._comm_stream)
    for coef, w in reg:  # d/dw coef*sum(w^2) = 2*coef*w
      off = w.data_ptr() - net.flat_params.data_ptr()
      g = grads[off // 4: off // 4 + w.numel()]
      _lib.call('b200rl_add_scaled', _lib.ptr(g), _lib.ptr(w), w.numel(),
                2.0 * float(coef) / self.replicas, _lib.stream())
    if self._grad_sync is not None and not bucketed:
      self._grad_sync(grads)
    if self._gradient_clipping is not None:    # eager_utils.clip_gradient_norms, per variable
      if self._clip_offsets is None:
        self._clip_offsets = torch.tensor(net.param_offsets, dtype=torch.int64,
                                          device=grads.device)
      _lib.call('b200rl_clip_by_norm_segments', _lib.ptr(grads), _lib.ptr(self._clip_offsets),
                len(net.param_offsets) - 1, float(self._gradient_clipping), _lib.stream())
    self._optimizer.apply_flat(net.flat_params, grads)
    self._bump_train_step(1)
    self._update_target()
    return tf_agent.LossInfo(loss.reshape(()), DqnLossInfo(td_loss=td_loss, td_error=td_error))

  def check_numerics(self):
    """Raises if any loss so far was inf/nan (dqn_agent.py:422); syncs the stream."""
    if int(self._nan_flag.item()) != 0:
      raise FloatingPointError('Loss is inf or nan')


class DdqnAgent(DqnAgent):
  """Double DQN (van Hasselt et al. 2015; dqn_agent.py:649-700)."""
  _DOUBLE_Q = True


class D3qnAgent(DqnAgent):
  """Double Dueling DQN (Wang et al. 2016; dqn_agent.py:704-753).

  Like DdqnAgent the bootstrap action comes from the ONLINE network evaluated at s_n, but it is
  a plain `tf.math.argmax` of that output (:731) -- it does not go through the greedy policy, so
  an `observation_and_action_constraint_splitter` mask is NOT applied to the selection (the
  reference's masked-action test expects 26.0 for this agent and 23.75 for the other two,
  dqn_agent_test.py:556).  The value is still read from the target network (:737-741).
  """
  _DOUBLE_Q = True
  _SELECT_UNMASKED = True
