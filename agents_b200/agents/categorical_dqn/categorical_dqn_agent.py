"""Categorical DQN (C51, Bellemare et al. 2017) on libb200rl.

Drop-in for `tf_agents.agents.categorical_dqn.categorical_dqn_agent.CategoricalDqnAgent`
(reference agents/categorical_dqn/categorical_dqn_agent.py:49-556): same constructor arguments,
`train(experience, weights)` returning `LossInfo(loss, DqnLossInfo(td_loss=(), td_error=()))`.

Everything but the loss is DqnAgent's: the online/target forward fork, the backward pass,
per-variable gradient clipping, the optimiser, the train-step counter, the Periodically target
update and the L2 terms.  The loss is one b200rl_c51_loss call (csrc/categorical_dqn.cu): target
softmax, expected-Q masked argmax, projection of the Bellman-shifted support, cross entropy of
the taken action's logits and its gradient.

Reference behaviour kept on purpose:
  * no LAST-step valid mask (DqnAgent masks, :271-518 does not);
  * `weights` is accepted and ignored: _loss never passes it to aggregate_losses (:463-466);
  * `td_errors_loss_fn` is accepted and unused;
  * DqnLossInfo(td_loss=(), td_error=()) (:516-518).
"""
import numpy as np
import torch

from agents_b200 import _lib
from agents_b200.agents.dqn import dqn_agent
from agents_b200.policies import categorical_q_policy
from agents_b200.policies import q_policy


def _linspace_f32(start, stop, num):
  """tf.linspace in float32 (:194-196): start, start + i * delta (i = 1 .. num-2), stop, with
  delta = (stop - start) / (num - 1) and every operation rounded to float32."""
  f32 = np.float32
  start, stop = f32(start), f32(stop)
  delta = f32(stop - start) / f32(num - 1)
  mid = (start + (np.arange(1, num - 1).astype(f32) * delta).astype(f32)).astype(f32)
  return np.concatenate([[start], mid, [stop]]).astype(f32)


def _check_atoms(net, label):
  try:
    return net.num_atoms
  except AttributeError:                                                      # :165-174
    raise TypeError('Expected {} to have property `num_atoms`, but it doesn\'t. (Note: you likely '
                    'want to use a CategoricalQNetwork.) Network is: {}'.format(label, net))


class CategoricalDqnAgent(dqn_agent.DqnAgent):
  """A Categorical DQN agent based on DqnAgent (categorical_dqn_agent.py:49-556)."""

  _FUSED_TD_LOSS = False

  def __init__(self, time_step_spec, action_spec, categorical_q_network, optimizer,
               observation_and_action_constraint_splitter=None, min_q_value=-10.0,
               max_q_value=10.0, epsilon_greedy=0.1, n_step_update=1, boltzmann_temperature=None,
               target_categorical_q_network=None, target_update_tau=1.0, target_update_period=1,
               td_errors_loss_fn=None, gamma=1.0, reward_scale_factor=1.0,
               gradient_clipping=None, debug_summaries=False, summarize_grads_and_vars=False,
               train_step_counter=None, name=None, seed=0):
    self._num_atoms = int(_check_atoms(categorical_q_network, 'categorical_q_network'))
    if target_categorical_q_network is not None:
      target_num_atoms = _check_atoms(target_categorical_q_network, 'target_categorical_q_network')
      if self._num_atoms != target_num_atoms:                                 # :184-190
        raise ValueError('categorical_q_network and target_categorical_q_network have different '
                         'numbers of atoms: {} vs. {}'.format(self._num_atoms, target_num_atoms))
    for net in (categorical_q_network, target_categorical_q_network):
      if net is not None and getattr(net, 'state_spec', ()):
        raise NotImplementedError('CategoricalDqnAgent supports stateless networks only; RNN '
                                  'Q-networks are not built.')
    self._min_q_value = min_q_value
    self._max_q_value = max_q_value
    self._support = torch.as_tensor(_linspace_f32(min_q_value, max_q_value, self._num_atoms),
                                    device=categorical_q_network.device)
    super(CategoricalDqnAgent, self).__init__(
        time_step_spec, action_spec, categorical_q_network, optimizer,
        observation_and_action_constraint_splitter=observation_and_action_constraint_splitter,
        epsilon_greedy=epsilon_greedy, n_step_update=n_step_update,
        boltzmann_temperature=boltzmann_temperature,
        target_q_network=target_categorical_q_network, target_update_tau=target_update_tau,
        target_update_period=target_update_period, td_errors_loss_fn=td_errors_loss_fn,
        gamma=gamma, reward_scale_factor=reward_scale_factor, gradient_clipping=gradient_clipping,
        debug_summaries=debug_summaries, summarize_grads_and_vars=summarize_grads_and_vars,
        train_step_counter=train_step_counter, name=name, seed=seed)

  def _check_network_output(self, net, label):
    """network_utils.check_single_floating_network_output against (A, N) (:264-269)."""
    out = net.create_variables()
    expected = (self._num_actions, self._num_atoms)
    if tuple(out.shape) != expected:
      raise ValueError('Expected {} to emit a floating point tensor with inner dims {}; but saw '
                       'network output spec: {}'.format(label, expected, out))

  def _setup_policy(self, time_step_spec, action_spec):
    """:222-262 (the Boltzmann collect policy is not built: DqnAgent raises for it)."""
    policy = categorical_q_policy.CategoricalQPolicy(
        time_step_spec, action_spec, self._q_network, self._min_q_value, self._max_q_value,
        observation_and_action_constraint_splitter=self._splitter)
    collect_policy = q_policy.EpsilonGreedyPolicy(policy, epsilon=self._epsilon_greedy,
                                                  seed=self._seed)
    self._target_policy = categorical_q_policy.CategoricalQPolicy(
        time_step_spec, action_spec, self._target_q_network, self._min_q_value,
        self._max_q_value, observation_and_action_constraint_splitter=self._splitter)
    return q_policy.GreedyPolicy(policy), collect_policy

  def _td(self, exp, B, T, q, next_t, next_sel, next_mask, weights, tape):
    """Cross-entropy loss and dLoss/dlogits from the online and target logits (one call).

    `weights` is ignored like the reference's (:463-466).  The projection uses the agent's
    tf.linspace support (:196); the target greedy action is taken with the target policy's own
    np.linspace support (categorical_q_policy.py:141-144), as the reference's
    `_target_greedy_policy` does (:545-550)."""
    del next_sel, weights
    if self.replicas > 1:
      raise NotImplementedError('CategoricalDqnAgent trains on one replica.')
    dev = q.device
    actions, a_stride = self._column0(exp.action)
    rew = exp.reward.float().contiguous()
    disc = exp.discount.float().contiguous()
    if next_mask is not None:
      next_mask = next_mask.to(torch.int32).contiguous()
    A, N = self._num_actions, self._num_atoms
    loss = torch.empty(1, dtype=torch.float32, device=dev)
    dq = torch.empty((B, A * N), dtype=torch.float32, device=dev)
    rows = torch.empty(B, dtype=torch.float32, device=dev)
    _lib.call('b200rl_c51_loss', _lib.ptr(q), _lib.ptr(next_t), _lib.ptr(next_mask),
              _lib.dptr(actions), a_stride, _lib.ptr(rew), _lib.ptr(disc), _lib.ptr(self._support),
              _lib.ptr(self._target_policy.support), B, A, N, T, float(self._gamma),
              float(self._reward_scale_factor), float(B * self.replicas), _lib.ptr(loss), _lib.ptr(dq), _lib.ptr(self._nan_flag),
              _lib.ptr(rows), 4 * B, _lib.stream())
    reg = self._q_network.losses
    for coef, w in reg:                      # aggregate_losses regularization_loss (:463-466)
      _lib.call('b200rl_l2_sum', _lib.ptr(w), w.numel(), float(coef) / self.replicas,
                _lib.ptr(loss), _lib.stream())
    return loss, (), (), dq, tape, reg
