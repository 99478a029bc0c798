"""CategoricalQPolicy (policies/categorical_q_policy.py:38-192): a QPolicy over a categorical
Q-network whose `q_values` are the expected values of the per-action distributions
(common.convert_q_logits_to_values), one b200rl_c51_q_values launch.  GreedyPolicy and
EpsilonGreedyPolicy wrap it unchanged: the mask goes to their selection launch, which gives masked
actions the lowest logit (:184-187 use -inf; both leave only allowed actions as the argmax).
"""
import numpy as np
import torch

from agents_b200 import _lib
from agents_b200.policies import q_policy
from agents_b200.specs import tensor_spec


class CategoricalQPolicy(q_policy.QPolicy):

  def __init__(self, time_step_spec, action_spec, q_network, min_q_value, max_q_value,
               observation_and_action_constraint_splitter=None, name=None):
    if not isinstance(action_spec, tensor_spec.BoundedTensorSpec):            # :97-100
      raise TypeError('action_spec must be a BoundedTensorSpec. Got: %s' % (action_spec,))
    if action_spec.minimum != 0:                                              # :103-110
      raise ValueError('Action specs should have minimum of 0, but saw: {0}.'.format(action_spec))
    try:
      num_atoms = q_network.num_atoms
    except AttributeError:                                                    # :113-120
      raise ValueError('Expected q_network to have property `num_atoms`, but it doesn\'t. '
                       '(Note: you likely want to use a CategoricalQNetwork.) Network is: %s'
                       % q_network)
    super(CategoricalQPolicy, self).__init__(
        time_step_spec, action_spec, q_network,
        observation_and_action_constraint_splitter=observation_and_action_constraint_splitter,
        name=name)
    self._num_atoms = int(num_atoms)
    out = q_network.create_variables()
    if tuple(out.shape) != (self._num_actions, self._num_atoms):              # :123-125
      raise ValueError('Expected q_network to emit a floating point tensor with inner dims {}; '
                       'but saw network output spec: {}'.format(
                           (self._num_actions, self._num_atoms), out))
    # np.linspace in float32, as the reference builds it (:141-144)
    self._support = torch.as_tensor(
        np.linspace(min_q_value, max_q_value, self._num_atoms, dtype=np.float32),
        device=q_network.device)

  @property
  def support(self):
    return self._support

  def q_values(self, time_step, policy_state=()):
    obs, mask = time_step.observation, None
    if self._splitter is not None:
      obs, mask = self._splitter(obs)
    logits, _ = self._q_network(obs, step_type=time_step.step_type)
    logits = logits.contiguous()
    b = logits.shape[0]
    q = torch.empty((b, self._num_actions), dtype=torch.float32, device=logits.device)
    _lib.call('b200rl_c51_q_values', _lib.ptr(logits), _lib.ptr(self._support), b,
              self._num_actions, self._num_atoms, _lib.ptr(q), _lib.stream())
    return q, mask, policy_state
