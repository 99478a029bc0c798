"""RandomTFPolicy: uniform random discrete actions, optionally restricted by an action mask.

Reference: policies/random_tf_policy.py:80-161 (masked case: sample among the allowed actions,
:104-131; unmasked: `tensor_spec.sample_spec_nest`, :137).  Device work: the shared
b200rl_epsilon_greedy launch with epsilon = 2 (always the random branch) over zero Q values.
A bounded float spec of rank 0 or 1 draws uniform actions in [minimum, maximum) instead
(b200rl_epsilon_uniform with epsilon = 2, greedy_policy._FloatUniform).
"""
import torch

from agents_b200.policies.greedy_policy import _FloatUniform
from agents_b200.policies.greedy_policy import _Selecting
from agents_b200.trajectories import policy_step
from agents_b200.utils import nest


class RandomTFPolicy(_Selecting):
  """Uniform random discrete actions (random_tf_policy.py:137)."""

  def __init__(self, time_step_spec, action_spec, seed=0,
               observation_and_action_constraint_splitter=None, name=None):
    super().__init__(time_step_spec, action_spec, seed=seed, name=name)
    spec = nest.flatten(action_spec)[0]
    self._float = None
    if spec.dtype.is_floating_point:
      if observation_and_action_constraint_splitter is not None:
        raise NotImplementedError('Action masks apply to discrete actions only.')
      self._float = _FloatUniform(spec, self._seed, torch.device('cuda'))
      self._uniform_rng = self._float.rng
      self._float_shape = tuple(spec.shape)
      return
    self._num_actions = int(spec.maximum - spec.minimum + 1)
    self._action_dtype = spec.dtype
    self._splitter = observation_and_action_constraint_splitter
    self._zeros = None

  def _action(self, time_step, policy_state, seed):
    b = time_step.step_type.shape[0]
    dev = time_step.step_type.device
    if self._float is not None:
      act = torch.empty((b,) + self._float_shape, dtype=torch.float32, device=dev)
      return policy_step.PolicyStep(self._float.apply(act, 2.0), policy_state, ())
    mask = None
    if self._splitter is not None:
      _, mask = self._splitter(time_step.observation)
    if self._zeros is None or self._zeros.shape[0] != b or self._zeros.device != dev:
      self._zeros = torch.zeros((b, self._num_actions), dtype=torch.float32, device=dev)
    act = self._select(self._zeros, mask, 2.0, self._action_dtype)
    return policy_step.PolicyStep(act, policy_state, ())
