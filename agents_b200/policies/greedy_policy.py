"""GreedyPolicy and the action-selection launch shared by the discrete policies.

Reference: policies/greedy_policy.py:70-89 (the mode of a Categorical over the Q values == the
first argmax; masked actions get dtype.min logits, q_policy.py:174-183).  `_Selecting._select` is
the ONE launch (b200rl_epsilon_greedy, csrc/env.cu) behind GreedyPolicy (epsilon = -1: never
random), EpsilonGreedyPolicy (epsilon_greedy_policy.py) and RandomTFPolicy (epsilon = 2: always
random, random_tf_policy.py): Philox draw, masked argmax and masked uniform choice per batch row.
"""
import numpy as np
import torch

from agents_b200 import _lib
from agents_b200.policies import tf_policy
from agents_b200.trajectories import policy_step
from agents_b200.utils import nest

_POLICY_SEED_TAG = 0x9E3779B97F4A7C15


class _Selecting(tf_policy.TFPolicy):
  """Shared launch of b200rl_epsilon_greedy for the three selection policies."""

  def __init__(self, time_step_spec, action_spec, seed=0, name=None, policy_state_spec=()):
    super().__init__(time_step_spec, action_spec, policy_state_spec=policy_state_spec, name=name)
    self._seed = (int(seed) ^ _POLICY_SEED_TAG) & 0xFFFFFFFFFFFFFFFF
    self._rng = None

  def _select(self, q, mask, eps, dtype):
    b, a = q.shape
    if self._rng is None or self._rng.device != q.device:
      self._rng = torch.zeros(2, dtype=torch.int64, device=q.device)
    out = torch.empty(b, dtype=torch.int32, device=q.device)
    if mask is not None:
      mask = mask.to(torch.int32).contiguous()
    _lib.call('b200rl_epsilon_greedy', _lib.ptr(q.contiguous()), _lib.ptr(mask), b, a,
              float(eps), self._seed, _lib.ptr(self._rng), None, None, _lib.ptr(out),
              _lib.stream())
    # column j of q is action minimum + j (the reference's ShiftedCategorical)
    spec = nest.flatten(self.action_spec)[0]
    minimum = int(np.asarray(getattr(spec, 'minimum', 0)).reshape(-1)[0])
    if minimum != 0:
      out += minimum
    return out if dtype == torch.int32 else out.to(dtype)


class _FloatUniform(object):
  """The float-spec branch shared by EpsilonGreedyPolicy and RandomTFPolicy: one
  b200rl_epsilon_uniform launch replaces a row, with probability epsilon, by a uniform draw in
  [minimum, maximum) of a bounded float spec of rank 0 or 1 (tensor_spec.sample_spec_nest).  The
  Philox counter is a device tensor allocated here, so a captured collect step draws fresh values
  on every replay."""

  def __init__(self, spec, seed, device):
    a = int(np.prod(spec.shape)) if len(spec.shape) else 1
    if len(spec.shape) > 1:
      raise NotImplementedError('Float actions of rank > 1 are not supported.')
    self.num_actions = a
    self.amin = torch.as_tensor(np.broadcast_to(np.asarray(spec.minimum, np.float32), (a,)).copy(),
                                device=device)
    self.amax = torch.as_tensor(np.broadcast_to(np.asarray(spec.maximum, np.float32), (a,)).copy(),
                                device=device)
    self.seed = seed
    self.rng = torch.zeros(2, dtype=torch.int64, device=device)

  def apply(self, action, eps):
    """Overwrites rows of `action` ([N, A], or [N] for a scalar spec) in place."""
    n = action.shape[0]
    _lib.call('b200rl_epsilon_uniform', _lib.ptr(action), self.num_actions, n, self.num_actions,
              float(eps), _lib.ptr(self.amin), _lib.ptr(self.amax), self.seed,
              _lib.ptr(self.rng), _lib.stream())
    return action


class GreedyPolicy(_Selecting):
  """argmax_a Q(s,a) (greedy_policy.py:70-89).  The state is the wrapped QPolicy's."""

  def __init__(self, policy, name=None):
    super().__init__(policy.time_step_spec, policy.action_spec, name=name,
                     policy_state_spec=policy.policy_state_spec)
    self._wrapped_policy = policy

  @property
  def wrapped_policy(self):
    return self._wrapped_policy

  def variables(self):
    return self._wrapped_policy.variables()

  def get_initial_state(self, batch_size=None):
    return self._wrapped_policy.get_initial_state(batch_size)

  def _action(self, time_step, policy_state, seed):
    q, mask, state = self._wrapped_policy.q_values(time_step, policy_state)
    act = self._select(q, mask, -1.0, self._wrapped_policy._action_dtype)
    return policy_step.PolicyStep(act, state, ())
