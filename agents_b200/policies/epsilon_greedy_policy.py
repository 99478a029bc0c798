"""EpsilonGreedyPolicy: where(u >= epsilon, greedy action, uniform random allowed action).

Reference: policies/epsilon_greedy_policy.py:120-145 (`u ~ U[0, 1)` per batch row, the random
branch is `RandomTFPolicy` over the same action mask).  Device work: one b200rl_epsilon_greedy
launch (greedy_policy._Selecting).  `epsilon` may be a float or a callable evaluated on the host at
every call (:93-99).  With a recurrent Q network the returned state is the greedy branch's new
state on every row, including the rows that take the random action (the reference returns
`greedy_action.state`).

For a bounded float action spec (QtOptAgent's collect policy over CEMPolicy) the wrapped policy's
action is taken and, per row with probability epsilon, replaced by a uniform draw in
[minimum, maximum) (one b200rl_epsilon_uniform launch, greedy_policy._FloatUniform).
"""
import warnings

import torch

from agents_b200.policies.greedy_policy import _FloatUniform
from agents_b200.policies.greedy_policy import _Selecting
from agents_b200.trajectories import policy_step
from agents_b200.utils import nest


class EpsilonGreedyPolicy(_Selecting):
  """where(u >= epsilon, greedy, uniform random) (epsilon_greedy_policy.py:120-145)."""

  def __init__(self, policy, epsilon, seed=0, name=None):
    super().__init__(policy.time_step_spec, policy.action_spec, seed=seed, name=name,
                     policy_state_spec=policy.policy_state_spec)
    self._wrapped_policy = policy
    self._epsilon = epsilon
    self._warned_capture = False
    self._float = None
    spec = nest.flatten(policy.action_spec)[0]
    if spec.dtype.is_floating_point:
      net = getattr(policy, 'q_network', None)
      self._float = _FloatUniform(spec, self._seed,
                                  net.device if net is not None else torch.device('cuda'))
      self._uniform_rng = self._float.rng

  @property
  def wrapped_policy(self):
    return self._wrapped_policy

  def variables(self):
    return self._wrapped_policy.variables()

  def get_initial_state(self, batch_size=None):
    return self._wrapped_policy.get_initial_state(batch_size)

  def _get_epsilon(self):
    if not callable(self._epsilon):
      return self._epsilon
    if (not self._warned_capture and torch.cuda.is_available() and
        torch.cuda.is_current_stream_capturing()):
      # the launch takes epsilon BY VALUE: inside common.function (a CUDA graph) the value seen
      # at capture time is replayed, unlike a tf.Variable read inside a tf.function
      warnings.warn('EpsilonGreedyPolicy: a callable epsilon is evaluated once when the collect '
                    'step is captured by common.function; call the policy outside the captured '
                    'function (or re-capture) to follow an epsilon schedule.')
      self._warned_capture = True
    return self._epsilon()

  def _action(self, time_step, policy_state, seed):
    if self._float is not None:
      step = self._wrapped_policy.action(time_step, policy_state, seed)
      act = self._float.apply(step.action.float().clone(), self._get_epsilon())
      return policy_step.PolicyStep(act, step.state, step.info)
    q, mask, state = self._wrapped_policy.q_values(time_step, policy_state)
    act = self._select(q, mask, self._get_epsilon(), self._wrapped_policy._action_dtype)
    return policy_step.PolicyStep(act, state, ())
