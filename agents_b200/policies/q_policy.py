"""QPolicy: holds the Q network and evaluates it on a TimeStep.

Reference: policies/q_policy.py:150-194 (Q-net logits; an action mask from
`observation_and_action_constraint_splitter` is applied by the selecting policy, which gives
masked actions dtype.min).  The selection itself lives in greedy_policy.py /
epsilon_greedy_policy.py / random_tf_policy.py (one b200rl_epsilon_greedy launch); their classes
are re-exported here because DqnAgent builds `EpsilonGreedyPolicy(QPolicy(...))` from this module.
A recurrent Q network (QRnnNetwork) gives the policy its state: `policy_state_spec` is the
network's `state_spec`, and `q_values` runs one [B, 1] step from that state (zero at FIRST) and
returns the new state.
"""
from agents_b200.policies import tf_policy
from agents_b200.policies.epsilon_greedy_policy import EpsilonGreedyPolicy  # noqa: F401
from agents_b200.policies.greedy_policy import GreedyPolicy
from agents_b200.policies.greedy_policy import _Selecting  # noqa: F401
from agents_b200.policies.random_tf_policy import RandomTFPolicy  # noqa: F401
from agents_b200.utils import nest


class QPolicy(tf_policy.TFPolicy):
  """Holds the Q network; `q_values(time_step, policy_state)` evaluates it
  (q_policy.py:150-194)."""

  def __init__(self, time_step_spec, action_spec, q_network,
               observation_and_action_constraint_splitter=None, emit_log_probability=False,
               name=None):
    super().__init__(time_step_spec, action_spec, policy_state_spec=getattr(q_network, 'state_spec', ()),
                     name=name)
    flat = nest.flatten(action_spec)
    if len(flat) > 1:
      raise ValueError('Only scalar actions are supported now.')
    spec = flat[0]
    self._num_actions = int(spec.maximum - spec.minimum + 1)
    self._action_dtype = spec.dtype
    self._q_network = q_network
    self._splitter = observation_and_action_constraint_splitter

  @property
  def observation_and_action_constraint_splitter(self):
    return self._splitter

  @property
  def num_actions(self):
    return self._num_actions

  def variables(self):
    return self._q_network.variables

  def get_initial_state(self, batch_size=None):
    if not self._policy_state_spec:
      return ()
    return self._q_network.get_initial_state(batch_size)

  def _check_state(self, policy_state):
    if len(nest.flatten(policy_state)) != len(nest.flatten(self._policy_state_spec)):
      raise ValueError('This QPolicy is stateful (its Q network is recurrent): pass the '
                       'policy_state from get_initial_state(batch_size) or from the previous '
                       'action().')

  def q_values(self, time_step, policy_state=()):
    """Returns (q [B, A], action mask or None, new policy_state)."""
    obs, mask = time_step.observation, None
    if self._splitter is not None:
      obs, mask = self._splitter(obs)
    if not self._policy_state_spec:
      q, _ = self._q_network(obs, step_type=time_step.step_type)
      return q, mask, policy_state
    self._check_state(policy_state)
    q, state = self._q_network(obs, step_type=time_step.step_type, network_state=policy_state)
    return q, mask, state

  def _action(self, time_step, policy_state, seed):
    return GreedyPolicy(self)._action(time_step, policy_state, seed)
