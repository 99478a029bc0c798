"""PPOPolicy (tf_agents/agents/ppo/ppo_policy.py:40-): ActorPolicy that also records the
distribution parameters (and optionally the value prediction) in `policy_info`
(ppo_policy.py:156-159), so that PPOAgent.train can recompute the behaviour log-probs.

collect=True  -> actions are sampled from Normal(loc, scale) and clipped to the spec
                 (ActorPolicy clip=True); info = {'dist_params': {'loc', 'scale'}[, 'value_prediction']}.
collect=False -> the greedy policy (mode of the distribution = loc), empty info.
For a discrete action spec the actor emits Categorical logits: collect draws with
b200rl_categorical_sample and records {'dist_params': {'logits'}}; the greedy policy is the
first argmax (b200rl_epsilon_greedy with epsilon 0); `clip` does not apply.
The draws and the mode are ActorPolicy's; PPOPolicy keeps its own seed tag, so its draws do not
change with the extraction.
A recurrent actor (ActorDistributionRnnNetwork) gives the policy a state (ppo_policy.py:163-173):
{'actor_network_state'} and, for a collect policy that records value predictions
(compute_value_and_advantage_in_train=False) with a recurrent value net, 'value_network_state'.
`action` runs one [B, 1] step from that state, starting from zero at FIRST, and returns the new
state.  With feed-forward networks the state is () and nothing changes.
"""
import torch

from agents_b200.policies import actor_policy
from agents_b200.specs import tensor_spec
from agents_b200.trajectories import policy_step

_PPO_SEED_TAG = 0x50504F5F504F4C49


class PPOPolicy(actor_policy.ActorPolicy):

  _SEED_TAG = _PPO_SEED_TAG
  _STATEFUL_ACTOR = True

  def __init__(self, time_step_spec, action_spec, actor_net, value_net,
               observation_normalizer=None, clip=True, collect=True,
               compute_value_and_advantage_in_train=True, seed=0):
    actor_policy.reject_tanh_normal(actor_net, 'PPOPolicy')
    info_spec = ()
    if collect:
      info_spec = {'dist_params': actor_net.dist_params_spec()}
      if not compute_value_and_advantage_in_train:
        info_spec['value_prediction'] = tensor_spec.TensorSpec((), torch.float32,
                                                               'value_prediction')
    state_spec = {}
    if actor_net.state_spec:
      state_spec['actor_network_state'] = actor_net.state_spec
    if collect and value_net.state_spec and not compute_value_and_advantage_in_train:
      state_spec['value_network_state'] = value_net.state_spec
    super().__init__(time_step_spec, action_spec, actor_net, clip=clip, collect=collect,
                     seed=seed, info_spec=info_spec, policy_state_spec=state_spec or ())
    self._value_net = value_net
    self._observation_normalizer = observation_normalizer
    self._value_in_info = collect and not compute_value_and_advantage_in_train

  def get_initial_state(self, batch_size=None):
    if not self._policy_state_spec:
      return ()
    out = {'actor_network_state': self._actor_net.get_initial_state(batch_size)} \
        if self._actor_net.state_spec else {}
    if 'value_network_state' in self._policy_state_spec:
      out['value_network_state'] = self._value_net.get_initial_state(batch_size)
    return out

  def variables(self):
    return self._actor_net.variables + self._value_net.variables

  def _normalized(self, observation):
    if self._observation_normalizer is None:
      return observation
    return self._observation_normalizer.normalize(observation)

  def apply_value_network(self, observations, step_types=None, value_state=None, training=False):
    """Value predictions for `[N, ...]` observations (ppo_policy.py apply_value_network); a
    recurrent value net takes `[B, T, ...]` observations with their step types and returns its
    final state too."""
    if self._value_net.state_spec:
      return self._value_net(self._normalized(observations), step_types, value_state or ())
    v, _ = self._value_net(self._normalized(observations))
    return v, ()

  def _check_state(self, policy_state):
    if not isinstance(policy_state, dict) or set(policy_state) != set(self._policy_state_spec):
      raise ValueError('This PPOPolicy is stateful: pass the policy_state from '
                       'get_initial_state(batch_size) or from the previous action(), with keys '
                       f'{sorted(self._policy_state_spec)}.')

  def distribution_params(self, time_step, policy_state=()):
    """The actor's distribution parameters for `time_step`; with a recurrent actor, from
    `policy_state` (the new state is returned by `action`)."""
    if not self._actor_net.state_spec:
      return super().distribution_params(time_step)
    self._check_state(policy_state)
    params, _ = self._actor_net.distribution_params(
        self._normalized(time_step.observation), time_step.step_type,
        policy_state['actor_network_state'])
    return params

  def _action(self, time_step, policy_state, seed):
    if not self._policy_state_spec:
      return super()._action(time_step, policy_state, seed)
    self._check_state(policy_state)
    obs = self._normalized(time_step.observation)
    new_state = dict(policy_state)
    if self._actor_net.state_spec:
      params, new_state['actor_network_state'] = self._actor_net.distribution_params(
          obs, time_step.step_type, policy_state['actor_network_state'])
    else:
      params = self._actor_net.distribution_params(obs)
    if self._actor_net.discrete:
      act = self._categorical_action(params)
    else:
      act = self._normal_action(*params)
    info = ()
    if self._collect:
      info = {'dist_params': ({'logits': params} if self._actor_net.discrete else
                              {'loc': params[0], 'scale': params[1]})}
      if self._value_in_info:
        if 'value_network_state' in policy_state:
          info['value_prediction'], new_state['value_network_state'] = self._value_net(
              obs, time_step.step_type, policy_state['value_network_state'])
        else:
          info['value_prediction'], _ = self._value_net(obs)
    return policy_step.PolicyStep(act, new_state, info)

  def _info(self, observation, params):
    if not self._collect:
      return ()
    if self._actor_net.discrete:
      info = {'dist_params': {'logits': params}}
    else:
      info = {'dist_params': {'loc': params[0], 'scale': params[1]}}
    if self._value_in_info:
      info['value_prediction'], _ = self._value_net(observation)
    return info
