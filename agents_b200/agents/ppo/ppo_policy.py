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
"""
import torch

from agents_b200.policies import actor_policy
from agents_b200.specs import tensor_spec

_PPO_SEED_TAG = 0x50504F5F504F4C49


class PPOPolicy(actor_policy.ActorPolicy):

  _SEED_TAG = _PPO_SEED_TAG

  def __init__(self, time_step_spec, action_spec, actor_net, value_net,
               observation_normalizer=None, clip=True, collect=True,
               compute_value_and_advantage_in_train=True, seed=0):
    info_spec = ()
    if collect:
      info_spec = {'dist_params': actor_net.dist_params_spec()}
      if not compute_value_and_advantage_in_train:
        info_spec['value_prediction'] = tensor_spec.TensorSpec((), torch.float32,
                                                               'value_prediction')
    super().__init__(time_step_spec, action_spec, actor_net, clip=clip, collect=collect,
                     seed=seed, info_spec=info_spec)
    self._value_net = value_net
    self._observation_normalizer = observation_normalizer
    self._value_in_info = collect and not compute_value_and_advantage_in_train

  def variables(self):
    return self._actor_net.variables + self._value_net.variables

  def _normalized(self, observation):
    if self._observation_normalizer is None:
      return observation
    return self._observation_normalizer.normalize(observation)

  def apply_value_network(self, observations, step_types=None, value_state=None, training=False):
    """Value predictions for `[N, ...]` observations (ppo_policy.py apply_value_network)."""
    v, _ = self._value_net(self._normalized(observations))
    return v, ()

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
