"""PPOPolicy (tf_agents/agents/ppo/ppo_policy.py:40-): ActorPolicy that also records the
distribution parameters (and optionally the value prediction) in `policy_info`
(ppo_policy.py:156-159), so that PPOAgent.train can recompute the behaviour log-probs.

collect=True  -> actions are sampled from Normal(loc, scale) and clipped to the spec
                 (ActorPolicy clip=True); info = {'dist_params': {'loc', 'scale'}[, 'value_prediction']}.
collect=False -> the greedy policy (mode of the distribution = loc), empty info.
For a discrete action spec the actor emits Categorical logits: collect draws with
b200rl_categorical_sample and records {'dist_params': {'logits'}}; the greedy policy is the
first argmax (b200rl_epsilon_greedy with epsilon 0); `clip` does not apply.
"""
import torch

from agents_b200 import _lib
from agents_b200.policies import tf_policy
from agents_b200.specs import tensor_spec
from agents_b200.trajectories import policy_step
from agents_b200.utils import nest

_PPO_SEED_TAG = 0x50504F5F504F4C49


class PPOPolicy(tf_policy.TFPolicy):

  def __init__(self, time_step_spec, action_spec, actor_net, value_net,
               observation_normalizer=None, clip=True, collect=True,
               compute_value_and_advantage_in_train=True, seed=0):
    spec = nest.flatten(action_spec)[0]
    info_spec = ()
    if collect:
      info_spec = {'dist_params': actor_net.dist_params_spec()}
      if not compute_value_and_advantage_in_train:
        info_spec['value_prediction'] = tensor_spec.TensorSpec((), torch.float32,
                                                               'value_prediction')
    super().__init__(time_step_spec, action_spec, info_spec=info_spec)
    self._actor_net, self._value_net = actor_net, value_net
    self._observation_normalizer = observation_normalizer
    self._clip, self._collect = clip, collect
    self._value_in_info = collect and not compute_value_and_advantage_in_train
    self._seed = (int(seed) ^ _PPO_SEED_TAG) & 0xFFFFFFFFFFFFFFFF
    self._rng = None
    self._action_spec_leaf = spec

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

  def distribution_params(self, time_step):
    return self._actor_net.distribution_params(self._normalized(time_step.observation))

  def _rng_block(self, device):
    if self._rng is None or self._rng.device != device:
      self._rng = torch.zeros(2, dtype=torch.int64, device=device)
    return self._rng

  def _categorical_action(self, obs, policy_state):
    logits = self._actor_net.distribution_params(obs)
    n, a = logits.shape
    act = torch.empty(n, dtype=torch.int32, device=logits.device)
    if self._collect:
      _lib.call('b200rl_categorical_sample', _lib.ptr(logits), a, n, a, self._seed,
                _lib.ptr(self._rng_block(logits.device)), _lib.ptr(act), _lib.stream())
    else:       # mode of the Categorical: the first argmax (epsilon 0 never picks at random)
      _lib.call('b200rl_epsilon_greedy', _lib.ptr(logits), None, n, a, 0.0, self._seed,
                _lib.ptr(self._rng_block(logits.device)), None, None, _lib.ptr(act),
                _lib.stream())
    spec = self._action_spec_leaf
    act = act.reshape((n,) + tuple(spec.shape))
    if spec.dtype != torch.int32:
      act = act.to(spec.dtype)
    info = ()
    if self._collect:
      info = {'dist_params': {'logits': logits}}
      if self._value_in_info:
        info['value_prediction'], _ = self._value_net(obs)
    return policy_step.PolicyStep(act, policy_state, info)

  def _action(self, time_step, policy_state, seed):
    obs = self._normalized(time_step.observation)
    if self._actor_net.discrete:
      return self._categorical_action(obs, policy_state)
    loc, scale = self._actor_net.distribution_params(obs)
    if not self._collect:
      return policy_step.PolicyStep(loc, policy_state, ())
    n, a = loc.shape
    if self._rng is None or self._rng.device != loc.device:
      self._rng = torch.zeros(2, dtype=torch.int64, device=loc.device)
    act = torch.empty_like(loc)
    _lib.call('b200rl_normal_sample', _lib.ptr(loc), _lib.ptr(scale), a, n, a,
              _lib.ptr(self._actor_net.action_min) if self._clip else None,
              _lib.ptr(self._actor_net.action_max) if self._clip else None, self._seed,
              _lib.ptr(self._rng), _lib.ptr(act), _lib.stream())
    info = {'dist_params': {'loc': loc, 'scale': scale}}
    if self._value_in_info:
      info['value_prediction'], _ = self._value_net(obs)
    return policy_step.PolicyStep(act, policy_state, info)
