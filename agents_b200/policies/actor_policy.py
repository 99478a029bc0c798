"""ActorPolicy (tf_agents/policies/actor_policy.py): actions from the distribution an
ActorDistributionNetwork emits.

collect=True  -> a draw from the distribution: Normal(loc, scale) through b200rl_normal_sample,
                 clipped to the action spec when `clip` (the reference's clip=True default), or
                 Categorical(logits) through b200rl_categorical_sample (`clip` does not apply).
collect=False -> the greedy policy, the mode of the distribution: loc for a Normal, the first
                 argmax of the logits for a Categorical (b200rl_epsilon_greedy with epsilon 0).
A deterministic network (ActorNetwork, `deterministic = True`) gives its scale_to_spec action,
clamped to the action spec when `clip`; `collect` does not apply.  A recurrent deterministic actor
(ActorRnnNetwork) makes the policy stateful: `policy_state_spec` is the actor's `state_spec`, and
each call runs one [B, 1] step from the given state (the zero state where step_type is FIRST) and
returns the new state.
Draws use a device {call, ticket} counter, so a captured collect step draws fresh values on every
replay.  Subclasses record extra `policy_info` through `_info` (PPOPolicy).
"""
import torch

from agents_b200 import _lib
from agents_b200.policies import tf_policy
from agents_b200.trajectories import policy_step
from agents_b200.utils import nest

_ACTOR_SEED_TAG = 0x4143544F52504F4C


def reject_tanh_normal(actor_network, who):
  """The tanh-Normal recurrent actor emits a raw [N, 2A] head that only SacPolicy samples."""
  if getattr(actor_network, 'tanh_normal', False):
    raise NotImplementedError('{} does not support a tanh-Normal actor (TanhNormalProjection'
                              'Network head); use it with SacAgent / SacPolicy.'.format(who))


class ActorPolicy(tf_policy.TFPolicy):

  _SEED_TAG = _ACTOR_SEED_TAG
  _STATEFUL_ACTOR = False        # subclasses that thread a recurrent actor's state set True

  def __init__(self, time_step_spec, action_spec, actor_network, clip=True, collect=True, seed=0,
               info_spec=(), policy_state_spec=()):
    reject_tanh_normal(actor_network, type(self).__name__)
    self._stateful_deterministic = False
    if getattr(actor_network, 'state_spec', ()) and not self._STATEFUL_ACTOR:
      if not getattr(actor_network, 'deterministic', False):
        raise NotImplementedError('ActorPolicy supports stateless actor networks and recurrent '
                                  'deterministic actors (ActorRnnNetwork) only.')
      self._stateful_deterministic = True
      policy_state_spec = actor_network.state_spec
    super().__init__(time_step_spec, action_spec, policy_state_spec=policy_state_spec,
                     info_spec=info_spec)
    self._actor_net = actor_network
    self._clip, self._collect = clip, collect
    self._seed = (int(seed) ^ self._SEED_TAG) & 0xFFFFFFFFFFFFFFFF
    self._rng = None
    self._action_spec_leaf = nest.flatten(action_spec)[0]

  @property
  def actor_network(self):
    return self._actor_net

  def variables(self):
    return self._actor_net.variables

  def get_initial_state(self, batch_size=None):
    if not self._stateful_deterministic:
      return super().get_initial_state(batch_size)
    return self._actor_net.get_initial_state(batch_size)

  def _normalized(self, observation):
    return observation

  def distribution_params(self, time_step):
    return self._actor_net.distribution_params(self._normalized(time_step.observation))

  def _rng_block(self, device):
    if self._rng is None or self._rng.device != device:
      self._rng = torch.zeros(2, dtype=torch.int64, device=device)
    return self._rng

  def _categorical_action(self, logits):
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
    return act

  def _normal_action(self, loc, scale):
    if not self._collect:
      return loc
    n, a = loc.shape
    act = torch.empty_like(loc)
    _lib.call('b200rl_normal_sample', _lib.ptr(loc), _lib.ptr(scale), a, n, a,
              _lib.ptr(self._actor_net.action_min) if self._clip else None,
              _lib.ptr(self._actor_net.action_max) if self._clip else None, self._seed,
              _lib.ptr(self._rng_block(loc.device)), _lib.ptr(act), _lib.stream())
    return act

  def _info(self, observation, params):
    """policy_info of a step; `params` are the distribution parameters."""
    return ()

  def _action(self, time_step, policy_state, seed):
    obs = self._normalized(time_step.observation)
    if self._stateful_deterministic:
      if len(nest.flatten(policy_state)) != len(nest.flatten(self._policy_state_spec)):
        raise ValueError('This ActorPolicy is stateful (its actor is recurrent): pass the '
                         'policy_state from get_initial_state(batch_size) or from the previous '
                         'action().')
      act, state = self._actor_net.action(obs, time_step.step_type, policy_state, clip=self._clip)
      return policy_step.PolicyStep(act, state, self._info(obs, act))
    if getattr(self._actor_net, 'deterministic', False):
      act = self._actor_net.action(obs, clip=self._clip)
      return policy_step.PolicyStep(act, policy_state, self._info(obs, act))
    params = self._actor_net.distribution_params(obs)
    if self._actor_net.discrete:
      act = self._categorical_action(params)
    else:
      act = self._normal_action(*params)
    return policy_step.PolicyStep(act, policy_state, self._info(obs, params))
