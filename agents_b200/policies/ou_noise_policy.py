"""OUNoisePolicy (tf_agents/policies/ou_noise_policy.py): the wrapped policy's action plus
Ornstein-Uhlenbeck noise (utils/common.py OUProcess), clipped to the action spec when `clip`.

The OU state x has the unbatched action shape [A] and starts at zeros.  Each `action()` call
advances it once, x <- (1 - ou_damping) x + N(0, ou_stddev), and adds the same x to every row of
the batch; as in the reference the state is never reset at episode boundaries.  A stateful
wrapped policy (a recurrent actor) owns the policy state: its new state is returned as is.  One
b200rl_ou_noise launch per call does both.  The state and the {call, ticket} Philox counter are
device tensors allocated here, so a captured collect step advances them on every replay.
"""
import numpy as np
import torch

from agents_b200 import _lib
from agents_b200.policies import tf_policy
from agents_b200.trajectories import policy_step
from agents_b200.utils import nest

_OU_SEED_TAG = 0x4F555F4E4F495345


class OUNoisePolicy(tf_policy.TFPolicy):
  """Actor policy with Ornstein-Uhlenbeck exploration noise."""

  def __init__(self, wrapped_policy, ou_stddev=1.0, ou_damping=1.0, clip=True, name=None,
               seed=0):
    spec = nest.flatten(wrapped_policy.action_spec)
    for s in spec:
      if not s.dtype.is_floating_point:
        raise ValueError('OU Noise is applicable only to continuous actions.')
    if len(spec) != 1 or len(spec[0].shape) != 1:
      raise NotImplementedError('OUNoisePolicy supports one rank-1 continuous action.')
    super().__init__(wrapped_policy.time_step_spec, wrapped_policy.action_spec,
                     wrapped_policy.policy_state_spec, wrapped_policy.info_spec, name=name)
    self._wrapped_policy = wrapped_policy
    self._ou_stddev, self._ou_damping = float(ou_stddev), float(ou_damping)
    self._clip = clip
    self._seed = (int(seed) ^ _OU_SEED_TAG) & 0xFFFFFFFFFFFFFFFF
    a = int(spec[0].shape[0])
    net = getattr(wrapped_policy, 'actor_network', None)
    device = net.device if net is not None else torch.device('cuda')
    amin = np.broadcast_to(np.asarray(spec[0].minimum, np.float32), (a,)).copy()
    amax = np.broadcast_to(np.asarray(spec[0].maximum, np.float32), (a,)).copy()
    self._amin = torch.as_tensor(amin, device=device)
    self._amax = torch.as_tensor(amax, device=device)
    self._ou_state = torch.zeros(a, dtype=torch.float32, device=device)
    self._ou_rng = torch.zeros(2, dtype=torch.int64, device=device)

  @property
  def wrapped_policy(self):
    return self._wrapped_policy

  @property
  def ou_state(self):
    """The OU process value x [A] after the last `action()` call."""
    return self._ou_state

  def get_initial_state(self, batch_size=None):
    return self._wrapped_policy.get_initial_state(batch_size)

  def variables(self):
    return self._wrapped_policy.variables()

  def _action(self, time_step, policy_state, seed):
    step = self._wrapped_policy.action(time_step, policy_state, seed)
    loc = step.action
    if loc.stride(-1) != 1:
      loc = loc.contiguous()
    n, a = loc.shape
    act = torch.empty((n, a), dtype=torch.float32, device=loc.device)
    _lib.call('b200rl_ou_noise', _lib.dptr(loc), loc.stride(0), n, a, _lib.ptr(self._ou_state),
              self._ou_damping, self._ou_stddev, None, self._seed,
              _lib.ptr(self._ou_rng), _lib.ptr(self._amin) if self._clip else None,
              _lib.ptr(self._amax) if self._clip else None, _lib.ptr(act), a, _lib.stream())
    return policy_step.PolicyStep(act, step.state, step.info)

  def distribution(self, time_step, policy_state=()):
    raise NotImplementedError('Distributions are not implemented yet.')
