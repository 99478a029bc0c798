"""GaussianPolicy (tf_agents/policies/gaussian_policy.py): the wrapped policy's action plus
N(0, scale) noise, clipped to the action spec when `clip`.

One b200rl_normal_sample launch with loc = the wrapped action and a cached [N, A] scale tensor:
clip(loc + scale * z), z drawn on the device with a {call, ticket} counter, so a captured collect
step draws fresh noise on every replay.
"""
import numpy as np
import torch

from agents_b200 import _lib
from agents_b200.policies import tf_policy
from agents_b200.trajectories import policy_step
from agents_b200.utils import nest

_GAUSSIAN_SEED_TAG = 0x47415553535F504F


class GaussianPolicy(tf_policy.TFPolicy):

  def __init__(self, wrapped_policy, scale=1.0, clip=True, name=None, seed=0):
    spec = nest.flatten(wrapped_policy.action_spec)
    if len(spec) != 1 or not spec[0].dtype.is_floating_point or len(spec[0].shape) != 1:
      raise ValueError('GaussianPolicy supports one rank-1 continuous action.')
    super().__init__(wrapped_policy.time_step_spec, wrapped_policy.action_spec,
                     wrapped_policy.policy_state_spec, wrapped_policy.info_spec, name=name)
    self._wrapped_policy = wrapped_policy
    self._scale = float(scale)
    self._clip = clip
    self._seed = (int(seed) ^ _GAUSSIAN_SEED_TAG) & 0xFFFFFFFFFFFFFFFF
    a = int(spec[0].shape[0])
    self._amin = np.broadcast_to(np.asarray(spec[0].minimum, np.float32), (a,)).copy()
    self._amax = np.broadcast_to(np.asarray(spec[0].maximum, np.float32), (a,)).copy()
    self._bounds = None
    self._scale_t = None
    self._rng = None

  @property
  def wrapped_policy(self):
    return self._wrapped_policy

  def variables(self):
    return self._wrapped_policy.variables()

  def _buffers(self, n, a, device):
    if self._rng is None or self._rng.device != device:
      self._rng = torch.zeros(2, dtype=torch.int64, device=device)
      self._bounds = (torch.as_tensor(self._amin, device=device),
                      torch.as_tensor(self._amax, device=device))
    if self._scale_t is None or self._scale_t.shape != (n, a) or self._scale_t.device != device:
      self._scale_t = torch.full((n, a), self._scale, dtype=torch.float32, device=device)
    return self._scale_t, self._bounds, self._rng

  def _action(self, time_step, policy_state, seed):
    step = self._wrapped_policy.action(time_step, policy_state, seed)
    loc = step.action.contiguous()
    n, a = loc.shape
    scale, (amin, amax), rng = self._buffers(n, a, loc.device)
    act = torch.empty_like(loc)
    _lib.call('b200rl_normal_sample', _lib.ptr(loc), _lib.ptr(scale), a, n, a,
              _lib.ptr(amin) if self._clip else None, _lib.ptr(amax) if self._clip else None,
              self._seed, _lib.ptr(rng), _lib.ptr(act), _lib.stream())
    return policy_step.PolicyStep(act, step.state, step.info)
