"""Deterministic ActorNetwork (tf_agents/agents/ddpg/actor_network.py), the actor of TD3.

fc layers (ReLU) -> Dense(A, tanh) -> `common.scale_to_spec`: action = means + magnitudes * y with
means / magnitudes the centre / half-width of the bounded action spec.  Kernels default to
VarianceScaling(1/3, fan_in, uniform) for the hidden layers and U(-0.003, 0.003) for the action
layer; biases start at zero.  The layer stack ends at the tanh output y; scale_to_spec (with TD3's
optional target-policy noise and the clamp of a clipping policy) runs in csrc/td3.cu.
"""
import math

import numpy as np
import torch

from agents_b200 import _lib
from agents_b200.networks import layers as L
from agents_b200.networks import network
from agents_b200.utils import nest


def _hidden_init(shape, fan_in, generator):
  """VarianceScaling(scale=1/3, mode='fan_in', distribution='uniform')."""
  limit = math.sqrt(3.0 * (1.0 / 3.0) / max(1.0, fan_in))
  return (torch.rand(shape, dtype=torch.float32, generator=generator) * 2 - 1) * limit


def _last_init(shape, fan_in, generator):
  """RandomUniform(-0.003, 0.003)."""
  return (torch.rand(shape, dtype=torch.float32, generator=generator) * 2 - 1) * 0.003


class ActorNetwork(network.Network):
  """Maps an observation to one bounded continuous action."""

  deterministic = True

  def __init__(self, input_tensor_spec, output_tensor_spec, fc_layer_params=None,
               activation_fn='relu', kernel_initializer=None, last_kernel_initializer=None,
               name='ActorNetwork', device='cuda'):
    if len(nest.flatten(input_tensor_spec)) > 1:
      raise ValueError('Only a single observation is supported by this network')
    spec = nest.flatten(output_tensor_spec)
    if len(spec) > 1:
      raise ValueError('Only a single action is supported by this network')
    if not spec[0].dtype.is_floating_point:
      raise ValueError('Only float actions are supported by this network.')
    if len(spec[0].shape) != 1:
      raise ValueError('ActorNetwork here supports one rank-1 continuous action.')
    super().__init__(input_tensor_spec=input_tensor_spec, state_spec=(), name=name, device=device)
    self.num_actions = int(spec[0].shape[0])
    kinit = kernel_initializer or _hidden_init
    layers = [L.Dense(units, activation=activation_fn, kernel_initializer=kinit)
              for units in (fc_layer_params or [])]
    layers.append(L.Dense(self.num_actions, activation='tanh',
                          kernel_initializer=last_kernel_initializer or _last_init))
    self._layers = layers
    amin = np.broadcast_to(np.asarray(spec[0].minimum, np.float32), (self.num_actions,)).copy()
    amax = np.broadcast_to(np.asarray(spec[0].maximum, np.float32), (self.num_actions,)).copy()
    self._amin = torch.as_tensor(amin, device=self._device)
    self._amax = torch.as_tensor(amax, device=self._device)

  @property
  def action_min(self):
    return self._amin

  @property
  def action_max(self):
    return self._amax

  def tanh_output(self, observation):
    """The action layer's output y [N, A] in [-1, 1], before scale_to_spec; no tape."""
    return self._run(observation, keep=False)[0]

  def scale_to_spec(self, y, out=None, clip=False, noise_std=0.0, noise_clip=0.0, noise=None,
                    seed=0, rng=None):
    """means + magnitudes * y (+ clip(noise_std * z, +-noise_clip)), clamped to the spec when
    `clip`.  `out` may be a strided [N, A] view (the action columns of a critic input) and may
    alias `y`; z is `noise` [N, A] when given, else drawn on the device with `seed` and the
    {call, ticket} counter `rng`."""
    n = y.shape[0]
    if out is None:
      out = torch.empty((n, self.num_actions), dtype=torch.float32, device=y.device)
    if noise is not None:
      noise = torch.as_tensor(noise, dtype=torch.float32, device=y.device).contiguous()
    _lib.call('b200rl_td3_scale_to_spec', _lib.dptr(y), y.stride(0), n, self.num_actions,
              _lib.ptr(self._amin), _lib.ptr(self._amax), float(noise_std), float(noise_clip),
              _lib.ptr(noise), seed, _lib.ptr(rng), int(clip), _lib.dptr(out), out.stride(0),
              _lib.stream())
    return out

  def action(self, observation, clip=False):
    return self.scale_to_spec(self.tanh_output(observation), clip=clip)

  def __call__(self, observation, step_type=None, network_state=(), training=False):
    return self.action(observation), network_state
