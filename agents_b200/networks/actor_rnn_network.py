"""ActorRnnNetwork (tf_agents/agents/ddpg/actor_rnn_network.py): the recurrent deterministic actor
of DDPG.

input encoder (optional Conv2D stack, input_fc (200, 100), glorot_uniform kernels, activation_fn)
-> LSTM layers (lstm_size (40,)) -> output_fc (200, 100) (always ReLU, VarianceScaling(2.0,
fan_in, truncated normal), the `mlp_layers` default) -> Dense(A, tanh) with U(-0.003, 0.003)
kernels -> `common.scale_to_spec`.  It is an LSTMEncodingNetwork whose output stack ends at the tanh
output y; scale_to_spec runs in csrc/td3.cu as for ActorNetwork.

The state is the reference's list nest, `list(cell.state_size)`: [h, c] for one LSTM layer (both
specs named 'network_state_spec') and a list of [h, c] per layer when stacked.
"""
import numpy as np
import torch

from agents_b200.networks import actor_distribution_network
from agents_b200.networks import actor_network
from agents_b200.networks import layers as L
from agents_b200.networks import lstm_encoding_network
from agents_b200.networks import q_network
from agents_b200.specs import tensor_spec
from agents_b200.utils import nest


def _list_state(finals):
  """[h, c] per layer; the bare [h, c] for one layer."""
  layers = [list(f) for f in finals]
  return layers[0] if len(layers) == 1 else layers


class ActorRnnNetwork(lstm_encoding_network.LSTMEncodingNetwork):
  """Maps an observation sequence to one bounded continuous action per step."""

  deterministic = True

  def __init__(self, input_tensor_spec, output_tensor_spec, conv_layer_params=None,
               input_fc_layer_params=(200, 100), lstm_size=(40,),
               output_fc_layer_params=(200, 100), activation_fn='relu', name='ActorRnnNetwork',
               device='cuda'):
    if len(nest.flatten(input_tensor_spec)) > 1:
      raise ValueError('Only a single observation is supported by this network')
    spec = nest.flatten(output_tensor_spec)
    if len(spec) != 1 or not spec[0].dtype.is_floating_point or len(spec[0].shape) != 1:
      raise NotImplementedError('ActorRnnNetwork here supports one rank-1 continuous action.')
    super().__init__(input_tensor_spec, conv_layer_params=conv_layer_params,
                     input_fc_layer_params=None, lstm_size=lstm_size,
                     output_fc_layer_params=None, name=name, device=device)
    self._state_spec = self._spec_nest(lstm_size)
    self._pre = actor_distribution_network.encoder_layers(
        None, conv_layer_params, input_fc_layer_params, activation_fn, None)   # glorot_uniform
    self.num_actions = int(spec[0].shape[0])
    self._post = [L.Dense(n, activation='relu', kernel_initializer=q_network._vs_init)
                  for n in (output_fc_layer_params or ())]
    self._post.append(L.Dense(self.num_actions, activation='tanh',
                              kernel_initializer=actor_network._last_init))
    self._layers = self._pre + self._cells + self._post
    amin = np.broadcast_to(np.asarray(spec[0].minimum, np.float32), (self.num_actions,)).copy()
    amax = np.broadcast_to(np.asarray(spec[0].maximum, np.float32), (self.num_actions,)).copy()
    self._amin = torch.as_tensor(amin, device=self._device)
    self._amax = torch.as_tensor(amax, device=self._device)

  @staticmethod
  def _spec_nest(lstm_size):
    def cell(n):
      return [tensor_spec.TensorSpec((n,), torch.float32, 'network_state_spec')] * 2
    return cell(lstm_size[0]) if len(lstm_size) == 1 else [cell(n) for n in lstm_size]

  action_min = actor_network.ActorNetwork.action_min
  action_max = actor_network.ActorNetwork.action_max
  scale_to_spec = actor_network.ActorNetwork.scale_to_spec

  def _pack_state(self, finals):
    return _list_state(finals)

  def tanh_output(self, observation, step_type=None, network_state=()):
    """(y [B*T, A] in [-1, 1] over the B*T rows in batch-major order, new_state); no tape."""
    obs, st, B, T, _ = self._sequence(observation, step_type)
    y, state, _ = self._run_seq(obs, st, B, T, network_state)
    return y, state

  def action(self, observation, step_type=None, network_state=(), clip=False):
    """(scale_to_spec action with the outer shape of `observation`, new_state)."""
    obs, st, B, T, has_time = self._sequence(observation, step_type)
    y, state, _ = self._run_seq(obs, st, B, T, network_state)
    return self._unflatten(self.scale_to_spec(y, clip=clip), B, T, has_time), state

  def __call__(self, observation, step_type=None, network_state=(), training=False):
    return self.action(observation, step_type, network_state)
