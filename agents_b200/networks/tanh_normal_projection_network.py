"""Actor network with a TanhNormalProjectionNetwork head (SAC).

Reference: networks/actor_distribution_network.py with
`continuous_projection_net=tanh_normal_projection_network.TanhNormalProjectionNetwork`
(examples/sac/haarnoja18/sac_train_eval.py:188-196) and
agents/sac/tanh_normal_projection_network.py:38-143: a Dense(2A) projection
(variance_scaling(0.1)) split into loc and log-std, std = exp(log_std), distribution
SquashToSpecNormal (distributions/utils.py:40-160).  The network output here is the raw
[N, 2A] head; sampling / log-prob / their backward run in csrc/sac.cu.

`TanhNormalProjectionNetwork` is the callable the reference passes as `continuous_projection_net`
to ActorDistributionRnnNetwork (agents/sac/examples/v2/train_eval_rnn.py): it holds the
projection layer, a Keras-default Dense(2A) (glorot_uniform kernel, zero bias, no activation).
"""
import numpy as np
import torch

from agents_b200.networks import actor_distribution_network as adn
from agents_b200.networks import layers as L
from agents_b200.networks import network
from agents_b200.networks import q_network
from agents_b200.utils import nest


class TanhNormalProjectionNetwork(object):
  """The tanh-squashed diagonal Normal head over `sample_spec`: one Dense(2A) layer whose output
  is (loc | log_std), std = exp(log_std).  Only the reference defaults (activation_fn None,
  std_transform exp) are supported: the sampling kernels assume them."""

  def __init__(self, sample_spec, activation_fn=None, std_transform=torch.exp,
               name='TanhNormalProjectionNetwork'):
    if len(nest.flatten(sample_spec)) != 1:
      raise ValueError('Tanh Normal Projection network only supports single spec samples.')
    if activation_fn is not None:
      raise NotImplementedError('TanhNormalProjectionNetwork supports activation_fn=None only.')
    if std_transform is not torch.exp and std_transform is not np.exp:
      raise NotImplementedError('TanhNormalProjectionNetwork supports std_transform=exp only.')
    spec = nest.flatten(sample_spec)[0]
    if len(spec.shape) != 1:
      raise ValueError('TanhNormalProjectionNetwork supports one rank-1 continuous action.')
    self.name = name
    self.sample_spec = spec
    self.num_actions = int(spec.shape[0])
    self.projection_layer = L.Dense(2 * self.num_actions, activation=None)


class TanhNormalActorNetwork(network.Network):

  def __init__(self, input_tensor_spec, output_tensor_spec, fc_layer_params=(256, 256),
               activation_fn='relu', kernel_initializer=None,
               name='ActorDistributionNetwork', device='cuda'):
    super().__init__(input_tensor_spec=input_tensor_spec, state_spec=(), name=name, device=device)
    spec = nest.flatten(output_tensor_spec)
    if len(spec) != 1 or len(spec[0].shape) != 1:
      raise ValueError('TanhNormalActorNetwork supports one rank-1 continuous action.')
    self.num_actions = int(spec[0].shape[0])
    kinit = kernel_initializer or q_network._vs_init
    layers = []
    for units in (fc_layer_params or []):
      layers.append(L.Dense(units, activation=activation_fn, kernel_initializer=kinit))
    layers.append(L.Dense(2 * self.num_actions, activation=None, kernel_initializer=adn._mean_init))
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
