"""ValueNetwork (tf_agents/networks/value_network.py): encoder + Dense(1), output squeezed.

Defaults follow the reference (fc_layer_params=(75, 40), relu); the PPO examples use
(200, 100) tanh (agents/ppo/examples/v2/train_eval_clip_agent.py:101-102).  The value head uses
uniform(-0.03, 0.03) kernels like the reference.  preprocessing_layers / conv_layer_params put a
Conv2D stack and Flatten in front of the dense layers (the Atari-shape PPO nets).
"""
import torch

from agents_b200.networks import actor_distribution_network
from agents_b200.networks import layers as L
from agents_b200.networks import network
from agents_b200.networks import q_network


class ValueNetwork(network.Network):

  def __init__(self, input_tensor_spec, fc_layer_params=(75, 40), activation_fn='relu',
               kernel_initializer=None, name='ValueNetwork', device='cuda',
               preprocessing_layers=None, conv_layer_params=None):
    super().__init__(input_tensor_spec=input_tensor_spec, state_spec=(), name=name, device=device)
    kinit = kernel_initializer or q_network._vs_init
    layers = actor_distribution_network.encoder_layers(
        preprocessing_layers, conv_layer_params, fc_layer_params, activation_fn, kinit)
    layers.append(L.Dense(1, activation=None, kernel_initializer=q_network._q_head_init))
    self._layers = layers

  def __call__(self, observation, step_type=None, network_state=(), training=False):
    out, _ = self._run(observation, keep=False)
    return out.squeeze(-1), network_state
