"""CategoricalQNetwork (tf_agents/networks/categorical_q_network.py:33-144): a QNetwork whose
Dense head has num_actions * num_atoms units (same uniform(-0.03, 0.03) kernel / -0.2 bias
initialisers), read as [B, num_actions, num_atoms] logits.

`net(obs)[0]` is a [B, A, N] view of the head's output; `forward_train` keeps the flat [B, A*N]
tensor, which is what the C51 loss kernel and the backward pass consume (no copy either way).
`preprocessing_layers=CastScale(255.)` gives the Atari example's AtariCategoricalQNetwork
(agents/categorical_dqn/examples/train_eval_atari.py).
"""
import torch

from agents_b200.networks import q_network
from agents_b200.specs import tensor_spec


class CategoricalQNetwork(q_network.QNetwork):

  def __init__(self, input_tensor_spec, action_spec, num_atoms=51, preprocessing_layers=None,
               conv_layer_params=None, fc_layer_params=None, activation_fn='relu',
               name='CategoricalQNetwork', device='cuda'):
    if not isinstance(action_spec, tensor_spec.BoundedTensorSpec):           # :100-103
      raise TypeError('action_spec must be a BoundedTensorSpec. Got: %s' % (action_spec,))
    self._num_actions = int(action_spec.maximum - action_spec.minimum + 1)
    self._num_atoms = int(num_atoms)
    head_spec = tensor_spec.BoundedTensorSpec(                                # :108-110
        (), torch.int32, 0, self._num_actions * self._num_atoms - 1)
    super(CategoricalQNetwork, self).__init__(
        input_tensor_spec, head_spec, preprocessing_layers=preprocessing_layers,
        conv_layer_params=conv_layer_params, fc_layer_params=fc_layer_params,
        activation_fn=activation_fn, name=name, device=device)

  @property
  def num_atoms(self):
    return self._num_atoms

  def create_variables(self, input_tensor_spec=None, **kwargs):
    super(CategoricalQNetwork, self).create_variables(input_tensor_spec, **kwargs)
    return tensor_spec.TensorSpec((self._num_actions, self._num_atoms), torch.float32)

  def __call__(self, observation, step_type=None, network_state=(), training=False):
    logits, network_state = super(CategoricalQNetwork, self).__call__(
        observation, step_type, network_state, training)
    return logits.view(-1, self._num_actions, self._num_atoms), network_state   # :143
