"""ValueRnnNetwork (tf_agents/networks/value_rnn_network.py): an LSTMEncodingNetwork
(input_fc (75, 40), lstm_size (40,), output_fc (75, 40)) followed by Dense(1) with
uniform(-0.03, 0.03) kernels; the output is squeezed to [B] or [B, T]."""
from agents_b200.networks import layers as L
from agents_b200.networks import lstm_encoding_network
from agents_b200.networks import q_network


class ValueRnnNetwork(lstm_encoding_network.LSTMEncodingNetwork):

  def __init__(self, input_tensor_spec, preprocessing_layers=None, preprocessing_combiner=None,
               conv_layer_params=None, input_fc_layer_params=(75, 40),
               input_dropout_layer_params=None, lstm_size=(40,), output_fc_layer_params=(75, 40),
               activation_fn='relu', dtype=None, name='ValueRnnNetwork', device='cuda'):
    if input_dropout_layer_params:
      raise NotImplementedError('Dropout layer is not supported.')
    super().__init__(input_tensor_spec, preprocessing_layers=preprocessing_layers,
                     preprocessing_combiner=preprocessing_combiner,
                     conv_layer_params=conv_layer_params,
                     input_fc_layer_params=input_fc_layer_params, lstm_size=lstm_size,
                     output_fc_layer_params=output_fc_layer_params, activation_fn=activation_fn,
                     name=name, device=device)
    self._post.append(L.Dense(1, activation=None, kernel_initializer=q_network._q_head_init))
    self._layers = self._pre + self._cells + self._post

  def __call__(self, observation, step_type=None, network_state=(), training=False):
    out, state = super().__call__(observation, step_type, network_state, training)
    return out.squeeze(-1), state
