"""QRnnNetwork (tf_agents/networks/q_rnn_network.py): an LSTMEncodingNetwork (input_fc (75, 40),
lstm_size, output_fc (75, 40)) followed by Dense(num_actions) with uniform(-0.03, 0.03) kernels and
a -0.2 bias.  Outputs Q values [B, A] for one step or [B, T, A] for a sequence, and the new state."""
from agents_b200.networks import layers as L
from agents_b200.networks import lstm_encoding_network
from agents_b200.networks import q_network
from agents_b200.utils import nest


class QRnnNetwork(lstm_encoding_network.LSTMEncodingNetwork):

  def __init__(self, input_tensor_spec, action_spec, preprocessing_layers=None,
               preprocessing_combiner=None, conv_layer_params=None,
               input_fc_layer_params=(75, 40), lstm_size=None, output_fc_layer_params=(75, 40),
               activation_fn='relu', rnn_construction_fn=None, rnn_construction_kwargs=None,
               dtype=None, name='QRnnNetwork', device='cuda'):
    q_network.validate_specs(action_spec, input_tensor_spec)
    action_spec = nest.flatten(action_spec)[0]
    num_actions = int(action_spec.maximum - action_spec.minimum + 1)
    super().__init__(input_tensor_spec, preprocessing_layers=preprocessing_layers,
                     preprocessing_combiner=preprocessing_combiner,
                     conv_layer_params=conv_layer_params,
                     input_fc_layer_params=input_fc_layer_params, lstm_size=lstm_size,
                     output_fc_layer_params=output_fc_layer_params, activation_fn=activation_fn,
                     rnn_construction_fn=rnn_construction_fn,
                     rnn_construction_kwargs=rnn_construction_kwargs, name=name, device=device)
    self._post.append(L.Dense(num_actions, activation=None,
                              kernel_initializer=q_network._q_head_init, bias_initializer=-0.2))
    self._layers = self._pre + self._cells + self._post
