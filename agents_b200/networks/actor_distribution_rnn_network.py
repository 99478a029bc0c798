"""ActorDistributionRnnNetwork (tf_agents/networks/actor_distribution_rnn_network.py): an
LSTMEncodingNetwork (input_fc (200, 100), LSTM layers, output_fc (200, 100)) followed by the
Normal or Categorical head of ActorDistributionNetwork.  The Normal head starts its std bias at
log(exp(0.35) - 1), as the reference's `_normal_projection_net` does (:39-49).

`distribution_params(observation, step_type, network_state)` returns (params, new_state) with
params over the B*T rows in batch-major order: (loc, scale) each [B*T, A], or logits [B*T, A].

`continuous_projection_net=tanh_normal_projection_network.TanhNormalProjectionNetwork` (SAC's
recurrent actor, agents/sac/examples/v2/train_eval_rnn.py) puts the tanh-Normal head after the
output stack instead: one Dense(2A), so the variables are input_fc, LSTM, output_fc, projection.
Its params are the raw (loc | log_std) head [B*T, 2A] (`__call__`: [B, T, 2A] or [B, 2A]);
sampling, log-probs and their backward run in csrc/sac.cu (SacPolicy), and `backward` takes
dLoss/dhead [B*T, 2A].
"""
import math

import numpy as np
import torch

from agents_b200.networks import actor_distribution_network as adn
from agents_b200.networks import layers as L
from agents_b200.networks import lstm_encoding_network
from agents_b200.networks import tanh_normal_projection_network
from agents_b200.utils import nest

_INIT_ACTION_STDDEV = 0.35


class ActorDistributionRnnNetwork(lstm_encoding_network.LSTMEncodingNetwork):

  def __init__(self, input_tensor_spec, output_tensor_spec, preprocessing_layers=None,
               preprocessing_combiner=None, conv_layer_params=None,
               input_fc_layer_params=(200, 100), input_dropout_layer_params=None, lstm_size=None,
               output_fc_layer_params=(200, 100), activation_fn='relu', dtype=None,
               continuous_projection_net=None, rnn_construction_fn=None,
               rnn_construction_kwargs=None, name='ActorDistributionRnnNetwork', device='cuda'):
    if input_dropout_layer_params:
      raise NotImplementedError('Dropout layer is not supported.')
    super().__init__(input_tensor_spec, preprocessing_layers=preprocessing_layers,
                     preprocessing_combiner=preprocessing_combiner,
                     conv_layer_params=conv_layer_params,
                     input_fc_layer_params=input_fc_layer_params, lstm_size=lstm_size,
                     output_fc_layer_params=output_fc_layer_params, activation_fn=activation_fn,
                     rnn_construction_fn=rnn_construction_fn,
                     rnn_construction_kwargs=rnn_construction_kwargs, name=name, device=device)
    spec = nest.flatten(output_tensor_spec)
    discrete = [not s.dtype.is_floating_point for s in spec]
    if len(spec) != 1 or (not discrete[0] and len(spec[0].shape) != 1):
      raise ValueError('ActorDistributionRnnNetwork supports one discrete action or one rank-1 '
                       'continuous action.')
    self._action_spec = spec[0]
    self.distribution = adn.CATEGORICAL if discrete[0] else adn.NORMAL
    self.tanh_normal = False
    if continuous_projection_net is not None and not discrete[0]:
      proj = continuous_projection_net(spec[0])
      if not isinstance(proj, tanh_normal_projection_network.TanhNormalProjectionNetwork):
        raise NotImplementedError('ActorDistributionRnnNetwork supports the default Normal head or '
                                  'TanhNormalProjectionNetwork as continuous_projection_net.')
      self.tanh_normal = True
      self.num_actions = proj.num_actions
      self._post.append(proj.projection_layer)
    elif self.discrete:
      self.num_actions = adn._discrete_num_actions(spec[0])
      self._post.append(L.Dense(self.num_actions, activation=None,
                                kernel_initializer=adn._mean_init))
    else:
      self.num_actions = int(spec[0].shape[0])
      self._post.append(L.Dense(self.num_actions, activation=None,
                                kernel_initializer=adn._mean_init))
      self._std = adn.StdBias(self.num_actions,
                              math.log(math.expm1(_INIT_ACTION_STDDEV)))
      self._post.append(self._std)
    if not self.discrete:
      amin = np.broadcast_to(np.asarray(spec[0].minimum, np.float32), (self.num_actions,))
      amax = np.broadcast_to(np.asarray(spec[0].maximum, np.float32), (self.num_actions,))
      self._amin = torch.as_tensor(amin.copy(), device=self._device)
      self._amax = torch.as_tensor(amax.copy(), device=self._device)
    self._layers = self._pre + self._cells + self._post

  discrete = adn.ActorDistributionNetwork.discrete
  dist_params_spec = adn.ActorDistributionNetwork.dist_params_spec
  action_min = adn.ActorDistributionNetwork.action_min
  action_max = adn.ActorDistributionNetwork.action_max

  def _head_params(self, m_raw):
    if self.discrete or self.tanh_normal:
      return m_raw
    return adn.normal_head_fwd(m_raw, self._std.bias, self._amin, self._amax)

  def distribution_params(self, observation, step_type=None, network_state=()):
    """(params over the B*T rows, new_state); no tape."""
    obs, st, B, T, _ = self._sequence(observation, step_type)
    m_raw, state, _ = self._run_seq(obs, st, B, T, network_state)
    return self._head_params(m_raw), state

  def forward_train(self, observation, step_type=None):
    m_raw, tape = super().forward_train(observation, step_type)
    return self._head_params(m_raw), (tape, m_raw)

  def backward(self, ctx, dparams):
    """dparams = (dloc, dscale), each [B*T, A]; dlogits [B*T, A] for a discrete action; dhead
    [B*T, 2A] for the tanh-Normal head."""
    tape, m_raw = ctx
    if self.discrete or self.tanh_normal:
      return super().backward(tape, dparams)
    dm, ds_part = adn.normal_head_bwd(m_raw, self._std.bias, self._amin, self._amax, dparams)
    grads = super().backward(tape, dm)
    adn.reduce_std_grad(ds_part, self._std.d_bias)
    return grads

  def __call__(self, observation, step_type=None, network_state=(), training=False):
    obs, st, B, T, has_time = self._sequence(observation, step_type)
    m_raw, state, _ = self._run_seq(obs, st, B, T, network_state)
    params = self._head_params(m_raw)
    return nest.map_structure(lambda p: self._unflatten(p, B, T, has_time), params), state
