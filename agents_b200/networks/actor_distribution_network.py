"""ActorDistributionNetwork: encoder + a NormalProjectionNetwork head for continuous actions or a
CategoricalProjectionNetwork head for discrete ones.

Reference: networks/actor_distribution_network.py (encoder, default fc_layer_params (200, 100);
the head follows the action spec, :34-38,157-158).
Continuous (networks/normal_projection_network.py): means = Dense(A, variance_scaling(0.1)),
squashed to the action spec with tanh (`tanh_squash_to_spec`); standard deviations are a
state-independent bias passed through softplus (std_bias_initializer_value=0.0).  The head
transform and its backward run in csrc/ppo.cu (b200rl_normal_proj_fwd/bwd).
Discrete (networks/categorical_projection_network.py:88-95): logits = Dense(A,
variance_scaling(0.1), zero bias) with A = maximum + 1; the logits are the distribution
parameters and their gradient goes straight into the layer stack.
The optional preprocessing_layers / conv_layer_params build a Conv2D stack and Flatten in front
of the dense layers, as in QNetwork (encoding_network.py:240-300).
"""
import numpy as np
import torch

from agents_b200 import _lib
from agents_b200.networks import layers as L
from agents_b200.networks import network
from agents_b200.utils import nest
from agents_b200.utils import workspace


def _mean_init(shape, fan_in, generator):
  return L.variance_scaling(shape, fan_in, 0.1, generator)


class StdBias(L.Layer):
  """The BiasLayer of NormalProjectionNetwork: a trainable [A] vector; identity in the chain."""
  has_params = True

  def __init__(self, num_actions, init_value=0.0):
    self.num_actions = num_actions
    self.init_value = float(init_value)
    self.l2 = 0.0

  def build(self, input_shape):
    return tuple(input_shape)

  def param_shapes(self):
    return [(self.num_actions,)]

  def bind(self, params, grads):
    self.bias, self.d_bias = params[0], grads[0]

  def init_params(self, generator):
    self.bias.fill_(self.init_value)

  def forward(self, x):
    return x

  def backward(self, x, y, dy, need_dx):
    return dy


NORMAL = 'normal'
CATEGORICAL = 'categorical'


def _discrete_num_actions(spec):
  """Number of categories of a discrete action spec; rejects what the Categorical head cannot
  represent (the reference's CategoricalProjectionNetwork needs one scalar action from 0)."""
  if spec.shape not in ((), (1,)):
    raise ValueError('ActorDistributionNetwork supports a discrete action of shape () or (1,), '
                     f'got shape {spec.shape}.')
  if not hasattr(spec, 'minimum') or not hasattr(spec, 'maximum'):
    raise ValueError('A discrete action needs a BoundedTensorSpec (its maximum gives the number '
                     'of categories).')
  lo = np.asarray(spec.minimum)
  hi = np.asarray(spec.maximum)
  if lo.size != 1 or hi.size != 1:
    raise ValueError('A discrete action needs scalar minimum and maximum bounds.')
  if int(lo.reshape(())) != 0:
    raise ValueError('A discrete action spec must have minimum == 0 (the logits index the '
                     f'actions), got minimum {int(lo.reshape(()))}.')
  return int(hi.reshape(())) + 1


def encoder_layers(preprocessing_layers, conv_layer_params, fc_layer_params, activation_fn, kinit):
  """[preprocessing] + Conv2D stack + Flatten + Dense stack (the Flatten only with a conv or
  preprocessing front, so an MLP encoder stays a plain Dense stack)."""
  layers = []
  if preprocessing_layers is not None:
    layers.append(preprocessing_layers)
  for (filters, kernel_size, strides) in (conv_layer_params or []):
    layers.append(L.Conv2D(filters, kernel_size, strides, activation=activation_fn,
                           kernel_initializer=kinit))
  if layers:
    layers.append(L.Flatten())
  for units in (fc_layer_params or []):
    layers.append(L.Dense(units, activation=activation_fn, kernel_initializer=kinit))
  return layers


def normal_head_fwd(m_raw, std_bias, amin, amax):
  """(loc, scale) [N, A] of the NormalProjectionNetwork head from the mean layer's output."""
  n, a = m_raw.shape
  loc = torch.empty_like(m_raw)
  scale = torch.empty_like(m_raw)
  _lib.call('b200rl_normal_proj_fwd', _lib.ptr(m_raw), _lib.ptr(std_bias), _lib.ptr(amin),
            _lib.ptr(amax), n, a, _lib.ptr(loc), _lib.ptr(scale), _lib.stream())
  return loc, scale


def normal_head_bwd(m_raw, std_bias, amin, amax, dparams):
  """(dm_raw, per-row std-bias gradient) from dparams = (dloc, dscale), each [N, A]."""
  dloc, dscale = dparams
  n, a = m_raw.shape
  dm = torch.empty_like(m_raw)
  ds_part = torch.empty_like(m_raw)
  _lib.call('b200rl_normal_proj_bwd', _lib.ptr(m_raw), _lib.ptr(std_bias), _lib.ptr(amin),
            _lib.ptr(amax), _lib.ptr(dloc), _lib.ptr(dscale), n, a, _lib.ptr(dm),
            _lib.ptr(ds_part), _lib.stream())
  return dm, ds_part


def reduce_std_grad(ds_part, d_std_bias):
  """d_std_bias <- column sums of the per-row std-bias gradient."""
  n, a = ds_part.shape
  ws, nb = workspace.get(ds_part.device)
  _lib.call('b200rl_colsum', _lib.ptr(ds_part), None, 0, n, a, 1.0, _lib.ptr(d_std_bias),
            _lib.ptr(ws), nb, _lib.stream())


class ActorDistributionNetwork(network.Network):
  """Emits the parameters of the action distribution: (loc, scale) of a diagonal Normal over
  bounded continuous actions, or the [N, A] logits of a Categorical over discrete ones."""

  def __init__(self, input_tensor_spec, output_tensor_spec, fc_layer_params=(200, 100),
               activation_fn='relu', kernel_initializer=None, std_bias_initializer_value=0.0,
               name='ActorDistributionNetwork', device='cuda', preprocessing_layers=None,
               conv_layer_params=None):
    super().__init__(input_tensor_spec=input_tensor_spec, state_spec=(), name=name, device=device)
    spec = nest.flatten(output_tensor_spec)
    discrete = [not s.dtype.is_floating_point for s in spec]
    if any(discrete) and len(spec) != 1:
      raise ValueError('ActorDistributionNetwork supports a single discrete action; nested or '
                       'multiple action specs are not supported.')
    if not any(discrete) and (len(spec) != 1 or len(spec[0].shape) != 1):
      raise ValueError('ActorDistributionNetwork here supports one rank-1 continuous action.')
    self._action_spec = spec[0]
    self.distribution = CATEGORICAL if discrete[0] else NORMAL
    from agents_b200.networks import q_network
    kinit = kernel_initializer or q_network._vs_init  # EncodingNetwork default initializer
    layers = encoder_layers(preprocessing_layers, conv_layer_params, fc_layer_params,
                            activation_fn, kinit)
    if self.distribution == CATEGORICAL:
      self.num_actions = _discrete_num_actions(spec[0])
      layers.append(L.Dense(self.num_actions, activation=None, kernel_initializer=_mean_init))
      self._layers = layers
      return
    self.num_actions = int(spec[0].shape[0])
    layers.append(L.Dense(self.num_actions, activation=None, kernel_initializer=_mean_init))
    self._std = StdBias(self.num_actions, std_bias_initializer_value)
    layers.append(self._std)
    self._layers = layers
    amin = np.broadcast_to(np.asarray(spec[0].minimum, np.float32), (self.num_actions,)).copy()
    amax = np.broadcast_to(np.asarray(spec[0].maximum, np.float32), (self.num_actions,)).copy()
    self._amin = torch.as_tensor(amin, device=self._device)
    self._amax = torch.as_tensor(amax, device=self._device)

  @property
  def discrete(self):
    return self.distribution == CATEGORICAL

  def dist_params_spec(self):
    """Specs of the distribution parameters the PPO policy records in policy_info."""
    from agents_b200.specs import tensor_spec
    if self.discrete:
      return {'logits': tensor_spec.TensorSpec((self.num_actions,), torch.float32, 'logits')}
    a = self._action_spec.shape
    return {'loc': tensor_spec.TensorSpec(a, torch.float32, 'loc'),
            'scale': tensor_spec.TensorSpec(a, torch.float32, 'scale')}

  @property
  def action_min(self):
    return self._amin

  @property
  def action_max(self):
    return self._amax

  def _head(self, m_raw):
    return normal_head_fwd(m_raw, self._std.bias, self._amin, self._amax)

  def distribution_params(self, observation):
    """(loc, scale) each [N, A], or logits [N, A] for a discrete action; no tape."""
    m_raw, _ = self._run(observation, keep=False)
    if self.discrete:
      return m_raw
    return self._head(m_raw)

  def forward_train(self, observation):
    m_raw, tape = self._run(observation, keep=True)
    if self.discrete:
      return m_raw, tape
    loc, scale = self._head(m_raw)
    return (loc, scale), (tape, m_raw)

  def backward(self, ctx, dparams):
    """dparams = (dloc, dscale), each [N, A] contiguous; or dlogits [N, A] for a discrete action."""
    if self.discrete:
      return super().backward(ctx, dparams)
    tape, m_raw = ctx
    dm, ds_part = normal_head_bwd(m_raw, self._std.bias, self._amin, self._amax, dparams)
    grads = super().backward(tape, dm)      # zeroes the flat gradient, then accumulates
    reduce_std_grad(ds_part, self._std.d_bias)
    return grads

  def __call__(self, observation, step_type=None, network_state=(), training=False):
    return self.distribution_params(observation), network_state
