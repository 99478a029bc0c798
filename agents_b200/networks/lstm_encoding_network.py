"""LSTMEncodingNetwork (tf_agents/networks/lstm_encoding_network.py): input encoder (optional
preprocessing / Conv2D stack, Dense stack) -> one LSTM layer per `lstm_size` entry -> output Dense
stack, over `[B, ...]` single steps or `[B, T, ...]` sequences.

The LSTM layer is keras LSTMCell (implementation=2) under DynamicUnroll: a step whose step_type is
FIRST starts from the zero state.  Its input projection x W + b over all B*T rows is one
b200rl_dense_fwd; the recurrence runs all T steps in one b200rl_lstm_seq_fwd launch (csrc/lstm.cu).
The backward is one b200rl_lstm_seq_bwd launch to the gate gradients dG, then GEMMs over the B*T
rows: dW, db and dx from (x, dG), dU from (h_used, dG).  Stacked cells run layer by layer over the
whole sequence, which equals StackedRNNCells stepping (layer l at t reads layer l-1 at t and layer
l at t-1 only).  Training always starts from the zero state, so no gradient reaches the initial
state.
"""
import torch

from agents_b200 import _lib
from agents_b200.networks import actor_distribution_network
from agents_b200.networks import layers as L
from agents_b200.networks import network
from agents_b200.networks import q_network
from agents_b200.specs import tensor_spec
from agents_b200.utils import nest
from agents_b200.utils import workspace

MAX_UNITS = 256
_STEP_MID = 1


def _orthogonal(shape, generator):
  """keras Orthogonal(gain=1): the Q factor of a normal matrix, shaped [rows, cols]."""
  rows, cols = shape
  a = torch.randn((max(rows, cols), min(rows, cols)), dtype=torch.float64, generator=generator)
  q, r = torch.linalg.qr(a)
  q = q * torch.sign(torch.diagonal(r))
  if rows < cols:
    q = q.t()
  return q.float().contiguous()


class LSTM(L.Layer):
  """One LSTM layer: kernel [in, 4H], recurrent_kernel [H, 4H], bias [4H] (gates i, f, g, o)."""
  has_params = True

  def __init__(self, units):
    self.units = int(units)
    if not 1 <= self.units <= MAX_UNITS:
      raise ValueError(f'LSTM units must be in [1, {MAX_UNITS}], got {self.units}.')
    self.l2 = 0.0

  def build(self, input_shape):
    if len(input_shape) != 1:
      raise ValueError(f'LSTM expects rank-1 inputs per step, got {input_shape}.')
    self.in_features = int(input_shape[0])
    return (self.units,)

  def param_shapes(self):
    h4 = 4 * self.units
    return [(self.in_features, h4), (self.units, h4), (h4,)]

  def bind(self, params, grads):
    self.kernel, self.recurrent_kernel, self.bias = params
    self.d_kernel, self.d_recurrent_kernel, self.d_bias = grads

  def init_params(self, generator):
    h = self.units
    self.kernel.copy_(L.glorot_uniform((self.in_features, 4 * h), self.in_features, 4 * h,
                                       generator))
    self.recurrent_kernel.copy_(_orthogonal((h, 4 * h), generator))
    self.bias.zero_()
    self.bias[h:2 * h] = 1.0                                     # unit_forget_bias

  def forward_seq(self, x, step_type, B, T, state=None):
    """x [B*T, in] (batch-major rows), step_type int32 [B, T], state (h0, c0) [B, H] or None.
    Returns (h [B*T, H], (h_T, c_T), ctx)."""
    H, dev = self.units, x.device
    x = x.contiguous()
    n = B * T
    xw = torch.empty((n, 4 * H), dtype=torch.float32, device=dev)
    ws, nb = workspace.get(dev)
    _lib.call('b200rl_dense_fwd', _lib.ptr(x), self.in_features, _lib.ptr(self.kernel),
              _lib.ptr(self.bias), _lib.ptr(xw), n, self.in_features, 4 * H, _lib.ACT_NONE,
              _lib.ptr(ws), nb, _lib.stream())
    h = torch.empty((n, H), dtype=torch.float32, device=dev)
    gates = torch.empty((n, 4 * H), dtype=torch.float32, device=dev)
    c = torch.empty((n, H), dtype=torch.float32, device=dev)
    h_used = torch.empty((n, H), dtype=torch.float32, device=dev)
    hT = torch.empty((B, H), dtype=torch.float32, device=dev)
    cT = torch.empty((B, H), dtype=torch.float32, device=dev)
    h0, c0 = (None, None) if state is None else (state[0].float().contiguous(),
                                                  state[1].float().contiguous())
    _lib.call('b200rl_lstm_seq_fwd', _lib.ptr(xw), _lib.ptr(self.recurrent_kernel),
              _lib.ptr(step_type), _lib.ptr(h0), _lib.ptr(c0), B, T, H, _lib.ptr(h),
              _lib.ptr(gates), _lib.ptr(c), _lib.ptr(h_used), _lib.ptr(hT), _lib.ptr(cT),
              _lib.stream())
    return h, (hT, cT), (x, gates, c, h_used, c0, step_type, B, T)

  def backward_seq(self, ctx, dh, need_dx, need_param_grads=True):
    """Accumulates dW, dU, db into the gradient views; returns dx [B*T, in] (or None).
    need_param_grads=False runs only the BPTT and the dx GEMM: the gradient views are untouched
    (DDPG's dQ/da through a recurrent critic)."""
    x, gates, c, h_used, c0, step_type, B, T = ctx
    H, dev = self.units, x.device
    n = B * T
    dh = dh.contiguous()
    dG = torch.empty((n, 4 * H), dtype=torch.float32, device=dev)
    _lib.call('b200rl_lstm_seq_bwd', _lib.ptr(dh), _lib.ptr(gates), _lib.ptr(c), _lib.ptr(c0),
              _lib.ptr(self.recurrent_kernel), _lib.ptr(step_type), B, T, H, _lib.ptr(dG),
              _lib.stream())
    dx = torch.empty((n, self.in_features), dtype=torch.float32, device=dev) if need_dx else None
    if not (need_dx or need_param_grads):
      return None
    ws, nb = workspace.get(dev)
    dw, db = (self.d_kernel, self.d_bias) if need_param_grads else (None, None)
    _lib.call('b200rl_dense_bwd', _lib.ptr(x), self.in_features, _lib.ptr(self.kernel),
              _lib.ptr(dG), _lib.ptr(dx), _lib.ptr(dw), _lib.ptr(db), n,
              self.in_features, 4 * H, 1, _lib.ACT_NONE, _lib.ptr(ws), nb, _lib.stream())
    if need_param_grads:
      _lib.call('b200rl_dense_bwd', _lib.ptr(h_used), H, _lib.ptr(self.recurrent_kernel),
                _lib.ptr(dG), None, _lib.ptr(self.d_recurrent_kernel), None, n, H, 4 * H, 1,
                _lib.ACT_NONE, _lib.ptr(ws), nb, _lib.stream())
    return dx


class LSTMEncodingNetwork(network.Network):
  """`__call__(observation, step_type, network_state)` -> (output, new_state).  Observations are
  `[B, ...]` (one step; a time axis of 1 is added) or `[B, T, ...]`; outputs keep that outer
  shape.  The state is (h, c) for one LSTM layer and a tuple of (h, c) per layer when stacked."""

  def __init__(self, input_tensor_spec, preprocessing_layers=None, preprocessing_combiner=None,
               conv_layer_params=None, input_fc_layer_params=(75, 40), lstm_size=None,
               output_fc_layer_params=(75, 40), activation_fn='relu', rnn_construction_fn=None,
               rnn_construction_kwargs=None, dtype=None, name='LSTMEncodingNetwork',
               device='cuda'):
    if rnn_construction_fn is not None:
      raise NotImplementedError('rnn_construction_fn is not supported: the LSTM layers run on '
                                'the fused sequence kernels; give lstm_size instead.')
    if preprocessing_combiner is not None:
      raise NotImplementedError('preprocessing_combiner (multi-input observations) is not '
                                'supported by the recurrent networks.')
    if not lstm_size:
      raise ValueError('Need to provide either custom rnn_construction_fn or lstm_size.')
    counter = iter(range(2 * len(lstm_size)))
    specs = tuple((tensor_spec.TensorSpec((n,), torch.float32, 'network_state_%d' % next(counter)),
                   tensor_spec.TensorSpec((n,), torch.float32, 'network_state_%d' % next(counter)))
                  for n in lstm_size)
    super().__init__(input_tensor_spec=input_tensor_spec,
                     state_spec=specs[0] if len(specs) == 1 else specs, name=name, device=device)
    kinit = q_network._vs_init
    self._pre = actor_distribution_network.encoder_layers(
        preprocessing_layers, conv_layer_params, input_fc_layer_params, activation_fn, kinit)
    self._cells = [LSTM(n) for n in lstm_size]
    self._post = [L.Dense(n, activation=activation_fn, kernel_initializer=kinit)
                  for n in (output_fc_layer_params or ())]
    self._layers = self._pre + self._cells + self._post

  def copy(self, **kwargs):
    """Network.copy replaces `_layers` only; the copy's encoder, cell and output lists must hold
    the copied layers (bound to the copy's variables), not the original's."""
    new = super().copy(**kwargs)
    n_pre, n_cells = len(self._pre), len(self._cells)
    new._pre = new._layers[:n_pre]
    new._cells = new._layers[n_pre:n_pre + n_cells]
    new._post = new._layers[n_pre + n_cells:]
    return new

  # ---- state ------------------------------------------------------------------------------
  def get_initial_state(self, batch_size=None):
    return nest.map_structure(
        lambda s: torch.zeros((batch_size,) + tuple(s.shape), dtype=torch.float32,
                              device=self._device), self._state_spec)

  def _layer_states(self, network_state):
    if network_state is None or (isinstance(network_state, (tuple, list)) and
                                 len(network_state) == 0):
      return [None] * len(self._cells)
    if len(self._cells) == 1:
      return [network_state]
    return list(network_state)

  def _pack_state(self, finals):
    return finals[0] if len(finals) == 1 else tuple(finals)

  # ---- execution --------------------------------------------------------------------------
  def _sequence(self, observation, step_type):
    """Returns (obs [B*T, ...], step_type int32 [B, T], B, T, has_time_dim).  `observation` may
    also be the B*T rows of a [B, T] sequence already flattened, with step_type [B, T]."""
    self._require_built()
    obs = nest.flatten(observation)[0]
    rank = len(self._input_shape)
    outer = obs.dim() - rank
    if outer == 1 and step_type is not None and step_type.dim() == 2 and \
        step_type.numel() == obs.shape[0]:
      B, T = step_type.shape
      has_time = True
    elif outer == 1:
      B, T, has_time = obs.shape[0], 1, False
    elif outer == 2:
      B, T, has_time = obs.shape[0], obs.shape[1], True
    else:
      raise ValueError('Input observation must have a batch or batch x time outer shape.')
    obs = obs.reshape((B * T,) + tuple(obs.shape[outer:]))
    if step_type is None:
      st = torch.full((B, T), _STEP_MID, dtype=torch.int32, device=obs.device)
    else:
      st = step_type.to(torch.int32).reshape(B, T).contiguous()
    return obs, st, B, T, has_time

  @staticmethod
  def _run_stack(layers, x, tape):
    for l in layers:
      if isinstance(l, L.CastScale):
        continue
      y = l.forward(x)
      tape.append((l, x, y))
      x = y
    return x

  def _run_seq(self, obs, st, B, T, network_state):
    """Returns (output [B*T, ...], new_state, tape)."""
    pre_tape = []
    x = self._run_stack(self._pre, obs, pre_tape)
    x, state, ctxs, post_tape = self._run_recurrent(x, st, B, T, network_state)
    return x, state, (pre_tape, ctxs, post_tape)

  def _run_recurrent(self, x, st, B, T, network_state):
    """The LSTM layers and the output stack over the encoded rows x [B*T, ...]; returns
    (output [B*T, ...], new_state, cell contexts, output-stack tape)."""
    post_tape, ctxs, finals = [], [], []
    for cell, s in zip(self._cells, self._layer_states(network_state)):
      x, fin, ctx = cell.forward_seq(x, st, B, T, s)
      ctxs.append(ctx)
      finals.append(fin)
    x = self._run_stack(self._post, x, post_tape)
    return x, self._pack_state(finals), ctxs, post_tape

  def _unflatten(self, out, B, T, has_time):
    return out.reshape(((B, T) if has_time else (B,)) + tuple(out.shape[1:]))

  def __call__(self, observation, step_type=None, network_state=(), training=False):
    obs, st, B, T, has_time = self._sequence(observation, step_type)
    out, state, _ = self._run_seq(obs, st, B, T, network_state)
    return self._unflatten(out, B, T, has_time), state

  def forward_train(self, observation, step_type=None):
    """[B, T] forward from the zero state that records the tape; returns (output [B*T, ...],
    tape)."""
    obs, st, B, T, _ = self._sequence(observation, step_type)
    out, _, tape = self._run_seq(obs, st, B, T, ())
    return out, tape

  def backward(self, tape, dy):
    """Back-propagates dLoss/d(output [B*T, ...]) through `tape`, OVERWRITING flat_grads."""
    pre_tape, ctxs, post_tape = tape
    need_pre = any(l.has_params for l, _, _ in pre_tape)
    dh = self._backward_recurrent(ctxs, post_tape, dy, need_pre)
    if need_pre:
      super().backward(pre_tape, dh, zero_grads=False)
    return self._grads

  def _backward_recurrent(self, ctxs, post_tape, dy, need_dx, need_param_grads=True):
    """Back-propagates dy through the output stack and the LSTM layers of `_run_recurrent`;
    returns dLoss/d(the first LSTM layer's input) when need_dx.  With need_param_grads the
    gradients are OVERWRITTEN from here on; without, flat_grads is left untouched."""
    if any(l.has_params for l, _, _ in post_tape):
      _, dh = network.Network.backward(self, post_tape, dy, need_input_grad=True,
                                       need_param_grads=need_param_grads)
    else:
      if need_param_grads:
        self._grads.zero_()
      dh = dy
    for i in range(len(self._cells) - 1, -1, -1):
      dh = self._cells[i].backward_seq(ctxs[i], dh, need_dx=i > 0 or need_dx,
                                       need_param_grads=need_param_grads)
    return dh
