"""Network base class (tf_agents/networks/network.py:111).

A Network owns ONE flat fp32 parameter buffer and ONE flat gradient buffer on its device;
layers hold views.  `__call__(observation, step_type=None, network_state=(), training=False)`
returns `(output, network_state)` like the reference; `forward_train` additionally records
the activations needed by `backward`.
"""
import copy as _copy

import numpy as np
import torch

from agents_b200.networks import layers as layers_lib
from agents_b200.utils import nest
from agents_b200.utils import workspace


class Network(object):

  def __init__(self, input_tensor_spec=None, state_spec=(), name=None, device='cuda'):
    self._input_tensor_spec = input_tensor_spec
    self._state_spec = state_spec
    self._name = name or type(self).__name__
    self._device = torch.device(device)
    self._layers = []
    self._built = False
    self._params = None
    self._grads = None
    self._seed = None

  # ---- reference surface ------------------------------------------------------------------
  @property
  def name(self):
    return self._name

  @property
  def input_tensor_spec(self):
    return self._input_tensor_spec

  @property
  def state_spec(self):
    return self._state_spec

  @property
  def device(self):
    return self._device

  @property
  def layers(self):
    return list(self._layers)

  def create_variables(self, input_tensor_spec=None, **kwargs):
    """Builds parameters for `input_tensor_spec`; returns the output spec
    (network.py `create_variables`)."""
    from agents_b200.specs import tensor_spec
    if input_tensor_spec is not None:
      if self._input_tensor_spec is None:
        self._input_tensor_spec = input_tensor_spec
    if not self._built:
      if self._input_tensor_spec is None:
        raise ValueError('Network needs an input_tensor_spec to create its variables.')
      self._build(nest.flatten(self._input_tensor_spec)[0].shape)
    return tensor_spec.TensorSpec(self._output_shape, torch.float32)

  @property
  def variables(self):
    self._require_built()
    return list(self._param_views)

  @property
  def trainable_weights(self):
    return self.variables

  @property
  def non_trainable_weights(self):
    return []

  @property
  def trainable_variables(self):
    return self.variables

  @property
  def losses(self):
    """Regularisation losses as (coef, tensor) pairs (Keras `layer.losses`)."""
    out = []
    for l in self._layers:
      if getattr(l, 'l2', 0.0):
        out.append((l.l2, l.kernel))
    return out

  def copy(self, **kwargs):
    """Same architecture, freshly allocated variables (network.py `copy`)."""
    new = _copy.copy(self)
    new._layers = [_copy.copy(l) for l in self._layers]
    new._built = False
    new._params = None
    new._grads = None
    if 'name' in kwargs:
      new._name = kwargs['name']
    if self._built:
      new._build(self._input_shape)
    return new

  # ---- flat storage -----------------------------------------------------------------------
  @property
  def flat_params(self):
    self._require_built()
    return self._params

  @property
  def flat_grads(self):
    self._require_built()
    return self._grads

  @property
  def param_offsets(self):
    """int64 offsets [n_vars+1] of each variable inside the flat buffer."""
    self._require_built()
    return self._offsets

  def _require_built(self):
    if not self._built:
      self.create_variables()

  def set_seed(self, seed):
    self._seed = seed
    return self

  def _build(self, input_shape):
    shape = tuple(int(d) for d in input_shape)
    self._input_shape = shape
    sizes = []
    pending_div = None
    for l in self._layers:
      if isinstance(l, layers_lib.CastScale):
        pending_div = l.divisor
        shape = l.build(shape)
        continue
      if pending_div is not None:
        if not isinstance(l, layers_lib.Conv2D):
          raise ValueError('CastScale must be followed by a Conv2D layer (it is fused into it).')
        l.pre_divisor = pending_div
        pending_div = None
      shape = l.build(shape)
      for ps in l.param_shapes():
        sizes.append(int(np.prod(ps)))
    self._output_shape = shape
    total = int(sum(sizes))
    # pad each variable to 4 floats so views stay 16 B aligned
    offs = [0]
    for s in sizes:
      offs.append(offs[-1] + (s + 3) // 4 * 4)
    self._params = torch.zeros(max(offs[-1], 4), dtype=torch.float32, device=self._device)
    self._grads = torch.zeros_like(self._params)
    self._offsets = offs
    self._param_views = []
    self._grad_views = []
    i = 0
    for l in self._layers:
      shapes = l.param_shapes()
      if not shapes:
        continue
      pv, gv = [], []
      for ps in shapes:
        n = int(np.prod(ps))
        pv.append(self._params[offs[i]:offs[i] + n].view(ps))
        gv.append(self._grads[offs[i]:offs[i] + n].view(ps))
        i += 1
      l.bind(pv, gv)
      self._param_views.extend(pv)
      self._grad_views.extend(gv)
    self._n_params = total
    gen = None
    if self._seed is not None:
      gen = torch.Generator().manual_seed(int(self._seed))
    with torch.no_grad():
      for l in self._layers:
        if l.has_params:
          l.init_params(gen)
    self._built = True

  def _layer_range(self, layer):
    """[lo, hi) of `layer`'s gradients inside the flat gradient buffer (elements)."""
    first = layer.d_kernel
    lo = (first.data_ptr() - self._grads.data_ptr()) // 4
    last = layer.d_bias if getattr(layer, 'd_bias', None) is not None else layer.d_kernel
    hi = (last.data_ptr() - self._grads.data_ptr()) // 4 + last.numel()
    return lo, (hi + 3) // 4 * 4

  # ---- execution --------------------------------------------------------------------------
  def _run(self, x, keep):
    self._require_built()
    tape = []
    for l in self._layers:
      if isinstance(l, layers_lib.CastScale):
        continue
      y = l.forward(x)
      if keep:
        tape.append((l, x, y))
      x = y
    return x, tape

  def __call__(self, observation, step_type=None, network_state=(), training=False):
    out, _ = self._run(observation, keep=False)
    return out, network_state

  def forward_train(self, observation):
    """Forward that records activations; returns (output, tape)."""
    return self._run(observation, keep=True)

  def backward(self, tape, dy, need_input_grad=False, need_param_grads=True, grad_hook=None,
               zero_grads=True):
    """Back-propagates dLoss/d(output) through `tape`, OVERWRITING flat_grads.

    grad_hook(lo, hi): called right after the parameter gradients of a layer have been enqueued,
    with that layer's range of the flat gradient buffer, on the stream that produces them (the
    side stream inside a captured graph).  Layers are visited last to first, so successive calls
    cover a growing suffix of the buffer: data-parallel agents use it to start the gradient
    all-reduce of the large tail (fc layers) while the convolution gradients are still running.

    need_input_grad: also return dLoss/d(input) (SAC's actor loss differentiates the critics
    w.r.t. their action input); need_param_grads=False skips the weight gradients (dense only).
    zero_grads=False accumulates into flat_grads as they are (a network whose tape is run in two
    parts, the CriticNetwork observation branch).
    Returns flat_grads, or (flat_grads, d_input) when need_input_grad."""
    first = next(i for i, (l, _, _) in enumerate(tape) if l.has_params)
    # Inside a captured graph the parameter gradients (dW GEMM + fused bias column sums) of every
    # layer are forked onto a side stream: only the dX chain stays on the critical path.
    side = _side_stream(self._device) if (
        need_param_grads and torch.cuda.is_current_stream_capturing()) else None
    main = torch.cuda.current_stream() if side is not None else None
    # The flat gradient is zeroed ONCE and every layer accumulates into its views (split-K weight
    # gradients and the fused bias sums are red.global.add epilogues): one fill instead of one
    # memset node per layer.
    zeroed = not (need_param_grads and zero_grads)
    if not zeroed and side is None:
      self._grads.zero_()
      zeroed = True

    def producer_act(i):
      """Activation code of the layer whose output is tape[i]'s input (Flatten is a view)."""
      j = i - 1
      while j >= 0 and isinstance(tape[j][0], layers_lib.Flatten):
        j -= 1
      if j < 0 or not hasattr(tape[j][0], 'backward_parts'):
        return _ACT_NONE
      return tape[j][0]._act

    dy_is_preact = False     # dy already carries act' of the layer it is handed to
    for i in range(len(tape) - 1, -1, -1):
      l, x, y = tape[i]
      need_dx = need_input_grad or i > first
      if not hasattr(l, 'backward_parts'):
        dy = l.backward(x, y, dy, need_dx=need_dx)       # Flatten: reshape, flag carries through
        continue
      dz = dy.contiguous() if dy_is_preact else l.backward_act(y, dy)
      # Dense consumers fold act'(x) into their dX epilogue (one coalesced read per output row);
      # for Conv2D consumers the col2im epilogue would need a scattered read per red.add, which
      # measured slower than the separate vectorised act_bwd pass (profiles/r2/README.md)
      x_act = producer_act(i) if need_dx and isinstance(l, layers_lib.Dense) else _ACT_NONE
      if side is not None:
        side.wait_stream(main)                   # dz (and everything before it) is ready
        dz.record_stream(side)
        with torch.cuda.stream(side), workspace.slot(1):
          if not zeroed:
            self._grads.zero_()
            zeroed = True
          l.backward_parts(x, dz, need_dx=False, need_dw=True, accumulate=1)
          if grad_hook is not None:
            grad_hook(*self._layer_range(l))
        dy = l.backward_parts(x, dz, need_dx=True, need_dw=False, x_act=x_act) if need_dx else None
      elif not need_param_grads:
        if isinstance(l, layers_lib.Dense):
          dy = l.backward_parts(x, dz, need_dx=need_dx, need_dw=False, x_act=x_act)
        else:
          raise NotImplementedError('need_param_grads=False is only supported for Dense stacks.')
      else:
        dy = l.backward_parts(x, dz, need_dx=need_dx, need_dw=True, x_act=x_act, accumulate=1)
        if grad_hook is not None:
          grad_hook(*self._layer_range(l))
      dy_is_preact = x_act != _ACT_NONE
    if side is not None:
      main.wait_stream(side)
    elif not torch.cuda.is_current_stream_capturing():
      workspace.mirror(self._device, 1)          # size the side-stream scratch for a later capture
      _side_stream(self._device)
    if need_input_grad:
      return self._grads, dy
    return self._grads


_ACT_NONE = 0
_SIDE_STREAMS = {}


def _side_stream(device):
  device = torch.device(device)
  key = device.index if device.index is not None else torch.cuda.current_device()
  if key not in _SIDE_STREAMS:
    _SIDE_STREAMS[key] = torch.cuda.Stream(device=device)
  return _SIDE_STREAMS[key]


def allocate_jointly(networks):
  """Re-homes the parameters of several built Networks into ONE flat buffer (and one gradient
  buffer) so a single optimiser / clip / all-reduce launch covers all of them — the reference
  applies one optimizer to `actor_net.trainable_weights + value_net.trainable_weights`
  (agents/ppo/ppo_agent.py:916-923).  Returns (flat_params, flat_grads)."""
  for n in networks:
    n._require_built()
  total = sum(n._params.numel() for n in networks)
  dev = networks[0].device
  params = torch.zeros(total, dtype=torch.float32, device=dev)
  grads = torch.zeros_like(params)
  off = 0
  for n in networks:
    k = n._params.numel()
    params[off:off + k].copy_(n._params)
    n._params = params[off:off + k]
    n._grads = grads[off:off + k]
    n._param_views, n._grad_views = [], []
    i = 0
    for l in n._layers:
      shapes = l.param_shapes()
      if not shapes:
        continue
      pv, gv = [], []
      for ps in shapes:
        cnt = int(np.prod(ps))
        o = n._offsets[i]
        pv.append(n._params[o:o + cnt].view(ps))
        gv.append(n._grads[o:o + cnt].view(ps))
        i += 1
      l.bind(pv, gv)
      n._param_views.extend(pv)
      n._grad_views.extend(gv)
    off += k
  return params, grads
