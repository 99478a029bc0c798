"""Layers with explicit forward/backward over libb200rl (no autograd tape).

Stand-ins for the Keras layers the reference's networks are built from
(networks/encoding_network.py:224-312): Dense, Conv2D (NHWC, VALID), Flatten and the
cast-and-scale Lambda of the Atari net (examples/dqn/mnih15/dqn_train_eval_atari.py:104).
Parameters are views into one flat fp32 buffer owned by the enclosing Network, gradients are
views into a matching flat buffer, so optimiser / Polyak / all-reduce are single launches.
"""
import ctypes
import math

import numpy as np
import torch

from agents_b200 import _lib
from agents_b200.utils import workspace

_ACTS = {None: _lib.ACT_NONE, 'linear': _lib.ACT_NONE, 'relu': _lib.ACT_RELU,
         'tanh': _lib.ACT_TANH}


def _act_code(act):
  if callable(act):
    act = getattr(act, '__name__', None)
  if act not in _ACTS:
    raise ValueError(f'Unsupported activation {act!r}; supported: relu, tanh, None.')
  return _ACTS[act]


def variance_scaling(shape, fan_in, scale=2.0, generator=None):
  """variance_scaling_initializer(scale, fan_in, truncated_normal) (encoding_network.py:224-226)."""
  stddev = math.sqrt(scale / max(1.0, fan_in)) / 0.87962566103423978
  t = torch.empty(shape, dtype=torch.float32)
  torch.nn.init.trunc_normal_(t, mean=0.0, std=stddev, a=-2 * stddev, b=2 * stddev,
                              generator=generator)
  return t


def glorot_uniform(shape, fan_in, fan_out, generator=None):
  limit = math.sqrt(6.0 / (fan_in + fan_out))
  return (torch.rand(shape, dtype=torch.float32, generator=generator) * 2 - 1) * limit


class Layer(object):
  """Base: subclasses define build/forward/backward; params are bound by the Network."""
  has_params = False

  def build(self, input_shape):
    """Returns output shape (without batch dim)."""
    raise NotImplementedError

  def param_shapes(self):
    return []

  def bind(self, params, grads):
    pass

  def init_params(self, generator):
    pass

  def forward(self, x):
    raise NotImplementedError

  def backward(self, x, y, dy, need_dx):
    raise NotImplementedError


def _batch_strided(x, inner_elems):
  """Accepts tensors whose only non-standard stride is the batch stride. Returns (tensor,
  batch_stride_in_elements)."""
  if x.is_contiguous():
    return x, inner_elems
  inner = x[0]
  if x.dim() >= 2 and inner.is_contiguous() and x.stride(0) >= inner_elems:
    return x, x.stride(0)
  x = x.contiguous()
  return x, inner_elems


class CastScale(Layer):
  """tf.cast(obs, float32) / divisor as a preprocessing layer; fused into the next layer."""

  def __init__(self, divisor=255.0):
    self.divisor = float(divisor)

  def build(self, input_shape):
    return tuple(input_shape)


class Flatten(Layer):

  def build(self, input_shape):
    self._in_shape = tuple(input_shape)
    return (int(np.prod(input_shape)),)

  def forward(self, x):
    return x.reshape(x.shape[0], -1)

  def backward(self, x, y, dy, need_dx):
    return dy.reshape(x.shape) if need_dx else None


class Dense(Layer):
  """y = act(x @ kernel + bias), kernel [in, units] (Keras layout)."""
  has_params = True

  def __init__(self, units, activation=None, use_bias=True, kernel_initializer=None,
               bias_initializer=None, kernel_regularizer_l2=0.0):
    self.units = int(units)
    self.activation = activation
    self._act = _act_code(activation)
    self.use_bias = use_bias
    self.kernel_initializer = kernel_initializer
    self.bias_initializer = bias_initializer
    self.l2 = float(kernel_regularizer_l2 or 0.0)

  def build(self, input_shape):
    if len(input_shape) != 1:
      raise ValueError(f'Dense expects rank-1 inputs per example, got {input_shape}.')
    self.in_features = int(input_shape[0])
    return (self.units,)

  def param_shapes(self):
    shapes = [(self.in_features, self.units)]
    if self.use_bias:
      shapes.append((self.units,))
    return shapes

  def bind(self, params, grads):
    self.kernel, self.d_kernel = params[0], grads[0]
    self.bias, self.d_bias = (params[1], grads[1]) if self.use_bias else (None, None)

  def init_params(self, generator):
    init = self.kernel_initializer
    if init is None:
      w = glorot_uniform((self.in_features, self.units), self.in_features, self.units, generator)
    elif callable(init):
      w = init((self.in_features, self.units), self.in_features, generator)
    else:
      w = torch.as_tensor(np.asarray(init, dtype=np.float32)).reshape(self.in_features, self.units)
    self.kernel.copy_(w)
    if self.use_bias:
      b = self.bias_initializer
      if b is None:
        self.bias.zero_()
      elif callable(b):
        self.bias.copy_(b((self.units,), self.in_features, generator))
      else:
        self.bias.copy_(torch.as_tensor(np.broadcast_to(
            np.asarray(b, dtype=np.float32).reshape(-1), (self.units,)).copy()))

  def forward(self, x):
    x, ldx = _batch_strided(x, self.in_features)
    m = x.shape[0]
    y = torch.empty((m, self.units), dtype=torch.float32, device=x.device)
    ws, nb = workspace.get(x.device)
    _lib.call('b200rl_dense_fwd', _lib.dptr(x), ldx, _lib.ptr(self.kernel), _lib.ptr(self.bias), _lib.ptr(y), m, self.in_features,
              self.units, self._act, _lib.ptr(ws), nb, _lib.stream())
    return y

  def backward_act(self, y, dy):
    """dLoss/d(pre-activation) from dLoss/d(output)."""
    dy = dy.contiguous()
    if self._act == _lib.ACT_NONE:
      return dy
    dz = torch.empty_like(dy)
    _lib.call('b200rl_act_bwd', _lib.ptr(y), _lib.ptr(dy), _lib.ptr(dz), dy.numel(), self._act,
              _lib.stream())
    return dz

  def backward_parts(self, x, dz, need_dx, need_dw, x_act=_lib.ACT_NONE, accumulate=0):
    """Input gradient and/or parameter gradients from dz (either half may be skipped, so that the
    two halves can run on different streams).  `x_act`: activation code of the layer that
    produced `x`; the returned input gradient is then w.r.t. that layer's pre-activation (the
    act' factor is applied in the GEMM epilogue).  `accumulate`: add into the gradient views
    (the Network zeroes its flat gradient buffer once per backward pass)."""
    x, ldx = _batch_strided(x, self.in_features)
    m = x.shape[0]
    dx = torch.empty((m, self.in_features), dtype=torch.float32, device=x.device) if need_dx else None
    ws, nb = workspace.get(x.device)
    _lib.call('b200rl_dense_bwd', _lib.dptr(x), ldx, _lib.ptr(self.kernel), _lib.ptr(dz),
              _lib.ptr(dx), _lib.ptr(self.d_kernel) if need_dw else None,
              _lib.ptr(self.d_bias) if need_dw else None, m, self.in_features,
              self.units, int(accumulate), int(x_act), _lib.ptr(ws), nb, _lib.stream())
    return dx

  def backward(self, x, y, dy, need_dx, need_dw=True, x_act=_lib.ACT_NONE):
    return self.backward_parts(x, self.backward_act(y, dy), need_dx, need_dw, x_act)


class Conv2D(Layer):
  """NHWC VALID convolution, kernel [KH, KW, C, F] (Keras HWIO)."""
  has_params = True

  def __init__(self, filters, kernel_size, strides=1, activation=None, kernel_initializer=None):
    self.filters = int(filters)
    ks = kernel_size if isinstance(kernel_size, (tuple, list)) else (kernel_size, kernel_size)
    self.kh, self.kw = int(ks[0]), int(ks[1])
    st = strides if not isinstance(strides, (tuple, list)) else strides[0]
    self.stride = int(st)
    self.activation = activation
    self._act = _act_code(activation)
    self.kernel_initializer = kernel_initializer
    self.pre_divisor = None   # set by the Network when preceded by CastScale
    self.l2 = 0.0
    self.use_bias = True

  def build(self, input_shape):
    if len(input_shape) != 3:
      raise ValueError(f'Conv2D expects [H,W,C] inputs per example, got {input_shape}.')
    self.h, self.w, self.c = [int(d) for d in input_shape]
    self.oh = (self.h - self.kh) // self.stride + 1
    self.ow = (self.w - self.kw) // self.stride + 1
    return (self.oh, self.ow, self.filters)

  def param_shapes(self):
    return [(self.kh, self.kw, self.c, self.filters), (self.filters,)]

  def bind(self, params, grads):
    self.kernel, self.bias = params
    self.d_kernel, self.d_bias = grads

  def init_params(self, generator):
    fan_in = self.kh * self.kw * self.c
    shape = (self.kh, self.kw, self.c, self.filters)
    init = self.kernel_initializer
    if init is None:
      w = glorot_uniform(shape, fan_in, self.kh * self.kw * self.filters, generator)
    elif callable(init):
      w = init(shape, fan_in, generator)
    else:
      w = torch.as_tensor(np.asarray(init, dtype=np.float32)).reshape(shape)
    self.kernel.copy_(w)
    self.bias.zero_()

  def _geom(self, x):
    g = _lib.ConvGeom()
    g.N, g.H, g.W, g.C = x.shape[0], self.h, self.w, self.c
    g.KH, g.KW, g.F, g.stride = self.kh, self.kw, self.filters, self.stride
    return g

  def _input(self, x):
    is_u8 = x.dtype == torch.uint8
    if is_u8 and self.pre_divisor is None:
      raise ValueError('uint8 inputs need a CastScale preprocessing layer before Conv2D.')
    if not is_u8 and x.dtype != torch.float32:
      x = x.float()
    x, bstride = _batch_strided(x, self.h * self.w * self.c)
    return x, bstride, is_u8

  def forward(self, x):
    x, bstride, is_u8 = self._input(x)
    g = self._geom(x)
    g.x_batch_stride = bstride
    y = torch.empty((x.shape[0], self.oh, self.ow, self.filters), dtype=torch.float32,
                    device=x.device)
    ws, nb = workspace.get(x.device)
    _lib.call('b200rl_conv2d_fwd', _lib.dptr(x), int(is_u8), float(self.pre_divisor or 1.0),
              _lib.ptr(self.kernel), _lib.ptr(self.bias), _lib.ptr(y), ctypes.byref(g), self._act,
              _lib.ptr(ws), nb, _lib.stream())
    return y

  def backward_act(self, y, dy):
    dy = dy.contiguous()
    if self._act == _lib.ACT_NONE:
      return dy
    dz = torch.empty_like(dy)
    _lib.call('b200rl_act_bwd', _lib.ptr(y), _lib.ptr(dy), _lib.ptr(dz), dy.numel(), self._act,
              _lib.stream())
    return dz

  def backward_parts(self, x, dz, need_dx, need_dw, x_act=_lib.ACT_NONE, accumulate=0):
    x, bstride, is_u8 = self._input(x)
    g = self._geom(x)
    g.x_batch_stride = bstride
    dx = None
    need = 0
    if need_dx:
      dx = torch.empty((x.shape[0], self.h, self.w, self.c), dtype=torch.float32, device=x.device)
      need = x.shape[0] * self.oh * self.ow * self.kh * self.kw * self.c * 4
    ws, nb = workspace.get(x.device, need)
    _lib.call('b200rl_conv2d_bwd', _lib.dptr(x), int(is_u8), float(self.pre_divisor or 1.0),
              _lib.ptr(self.kernel), _lib.ptr(dz), _lib.ptr(dx),
              _lib.ptr(self.d_kernel) if need_dw else None,
              _lib.ptr(self.d_bias) if need_dw else None, ctypes.byref(g), int(accumulate),
              int(x_act), _lib.ptr(ws), nb, _lib.stream())
    return dx

  def backward(self, x, y, dy, need_dx, need_dw=True, x_act=_lib.ACT_NONE):
    return self.backward_parts(x, self.backward_act(y, dy), need_dx, need_dw, x_act)
