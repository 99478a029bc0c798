"""Optimisers on flat fp32 parameter buffers, TensorFlow update rules.

The reference passes a TF optimiser object to the agents (e.g.
agents/dqn/examples/v2/train_eval.py:180 `tf.compat.v1.train.AdamOptimizer(1e-3)`;
examples/dqn/mnih15/dqn_train_eval_atari.py:176-182 RMSProp(2.5e-4, decay .95, eps 1e-5,
centered)); `optimizer.apply_gradients` then runs TF's ApplyAdam / ApplyRMSProp kernels.  These
classes keep that constructor surface and run ONE fused launch of libb200rl over the network's
flat buffer (csrc/optim.cu).  Slot variables are created lazily like TF's.
"""
import torch

from agents_b200 import _lib


class Optimizer(object):

  def __init__(self):
    self._slots = {}

  def variables(self):
    out = []
    for s in self._slots.values():
      out.extend(s.values())
    return out

  def apply_flat(self, params, grads, grad_scale=None):
    raise NotImplementedError

  def apply_gradients(self, grads_and_vars):
    """Keras-style entry: a single (flat_grads, flat_params) pair per network."""
    for g, v in grads_and_vars:
      self.apply_flat(v, g)


class AdamOptimizer(Optimizer):
  """tf.compat.v1.train.AdamOptimizer (epsilon 1e-8)."""

  def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8):
    super().__init__()
    self.learning_rate, self.beta1, self.beta2, self.epsilon = (
        float(learning_rate), float(beta1), float(beta2), float(epsilon))

  def _get_slots(self, params):
    key = params.data_ptr()
    if key not in self._slots:
      self._slots[key] = dict(
          m=torch.zeros_like(params), v=torch.zeros_like(params),
          step=torch.zeros(2, dtype=torch.int64, device=params.device))
    return self._slots[key]

  def iterations(self, params):
    return self._get_slots(params)['step'][0]

  def apply_flat(self, params, grads, grad_scale=None, gate=None):
    """gate=(counter, period): apply (and count the step) only when the int64 device `counter`
    is a multiple of `period`, decided on the device so the call can sit in a captured graph."""
    s = self._get_slots(params)
    if gate is None:
      _lib.call('b200rl_adam_tf', _lib.ptr(params), _lib.ptr(grads), _lib.ptr(s['m']),
                _lib.ptr(s['v']), params.numel(), self.learning_rate, self.beta1, self.beta2,
                self.epsilon, _lib.ptr(s['step']), _lib.ptr(grad_scale), _lib.stream())
      return
    counter, period = gate
    _lib.call('b200rl_adam_tf_gated', _lib.ptr(params), _lib.ptr(grads), _lib.ptr(s['m']),
              _lib.ptr(s['v']), params.numel(), self.learning_rate, self.beta1, self.beta2,
              self.epsilon, _lib.ptr(s['step']), _lib.ptr(grad_scale), _lib.ptr(counter),
              int(period), _lib.stream())


class Adam(AdamOptimizer):
  """tf.keras.optimizers.Adam (epsilon 1e-7, beta_1/beta_2 names)."""

  def __init__(self, learning_rate=0.001, beta_1=0.9, beta_2=0.999, epsilon=1e-7):
    super().__init__(learning_rate, beta_1, beta_2, epsilon)


class RMSPropOptimizer(Optimizer):
  """tf.compat.v1.train.RMSPropOptimizer (ms slot initialised to ones)."""
  _MS_INIT = 1.0

  def __init__(self, learning_rate, decay=0.9, momentum=0.0, epsilon=1e-10, centered=False):
    super().__init__()
    self.learning_rate, self.decay, self.momentum, self.epsilon, self.centered = (
        float(learning_rate), float(decay), float(momentum), float(epsilon), bool(centered))

  def _get_slots(self, params):
    key = params.data_ptr()
    if key not in self._slots:
      self._slots[key] = dict(ms=torch.full_like(params, self._MS_INIT),
                              mg=torch.zeros_like(params), mom=torch.zeros_like(params))
    return self._slots[key]

  def apply_flat(self, params, grads, grad_scale=None):
    s = self._get_slots(params)
    _lib.call('b200rl_rmsprop_tf', _lib.ptr(params), _lib.ptr(grads), _lib.ptr(s['ms']),
              _lib.ptr(s['mg']), _lib.ptr(s['mom']), params.numel(), self.learning_rate,
              self.decay, self.momentum, self.epsilon, int(self.centered),
              _lib.ptr(grad_scale), _lib.stream())


class RMSprop(RMSPropOptimizer):
  """tf.keras.optimizers.RMSprop (rho name, epsilon 1e-7, ms slot initialised to zeros)."""
  _MS_INIT = 0.0

  def __init__(self, learning_rate=0.001, rho=0.9, momentum=0.0, epsilon=1e-7, centered=False):
    super().__init__(learning_rate, rho, momentum, epsilon, centered)
