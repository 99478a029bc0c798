"""GaussianActionsSampler (tf_agents/policies/samplers/qtopt_cem_actions_sampler_continuous.py):
the sampling distribution of CEMPolicy's search over one rank-1 bounded float action.

`sample_batch_and_clip` draws [B, N, A] actions N(mean, var) and clips them to the spec
(b200rl_cem_sample); `refit_distribution_to` refits mean and var [B, A] to the samples at the
given [B, M] indices with tf.nn.moments semantics, the mean first, then the mean of squared
deviations, both divided by M (b200rl_cem_refit).  CEMPolicy does not call these two methods: it
runs the same kernels with the selection fused into the refit and the samples written straight
into the critic's input.  Sample clippers and rejecters, integer actions and nested specs are not
supported.
"""
import numpy as np
import torch

from agents_b200 import _lib
from agents_b200.utils import nest

_SAMPLER_SEED_TAG = 0x43454D5F53414D50


class GaussianActionsSampler(object):
  """Continuous Gaussian actions sampler over one rank-1 bounded float action."""

  def __init__(self, action_spec, sample_clippers=None, sample_rejecters=None,
               max_rejection_iterations=10, support_integer=False, seed=0):
    flat = nest.flatten(action_spec)
    if len(flat) != 1:
      raise NotImplementedError('GaussianActionsSampler supports one action tensor, not a nest.')
    spec = flat[0]
    if not spec.dtype.is_floating_point:
      raise ValueError('Only continuous action is supported by this sampler. The action_spec: {} '
                       'contains discrete action'.format(action_spec))
    if len(spec.shape) != 1:
      raise ValueError('Only 1d action is supported by this sampler. The action_spec: {} contains '
                       'an action whose rank is not 1.'.format(action_spec))
    if sample_clippers or sample_rejecters:
      raise NotImplementedError('sample_clippers and sample_rejecters are not supported.')
    if support_integer:
      raise NotImplementedError('support_integer is not supported.')
    self._action_spec = action_spec
    self._num_actions = int(spec.shape[0])
    a = self._num_actions
    self._minimum = np.broadcast_to(np.asarray(spec.minimum, np.float32), (a,)).copy()
    self._maximum = np.broadcast_to(np.asarray(spec.maximum, np.float32), (a,)).copy()
    self._bounds = {}
    self._seed = (int(seed) ^ _SAMPLER_SEED_TAG) & 0xFFFFFFFFFFFFFFFF
    self._rng = None

  @property
  def action_spec(self):
    return self._action_spec

  @property
  def num_actions(self):
    return self._num_actions

  def bounds(self, device):
    """(amin, amax) [A] float32 tensors on `device`."""
    device = torch.device(device)
    if device not in self._bounds:
      self._bounds[device] = (torch.as_tensor(self._minimum, device=device),
                              torch.as_tensor(self._maximum, device=device))
    return self._bounds[device]

  def sample_batch_and_clip(self, num_samples, mean, var, state=None, z=None):
    """[B, N, A] actions clip(mean + sqrt(var) z, spec) for mean, var [B, A]; z [B, N, A] supplies
    the N(0, 1) draws (else Philox on the device)."""
    del state
    mean, var = mean.float().contiguous(), var.float().contiguous()
    B, A = mean.shape
    dev = mean.device
    if self._rng is None:
      self._rng = torch.zeros(2, dtype=torch.int64, device=dev)
    lo, hi = self.bounds(dev)
    out = torch.empty((B, int(num_samples), A), dtype=torch.float32, device=dev)
    z = None if z is None else z.float().contiguous()
    _lib.call('b200rl_cem_sample', None, 0, B, int(num_samples), 0, A, _lib.ptr(mean), A,
              _lib.ptr(var), A, 0.0, _lib.ptr(lo), _lib.ptr(hi), _lib.ptr(z), self._seed,
              _lib.ptr(self._rng), _lib.ptr(out), A, _lib.stream())
    return out

  def refit_distribution_to(self, target_sample_indices, samples):
    """(mean, var) [B, A] of samples [B, N, A] at target_sample_indices [B, M], in index order."""
    samples = samples.float().contiguous()
    B, N, A = samples.shape
    ind = target_sample_indices.to(torch.int32).contiguous()
    mean = torch.empty((B, A), dtype=torch.float32, device=samples.device)
    var = torch.empty_like(mean)
    _lib.call('b200rl_cem_refit', None, _lib.ptr(ind), _lib.ptr(samples), A, 0, B, N,
              ind.shape[1], A, 0.0, None, None, 1, None, 0, None, _lib.ptr(mean), _lib.ptr(var),
              None, None, _lib.stream())
    return mean, var
