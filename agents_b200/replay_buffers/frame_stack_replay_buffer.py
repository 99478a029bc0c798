"""FrameStackReplayBuffer: TFUniformReplayBuffer semantics with frame de-duplicated storage.

The reference's Atari pipelines store the `[84, 84, 4]` stack the FrameStack4 wrapper emits
(environments/atari_wrappers.py:82-126) in every slot, i.e. each frame four times; de-duplication
exists only in the host-side `PyHashedReplayBuffer` (replay_buffers/py_hashed_replay_buffer.py).
This buffer keeps ONE frame per slot (4x capacity for the same HBM) and rebuilds
`[B, T, H, W, K]` observations in the gather (`b200rl_rb_gather_frame_stack`).

Contract (oracle/frame_stack.py): the producer follows the frame-stack rule (stack filled with the
first frame at FIRST steps, newest frame last); `add_batch` accepts either the stacked observation
`[B_env, H, W, K]` (the newest frame is stored) or the single frame `[B_env, H, W]`; sampled
windows are drawn from the plain range until the ring wraps and from ids with K-1 stored
predecessors afterwards, so a rebuilt stack never reads an overwritten slot; BufferInfo carries the
probability of that range.
Everything else (ring layout, Philox draws, BufferInfo) is the wrapped TFUniformReplayBuffer.

Validated on the GPU (tests/test_zz_late_gpu.py: rebuilt stacks are bit-identical to what a
FrameStack-K producer emitted, before and after the ring wraps).
"""
import ctypes

import numpy as np
import torch

from agents_b200 import _lib
from agents_b200.replay_buffers import table
from agents_b200.replay_buffers import tf_uniform_replay_buffer as rb_mod
from agents_b200.specs import tensor_spec
from agents_b200.utils import nest


class FrameStackReplayBuffer(object):

  def __init__(self, data_spec, batch_size, max_length=1000, device='cuda', seed=0):
    obs = data_spec.observation
    if not isinstance(obs, tensor_spec.TensorSpec) or obs.dtype != torch.uint8 or len(obs.shape) != 3:
      raise ValueError('FrameStackReplayBuffer needs a uint8 [H, W, K] observation spec.')
    self._h, self._w, self._k = [int(d) for d in obs.shape]
    if not 1 <= self._k <= 4 or (self._h * self._w) % 4:
      raise ValueError('Stack depth must be 1..4 and H*W a multiple of 4.')
    self._data_spec = data_spec
    frame_spec = tensor_spec.TensorSpec((self._h, self._w), torch.uint8, obs.name or 'observation')
    self._inner_spec = data_spec._replace(observation=frame_spec)
    self._rb = rb_mod.TFUniformReplayBuffer(self._inner_spec, batch_size=batch_size,
                                            max_length=max_length, device=device, seed=seed)
    flat = nest.flatten(self._inner_spec)
    self._obs_index = next(i for i, s in enumerate(flat) if s is frame_spec)
    self._step_type_index = next(i for i, s in enumerate(flat) if s is self._inner_spec.step_type)
    if self._inner_spec.step_type.dtype != torch.int32:
      raise ValueError('FrameStackReplayBuffer reads step_type as int32 inside the gather kernel; '
                       'got {}.'.format(self._inner_spec.step_type.dtype))

  @property
  def data_spec(self):
    return self._data_spec

  @property
  def batch_size(self):
    return self._rb.batch_size

  @property
  def max_length(self):
    return self._rb.max_length

  @property
  def device(self):
    return self._rb.device

  @property
  def stack_depth(self):
    return self._k

  def num_frames(self):
    return self._rb.num_frames()

  def clear(self):
    return self._rb.clear()

  def add_batch(self, items):
    obs = items.observation
    if obs.dim() == 4:                     # stacked [B_env, H, W, K]: keep the newest frame
      obs = obs[..., -1].contiguous()
    return self._rb.add_batch(items._replace(observation=obs))

  def _valid_range(self, num_steps):
    """oracle/frame_stack.valid_range_ids: the plain T-range; once the ring has wrapped the
    lower bound moves up by K-1 (the look-back of the oldest ids would read overwritten slots)."""
    rb, k = self._rb, self._k
    last = rb._get_last_id()
    lo, hi = rb_mod._valid_range_ids(last, rb.max_length, num_steps)
    wrapped = last + 1 > rb.max_length
    if wrapped:
      lo += k - 1
    return lo, hi, wrapped

  def get_next(self, sample_batch_size=None, num_steps=None):
    """Like TFUniformReplayBuffer.get_next with observations rebuilt to [B, T, H, W, K]."""
    rb, k = self._rb, self._k
    B = 1 if sample_batch_size is None else int(sample_batch_size)
    T = 1 if num_steps is None else int(num_steps)
    if T > rb.max_length:
      raise ValueError('num_steps ({}) is bigger than max_length ({}).'.format(T, rb.max_length))
    lo, hi, wrapped = self._valid_range(T)
    if hi <= lo:
      raise rb_mod.InvalidArgumentError(
          'TFUniformReplayBuffer is empty. Make sure to add items before sampling the buffer.')
    dev = rb.device
    with torch.cuda.device(dev):
      ring = table.make_ring([], [], rb.batch_size, rb.max_length, last_id=rb._last_id,
                             ticket=rb._ctrl[2:3])
      ids = torch.empty(B, dtype=torch.int64, device=dev)
      offs = torch.empty(B, dtype=torch.int64, device=dev)
      # The device draw covers [lo_T, last + 2 - span) for `span` steps.  Before the ring wraps the
      # sampleable range is the plain T-range; afterwards it is [lo_T + K - 1, hi_T), which is the
      # (T + K - 1)-range shifted by K - 1.
      span = T + k - 1 if wrapped else T
      _lib.call('b200rl_rb_draw', ctypes.byref(ring), B, span, rb._seed, _lib.ptr(rb._ctrl[0:1]),
                _lib.ptr(ids), _lib.ptr(offs), _lib.stream())
      if wrapped:
        ids = ids + (k - 1)
      # small leaves + ids through the fused sampler on a ring WITHOUT the frame leaf (its rows are
      # only needed inside the stack rebuild below)
      storage = rb._data_table.variables()
      keep = [i for i in range(len(storage)) if i != self._obs_index]
      specs = [rb._flat_specs[i] for i in keep]
      small = table.make_ring([storage[i] for i in keep], specs, rb.batch_size, rb.max_length,
                              id_table=rb._id_table.variables()[0], last_id=rb._last_id,
                              ticket=rb._ctrl[2:3])
      outs = [torch.empty((B, T) + sp.shape, dtype=sp.dtype, device=dev) for sp in specs]
      out_ids = torch.empty((B, T), dtype=torch.int64, device=dev)
      _lib.call('b200rl_rb_sample', ctypes.byref(small), B, T, _lib.ptr(ids), _lib.ptr(offs),
                rb._seed, _lib.ptr(rb._ctrl[0:1]), _lib.ptr_array(outs), _lib.ptr(out_ids), None,
                None, _lib.ptr(rb._ctrl[1:2]), _lib.stream())
      out = torch.empty((B, T, self._h, self._w, k), dtype=torch.uint8, device=dev)
      _lib.call('b200rl_rb_gather_frame_stack', _lib.ptr(storage[self._obs_index]),
                _lib.ptr(storage[self._step_type_index]), self._h * self._w, rb.max_length,
                _lib.ptr(ids), _lib.ptr(offs), B, T, k, _lib.ptr(out), _lib.stream())
      # probability of each drawn window under the range actually sampled from
      prob = np.float32(1.0) / np.float32((hi - lo) * rb.batch_size)
      probs = torch.full((B,), float(prob), dtype=torch.float32, device=dev)
    flat = list(outs)
    flat.insert(self._obs_index, out)
    data = nest.pack_sequence_as(self._data_spec, flat)

    # squeeze like the reference does when sample_batch_size / num_steps are None (:286-306)
    def fix(t, has_time=True):
      if num_steps is None and has_time:
        t = t[:, 0]
      if sample_batch_size is None:
        t = t[0]
      return t
    data = nest.map_structure(fix, data)
    info = rb_mod.BufferInfo(ids=fix(out_ids), probabilities=fix(probs, has_time=False))
    return data, info

  def as_dataset(self, sample_batch_size=None, num_steps=None, **unused):
    while True:
      yield self.get_next(sample_batch_size, num_steps)
