"""Distribution strategy for the learner: one process per GPU over torch.distributed.

Stands in for `tf.distribute.MirroredStrategy` as returned by
tf_agents/train/utils/strategy_utils.py:36-61.  The reference's data-parallel scheme (SURVEY.md
§2.3): every replica computes per-example losses divided by the GLOBAL batch
(utils/common.py:1465-1467), gradients are SUM-all-reduced, every replica applies the same
optimiser step and target update, LossInfo is SUM-reduced (train/learner.py:322-336).  Here the
all-reduce is ONE NCCL call on the flat gradient buffer (NVLink/NVSwitch); on CPU test boxes the
same code runs over gloo.
"""
import os

import torch
import torch.distributed as dist


class SingleProcessStrategy(object):
  """The default (no-op) strategy: one replica."""
  num_replicas_in_sync = 1
  rank = 0

  def all_reduce_sum(self, tensor):
    return tensor

  def broadcast(self, tensor, src=0):
    return tensor

  def barrier(self):
    pass

  def shard_range(self, n):
    return 0, n


def configure_nccl_env():
  """Call before `init_process_group('nccl')`.  The gradient all-reduce runs beside the backward
  pass, whose persistent GEMM kernels want every SM: cap NCCL at 8 CTAs (it holds 8 SMs instead of
  16-32; measured on 2 B200s: 5305 -> 5403 steps/s with the dynamic tile scheduler).  A value
  already in the environment wins."""
  os.environ.setdefault('NCCL_MAX_CTAS', '8')


class ProcessGroupStrategy(object):
  """Data parallelism over an initialised torch.distributed process group (nccl or gloo)."""

  def __init__(self, group=None):
    if not dist.is_initialized():
      raise RuntimeError('torch.distributed is not initialised; launch with torchrun or call '
                         'init_process_group first.')
    self._group = group
    self.num_replicas_in_sync = dist.get_world_size(group)
    self.rank = dist.get_rank(group)

  def all_reduce_sum(self, tensor):
    dist.all_reduce(tensor, op=dist.ReduceOp.SUM, group=self._group)
    return tensor

  def broadcast(self, tensor, src=0):
    dist.broadcast(tensor, src=src, group=self._group)
    return tensor

  def barrier(self):
    dist.barrier(group=self._group)

  def shard_range(self, n):
    """Contiguous slice [lo, hi) of `n` buffer segments / batch rows owned by this rank
    (replay storage is already `batch_size` independent segments,
    replay_buffers/tf_uniform_replay_buffer.py:64-94)."""
    w = self.num_replicas_in_sync
    if n % w:
      raise ValueError(f'{n} segments do not divide over {w} replicas.')
    per = n // w
    return self.rank * per, (self.rank + 1) * per


def get_strategy(tpu=None, use_gpu=True):
  """Returns the strategy for this process (strategy_utils.py:36-61): the process-group
  strategy when launched under torchrun with WORLD_SIZE > 1, else the single-replica default."""
  if tpu:
    raise NotImplementedError('TPUStrategy has no CUDA equivalent.')
  if dist.is_initialized() and dist.get_world_size() > 1:
    return ProcessGroupStrategy()
  if int(os.environ.get('WORLD_SIZE', '1')) > 1 and not dist.is_initialized():
    backend = 'nccl' if (use_gpu and torch.cuda.is_available()) else 'gloo'
    if backend == 'nccl':
      torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', '0')))
      configure_nccl_env()
    dist.init_process_group(backend)
    return ProcessGroupStrategy()
  return SingleProcessStrategy()
