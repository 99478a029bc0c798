"""PPOLearner (tf_agents/train/ppo_learner.py:41-349): minibatch PPO training on cached data.

Reference behaviour kept:
  * constructor checks and messages (:172-192): `shuffle_buffer_size` required with
    `minibatch_size`; `compute_value_and_advantage_in_train` must be False with minibatching;
    `agent.update_normalizers_in_train` must be False (the learner updates them);
  * `run()` (:253-304): first `_update_normalizers` over `num_samples` batches of the
    normalisation dataset (:306-337) and count the frames, then
    `int(num_frames / minibatch_size) * num_epochs / num_replicas` train iterations (or
    `num_samples * num_epochs / num_replicas` full-sequence iterations) through the generic
    `Learner`; raises when that is 0;
  * the training stream (:220-250): `take(num_samples).cache().repeat(num_epochs)` and, for
    minibatches, `[B, T, ...] -> unbatch -> shuffle(S) -> batch(1) -> batch(mb,
    drop_remainder=True)`, one such inner dataset per `Counter()` value; the iterator persists
    across `run()` calls, so minibatches left over from one inner dataset are consumed first
    by the next `run()` exactly as in the reference.

What is different: the cache is the set of device tensors the replay buffer returned (no copy);
the shuffle order comes from libb200rl (`b200rl_shuffle_order`, Philox, host side like tf.data)
and every minibatch is ONE multi-leaf gather launch (`b200rl_rb_read_rows`) into `[mb, 1, ...]`
tensors.  The order itself is unpinned in the reference (tf.data RNG).
"""
import ctypes

import numpy as np
import torch

from agents_b200 import _lib
from agents_b200.replay_buffers import table as table_lib
from agents_b200.specs import tensor_spec
from agents_b200.train import learner
from agents_b200.train.utils import strategy_utils
from agents_b200.utils import nest

_SHUFFLE_SEED_TAG = 0x5050_4F4C_5348_5546


def shuffle_order(n, buffer_size, seed, call):
  """int64 numpy array: emission order of `shuffle(buffer_size)` over a stream of n elements."""
  out = np.empty(int(n), dtype=np.int64)
  _lib.call('b200rl_shuffle_order', int(n), int(buffer_size), int(seed) & 0xFFFFFFFFFFFFFFFF,
            int(call), out.ctypes.data_as(ctypes.c_void_p))
  return out


def _split_sample(sample):
  if isinstance(sample, tuple) and len(sample) == 2 and not hasattr(sample, '_fields'):
    return sample
  return sample, ()


class PPOLearner(object):
  """Manages all the learning details needed when training an PPO agent."""

  def __init__(self, root_dir, train_step, agent, experience_dataset_fn,
               normalization_dataset_fn, num_samples, num_epochs=1, minibatch_size=None,
               shuffle_buffer_size=None, after_train_strategy_step_fn=None, triggers=None,
               checkpoint_interval=100000, summary_interval=1000,
               use_kwargs_in_agent_train=False, strategy=None, seed=0):
    if minibatch_size and shuffle_buffer_size is None:
      raise ValueError('shuffle_buffer_size must be provided if minibatch_size is not None.')
    if minibatch_size and getattr(agent, 'recurrent', False):        # ppo_learner.py:174-177
      raise ValueError('minibatch_size must be set to None for RNN networks.')
    if minibatch_size and agent._compute_value_and_advantage_in_train:
      raise ValueError('agent.compute_value_and_advantage_in_train should be set to False '
                       'when mini batching is used.')
    if agent.update_normalizers_in_train:
      raise ValueError('agent.update_normalizers_in_train should be set to False when '
                       'PPOLearner is used.')
    strategy = strategy or strategy_utils.get_strategy()
    self._agent = agent
    self._minibatch_size = minibatch_size
    self._shuffle_buffer_size = shuffle_buffer_size
    self._num_epochs = num_epochs
    self._experience_dataset_fn = experience_dataset_fn
    self._normalization_dataset_fn = normalization_dataset_fn
    self._num_samples = num_samples
    self._seed = (int(seed) ^ _SHUFFLE_SEED_TAG) + strategy.rank
    self._generic_learner = learner.Learner(
        root_dir, train_step, agent, experience_dataset_fn=None,
        after_train_strategy_step_fn=after_train_strategy_step_fn, triggers=triggers,
        checkpoint_interval=checkpoint_interval, summary_interval=summary_interval,
        use_kwargs_in_agent_train=use_kwargs_in_agent_train, strategy=strategy)
    self.num_replicas = strategy.num_replicas_in_sync
    self._train_iterator = self._train_stream()
    self._normalization_iterator = self._normalization_stream()
    self.num_frames_for_training = 0

  # ---- datasets (ppo_learner.py:206-251) ----------------------------------------------------------
  def _normalization_stream(self):
    while True:                                    # Counter().flat_map(normalization_dataset_fn)
      for sample in self._normalization_dataset_fn():
        yield sample

  def _train_stream(self):
    call = 0
    while True:                                    # Counter().flat_map(_make_dataset)
      it = iter(self._experience_dataset_fn())
      cache = [_split_sample(next(it)) for _ in range(self._num_samples)]   # take().cache()
      if not self._minibatch_size:
        for _ in range(self._num_epochs):          # repeat(num_epochs)
          for sample in cache:
            yield sample
      else:
        for sample in self._minibatches(cache, call):
          yield sample
      call += 1

  def _minibatches(self, cache, call):
    """unbatch -> shuffle -> batch(1) -> batch(mb, drop_remainder=True) over the cached samples."""
    mb = int(self._minibatch_size)
    outer = [tuple(traj.reward.shape[:2]) for traj, _ in cache]

    # sample info that cannot be unbatched over [B, T] (e.g. BufferInfo.probabilities [B]) is
    # dropped; the reference pipeline needs [B, T] info leaves (Reverb SampleInfo) as well
    keep_info = all(all(tuple(l.shape[:2]) == o for l in nest.flatten(info))
                    for (_, info), o in zip(cache, outer))
    if not keep_info:
      cache = [(traj, ()) for traj, _ in cache]
    structure = cache[0]
    flats = [nest.flatten(s) for s in cache]
    leaves = []
    for i in range(len(flats[0])):                 # BatchSquash(2).flatten + unbatch: [B*T, ...]
      parts = [f[i].reshape((-1,) + tuple(f[i].shape[2:])) for f in flats]
      leaves.append((parts[0] if len(parts) == 1 else torch.cat(parts, 0)).contiguous())
    n = int(leaves[0].shape[0])
    dev = leaves[0].device
    stream = n * int(self._num_epochs)
    order = shuffle_order(stream, self._shuffle_buffer_size, self._seed, call) % n
    nb = stream // mb
    if nb == 0:
      return
    rows = torch.from_numpy(order[:nb * mb]).to(dev)
    specs = [tensor_spec.TensorSpec(tuple(l.shape[1:]), l.dtype) for l in leaves]
    ring = table_lib.make_ring(leaves, specs, 1, n)
    with torch.cuda.device(dev):
      for b in range(nb):
        outs = [torch.empty((mb, 1) + s.shape, dtype=s.dtype, device=dev) for s in specs]
        out_ptrs = _lib.ptr_array(outs)
        _lib.call('b200rl_rb_read_rows', ctypes.byref(ring), _lib.ptr(rows[b * mb:(b + 1) * mb]),
                  mb, out_ptrs, None, _lib.stream())
        yield nest.pack_sequence_as(structure, outs)

  # ---- run (ppo_learner.py:253-337) ---------------------------------------------------------------
  def run(self, parallel_iterations=10):
    """Train `num_samples` batches repeating for `num_epochs` of iterations."""
    num_frames = self._update_normalizers(self._normalization_iterator)
    self.num_frames_for_training = num_frames
    if self._minibatch_size:
      num_total_batches = int(num_frames / self._minibatch_size) * self._num_epochs
    else:
      num_total_batches = self._num_samples * self._num_epochs
    iterations = int(num_total_batches / self.num_replicas)
    if iterations == 0:
      raise ValueError(
          'Cannot distribute {} batches across {} replicas. Please increase '
          'PPOLearner.num_samples. See PPOLeaner.num_samples documentation for more '
          'details.'.format(num_total_batches, self.num_replicas))
    return self._generic_learner.run(iterations, self._train_iterator,
                                     parallel_iterations=parallel_iterations)

  def _update_normalizers(self, iterator):
    """Update the normalizers and count the total number of frames (:306-337)."""
    num_frames = 0
    for _ in range(self._num_samples):
      traj, _ = _split_sample(next(iterator))
      self._agent.update_observation_normalizer(traj.observation)
      self._agent.update_reward_normalizer(traj.reward)
      shape = tuple(traj.reward.shape)
      if shape:
        batch = shape[0]
        if len(shape) > 1:
          batch *= shape[1]
      else:
        batch = 1
      num_frames += int(batch)
    return num_frames

  @property
  def train_step_numpy(self):
    return self._generic_learner.train_step_numpy
