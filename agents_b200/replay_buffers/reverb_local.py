"""In-process table server with Reverb's data model, steps resident in HBM.

The reference's `ReverbReplayBuffer` / `Reverb*Observer` classes
(tf_agents/replay_buffers/reverb_replay_buffer.py:37, reverb_utils.py:34,270,509) speak to an
external `dm-reverb` gRPC server through three objects: a *trajectory writer* (`append` one step,
`history[-n:]` column slices, `create_item(table, trajectory, priority)`, `end_episode`), a
*table* (sampler, remover, `max_size`, `max_times_sampled`, rate limiter) and a *client*
(`server_info`, `reset`, `mutate_priorities`).  dm-reverb is not part of the reference repository
(go.mod-style external dependency, un-vendored), so this module restates that model — the format
in which the observers hand data over — as a single-process server whose payload lives on the GPU:

  * every appended step is written ONCE into a row of a device-resident step store
    (`HbmStepStore` over `replay_buffers/table.Table`); items are `(key, priority, rows[])`
    records that reference those rows, so overlapping windows (stride < sequence_length) share
    storage exactly like Reverb chunks do.  Rows are reference counted (writer keep-alive window +
    items) and recycled through a free list;
  * appends are staged in pinned host memory and flushed with one asynchronous H2D copy per leaf
    plus ONE `b200rl_rb_write_rows` launch per flush; a sampled batch of `B` items x `T` steps is
    ONE `b200rl_rb_read_rows` launch over the `[B, T]` row matrix (the same TMA bulk-copy gather
    kernel `TFUniformReplayBuffer.get_next` uses);
  * table bookkeeping (keys, priorities, FIFO order, times-sampled, removal) is host state, as it
    is in the Reverb server; it is kept in dense numpy arrays (priority / key / times-sampled per
    position, a sum tree for the Prioritized selector, a `[position, T]` matrix of step rows while
    all items have one length) so that a whole batch is drawn without python work per sample
    (`Table.sample_rows`: 0.06 ms of host time for 256 items, 19 us per appended step + item).

What is deliberately different from dm-reverb: no network transport (a `Client` is bound to a
`Server` object, or to `'localhost:<port>'` of a server of this process), no blocking rate
limiter (a sample that Reverb would block on raises `RateLimited`; see `Table.sample`), keys are a
counter instead of random 64-bit values, and all columns of an item must cover the same step range.
Not thread-safe (one collect loop, like `table.py:21` of the reference).
"""
import collections
import itertools

import numpy as np

from agents_b200.utils import nest


class RateLimited(RuntimeError):
  """Raised where dm-reverb would block (or time out) on the table's rate limiter."""


# ---- selectors / rate limiters (reverb.selectors.*, reverb.rate_limiters.*) ------------------------
class _Selector(object):
  is_deterministic = False

  def __repr__(self):
    return type(self).__name__ + '()'


class Uniform(_Selector):
  pass


class Fifo(_Selector):
  is_deterministic = True


class Lifo(_Selector):
  is_deterministic = True


class MaxHeap(_Selector):
  is_deterministic = True


class MinHeap(_Selector):
  is_deterministic = True


class Prioritized(_Selector):
  """P(i) = p_i^exponent / sum_j p_j^exponent."""

  def __init__(self, priority_exponent=1.0):
    self.priority_exponent = float(priority_exponent)


class selectors(object):  # pylint: disable=invalid-name
  Uniform, Fifo, Lifo, MaxHeap, MinHeap, Prioritized = Uniform, Fifo, Lifo, MaxHeap, MinHeap, Prioritized


class MinSize(object):
  """Sampling is allowed once the table holds `min_size_to_sample` items."""

  def __init__(self, min_size_to_sample):
    self.min_size_to_sample = int(min_size_to_sample)
    self.max_size = None


class Queue(object):
  """Rate limiter of `Table.queue`: every item is sampled exactly once, inserts stop when full."""

  def __init__(self, size):
    self.min_size_to_sample = 1
    self.max_size = int(size)


class rate_limiters(object):  # pylint: disable=invalid-name
  MinSize, Queue = MinSize, Queue


TableInfo = collections.namedtuple('TableInfo', [
    'name', 'sampler_options', 'remover_options', 'max_size', 'max_times_sampled', 'current_size',
    'num_unique_samples', 'signature', 'rate_limiter_info'])

SampleInfo = collections.namedtuple('SampleInfo', [
    'key', 'probability', 'table_size', 'priority', 'times_sampled'])

ReplaySample = collections.namedtuple('ReplaySample', ['info', 'data'])


class _Item(object):
  """`pos` = index into the table's dense arrays (priority, times sampled, key, rows)."""
  __slots__ = ('key', 'priority', 'rows', 'store', 'pos')

  def __init__(self, key, priority, rows, store):
    self.key, self.priority, self.rows, self.store = key, float(priority), rows, store
    self.pos = -1


class _SumTree(object):
  """Weights of the dense item positions in a complete binary tree (numpy array, leaves in the
  second half): `set` and `find` are O(log n), so a prioritized draw does not scan the table
  (dm-reverb's Prioritized selector keeps the same structure)."""

  def __init__(self, capacity=64):
    self._cap = 1
    while self._cap < capacity:
      self._cap *= 2
    self._t = np.zeros(2 * self._cap, np.float64)

  @property
  def total(self):
    return float(self._t[1])

  def _grow(self, n):
    cap = self._cap
    while cap < n:
      cap *= 2
    leaves = self._t[self._cap:2 * self._cap].copy()
    self._cap = cap
    self._t = np.zeros(2 * cap, np.float64)
    self._t[cap:cap + leaves.shape[0]] = leaves
    for i in range(cap - 1, 0, -1):               # rebuild the inner nodes once per doubling
      self._t[i] = self._t[2 * i] + self._t[2 * i + 1]

  def set(self, pos, weight):
    if pos >= self._cap:
      self._grow(pos + 1)
    i = pos + self._cap
    self._t[i] = weight
    i >>= 1
    while i >= 1:
      self._t[i] = self._t[2 * i] + self._t[2 * i + 1]
      i >>= 1

  def get(self, pos):
    return float(self._t[pos + self._cap]) if pos < self._cap else 0.0

  def find_many(self, u):
    """`find` for a vector of `u`: one numpy step per tree level."""
    i = np.ones(u.shape, np.int64)
    u = u.astype(np.float64).copy()
    cap = self._cap
    while cap > 1:
      left = self._t[2 * i]
      right = u >= left
      u -= np.where(right, left, 0.0)
      i = 2 * i + right
      cap >>= 1
    return i - self._cap

  def find(self, u):
    """Position whose cumulative-weight interval contains `u` in [0, total)."""
    i = 1
    while i < self._cap:
      left = self._t[2 * i]
      if u < left:
        i = 2 * i
      else:
        u -= left
        i = 2 * i + 1
    return i - self._cap


class Table(object):
  """One named collection of items (reverb.Table)."""

  def __init__(self, name, sampler, remover, max_size, rate_limiter, max_times_sampled=0,
               signature=None):
    if max_size < 1:
      raise ValueError('max_size must be >= 1.')
    self.name = name
    self._sampler, self._remover = sampler, remover
    self._max_size = int(max_size)
    self._rate_limiter = rate_limiter
    self._max_times_sampled = int(max_times_sampled)
    self.signature = signature
    self._by_key = collections.OrderedDict()      # insertion order = FIFO order
    self._dense = []                              # positions for O(1) uniform draws
    self._prio = np.zeros(64, np.float64)         # priorities aligned with _dense
    self._times = np.zeros(64, np.int64)          # times sampled, aligned with _dense
    self._keys = np.zeros(64, np.int64)           # item keys, aligned with _dense
    # [position, T] step rows while every item has the same length and row pool (the vectorised
    # batch path of `sample_rows`); None once items of another length / pool were inserted
    self._rows2d = None
    self._rows_ok = True
    self._pool = None
    self._num_unique_samples = 0
    self._server = None
    self._tree = _SumTree() if isinstance(sampler, Prioritized) else None   # p^exponent per position

  @classmethod
  def queue(cls, name, max_size, signature=None):
    """FIFO in, FIFO out, each item delivered once (reverb.Table.queue)."""
    return cls(name, Fifo(), Fifo(), max_size, Queue(max_size), max_times_sampled=1,
               signature=signature)

  # -- introspection --------------------------------------------------------------------------
  @property
  def current_size(self):
    return len(self._dense)

  @property
  def info(self):
    return TableInfo(self.name, self._sampler, self._remover, self._max_size,
                     self._max_times_sampled, self.current_size, self._num_unique_samples,
                     self.signature, self._rate_limiter)

  def can_sample(self, num_samples=1):
    del num_samples  # MinSize / Queue only look at the current size
    return self.current_size >= max(1, self._rate_limiter.min_size_to_sample)

  def can_insert(self, num_inserts=1):
    cap = self._rate_limiter.max_size
    return cap is None or self.current_size + num_inserts <= cap

  # -- mutation -------------------------------------------------------------------------------
  def _set_weight(self, pos, priority):
    self._prio[pos] = priority
    if self._tree is not None:
      self._tree.set(pos, float(np.power(priority, self._sampler.priority_exponent)) if priority > 0
                     else 0.0)

  def _put(self, item):
    pos = item.pos = len(self._dense)
    self._dense.append(item)
    if pos >= self._prio.shape[0]:
      self._prio = np.concatenate([self._prio, np.zeros_like(self._prio)])
      self._times = np.concatenate([self._times, np.zeros_like(self._times)])
      self._keys = np.concatenate([self._keys, np.zeros_like(self._keys)])
      if self._rows2d is not None:
        self._rows2d = np.concatenate([self._rows2d, np.zeros_like(self._rows2d)])
    self._set_weight(pos, item.priority)
    self._times[pos] = 0
    self._keys[pos] = item.key
    self._by_key[item.key] = item
    # the [position, T] row matrix of the vectorised batch path
    if self._rows_ok:
      if self._rows2d is None and self._pool is None:
        self._pool = item.store
        self._rows2d = np.zeros((self._prio.shape[0], item.rows.shape[0]), np.int64)
      if item.store is not self._pool or item.rows.shape[0] != self._rows2d.shape[1]:
        self._rows_ok, self._rows2d = False, None       # mixed lengths / pools: generic path only
      else:
        self._rows2d[pos] = item.rows

  def _drop(self, item):
    last = self._dense.pop()
    n = len(self._dense)
    self._set_weight(n, 0.0)                      # the vacated last position
    if last is not item:
      pos = item.pos
      self._dense[pos] = last
      last.pos = pos
      self._set_weight(pos, last.priority)
      self._times[pos] = self._times[n]
      self._keys[pos] = self._keys[n]
      if self._rows2d is not None:
        self._rows2d[pos] = self._rows2d[n]
    del self._by_key[item.key]
    item.store.release(item.rows)
    if not self._dense and not self._rows_ok:     # an emptied table may take the fast path again
      self._rows_ok, self._rows2d, self._pool = True, None, None

  def _victim(self):
    r = self._remover
    if isinstance(r, Fifo):
      return next(iter(self._by_key.values()))
    if isinstance(r, Lifo):
      return next(reversed(self._by_key.values()))
    n = len(self._dense)
    if isinstance(r, MinHeap):
      return self._dense[int(np.argmin(self._prio[:n]))]
    if isinstance(r, MaxHeap):
      return self._dense[int(np.argmax(self._prio[:n]))]
    if isinstance(r, Uniform):
      return self._dense[int(self._server.rng.integers(n))]
    raise ValueError('Unsupported remover {!r}'.format(r))

  def insert(self, key, priority, rows, store):
    if not self.can_insert(1):
      raise RateLimited(
          'Table {!r} is a queue of {} items and is full; dm-reverb would block the writer until '
          'an item is sampled.'.format(self.name, self._rate_limiter.max_size))
    store.retain(rows)
    self._put(_Item(key, priority, rows, store))
    while len(self._dense) > self._max_size:     # the remover also sees the new item, as in Reverb
      self._drop(self._victim())

  def reset(self):
    for item in list(self._dense):
      self._drop(item)

  def mutate(self, updates=None, deletes=None):
    for key, p in (updates or {}).items():
      item = self._by_key.get(int(key))
      if item is not None:                         # unknown keys are ignored, as in Reverb
        item.priority = float(p)
        self._set_weight(item.pos, item.priority)
    for key in deletes or ():
      item = self._by_key.get(int(key))
      if item is not None:
        self._drop(item)

  # -- sampling -------------------------------------------------------------------------------
  def _pick(self):
    """One draw of the sampler: (item, probability)."""
    s, n = self._sampler, len(self._dense)
    if isinstance(s, Uniform):
      return self._dense[int(self._server.rng.integers(n))], 1.0 / n
    if isinstance(s, Fifo):
      return next(iter(self._by_key.values())), 1.0
    if isinstance(s, Lifo):
      return next(reversed(self._by_key.values())), 1.0
    if isinstance(s, MaxHeap):
      return self._dense[int(np.argmax(self._prio[:n]))], 1.0
    if isinstance(s, MinHeap):
      return self._dense[int(np.argmin(self._prio[:n]))], 1.0
    if isinstance(s, Prioritized):
      total = self._tree.total
      if not total > 0:                            # all priorities zero: uniform, like Reverb
        return self._dense[int(self._server.rng.integers(n))], 1.0 / n
      i = self._tree.find(self._server.rng.random() * total)
      if i >= n or not self._tree.get(i) > 0:      # rounding at an interval edge: nearest live item
        i = int(np.argmax(self._prio[:n] > 0))
      return self._dense[i], self._tree.get(i) / total
    raise ValueError('Unsupported sampler {!r}'.format(s))

  def sample(self, num_samples=1):
    """`num_samples` sequential draws -> list of (item, SampleInfo).

    An item that reaches `max_times_sampled` is removed before the next draw (its rows stay
    alive until `release_samples` is called with the returned list, so the caller can still read
    them).  Raises `RateLimited` where dm-reverb would block."""
    out = []
    for _ in range(num_samples):
      if not self.can_sample(1):
        if out:
          self.release_samples(out)
        raise RateLimited(
            'Table {!r} holds {} item(s); its rate limiter needs {} to sample.'.format(
                self.name, self.current_size, max(1, self._rate_limiter.min_size_to_sample)))
      item, prob = self._pick()
      if self._times[item.pos] == 0:
        self._num_unique_samples += 1
      self._times[item.pos] += 1
      times = int(self._times[item.pos])
      info = SampleInfo(item.key, prob, self.current_size, item.priority, times)
      item.store.retain(item.rows)                 # pinned for the reader
      out.append((item, info))
      if self._max_times_sampled > 0 and times >= self._max_times_sampled:
        self._drop(item)
    return out

  def sample_rows(self, num_samples):
    """Vectorised batch draw: `(pool, rows[num_samples, T], SampleInfo of arrays)`, or None when the
    table needs the item-by-item path (`max_times_sampled`, items of different lengths or row
    pools, a sampler other than Uniform / Prioritized).  No python work per sample: positions are
    drawn at once (sum-tree descent over the whole vector for Prioritized) and the step rows come
    from the dense `[position, T]` matrix, ready for ONE gather launch."""
    n = len(self._dense)
    if (self._max_times_sampled > 0 or self._rows2d is None or
        not isinstance(self._sampler, (Uniform, Prioritized))):
      return None
    if not self.can_sample(1):
      raise RateLimited(
          'Table {!r} holds {} item(s); its rate limiter needs {} to sample.'.format(
              self.name, n, max(1, self._rate_limiter.min_size_to_sample)))
    rng = self._server.rng
    total = self._tree.total if self._tree is not None else 0.0
    if self._tree is not None and total > 0:
      pos = self._tree.find_many(rng.random(num_samples) * total)
      w = self._tree._t[self._tree._cap + np.minimum(pos, n - 1)]
      bad = (pos >= n) | ~(w > 0)                  # rounding at an interval edge
      if bad.any():
        pos = np.where(bad, int(np.argmax(self._prio[:n] > 0)), pos)
        w = self._tree._t[self._tree._cap + pos]
      prob = w / total
    else:
      pos = rng.integers(n, size=num_samples)
      prob = np.full(num_samples, 1.0 / n)
    fresh = np.unique(pos[self._times[pos] == 0])
    self._num_unique_samples += int(fresh.size)
    np.add.at(self._times, pos, 1)
    info = SampleInfo(self._keys[pos].copy(), prob, np.full(num_samples, n, np.int64),
                      self._prio[pos].copy(), self._times[pos].copy())
    return self._pool, self._rows2d[pos], info

  @staticmethod
  def release_samples(samples):
    for item, _ in samples:
      item.store.release(item.rows)


# ---- step store --------------------------------------------------------------------------------------
class HbmStepStore(object):
  """Rows of steps in HBM: one `[capacity, *leaf.shape]` CUDA tensor per leaf (`Table`).

  `staging()` hands out pinned host arrays `[stage, *leaf.shape]`; `commit(rows, n)` uploads the
  first `n` staged steps (async H2D per leaf) and scatters them with one `b200rl_rb_write_rows`
  launch; two staging sets alternate, an event per set guards the reuse of its pinned memory.
  `read(rows)` gathers `rows.shape + leaf.shape` tensors with one `b200rl_rb_read_rows` launch."""

  def __init__(self, flat_specs, capacity, device='cuda', stage=256):
    import torch
    from agents_b200.replay_buffers import table as table_lib
    self._torch = torch
    self._specs = list(flat_specs)
    self._device = torch.device(device)
    if self._device.type != 'cuda':
      raise ValueError('HbmStepStore needs a CUDA device (there is no host fallback).')
    self._table_lib = table_lib
    self._table = table_lib.Table(self._specs, capacity, device=self._device)
    self.capacity = int(capacity)
    self.stage = int(stage)
    self._pinned = [[torch.empty((self.stage,) + s.shape, dtype=s.dtype).pin_memory()
                     for s in self._specs] for _ in range(2)]
    self._views = [[p.numpy() for p in ps] for ps in self._pinned]
    self._done = [torch.cuda.Event(), torch.cuda.Event()]
    self._used = [False, False]
    self._slot = 0

  def staging(self):
    if self._used[self._slot]:
      self._done[self._slot].synchronize()
      self._used[self._slot] = False
    return self._views[self._slot]

  def commit(self, rows, n):
    torch = self._torch
    slot = self._slot
    with torch.cuda.device(self._device):
      values = [p[:n].to(self._device, non_blocking=True) for p in self._pinned[slot]]
      self._table.write(torch.from_numpy(np.ascontiguousarray(rows[:n])), values)
      self._done[slot].record()
    self._used[slot] = True
    self._slot ^= 1

  def read(self, rows):
    with self._torch.cuda.device(self._device):
      return self._table.read(self._torch.from_numpy(np.ascontiguousarray(rows)))

  def grow(self, capacity):
    old = self._table.variables()
    new = self._table_lib.Table(self._specs, capacity, device=self._device)
    for dst, src in zip(new.variables(), old):
      dst[:src.shape[0]].copy_(src)
    self._table, self.capacity = new, int(capacity)


class _RowPool(object):
  """Row allocation, reference counts and append staging in front of a step store."""

  def __init__(self, store, specs):
    self._store = store
    self.store_specs = specs
    self._refs = np.zeros(store.capacity, np.int32)
    self._free = list(range(store.capacity - 1, -1, -1))
    self._pending_rows = np.zeros(store.stage, np.int64)
    self._n_pending = 0
    self._pending = set()         # rows staged but not yet written
    self._deferred = []           # rows that died while staged: reusable after the flush

  @property
  def store(self):
    return self._store

  def append(self, flat_step):
    """Stages one step, returns its row (holding one reference for the caller)."""
    if not self._free:
      self.flush()
      old = self._store.capacity
      self._store.grow(2 * old)
      self._refs = np.concatenate([self._refs, np.zeros(old, np.int32)])
      self._free = list(range(2 * old - 1, old - 1, -1))
    row = self._free.pop()
    self._refs[row] = 1
    bufs = self._store.staging()
    i = self._n_pending
    for buf, leaf in zip(bufs, flat_step):
      buf[i] = leaf
    self._pending_rows[i] = row
    self._pending.add(row)
    self._n_pending = i + 1
    if self._n_pending == self._store.stage:
      self.flush()
    return row

  def flush(self):
    if self._n_pending:
      self._store.commit(self._pending_rows, self._n_pending)
      self._n_pending = 0
      self._pending.clear()
      self._free.extend(self._deferred)
      del self._deferred[:]

  def retain(self, rows):
    np.add.at(self._refs, rows, 1)

  def release(self, rows):
    np.subtract.at(self._refs, rows, 1)
    rows = np.unique(rows)
    dead = rows[self._refs[rows] == 0]
    for r in dead:
      # a row that dies while still staged must not be handed out again before the flush: one
      # write launch would then carry two values for the same row
      r = int(r)
      (self._deferred if r in self._pending else self._free).append(r)

  def read(self, rows):
    self.flush()
    return self._store.read(rows)

  def live_rows(self):
    return int(np.count_nonzero(self._refs))


# ---- writer ----------------------------------------------------------------------------------------
class _Column(object):
  """`writer.history` leaf: slicing yields a reference to a range of the episode's steps."""

  def __init__(self, writer, leaf_index):
    self._writer, self._leaf = writer, leaf_index

  def __len__(self):
    return len(self._writer._episode_rows)

  def __getitem__(self, idx):
    n = len(self)
    if isinstance(idx, slice):
      start, stop, step = idx.indices(n)
      if step != 1:
        raise ValueError('history slices must be contiguous.')
    else:
      i = idx + n if idx < 0 else idx
      if not 0 <= i < n:
        raise IndexError('history index out of range')
      start, stop = i, i + 1
    return _ColumnRef(self._writer, self._leaf, start, max(start, stop))


class _ColumnRef(object):
  """Steps [start, stop) of one column of a writer's episode (a nest LEAF, hence not a tuple)."""
  __slots__ = ('writer', 'leaf', 'start', 'stop')

  def __init__(self, writer, leaf, start, stop):
    self.writer, self.leaf, self.start, self.stop = writer, leaf, start, stop

  def __len__(self):
    return self.stop - self.start


class TrajectoryWriter(object):
  """reverb.TrajectoryWriter: append steps, reference windows of them in items."""

  def __init__(self, server, num_keep_alive_refs, validate_items=True):
    if num_keep_alive_refs < 1:
      raise ValueError('num_keep_alive_refs must be >= 1.')
    self._server = server
    self._keep = int(num_keep_alive_refs)
    self._validate = validate_items
    self._pool = None
    self._structure = None
    self._history = None
    self._episode_rows = []       # row of every step of the current episode
    self._released_upto = 0       # steps [0, _released_upto) fell out of the keep-alive window
    self._closed = False

  def __enter__(self):
    return self

  def __exit__(self, *exc):
    self.close()

  @property
  def history(self):
    if self._history is None:
      raise RuntimeError('history is not available before the first append.')
    return self._history

  @property
  def episode_steps(self):
    return len(self._episode_rows)

  def append(self, data):
    if self._closed:
      raise RuntimeError('Calling method append after close has been called')
    flat = [np.asarray(x) for x in nest.flatten(data)]
    if self._pool is None:
      self._pool = self._server._pool_for(data, flat)
      self._structure = data
      self._history = nest.pack_sequence_as(
          data, [_Column(self, i) for i in range(len(flat))]) if nest.is_nested(data) else _Column(self, 0)
    elif len(flat) != len(self._pool.store_specs):
      raise ValueError('append: the step does not match the structure of earlier steps.')
    for a, spec in zip(flat, self._pool.store_specs):
      if tuple(a.shape) != tuple(spec.shape):      # numpy would silently broadcast a smaller leaf
        raise ValueError('append: leaf {!r} has shape {}, the step store holds {}.'.format(
            spec.name, tuple(a.shape), tuple(spec.shape)))
    self._episode_rows.append(self._pool.append(flat))
    # keep-alive window: the writer's own reference on steps older than `keep` is dropped
    limit = len(self._episode_rows) - self._keep
    while self._released_upto < limit:
      self._pool.release(np.asarray([self._episode_rows[self._released_upto]], np.int64))
      self._released_upto += 1

  def create_item(self, table, priority, trajectory):
    if self._closed:
      raise RuntimeError('Calling method create_item after close has been called')
    refs = nest.flatten(trajectory)
    if not refs or not all(isinstance(r, _ColumnRef) for r in refs):
      raise ValueError('trajectory must be a (nest of) slices of writer.history.')
    start, stop = refs[0].start, refs[0].stop
    for r in refs:
      if r.writer is not self or (r.start, r.stop) != (start, stop):
        raise ValueError('All columns of an item must reference the same steps of this writer '
                         '(got [{}, {}) and [{}, {})).'.format(start, stop, r.start, r.stop))
    if stop <= start:
      raise ValueError('An item must reference at least one step.')
    if start < self._released_upto:
      raise ValueError(
          'Item references step {} of the episode, but only the last {} steps are kept alive '
          '(num_keep_alive_refs).'.format(start, self._keep))
    rows = np.asarray(self._episode_rows[start:stop], np.int64)
    self._server._table(table).insert(self._server._new_key(), priority, rows, self._pool)

  def end_episode(self, clear_buffers=True, timeout_ms=None):
    del timeout_ms
    if clear_buffers and self._pool is not None:
      live = self._episode_rows[self._released_upto:]
      if live:
        self._pool.release(np.asarray(live, np.int64))
      self._episode_rows = []
      self._released_upto = 0

  def flush(self, block_until_num_items=0, timeout_ms=None):
    del block_until_num_items, timeout_ms
    if self._pool is not None:
      self._pool.flush()

  def close(self):
    if not self._closed:
      self.end_episode()
      self.flush()
      self._closed = True


# ---- server / client -------------------------------------------------------------------------------
_SERVERS = {}
_PORTS = itertools.count(41000)


class Server(object):
  """Holds the tables and the HBM step stores (reverb.Server)."""

  def __init__(self, tables, port=None, seed=0, device='cuda', initial_step_capacity=4096,
               stage_steps=256, store_factory=None):
    self._tables = collections.OrderedDict()
    for t in tables:
      if t.name in self._tables:
        raise ValueError('Duplicate table name {!r}.'.format(t.name))
      t._server = self
      self._tables[t.name] = t
    self.port = next(_PORTS) if port is None else int(port)
    _SERVERS[self.port] = self
    self.rng = np.random.Generator(np.random.Philox(seed))
    self._device = device
    self._cap0, self._stage = int(initial_step_capacity), int(stage_steps)
    self._store_factory = store_factory or (
        lambda specs, cap: HbmStepStore(specs, cap, device=self._device, stage=self._stage))
    self._pools = {}
    self._keys = itertools.count(1)

  def _new_key(self):
    return next(self._keys)

  def _table(self, name):
    try:
      return self._tables[name]
    except KeyError:
      raise ValueError('Unknown table {!r}; the server has {}.'.format(name, list(self._tables)))

  def _pool_for(self, structure, flat):
    """The row pool of steps shaped like `flat` (created on first use)."""
    from agents_b200.specs import tensor_spec
    sig_nest = nest.map_structure(lambda _: 0, structure) if nest.is_nested(structure) else 0
    dtypes = self._signature_dtypes(len(flat))
    leaves = []
    for i, a in enumerate(flat):
      dt = dtypes[i] if dtypes is not None else (np.dtype(np.float32) if a.dtype == np.float64 else a.dtype)
      leaves.append((np.dtype(dt).str, tuple(a.shape)))
    sig = (repr(sig_nest), tuple(leaves))
    pool = self._pools.get(sig)
    if pool is None:
      specs = [tensor_spec.TensorSpec(shape, np.dtype(dt), 'leaf%d' % i)
               for i, (dt, shape) in enumerate(leaves)]
      pool = _RowPool(self._store_factory(specs, self._cap0), specs)
      self._pools[sig] = pool
    return pool

  def _signature_dtypes(self, n_leaves):
    """Leaf dtypes of the first table signature with `n_leaves` leaves (python scalars appended
    before any typed array would otherwise default to int64 / float32)."""
    from agents_b200.specs import tensor_spec
    for t in self._tables.values():
      if t.signature is not None:
        flat = nest.flatten(t.signature)
        if len(flat) == n_leaves:
          return [tensor_spec.as_numpy_dtype(s.dtype) for s in flat]
    return None

  def localhost_client(self):
    return Client(self)

  def stop(self):
    _SERVERS.pop(self.port, None)

  def live_rows(self):
    return sum(p.live_rows() for p in self._pools.values())


class Client(object):
  """reverb.Client bound to a `Server` of this process."""

  def __init__(self, server_or_address):
    if isinstance(server_or_address, Server):
      self._server = server_or_address
    else:
      host, _, port = str(server_or_address).rpartition(':')
      srv = _SERVERS.get(int(port)) if port.isdigit() else None
      if srv is None or host not in ('localhost', '127.0.0.1', ''):
        raise NotImplementedError(
            'No network transport: {!r} does not name a reverb_local.Server of this process.'.format(
                server_or_address))
      self._server = srv

  @property
  def server(self):
    return self._server

  def trajectory_writer(self, num_keep_alive_refs, validate_items=True):
    return TrajectoryWriter(self._server, num_keep_alive_refs, validate_items)

  def server_info(self, timeout=None):
    del timeout
    return {name: t.info for name, t in self._server._tables.items()}

  def reset(self, table):
    self._server._table(table).reset()

  def mutate_priorities(self, table, updates=None, deletes=None):
    self._server._table(table).mutate(updates, deletes)

  def update_priorities(self, table, keys, priorities):
    """reverb.TFClient.update_priorities: parallel arrays of keys and new priorities."""
    self.mutate_priorities(table, updates={int(k): float(p) for k, p in zip(keys, priorities)})

  def sample(self, table, num_samples=1):
    """Yields `ReplaySample(info, data)` with `data` a nest of `[T, ...]` device tensors."""
    tbl = self._server._table(table)
    for _ in range(num_samples):
      picked = tbl.sample(1)
      try:
        yield read_items(picked)[0]
      finally:
        Table.release_samples(picked)


def read_items(samples, structure=None):
  """[(item, info)] -> [ReplaySample]: one gather launch per item (variable lengths allowed)."""
  out = []
  for item, info in samples:
    flat = item.store.read(item.rows)
    data = flat if structure is None else nest.pack_sequence_as(structure, flat)
    out.append(ReplaySample(info, data))
  return out
