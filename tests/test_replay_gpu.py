"""TFUniformReplayBuffer on the GPU: reference-test replays through the product API and
bit-exact parity against the oracle (oracle/replay.py) on the same seeded inputs."""
import numpy as np
import pytest
import torch

from agents_b200.replay_buffers import table
from agents_b200.replay_buffers import tf_uniform_replay_buffer as rb_mod
from agents_b200.specs import tensor_spec
from agents_b200.trajectories import trajectory
from oracle import replay as oreplay

pytestmark = pytest.mark.gpu


def _scalar_rb(cuda, batch_size, max_length=1000, dtype=torch.int64, **kw):
  return rb_mod.TFUniformReplayBuffer(tensor_spec.TensorSpec([], dtype, 'action'),
                                      batch_size=batch_size, max_length=max_length, device=cuda,
                                      **kw)


# ---- replays of replay_buffers/tf_uniform_replay_buffer_test.py ----------------------------
@pytest.mark.parametrize('batch_size', [1, 5])
def test_gather_all(cuda, batch_size):  # :313-333
  rb = _scalar_rb(cuda, batch_size)
  for i in range(10):
    rb.add_batch(torch.arange(i, i + batch_size, dtype=torch.int64, device=cuda))
  assert rb.gather_all().cpu().tolist() == [list(range(i, i + 10)) for i in range(batch_size)]


@pytest.mark.parametrize('batch_size', [1, 5])
def test_gather_all_over_capacity(cuda, batch_size):  # :339-361
  rb = _scalar_rb(cuda, batch_size, max_length=10)
  for i in range(15):
    rb.add_batch(torch.arange(0, batch_size * 100, 100, dtype=torch.int64, device=cuda) + i)
  want = [list(range(5 + x * 100, 15 + x * 100)) for x in range(batch_size)]
  assert rb.gather_all().cpu().tolist() == want


@pytest.mark.parametrize('batch_size', [1, 5])
def test_gather_all_empty(cuda, batch_size):  # :367-378
  rb = _scalar_rb(cuda, batch_size, dtype=torch.int32)
  assert tuple(rb.gather_all().shape) == (batch_size, 0)


def test_empty_sample_raises(cuda):  # :96-109
  rb = _scalar_rb(cuda, 1, max_length=10)
  with pytest.raises(rb_mod.InvalidArgumentError, match='TFUniformReplayBuffer is empty'):
    rb.get_next()
  rb.add_batch(torch.zeros(1, dtype=torch.int64, device=cuda))
  with pytest.raises(rb_mod.InvalidArgumentError):
    rb.get_next(num_steps=2)   # one item cannot give a 2-step window


@pytest.mark.parametrize('batch_size', [1, 5])
def test_probabilities(cuda, batch_size):  # :384-447
  rb = _scalar_rb(cuda, batch_size, max_length=3, dtype=torch.int32)
  for i in range(1, 5):
    rb.add_batch(torch.full((batch_size,), i, dtype=torch.int32, device=cuda))
    _, info = rb.get_next()
    want = 1.0 / min(i * batch_size, 3 * batch_size)
    np.testing.assert_allclose(info.probabilities.item(), want, rtol=1e-6)
    _, info = rb.get_next(sample_batch_size=2)
    np.testing.assert_allclose(info.probabilities.cpu().numpy(), [want] * 2, rtol=1e-6)


def test_multi_step_windows(cuda):  # :227-307
  rb = _scalar_rb(cuda, 1, max_length=10)
  for i in range(25):
    rb.add_batch(torch.tensor([i % 10], dtype=torch.int64, device=cuda))
  for _ in range(20):
    steps, _ = rb.get_next(sample_batch_size=3, num_steps=2)
    s = steps.cpu().numpy()
    assert s.shape == (3, 2) and ((s[:, 0] + 1) % 10 == s[:, 1]).all()
  steps, info = rb.get_next(num_steps=2)                  # unbatched, stacked -> [T]
  assert tuple(steps.shape) == (2,) and tuple(info.ids.shape) == (2,)
  steps, info = rb.get_next(sample_batch_size=4, num_steps=2, time_stacked=False)
  assert isinstance(steps, tuple) and len(steps) == 2 and tuple(steps[0].shape) == (4,)
  assert (((steps[0] + 1) % 10) == steps[1]).all()


def test_num_frames_and_clear(cuda):  # :673-699, :129-221
  rb = _scalar_rb(cuda, 5, max_length=4, dtype=torch.int32)
  assert int(rb.num_frames()) == 0
  for i in range(1, 7):
    rb.add_batch(torch.zeros(5, dtype=torch.int32, device=cuda))
    assert int(rb.num_frames()) == min(i * 5, 20)
  rb.clear()
  assert int(rb.num_frames()) == 0 and int(rb._last_id.item()) == -1
  with pytest.raises(rb_mod.InvalidArgumentError):
    rb.get_next()
  rb.add_batch(torch.full((5,), 9, dtype=torch.int32, device=cuda))
  rb.clear(clear_all_variables=True)
  assert int(rb.variables()[0].abs().sum().item()) == 0


def _collect(cuda, max_length, bbs, num_adds, sample_batch_size, num_steps=None):
  rb = _scalar_rb(cuda, bbs, max_length=max_length, dtype=torch.int32)
  ds = rb.as_dataset(single_deterministic_pass=True, sample_batch_size=sample_batch_size,
                     num_steps=num_steps)
  for ix in range(num_adds):
    rb.add_batch(10 * torch.arange(bbs, dtype=torch.int32, device=cuda) + ix)
  return np.asarray([d.cpu().numpy() for d, _ in ds])


def test_deterministic_pass_datasets(cuda):  # :548-641
  for bbs in (1, 5):
    got = _collect(cuda, 3, bbs, 3, None)
    assert got.tolist() == np.hstack([np.arange(3) + 10 * i for i in range(bbs)]).tolist()
    got = _collect(cuda, 3, bbs, 3, bbs)
    assert got.tolist() == np.vstack([10 * np.arange(bbs) + i for i in range(3)]).tolist()
  got = _collect(cuda, 4, 5, 4, None, num_steps=2)
  assert got.tolist() == [[0, 1], [2, 3], [10, 11], [12, 13], [20, 21], [22, 23], [30, 31],
                          [32, 33], [40, 41], [42, 43]]
  got = _collect(cuda, 4, 6, 4, 3, num_steps=2)
  assert got.tolist() == [[[0, 1], [10, 11], [20, 21]], [[2, 3], [12, 13], [22, 23]],
                          [[30, 31], [40, 41], [50, 51]], [[32, 33], [42, 43], [52, 53]]]


def test_deterministic_pass_value_errors(cuda):  # :643-667
  rb = _scalar_rb(cuda, 2, max_length=3, dataset_drop_remainder=True)
  with pytest.raises(ValueError, match='ALL data will be dropped'):
    rb.as_dataset(single_deterministic_pass=True, sample_batch_size=3)
  with pytest.raises(ValueError, match='ALL data will be dropped'):
    rb.as_dataset(single_deterministic_pass=True, num_steps=4)


def test_add_batch_shape_errors(cuda):
  rb = _scalar_rb(cuda, 3)
  with pytest.raises(ValueError):
    rb.add_batch(torch.zeros(2, dtype=torch.int64, device=cuda))
  with pytest.raises(ValueError):
    rb.add_batch((torch.zeros(3, dtype=torch.int64, device=cuda),) * 2)


# ---- parity with the oracle ---------------------------------------------------------------------
def _traj_spec(obs_shape, obs_dtype, act_dtype=torch.int32, act_shape=()):
  return trajectory.Trajectory(
      step_type=tensor_spec.TensorSpec([], torch.int32, 'step_type'),
      observation=tensor_spec.TensorSpec(obs_shape, obs_dtype, 'observation'),
      action=tensor_spec.TensorSpec(act_shape, act_dtype, 'action'),
      policy_info=(),
      next_step_type=tensor_spec.TensorSpec([], torch.int32, 'next_step_type'),
      reward=tensor_spec.TensorSpec([], torch.float32, 'reward'),
      discount=tensor_spec.TensorSpec([], torch.float32, 'discount'))


def _random_items(rng, spec_flat, B):
  items = []
  for s in spec_flat:
    npdt = tensor_spec.as_numpy_dtype(s.dtype)
    if npdt == np.uint8:
      items.append(rng.randint(0, 256, size=(B,) + s.shape).astype(np.uint8))
    elif np.issubdtype(npdt, np.integer):
      items.append(rng.randint(0, 3, size=(B,) + s.shape).astype(npdt))
    else:
      items.append(rng.rand(*((B,) + s.shape)).astype(npdt))
  return items


def _pair(cuda, spec, B_env, L, seed=7):
  from agents_b200.utils import nest
  flat = nest.flatten(spec)
  rb = rb_mod.TFUniformReplayBuffer(spec, batch_size=B_env, max_length=L, device=cuda, seed=seed)
  orc = oreplay.UniformReplayOracle([s.shape for s in flat],
                                    [tensor_spec.as_numpy_dtype(s.dtype) for s in flat], B_env, L,
                                    seed=seed)
  return rb, orc, flat


def _fill(cuda, rb, orc, flat, spec, n, rng):
  from agents_b200.utils import nest
  for _ in range(n):
    items = _random_items(rng, flat, orc.batch_size)
    orc.add_batch(items)
    rb.add_batch(nest.pack_sequence_as(spec, [torch.as_tensor(x, device=cuda) for x in items]))


@pytest.mark.parametrize('obs_shape,obs_dtype,B_env,L,adds', [
    ((84, 84, 4), torch.uint8, 3, 8, 13),     # Atari row: one big leaf (2 pieces) + smalls; wraps
    ((17,), torch.float32, 5, 16, 9),         # MuJoCo row: all-small path, not full
    ((1000,), torch.uint8, 2, 4, 6),          # 1000 B leaf: 8 B vectors
    ((3, 7), torch.uint8, 2, 4, 5),           # 21 B leaf: byte path
    ((40000,), torch.uint8, 2, 3, 4),         # 3 pieces
])
def test_sample_parity_bit_exact(cuda, obs_shape, obs_dtype, B_env, L, adds):
  from agents_b200.utils import nest
  spec = _traj_spec(obs_shape, obs_dtype)
  rb, orc, flat = _pair(cuda, spec, B_env, L)
  rng = np.random.RandomState(0)
  _fill(cuda, rb, orc, flat, spec, adds, rng)
  torch.cuda.synchronize()
  assert int(rb._last_id.item()) == orc.last_id
  np.testing.assert_array_equal(rb._id_table.variables()[0].cpu().numpy(), orc.id_table)
  for st, ot in zip(rb._data_table.variables(), orc.storage):
    np.testing.assert_array_equal(st.cpu().numpy(), ot)
  for (B, T) in [(4, 1), (7, 2), (16, 3)]:
    if T > min(L, adds):
      continue
    want, want_ids, want_rows, want_prob = orc.get_next(B, T)       # Philox draw #k on both
    data, info = rb.get_next(sample_batch_size=B, num_steps=T)
    got = nest.flatten(data)
    for g, w in zip(got, want):
      np.testing.assert_array_equal(g.cpu().numpy(), w)
    np.testing.assert_array_equal(info.ids.cpu().numpy(), want_ids)
    np.testing.assert_array_equal(info.probabilities.cpu().numpy(), want_prob)
  # oracle mode: externally supplied draws
  lo, hi = oreplay.valid_range_ids(orc.last_id, L, 2)
  ids = rng.randint(lo, hi, size=5).astype(np.int64)
  offs = rng.randint(0, B_env, size=5).astype(np.int64)
  want, want_ids, _, _ = orc.get_next(5, 2, ids=ids, batch_offsets=offs)
  data, info = rb.get_next(sample_batch_size=5, num_steps=2, ids=ids, batch_offsets=offs)
  for g, w in zip(nest.flatten(data), want):
    np.testing.assert_array_equal(g.cpu().numpy(), w)
  np.testing.assert_array_equal(info.ids.cpu().numpy(), want_ids)
  # gather_all
  for g, w in zip(nest.flatten(rb.gather_all()), orc.gather_all()):
    np.testing.assert_array_equal(g.cpu().numpy(), w)


def test_rng_call_counter_advances_like_oracle(cuda):
  spec = tensor_spec.TensorSpec([], torch.int64, 'x')
  rb, orc, flat = _pair(cuda, spec, 4, 32, seed=123)
  for i in range(40):
    v = np.arange(4, dtype=np.int64) * 1000 + i
    orc.add_batch([v])
    rb.add_batch(torch.as_tensor(v, device=cuda))
  seen = []
  for _ in range(5):
    (want,), _, _, _ = orc.get_next(64, 2)
    got, _ = rb.get_next(sample_batch_size=64, num_steps=2)
    np.testing.assert_array_equal(got.cpu().numpy(), want)
    seen.append(want[:, 0].tolist())
  assert len({tuple(s) for s in seen}) == 5      # every call draws fresh ids
  assert int(rb._ctrl[0].item()) == orc.rng_call == 5
  assert int(rb._ctrl[2].item()) == 0            # ticket returned to 0


def test_table_read_write(cuda):  # replay_buffers/table_test.py semantics
  spec = (tensor_spec.TensorSpec([2], torch.float32, 'a'), tensor_spec.TensorSpec([], torch.int32, 'b'))
  t = table.Table(spec, capacity=6, device=cuda)
  t.write([1, 4], (torch.tensor([[1., 2.], [3., 4.]], device=cuda), torch.tensor([7, 9], device=cuda, dtype=torch.int32)))
  a, b = t.read([4, 1, 0])
  assert a.cpu().tolist() == [[3., 4.], [1., 2.], [0., 0.]] and b.cpu().tolist() == [9, 7, 0]
  a1 = t.read(4, slots=t.slots[0])
  assert a1.cpu().tolist() == [3., 4.]
  (bb,) = t.read(torch.tensor([[1, 4]], device=cuda), slots=(t.slots[1],))
  assert bb.cpu().tolist() == [[7, 9]]


def test_custom_table_fn_uses_generic_path(cuda):
  class MyTable(table.Table):
    pass

  class Wrapper(object):            # not a table.Table instance: forces the generic path
    def __init__(self, spec, capacity, device='cuda'):
      self._t = table.Table(spec, capacity, device=device)
    def __getattr__(self, n):
      return getattr(self._t, n)

  spec = tensor_spec.TensorSpec([], torch.int64, 'x')
  rb = rb_mod.TFUniformReplayBuffer(spec, batch_size=2, max_length=10, device=cuda, table_fn=Wrapper,
                                    seed=5)
  orc = oreplay.UniformReplayOracle([()], [np.int64], 2, 10, seed=5)
  for i in range(12):
    v = np.array([i, 100 + i], dtype=np.int64)
    orc.add_batch([v])
    rb.add_batch(torch.as_tensor(v, device=cuda))
  (want,), want_ids, _, want_p = orc.get_next(9, 2)
  got, info = rb.get_next(sample_batch_size=9, num_steps=2)
  np.testing.assert_array_equal(got.cpu().numpy(), want)
  np.testing.assert_array_equal(info.ids.cpu().numpy(), want_ids)
  np.testing.assert_array_equal(info.probabilities.cpu().numpy(), want_p)
  np.testing.assert_array_equal(rb.gather_all().cpu().numpy(), orc.gather_all()[0])
  # a draw over several blocks advances the call once and returns the ticket to 0
  (want,), want_ids, _, _ = orc.get_next(600, 2)
  got, info = rb.get_next(sample_batch_size=600, num_steps=2)
  np.testing.assert_array_equal(got.cpu().numpy(), want)
  np.testing.assert_array_equal(info.ids.cpu().numpy(), want_ids)
  assert int(rb._ctrl[0].item()) == orc.rng_call == 2 and int(rb._ctrl[2].item()) == 0


def test_full_size_properties(cuda):
  """BASELINE config #2 geometry (256 x 4096 = 1M slots, 28 244 B rows, batch 256, T=2) through
  size-independent properties: every sampled frame carries its own row index, windows are
  contiguous inside one segment, ids match the id table, probabilities are 1/(n_ids*B_env)."""
  free, _ = torch.cuda.mem_get_info()
  B_env, L = 256, 4096
  if free < 40 << 30:
    B_env, L = 64, 1024
  spec = _traj_spec((84, 84, 4), torch.uint8)
  rb = rb_mod.TFUniformReplayBuffer(spec, batch_size=B_env, max_length=L, device=cuda, seed=99)
  cap = B_env * L
  obs = rb._data_table.variables()[1]          # observation storage [cap, 84, 84, 4]
  rows = torch.arange(cap, dtype=torch.int64, device=cuda)
  tag = obs.view(cap, -1)[:, :8]
  tag.copy_(rows.view(-1, 1).view(torch.uint8).view(cap, 8))     # row index in the first 8 bytes
  tail = obs.view(cap, -1)[:, -8:]
  tail.copy_((rows * 3 + 1).view(-1, 1).view(torch.uint8).view(cap, 8))
  last_id = L + 1234                            # wrapped ring
  seg_pos = rows % L
  ids = torch.where(seg_pos <= last_id % L, last_id - (last_id % L) + seg_pos,
                    last_id - (last_id % L) - L + seg_pos)
  rb._id_table.variables()[0].copy_(ids)
  rb._last_id.fill_(last_id)
  rb._last_id_host = last_id
  for _ in range(3):
    data, info = rb.get_next(sample_batch_size=256, num_steps=2)
    o = data.observation.reshape(256, 2, -1)
    got_rows = o[:, :, :8].contiguous().view(torch.int64).reshape(256, 2)
    got_tail = o[:, :, -8:].contiguous().view(torch.int64).reshape(256, 2)
    assert bool((got_tail == got_rows * 3 + 1).all())
    seg = got_rows // L
    assert bool((seg[:, 0] == seg[:, 1]).all())
    assert bool((got_rows[:, 1] % L == (got_rows[:, 0] % L + 1) % L).all())
    assert bool((info.ids == ids[got_rows]).all())
    assert bool((info.ids[:, 1] == info.ids[:, 0] + 1).all())
    assert bool((info.ids >= last_id + 1 - L).all()) and bool((info.ids <= last_id).all())
    np.testing.assert_allclose(info.probabilities.cpu().numpy(),
                               np.float32(1.0) / np.float32((L - 1) * B_env), rtol=0)
  assert len(torch.unique(seg)) > 1


def test_add_batch_inside_a_captured_step_keeps_the_host_mirror(cuda):
  """`add_batch` replayed from a common.function graph advances the device-resident last_id; the
  host mirror (used by gather_all / num_frames / the empty check) must follow every replay."""
  from agents_b200.utils import common
  rb = _scalar_rb(cuda, 3, max_length=16)
  item = torch.zeros(3, dtype=torch.int64, device=cuda)

  def step():
    item.add_(1)
    rb.add_batch(item)
    return item

  fn = common.function(step, warmup=1)
  for _ in range(6):                       # 1 eager + capture/replay + 4 replays
    fn()
  torch.cuda.synchronize()
  assert int(rb._last_id.item()) == 5 == rb._get_last_id()
  assert int(rb.num_frames()) == 18
  got = rb.gather_all().cpu().tolist()
  assert got == [[1, 2, 3, 4, 5, 6]] * 3
  data, _ = rb.get_next(sample_batch_size=4, num_steps=2)      # no spurious "buffer is empty"
  assert tuple(data.shape) == (4, 2)
