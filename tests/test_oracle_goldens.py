"""Pins the CPU oracle to the reference's own test goldens (SURVEY.md §8c).

Each test names the reference test it replays (paths relative to
tf_agents/ in the reference repository).  No GPU, no reference import: the literals below are the
reference's expected values.
"""
import numpy as np
import pytest

from oracle import dqn as odqn
from oracle import nn as onn
from oracle import optim as ooptim
from oracle import replay as oreplay
from oracle import value_ops as ovo

f32 = np.float32


def _rb(batch_size, max_length, dtype=np.int64):
  return oreplay.UniformReplayOracle([()], [dtype], batch_size, max_length)


# ---- replay_buffers/tf_uniform_replay_buffer_test.py ---------------------------------------
@pytest.mark.parametrize('batch_size', [1, 5])
def test_gather_all(batch_size):  # :313-333 testGatherAll (default max_length=1000)
  rb = _rb(batch_size, 1000)
  for i in range(10):
    rb.add_batch([np.arange(i, i + batch_size, dtype=np.int64)])
  (items,) = rb.gather_all()
  assert items.tolist() == [list(range(i, i + 10)) for i in range(batch_size)]


@pytest.mark.parametrize('batch_size', [1, 5])
def test_gather_all_over_capacity(batch_size):  # :339-361
  rb = _rb(batch_size, 10)
  for i in range(15):
    rb.add_batch([np.arange(0, batch_size * 100, 100, dtype=np.int64) + i])
  (items,) = rb.gather_all()
  assert items.tolist() == [list(range(5 + x * 100, 15 + x * 100)) for x in range(batch_size)]


@pytest.mark.parametrize('batch_size', [1, 5])
def test_gather_all_empty(batch_size):  # :367-378
  rb = _rb(batch_size, 1000, np.int32)
  (items,) = rb.gather_all()
  assert items.shape == (batch_size, 0)


@pytest.mark.parametrize('batch_size', [1, 5])
def test_sample_batch_probabilities(batch_size):  # :384-418
  rb = _rb(batch_size, 4, np.int32)
  for i in range(1, 3):
    rb.add_batch([np.full(batch_size, i - 1, np.int32)])
    _, _, _, prob = rb.get_next(2, 1)
    np.testing.assert_allclose(prob, [1.0 / (i * batch_size)] * 2, rtol=1e-6)


@pytest.mark.parametrize('batch_size', [1, 5])
def test_sample_single_probability_saturates(batch_size):  # :424-447
  max_length = 3
  rb = _rb(batch_size, max_length, np.int32)
  for i in range(1, 5):
    rb.add_batch([np.full(batch_size, i - 1, np.int32)])
    _, _, _, prob = rb.get_next(1, 1)
    np.testing.assert_allclose(prob[0], 1.0 / min(i * batch_size, max_length * batch_size),
                               rtol=1e-6)


def test_multi_step_windows_wrap_inside_segment():  # :227-307 ((x+1)%10 == next)
  rb = _rb(1, 10)
  for i in range(25):
    rb.add_batch([np.array([i % 10], dtype=np.int64)])
  for _ in range(100):
    (steps,), _, _, _ = rb.get_next(3, 2)
    assert ((steps[:, 0] + 1) % 10 == steps[:, 1]).all()


def test_get_next_two_segments():  # :701-723 testGetNext (B=256, T=2 across 2 segments)
  rb = _rb(2, 10)
  for i in range(10):
    rb.add_batch([np.array([i, 100 + i], dtype=np.int64)])
  (steps,), ids, rows, _ = rb.get_next(256, 2)
  assert steps.shape == (256, 2)
  assert (steps[:, 1] == steps[:, 0] + 1).all()           # never crosses a segment
  assert set(np.unique(rows // 10)) <= {0, 1}
  assert (ids[:, 1] == ids[:, 0] + 1).all()


def test_num_frames():  # :673-699
  rb = _rb(5, 4, np.int32)
  assert rb.num_frames() == 0
  for i in range(1, 7):
    rb.add_batch([np.zeros(5, np.int32)])
    assert rb.num_frames() == min(i * 5, 20)


def test_empty_raises():  # :96-109
  with pytest.raises(ValueError, match='TFUniformReplayBuffer is empty'):
    _rb(1, 10).get_next(1, 1)


def test_clear():  # :129-221
  rb = _rb(1, 10)
  rb.add_batch([np.array([7], dtype=np.int64)])
  rb.clear()
  assert rb.last_id == -1 and rb.num_frames() == 0
  assert rb.storage[0][0] == 7           # contents only unlinked
  rb.add_batch([np.array([3], dtype=np.int64)])
  rb.clear(clear_all_variables=True)
  assert rb.storage[0].sum() == 0


def _collect_deterministic(max_length, buffer_batch_size, num_adds, sample_batch_size,
                           num_steps=None):
  # _create_collect_rb_dataset :488-546
  rb = _rb(buffer_batch_size, max_length, np.int32)
  for ix in range(num_adds):
    rb.add_batch([10 * np.arange(buffer_batch_size, dtype=np.int32) + ix])
  vals = []
  for ids in rb.deterministic_row_ids(sample_batch_size, num_steps):
    vals.append(rb.storage[0][np.asarray(ids) % rb.capacity])
  return vals


@pytest.mark.parametrize('bbs', [1, 5])
def test_deterministic_dataset(bbs):  # :548-558
  vals = _collect_deterministic(3, bbs, 3, None)
  assert np.asarray(vals).tolist() == np.hstack(
      [np.arange(3) + 10 * i for i in range(bbs)]).tolist()


def test_deterministic_dataset_num_steps():  # :560-590
  vals = _collect_deterministic(4, 5, 4, None, num_steps=2)
  want = [[0, 1], [2, 3], [10, 11], [12, 13], [20, 21], [22, 23], [30, 31], [32, 33],
          [40, 41], [42, 43]]
  assert np.asarray(vals).tolist() == want


@pytest.mark.parametrize('bbs', [1, 5])
def test_deterministic_dataset_sample_batch(bbs):  # :596-614
  vals = _collect_deterministic(3, bbs, 3, bbs)
  assert np.asarray(vals).tolist() == np.vstack(
      [10 * np.arange(bbs) + i for i in range(3)]).tolist()


def test_deterministic_dataset_num_steps_and_sample_batch():  # :616-641
  vals = _collect_deterministic(4, 6, 4, 3, num_steps=2)
  want = [[[0, 1], [10, 11], [20, 21]], [[2, 3], [12, 13], [22, 23]],
          [[30, 31], [40, 41], [50, 51]], [[32, 33], [42, 43], [52, 53]]]
  assert np.asarray(vals).tolist() == want


# ---- utils/value_ops_test.py -----------------------------------------------------------------
def test_discounted_return_final_value_precomputed():  # :179-206
  got = ovo.discounted_return(np.ones(9, f32)[:, None],
                              np.array([1, 1, 1, 1, 0, .9, .9, .9, .9], f32)[:, None],
                              final_value=np.array([8], f32))[:, 0]
  want = [5, 4, 3, 2, 1, 8 * 0.9**4 + 3.439, 8 * 0.9**3 + 2.71, 8 * 0.9**2 + 1.9, 8 * 0.9 + 1]
  np.testing.assert_allclose(got, want, rtol=1e-6)


def test_discounted_return_vs_naive():  # :28-92 randomised vs naive numpy
  rng = np.random.RandomState(0)
  T, B = 9, 7
  r, d = rng.rand(T, B).astype(f32), rng.rand(T, B).astype(f32)
  fv = rng.rand(B).astype(f32)
  want = np.zeros((T, B))
  acc = fv.astype(np.float64)
  for t in range(T - 1, -1, -1):
    acc = r[t] + d[t] * acc
    want[t] = acc
  np.testing.assert_allclose(ovo.discounted_return(r, d, fv), want, rtol=1e-5)
  np.testing.assert_allclose(ovo.discounted_return(r.T, d.T, fv, time_major=False), want.T,
                             rtol=1e-5)
  np.testing.assert_allclose(
      ovo.discounted_return(r, d, fv, provide_all_returns=False), want[0], rtol=1e-5)


def test_gae_precomputed():  # :239-278 testAdvantagesMatchPrecomputedResult
  d = np.array([[1, 1, 1, 1, 0, .9, .9, .9, 0]] * 2, f32)
  adv = ovo.generalized_advantage_estimation(
      values=np.full((2, 9), 3, f32), final_value=np.full(2, 3, f32), discounts=d,
      rewards=np.ones((2, 9), f32), td_lambda=0.95, time_major=False)
  want = [2.0808625, 1.13775, 0.145, -0.9, -2.0, 0.56016475, -0.16355, -1.01, -2.0]
  np.testing.assert_allclose(adv, [want, want], rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize('lam', [0.7, 0.0, 1.0])
def test_gae_vs_naive(lam):  # :214-237 with _naive_gae_as_ground_truth :95-127
  rng = np.random.RandomState(1)
  T, B = 9, 7
  r, d, v = [rng.rand(T, B).astype(f32) for _ in range(3)]
  fv = rng.rand(B).astype(f32)
  nv = np.concatenate([v[1:], fv[None]], 0).astype(np.float64)
  delta = r + d * nv - v
  want = np.zeros((T, B))
  for t in range(T):
    acc, w = np.zeros(B), np.ones(B)
    for k in range(t, T):
      acc = acc + w * delta[k]
      w = w * lam * d[k]
    want[t] = acc
  np.testing.assert_allclose(ovo.generalized_advantage_estimation(v, fv, d, r, lam), want,
                             rtol=1e-5, atol=1e-6)


# ---- trajectories/trajectory_test.py -------------------------------------------------------
def test_n_step_n1():  # :241-274
  R, D = ovo.n_step_reduce(np.array([[-1.0, 0.0]], f32), np.array([[0.9, 0.0]], f32), 0.5)
  assert R.tolist() == [-1.0] and D.tolist() == [f32(0.9)]


def test_n_step_n3():  # :276-317
  g = 0.5
  R, D = ovo.n_step_reduce(np.array([[-1.0, 1.0, 2.0, 0.0]], f32),
                           np.array([[0.9, 0.95, 1.0, 0.0]], f32), g)
  np.testing.assert_allclose(R, [-1.0 + 1.0 * g * 0.9 + 2.0 * g**2 * 0.9 * 0.95], rtol=1e-6)
  np.testing.assert_allclose(D, [g**2 * 0.9 * 0.95 * 1.0], rtol=1e-6)


# ---- agents/dqn/dqn_agent_test.py ------------------------------------------------------------
def _dummy_net(l2=0.0):
  # DummyNet :38-69: Dense(2) kernel [[2,1],[1,1]] (in x out), bias [1,1]
  return onn.Sequential([dict(kind='dense', w=np.array([[2, 1], [1, 1]], f32),
                              b=np.array([1, 1], f32), act=None)])


def _exp(obs_seq, step_types, rewards, discounts, actions=(0, 1)):
  B = 2
  T = len(obs_seq)
  return dict(
      observation=np.stack([np.asarray(o, f32) for o in obs_seq], axis=1),
      step_type=np.stack([np.full(B, s, np.int32) for s in step_types], axis=1),
      action=np.stack([np.asarray(actions, np.int32)] * T, axis=1),
      reward=np.stack([np.asarray(r, f32) for r in rewards], axis=1),
      discount=np.stack([np.asarray(d, f32) for d in discounts], axis=1))


def test_td_targets():  # :74-82
  got = odqn.compute_td_targets(np.array([10, 20], f32), np.array([10, 20], f32),
                                np.array([.9, .9], f32))
  np.testing.assert_allclose(got, [19.0, 38.0], rtol=1e-6)


@pytest.mark.parametrize('ddqn', [False, True])
def test_dqn_loss(ddqn):  # :178-218 -> 26.0
  agent = odqn.DqnOracle(_dummy_net(), None, ddqn=ddqn)
  exp = _exp([[[1, 2], [3, 4]], [[5, 6], [7, 8]]], [0, 1], [[10, 20]] * 2, [[.9, .9]] * 2)
  np.testing.assert_allclose(agent.loss(exp)['loss'], 26.0, rtol=1e-6)


@pytest.mark.parametrize('ddqn', [False, True])
def test_dqn_loss_changed_optimal_actions(ddqn):  # :220-267 -> 9.8
  agent = odqn.DqnOracle(_dummy_net(), None, ddqn=ddqn)
  exp = _exp([[[1, 2], [3, 4]], [[-5, 6], [-7, 8]]], [0, 1], [[10, 20]] * 2, [[.9, .9]] * 2)
  np.testing.assert_allclose(agent.loss(exp)['loss'], 9.8, rtol=1e-6)


def test_dqn_loss_l2():  # :269-299 -> 33.0 (26.0 + 7.0)
  net = _dummy_net()
  agent = odqn.DqnOracle(net, None)
  exp = _exp([[[1, 2], [3, 4]], [[5, 6], [7, 8]]], [0, 1], [[10, 20]] * 2, [[.9, .9]] * 2)
  base = agent.loss(exp)
  reg = float(np.sum(net.layers[0]['w'] ** 2))
  assert reg == 7.0
  np.testing.assert_allclose(base['loss'] + reg, 33.0, rtol=1e-6)


def test_dqn_loss_nstep():  # :301-355 -> 47.42 (n=2)
  agent = odqn.DqnOracle(_dummy_net(), None, n_step_update=2)
  exp = _exp([[[1, 2], [3, 4]], [[5, 6], [7, 8]], [[9, 10], [11, 12]]], [0, 1, 1],
             [[10, 20]] * 3, [[.9, .9]] * 3)
  np.testing.assert_allclose(agent.loss(exp)['loss'], 47.42, rtol=1e-6)


def test_dqn_loss_nstep_mid_mid_last_first():  # :416-481 -> 21.5 (n=3, LAST zeroes bootstrap)
  agent = odqn.DqnOracle(_dummy_net(), None, n_step_update=3)
  exp = _exp([[[1, 2], [3, 4]], [[5, 6], [7, 8]], [[9, 10], [11, 12]], [[13, 14], [15, 16]]],
             [1, 1, 2, 0], [[10, 20], [10, 20], [0, 0], [0, 0]],
             [[.9, .9], [0, 0], [1, 1], [1, 1]])
  np.testing.assert_allclose(agent.loss(exp)['loss'], 21.5, rtol=1e-6)


def test_dqn_loss_masked_actions():  # :483-561 -> 23.75
  net = _dummy_net()
  obs0 = np.array([[1, 2], [3, 4]], f32)
  obsn = np.array([[5, 6], [7, 8]], f32)
  out = odqn.dqn_loss(net.forward(obs0), net.forward(obsn), net.forward(obsn), [0, 1], [0, 0],
                      np.array([[10, 0], [20, 0]], f32), np.array([[.9, 1], [.9, 1]], f32),
                      next_mask=np.array([[0, 1], [1, 0]]))
  np.testing.assert_allclose(out['loss'], 23.75, rtol=1e-6)
  # D3qnAgent selects with a raw argmax of the online network (dqn_agent.py:731), so the same
  # case without the mask is what the reference expects for it: 26.0 (dqn_agent_test.py:556)
  out = odqn.dqn_loss(net.forward(obs0), net.forward(obsn), net.forward(obsn), [0, 1], [0, 0],
                      np.array([[10, 0], [20, 0]], f32), np.array([[.9, 1], [.9, 1]], f32),
                      next_mask=None)
  np.testing.assert_allclose(out['loss'], 26.0, rtol=1e-6)


def test_huber_matches_test_comment():  # dqn_agent_test.py:205-213 ("Huber loss subtracts 0.5")
  np.testing.assert_allclose(odqn.huber(np.array([25.3, 40.7], f32), np.array([5, 8], f32)),
                             [19.8, 32.2], rtol=1e-6)
  np.testing.assert_allclose(odqn.huber(np.array([0.3], f32), np.array([0.0], f32)), [0.045],
                             rtol=1e-6)


# ---- utils/common_test.py --------------------------------------------------------------------
def test_soft_update():  # :83-143
  s, t = [np.array([1.0, 2.0], f32)], [np.array([3.0, 5.0], f32)]
  ooptim.soft_variables_update(s, t, tau=0.1)
  np.testing.assert_allclose(t[0], [0.9 * 3 + 0.1 * 1, 0.9 * 5 + 0.1 * 2], rtol=1e-6)
  ooptim.soft_variables_update(s, t, tau=1.0)
  assert t[0].tolist() == [1.0, 2.0]


def test_periodically():  # :230-331: fires on the `period`-th, 2*period-th ... call
  fired = []
  p = ooptim.Periodically(lambda: fired.append(1), 3)
  pattern = [p() for _ in range(7)]
  assert pattern == [False, False, True, False, False, True, False]
  q = ooptim.Periodically(lambda: None, 1)
  assert [q() for _ in range(3)] == [True, True, True]


def test_index_with_actions():  # :164-228
  q = np.array([[1, 2, 3], [4, 5, 6]], f32)
  assert odqn.index_with_actions(q, [2, 0]).tolist() == [3.0, 4.0]
