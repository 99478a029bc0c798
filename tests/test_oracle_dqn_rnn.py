"""Host checks of the recurrent DQN oracle (tests/dqn_rnn_oracle.py): the reference's RNN smoke
loss, the sequence loss and its dLoss/dq against float64 torch autograd, and the T-1 = 1 case
against the feed-forward oracle."""
import numpy as np
import pytest

from oracle import dqn as odqn
from oracle import lstm as olstm
from oracle import optim as ooptim

import dqn_rnn_oracle as O

f32 = np.float32


@pytest.mark.parametrize('ddqn', [False, True])
def test_reference_rnn_smoke_loss(ddqn):
  exp, cell = O.reference_smoke_case()
  orc = O.RecurrentDqnOracle(olstm.RnnNet([], [cell], []), None, gamma=1.0, ddqn=ddqn)
  assert np.isclose(float(orc.loss(exp)['loss']), O.REFERENCE_SMOKE_LOSS, rtol=1e-6, atol=0)
  orc.gamma = 0.95
  assert np.isclose(float(orc.loss(exp)['loss']), 28.657658, rtol=1e-6, atol=0)


@pytest.mark.parametrize('kind', ['huber', 'squared'])
@pytest.mark.parametrize('B,Tm,A', [(1, 1, 1), (7, 10, 6), (5, 80, 2)])
@pytest.mark.parametrize('wkind', ['none', 'scalar', 'row'])
def test_seq_loss_matches_float64(kind, B, Tm, A, wkind):
  rng = np.random.RandomState(B * 100 + Tm + A)
  N = B * Tm
  q, nt, ns = (rng.randn(N, A).astype(f32) * 2 for _ in range(3))
  act = rng.randint(0, A, (B, Tm)).astype(np.int32)
  st = rng.choice([0, 1, 2], (B, Tm), p=[0.2, 0.6, 0.2]).astype(np.int32)
  r = rng.randn(B, Tm).astype(f32)
  d = (rng.rand(B, Tm) > 0.2).astype(f32)
  mask = (rng.rand(N, A) > 0.3).astype(np.int32)
  mask[:, 0] = 1
  w = None if wkind == 'none' else (f32(0.7) if wkind == 'scalar' else
                                    np.where(rng.rand(B) < 0.3, 0, rng.rand(B)).astype(f32))
  got = O.dqn_seq_loss(q, nt, ns, act, st, r, d, 0.9, 1.5, kind, w, mask)
  want = O.seq_loss_float64(q, nt, ns, act, st, r, d, 0.9, 1.5, kind, w, mask)
  np.testing.assert_allclose(got['loss'], want[0], rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(got['td_loss'], want[1], rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(got['td_error'], want[2], rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(got['dq'], want[3], rtol=1e-5, atol=1e-7)


def test_one_transition_is_the_feed_forward_loss():
  rng = np.random.RandomState(3)
  B, A = 9, 4
  q, nt, ns = (rng.randn(B, A).astype(f32) for _ in range(3))
  act = rng.randint(0, A, (B, 2)).astype(np.int32)
  st = rng.randint(0, 3, (B, 2)).astype(np.int32)
  r, d = rng.randn(B, 2).astype(f32), rng.rand(B, 2).astype(f32)
  seq = O.dqn_seq_loss(q, nt, ns, act[:, :1], st[:, :1], r[:, :1], d[:, :1], 0.95)
  ff = odqn.dqn_loss(q, nt, ns, act[:, 0], st[:, 0], r, d, 0.95)
  for k in ('loss', 'td_loss', 'dq'):
    np.testing.assert_array_equal(np.asarray(seq[k]).reshape(-1), np.asarray(ff[k]).reshape(-1))


def test_train_moves_target_by_polyak_update():
  rng = np.random.RandomState(4)
  exp, cell = O.reference_smoke_case()
  post = [dict(w=rng.randn(2, 2).astype(f32), b=np.zeros(2, f32), act=None)]
  orc = O.RecurrentDqnOracle(olstm.RnnNet([], [cell], post), ooptim.AdamTF(1e-2),
                             target_update_tau=0.5, gradient_clipping=0.5, ddqn=True,
                             l2=[(3, 0.01)])
  before = [p.copy() for p in orc.target_net.params()]
  out = orc.train(exp, weights=np.array([1.0, 0.5], f32))
  for p, t, b in zip(orc.q_net.params(), orc.target_net.params(), before):
    np.testing.assert_allclose(t, 0.5 * b + 0.5 * p, rtol=1e-6, atol=1e-7)
  assert all(np.linalg.norm(g) <= 0.5 + 1e-6 for g in out['grads'])
  assert orc.train_step_counter == 1
