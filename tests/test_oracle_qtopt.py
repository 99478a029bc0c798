"""Host checks of the QT-Opt oracle (oracle/qtopt.py): the reference test's golden loss, the
gradient against float64 autograd, the CEM search's top-k tie order, moments and bounds, and the
n-step reduction."""
import numpy as np
import torch

from oracle import nn as onn
from oracle import qtopt as oq
from oracle.td3 import Critic

f32 = np.float32


def _dense(w, b, act=None):
  return dict(kind='dense', w=np.asarray(w, f32), b=np.asarray(b, f32), act=act)


def _golden_exp():
  # agents/qtopt/qtopt_agent_test.py testLoss: restart time steps, then a transition
  return dict(observation=np.array([[[1, 2], [5, 6]], [[3, 4], [7, 8]]], f32),
              action=np.zeros((2, 2, 1), f32), reward=np.array([[10, 0], [20, 0]], f32),
              discount=np.array([[.9, 1], [.9, 1]], f32),
              step_type=np.array([[0, 1], [0, 1]], np.int32))


def test_reference_golden_loss():
  # DummyNet: Dense(1) of the observation with kernel [2, 1], bias 2 (q, target, delayed_2) or 1
  # (delayed); a CriticNetwork with no hidden layers and a zero action weight is the same network.
  net = lambda bias: Critic(onn.Sequential([_dense([[2], [1], [0]], [bias])]))
  orc = oq.QtOptOracle(net(2.0), [0.0], [1.0], [0.5], [0.08])
  orc.delayed = net(1.0)
  z = np.random.RandomState(0).randn(3, 2, 32, 1).astype(f32)
  out, _ = orc.loss_and_grads(_golden_exp(), z)
  np.testing.assert_allclose(out['loss'], 23.5, rtol=1e-6)
  np.testing.assert_allclose(out['td_loss'].mean(), 23.5, rtol=1e-6)
  np.testing.assert_allclose(out['y'], [25.3, 40.7], rtol=1e-6)
  assert (out['next_action'] >= 0).all() and (out['next_action'] <= 1).all()


def test_top_k_breaks_ties_to_the_lower_index():
  rng = np.random.RandomState(3)
  s = rng.randint(0, 4, (50, 33)).astype(f32)           # many ties
  idx = oq.top_k(s, 7)
  for b in range(50):
    want = sorted(range(33), key=lambda n: (-s[b, n], n))[:7]
    assert list(idx[b]) == want
  assert list(oq.top_k(np.zeros((1, 5), f32), 5)[0]) == [0, 1, 2, 3, 4]


def test_moments_match_numpy_and_sampling_clips():
  rng = np.random.RandomState(4)
  x = rng.randn(20, 9, 5).astype(f32)
  mean, var = oq.moments(x)
  np.testing.assert_allclose(mean, x.astype(np.float64).mean(1), rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(var, x.astype(np.float64).var(1), rtol=1e-5, atol=1e-6)
  lo, hi = np.array([-2, -1, 0], f32), np.array([3, 1, 0.5], f32)
  a = oq.sample(np.zeros((4, 3), f32), np.full((4, 3), 1e-9, f32), rng.randn(4, 100, 3) * 50,
                1e-4, lo, hi)
  assert (a >= lo).all() and (a <= hi).all()
  # the variance floor: sqrt(1e-4) * z before the clip
  a = oq.sample(np.zeros((1, 3), f32), np.zeros((1, 3), f32), np.ones((1, 1, 3), f32), 1e-4,
                lo, hi)
  np.testing.assert_allclose(a[0, 0], [0.01, 0.01, 0.01], rtol=1e-6)


def test_cem_search_finds_the_maximum_of_a_concave_score():
  rng = np.random.RandomState(5)
  B, N, A = 64, 64, 3
  target = rng.uniform(-0.8, 0.8, (B, A)).astype(f32)
  tiled = np.repeat(target, N, axis=0)
  score = lambda a: -np.sum((a - tiled) ** 2, axis=1)
  z = rng.randn(6, B, N, A).astype(f32)
  best, s = oq.cem_search(score, B, np.zeros(A), np.full(A, 0.3), z, 6, 1e-4, -np.ones(A, f32),
                          np.ones(A, f32))
  assert np.abs(best - target).max() < 0.1 and np.abs(best - target).mean() < 0.01
  np.testing.assert_allclose(s, -np.sum((best - target) ** 2, axis=1), rtol=1e-5, atol=1e-7)


def test_nstep_reduce_matches_the_discounted_sum():
  rng = np.random.RandomState(6)
  r, d = rng.randn(10, 4).astype(f32), (rng.rand(10, 4) > .2).astype(f32)
  R, D = oq.nstep_reduce(r, d, 0.9)
  want_r = r[:, 0] + 0.9 * d[:, 0] * r[:, 1] + 0.81 * d[:, 0] * d[:, 1] * r[:, 2]
  np.testing.assert_allclose(R, want_r, rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(D, 0.81 * d[:, 0] * d[:, 1] * d[:, 2], rtol=1e-6)


def _torch_q(layers, obs, act):
  h = torch.cat([obs, act], 1)
  for w, b, act_fn in layers:
    h = h @ w + b
    if act_fn == 'relu':
      h = torch.relu(h)
  return h[:, 0]


def test_gradient_matches_float64_autograd():
  rng = np.random.RandomState(8)
  D, A, B, H = 5, 3, 32, 16
  seq = lambda: onn.Sequential([_dense(rng.randn(D + A, H) * .4, rng.randn(H) * .1, 'relu'),
                                _dense(rng.randn(H, 1) * .4, rng.randn(1) * .1)])
  orc = oq.QtOptOracle(Critic(seq()), -np.ones(A, f32), np.ones(A, f32), np.zeros(A),
                       np.full(A, .3), num_samples=8, num_elites=3, gamma=0.9, reward_scale=0.7)
  orc.delayed, orc.delayed_2 = Critic(seq()), Critic(seq())
  exp = dict(observation=rng.randn(B, 3, D).astype(f32),
             action=rng.uniform(-1, 1, (B, 3, A)).astype(f32),
             reward=(rng.randn(B, 3) * 3).astype(f32),
             discount=(rng.rand(B, 3) > .1).astype(f32),
             step_type=rng.randint(0, 3, (B, 3)).astype(np.int32))
  w = rng.rand(B).astype(f32)
  z = rng.randn(3, B, 8, A).astype(f32)
  out, grads = orc.loss_and_grads(exp, z, w)
  t64 = lambda a: torch.as_tensor(np.asarray(a, np.float64))
  obs2, a2 = t64(exp['observation'][:, -1]), t64(out['next_action'])
  nq = torch.minimum(*[_torch_q([(t64(l['w']), t64(l['b']), l['act']) for l in n.joint.layers],
                                obs2, a2) for n in (orc.delayed, orc.delayed_2)])
  r, d = exp['reward'].astype(np.float64), exp['discount'].astype(np.float64)
  R = t64(r[:, 0] + 0.9 * d[:, 0] * r[:, 1])
  Dn = t64(0.9 * d[:, 0] * d[:, 1])
  y = 0.7 * R + 0.9 * Dn * nq
  params = [(t64(l['w']).requires_grad_(), t64(l['b']).requires_grad_(), l['act'])
            for l in orc.q.joint.layers]
  q = _torch_q(params, t64(exp['observation'][:, 0]), t64(exp['action'][:, 0]))
  e = (y - q).abs()
  hub = torch.where(e <= 1, 0.5 * e * e, e - 0.5)
  m = t64(exp['step_type'][:, 0] != 2)
  loss = (m * hub * t64(w)).sum() / B
  np.testing.assert_allclose(out['loss'], loss.item(), rtol=1e-5)
  ref = torch.autograd.grad(loss, [t for p in params for t in p[:2]])
  for g, rf in zip(grads, ref):
    np.testing.assert_allclose(g, rf.numpy(), rtol=1e-4, atol=1e-5 * float(rf.abs().max()))
