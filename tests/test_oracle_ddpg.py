"""The numpy DDPG oracle against the reference's critic- and actor-loss goldens and against float64
autograd: Huber and squared TD losses, weights, the observation branch and dqda_clipping None /
0.5 / 0; and the OU recurrence with supplied draws (no GPU)."""
import numpy as np
import pytest
import torch

from oracle import ddpg as oddpg
from oracle import nn as onn
from oracle import optim as ooptim
from oracle import td3 as otd3

f32 = np.float32


def _dense(rng, i, o, act, scale=0.4):
  return dict(kind='dense', w=(rng.randn(i, o) * scale).astype(f32),
              b=(rng.randn(o) * 0.1).astype(f32), act=act)


def _nets(rng, D, A, obs_fc=(7,), joint_fc=(9,), actor_fc=(8,)):
  dims = [D] + list(actor_fc)
  actor = onn.Sequential([_dense(rng, a, b, 'relu') for a, b in zip(dims, dims[1:])] +
                         [_dense(rng, dims[-1], A, 'tanh')])
  obs, width = None, D
  if obs_fc:
    od = [D] + list(obs_fc)
    obs = onn.Sequential([_dense(rng, a, b, 'relu') for a, b in zip(od, od[1:])])
    width = od[-1]
  jd = [width + A] + list(joint_fc)
  joint = onn.Sequential([_dense(rng, a, b, 'relu') for a, b in zip(jd, jd[1:])] +
                         [_dense(rng, jd[-1], 1, None, scale=2.0)])   # large dQ/da: clips bind
  return actor, otd3.Critic(joint, obs)


def _t(a):
  return torch.tensor(np.asarray(a, np.float64), requires_grad=True)


def _mlp(seq, params, x):
  i = 0
  for l in seq.layers:
    x = x @ params[i] + params[i + 1]
    i += 2
    x = torch.relu(x) if l['act'] == 'relu' else torch.tanh(x) if l['act'] == 'tanh' else x
  return x


def _q(critic, params, obs, act):
  n_obs = 2 * len(critic.obs.layers) if critic.obs else 0
  h = _mlp(critic.obs, params[:n_obs], obs) if critic.obs else obs
  return _mlp(critic.joint, params[n_obs:], torch.cat([h, act], 1))[:, 0]


def _elem(y, q, kind):
  e = y - q
  if kind == otd3.HUBER:
    a = e.abs()
    return torch.where(a <= 1, 0.5 * e * e, a - 0.5)
  return e * e


def _golden_oracle():
  # agents/ddpg/ddpg_agent_test.py: unbounded linear actor (kernel [2, 1], bias 5), linear critic
  # on concat(obs, action) (kernel [1, 3, 2], bias 4)
  actor = onn.Sequential([dict(kind='dense', w=np.array([[2.], [1.]], f32), b=np.array([5.], f32),
                               act=None)])
  critic = otd3.Critic(onn.Sequential([dict(kind='dense', w=np.array([[1.], [3.], [2.]], f32),
                                            b=np.array([4.], f32), act=None)]))
  return oddpg.DdpgOracle(actor, critic, None, None)


def test_reference_critic_loss_golden():
  # testCriticLoss: q = [21, 31], q' = [69, 89], y = [72.1, 100.1], Huber -> 59.6
  orc = _golden_oracle()
  obs, obs2 = np.array([[1., 2.], [3., 4.]], f32), np.array([[5., 6.], [7., 8.]], f32)
  act = np.array([[5.], [6.]], f32)
  r, d = np.array([10., 20.], f32), np.array([0.9, 0.9], f32)
  loss, _ = orc.critic_grads(obs, act, r, d, obs2)
  np.testing.assert_allclose(loss, 59.6, rtol=1e-6)
  np.testing.assert_array_equal(orc.critic.forward(obs, act), [21., 31.])
  np.testing.assert_array_equal(orc.tc.forward(obs2, orc.ta.forward(obs2)), [69., 89.])


def test_reference_actor_loss_golden():
  # testActorLoss: dQ/da is the critic's action weight, 2, for every row -> mean(2^2) = 4
  orc = _golden_oracle()
  obs = np.array([[1., 2.], [3., 4.]], f32)
  np.testing.assert_array_equal(orc.dqda(obs, orc.actor.forward(obs)), [[2.], [2.]])
  loss, _ = orc.actor_grads(obs)
  assert loss == 4.0


@pytest.mark.parametrize('kind', [otd3.HUBER, otd3.SQUARED])
@pytest.mark.parametrize('weighted', [False, True])
@pytest.mark.parametrize('obs_fc', [None, (7,)])
@pytest.mark.parametrize('dqda_clipping', [None, 0.5, 0.0])
def test_gradients_match_float64_autograd(kind, weighted, obs_fc, dqda_clipping):
  rng = np.random.RandomState(3)
  D, A, B = 5, 3, 33
  actor, critic = _nets(rng, D, A, obs_fc=obs_fc)
  amin, amax = np.array([-1., -2., 0.], f32), np.array([1., 2., 3.], f32)
  orc = oddpg.DdpgOracle(actor, critic, amin, amax, gamma=0.9, reward_scale=1.5, loss=kind,
                         dqda_clipping=dqda_clipping)
  for p in orc.tc.params() + orc.ta.params():       # targets differ, as after some soft updates
    p += (rng.randn(*p.shape) * 0.05).astype(f32)
  obs, obs2 = rng.randn(B, D).astype(f32), rng.randn(B, D).astype(f32)
  act = rng.uniform(-1, 1, (B, A)).astype(f32) * amax
  r, d = (rng.randn(B) * 3).astype(f32), (rng.rand(B) > 0.2).astype(f32)
  w = rng.rand(B).astype(f32) if weighted else None
  closs, cgrads = orc.critic_grads(obs, act, r, d, obs2, w)
  aloss, agrads = orc.actor_grads(obs, w)

  T = lambda a: torch.tensor(np.asarray(a, np.float64))
  lo, hi = T(amin), T(amax)
  W = torch.ones(B, dtype=torch.float64) if w is None else T(w)
  a2 = (hi + lo) / 2 + (hi - lo) / 2 * _mlp(orc.ta, [T(p) for p in orc.ta.params()], T(obs2))
  y = 1.5 * T(r) + 0.9 * T(d) * _q(orc.tc, [T(p) for p in orc.tc.params()], T(obs2), a2)
  pc = [_t(p) for p in critic.params()]
  loss = (_elem(y, _q(critic, pc, T(obs), T(act)), kind) * W).mean()
  ref = torch.autograd.grad(loss, pc)
  np.testing.assert_allclose(closs, loss.item(), rtol=2e-5)
  for g, rf in zip(cgrads, ref):
    np.testing.assert_allclose(g, rf.numpy(), rtol=1e-4, atol=1e-6 * float(rf.abs().max()))

  # actor: the loss is mean_{b,k}(w_b ((a + c) - a)^2) with c = clip(dQ/da) held constant
  pa = [_t(p) for p in actor.params()]
  a = (hi + lo) / 2 + (hi - lo) / 2 * _mlp(actor, pa, T(obs))
  ad = a.detach().requires_grad_()
  dqda, = torch.autograd.grad(_q(critic, [T(p) for p in critic.params()], T(obs), ad).sum(), ad)
  c = dqda if dqda_clipping is None else dqda.clamp(-dqda_clipping, dqda_clipping)
  if dqda_clipping == 0.5:
    assert float((dqda.abs() > 0.5).double().mean()) > 0.1       # the clip binds on some rows
  aref = (((a.detach() + c) - a) ** 2 * W[:, None]).mean()
  ref = torch.autograd.grad(aref, pa)
  np.testing.assert_allclose(aloss, aref.item(), rtol=2e-5, atol=1e-7)
  for g, rf in zip(agrads, ref):
    np.testing.assert_allclose(g, rf.numpy(), rtol=1e-4, atol=1e-6 * max(float(rf.abs().max()), 1e-30))
  if dqda_clipping == 0.0:                # clipped to [0, 0]: no actor gradient (reference code)
    assert aloss == 0 and all(not np.any(g) for g in agrads)


def test_weights_apply_per_row():
  """w_b multiplies row b of the [B, A] loss; a scalar weight scales the whole loss."""
  rng = np.random.RandomState(6)
  dqda = rng.randn(5, 3).astype(f32)
  w = rng.rand(5).astype(f32)
  loss, da = oddpg.actor_loss(dqda, None, w)
  np.testing.assert_allclose(loss, np.sum(w[:, None] * dqda.astype(np.float64) ** 2) / 15, rtol=1e-6)
  np.testing.assert_allclose(da, -2 * w[:, None] * dqda / 15, rtol=1e-6)
  l1, _ = oddpg.actor_loss(dqda, None, np.full(5, 0.5, f32))
  l0, _ = oddpg.actor_loss(dqda)
  np.testing.assert_allclose(l1, 0.5 * l0, rtol=1e-6)


def test_train_updates_actor_every_step_and_targets_periodically():
  rng = np.random.RandomState(5)
  D, A, B = 4, 2, 16
  actor, critic = _nets(rng, D, A)
  orc = oddpg.DdpgOracle(actor, critic, -np.ones(A, f32), np.ones(A, f32), ooptim.AdamTF(1e-2),
                         ooptim.AdamTF(1e-2), tau=0.05, target_update_period=2, gamma=0.9)
  for step in range(5):
    before = [p.copy() for p in actor.params()]
    tbefore = [p.copy() for p in orc.ta.params()]
    e = dict(observation=rng.randn(B, 2, D).astype(f32),
             action=rng.uniform(-1, 1, (B, 2, A)).astype(f32),
             reward=rng.randn(B, 2).astype(f32), discount=np.ones((B, 2), f32))
    out = orc.train(e)
    assert np.isfinite(out['actor_loss']) and out['loss'] == f32(out['actor_loss'] + out['critic_loss'])
    assert any(not np.array_equal(a, b) for a, b in zip(before, actor.params())), step
    tmoved = any(not np.array_equal(a, b) for a, b in zip(tbefore, orc.ta.params()))
    assert tmoved == ((step + 1) % 2 == 0), step     # Periodically: ++counter % period
  assert orc.actor_opt.t == orc.critic_opt.t == 5 == orc.train_step_counter


@pytest.mark.parametrize('damping', [1.0, 0.15, 0.0])
def test_ou_recurrence_matches_closed_form(damping):
  """x_t = sum_{s<=t} rho^(t-s) sigma z_s with rho = 1 - damping, x_0 = 0; the same x_t is added to
  every row, and the sum is clipped to the spec."""
  rng = np.random.RandomState(7)
  A, N, T, sigma = 4, 3, 20, 0.3
  rho = 1.0 - damping
  z = rng.randn(T, A).astype(f32)
  loc = rng.uniform(-1, 1, (N, A)).astype(f32)
  amin, amax = np.full(A, -0.8, f32), np.full(A, 0.9, f32)
  x = np.zeros(A, f32)
  for t in range(T):
    x = oddpg.ou_step(x, z[t], damping, sigma)
    want = sum(rho ** (t - s) * sigma * z[s].astype(np.float64) for s in range(t + 1))
    np.testing.assert_allclose(x, want, rtol=1e-5, atol=1e-6)
    out = oddpg.ou_actions(loc, x, amin, amax)
    np.testing.assert_allclose(out, np.clip(loc + want, amin, amax), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(oddpg.ou_actions(loc, x) - loc, np.broadcast_to(x, (N, A)),
                               atol=1e-6)
