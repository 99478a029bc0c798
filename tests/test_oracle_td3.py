"""The numpy TD3 oracle against the reference's actor-loss golden and against float64 autograd:
Huber and squared TD losses, weights, target smoothing with injected noise, the observation branch
and the delayed-actor schedule (no GPU)."""
import numpy as np
import pytest
import torch

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

  def critic():
    obs = None
    width = D
    if obs_fc:
      od = [D] + list(obs_fc)
      obs = onn.Sequential([_dense(rng, a, b, 'relu') for a, b in zip(od, od[1:])])
      width = od[-1]
    jd = [width + A] + list(joint_fc)
    joint = onn.Sequential([_dense(rng, a, b, 'relu') for a, b in zip(jd, jd[1:])] +
                           [_dense(rng, jd[-1], 1, None)])
    return otd3.Critic(joint, obs)
  return actor, critic(), critic()


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


def test_reference_actor_loss_golden():
  # agents/td3/td3_agent_test.py testActorLoss: unbounded linear actor (kernel [2, 1], bias 5),
  # linear critic on concat(obs, action) (kernel [1, 3, 2], bias 4): actions 9 and 15, loss -39
  actor = onn.Sequential([dict(kind='dense', w=np.array([[2.], [1.]], f32), b=np.array([5.], f32),
                               act=None)])
  critic = otd3.Critic(onn.Sequential([dict(kind='dense', w=np.array([[1.], [3.], [2.]], f32),
                                            b=np.array([4.], f32), act=None)]))
  orc = otd3.Td3Oracle(actor, critic, critic, None, None)
  obs = np.array([[1., 2.], [3., 4.]], f32)
  np.testing.assert_array_equal(actor.forward(obs)[:, 0], [9., 15.])
  loss, _ = orc.actor_grads(obs)
  assert loss == -39.0


@pytest.mark.parametrize('kind', [otd3.HUBER, otd3.SQUARED])
@pytest.mark.parametrize('weighted', [False, True])
@pytest.mark.parametrize('obs_fc', [None, (7,)])
def test_gradients_match_float64_autograd(kind, weighted, obs_fc):
  rng = np.random.RandomState(3)
  D, A, B = 5, 3, 33
  actor, c1, c2 = _nets(rng, D, A, obs_fc=obs_fc)
  amin, amax = np.array([-1., -2., 0.], f32), np.array([1., 2., 3.], f32)
  orc = otd3.Td3Oracle(actor, c1, c2, amin, amax, gamma=0.9, reward_scale=1.5, loss=kind,
                       target_policy_noise=0.3, target_policy_noise_clip=0.4)
  # targets differ from the online nets, as after some soft updates
  for p in orc.t1.params() + orc.t2.params() + orc.ta.params():
    p += (rng.randn(*p.shape) * 0.05).astype(f32)
  obs, obs2 = rng.randn(B, D).astype(f32), rng.randn(B, D).astype(f32)
  act = rng.uniform(-1, 1, (B, A)).astype(f32) * amax
  r, d = (rng.randn(B) * 3).astype(f32), (rng.rand(B) > 0.2).astype(f32)
  z = (rng.randn(B, A) * 2).astype(f32)              # many draws beyond the noise clip
  w = rng.rand(B).astype(f32) if weighted else None
  closs, cgrads = orc.critic_grads(obs, act, r, d, obs2, z, w)
  aloss, agrads = orc.actor_grads(obs, w)

  T = lambda a: torch.tensor(np.asarray(a, np.float64))
  lo, hi = T(amin), T(amax)
  ta = [T(p) for p in orc.ta.params()]
  a2 = (hi + lo) / 2 + (hi - lo) / 2 * _mlp(orc.ta, ta, T(obs2))
  a2 = a2 + torch.clamp(0.3 * T(z), -0.4, 0.4)
  tq = torch.minimum(_q(orc.t1, [T(p) for p in orc.t1.params()], T(obs2), a2),
                     _q(orc.t2, [T(p) for p in orc.t2.params()], T(obs2), a2))
  y = 1.5 * T(r) + 0.9 * T(d) * tq
  p1, p2 = [_t(p) for p in c1.params()], [_t(p) for p in c2.params()]
  per = _elem(y, _q(c1, p1, T(obs), T(act)), kind) + _elem(y, _q(c2, p2, T(obs), T(act)), kind)
  W = torch.ones(B, dtype=torch.float64) if w is None else T(w)
  loss = (per * W).mean()
  ref = torch.autograd.grad(loss, p1 + p2)
  np.testing.assert_allclose(closs, loss.item(), rtol=2e-5)
  for g, rf in zip(cgrads, ref):
    np.testing.assert_allclose(g, rf.numpy(), rtol=1e-4, atol=1e-6 * float(rf.abs().max()))
  pa = [_t(p) for p in actor.params()]
  a = (hi + lo) / 2 + (hi - lo) / 2 * _mlp(actor, pa, T(obs))
  aref = (-_q(c1, [T(p) for p in c1.params()], T(obs), a) * W).sum() / B
  ref = torch.autograd.grad(aref, pa)
  np.testing.assert_allclose(aloss, aref.item(), rtol=2e-5, atol=1e-6)
  for g, rf in zip(agrads, ref):
    np.testing.assert_allclose(g, rf.numpy(), rtol=1e-4, atol=1e-6 * float(rf.abs().max()))


def test_target_actions_are_smoothed_but_not_clamped():
  rng = np.random.RandomState(4)
  actor, c1, c2 = _nets(rng, 4, 2)
  actor.layers[-1]['b'][:] = 50.0                   # tanh saturates: the action sits at the bound
  orc = otd3.Td3Oracle(actor, c1, c2, -np.ones(2, f32), np.ones(2, f32), target_policy_noise=0.2,
                       target_policy_noise_clip=0.5)
  obs2 = rng.randn(64, 4).astype(f32)
  z = np.full((64, 2), 10.0, f32)
  a2 = orc.target_actions(obs2, z)
  np.testing.assert_allclose(a2, 1.5, rtol=1e-6)   # noise clipped at 0.5, sum not clamped to 1
  np.testing.assert_allclose(orc.target_actions(obs2, -z), 0.5, rtol=1e-4)


@pytest.mark.parametrize('period', [1, 2, 3])
def test_delayed_actor_schedule(period):
  rng = np.random.RandomState(5)
  D, A, B = 4, 2, 16
  actor, c1, c2 = _nets(rng, D, A)
  orc = otd3.Td3Oracle(actor, c1, c2, -np.ones(A, f32), np.ones(A, f32), ooptim.AdamTF(1e-2),
                       ooptim.AdamTF(1e-2), actor_update_period=period, tau=0.05,
                       target_update_period=2)
  for step in range(7):
    before = [p.copy() for p in actor.params()]
    tbefore = [p.copy() for p in orc.ta.params()]
    e = dict(observation=rng.randn(B, 2, D).astype(f32), action=rng.uniform(-1, 1, (B, 2, A)).astype(f32),
             reward=rng.randn(B, 2).astype(f32), discount=np.ones((B, 2), f32))
    out = orc.train(e, rng.randn(B, A).astype(f32))
    assert np.isfinite(out['actor_loss'])             # returned on every step
    moved = any(not np.array_equal(a, b) for a, b in zip(before, actor.params()))
    assert moved == (step % period == 0), step
    tmoved = any(not np.array_equal(a, b) for a, b in zip(tbefore, orc.ta.params()))
    assert tmoved == ((step + 1) % 2 == 0), step     # Periodically: ++counter % period
  assert orc.actor_updates == len([s for s in range(7) if s % period == 0])
  assert orc.actor_opt.t == orc.actor_updates and orc.critic_opt.t == 7
