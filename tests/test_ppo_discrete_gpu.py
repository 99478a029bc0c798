"""Discrete-action PPO on the GPU: the categorical loss / log-prob / KL / sampling kernels against
oracle/ppo_discrete.py, the Categorical PPOPolicy, and PPOClipAgent / PPOAgent / PPOLearner
training parity with a Categorical actor (MLP and Atari-shape conv torsos)."""
import ctypes

import numpy as np
import pytest
import torch

from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.agents.ppo import ppo_agent
from agents_b200.agents.ppo import ppo_clip_agent
from agents_b200.networks import actor_distribution_network
from agents_b200.networks import layers as L
from agents_b200.networks import value_network
from agents_b200.specs import tensor_spec
from agents_b200.train import ppo_learner
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory
from agents_b200.utils import common
from agents_b200.utils import workspace
from oracle import nn as onn
from oracle import optim as ooptim
from oracle import ppo_discrete as opd
from oracle import ppo_learner as opl

from conftest import record_parity

pytestmark = pytest.mark.gpu
f32 = np.float32
CANARY = 64


def _dev(cuda, a, dtype=None):
  return torch.as_tensor(np.ascontiguousarray(a, dtype=dtype), device=cuda)


def _case(rng, N, A):
  z = (rng.randn(N, A) * 2).astype(f32)
  zo = (z + rng.randn(N, A) * 0.4).astype(f32)
  a = rng.randint(0, A, N).astype(np.int32)
  a[:3] = 0
  a[3:6] = A - 1                                 # both ends of the action range
  old_logp = (opd.categorical_log_prob(zo, a)).astype(f32)
  adv, ret = rng.randn(N).astype(f32), rng.randn(N).astype(f32)
  v = rng.randn(N).astype(f32)
  v_old = (v + rng.randn(N) * 0.3).astype(f32)
  w = (rng.rand(N) > 0.2).astype(f32)            # weights with zeros
  return z, zo, a, old_logp, adv, ret, v, v_old, w


def _run_loss(cuda, z, zo, a, old_logp, adv, ret, v, v_old, w, T, kw, kl=None, ld_pad=0):
  """Launches b200rl_ppo_loss_categorical; ld_pad > 0 passes the logits as a strided view."""
  N, A = z.shape
  ld = A + ld_pad
  zbuf = np.full((N, ld), np.nan, f32)
  zbuf[:, :A] = z
  t = dict(z=_dev(cuda, zbuf), a=_dev(cuda, a), old=_dev(cuda, old_logp), adv=_dev(cuda, adv),
           ret=_dev(cuda, ret), v=_dev(cuda, v), vo=_dev(cuda, v_old), w=_dev(cuda, w))
  losses = torch.empty(6, device=cuda)
  dz = torch.full((N * A + CANARY,), 7.0, device=cuda)         # canary tail after the gradient
  dv = torch.full((N + CANARY,), 7.0, device=cuda)
  flag = torch.zeros(1, dtype=torch.int32, device=cuda)
  ws, nb = workspace.get(cuda)
  kl_arg, keep = None, []
  if kl is not None:
    beta = torch.tensor([kl['beta']], dtype=torch.float32, device=cuda)
    mean_kl = torch.empty(1, device=cuda)
    terms = torch.empty(3, device=cuda)
    zo_d = _dev(cuda, zo)
    _lib.call('b200rl_ppo_kl_categorical', _lib.ptr(t['z']), ld, _lib.ptr(zo_d), A, _lib.ptr(t['w']),
              N, A, 1.0 / N, None, _lib.ptr(mean_kl), _lib.ptr(ws), nb, _lib.stream())
    _lib.call('b200rl_ppo_kl_terms', _lib.ptr(mean_kl), _lib.ptr(beta), kl['factor'], kl['target'],
              kl['coef'], _lib.ptr(terms), _lib.stream())
    kl_arg = _lib.PpoKlLogits(_lib.ptr(zo_d), A, _lib.ptr(terms), 1.0 / N)
    keep = [beta, mean_kl, terms, zo_d]
  _lib.call('b200rl_ppo_loss_categorical', _lib.ptr(t['z']), ld, _lib.ptr(t['a']), _lib.ptr(t['old']),
            _lib.ptr(t['adv']), _lib.ptr(t['ret']), _lib.ptr(t['v']), _lib.ptr(t['vo']), _lib.ptr(t['w']),
            N, A, T, float(N // T), kw['clip_eps'], kw['value_clip'], kw['vf_coef'], kw['ent_coef'],
            kw['logp_clip'], _lib.ptr(losses), _lib.ptr(dz), A, _lib.ptr(dv), _lib.ptr(flag),
            ctypes.byref(kl_arg) if kl_arg is not None else None, _lib.ptr(ws), nb, _lib.stream())
  torch.cuda.synchronize()
  del keep
  dz, dv = dz.cpu().numpy(), dv.cpu().numpy()
  assert np.all(dz[N * A:] == 7.0) and np.all(dv[N:] == 7.0)
  return losses.cpu().numpy(), dz[:N * A].reshape(N, A), dv[:N], int(flag.item())


_CFGS = {
    'clip': dict(clip_eps=0.2),
    'clip_vclip_ent_logpclip': dict(clip_eps=0.2, value_clip=0.3, ent_coef=0.01, logp_clip=2.0),
    'kl_cutoff_adaptive': dict(clip_eps=0.0, ent_coef=0.02,
                               kl=dict(beta=0.7, factor=2.0, target=0.01, coef=1000.0)),
}


@pytest.mark.parametrize('A', [2, 6, 18, 300])
@pytest.mark.parametrize('name', sorted(_CFGS))
def test_loss_kernel_parity(cuda, A, name):
  cfg = dict(_CFGS[name])
  kl = cfg.pop('kl', None)
  kw = dict(clip_eps=0.2, value_clip=0.0, vf_coef=0.5, ent_coef=0.0, logp_clip=0.0)
  kw.update(cfg)
  rng = np.random.RandomState(A)
  B, T = 41, 9
  N = B * T
  z, zo, a, old_logp, adv, ret, v, v_old, w = _case(rng, N, A)
  losses, dz, dv, flag = _run_loss(cuda, z, zo, a, old_logp, adv, ret, v, v_old, w, T, kw, kl,
                                   ld_pad=3 if A == 18 else 0)
  assert flag == 0
  okw = dict(clip_eps=kw['clip_eps'], vf_coef=kw['vf_coef'], ent_coef=kw['ent_coef'],
             value_clip=kw['value_clip'], logp_clip=kw['logp_clip'])
  if kl:
    okw.update(kl_cutoff_factor=kl['factor'], kl_cutoff_coef=kl['coef'],
               initial_adaptive_kl_beta=kl['beta'], adaptive_kl_target=kl['target'])
  actor = onn.Sequential([dict(kind='dense', w=np.eye(A, dtype=f32), b=np.zeros(A, f32))])
  orc = opd.CategoricalPPOOracle(actor, onn.Sequential([]), ooptim.AdamTF(1e-3), **okw)
  # the loss kernel takes v as an input: the oracle's value net returns the same predictions
  orc.value = _Const(v)
  info, _, want_dz, want_dv = orc.loss_and_grads(z, a, old_logp, ret, adv, v_old, w, B, T,
                                                 old_logits=zo)
  rel = lambda g, w_: abs(float(g) - float(w_)) / max(abs(float(w_)), 1e-30)
  record_parity('ppo_discrete_loss', total_rel=rel(losses[4], info['loss']),
                pg_rel=rel(losses[0], info['pg']), ent_rel=rel(losses[2], info['ent']))
  np.testing.assert_allclose(losses[0], info['pg'], rtol=1e-5, atol=1e-7)
  np.testing.assert_allclose(losses[1], info['ve'], rtol=1e-5)
  np.testing.assert_allclose(losses[2], info['ent'], rtol=1e-5, atol=1e-9)
  np.testing.assert_allclose(losses[3], info['clip_fraction'], rtol=1e-6)
  np.testing.assert_allclose(losses[5], info['kl'], rtol=1e-5, atol=1e-9)
  np.testing.assert_allclose(losses[4], info['loss'], rtol=1e-5, atol=1e-7)
  scale = np.abs(want_dz).max()
  record_parity('ppo_discrete_loss', dlogits_err_rel_to_max=float(np.abs(dz - want_dz).max()) / scale)
  np.testing.assert_allclose(dz, want_dz, rtol=1e-4, atol=1e-5 * scale)
  np.testing.assert_allclose(dv, want_dv, rtol=1e-5, atol=1e-9)


class _Const(object):
  """A stand-in value net that returns fixed predictions (the loss kernel takes v as input)."""

  def __init__(self, v):
    self.v = v

  def forward(self, x, keep=False):
    out = self.v[:, None]
    return (out, None) if keep else out

  def backward(self, tape, dy):
    return []

  def params(self):
    return []


def test_out_of_range_action_raises_flag_and_stays_in_bounds(cuda):
  rng = np.random.RandomState(1)
  N, A, T = 300, 6, 3
  z, zo, a, old_logp, adv, ret, v, v_old, w = _case(rng, N, A)
  a[10], a[20] = A, -1
  kw = dict(clip_eps=0.2, value_clip=0.0, vf_coef=0.5, ent_coef=0.01, logp_clip=0.0)
  losses, dz, dv, flag = _run_loss(cuda, z, zo, a, old_logp, adv, ret, v, v_old, w, T, kw)
  assert flag == 1                     # canary tails were checked inside _run_loss
  assert np.all(np.isfinite(dz)) and np.all(np.isfinite(losses))
  out = torch.empty(N, device=cuda)
  f2 = torch.zeros(1, dtype=torch.int32, device=cuda)
  zd, ad = _dev(cuda, z), _dev(cuda, a)
  _lib.call('b200rl_categorical_logp', _lib.ptr(zd), A, _lib.ptr(ad), N, A, _lib.ptr(out), _lib.ptr(f2),
            _lib.stream())
  assert int(f2.item()) == 1


@pytest.mark.parametrize('A', [2, 6, 18, 300])
def test_logp_and_kl_kernels(cuda, A):
  rng = np.random.RandomState(10 + A)
  N = 1111
  z, zo, a, _, _, _, _, _, w = _case(rng, N, A)
  zd, zod, ad, wd = _dev(cuda, z), _dev(cuda, zo), _dev(cuda, a), _dev(cuda, w)
  out = torch.empty(N, device=cuda)
  flag = torch.zeros(1, dtype=torch.int32, device=cuda)
  _lib.call('b200rl_categorical_logp', _lib.ptr(zd), A, _lib.ptr(ad), N, A, _lib.ptr(out), _lib.ptr(flag),
            _lib.stream())
  np.testing.assert_allclose(out.cpu().numpy(), opd.categorical_log_prob(z, a), rtol=1e-5, atol=1e-6)
  assert int(flag.item()) == 0
  kl = torch.empty(N, device=cuda)
  s = torch.empty(1, device=cuda)
  ws, nb = workspace.get(cuda)
  _lib.call('b200rl_ppo_kl_categorical', _lib.ptr(zd), A, _lib.ptr(zod), A, _lib.ptr(wd), N, A, 1.0 / N,
            _lib.ptr(kl), _lib.ptr(s), _lib.ptr(ws), nb, _lib.stream())
  want = (opd.categorical_kl(zo, z) * w).astype(f32)
  np.testing.assert_allclose(kl.cpu().numpy(), want, rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(s.item(), want.mean(dtype=np.float64), rtol=1e-5)


def _sample(cuda, logits_d, rng_block, seed):
  n, a = logits_d.shape
  out = torch.empty(n, dtype=torch.int32, device=cuda)
  _lib.call('b200rl_categorical_sample', _lib.ptr(logits_d), a, n, a, seed, _lib.ptr(rng_block),
            _lib.ptr(out), _lib.stream())
  return out


def test_sampling_matches_oracle_and_distribution(cuda):
  rng = np.random.RandomState(5)
  seed = 0x1234_5678_9ABC
  for A in (2, 6, 18, 300):
    N = 4099
    z = (rng.randn(N, A) * 2).astype(f32)
    zd = _dev(cuda, z)
    block = torch.zeros(2, dtype=torch.int64, device=cuda)
    for call in range(2):
      got = _sample(cuda, zd, block, seed).cpu().numpy()
      want, u = opd.categorical_sample(z, seed, call)
      cdf = opd.categorical_cdf(z)
      near = (np.abs(cdf - u[:, None]) < 1e-6).any(axis=1)
      assert near.mean() < 0.01
      np.testing.assert_array_equal(got[~near], want[~near])
      assert got.min() >= 0 and got.max() < A
    assert int(block[0].item()) == 2 and int(block[1].item()) == 0   # counter advanced, ticket reset
  # frequencies over >= 1M draws against softmax(logits)
  from scipy import stats
  A = 6
  z = (rng.randn(1, A) * 1.2).astype(f32)
  zd = _dev(cuda, np.tile(z, (1 << 20, 1)))
  counts = np.bincount(_sample(cuda, zd, torch.zeros(2, dtype=torch.int64, device=cuda), seed).cpu().numpy(),
                       minlength=A)
  p = torch.softmax(torch.tensor(z[0], dtype=torch.float64), 0).numpy()
  assert stats.chisquare(counts, p * counts.sum()).pvalue > 1e-4


def test_sampling_under_graph_replay_draws_fresh_values(cuda):
  z = torch.randn(2048, 6, device=cuda)
  block = torch.zeros(2, dtype=torch.int64, device=cuda)
  out = torch.empty(2048, dtype=torch.int32, device=cuda)
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  g = torch.cuda.CUDAGraph()
  with torch.cuda.stream(s):
    _lib.call('b200rl_categorical_sample', _lib.ptr(z), 6, 2048, 6, 7, _lib.ptr(block), _lib.ptr(out),
              _lib.stream())                                   # warm-up (call 0)
    torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=s):
      _lib.call('b200rl_categorical_sample', _lib.ptr(z), 6, 2048, 6, 7, _lib.ptr(block), _lib.ptr(out),
                _lib.stream())
  torch.cuda.current_stream().wait_stream(s)
  g.replay()
  first = out.clone()
  g.replay()
  second = out.clone()
  torch.cuda.synchronize()
  assert int(block[0].item()) == 3
  assert not torch.equal(first, second)
  want1, _ = opd.categorical_sample(z.cpu().numpy(), 7, 1)
  assert (first.cpu().numpy() == want1).mean() > 0.99


# ---- networks / policy / agent -----------------------------------------------------------------
def _nets(cuda, obs_spec, act_spec, hidden=(64, 32), act='tanh', conv=None):
  extra = {}
  if conv is not None:
    extra = dict(preprocessing_layers=L.CastScale(255.), conv_layer_params=conv)
  actor = actor_distribution_network.ActorDistributionNetwork(
      obs_spec, act_spec, fc_layer_params=hidden, activation_fn=act, device=cuda, **extra).set_seed(1)
  extra = dict(extra)
  if conv is not None:
    extra['preprocessing_layers'] = L.CastScale(255.)
  value = value_network.ValueNetwork(obs_spec, fc_layer_params=hidden, activation_fn=act, device=cuda,
                                     **extra).set_seed(2)
  return actor, value


def _mirror(net):
  layers = []
  for l in net.layers:
    if isinstance(l, L.CastScale):
      layers.append(dict(kind='cast_scale', divisor=l.divisor))
    elif isinstance(l, L.Conv2D):
      layers.append(dict(kind='conv', w=l.kernel.cpu().numpy().copy(), b=l.bias.cpu().numpy().copy(),
                         stride=l.stride, act=l.activation))
    elif isinstance(l, L.Flatten):
      layers.append(dict(kind='flatten'))
    elif isinstance(l, L.Dense):
      layers.append(dict(kind='dense', w=l.kernel.cpu().numpy().copy(), b=l.bias.cpu().numpy().copy(),
                         act=l.activation))
  return onn.Sequential(layers)


def test_policy_collect_and_greedy(cuda):
  obs_spec = tensor_spec.TensorSpec((17,), torch.float32, 'observation')
  for dtype, shape in ((torch.int64, ()), (torch.int32, (1,))):
    act_spec = tensor_spec.BoundedTensorSpec(shape, dtype, 0, 17, 'action')
    actor, value = _nets(cuda, obs_spec, act_spec, hidden=(32,))
    agent = ppo_clip_agent.PPOClipAgent(ts.time_step_spec(obs_spec), act_spec, optimizer=optimizers.Adam(1e-3),
                                        actor_net=actor, value_net=value, importance_ratio_clipping=0.2,
                                        use_gae=True, normalize_observations=False)
    agent.initialize()
    obs = torch.randn(4096, 17, device=cuda)
    step = agent.collect_policy.action(ts.restart(obs, batch_size=4096))
    assert step.action.dtype == dtype and tuple(step.action.shape) == (4096,) + shape
    assert int(step.action.min()) >= 0 and int(step.action.max()) < 18
    assert set(step.info) == {'dist_params'} and set(step.info['dist_params']) == {'logits'}
    logits = step.info['dist_params']['logits']
    assert tuple(logits.shape) == (4096, 18)
    torch.testing.assert_close(logits, actor(obs)[0])
    step2 = agent.collect_policy.action(ts.restart(obs, batch_size=4096))
    assert not torch.equal(step.action, step2.action)
    greedy = agent.policy.action(ts.restart(obs, batch_size=4096))
    assert greedy.info == ()
    np.testing.assert_array_equal(greedy.action.reshape(-1).cpu().numpy(),
                                  logits.cpu().numpy().argmax(axis=1))
  # ties: the mode is the FIRST argmax
  net_logits = torch.tensor([[1., 3., 3., 0.], [2., 2., 2., 2.], [0., -1., 5., 5.]], device=cuda)
  out = torch.empty(3, dtype=torch.int32, device=cuda)
  blk = torch.zeros(2, dtype=torch.int64, device=cuda)
  _lib.call('b200rl_epsilon_greedy', _lib.ptr(net_logits), None, 3, 4, 0.0, 1, _lib.ptr(blk), None, None,
            _lib.ptr(out), _lib.stream())
  assert out.cpu().tolist() == [1, 0, 2]


def _experience(rng, B, T, obs_shape, A, u8=False):
  obs = (rng.randint(0, 256, (B, T) + obs_shape).astype(np.uint8) if u8
         else rng.randn(B, T, *obs_shape).astype(f32))
  e = dict(observation=obs, action=rng.randint(0, A, (B, T)).astype(np.int64),
           logits=(rng.randn(B, T, A) * 0.5).astype(f32), reward=rng.rand(B, T).astype(f32),
           discount=np.ones((B, T), f32), step_type=np.ones((B, T), np.int32),
           next_step_type=np.ones((B, T), np.int32))
  ends = rng.rand(B, T) < 0.05
  e['next_step_type'][ends] = 2
  e['discount'][ends] = 0
  e['step_type'][:, 1:][ends[:, :-1]] = 2
  return e


def _to_traj(cuda, e, extra_info=None):
  d = lambda a: torch.as_tensor(a, device=cuda)
  info = {'dist_params': {'logits': d(e['logits'])}}
  for k in (extra_info or ()):
    info[k] = d(e[k])
  return trajectory.Trajectory(d(e['step_type']), d(e['observation']), d(e['action']), info,
                               d(e['next_step_type']), d(e['reward']), d(e['discount']))


def _check_params(tag, nets, orc, steps, lr):
  """Post-Adam parameters: at most 0.1 % of elements beyond 2e-3 relative + 2e-5, none beyond
  steps * lr (Adam moves a parameter by at most ~lr per step, so a 1e-7 gradient difference on a
  near-zero gradient can flip a whole step)."""
  got = np.concatenate([v.cpu().numpy().reshape(-1) for n in nets for v in n.variables])
  want = np.concatenate([p.reshape(-1) for p in orc.params()])
  err = np.abs(got - want)
  out = err > 2e-3 * np.abs(want) + 2e-5
  record_parity(tag, param_max_abs=float(err.max()), param_outlier_frac=float(out.mean()))
  assert out.mean() <= 1e-3, out.mean()
  assert err.max() <= steps * lr, err.max()


@pytest.mark.parametrize('kind', ['clip', 'kl'])
def test_agent_train_parity_mlp(cuda, kind):
  rng = np.random.RandomState(7)
  B, T, D, A, epochs = 32, 17, 17, 18, 3
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int64, 0, A - 1, 'action')
  actor, value = _nets(cuda, obs_spec, act_spec)
  common_kw = dict(use_gae=True, lambda_value=0.95, discount_factor=0.99, num_epochs=epochs,
                   normalize_rewards=True, normalize_observations=True, entropy_regularization=0.01)
  okw = dict(num_epochs=epochs, vf_coef=0.5, ent_coef=0.01, gamma=0.99, lam=0.95, normalize_rewards=True,
             normalize_observations=True, obs_dim=D)
  if kind == 'clip':
    agent = ppo_clip_agent.PPOClipAgent(ts.time_step_spec(obs_spec), act_spec, optimizer=optimizers.Adam(1e-3),
                                        actor_net=actor, value_net=value, importance_ratio_clipping=0.2,
                                        gradient_clipping=0.5, value_clipping=0.2, **common_kw)
    okw.update(clip_eps=0.2, gradient_clipping=0.5, value_clip=0.2)
  else:
    kl = dict(kl_cutoff_factor=2.0, kl_cutoff_coef=1000.0, initial_adaptive_kl_beta=1.0,
              adaptive_kl_target=0.01, adaptive_kl_tolerance=0.3)
    agent = ppo_agent.PPOAgent(ts.time_step_spec(obs_spec), act_spec, optimizers.Adam(1e-3), actor_net=actor,
                               value_net=value, importance_ratio_clipping=0.0, **kl, **common_kw)
    okw.update(clip_eps=0.0, **kl)
  agent.initialize()
  orc = opd.CategoricalPPOOracle(_mirror(actor), _mirror(value), ooptim.AdamTF(1e-3, eps=1e-7), **okw)
  for _ in range(3):
    e = _experience(rng, B, T, (D,), A)
    want = orc.train(e)[-1]
    got = agent.train(_to_traj(cuda, e))
    rel = abs(got.loss.item() - want['loss']) / max(abs(want['loss']), 1e-30)
    record_parity('ppo_discrete_train_' + kind, loss_rel=rel)
    np.testing.assert_allclose(got.loss.item(), want['loss'], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(got.extra.policy_gradient_loss.item(), want['pg'], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(got.extra.value_estimation_loss.item(), want['ve'], rtol=1e-5)
    np.testing.assert_allclose(got.extra.entropy_regularization_loss.item(), want['ent'], rtol=1e-5)
    np.testing.assert_allclose(got.extra.kl_penalty_loss.item(), want['kl'], rtol=1e-5, atol=1e-7)
    if kind == 'kl':
      np.testing.assert_allclose(agent._adaptive_kl_beta.item(), orc.beta, rtol=1e-6)
  assert int(agent.train_step_counter.item()) == 3 * epochs
  _check_params('ppo_discrete_train_' + kind, [actor, value], orc, 3 * epochs, 1e-3)
  agent.check_numerics()


def test_agent_train_parity_conv_torso(cuda):
  rng = np.random.RandomState(8)
  B, T, A, epochs = 4, 8, 6, 2
  obs_spec = tensor_spec.TensorSpec((84, 84, 4), torch.uint8, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, A - 1, 'action')
  conv = ((32, 8, 4), (64, 4, 2), (64, 3, 1))
  actor, value = _nets(cuda, obs_spec, act_spec, hidden=(512,), act='relu', conv=conv)
  agent = ppo_clip_agent.PPOClipAgent(ts.time_step_spec(obs_spec), act_spec, optimizer=optimizers.Adam(2.5e-4),
                                      actor_net=actor, value_net=value, importance_ratio_clipping=0.1,
                                      use_gae=True, num_epochs=epochs, normalize_observations=False,
                                      normalize_rewards=False, entropy_regularization=0.01)
  agent.initialize()
  orc = opd.CategoricalPPOOracle(_mirror(actor), _mirror(value), ooptim.AdamTF(2.5e-4, eps=1e-7),
                                 num_epochs=epochs, clip_eps=0.1, vf_coef=0.5, ent_coef=0.01)
  for _ in range(2):
    e = _experience(rng, B, T, (84, 84, 4), A, u8=True)
    want = orc.train(e)[-1]
    got = agent.train(_to_traj(cuda, e))
    record_parity('ppo_discrete_train_conv',
                  loss_rel=abs(got.loss.item() - want['loss']) / max(abs(want['loss']), 1e-30))
    np.testing.assert_allclose(got.loss.item(), want['loss'], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(got.extra.value_estimation_loss.item(), want['ve'], rtol=1e-5)
    np.testing.assert_allclose(got.extra.entropy_regularization_loss.item(), want['ent'], rtol=1e-5)
  _check_params('ppo_discrete_train_conv', [actor, value], orc, 2 * epochs, 2.5e-4)
  agent.check_numerics()


def test_ppo_learner_minibatches(cuda, tmp_path):
  rng = np.random.RandomState(5)
  B, T, D, A, mb, epochs, buf, seed = 16, 13, 17, 6, 30, 3, 50, 9
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int64, 0, A - 1, 'action')
  actor, value = _nets(cuda, obs_spec, act_spec)
  agent = ppo_clip_agent.PPOClipAgent(
      ts.time_step_spec(obs_spec), act_spec, optimizer=optimizers.Adam(1e-3), actor_net=actor, value_net=value,
      importance_ratio_clipping=0.2, use_gae=True, lambda_value=0.95, discount_factor=0.99, num_epochs=1,
      normalize_observations=False, normalize_rewards=False, compute_value_and_advantage_in_train=False,
      update_normalizers_in_train=False)
  agent.initialize()
  orc = opd.CategoricalPPOOracle(_mirror(actor), _mirror(value), ooptim.AdamTF(1e-3, eps=1e-7), num_epochs=1,
                                 clip_eps=0.2, vf_coef=0.5, gamma=0.99, lam=0.95)
  batches = []
  for _ in range(2):
    e = _experience(rng, B, T, (D,), A)
    e['value_prediction'] = rng.randn(B, T).astype(f32)
    batches.append(e)

  def dataset():
    while True:
      for e in batches:
        yield agent.preprocess_sequence(_to_traj(cuda, e, ['value_prediction'])), ()

  lrn = ppo_learner.PPOLearner(str(tmp_path), agent.train_step_counter, agent, dataset, dataset,
                               num_samples=2, num_epochs=epochs, minibatch_size=mb, shuffle_buffer_size=buf,
                               checkpoint_interval=0, seed=seed)
  n = 2 * B * T
  per_run = opl.iterations_per_run(n, 2, epochs, mb, 1)
  info = lrn.run()
  pre = [orc.preprocess_sequence(e) for e in batches]
  flat = {k: np.concatenate([p[k].reshape((B * T,) + p[k].shape[2:]) for p in pre], 0) for k in pre[0]}
  rows = opl.minibatch_rows(n, epochs, mb, buf, (seed ^ ppo_learner._SHUFFLE_SEED_TAG), 0)
  infos = [orc.train({k: v[r][:, None] for k, v in flat.items()}, preprocessed=True,
                     update_normalizers=False)[-1] for r in rows[:per_run]]
  np.testing.assert_allclose(info.loss.item(), infos[-1]['loss'], rtol=2e-5, atol=1e-6)
  np.testing.assert_allclose(info.extra.value_estimation_loss.item(), infos[-1]['ve'], rtol=2e-5)
  assert int(agent.train_step_counter.item()) == per_run
  _check_params('ppo_discrete_learner', [actor, value], orc, per_run, 1e-3)


def test_graph_captured_train_matches_eager(cuda):
  rng = np.random.RandomState(6)
  B, T, D, A = 4, 16, 5, 3                     # N = 64: the loss kernel runs as a single CTA
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, A - 1, 'action')

  def make():
    actor, value = _nets(cuda, obs_spec, act_spec, hidden=(16,))
    agent = ppo_agent.PPOAgent(ts.time_step_spec(obs_spec), act_spec, optimizers.Adam(1e-3), actor_net=actor,
                               value_net=value, use_gae=True, num_epochs=2, normalize_observations=False,
                               normalize_rewards=False, importance_ratio_clipping=0.2,
                               initial_adaptive_kl_beta=1.0, kl_cutoff_factor=2.0)
    agent.initialize()
    return agent

  eager, graphed = make(), make()
  train_fn = common.function(graphed.train)
  e = _experience(rng, B, T, (D,), A)
  traj = _to_traj(cuda, e)
  for _ in range(5):
    l1 = eager.train(traj).loss.item()
    l2 = train_fn(traj).loss.item()
    np.testing.assert_allclose(l2, l1, rtol=1e-6)
  # Inside a captured graph the parameter gradients run on a side stream (network.backward), so
  # their fp32 sums may round differently from the eager order: parameters agree to rounding.
  diff = (eager._flat_params - graphed._flat_params).abs().max().item()
  record_parity('ppo_discrete_graph_vs_eager', param_max_abs=diff)
  torch.testing.assert_close(graphed._flat_params, eager._flat_params, rtol=1e-5, atol=1e-6)
  torch.testing.assert_close(graphed._adaptive_kl_beta, eager._adaptive_kl_beta, rtol=1e-6, atol=0)


def test_cartpole_end_to_end_learns(cuda):
  """Device CartPole -> DynamicStepDriver(collect policy) -> TFUniformReplayBuffer -> gather_all
  -> PPOClipAgent.train -> clear, 40 iterations of 16 envs x 128 steps; then the greedy policy's
  mean first-episode length over 16 evaluation envs must reach 100.
  Threshold: the same configuration run on the CPU through oracle/ppo_discrete.py (oracle
  CartPole, oracle categorical draws) gave 294, 455, 132, 470, 500, 140, 358 and 184
  for seeds 0-7 after 40 iterations (median ~325); an untrained policy lasts ~20 steps.  100 sits
  below the smallest of those with margin and is ~5x the untrained length."""
  from agents_b200.drivers import dynamic_step_driver
  from agents_b200.environments import random_tf_environment
  from agents_b200.replay_buffers import tf_uniform_replay_buffer as rb_mod
  B, T, iters = 16, 128, 40
  env = random_tf_environment.CartPoleTFEnvironment(batch_size=B, seed=0, device=cuda)
  tss, act_spec = env.time_step_spec(), env.action_spec()
  actor, value = _nets(cuda, tss.observation, act_spec, hidden=(64, 64))
  agent = ppo_clip_agent.PPOClipAgent(tss, act_spec, optimizer=optimizers.Adam(1e-3), actor_net=actor,
                                      value_net=value, importance_ratio_clipping=0.2, use_gae=True,
                                      lambda_value=0.95, discount_factor=0.99, num_epochs=10)
  agent.initialize()
  rb = rb_mod.TFUniformReplayBuffer(agent.collect_data_spec, batch_size=B, max_length=T, device=cuda)
  driver = dynamic_step_driver.DynamicStepDriver(env, agent.collect_policy, observers=[rb.add_batch],
                                                 num_steps=B * T)
  time_step, policy_state = env.reset(), None
  for _ in range(iters):
    time_step, policy_state = driver.run(time_step, policy_state, maximum_iterations=T)
    exp = rb.gather_all()
    assert tuple(exp.action.shape) == (B, T) and set(exp.policy_info['dist_params']) == {'logits'}
    agent.train(exp)
    rb.clear()
  agent.check_numerics()
  ev = random_tf_environment.CartPoleTFEnvironment(batch_size=16, seed=7, device=cuda)
  step = ev.reset()
  length = torch.zeros(16, dtype=torch.int32, device=cuda)
  alive = torch.ones(16, dtype=torch.bool, device=cuda)
  for _ in range(500):
    step = ev.step(agent.policy.action(step).action)
    length += alive.to(torch.int32)
    alive &= step.step_type != ts.StepType.LAST
    if not bool(alive.any()):
      break
  mean_len = float(length.float().mean())
  record_parity('ppo_discrete_cartpole', mean_episode_length=mean_len)
  assert mean_len >= 100, mean_len
