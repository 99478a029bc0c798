"""DDPG on the GPU: the ddpg.cu kernels against float64 and the reference goldens, the OU noise
(supplied and device draws), DdpgAgent.train against the numpy oracle, gradients before the
optimiser, graph replay of train and of the collect policy, Learner checkpoints, the policies, and
an offline learning check."""
import tempfile

import numpy as np
import pytest
import torch

import grad_refs as R
from conftest import record_parity
from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.agents.ddpg import ddpg_agent
from agents_b200.networks import actor_network
from agents_b200.networks import critic_network
from agents_b200.networks import layers as L
from agents_b200.policies import ou_noise_policy
from agents_b200.specs import tensor_spec
from agents_b200.train import learner as learner_lib
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory
from agents_b200.utils import common
from oracle import ddpg as oddpg
from oracle import nn as onn
from oracle import optim as ooptim

pytestmark = pytest.mark.gpu
f32 = np.float32
F64 = torch.float64


def _d(cuda, a):
  return torch.as_tensor(np.ascontiguousarray(a, dtype=f32), device=cuda)


def _specs(D, A, lo=-1.0, hi=1.0):
  obs = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act = tensor_spec.BoundedTensorSpec((A,), torch.float32, lo, hi, 'action')
  return obs, act


def _make(cuda, D=17, A=6, actor_fc=(400, 300), obs_fc=(400,), joint_fc=(300,), lr=1e-3,
          bounds=(-1.0, 1.0), **kw):
  obs_spec, act_spec = _specs(D, A, *bounds)
  actor = actor_network.ActorNetwork(obs_spec, act_spec, fc_layer_params=actor_fc,
                                     device=cuda).set_seed(1)
  critic = critic_network.CriticNetwork((obs_spec, act_spec), observation_fc_layer_params=obs_fc,
                                        joint_fc_layer_params=joint_fc, device=cuda).set_seed(2)
  agent = ddpg_agent.DdpgAgent(ts.time_step_spec(obs_spec), act_spec, actor_network=actor,
                               critic_network=critic, actor_optimizer=optimizers.Adam(lr),
                               critic_optimizer=optimizers.Adam(lr), **kw)
  agent.initialize()
  return agent


def _seq(dense_layers):
  return onn.Sequential([dict(kind='dense', w=l.kernel.cpu().numpy().copy(),
                              b=l.bias.cpu().numpy().copy(), act=l.activation)
                         for l in dense_layers])


def _mirror_critic(net):
  dense = [l for l in net.layers if isinstance(l, L.Dense)]
  k = net._n_obs_layers
  return oddpg.Critic(_seq(dense[k:]), _seq(dense[:k]) if k else None)


def _oracle(agent, **kw):
  a = agent._actor_network
  return oddpg.DdpgOracle(_seq(a.layers), _mirror_critic(agent._critic_network),
                          a.action_min.cpu().numpy(), a.action_max.cpu().numpy(), **kw)


def _batch(rng, B, D, A):
  return dict(observation=rng.randn(B, 2, D).astype(f32),
              action=rng.uniform(-1, 1, (B, 2, A)).astype(f32),
              reward=(rng.randn(B, 2) * 2).astype(f32),
              discount=(rng.rand(B, 2) > .1).astype(f32))


def _traj(cuda, e):
  B = e['reward'].shape[0]
  one = torch.ones(B, 2, dtype=torch.int32, device=cuda)
  return trajectory.Trajectory(one, _d(cuda, e['observation']), _d(cuda, e['action']), (), one,
                               _d(cuda, e['reward']), _d(cuda, e['discount']))


def _critic_loss(cuda, q, tq, r, d, w, B, gamma, rs, kind):
  loss, dq, y = (torch.empty(1, device=cuda), torch.empty(B, device=cuda),
                 torch.empty(B, device=cuda))
  ins = [_d(cuda, a) for a in (q, tq, r, d)]           # held until the call has been enqueued
  tw = None if w is None else _d(cuda, w)
  _lib.call('b200rl_ddpg_critic_loss', *[_lib.ptr(t) for t in ins], _lib.ptr(tw), B, gamma, rs,
            kind, _lib.ptr(loss), _lib.ptr(dq), _lib.ptr(y), None, _lib.stream())
  return loss, dq, y


def _actor_loss(cuda, dqda, off, A, w, clip, lo, hi):
  B, ld = dqda.shape
  loss = torch.empty(1, device=cuda)
  dy = torch.full((B * A + 7,), 7.0, device=cuda)               # canary tail
  src, tlo, thi = _d(cuda, dqda), _d(cuda, lo), _d(cuda, hi)
  tw = None if w is None else _d(cuda, w)
  _lib.call('b200rl_ddpg_actor_loss', src.data_ptr() + 4 * off, ld, _lib.ptr(tw), B, A,
            int(clip is not None), 0.0 if clip is None else clip, _lib.ptr(tlo), _lib.ptr(thi),
            _lib.ptr(loss), _lib.ptr(dy), None, _lib.stream())
  assert bool((dy[B * A:] == 7).all())
  assert np.array_equal(src.cpu().numpy(), dqda)             # the critic's gradient is read only
  return loss, dy[:B * A].reshape(B, A)


# ---- 1. kernels against float64 -----------------------------------------------------------------
@pytest.mark.parametrize('B', [1, 7, 256, 1000, 5000])
@pytest.mark.parametrize('A', [1, 6, 17])
def test_kernels_match_float64(cuda, B, A):
  rng = np.random.RandomState(B * 37 + A)
  lo = rng.uniform(-3, -0.5, A).astype(f32)
  hi = rng.uniform(0.5, 2, A).astype(f32)
  LO, HI = R.t64(lo), R.t64(hi)
  for kind in (_lib.LOSS_HUBER, _lib.LOSS_SQUARED):
    for weighted in (False, True):
      q, tq = (rng.randn(B) * 2).astype(f32), (rng.randn(B) * 2).astype(f32)
      r, dsc = (rng.randn(B) * 2).astype(f32), (rng.rand(B) > .2).astype(f32)
      w = rng.rand(B).astype(f32) if weighted else None
      loss, dq, yt = _critic_loss(cuda, q, tq, r, dsc, w, B, 0.97, 1.3, kind)
      Q = R.t64(q).requires_grad_()
      yref = 1.3 * R.t64(r) + 0.97 * R.t64(dsc) * R.t64(tq)
      el = R.huber if kind == _lib.LOSS_HUBER else (lambda e: e * e)
      W = torch.ones(B, dtype=F64) if w is None else R.t64(w)
      ref = (el(yref - Q) * W).sum() / B
      np.testing.assert_allclose(loss.item(), ref.item(), rtol=1e-5)
      torch.testing.assert_close(yt.cpu().double(), yref, rtol=1e-6, atol=1e-5)
      R.assert_grad_close('ddpg dq', dq, torch.autograd.grad(ref, Q)[0], 1e-5, 1e-5)
  ld, off = A + 5, 3                                   # strided rows, like a critic's input gradient
  dqda = (rng.randn(B, ld) * 0.6).astype(f32)          # about 40 % of |dqda| exceed 0.5
  D = R.t64(dqda[:, off:off + A])
  for clip in (None, 0.5, 0.0):
    for weighted in (False, True):
      w = rng.rand(B).astype(f32) if weighted else None
      loss, dy = _actor_loss(cuda, dqda, off, A, w, clip, lo, hi)
      W = (torch.ones(B, dtype=F64) if w is None else R.t64(w))[:, None]
      c = D if clip is None else D.clamp(-clip, clip)
      ref = (c * c * W).sum() / (B * A)
      want_dy = (HI - LO) / 2 * (-2 * W * c / (B * A))
      np.testing.assert_allclose(loss.item(), ref.item(), rtol=1e-5, atol=0)
      torch.testing.assert_close(dy.cpu().double(), want_dy, rtol=2e-6, atol=0)
      if clip == 0.0:                                  # clipped to [0, 0]: no actor gradient
        assert loss.item() == 0 and not bool(dy.any())
  # OU step with supplied draws, written at a row stride between canary columns
  x0 = rng.randn(A).astype(f32)
  z = rng.randn(A).astype(f32)
  tz, tlo, thi = _d(cuda, z), _d(cuda, lo), _d(cuda, hi)
  loc = rng.uniform(-2, 2, (B, ld)).astype(f32)
  for clamp in (False, True):
    state, tloc = _d(cuda, x0), _d(cuda, loc)
    ctr = torch.zeros(2, dtype=torch.int64, device=cuda)
    out = torch.full((B, ld), 7.0, device=cuda)
    _lib.call('b200rl_ou_noise', tloc.data_ptr() + 4 * off, ld, B, A, _lib.ptr(state), 0.15, 0.3,
              _lib.ptr(tz), 0, _lib.ptr(ctr), _lib.ptr(tlo) if clamp else None,
              _lib.ptr(thi) if clamp else None, out.data_ptr() + 4 * 2, ld, _lib.stream())
    xn = 0.85 * R.t64(x0) + 0.3 * R.t64(z)
    want = R.t64(loc[:, off:off + A]) + xn[None, :]
    if clamp:
      want = torch.minimum(torch.maximum(want, LO), HI)
    o = out.cpu()
    torch.testing.assert_close(state.cpu().double(), xn, rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(o[:, 2:2 + A].double(), want, rtol=1e-6, atol=1e-6)
    assert bool((o[:, :2] == 7).all()) and bool((o[:, 2 + A:] == 7).all())
    assert ctr.cpu().tolist() == [0, 0]                # supplied draws leave the call counter


def test_reference_goldens_through_the_kernels(cuda):
  # agents/ddpg/ddpg_agent_test.py testCriticLoss / testActorLoss
  loss, _, y = _critic_loss(cuda, np.array([21., 31.], f32), np.array([69., 89.], f32),
                            np.array([10., 20.], f32), np.array([.9, .9], f32), None, 2, 1.0, 1.0,
                            _lib.LOSS_HUBER)
  np.testing.assert_allclose(loss.item(), 59.6, rtol=1e-6)
  np.testing.assert_allclose(y.cpu().numpy(), [72.1, 100.1], rtol=1e-6)
  loss, _ = _actor_loss(cuda, np.full((2, 3), 2.0, f32), 2, 1, None, None, np.array([-1.], f32),
                        np.array([1.], f32))
  assert loss.item() == 4.0


# ---- 2. OU noise ----------------------------------------------------------------------------------
@pytest.mark.parametrize('clip', [False, True])
def test_ou_noise_supplied_draws_match_recurrence(cuda, clip):
  N, A, T, sigma, damping = 1500, 5, 20, 0.4, 0.2    # N * A spans 30 blocks
  rng = np.random.RandomState(21)
  lo, hi = np.array([-1, -2, -.5, -1, 0], f32), np.array([1, 2, .5, 3, 1], f32)
  loc = _d(cuda, rng.uniform(-1, 1, (N, A)) * hi)
  tlo, thi = _d(cuda, lo), _d(cuda, hi)
  state, ctr = torch.zeros(A, device=cuda), torch.zeros(2, dtype=torch.int64, device=cuda)
  x = torch.zeros(A, dtype=F64)
  clipped = 0
  for t in range(T):
    z = rng.randn(A).astype(f32)
    tz, out = _d(cuda, z), torch.empty(N, A, device=cuda)
    _lib.call('b200rl_ou_noise', _lib.ptr(loc), A, N, A, _lib.ptr(state), damping, sigma,
              _lib.ptr(tz), 0, _lib.ptr(ctr), _lib.ptr(tlo) if clip else None,
              _lib.ptr(thi) if clip else None, _lib.ptr(out), A, _lib.stream())
    x = (1 - damping) * x + sigma * R.t64(z)
    torch.testing.assert_close(state.cpu().double(), x, rtol=1e-6, atol=1e-7)
    want = R.t64(loc) + x[None, :]
    if clip:
      outside = (want < R.t64(lo)) | (want > R.t64(hi))
      clipped += int(outside.sum())
      want = torch.minimum(torch.maximum(want, R.t64(lo)), R.t64(hi))
    else:                                              # the same x on every row
      noise = (out - loc).cpu()
      assert float((noise - noise[:1]).abs().max()) <= 2e-7 * 4
    torch.testing.assert_close(out.cpu().double(), want, rtol=1e-6, atol=1e-6)
  assert ctr.cpu().tolist() == [0, 0]
  assert not clip or clipped > 100


def test_ou_noise_device_draws_match_closed_form_moments(cuda):
  A, T, sigma, damping = 4096, 200, 0.3, 0.1           # components are independent samples
  rho = 1.0 - damping
  loc = torch.zeros(1, A, device=cuda)
  state, ctr = torch.zeros(A, device=cuda), torch.zeros(2, dtype=torch.int64, device=cuda)
  out = torch.empty(1, A, device=cuda)
  xs = []
  for _ in range(T):
    _lib.call('b200rl_ou_noise', _lib.ptr(loc), A, 1, A, _lib.ptr(state), damping, sigma, None, 5,
              _lib.ptr(ctr), None, None, _lib.ptr(out), A, _lib.stream())
    assert torch.equal(out[0], state)
    xs.append(state.cpu().double().numpy().copy())
  assert ctr.cpu().tolist() == [T, 0]
  var = lambda t: sigma ** 2 * (1 - rho ** (2 * t)) / (1 - rho ** 2)
  worst = 0.0
  for t in range(1, T + 1):                            # 5 standard errors of each estimate
    x = xs[t - 1]
    v = var(t)
    assert abs(x.mean()) <= 5 * np.sqrt(v / A), t
    se = np.sqrt(2.0) * v / np.sqrt(A)
    assert abs(np.mean(x * x) - v) <= 5 * se, (t, np.mean(x * x), v)
    worst = max(worst, abs(np.mean(x * x) - v) / se)
    if t > 1:
      c, vp = rho * var(t - 1), var(t - 1)
      se_c = np.sqrt((v * vp + c * c) / A)
      assert abs(np.mean(x * xs[t - 2]) - c) <= 5 * se_c, (t, np.mean(x * xs[t - 2]), c)
  record_parity('ddpg_ou_device_moments', worst_var_z=worst)


# ---- 3. DdpgAgent.train against the oracle --------------------------------------------------------
_CONFIGS = [
    # (obs_fc, loss, weighted, dqda_clipping, gradient clipping, target_update_period, bounds)
    ((400,), oddpg.HUBER, True, 0.5, 0.5, 5, (-2.0, 3.0)),
    ((400,), oddpg.SQUARED, False, None, None, 1, (-1.0, 1.0)),
    ((400,), oddpg.HUBER, False, 0.0, None, 5, (-1.0, 1.0)),
    (None, oddpg.SQUARED, True, 0.0, None, 1, (-2.0, 3.0)),
    (None, oddpg.HUBER, False, None, 0.5, 5, (-2.0, 3.0)),
    (None, oddpg.HUBER, True, 0.03, None, 1, (-1.0, 1.0)),
]
# At these initialisations |dQ/da| is 0.006 / 0.03-0.06 / 0.08-0.13 at its 10th / 50th / 90th
# percentile, so 0.5 leaves dQ/da unclipped and 0.03 clips about half of it.


@pytest.mark.parametrize(
    'cfg', _CONFIGS, ids=lambda c: f'{c[0]}-{c[1]}-w{c[2]}-q{c[3]}-c{c[4]}-t{c[5]}-{c[6][0]}_{c[6][1]}')
def test_agent_train_matches_oracle(cuda, cfg):
  obs_fc, kind, weighted, dqda_clip, clip, tup, bounds = cfg
  D, A, B = 17, 6, 256
  fn = common.element_wise_huber_loss if kind == oddpg.HUBER else common.element_wise_squared_loss
  agent = _make(cuda, D, A, obs_fc=obs_fc, joint_fc=(300,) if obs_fc else (400, 300),
                target_update_tau=0.05, target_update_period=tup, td_errors_loss_fn=fn,
                gamma=0.99, reward_scale_factor=0.5, gradient_clipping=clip,
                dqda_clipping=dqda_clip, bounds=bounds)
  orc = _oracle(agent, actor_opt=ooptim.AdamTF(1e-3, eps=1e-7),
                critic_opt=ooptim.AdamTF(1e-3, eps=1e-7), gamma=0.99, reward_scale=0.5, tau=0.05,
                target_update_period=tup, loss=kind, dqda_clipping=dqda_clip,
                gradient_clipping=clip)
  rng = np.random.RandomState(7)
  name = 'ddpg_agent_train_' + '_'.join(str(c) for c in cfg)
  for step in range(6):
    e = _batch(rng, B, D, A)
    w = rng.rand(B).astype(f32) if weighted else None
    want = orc.train(e, w)
    got = agent.train(_traj(cuda, e), weights=None if w is None else _d(cuda, w))
    for k in ('critic_loss', 'actor_loss'):
      g, wv = getattr(got.extra, k).item(), float(want[k])
      record_parity(name, **{k + '_rel': abs(g - wv) / max(abs(wv), 1e-30)})
      np.testing.assert_allclose(g, wv, rtol=1e-5, atol=0, err_msg=f'step {step} {k}')
    np.testing.assert_allclose(got.loss.item(), want['loss'], rtol=1e-5)
    if dqda_clip == 0.0:
      assert got.extra.actor_loss.item() == 0.0
  assert int(agent.train_step_counter.item()) == 6
  assert int(agent._actor_optimizer.iterations(agent._actor_network.flat_params).item()) == 6
  # Parameters after six Adam steps, with the criterion of the baseline parity tests: Adam divides
  # by sqrt(v), so a last-bit difference in a near-zero gradient (a dead-ReLU path) can move a
  # parameter by up to lr per step.  At most 0.1 % of the elements may leave rtol 1e-3 / atol
  # 1e-5, and none by more than steps * lr.
  for net, ref in ((agent._actor_network, orc.actor), (agent._target_actor_network, orc.ta),
                   (agent._critic_network, orc.critic), (agent._target_critic_network, orc.tc)):
    got = np.concatenate([v.cpu().numpy().ravel() for v in net.variables])
    want = np.concatenate([w.ravel() for w in ref.params()])
    diff = np.abs(got - want)
    out = diff > 1e-5 + 1e-3 * np.abs(want)
    record_parity(name, **{net.name + '_outlier_frac': out.mean(), net.name + '_max_abs': diff.max()})
    assert out.mean() <= 1e-3 and diff.max() <= 6 * 1e-3, (net.name, out.mean(), diff.max())
  agent.check_numerics()


# ---- 4. gradients before the optimiser ------------------------------------------------------------
def _torch_critic(net):
  dense = [l for l in net.layers if isinstance(l, L.Dense)]
  return [(R.t64(l.kernel).requires_grad_(), R.t64(l.bias).requires_grad_(), l.activation)
          for l in dense], net._n_obs_layers


def _q64(layers, k, obs, act):
  h = R.mlp(layers[:k], obs) if k else obs
  return R.mlp(layers[k:], torch.cat([h, act], 1))[:, 0]


@pytest.mark.parametrize('obs_fc', [(400,), None])
def test_gradients_before_the_optimizer_match_float64(cuda, obs_fc):
  D, A, B = 17, 6, 256
  agent = _make(cuda, D, A, obs_fc=obs_fc, joint_fc=(300,), lr=0.0, gamma=0.9, dqda_clipping=0.03,
                bounds=(-2.0, 3.0))
  mean, mag = 0.5, 2.5                                   # scale_to_spec of the spec [-2, 3]
  rng = np.random.RandomState(9)
  agent._target_params.add_(torch.randn_like(agent._target_params) * 0.01)   # targets differ
  ta = [(R.t64(l.kernel), R.t64(l.bias), l.activation) for l in agent._target_actor_network.layers]
  tc, k = _torch_critic(agent._target_critic_network)
  e, w = _batch(rng, B, D, A), rng.rand(B).astype(f32)
  agent.train(_traj(cuda, e), weights=_d(cuda, w))
  obs, obs2, act = R.t64(e['observation'][:, 0]), R.t64(e['observation'][:, 1]), R.t64(e['action'][:, 0])
  W, r, dsc = R.t64(w), R.t64(e['reward'][:, 0]), R.t64(e['discount'][:, 0])
  a2 = mean + mag * R.mlp(ta, obs2)
  y = r + 0.9 * dsc * _q64(tc, k, obs2, a2)
  c, _ = _torch_critic(agent._critic_network)
  params = [t for l in c for t in l[:2]]
  ref = torch.autograd.grad((R.huber(y - _q64(c, k, obs, act)) * W).sum() / B, params)
  for i, (g, rf) in enumerate(zip(agent._critic_network._grad_views, ref)):
    e_ = R.grad_errors(g, rf)
    record_parity(f'ddpg_grads_critic_{obs_fc}', **{f'{i}_rel_l2': e_[0], f'{i}_max': e_[1]})
    R.assert_grad_close(f'ddpg critic/{i}', g, rf, 1e-4, 1e-4)
  pa = [(R.t64(l.kernel).requires_grad_(), R.t64(l.bias).requires_grad_(), l.activation)
        for l in agent._actor_network.layers]
  a = mean + mag * R.mlp(pa, obs)
  ad = a.detach().requires_grad_()
  dqda, = torch.autograd.grad(_q64(c, k, obs, ad).sum(), ad)
  cl = dqda.clamp(-0.03, 0.03)
  frac = float((dqda.abs() > 0.03).double().mean())
  record_parity(f'ddpg_grads_actor_{obs_fc}', dqda_clipped_frac=frac)
  assert 0.1 < frac < 0.9, frac                        # the clip binds on part of the batch
  aloss = (((a.detach() + cl) - a) ** 2 * W[:, None]).mean()
  ref = torch.autograd.grad(aloss, [t for l in pa for t in l[:2]])
  for i, (g, rf) in enumerate(zip(agent._actor_network._grad_views, ref)):
    e_ = R.grad_errors(g, rf)
    record_parity(f'ddpg_grads_actor_{obs_fc}', **{f'{i}_rel_l2': e_[0], f'{i}_max': e_[1]})
    R.assert_grad_close(f'ddpg actor/{i}', g, rf, 1e-4, 1e-4)


# ---- 5. graph replay ------------------------------------------------------------------------------
_SMALL = dict(D=6, A=2, actor_fc=(16,), obs_fc=(16,), joint_fc=(16,), target_update_tau=0.05,
              target_update_period=3, dqda_clipping=0.5, ou_stddev=0.3, ou_damping=0.15)


def test_graph_replay_matches_eager_bit_for_bit(cuda):
  eager, graphed = _make(cuda, **_SMALL), _make(cuda, **_SMALL)
  train_fn = common.function(graphed.train)
  rng = np.random.RandomState(11)
  for step in range(8):                                # crosses target-update steps
    traj = _traj(cuda, _batch(rng, 8, 6, 2))
    l1 = eager.train(traj)
    l2 = train_fn(traj)
    assert l1.extra.critic_loss.item() == l2.extra.critic_loss.item(), step
    assert l1.extra.actor_loss.item() == l2.extra.actor_loss.item(), step
  assert int(graphed.train_step_counter.item()) == 8 and graphed._train_step_host == 8
  assert torch.equal(eager._online_params, graphed._online_params)
  assert torch.equal(eager._target_params, graphed._target_params)


def test_captured_collect_step_matches_eager_calls(cuda):
  eager, graphed = _make(cuda, seed=4, **_SMALL), _make(cuda, seed=4, **_SMALL)
  step = ts.restart(torch.randn(5, 6, device=cuda), batch_size=5)
  act_fn = common.function(lambda t: graphed.collect_policy.action(t).action)
  for call in range(6):                                # 2 eager warm-up calls, capture, replays
    a1 = eager.collect_policy.action(step).action
    a2 = act_fn(step)
    assert torch.equal(a1, a2), call
    assert torch.equal(eager.collect_policy.ou_state, graphed.collect_policy.ou_state), call
  assert graphed.collect_policy._ou_rng.cpu().tolist() == [6, 0]


# ---- 6. Learner checkpoints -----------------------------------------------------------------------
def test_learner_checkpoint_restore_reproduces_losses_and_noise(cuda):
  # 8 rows: every launch is one CTA, so the step is bit-reproducible (larger batches split the
  # weight-gradient reductions over CTAs that add with float atomics, DESIGN.md §4)
  rng = np.random.RandomState(12)
  batches = [_batch(rng, 8, 6, 2) for _ in range(7)]
  step_obs = ts.restart(torch.randn(3, 6, device=cuda), batch_size=3)
  root = tempfile.mkdtemp()

  def make(perturb):
    from agents_b200.train.utils import train_utils
    step = train_utils.create_train_step(cuda)
    agent = _make(cuda, train_step_counter=step, **_SMALL)
    if perturb:                                        # other weights and noise, then restored
      agent._online_params.mul_(0.5)
      agent._target_params.mul_(0.5)
      agent.collect_policy.action(step_obs)
    it = iter([_traj(cuda, e) for e in batches])
    return agent, step, learner_lib.Learner(root, step, agent, experience_dataset_fn=lambda: it,
                                            checkpoint_interval=4)

  agent, step, lrn = make(False)
  for _ in range(3):
    agent.collect_policy.action(step_obs)
  lrn.run(iterations=4)
  want_act = [agent.collect_policy.action(step_obs).action.clone() for _ in range(3)]
  want = [agent.train(_traj(cuda, e)).extra for e in batches[4:]]
  agent2, step2, _ = make(True)
  assert int(step2.item()) == 4
  got_act = [agent2.collect_policy.action(step_obs).action.clone() for _ in range(3)]
  got = [agent2.train(_traj(cuda, e)).extra for e in batches[4:]]
  for g, w in zip(got_act, want_act):
    assert torch.equal(g, w)
  for g, w in zip(got, want):
    assert g.critic_loss.item() == w.critic_loss.item() and g.actor_loss.item() == w.actor_loss.item()


# ---- 7. policies ----------------------------------------------------------------------------------
def test_policies_stay_in_bounds_and_collect_noise_is_correlated(cuda):
  D, A, N = 5, 3, 512
  obs_spec, act_spec = _specs(D, A, -0.5, 2.0)
  actor = actor_network.ActorNetwork(obs_spec, act_spec, fc_layer_params=(32,), device=cuda).set_seed(3)
  critic = critic_network.CriticNetwork((obs_spec, act_spec), joint_fc_layer_params=(32,), device=cuda)
  agent = ddpg_agent.DdpgAgent(ts.time_step_spec(obs_spec), act_spec, actor, critic,
                               optimizers.Adam(1e-3), optimizers.Adam(1e-3), ou_stddev=0.5,
                               ou_damping=0.05)
  assert isinstance(agent.collect_policy, ou_noise_policy.OUNoisePolicy)
  actor.layers[-1].kernel.mul_(1000.0)                 # saturate tanh so clipping matters
  step = ts.restart(torch.randn(N, D, device=cuda), batch_size=N)
  g1, g2 = agent.policy.action(step).action, agent.policy.action(step).action
  assert torch.equal(g1, g2)
  raw, _ = actor(step.observation)
  torch.testing.assert_close(g1, raw.clamp(-0.5, 2.0))
  xs, prev = [], None
  for _ in range(60):
    c = agent.collect_policy.action(step).action
    x = agent.collect_policy.ou_state.clone()
    assert tuple(c.shape) == (N, A) and float(c.min()) >= -0.5 and float(c.max()) <= 2.0
    torch.testing.assert_close(c, (raw + x).clamp(-0.5, 2.0), rtol=0, atol=0)
    assert prev is None or not torch.equal(c, prev)
    prev = c
    xs.append(x.cpu().double().numpy())
  xs = np.stack(xs)                                    # [T, A]; rho = 0.95
  lag1 = np.sum(xs[1:] * xs[:-1]) / np.sum(xs[:-1] ** 2)
  assert lag1 > 0.8, lag1
  with pytest.raises(NotImplementedError):
    agent.collect_policy.distribution(step)
  int_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 3, 'action')
  from agents_b200.policies import random_tf_policy
  with pytest.raises(ValueError):
    ou_noise_policy.OUNoisePolicy(random_tf_policy.RandomTFPolicy(ts.time_step_spec(obs_spec),
                                                                  int_spec))


def test_optimizer_none_and_unsupported_loss_raise(cuda):
  obs_spec, act_spec = _specs(4, 2)
  actor = actor_network.ActorNetwork(obs_spec, act_spec, fc_layer_params=(8,), device=cuda)
  critic = critic_network.CriticNetwork((obs_spec, act_spec), joint_fc_layer_params=(8,), device=cuda)
  agent = ddpg_agent.DdpgAgent(ts.time_step_spec(obs_spec), act_spec, actor, critic)
  assert agent.policy is not None and agent.collect_policy is not None
  with pytest.raises(ValueError, match='Optimizer is undefined'):
    agent.train(_traj(cuda, _batch(np.random.RandomState(0), 4, 4, 2)))
  with pytest.raises(ValueError):
    ddpg_agent.DdpgAgent(ts.time_step_spec(obs_spec), act_spec, actor, critic,
                         td_errors_loss_fn=lambda y, q: (y - q).abs())


# ---- 8. learning -----------------------------------------------------------------------------------
def learning_task(seed, D=8, A=3, n=4096):
  """Offline, gamma 0: reward -||a - tanh(s W)||^2 over uniform random actions."""
  rng = np.random.RandomState(seed)
  Wm = (rng.randn(D, A) * 0.5).astype(f32)
  obs = rng.randn(n, 2, D).astype(f32)
  act = rng.uniform(-1, 1, (n, 2, A)).astype(f32)
  best = np.tanh(obs[:, 0] @ Wm).astype(f32)
  rew = -np.sum((act[:, 0] - best) ** 2, axis=1).astype(f32)
  data = dict(observation=obs, action=act, reward=np.stack([rew, rew], 1),
              discount=np.zeros((n, 2), f32))
  eval_obs = rng.randn(1024, D).astype(f32)
  return data, eval_obs, np.tanh(eval_obs @ Wm).astype(f32), rng


LEARN_STEPS, LEARN_B = 1500, 64
LEARN_KW = dict(target_update_tau=0.05, gamma=0.0)
# Greedy error mean ||pi(s) - tanh(s W)||^2 of the numpy oracle (oracle/ddpg.py) on this task with
# the same networks, optimisers and batches, seeds 0-7:
#   initial 1.657 1.574 1.561 1.494 1.141 1.485 1.557 1.502
#   after LEARN_STEPS 0.0315 0.0289 0.0308 0.0225 0.0343 0.0586 0.0533 0.0314
# The threshold is twice the worst of those and far below every initial error.
LEARN_THRESHOLD = 0.12


def test_offline_learning_reduces_greedy_error(cuda):
  data, eval_obs, eval_best, rng = learning_task(0)
  agent = _make(cuda, D=8, A=3, actor_fc=(64, 64), obs_fc=None, joint_fc=(64, 64), **LEARN_KW)
  obs_t = _d(cuda, eval_obs)

  def err():
    a = agent.policy.action(ts.restart(obs_t, batch_size=obs_t.shape[0])).action
    return float(((a.cpu().numpy() - eval_best) ** 2).sum(1).mean())

  e0 = err()
  full = {k: _d(cuda, v) for k, v in data.items()}
  one = torch.ones(LEARN_B, 2, dtype=torch.int32, device=cuda)
  for _ in range(LEARN_STEPS):
    idx = torch.as_tensor(rng.randint(0, data['reward'].shape[0], LEARN_B), device=cuda)
    traj = trajectory.Trajectory(one, full['observation'][idx], full['action'][idx], (), one,
                                 full['reward'][idx], full['discount'][idx])
    agent.train(traj)
  e1 = err()
  record_parity('ddpg_learning', initial=e0, final=e1)
  assert e1 < LEARN_THRESHOLD < e0, (e0, e1)
