"""TD3 on the GPU: the td3.cu kernels and the gated Adam against float64, the device noise,
Td3Agent.train against the numpy oracle, gradients before the optimiser, graph replay, Learner
checkpoints, the policies, the CriticNetwork observation branch, and an offline learning check."""
import tempfile

import numpy as np
import pytest
import torch

import grad_refs as R
from conftest import record_parity
from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.agents.td3 import td3_agent
from agents_b200.networks import actor_network
from agents_b200.networks import critic_network
from agents_b200.networks import layers as L
from agents_b200.specs import tensor_spec
from agents_b200.train import learner as learner_lib
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory
from agents_b200.utils import common
from oracle import nn as onn
from oracle import optim as ooptim
from oracle import td3 as otd3

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
  agent = td3_agent.Td3Agent(ts.time_step_spec(obs_spec), act_spec, actor_network=actor,
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
  return otd3.Critic(_seq(dense[k:]), _seq(dense[:k]) if k else None)


def _oracle(agent, **kw):
  a = agent._actor_network
  return otd3.Td3Oracle(_seq(a.layers), _mirror_critic(agent._critic_network_1),
                        _mirror_critic(agent._critic_network_2), a.action_min.cpu().numpy(),
                        a.action_max.cpu().numpy(), **kw)


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


# ---- 1. kernels against float64 -----------------------------------------------------------------
@pytest.mark.parametrize('B', [1, 7, 256, 1000, 5000])
@pytest.mark.parametrize('A', [1, 6, 17])
def test_kernels_match_float64(cuda, B, A):
  rng = np.random.RandomState(B * 31 + A)
  lo = rng.uniform(-3, -0.5, A).astype(f32)
  hi = rng.uniform(0.5, 2, A).astype(f32)
  ld = A + 5                                             # strided rows, like a critic's joint input
  y = np.tanh(rng.randn(B, ld) * 2).astype(f32)
  z = (rng.randn(B, A) * 2).astype(f32)
  tlo, thi, ty, tz = _d(cuda, lo), _d(cuda, hi), _d(cuda, y), _d(cuda, z)
  Y, Z, LO, HI = R.t64(y[:, 3:3 + A]), R.t64(z), R.t64(lo), R.t64(hi)
  base = (HI + LO) / 2 + (HI - LO) / 2 * Y
  for clamp, std in ((0, 0.0), (1, 0.0), (0, 0.3), (1, 0.3)):
    out = torch.full((B, ld), 7.0, device=cuda)
    _lib.call('b200rl_td3_scale_to_spec', ty.data_ptr() + 12, ld, B, A, _lib.ptr(tlo), _lib.ptr(thi),
              std, 0.5, _lib.ptr(tz) if std else None, 0, None, clamp, out.data_ptr() + 8, ld,
              _lib.stream())
    want = base + torch.clamp(std * Z, -0.5, 0.5)
    if clamp:
      want = torch.minimum(torch.maximum(want, LO), HI)
    o = out.cpu()
    torch.testing.assert_close(o[:, 2:2 + A].double(), want, rtol=1e-6, atol=1e-6)
    assert bool((o[:, :2] == 7).all()) and bool((o[:, 2 + A:] == 7).all())   # other columns kept
    if std and not clamp:                                # target actions may leave the spec
      assert B < 64 or bool(((o[:, 2:2 + A].double() > HI) | (o[:, 2:2 + A].double() < LO)).any())
  for kind in (_lib.LOSS_HUBER, _lib.LOSS_SQUARED):
    for weighted in (False, True):
      q1, q2, tq1, tq2 = [(rng.randn(B) * 2).astype(f32) for _ in range(4)]
      r, dsc = (rng.randn(B) * 2).astype(f32), (rng.rand(B) > .2).astype(f32)
      w = rng.rand(B).astype(f32) if weighted else None
      tens = [_d(cuda, a) for a in (q1, q2, tq1, tq2, r, dsc)]
      tw = _d(cuda, w) if weighted else None
      loss, g1, g2, yt = (torch.empty(1, device=cuda), torch.empty(B, device=cuda),
                          torch.empty(B, device=cuda), torch.empty(B, device=cuda))
      _lib.call('b200rl_td3_critic_loss', *[_lib.ptr(t) for t in tens], _lib.ptr(tw), B, 0.97, 1.3,
                kind, _lib.ptr(loss), _lib.ptr(g1), _lib.ptr(g2), _lib.ptr(yt), None, _lib.stream())
      Q1, Q2 = R.t64(q1).requires_grad_(), R.t64(q2).requires_grad_()
      yref = 1.3 * R.t64(r) + 0.97 * R.t64(dsc) * torch.minimum(R.t64(tq1), R.t64(tq2))
      el = (lambda e: R.huber(e)) if kind == _lib.LOSS_HUBER else (lambda e: e * e)
      W = torch.ones(B, dtype=F64) if w is None else R.t64(w)
      ref = ((el(yref - Q1) + el(yref - Q2)) * W).sum() / B
      d1, d2 = torch.autograd.grad(ref, (Q1, Q2))
      np.testing.assert_allclose(loss.item(), ref.item(), rtol=1e-5)
      torch.testing.assert_close(yt.cpu().double(), yref, rtol=1e-6, atol=1e-5)
      R.assert_grad_close('td3 dq1', g1, d1, 1e-5, 1e-5)
      R.assert_grad_close('td3 dq2', g2, d2, 1e-5, 1e-5)
  qa = (rng.randn(B) * 3).astype(f32)
  for weighted in (False, True):
    w = rng.rand(B).astype(f32) if weighted else None
    tq, tw = _d(cuda, qa), (_d(cuda, w) if weighted else None)
    loss, dq = torch.empty(1, device=cuda), torch.empty(B, device=cuda)
    _lib.call('b200rl_td3_actor_loss', _lib.ptr(tq), _lib.ptr(tw), B, _lib.ptr(loss), _lib.ptr(dq),
              None, _lib.stream())
    Q = R.t64(qa).requires_grad_()
    ref = (-Q * (torch.ones(B, dtype=F64) if w is None else R.t64(w))).sum() / B
    np.testing.assert_allclose(loss.item(), ref.item(), rtol=1e-5, atol=1e-7)
    R.assert_grad_close('td3 actor dq', dq, torch.autograd.grad(ref, Q)[0], 1e-6, 1e-6)
  da = rng.randn(B, ld).astype(f32)
  tda, dy = _d(cuda, da), torch.empty(B, A, device=cuda)
  _lib.call('b200rl_td3_actor_bwd', tda.data_ptr() + 4 * 4, ld, _lib.ptr(tlo), _lib.ptr(thi), B, A,
            _lib.ptr(dy), _lib.stream())
  torch.testing.assert_close(dy.cpu().double(), (HI - LO) / 2 * R.t64(da[:, 4:4 + A]), rtol=1e-6,
                             atol=1e-7)


def test_gated_adam_skips_the_whole_update(cuda):
  n = 1000
  rng = np.random.RandomState(2)
  p0, g = rng.randn(n).astype(f32), rng.randn(n).astype(f32)
  p, tg = _d(cuda, p0), _d(cuda, g)
  opt, ref = optimizers.Adam(0.01), ooptim.AdamTF(0.01, eps=1e-7)
  rp = [p0.copy()]
  counter = torch.zeros((), dtype=torch.int64, device=cuda)
  for step in range(7):
    opt.apply_flat(p, tg, gate=(counter, 3))
    if step % 3 == 0:
      ref.apply(rp, [g])
    counter += 1
    np.testing.assert_allclose(p.cpu().numpy(), rp[0], rtol=1e-6, atol=1e-7)
  assert int(opt.iterations(p).item()) == ref.t == 3


# ---- 2. device noise ------------------------------------------------------------------------------
def test_device_noise_moments_and_clip_fraction(cuda):
  N, A = 20000, 6
  y = torch.zeros(N, A, device=cuda)
  lo, hi = -torch.ones(A, device=cuda), torch.ones(A, device=cuda)
  rng = torch.zeros(2, dtype=torch.int64, device=cuda)
  out = torch.empty(N, A, device=cuda)
  _lib.call('b200rl_td3_scale_to_spec', _lib.ptr(y), A, N, A, _lib.ptr(lo), _lib.ptr(hi), 0.2, 100.0,
            None, 11, _lib.ptr(rng), 0, _lib.ptr(out), A, _lib.stream())
  x = out.cpu().double().numpy()
  assert abs(x.mean()) < 0.004 and abs(x.std() - 0.2) < 0.004
  assert rng.cpu().tolist() == [1, 0]
  _lib.call('b200rl_td3_scale_to_spec', _lib.ptr(y), A, N, A, _lib.ptr(lo), _lib.ptr(hi), 0.2, 0.1,
            None, 11, _lib.ptr(rng), 0, _lib.ptr(out), A, _lib.stream())
  x2 = out.cpu().double().numpy()
  frac = np.mean(np.abs(x2) == f32(0.1))
  assert abs(frac - 0.617) < 0.01                      # P(|N(0, 0.2)| > 0.1) = 0.6171
  assert np.abs(x2).max() <= f32(0.1) and not np.array_equal(np.abs(x) > 0.1, np.abs(x2) >= 0.1)
  assert rng.cpu().tolist() == [2, 0]


# ---- 3. Td3Agent.train against the oracle ---------------------------------------------------------
_CONFIGS = [
    # (obs_fc, period, target_update_period, loss, weighted, clipping, action bounds)
    ((400,), 2, 5, otd3.HUBER, True, 0.5, (-2.0, 3.0)),
    ((400,), 1, 1, otd3.SQUARED, False, None, (-1.0, 1.0)),
    (None, 2, 1, otd3.SQUARED, True, None, (-1.0, 1.0)),
    (None, 1, 5, otd3.HUBER, False, 0.5, (-2.0, 3.0)),
]


@pytest.mark.parametrize(
    'cfg', _CONFIGS, ids=lambda c: f'{c[0]}-p{c[1]}-t{c[2]}-{c[3]}-w{c[4]}-c{c[5]}-{c[6][0]}_{c[6][1]}')
def test_agent_train_matches_oracle(cuda, cfg):
  obs_fc, period, tup, kind, weighted, clip, bounds = cfg
  D, A, B = 17, 6, 256
  fn = common.element_wise_huber_loss if kind == otd3.HUBER else common.element_wise_squared_loss
  agent = _make(cuda, D, A, obs_fc=obs_fc, joint_fc=(300,) if obs_fc else (400, 300),
                target_update_tau=0.05, target_update_period=tup, actor_update_period=period,
                td_errors_loss_fn=fn, gamma=0.99, reward_scale_factor=0.5, gradient_clipping=clip,
                bounds=bounds)
  orc = _oracle(agent, actor_opt=ooptim.AdamTF(1e-3, eps=1e-7),
                critic_opt=ooptim.AdamTF(1e-3, eps=1e-7), gamma=0.99, reward_scale=0.5, tau=0.05,
                target_update_period=tup, actor_update_period=period, loss=kind,
                gradient_clipping=clip)
  rng = np.random.RandomState(7)
  name = 'td3_agent_train_' + '_'.join(str(c) for c in cfg)
  for step in range(6):
    e = _batch(rng, B, D, A)
    z = rng.randn(B, A).astype(f32)
    w = rng.rand(B).astype(f32) if weighted else None
    want = orc.train(e, z, w)
    got = agent.train(_traj(cuda, e), weights=None if w is None else _d(cuda, w), noise=(_d(cuda, z),))
    # atol 1e-6: the actor loss is a mean of Q values of both signs, ~1e-2 at these weights, so
    # its relative error is that of a cancelling sum (measured errors are recorded)
    for k in ('critic_loss', 'actor_loss'):
      g, wv = getattr(got.extra, k).item(), float(want[k])
      record_parity(name, **{k + '_rel': abs(g - wv) / max(abs(wv), 1e-6)})
      np.testing.assert_allclose(g, wv, rtol=1e-5, atol=1e-6, err_msg=f'step {step} {k}')
    np.testing.assert_allclose(got.loss.item(), want['loss'], rtol=1e-5, atol=1e-6)
  assert int(agent.train_step_counter.item()) == 6
  assert int(agent._actor_optimizer.iterations(agent._actor_network.flat_params).item()) == \
      orc.actor_updates
  # Parameters after six Adam steps, with the criterion of the baseline parity tests: Adam divides
  # by sqrt(v), so a last-bit difference in a near-zero gradient (a dead-ReLU path) can move a
  # parameter by up to lr per step.  At most 0.1 % of the elements may leave rtol 1e-3 / atol
  # 1e-5, and none by more than steps * lr.
  for net, ref in ((agent._actor_network, orc.actor), (agent._target_actor_network, orc.ta),
                   (agent._critic_network_1, orc.c1), (agent._target_critic_network_2, orc.t2)):
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
  agent = _make(cuda, D, A, obs_fc=obs_fc, joint_fc=(300,), lr=0.0, target_policy_noise=0.3,
                target_policy_noise_clip=0.4, gamma=0.9, bounds=(-2.0, 3.0))
  mean, mag = 0.5, 2.5                                   # scale_to_spec of the spec [-2, 3]
  rng = np.random.RandomState(9)
  agent._target_params.add_(torch.randn_like(agent._target_params) * 0.01)   # targets differ
  ta = [(R.t64(l.kernel), R.t64(l.bias), l.activation) for l in agent._target_actor_network.layers]
  t1, k = _torch_critic(agent._target_critic_network_1)
  t2, _ = _torch_critic(agent._target_critic_network_2)
  e, z, w = _batch(rng, B, D, A), rng.randn(B, A).astype(f32), rng.rand(B).astype(f32)
  agent.train(_traj(cuda, e), weights=_d(cuda, w), noise=(_d(cuda, z),))
  obs, obs2, act = R.t64(e['observation'][:, 0]), R.t64(e['observation'][:, 1]), R.t64(e['action'][:, 0])
  W, r, dsc = R.t64(w), R.t64(e['reward'][:, 0]), R.t64(e['discount'][:, 0])
  a2 = mean + mag * R.mlp(ta, obs2) + torch.clamp(0.3 * R.t64(z), -0.4, 0.4)
  y = r + 0.9 * dsc * torch.minimum(_q64(t1, k, obs2, a2), _q64(t2, k, obs2, a2))
  c1, _ = _torch_critic(agent._critic_network_1)
  c2, _ = _torch_critic(agent._critic_network_2)
  per = R.huber(y - _q64(c1, k, obs, act)) + R.huber(y - _q64(c2, k, obs, act))
  params = [t for l in c1 + c2 for t in l[:2]]
  ref = torch.autograd.grad((per * W).sum() / B, params)
  got = [g for n in (agent._critic_network_1, agent._critic_network_2) for g in n._grad_views]
  for i, (g, rf) in enumerate(zip(got, ref)):
    e_ = R.grad_errors(g, rf)
    record_parity(f'td3_grads_critic_{obs_fc}', **{f'{i}_rel_l2': e_[0], f'{i}_max': e_[1]})
    R.assert_grad_close(f'td3 critic/{i}', g, rf, 1e-4, 1e-4)
  pa = [(R.t64(l.kernel).requires_grad_(), R.t64(l.bias).requires_grad_(), l.activation)
        for l in agent._actor_network.layers]
  aloss = (-_q64(c1, k, obs, mean + mag * R.mlp(pa, obs)) * W).sum() / B
  ref = torch.autograd.grad(aloss, [t for l in pa for t in l[:2]])
  for i, (g, rf) in enumerate(zip(agent._actor_network._grad_views, ref)):
    e_ = R.grad_errors(g, rf)
    record_parity(f'td3_grads_actor_{obs_fc}', **{f'{i}_rel_l2': e_[0], f'{i}_max': e_[1]})
    R.assert_grad_close(f'td3 actor/{i}', g, rf, 1e-4, 1e-4)


# ---- 5. graph replay ------------------------------------------------------------------------------
def test_graph_replay_matches_eager_bit_for_bit(cuda):
  kw = dict(D=6, A=2, actor_fc=(16,), obs_fc=(16,), joint_fc=(16,), target_update_tau=0.05,
            target_update_period=3, actor_update_period=2)
  eager, graphed = _make(cuda, **kw), _make(cuda, **kw)
  train_fn = common.function(graphed.train)
  rng = np.random.RandomState(11)
  for step in range(8):                                # crosses gated-off and target-update steps
    traj = _traj(cuda, _batch(rng, 8, 6, 2))
    l1 = eager.train(traj)
    l2 = train_fn(traj)
    assert l1.extra.critic_loss.item() == l2.extra.critic_loss.item(), step
    assert l1.extra.actor_loss.item() == l2.extra.actor_loss.item(), step
  assert int(graphed.train_step_counter.item()) == 8 and graphed._train_step_host == 8
  assert torch.equal(eager._online_params, graphed._online_params)
  assert torch.equal(eager._target_params, graphed._target_params)


# ---- 6. Learner checkpoints -----------------------------------------------------------------------
def test_learner_checkpoint_restore_reproduces_losses(cuda):
  # 8 rows: every launch is one CTA, so the step is bit-reproducible (larger batches split the
  # weight-gradient reductions over CTAs that add with float atomics, DESIGN.md §4)
  rng = np.random.RandomState(12)
  batches = [_batch(rng, 8, 6, 2) for _ in range(7)]
  root = tempfile.mkdtemp()
  kw = dict(D=6, A=2, actor_fc=(16,), obs_fc=(16,), joint_fc=(16,), target_update_tau=0.05,
            target_update_period=3, actor_update_period=2)

  def make(perturb):
    from agents_b200.train.utils import train_utils
    step = train_utils.create_train_step(cuda)
    agent = _make(cuda, train_step_counter=step, **kw)
    if perturb:                                        # other weights, then restored
      agent._online_params.mul_(0.5)
      agent._target_params.mul_(0.5)
    it = iter([_traj(cuda, e) for e in batches])
    return agent, step, learner_lib.Learner(root, step, agent, experience_dataset_fn=lambda: it,
                                            checkpoint_interval=4)

  agent, step, lrn = make(False)
  lrn.run(iterations=4)
  want = [agent.train(_traj(cuda, e)).extra for e in batches[4:]]
  agent2, step2, _ = make(True)
  assert int(step2.item()) == 4
  got = [agent2.train(_traj(cuda, e)).extra for e in batches[4:]]
  for g, w in zip(got, want):
    assert g.critic_loss.item() == w.critic_loss.item() and g.actor_loss.item() == w.actor_loss.item()


# ---- 7. policies ----------------------------------------------------------------------------------
def test_policies_stay_in_bounds_and_collect_differs(cuda):
  D, A, N = 5, 3, 512
  obs_spec, act_spec = _specs(D, A, -0.5, 2.0)
  actor = actor_network.ActorNetwork(obs_spec, act_spec, fc_layer_params=(32,), device=cuda).set_seed(3)
  critic = critic_network.CriticNetwork((obs_spec, act_spec), joint_fc_layer_params=(32,), device=cuda)
  agent = td3_agent.Td3Agent(ts.time_step_spec(obs_spec), act_spec, actor, critic,
                             optimizers.Adam(1e-3), optimizers.Adam(1e-3), exploration_noise_std=0.5)
  actor.layers[-1].kernel.mul_(1000.0)                 # saturate tanh so clipping matters
  step = ts.restart(torch.randn(N, D, device=cuda), batch_size=N)
  g1, g2 = agent.policy.action(step).action, agent.policy.action(step).action
  c1, c2 = agent.collect_policy.action(step).action, agent.collect_policy.action(step).action
  assert torch.equal(g1, g2) and not torch.equal(c1, c2) and not torch.equal(g1, c1)
  for a in (g1, c1, c2):
    assert tuple(a.shape) == (N, A) and float(a.min()) >= -0.5 and float(a.max()) <= 2.0
  raw, _ = actor(step.observation)
  torch.testing.assert_close(g1, raw.clamp(-0.5, 2.0))
  assert float(((c1 == -0.5) | (c1 == 2.0)).float().mean()) > 0.2   # noise pushed past the bounds


# ---- 8. CriticNetwork observation branch ----------------------------------------------------------
def test_critic_observation_branch_matches_float64(cuda):
  D, A, N = 7, 3, 300
  obs_spec, act_spec = _specs(D, A)
  net = critic_network.CriticNetwork((obs_spec, act_spec), observation_fc_layer_params=(24, 20),
                                     joint_fc_layer_params=(16,), device=cuda).set_seed(4)
  net.create_variables()
  rng = np.random.RandomState(13)
  obs, act = rng.randn(N, D).astype(f32), (-rng.rand(N, A) * 2).astype(f32)   # negative actions
  dq = rng.randn(N, 1).astype(f32)
  q, _ = net((_d(cuda, obs), _d(cuda, act)))
  x = net.joint_input(_d(cuda, obs), _d(cuda, act))
  q2, tape = net.forward_train_joint(x)
  grads, dx = net.backward(tape, _d(cuda, dq), need_input_grad=True)
  layers, k = _torch_critic(net)
  O, Aa = R.t64(obs), R.t64(act).requires_grad_()
  ref = _q64(layers, k, O, Aa)
  torch.testing.assert_close(q.cpu().double(), ref.detach(), rtol=1e-5, atol=1e-5)
  assert torch.equal(q, q2[:, 0])
  params = [t for l in layers for t in l[:2]]
  refs = torch.autograd.grad((ref * R.t64(dq[:, 0])).sum(), params + [Aa])
  for i, (g, rf) in enumerate(zip(net._grad_views, refs[:-1])):
    R.assert_grad_close(f'obs-branch critic/{i}', g, rf, 1e-4, 1e-4)
  col = net.action_column
  assert col == 20 and tuple(dx.shape) == (N, 20 + A)
  R.assert_grad_close('obs-branch dQ/da', dx[:, col:], refs[-1], 1e-4, 1e-4)
  # the input gradient alone leaves the parameter gradients alone
  before = net.flat_grads.clone()
  net.backward(tape, _d(cuda, dq) * 3, need_input_grad=True, need_param_grads=False)
  assert torch.equal(before, net.flat_grads)
  with pytest.raises(NotImplementedError):
    critic_network.CriticNetwork((obs_spec, act_spec), action_fc_layer_params=(8,), device=cuda)


# ---- 9. learning -----------------------------------------------------------------------------------
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
LEARN_KW = dict(actor_update_period=2, target_update_tau=0.05, gamma=0.0,
                target_policy_noise=0.2, target_policy_noise_clip=0.5)
# Greedy error mean ||pi(s) - tanh(s W)||^2 of the numpy oracle (oracle/td3.py) on this task with
# the same networks, optimisers and batches, seeds 0-7:
#   initial 1.657 1.574 1.561 1.494 1.141 1.485 1.557 1.502
#   after LEARN_STEPS 0.0287 0.0282 0.0271 0.0172 0.0255 0.0503 0.0490 0.0289
# The threshold is twice the worst of those and far below every initial error.
LEARN_THRESHOLD = 0.1


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
  record_parity('td3_learning', initial=e0, final=e1)
  assert e1 < LEARN_THRESHOLD < e0, (e0, e1)
