"""QT-Opt on the GPU: the qtopt.cu kernels against float64 (CEM sample / refit with ties and the
variance floor, the TD loss, the continuous epsilon-greedy draw), the device draws' moments, the
reference golden through QtOptAgent, QtOptAgent.train against the numpy oracle in noise mode, the
delayed target chain, gradients before the optimiser, graph replay of train and of the collect
step, Learner checkpoints, the policies, and an offline learning check."""
import tempfile

import numpy as np
import pytest
import torch

import grad_refs as R
from conftest import record_parity
from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.agents.qtopt import qtopt_agent
from agents_b200.networks import critic_network
from agents_b200.networks import layers as L
from agents_b200.policies import epsilon_greedy_policy
from agents_b200.policies import qtopt_cem_policy
from agents_b200.policies import random_tf_policy
from agents_b200.policies.samplers import qtopt_cem_actions_sampler_continuous as samplers
from agents_b200.specs import tensor_spec
from agents_b200.train import learner as learner_lib
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory
from agents_b200.utils import common
from oracle import nn as onn
from oracle import optim as ooptim
from oracle import qtopt as oq
from oracle.td3 import Critic

pytestmark = pytest.mark.gpu
f32 = np.float32
F64 = torch.float64


def _d(cuda, a):
  return torch.as_tensor(np.ascontiguousarray(a, dtype=f32), device=cuda)


def _specs(D, A, lo=-1.0, hi=1.0):
  obs = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act = tensor_spec.BoundedTensorSpec((A,), torch.float32, lo, hi, 'action')
  return obs, act


def _make(cuda, D=17, A=6, obs_fc=(400,), joint_fc=(300,), bounds=(-1.0, 1.0), lr=1e-3, N=32,
          M=4, I=3, **kw):
  obs_spec, act_spec = _specs(D, A, *bounds)
  critic = critic_network.CriticNetwork((obs_spec, act_spec), observation_fc_layer_params=obs_fc,
                                        joint_fc_layer_params=joint_fc, device=cuda).set_seed(2)
  lo, hi = bounds
  agent = qtopt_agent.QtOptAgent(
      ts.time_step_spec(obs_spec), act_spec, critic, optimizers.Adam(lr),
      samplers.GaussianActionsSampler(act_spec), init_mean_cem=np.full(A, (lo + hi) / 2),
      init_var_cem=np.full(A, ((hi - lo) / 4) ** 2), num_samples_cem=N, num_elites_cem=M,
      num_iter_cem=I, **kw)
  agent.initialize()
  return agent


def _seq(dense_layers):
  return onn.Sequential([dict(kind='dense', w=l.kernel.cpu().numpy().copy(),
                              b=l.bias.cpu().numpy().copy(), act=l.activation)
                         for l in dense_layers])


def _mirror(net):
  dense = [l for l in net.layers if isinstance(l, L.Dense)]
  k = net._n_obs_layers
  return Critic(_seq(dense[k:]), _seq(dense[:k]) if k else None)


def _batch(rng, B, D, A, T=2, lo=-1.0, hi=1.0):
  return dict(observation=rng.randn(B, T, D).astype(f32),
              action=rng.uniform(lo, hi, (B, T, A)).astype(f32),
              reward=(rng.randn(B, T) * 2).astype(f32),
              discount=(rng.rand(B, T) > .1).astype(f32),
              step_type=rng.choice([0, 1, 1, 1, 2], (B, T)).astype(np.int32))


def _traj(cuda, e):
  st = torch.as_tensor(e['step_type'], device=cuda)
  return trajectory.Trajectory(st, _d(cuda, e['observation']), _d(cuda, e['action']), (), st,
                               _d(cuda, e['reward']), _d(cuda, e['discount']))


def _ref_refit(x, scores, M):
  """float64 (idx, mean, var) of the top M of scores [B, N] (ties to the lower index)."""
  idx = np.argsort(-scores.astype(np.float64), axis=1, kind='stable')[:, :M]
  el = np.take_along_axis(x.astype(np.float64), idx[:, :, None], axis=1)
  return idx, el.mean(1), el.var(1)


# ---- 1. kernels against float64 -----------------------------------------------------------------
_SHAPES = [(B, N, M, A) for B in (1, 37, 5000) for N in (1, 7, 32, 33, 100)
           for M in sorted({1, 4, N}) if M <= N for A in (1, 17)
           if B * N * A <= 5000 * 100 * 17]


@pytest.mark.parametrize('B,N,M,A', _SHAPES)
def test_cem_kernels_match_float64(cuda, B, N, M, A):
  rng = np.random.RandomState(B * 7 + N * 3 + M + A)
  C, pad = 3, 2                                        # observation columns, canary columns
  W = C + A + pad
  for lo, hi in ((-1.0, 1.0), (-2.0, 3.0)):
    amin, amax = np.full(A, lo, f32), np.full(A, hi, f32)
    tlo, thi = _d(cuda, amin), _d(cuda, amax)
    # cem_sample: tiling + draws, an [A] distribution broadcast to every state
    src = rng.randn(B, C + 1).astype(f32)               # row stride C + 1
    m0, v0 = rng.uniform(lo, hi, A).astype(f32), rng.uniform(0, 1, A).astype(f32)
    v0[0] = 0.0                                          # the variance floor
    z = rng.randn(B, N, A).astype(f32)
    x = torch.full((B * N, W), 7.0, device=cuda)
    ctr = torch.zeros(2, dtype=torch.int64, device=cuda)
    ins = [_d(cuda, a) for a in (src, m0, v0, z)]
    _lib.call('b200rl_cem_sample', _lib.ptr(ins[0]), C + 1, B, N, C, A, _lib.ptr(ins[1]), 0,
              _lib.ptr(ins[2]), 0, 1e-4, _lib.ptr(tlo), _lib.ptr(thi), _lib.ptr(ins[3]), 0,
              _lib.ptr(ctr), _lib.ptr(x), W, _lib.stream())
    xs = x.cpu().numpy()
    want = np.clip(m0 + np.sqrt(np.maximum(v0.astype(np.float64), 1e-4)) * z, lo, hi)
    np.testing.assert_allclose(xs[:, C:C + A], want.reshape(B * N, A), rtol=1e-6, atol=1e-6)
    np.testing.assert_array_equal(xs[:, :C], np.repeat(src[:, :C], N, axis=0))
    assert (xs[:, C + A:] == 7).all() and ctr.cpu().tolist() == [0, 0]
    # cem_refit on scores with deliberate ties, then the next draws
    acts = rng.uniform(lo, hi, (B, N, A)).astype(f32)
    x[:, C:C + A] = _d(cuda, acts.reshape(B * N, A))
    scores = rng.randint(0, 5, (B, N)).astype(f32) * 0.25
    z2 = rng.randn(B, N, A).astype(f32)
    tsc, tz2 = _d(cuda, scores.ravel()), _d(cuda, z2)
    mean, var = torch.empty(B, A, device=cuda), torch.empty(B, A, device=cuda)
    _lib.call('b200rl_cem_refit', _lib.ptr(tsc), None, _lib.ptr(x), W, C, B, N, M, A, 1e-4,
              _lib.ptr(tlo), _lib.ptr(thi), 0, _lib.ptr(tz2), 0, _lib.ptr(ctr), _lib.ptr(mean),
              _lib.ptr(var), None, None, _lib.stream())
    idx, rm, rv = _ref_refit(acts, scores, M)
    np.testing.assert_allclose(mean.cpu().numpy(), rm, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(var.cpu().numpy(), rv, rtol=1e-4, atol=1e-6)
    xs2 = x.cpu().numpy()
    want = np.clip(rm[:, None] + np.sqrt(np.maximum(rv, 1e-4))[:, None] * z2, lo, hi)
    np.testing.assert_allclose(xs2[:, C:C + A], want.reshape(B * N, A), rtol=1e-5, atol=2e-6)
    np.testing.assert_array_equal(xs2[:, :C], xs[:, :C])
    assert (xs2[:, C + A:] == 7).all()
    # last iteration: best action and score instead of draws
    x[:, C:C + A] = _d(cuda, acts.reshape(B * N, A))
    best, bs = torch.empty(B, A, device=cuda), torch.empty(B, device=cuda)
    _lib.call('b200rl_cem_refit', _lib.ptr(tsc), None, _lib.ptr(x), W, C, B, N, M, A, 1e-4,
              _lib.ptr(tlo), _lib.ptr(thi), 1, None, 0, _lib.ptr(ctr), _lib.ptr(mean),
              _lib.ptr(var), _lib.ptr(best), _lib.ptr(bs), _lib.stream())
    rows = np.arange(B)
    np.testing.assert_array_equal(best.cpu().numpy(), acts[rows, idx[:, 0]])
    np.testing.assert_array_equal(bs.cpu().numpy(), scores[rows, idx[:, 0]])
    np.testing.assert_array_equal(x[:, C:C + A].cpu().numpy(), acts.reshape(B * N, A))
    assert ctr.cpu().tolist() == [0, 0]
  # the sampler's refit at given indices
  s = samplers.GaussianActionsSampler(_specs(2, A)[1])
  acts = rng.randn(B, N, A).astype(f32)
  ind = np.stack([rng.permutation(N)[:M] for _ in range(B)]).astype(np.int32)
  mean, var = s.refit_distribution_to(torch.as_tensor(ind, device=cuda), _d(cuda, acts))
  el = np.take_along_axis(acts.astype(np.float64), ind[:, :, None].astype(np.int64), axis=1)
  np.testing.assert_allclose(mean.cpu().numpy(), el.mean(1), rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(var.cpu().numpy(), el.var(1), rtol=1e-4, atol=1e-6)


def test_device_draws_match_the_sampling_moments(cuda):
  s = samplers.GaussianActionsSampler(_specs(2, 3, -100.0, 100.0)[1])
  mean = _d(cuda, [[0.5, -1.0, 2.0]])
  var = _d(cuda, [[0.04, 1.0, 9.0]])
  n = 200000
  a = s.sample_batch_and_clip(n, mean, var).cpu().double().numpy()[0]
  a2 = s.sample_batch_and_clip(n, mean, var).cpu().double().numpy()[0]
  assert s._rng.cpu().tolist() == [2, 0] and not np.array_equal(a, a2)
  m, v = mean.cpu().double().numpy()[0], var.cpu().double().numpy()[0]
  se_m, se_v = np.sqrt(v / n), v * np.sqrt(2.0 / n)
  assert (np.abs(a.mean(0) - m) <= 5 * se_m).all(), (a.mean(0), m)
  assert (np.abs(a.var(0) - v) <= 5 * se_v).all(), (a.var(0), v)
  record_parity('qtopt_draw_moments', mean_z=float(np.max(np.abs(a.mean(0) - m) / se_m)),
                var_z=float(np.max(np.abs(a.var(0) - v) / se_v)))


@pytest.mark.parametrize('B', [1, 300, 5000])
def test_td_loss_kernel_matches_float64(cuda, B):
  rng = np.random.RandomState(B)
  for kind in (_lib.LOSS_HUBER, _lib.LOSS_SQUARED):
    for twin in (False, True):
      for weighted in (False, True):
        q, t1, t2, r = [(rng.randn(B) * 2).astype(f32) for _ in range(4)]
        dsc = (rng.rand(B) > .2).astype(f32)
        st = np.stack([rng.randint(0, 3, B), np.zeros(B)], 1).astype(np.int32)   # stride 2
        w = rng.rand(B).astype(f32) if weighted else None
        ins = [_d(cuda, a) for a in (q, t1, t2, r, dsc)]
        tst, tw = torch.as_tensor(st, device=cuda), None if w is None else _d(cuda, w)
        loss, tl, te, dq = (torch.empty(1, device=cuda), torch.empty(B, device=cuda),
                            torch.empty(B, device=cuda), torch.empty(B, device=cuda))
        _lib.call('b200rl_qtopt_td_loss', _lib.ptr(ins[0]), _lib.ptr(ins[1]),
                  _lib.ptr(ins[2]) if twin else None, _lib.ptr(ins[3]), _lib.ptr(ins[4]),
                  _lib.ptr(tst), 2, _lib.ptr(tw), B, 0.97, 1.3, kind, _lib.ptr(loss),
                  _lib.ptr(tl), _lib.ptr(te), _lib.ptr(dq), None, _lib.stream())
        Q = R.t64(q).requires_grad_()
        nq = torch.minimum(R.t64(t1), R.t64(t2)) if twin else R.t64(t1)
        y = 1.3 * R.t64(r) + 0.97 * R.t64(dsc) * nq
        m = R.t64(st[:, 0] != 2)
        el = R.huber if kind == _lib.LOSS_HUBER else (lambda e: e * e)
        W = torch.ones(B, dtype=F64) if w is None else R.t64(w)
        per = m * el(y - Q)
        ref = (per * W).sum() / B
        np.testing.assert_allclose(loss.item(), ref.item(), rtol=1e-5)
        torch.testing.assert_close(tl.cpu().double(), per.detach(), rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(te.cpu().double(), m * (y - R.t64(q)), rtol=1e-5, atol=1e-5)
        R.assert_grad_close('qtopt dq', dq, torch.autograd.grad(ref, Q)[0], 1e-5, 1e-5)
  with pytest.raises(ValueError):
    _lib.call('b200rl_qtopt_td_loss', _lib.ptr(ins[0]), _lib.ptr(ins[1]), None, _lib.ptr(ins[3]),
              _lib.ptr(ins[4]), _lib.ptr(tst), 2, None, B, 0.97, 1.3, 7, _lib.ptr(loss),
              _lib.ptr(tl), _lib.ptr(te), _lib.ptr(dq), None, _lib.stream())


def test_epsilon_uniform_fraction_and_uniformity(cuda):
  N, A, eps = 100000, 3, 0.3
  lo, hi = np.array([-1, -2, 0], f32), np.array([1, 3, 0.5], f32)
  tlo, thi = _d(cuda, lo), _d(cuda, hi)
  act = torch.full((N, A), 100.0, device=cuda)
  ctr = torch.zeros(2, dtype=torch.int64, device=cuda)
  _lib.call('b200rl_epsilon_uniform', _lib.ptr(act), A, N, A, eps, _lib.ptr(tlo), _lib.ptr(thi), 3,
            _lib.ptr(ctr), _lib.stream())
  a = act.cpu().numpy()
  rep = (a != 100.0).all(1)
  assert ((a == 100.0).all(1) | rep).all()             # whole rows are replaced or kept
  frac = rep.mean()
  assert abs(frac - eps) <= 5 * np.sqrt(eps * (1 - eps) / N), frac
  u = (a[rep] - lo) / (hi - lo)
  assert (u >= 0).all() and (u < 1).all()
  for k in range(A):                                   # uniform: 10 equal bins, chi-square
    cnt, _ = np.histogram(u[:, k], bins=10, range=(0, 1))
    chi2 = float(((cnt - cnt.mean()) ** 2 / cnt.mean()).sum())
    assert chi2 < 30.0, (k, chi2)                      # 9 dof: p < 1e-3
  assert ctr.cpu().tolist() == [1, 0]
  record_parity('qtopt_epsilon_uniform', frac=float(frac))


# ---- 2. agent: golden, policies -------------------------------------------------------------------
def test_reference_golden_loss_through_the_agent(cuda):
  obs_spec, act_spec = _specs(2, 1, 0.0, 1.0)
  nets = []
  for bias in (2.0, 1.0):
    n = critic_network.CriticNetwork((obs_spec, act_spec), joint_fc_layer_params=(), device=cuda)
    n.create_variables()
    n.layers[-1].kernel.copy_(torch.tensor([[2.0], [1.0], [0.0]]))
    n.layers[-1].bias.fill_(bias)
    nets.append(n)
  agent = qtopt_agent.QtOptAgent(ts.time_step_spec(obs_spec), act_spec, nets[0], None,
                                 samplers.GaussianActionsSampler(act_spec), init_mean_cem=[0.5],
                                 init_var_cem=[0.08], num_samples_cem=32)
  agent.initialize()
  agent._target_q_network_delayed.flat_params.copy_(nets[1].flat_params)
  e = dict(observation=np.array([[[1, 2], [5, 6]], [[3, 4], [7, 8]]], f32),
           action=np.zeros((2, 2, 1), f32), reward=np.array([[10, 0], [20, 0]], f32),
           discount=np.array([[.9, 1], [.9, 1]], f32),
           step_type=np.array([[0, 1], [0, 1]], np.int32))
  info = agent._loss(_traj(cuda, e))
  np.testing.assert_allclose(info.loss.item(), 23.5, rtol=1e-6)
  np.testing.assert_allclose(info.extra.td_loss.mean().item(), 23.5, rtol=1e-6)
  with pytest.raises(ValueError, match='Optimizer is undefined'):
    agent.train(_traj(cuda, e))


def test_policies_stay_in_bounds(cuda):
  # agents/qtopt/qtopt_agent_test.py testPolicy, and the collect policy's uniform rows
  D, A, N = 2, 3, 512
  agent = _make(cuda, D=D, A=A, obs_fc=None, joint_fc=(32,), bounds=(-2.0, 3.0),
                epsilon_greedy=0.25)
  assert isinstance(agent.policy, qtopt_cem_policy.CEMPolicy)
  assert isinstance(agent.collect_policy, epsilon_greedy_policy.EpsilonGreedyPolicy)
  assert agent.policy_q_network is agent._target_q_network and agent.enable_td3
  step = ts.restart(torch.randn(N, D, device=cuda), batch_size=N)
  a1 = agent.policy.action(step).action
  assert tuple(a1.shape) == (N, A) and float(a1.min()) >= -2 and float(a1.max()) <= 3
  assert agent.policy._cem_rng.cpu().tolist() == [3, 0]
  # the action is the best sample of the last iteration: its score is the target's Q there
  best, score = agent.policy.search(step.observation)
  q, _ = agent._target_q_network((step.observation, best))
  torch.testing.assert_close(q, score, rtol=1e-5, atol=1e-5)
  c = agent.collect_policy.action(step).action
  assert float(c.min()) >= -2 and float(c.max()) <= 3
  rp = random_tf_policy.RandomTFPolicy(ts.time_step_spec(_specs(D, A)[0]), _specs(D, A, -2., 3.)[1])
  r = rp.action(step).action
  assert tuple(r.shape) == (N, A) and float(r.min()) >= -2 and float(r.max()) < 3
  assert float(r.std()) > 1.0


# ---- 3. QtOptAgent.train against the oracle ------------------------------------------------------
_CONFIGS = [
    # (enable_td3, n_step_update, loss, obs_fc, weighted, gradient clipping, bounds)
    (True, 1, oq.HUBER, (400,), True, None, (-1.0, 1.0)),
    (False, 1, oq.SQUARED, (400,), False, 0.5, (-2.0, 3.0)),
    (True, 2, oq.HUBER, None, False, None, (-2.0, 3.0)),
    (True, 1, oq.SQUARED, None, True, None, (-1.0, 1.0)),
    (False, 2, oq.HUBER, None, True, 0.5, (-1.0, 1.0)),
]


def _oracle(agent, bounds, **kw):
  lo, hi = bounds
  A = agent._sampler.num_actions
  return oq.QtOptOracle(_mirror(agent._q_network), np.full(A, lo, f32), np.full(A, hi, f32),
                        np.full(A, (lo + hi) / 2), np.full(A, ((hi - lo) / 4) ** 2), **kw)


@pytest.mark.parametrize('cfg', _CONFIGS,
                         ids=lambda c: f'td3{c[0]}-n{c[1]}-{c[2]}-{c[3]}-w{c[4]}-c{c[5]}-{c[6][0]}')
def test_agent_train_matches_oracle(cuda, cfg):
  td3, n, kind, obs_fc, weighted, clip, bounds = cfg
  D, A, B, N = 17, 6, 64, 32
  fn = common.element_wise_huber_loss if kind == oq.HUBER else common.element_wise_squared_loss
  kw = dict(enable_td3=td3, n_step_update=n, td_errors_loss_fn=fn, gamma=0.99,
            reward_scale_factor=0.5, gradient_clipping=clip, target_update_tau=0.05)
  if td3:
    kw['delayed_target_update_period'] = 2
  agent = _make(cuda, D, A, obs_fc=obs_fc, joint_fc=(300,) if obs_fc else (256, 256),
                bounds=bounds, **kw)
  orc = _oracle(agent, bounds, opt=ooptim.AdamTF(1e-3, eps=1e-7), gamma=0.99, reward_scale=0.5,
                tau=0.05, enable_td3=td3, delayed_target_update_period=2, loss=kind,
                gradient_clipping=clip)
  rng = np.random.RandomState(7)
  name = 'qtopt_agent_train_' + '_'.join(str(c) for c in cfg)
  for step in range(6):
    e = _batch(rng, B, D, A, n + 1, *bounds)
    w = rng.rand(B).astype(f32) if weighted else None
    z = rng.randn(3, B, N, A).astype(f32)
    want = orc.train(e, z, w)
    got = agent.train(_traj(cuda, e), weights=None if w is None else _d(cuda, w),
                      noise=(_d(cuda, z),))
    g, wv = got.loss.item(), float(want['loss'])
    record_parity(name, loss_rel=abs(g - wv) / max(abs(wv), 1e-30))
    np.testing.assert_allclose(g, wv, rtol=1e-5, err_msg=f'step {step}')
    np.testing.assert_allclose(got.extra.td_loss.cpu().numpy(), want['td_loss'], rtol=1e-4,
                               atol=1e-5)
    np.testing.assert_allclose(got.extra.td_error.cpu().numpy(), want['td_error'], rtol=1e-4,
                               atol=1e-5)
  assert int(agent.train_step_counter.item()) == 6
  nets = [(agent._q_network, orc.q), (agent._target_q_network, orc.target)]
  if td3:
    nets += [(agent._target_q_network_delayed, orc.delayed),
             (agent._target_q_network_delayed_2, orc.delayed_2)]
  for net, ref in nets:                                # as test_ddpg_gpu: Adam's last-bit outliers
    got = np.concatenate([v.cpu().numpy().ravel() for v in net.variables])
    want = np.concatenate([w.ravel() for w in ref.params()])
    diff = np.abs(got - want)
    out = diff > 1e-5 + 1e-3 * np.abs(want)
    record_parity(name, **{net.name + '_outlier_frac': out.mean(), net.name + '_max_abs': diff.max()})
    assert out.mean() <= 1e-3 and diff.max() <= 6 * 1e-3, (net.name, out.mean(), diff.max())
  agent.check_numerics()


def test_delayed_chain_lags_the_target(cuda):
  agent = _make(cuda, D=6, A=2, obs_fc=None, joint_fc=(16,), target_update_tau=1.0,
                delayed_target_update_period=5)
  rng = np.random.RandomState(3)
  tgt, d1, d2 = (agent._target_q_network.flat_params, agent._target_q_network_delayed.flat_params,
                 agent._target_q_network_delayed_2.flat_params)
  snaps = {}
  for step in range(1, 11):
    before, tgt_before = d1.clone(), tgt.clone()
    agent.train(_traj(cuda, _batch(rng, 8, 6, 2)))
    assert torch.equal(tgt, agent._q_network.flat_params)          # tau 1, period 1
    if step % 5 == 0:
      assert torch.equal(d2, before), step                         # delayed_2 <- the OLD delayed
      snaps[step] = tgt_before
      assert torch.equal(d1, tgt_before), step                     # delayed <- the OLD target
    else:
      assert torch.equal(d1, before), step
  assert torch.equal(d2, snaps[5]) and not torch.equal(d2, d1)


# ---- 4. gradients before the optimiser ------------------------------------------------------------
def _q64(net, obs, act):
  dense = [l for l in net.layers if isinstance(l, L.Dense)]
  ps = [(R.t64(l.kernel).requires_grad_(), R.t64(l.bias).requires_grad_(), l.activation)
        for l in dense]
  k = net._n_obs_layers
  h = R.mlp(ps[:k], obs) if k else obs
  return R.mlp(ps[k:], torch.cat([h, act], 1))[:, 0], ps


@pytest.mark.parametrize('obs_fc', [(400,), None])
def test_gradients_before_the_optimizer_match_float64(cuda, obs_fc):
  D, A, B, N = 17, 6, 256, 32
  agent = _make(cuda, D, A, obs_fc=obs_fc, joint_fc=(300,), lr=0.0, gamma=0.9,
                bounds=(-2.0, 3.0))
  rng = np.random.RandomState(9)
  for net in (agent._target_q_network_delayed, agent._target_q_network_delayed_2):
    net.flat_params.add_(torch.randn_like(net.flat_params) * 0.01)
  e, w = _batch(rng, B, D, A, 2, -2.0, 3.0), rng.rand(B).astype(f32)
  z = _d(cuda, rng.randn(3, B, N, A))
  obs2 = _d(cuda, e['observation'][:, 1])
  a2, _ = agent.policy.search(obs2, z=z)               # the search the train step repeats
  a2 = R.t64(a2)
  agent.train(_traj(cuda, e), weights=_d(cuda, w), noise=(z,))
  O2 = R.t64(e['observation'][:, 1])
  nq = torch.minimum(_q64(agent._target_q_network_delayed, O2, a2)[0],
                     _q64(agent._target_q_network_delayed_2, O2, a2)[0]).detach()
  y = R.t64(e['reward'][:, 0]) + 0.9 * R.t64(e['discount'][:, 0]) * nq
  q, ps = _q64(agent._q_network, R.t64(e['observation'][:, 0]), R.t64(e['action'][:, 0]))
  m = R.t64(e['step_type'][:, 0] != 2)
  ref = torch.autograd.grad((m * R.huber(y - q) * R.t64(w)).sum() / B,
                            [t for p in ps for t in p[:2]])
  for i, (g, rf) in enumerate(zip(agent._q_network._grad_views, ref)):
    e_ = R.grad_errors(g, rf)
    record_parity(f'qtopt_grads_{obs_fc}', **{f'{i}_rel_l2': e_[0], f'{i}_max': e_[1]})
    R.assert_grad_close(f'qtopt q/{i}', g, rf, 1e-4, 1e-4)


# ---- 5. graph replay ------------------------------------------------------------------------------
_SMALL = dict(D=6, A=2, obs_fc=(16,), joint_fc=(16,), target_update_tau=0.05,
              target_update_period=2, delayed_target_update_period=3, epsilon_greedy=0.3, N=9, M=3)


def test_graph_replay_matches_eager_bit_for_bit(cuda):
  eager, graphed = _make(cuda, **_SMALL), _make(cuda, **_SMALL)
  train_fn = common.function(graphed.train)
  rng = np.random.RandomState(11)
  for step in range(8):                                # crosses every target-update period
    traj = _traj(cuda, _batch(rng, 8, 6, 2))
    l1 = eager.train(traj)
    l2 = train_fn(traj)
    assert l1.loss.item() == l2.loss.item(), step
    assert torch.equal(l1.extra.td_error, l2.extra.td_error), step
  assert int(graphed.train_step_counter.item()) == 8 and graphed._train_step_host == 8
  for n in ('_q_network', '_target_q_network', '_target_q_network_delayed',
            '_target_q_network_delayed_2'):
    assert torch.equal(getattr(eager, n).flat_params, getattr(graphed, n).flat_params), n
  assert torch.equal(eager.policy._cem_rng, graphed.policy._cem_rng)
  assert eager.policy._cem_rng.cpu().tolist() == [8 * 3, 0]   # 3 drawing launches a search


def test_captured_collect_step_matches_eager_calls(cuda):
  eager, graphed = _make(cuda, seed=4, **_SMALL), _make(cuda, seed=4, **_SMALL)
  step = ts.restart(torch.randn(64, 6, device=cuda), batch_size=64)
  act_fn = common.function(lambda t: graphed.collect_policy.action(t).action)
  seen = set()
  for call in range(6):                                # 2 eager warm-up calls, capture, replays
    a1 = eager.collect_policy.action(step).action
    a2 = act_fn(step)
    assert torch.equal(a1, a2), call
    seen.add(a2.cpu().numpy().tobytes())
  assert len(seen) == 6                                # fresh draws on every replay
  assert graphed.collect_policy._uniform_rng.cpu().tolist() == [6, 0]
  assert graphed.policy._cem_rng.cpu().tolist() == [6 * 3, 0]


# ---- 6. Learner checkpoints -----------------------------------------------------------------------
def test_learner_checkpoint_restore_reproduces_losses_and_actions(cuda):
  # 8 rows: every launch is one CTA, so the step is bit-reproducible (DESIGN.md §4)
  rng = np.random.RandomState(12)
  batches = [_batch(rng, 8, 6, 2) for _ in range(9)]
  step_obs = ts.restart(torch.randn(3, 6, device=cuda), batch_size=3)
  root = tempfile.mkdtemp()

  def make(perturb):
    from agents_b200.train.utils import train_utils
    step = train_utils.create_train_step(cuda)
    agent = _make(cuda, train_step_counter=step, **_SMALL)
    if perturb:                                        # other weights and draws, then restored
      for n in (agent._q_network, agent._target_q_network, agent._target_q_network_delayed,
                agent._target_q_network_delayed_2):
        n.flat_params.mul_(0.5)
      agent.collect_policy.action(step_obs)
    it = iter([_traj(cuda, e) for e in batches])
    return agent, step, learner_lib.Learner(root, step, agent, experience_dataset_fn=lambda: it,
                                            checkpoint_interval=4)

  agent, step, lrn = make(False)
  for _ in range(3):
    agent.collect_policy.action(step_obs)
  lrn.run(iterations=4)
  want_act = [agent.collect_policy.action(step_obs).action.clone() for _ in range(3)]
  want = [agent.train(_traj(cuda, e)).loss.item() for e in batches[4:]]
  agent2, step2, _ = make(True)
  assert int(step2.item()) == 4
  got_act = [agent2.collect_policy.action(step_obs).action.clone() for _ in range(3)]
  got = [agent2.train(_traj(cuda, e)).loss.item() for e in batches[4:]]
  for g, w in zip(got_act, want_act):
    assert torch.equal(g, w)
  assert got == want


def test_unsupported_arguments_raise(cuda):
  obs_spec, act_spec = _specs(4, 2)
  critic = critic_network.CriticNetwork((obs_spec, act_spec), joint_fc_layer_params=(8,),
                                        device=cuda)
  s = samplers.GaussianActionsSampler(act_spec)
  tss = ts.time_step_spec(obs_spec)
  base = dict(init_mean_cem=[0.0, 0.0], init_var_cem=[0.3, 0.3])
  for kw, err in ((dict(in_graph_bellman_update=False), NotImplementedError),
                  (dict(emit_log_probability=True), NotImplementedError),
                  (dict(auxiliary_loss_fns=[lambda **k: 0]), NotImplementedError),
                  (dict(td_errors_loss_fn=lambda y, q: (y - q).abs()), ValueError),
                  (dict(init_mean_cem=None), ValueError)):
    with pytest.raises(err):
      qtopt_agent.QtOptAgent(tss, act_spec, critic, None, s, **{**base, **kw})
  with pytest.raises(NotImplementedError):
    samplers.GaussianActionsSampler(act_spec, sample_clippers=[lambda a, s: a])
  with pytest.raises(ValueError):
    samplers.GaussianActionsSampler(tensor_spec.BoundedTensorSpec((), torch.int32, 0, 3))
  with pytest.raises(NotImplementedError):
    qtopt_cem_policy.CEMPolicy(tss, act_spec, critic, s, [0.0, 0.0], [0.3, 0.3],
                               actor_policy=object())


# ---- 7. learning -----------------------------------------------------------------------------------
def learning_task(seed, D=8, A=3, n=4096):
  """Offline, discount 0: reward -||a - tanh(s W)||^2 over uniform random actions."""
  rng = np.random.RandomState(seed)
  Wm = (rng.randn(D, A) * 0.5).astype(f32)
  obs = rng.randn(n, 2, D).astype(f32)
  act = rng.uniform(-1, 1, (n, 2, A)).astype(f32)
  best = np.tanh(obs[:, 0] @ Wm).astype(f32)
  rew = -np.sum((act[:, 0] - best) ** 2, axis=1).astype(f32)
  data = dict(observation=obs, action=act, reward=np.stack([rew, rew], 1),
              discount=np.zeros((n, 2), f32), step_type=np.ones((n, 2), np.int32))
  eval_obs = rng.randn(1024, D).astype(f32)
  return data, eval_obs, np.tanh(eval_obs @ Wm).astype(f32), rng


LEARN_STEPS, LEARN_B = 1500, 64
LEARN_NET = dict(D=8, A=3, obs_fc=None, joint_fc=(64, 64), target_update_tau=0.05)
# Greedy error mean ||CEM(s) - tanh(s W)||^2 of the numpy oracle (oracle/qtopt.py) on this task with
# the same network, optimiser, batches and N = 32, M = 4, 3 iterations, seeds 0-7 (draws z from
# np.random.RandomState(100 + seed)):
#   initial       3.442 3.151 3.305 3.592 2.907 2.827 3.625 3.281
#   after 1500    0.1579 0.1626 0.1604 0.1338 0.1062 0.1624 0.1636 0.1306
# The threshold is twice the worst of those and far below every initial error.
LEARN_THRESHOLD = 0.33


def test_offline_learning_reduces_greedy_error(cuda):
  data, eval_obs, eval_best, rng = learning_task(0)
  agent = _make(cuda, **LEARN_NET)
  obs_t = _d(cuda, eval_obs)

  def err():
    a = agent.policy.action(ts.restart(obs_t, batch_size=obs_t.shape[0])).action
    return float(((a.cpu().numpy() - eval_best) ** 2).sum(1).mean())

  e0 = err()
  full = {k: torch.as_tensor(v, device=cuda) for k, v in data.items()}
  for _ in range(LEARN_STEPS):
    idx = torch.as_tensor(rng.randint(0, data['reward'].shape[0], LEARN_B), device=cuda)
    traj = trajectory.Trajectory(full['step_type'][idx], full['observation'][idx],
                                 full['action'][idx], (), full['step_type'][idx],
                                 full['reward'][idx], full['discount'][idx])
    agent.train(traj)
  e1 = err()
  record_parity('qtopt_learning', initial=e0, final=e1)
  assert e1 < LEARN_THRESHOLD < e0, (e0, e1)
