"""CQL-SAC on the GPU: the reference's goldens through csrc/cql.cu, the CQL loss / BC kernels
against float64 autograd, the candidate draws, CqlSacAgent.train against oracle/cql_sac.py
(every draw supplied), the agent's pre-optimizer gradients, graph == eager across the BC
boundary and Lagrange updates, and checkpoint -> restore."""
import math

import numpy as np
import pytest
import torch

import grad_refs as R
from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.agents.cql import cql_sac_agent
from agents_b200.networks import critic_network
from agents_b200.networks import layers as L
from agents_b200.networks import tanh_normal_projection_network as tnp
from agents_b200.specs import tensor_spec
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory
from agents_b200.utils import common
from conftest import record_parity
from oracle import cql_sac as ocql
from oracle import nn as onn
from oracle import optim as ooptim

pytestmark = pytest.mark.gpu
f32 = np.float32
# (a - shift) / half is exactly +-1 at these bounds, so dataset actions at the bounds stay finite
AMIN = np.array([-2.0, 0.0, -0.5, 0.25, -7.0, -1.0], f32)
AMAX = np.array([1.0, 10.0, 0.5, 0.75, -3.0, 1.0], f32)


def _d(cuda, a, dtype=torch.float32):
  return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device=cuda)


def _cql_loss_call(cuda, q1, q2, logp, B, N, ulogp, temp=1.0, alpha=None, log_alpha=None,
                   clip=(-math.inf, math.inf), tau=10.0, bc_debug=0, closs=0.0, dq_init=None):
  """Runs b200rl_cql_loss; returns (out[4], dq1, dq2, dlog_cql_alpha) as numpy."""
  R_ = B + 2 * B * N
  tq1, tq2, tlp = _d(cuda, q1), _d(cuda, q2), _d(cuda, logp)
  a = None if alpha is None else _d(cuda, np.float32(alpha))
  la = None if log_alpha is None else _d(cuda, np.array([log_alpha, 0, 0, 0], f32))
  dla = torch.full((4,), float('nan'), device=cuda)
  cl = _d(cuda, np.array([closs], f32))
  dq1 = torch.full((R_ + 3,), float('nan'), device=cuda)        # canary tail
  dq2 = torch.full((R_ + 3,), float('nan'), device=cuda)
  if dq_init is not None:
    dq1[:B] = _d(cuda, dq_init[0])
    dq2[:B] = _d(cuda, dq_init[1])
  out = torch.full((4,), float('nan'), device=cuda)
  ws = torch.zeros(256, device=cuda)
  nan = torch.zeros(1, dtype=torch.int32, device=cuda)
  _lib.call('b200rl_cql_loss', _lib.ptr(tq1), _lib.ptr(tq2), _lib.ptr(tlp), B, N, float(ulogp),
            float(temp), _lib.ptr(a), _lib.ptr(la), clip[0], clip[1], float(tau), int(bc_debug),
            _lib.ptr(cl), _lib.ptr(dq1), _lib.ptr(dq2), _lib.ptr(out), _lib.ptr(dla),
            _lib.ptr(nan), _lib.ptr(ws), 4 * 256, _lib.stream())
  assert torch.isnan(dq1[R_:]).all() and torch.isnan(dq2[R_:]).all()
  assert nan.item() == 0
  return (out.cpu().numpy(), dq1[:R_].cpu().numpy(), dq2[:R_].cpu().numpy(), dla.cpu().numpy())


def _mock_rows(a_unif):
  """testCqlLoss (cql_sac_agent_test.py:237-267) as joint-row critic outputs: q = obs[:, 1] + a,
  DummyActorPolicy candidates a = 1 with log_prob 10, the uniform actions a_unif [B, N]."""
  obs1 = np.tile(np.array([2, 4], f32), a_unif.shape[0] // 2)
  q = np.concatenate([obs1 + np.tile(np.array([5, 6], f32), a_unif.shape[0] // 2),
                      np.repeat(obs1 + 1, a_unif.shape[1]), (obs1[:, None] + a_unif).reshape(-1)])
  return q.astype(f32), np.full(a_unif.size, 10, f32)


def test_reference_goldens_through_kernels(cuda):
  # critic loss 2*MSE([16.3, 28.1], [7, 10]) without the entropy term: SAC's kernel, zero logp
  la = torch.zeros(4, device=cuda)
  q, tq = _d(cuda, [7., 10.]), _d(cuda, [7., 9.])
  zero, rew, disc = _d(cuda, [0., 0.]), _d(cuda, [10., 20.]), _d(cuda, [.9, .9])
  loss, dq1, dq2, y = (torch.empty(n, device=cuda) for n in (1, 2, 2, 2))
  _lib.call('b200rl_sac_critic_loss', _lib.ptr(q), _lib.ptr(q), _lib.ptr(tq), _lib.ptr(tq),
            _lib.ptr(zero), _lib.ptr(rew), _lib.ptr(disc), None, _lib.ptr(la), 2, 1.0, 1.0, 1.0, 2.0,
            _lib.ptr(loss), _lib.ptr(dq1), _lib.ptr(dq2), _lib.ptr(y), None, _lib.stream())
  np.testing.assert_allclose(y.cpu().numpy(), [16.3, 28.1], rtol=1e-6)
  np.testing.assert_allclose(loss.item(), 2 * np.mean((np.array([16.3, 28.1]) - [7, 10]) ** 2), rtol=1e-6)
  # CQL loss at all-zero uniform actions: -2.5042, and exactly x10 at cql_alpha 10
  qj, logp = _mock_rows(np.zeros((2, 10), f32))
  ulogp = ocql.uniform_log_prob(-1.0, 1.0, 1)
  out1 = _cql_loss_call(cuda, qj, qj, logp, 2, 10, ulogp, alpha=1.0)[0]
  out10 = _cql_loss_call(cuda, qj, qj, logp, 2, 10, ulogp, alpha=10.0)[0]
  np.testing.assert_allclose(out1[0], -2.5042, atol=1e-4)
  np.testing.assert_allclose(out10[2], 10 * out1[2], rtol=1e-6)        # alpha * cql_loss
  # Lagrange: cql_alpha 5 -> 5 e^-0.5 after one Adam step at lr 0.5 (:531-654)
  out, _, _, dla = _cql_loss_call(cuda, qj, qj, logp, 2, 10, ulogp, log_alpha=math.log(5.0),
                                  clip=(-1.0, 10.0))
  np.testing.assert_allclose(out[1], 5.0, rtol=1e-6)
  assert out[3] > 0 and dla[0] == out[3]
  p = _d(cuda, np.array([math.log(5.0), 0, 0, 0], f32))
  g = _d(cuda, np.array([dla[0], 0, 0, 0], f32))
  optimizers.Adam(0.5).apply_flat(p, g)
  np.testing.assert_allclose(math.exp(p[0].item()), 3.032653, rtol=1e-5)


@pytest.mark.parametrize('N', [1, 10, 40])
@pytest.mark.parametrize('mode', ['add', 'bc_debug', 'lagrange_in', 'lagrange_clipped'])
def test_cql_loss_kernel_vs_autograd(cuda, N, mode):
  rng = np.random.RandomState(N)
  B, temp, tau = 300, 0.8, -1.0
  R_ = B + 2 * B * N
  q1, q2 = (rng.randn(R_) * 4).astype(f32), (rng.randn(R_) * 4).astype(f32)
  logp = (rng.randn(B * N) * 3).astype(f32)
  ulogp = ocql.uniform_log_prob(AMIN, AMAX, 6)
  td = [(rng.randn(B) * .1).astype(f32) for _ in range(2)]
  kw = dict(alpha=2.5)
  if mode.startswith('lagrange'):
    kw = dict(log_alpha=1.2, clip=(-1.0, 2.0) if mode == 'lagrange_in' else (-1.0, 0.5))
  out, dq1, dq2, dla = _cql_loss_call(cuda, q1, q2, logp, B, N, ulogp, temp=temp, tau=tau,
                                      bc_debug=mode == 'bc_debug', closs=0.75, dq_init=td, **kw)
  Q1, Q2 = torch.tensor(q1.astype(np.float64), requires_grad=True), torch.tensor(
      q2.astype(np.float64), requires_grad=True)
  lp = R.t64(logp).reshape(B, N)
  terms = []
  for Q in (Q1, Q2):
    z = torch.cat([Q[B:B + B * N].reshape(B, N) * temp - lp,
                   Q[B + B * N:].reshape(B, N) * temp - float(ulogp)], 1)
    terms.append(torch.logsumexp(z, 1) / temp - Q[:B])
  cql = (terms[0] + terms[1]).mean() / 2
  alpha = 2.5 if mode in ('add', 'bc_debug') else math.exp(min(1.2, kw['clip'][1]))
  g1, g2 = torch.autograd.grad(alpha * cql, (Q1, Q2))
  if mode != 'bc_debug':
    g1[:B] += R.t64(td[0])
    g2[:B] += R.t64(td[1])
  e = max(abs(out[0] - cql.item()) / abs(cql.item()), *R.grad_errors(dq1, g1), *R.grad_errors(dq2, g2))
  record_parity('cql_loss_kernel', max_rel=e)
  np.testing.assert_allclose(out[0], cql.item(), rtol=1e-5)
  np.testing.assert_allclose(out[1], alpha, rtol=1e-6)
  np.testing.assert_allclose(out[2], alpha * cql.item() + (0 if mode == "bc_debug" else 0.75), rtol=1e-5)
  R.assert_grad_close('cql/dq1', dq1, g1, 1e-5, 1e-5)
  R.assert_grad_close('cql/dq2', dq2, g2, 1e-5, 1e-5)
  if mode.startswith('lagrange'):
    want = -alpha * (cql.item() - tau)
    np.testing.assert_allclose(out[3], want, rtol=1e-5)
    np.testing.assert_allclose(dla[0], want if mode == "lagrange_in" else 0.0, rtol=1e-5)
  else:
    assert out[3] == 0.0


@pytest.mark.parametrize('A', [1, 6])
def test_bc_kernels_vs_autograd(cuda, A):
  rng = np.random.RandomState(10 + A)
  B, lw, gb = 257, 0.7, 300.0
  amin, amax = AMIN[:A], AMAX[:A]
  head = (rng.randn(B, 2 * A) * .6).astype(f32)
  act = (amin + (amax - amin) * rng.rand(B, 2, A)).astype(f32)
  act[:5, 0], act[5:10, 0] = amin, amax                  # dataset actions at the bounds
  logp = rng.randn(B).astype(f32)
  w = (rng.rand(B) * 2).astype(f32)
  w[::7] = 0
  la = _d(cuda, np.array([0.3, 0, 0, 0], f32))
  th, ta, tmin, tmax, tlp, tw = (_d(cuda, x) for x in (head, act, amin, amax, logp, w))
  for step, bc in ((0, True), (3, False)):
    counter = _d(cuda, np.int64(step), torch.int64)
    loss = _d(cuda, np.array([123.0], f32))
    dq1, dq2 = torch.ones(B, device=cuda), torch.ones(B, device=cuda)
    dhead0 = rng.randn(B, 2 * A).astype(f32)
    dhead = _d(cuda, dhead0)
    nan = torch.zeros(1, dtype=torch.int32, device=cuda)
    ta0 = ta[:, 0]
    _lib.call('b200rl_cql_bc_actor_loss', _lib.ptr(th), _lib.dptr(ta0), 2 * A, _lib.ptr(tmin),
              _lib.ptr(tmax), _lib.ptr(tlp), _lib.ptr(tw), _lib.ptr(la), _lib.ptr(counter), 3, B, A,
              lw, gb, _lib.ptr(loss), _lib.ptr(dq1), _lib.ptr(dq2), _lib.ptr(nan), _lib.stream())
    _lib.call('b200rl_cql_bc_actor_bwd', _lib.ptr(th), _lib.dptr(ta0), 2 * A, _lib.ptr(tmin),
              _lib.ptr(tmax), _lib.ptr(tw), _lib.ptr(counter), 3, B, A, lw, gb, _lib.ptr(dhead),
              _lib.stream())
    if not bc:            # past the BC phase nothing is touched
      assert loss.item() == 123.0 and bool((dq1 == 1).all()) and bool((dq2 == 1).all())
      assert np.array_equal(dhead.cpu().numpy(), dhead0)
      continue
    assert nan.item() == 0 and bool((dq1 == 0).all()) and bool((dq2 == 0).all())
    bad = ta0.clone()
    bad[1, 0] = float(amax[0]) + 1.0   # (w[1] != 0) outside the spec: NaN, as in the reference
    _lib.call('b200rl_cql_bc_actor_loss', _lib.ptr(th), _lib.ptr(bad), A, _lib.ptr(tmin),
              _lib.ptr(tmax), _lib.ptr(tlp), _lib.ptr(tw), _lib.ptr(la), _lib.ptr(counter), 3, B, A,
              lw, gb, _lib.ptr(torch.empty(1, device=cuda)), _lib.ptr(torch.empty(B, device=cuda)),
              _lib.ptr(torch.empty(B, device=cuda)), _lib.ptr(nan), _lib.stream())
    assert nan.item() == 1
    h = torch.tensor(head.astype(np.float64), requires_grad=True)
    half, shift = R.t64((amax - amin) / 2), R.t64((amax + amin) / 2)
    y = torch.clamp((R.t64(act[:, 0]) - shift) / half, -float(ocql.TANH_CLIP), float(ocql.TANH_CLIP))
    u = torch.atanh(y)
    z = (u - h[:, :A]) / torch.exp(h[:, A:])
    lpd = (-0.5 * z * z - h[:, A:] - 0.5 * R.LOG2PI - torch.log(half)
           - 2 * (R.LOG2 - u - R.softplus(-2 * u))).sum(1)
    ref = lw * R.aggregate(math.exp(0.3) * R.t64(logp) - lpd, R.t64(w), gb)
    (g,) = torch.autograd.grad(ref, h)
    np.testing.assert_allclose(loss.item(), ref.item(), rtol=1e-5)
    got = dhead.cpu().double() - R.t64(dhead0)
    e = R.grad_errors(got, g)
    record_parity('cql_bc_kernels', rel_l2=e[0], max=e[1])
    R.assert_grad_close('bc/dhead', got, g, 1e-5, 1e-5)


def test_candidates_supplied_and_device_draws(cuda):
  rng = np.random.RandomState(2)
  B, N, D, A = 33, 10, 17, 6
  obs = rng.randn(B, 2, D).astype(f32)
  head = rng.randn(B, 2 * A).astype(f32)
  u = rng.rand(B * N, A).astype(f32)
  tobs, thead, tu, tmin, tmax = (_d(cuda, x) for x in (obs, head, u, AMIN, AMAX))
  x = torch.full((B + 2 * B * N, D + A), float('nan'), device=cuda)
  ht = torch.empty(B * N, 2 * A, device=cuda)
  o0 = tobs[:, 0]
  _lib.call('b200rl_cql_candidates', _lib.dptr(o0), 2 * D, B, N, D, A, _lib.ptr(tmin), _lib.ptr(tmax),
            _lib.ptr(tu), 0, None, _lib.ptr(thead), _lib.ptr(x), _lib.ptr(ht), _lib.stream())
  xs = x.cpu().numpy()
  BN = B * N
  np.testing.assert_array_equal(xs[B:, :D], np.tile(np.repeat(obs[:, 0], N, 0), (2, 1)))
  np.testing.assert_array_equal(xs[B + BN:, D:], ocql.uniform_actions(u, AMIN, AMAX))
  assert np.isnan(xs[:B]).all() and np.isnan(xs[B:B + BN, D:]).all()   # left to the caller
  np.testing.assert_array_equal(ht.cpu().numpy(), np.repeat(head, N, 0))
  # device draws: inside [min, max), uniform moments, one call per launch
  rngs = torch.zeros(2, dtype=torch.int64, device=cuda)
  Bd = 20000
  obsd = torch.zeros(Bd, D, device=cuda)
  headd = torch.zeros(Bd, 2 * A, device=cuda)
  xd = torch.empty(Bd + 2 * Bd * N, D + A, device=cuda)
  htd = torch.empty(Bd * N, 2 * A, device=cuda)
  _lib.call('b200rl_cql_candidates', _lib.ptr(obsd), D, Bd, N, D, A, _lib.ptr(tmin), _lib.ptr(tmax),
            None, 11, _lib.ptr(rngs), _lib.ptr(headd), _lib.ptr(xd), _lib.ptr(htd), _lib.stream())
  assert rngs.cpu().tolist() == [1, 0]
  a = xd[Bd + Bd * N:, D:].double()
  lo, hi = R.t64(AMIN).to(cuda), R.t64(AMAX).to(cuda)
  assert bool((a >= lo).all()) and bool((a <= hi).all())
  s = (a - lo) / (hi - lo)
  n = s.shape[0]
  assert float((s.mean(0) - 0.5).abs().max()) < 5 * math.sqrt(1 / 12 / n)
  assert float((s.var(0) - 1 / 12).abs().max()) < 5 * math.sqrt(1 / 180 / n)
  first = xd.clone()
  _lib.call('b200rl_cql_candidates', _lib.ptr(obsd), D, Bd, N, D, A, _lib.ptr(tmin), _lib.ptr(tmax),
            None, 11, _lib.ptr(rngs), _lib.ptr(headd), _lib.ptr(xd), _lib.ptr(htd), _lib.stream())
  assert rngs.cpu().tolist() == [2, 0] and not torch.equal(first, xd)


def test_device_rng_cql_loss_mean_matches_monte_carlo(cuda):
  """K copies of the testCqlLoss batch with device-drawn uniform actions: the mean CQL loss is the
  estimator's mean, -2.359 (oracle Monte Carlo, per-batch sd 0.127; the reference's one TF draw
  gave -2.307371)."""
  K, N = 10000, 10
  B = 2 * K
  obs = _d(cuda, np.tile(np.array([[1, 2], [3, 4]], f32), (K, 1)))
  lo, hi = _d(cuda, np.array([-1.0], f32)), _d(cuda, np.array([1.0], f32))
  rngs = torch.zeros(2, dtype=torch.int64, device=cuda)
  x = torch.empty(B + 2 * B * N, 3, device=cuda)
  ht = torch.empty(B * N, 2, device=cuda)
  head = torch.zeros(B, 2, device=cuda)
  _lib.call('b200rl_cql_candidates', _lib.ptr(obs), 2, B, N, 2, 1, _lib.ptr(lo), _lib.ptr(hi), None,
            5, _lib.ptr(rngs), _lib.ptr(head), _lib.ptr(x), _lib.ptr(ht), _lib.stream())
  a_unif = x[B + B * N:, 2].reshape(B, N).cpu().numpy()
  qj, logp = _mock_rows(a_unif)
  out = _cql_loss_call(cuda, qj, qj, logp, B, N, ocql.uniform_log_prob(-1.0, 1.0, 1), alpha=1.0)[0]
  record_parity('cql_device_rng_mean', abs_dev=abs(out[0] + 2.359))
  assert abs(out[0] - -2.359) < 5 * 0.127 / math.sqrt(K)


def test_reward_noise_kernel(cuda):
  B = 100000
  r = _d(cuda, np.linspace(-1, 1, B).astype(f32))
  std = _d(cuda, np.float32(0.3))
  z = _d(cuda, np.random.RandomState(0).randn(B).astype(f32))
  out = torch.empty(B, device=cuda)
  _lib.call('b200rl_cql_reward_noise', _lib.ptr(r), B, _lib.ptr(std), _lib.ptr(z), 0, None,
            _lib.ptr(out), _lib.stream())
  np.testing.assert_array_equal(out.cpu().numpy(), (r.cpu().numpy() + z.cpu().numpy() * f32(0.3)).astype(f32))
  rngs = torch.zeros(2, dtype=torch.int64, device=cuda)
  _lib.call('b200rl_cql_reward_noise', _lib.ptr(r), B, _lib.ptr(std), None, 3, _lib.ptr(rngs),
            _lib.ptr(out), _lib.stream())
  e = ((out - r) / 0.3).double()
  assert abs(e.mean().item()) < 5 / math.sqrt(B) and abs(e.std().item() - 1) < 0.02
  assert rngs.cpu().tolist() == [1, 0]
  std.fill_(0.0)          # a variable noise level set to 0: the rewards pass through
  _lib.call('b200rl_cql_reward_noise', _lib.ptr(r), B, _lib.ptr(std), None, 3, _lib.ptr(rngs),
            _lib.ptr(out), _lib.stream())
  assert torch.equal(out, r)


# ---- the agent ----------------------------------------------------------------------------------
D_OBS, A_ACT = 17, 6


def _mirror(net):
  return onn.Sequential([dict(kind='dense', w=l.kernel.cpu().numpy().copy(), b=l.bias.cpu().numpy().copy(),
                              act=l.activation) for l in net.layers if isinstance(l, L.Dense)])


def _make(cuda, opt=lambda: optimizers.Adam(3e-4), hidden=(64, 64), amin=-1.0, amax=1.0, **kw):
  obs_spec = tensor_spec.TensorSpec((D_OBS,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((A_ACT,), torch.float32, amin, amax, 'action')
  actor = tnp.TanhNormalActorNetwork(obs_spec, act_spec, fc_layer_params=hidden, device=cuda).set_seed(1)
  critic = critic_network.CriticNetwork((obs_spec, act_spec), joint_fc_layer_params=hidden,
                                        device=cuda).set_seed(2)
  base = dict(cql_alpha=2.0, num_cql_samples=10, include_critic_entropy_term=False,
              use_lagrange_cql_alpha=False, target_update_tau=0.005, gamma=0.99,
              reward_scale_factor=0.1, random_seed=3)
  base.update(kw)
  agent = cql_sac_agent.CqlSacAgent(ts.time_step_spec(obs_spec), act_spec, critic_network=critic,
                                    actor_network=actor, actor_optimizer=opt(),
                                    critic_optimizer=opt(), alpha_optimizer=opt(), **base)
  agent.initialize()
  return agent


def _oracle_of(agent, amin, amax, **kw):
  return ocql.CqlSacOracle(
      _mirror(agent._actor_network), _mirror(agent._critic_network_1), _mirror(agent._critic_network_2),
      np.broadcast_to(np.asarray(amin, f32), (A_ACT,)).copy(),
      np.broadcast_to(np.asarray(amax, f32), (A_ACT,)).copy(), ooptim.AdamTF(3e-4, eps=1e-7),
      ooptim.AdamTF(3e-4, eps=1e-7), ooptim.AdamTF(3e-4, eps=1e-7), gamma=0.99, reward_scale=0.1,
      tau=0.005, uniform_logp=agent._uniform_logp, **kw)


def _batch(rng, B, amin=-1.0, amax=1.0):
  lo = np.broadcast_to(np.asarray(amin, f32), (A_ACT,))
  hi = np.broadcast_to(np.asarray(amax, f32), (A_ACT,))
  act = (lo + (hi - lo) * rng.rand(B, 2, A_ACT)).astype(f32)
  act[:3, 0] = lo
  act[3:6, 0] = hi                       # dataset actions at the bounds
  return dict(observation=rng.randn(B, 2, D_OBS).astype(f32), action=act,
              reward=rng.rand(B, 2).astype(f32), discount=(rng.rand(B, 2) > .05).astype(f32))


def _traj(cuda, e):
  d = lambda a: torch.as_tensor(a, device=cuda)
  B = e['reward'].shape[0]
  ones = torch.ones(B, 2, dtype=torch.int32, device=cuda)
  return trajectory.Trajectory(ones, d(e['observation']), d(e['action']), (), ones, d(e['reward']),
                               d(e['discount']))


def _draws(rng, B, N, noise=False):
  return ([rng.randn(B, A_ACT).astype(f32) for _ in range(3)] +
          [rng.randn(B * N, A_ACT).astype(f32), rng.rand(B * N, A_ACT).astype(f32),
           rng.randn(B).astype(f32) if noise else None])


CONFIGS = {
    'plain': dict(),
    'entropy': dict(include_critic_entropy_term=True),
    'lagrange_clipped': dict(use_lagrange_cql_alpha=True, cql_alpha=5.0, cql_alpha_learning_rate=0.05,
                             cql_tau=1.0, log_cql_alpha_clipping=(-1.0, 1.62)),
    'bc_boundary': dict(num_bc_steps=2),
    'bc_debug': dict(bc_debug_mode=True),
    'reward_noise': dict(reward_noise_variance=0.3, softmax_temperature=0.5),
    'tensor_alpha': dict(),
    'per_dim_bounds': dict(),
}


@pytest.mark.parametrize('config', sorted(CONFIGS))
def test_cql_agent_train_parity(cuda, config):
  rng = np.random.RandomState(sorted(CONFIGS).index(config))
  B, N = 256, 10
  kw = dict(CONFIGS[config])
  amin, amax = (AMIN, AMAX) if config == 'per_dim_bounds' else (-1.0, 1.0)
  alpha_t = None
  if config == 'tensor_alpha':
    alpha_t = torch.tensor(2.0, device=cuda)
    kw['cql_alpha'] = alpha_t
  agent = _make(cuda, amin=amin, amax=amax, **kw)
  okw = {k: v for k, v in kw.items() if k not in ('cql_alpha',)}
  orc = _oracle_of(agent, amin, amax, cql_alpha=float(kw.get('cql_alpha', 2.0)), num_cql_samples=N,
                   **okw)
  for step in range(5):
    if alpha_t is not None and step == 2:
      alpha_t.fill_(3.5)                   # the reference's tf.Variable changed between steps
      orc.cql_alpha = f32(3.5)
    e = _batch(rng, B, amin, amax)
    draws = _draws(rng, B, N, noise='reward_noise_variance' in kw)
    want = orc.train(e, *draws)
    got = agent.train(_traj(cuda, e), noise=draws)
    fields = dict(loss=got.loss, **got.extra._asdict())
    for k, v in fields.items():
      rel = abs(v.item() - want[k]) / max(abs(want[k]), 1e-6)
      record_parity('cql_agent_parity_' + config, **{k: rel})
      # bc_debug_mode: the critics' output-bias CQL gradient is zero in exact arithmetic (each
      # state's softmax sums to 1 against -1 at its data row), so Adam turns its rounding into
      # lr-sized steps; the TD loss, which does not steer the critics there, drifts with them.
      rtol = 1e-3 if (config == 'bc_debug' and k == 'critic_loss') else 1e-5
      np.testing.assert_allclose(v.item(), want[k], rtol=rtol, atol=1e-6, err_msg=f'{config} step {step} {k}')
  agent.check_numerics()
  assert int(agent.train_step_counter.item()) == 5
  if kw.get('use_lagrange_cql_alpha'):
    np.testing.assert_allclose(agent.cql_alpha.item(), orc._alpha_now(), rtol=1e-5)
  # the device-RNG path draws fresh candidates and stays finite
  l1 = agent.train(_traj(cuda, e)).extra.cql_loss.item()
  l2 = agent.train(_traj(cuda, e)).extra.cql_loss.item()
  assert np.isfinite(l1) and np.isfinite(l2) and l1 != l2
  agent.check_numerics()


class RecordingOptimizer(optimizers.Optimizer):
  def __init__(self):
    super().__init__()
    self.calls = []

  def apply_flat(self, params, grads, grad_scale=None):
    self.calls.append(grads.clone())


def _layers64(net):
  return [(R.t64(l.kernel).requires_grad_(), R.t64(l.bias).requires_grad_(), l.activation)
          for l in net.layers if isinstance(l, L.Dense)]


def _params(layers):
  return [p for w, b, _ in layers for p in (w, b)]


def _views(net):
  return [g for l in net.layers if isinstance(l, L.Dense) for g in (l.d_kernel, l.d_bias)]


@pytest.mark.parametrize('bc', [False, True])
def test_cql_agent_gradients(cuda, bc):
  """Critic (TD + CQL) and actor (SAC or BC) gradients handed to the optimizer against float64
  autograd, per tensor, with the bounds of test_agent_grads_gpu.py."""
  rng = np.random.RandomState(30 + bc)
  B, N, temp, lw_c, lw_a = 200, 4, 0.7, 1.3, 0.8
  opts = iter([RecordingOptimizer() for _ in range(3)])
  agent = _make(cuda, opt=lambda: next(opts), amin=AMIN, amax=AMAX, cql_alpha=1.7, num_cql_samples=N,
                softmax_temperature=temp, critic_loss_weight=lw_c, actor_loss_weight=lw_a,
                include_critic_entropy_term=True, num_bc_steps=5 if bc else 0, initial_log_alpha=0.4)
  c1, c2, actor = agent._critic_network_1, agent._critic_network_2, agent._actor_network
  A64, C1, C2 = _layers64(actor), _layers64(c1), _layers64(c2)
  T1, T2 = _layers64(agent._target_critic_network_1), _layers64(agent._target_critic_network_2)
  e = _batch(rng, B, AMIN, AMAX)
  w = (rng.rand(B) * 2).astype(f32)
  w[rng.rand(B) < 0.2] = 0
  draws = _draws(rng, B, N)
  agent.train(_traj(cuda, e), weights=torch.as_tensor(w, device=cuda), noise=draws)
  agent.check_numerics()
  lo, hi = R.t64(AMIN), R.t64(AMAX)
  o0, o1 = R.t64(e['observation'][:, 0]), R.t64(e['observation'][:, 1])
  W = R.t64(w)
  eps_next, eps_actor, _, eps_cql, u_cql, _ = [None if x is None else R.t64(x) for x in draws]
  with torch.no_grad():
    a2, _, logp2 = R.sac_sample(R.mlp(A64, o1), eps_next, lo, hi)
    x2 = torch.cat([o1, a2], 1)
    tq1, tq2 = R.mlp(T1, x2)[:, 0], R.mlp(T2, x2)[:, 0]
    a_pi, _, logp_pi = R.sac_sample(R.mlp(A64, o0).repeat_interleave(N, 0), eps_cql, lo, hi)
    a_u = lo + u_cql * (hi - lo)
  x = torch.cat([torch.cat([o0, R.t64(e['action'][:, 0])], 1),
                 torch.cat([o0.repeat_interleave(N, 0), a_pi], 1),
                 torch.cat([o0.repeat_interleave(N, 0), a_u], 1)], 0)
  q1, q2 = R.mlp(C1, x)[:, 0], R.mlp(C2, x)[:, 0]
  closs, _ = R.sac_critic_loss(q1[:B], q2[:B], tq1, tq2, logp2, R.t64(e['reward'][:, 0]),
                               R.t64(e['discount'][:, 0]), 0.4, 0.99, 0.1, lw_c, float(B), W)
  ulogp = float(agent._uniform_logp)
  terms = []
  for q in (q1, q2):
    z = torch.cat([q[B:B + B * N].reshape(B, N) * temp - logp_pi.reshape(B, N),
                   q[B + B * N:].reshape(B, N) * temp - ulogp], 1)
    terms.append(torch.logsumexp(z, 1) / temp - q[:B])
  total = closs + 1.7 * (terms[0] + terms[1]).mean() / 2
  g = torch.autograd.grad(total, _params(C1) + _params(C2))
  got = agent._critic_optimizer.calls[0]
  base = agent._critic_grads.data_ptr()
  recorded = [got[(v.data_ptr() - base) // 4:(v.data_ptr() - base) // 4 + v.numel()].view(v.shape)
              for v in _views(c1) + _views(c2)]
  for i, (gg, rr) in enumerate(zip(recorded, g)):
    e_ = R.grad_errors(gg, rr)
    record_parity('cql_agent_grads_critic', **{f'{i}_rel_l2': e_[0], f'{i}_max': e_[1]})
    R.assert_grad_close(f'cql critic/{i}', gg, rr, 1e-4, 1e-4)
  # actor step: the critics have not moved (recording optimizer)
  a, _, logp = R.sac_sample(R.mlp(A64, o0), eps_actor, lo, hi)
  if bc:
    h = R.mlp(A64, o0)
    half, shift = (hi - lo) / 2, (hi + lo) / 2
    y = torch.clamp((R.t64(e['action'][:, 0]) - shift) / half, -float(ocql.TANH_CLIP), float(ocql.TANH_CLIP))
    u = torch.atanh(y)
    zz = (u - h[:, :A_ACT]) / torch.exp(h[:, A_ACT:])
    lpd = (-0.5 * zz * zz - h[:, A_ACT:] - 0.5 * R.LOG2PI - torch.log(half)
           - 2 * (R.LOG2 - u - R.softplus(-2 * u))).sum(1)
    aloss = lw_a * R.aggregate(math.exp(0.4) * logp - lpd, W, float(B))
  else:
    xa = torch.cat([o0, a], 1)
    aloss = R.sac_actor_loss(R.mlp(C1, xa)[:, 0], R.mlp(C2, xa)[:, 0], logp, 0.4, lw_a, float(B), W)
  g = torch.autograd.grad(aloss, _params(A64))
  got = agent._actor_optimizer.calls[0]
  base = actor.flat_grads.data_ptr()
  recorded = [got[(v.data_ptr() - base) // 4:(v.data_ptr() - base) // 4 + v.numel()].view(v.shape)
              for v in _views(actor)]
  for i, (gg, rr) in enumerate(zip(recorded, g)):
    e_ = R.grad_errors(gg, rr)
    record_parity('cql_agent_grads_actor_bc' if bc else 'cql_agent_grads_actor',
                  **{f'{i}_rel_l2': e_[0], f'{i}_max': e_[1]})
    R.assert_grad_close(f'cql actor/{i}', gg, rr, 1e-4, 1e-4)


def test_graph_replay_matches_eager_across_bc_boundary_and_lagrange(cuda):
  rng = np.random.RandomState(40)
  kw = dict(num_bc_steps=3, use_lagrange_cql_alpha=True, cql_alpha=5.0, cql_alpha_learning_rate=0.05,
            cql_tau=1.0, log_cql_alpha_clipping=(-1.0, 3.0), reward_noise_variance=0.2)
  eager, graphed = _make(cuda, **kw), _make(cuda, **kw)
  train_fn = common.function(graphed.train)
  e = _batch(rng, 256)
  traj = _traj(cuda, e)
  for step in range(7):
    l1 = eager.train(traj)
    l2 = train_fn(traj)
    for k in ('critic_loss', 'actor_loss', 'cql_loss', 'cql_alpha', 'cql_alpha_loss'):
      np.testing.assert_allclose(getattr(l2.extra, k).item(), getattr(l1.extra, k).item(), rtol=1e-5,
                                 atol=1e-6, err_msg=f'step {step} {k}')
  assert int(graphed.train_step_counter.item()) == 7 and graphed._train_step_host == 7
  torch.testing.assert_close(graphed._log_cql_alpha, eager._log_cql_alpha, rtol=1e-5, atol=1e-6)
  torch.testing.assert_close(graphed._actor_network.flat_params, eager._actor_network.flat_params,
                             rtol=1e-4, atol=1e-6)


def test_checkpoint_restore_reproduces_next_step(cuda, tmp_path):
  rng = np.random.RandomState(50)
  kw = dict(num_bc_steps=3, use_lagrange_cql_alpha=True, cql_alpha=5.0, cql_alpha_learning_rate=0.05,
            cql_tau=1.0)
  agent = _make(cuda, **kw)
  for _ in range(2):
    agent.train(_traj(cuda, _batch(rng, 64)), noise=_draws(rng, 64, 10))
  ck = common.Checkpointer(str(tmp_path), max_to_keep=1, agent=agent)
  ck.save(agent.train_step_counter)
  restored = _make(cuda, **dict(kw, cql_alpha=1.0))
  assert common.Checkpointer(str(tmp_path), max_to_keep=1, agent=restored).initialize_or_restore()
  assert int(restored.train_step_counter.item()) == 2
  for _ in range(2):                       # crosses the BC boundary (num_bc_steps = 3)
    e, draws = _batch(rng, 64), _draws(rng, 64, 10)
    l1 = agent.train(_traj(cuda, e), noise=draws)
    l2 = restored.train(_traj(cuda, e), noise=draws)
    for k, v in l1.extra._asdict().items():
      np.testing.assert_allclose(getattr(l2.extra, k).item(), v.item(), rtol=1e-5, atol=1e-7, err_msg=k)


def test_multi_replica_is_rejected(cuda):
  agent = _make(cuda)
  agent.replicas = 2
  with pytest.raises(NotImplementedError):
    agent.train(_traj(cuda, _batch(np.random.RandomState(0), 8)))
