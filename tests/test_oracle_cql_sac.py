"""Pins oracle/cql_sac.py to the scalar goldens of agents/cql/cql_sac_agent_test.py and checks its
hand-written gradients against float64 autograd (tests/grad_refs.py metric)."""
import numpy as np
import pytest
import torch

import grad_refs as R
from agents_b200.agents.cql import cql_sac_agent
from agents_b200.specs import tensor_spec
from oracle import cql_sac as ocql
from oracle import nn as onn
from oracle import optim as ooptim
from oracle import sac as osac

f32 = np.float32
OBS = np.array([[1, 2], [3, 4]], f32)
ACT = np.array([[5], [6]], f32)


def _dummy_critic(obs, act):
  # DummyCriticNet (cql_sac_agent_test.py:96-142): q = obs @ [0, 1] + act @ [1]
  return (obs[:, 1] + act[:, 0]).astype(f32)


def _mock_cql_loss(a_unif, cql_alpha=1.0, N=10):
  """testCqlLoss (:237-267) with DummyActorPolicy (action = spec.maximum = 1, log_prob 10) and
  the uniform actions a_unif [B, N] given; spec bounds (-1, 1), A = 1."""
  B = OBS.shape[0]
  q = _dummy_critic(OBS, ACT)
  q_pi = np.repeat(_dummy_critic(OBS, np.ones((B, 1), f32))[:, None], N, 1)
  q_u = (OBS[:, 1:2] + a_unif).astype(f32)
  loss, _ = ocql.cql_loss(q, q, q_pi, q_pi, np.full((B, N), 10, f32), q_u, q_u,
                          ocql.uniform_log_prob(-1.0, 1.0, 1))
  return f32(loss * f32(cql_alpha))


@pytest.mark.parametrize('entropy, want', [(False, [16.3, 28.1]), (True, [7.3, 19.1])])
def test_critic_loss_golden(entropy, want):  # :349-409
  q = _dummy_critic(OBS, ACT)
  tq = _dummy_critic(np.array([[5, 6], [7, 8]], f32), np.ones((2, 1), f32))
  loss, y = ocql.critic_loss(q, q, tq, tq, np.full(2, 10, f32), np.array([10, 20], f32),
                             np.array([.9, .9], f32), 0.0, entropy)
  np.testing.assert_allclose(y, want, rtol=1e-6)
  np.testing.assert_allclose(loss, 2 * np.mean((np.array(want) - [7., 10.]) ** 2), rtol=1e-6)


def test_critic_loss_reward_noise_before_scale():
  q = np.zeros(2, f32)
  z = np.array([1.5, -2.0], f32)
  _, y = ocql.critic_loss(q, q, q, q, np.zeros(2, f32), np.array([10, 20], f32), np.ones(2, f32),
                          0.0, False, reward_scale=3.0, noise_std=0.1, z_reward=z)
  np.testing.assert_allclose(y, 3.0 * (np.array([10, 20]) + 0.1 * z), rtol=1e-6)


def test_actor_loss_goldens():  # :411-437
  q = _dummy_critic(OBS, np.ones((2, 1), f32))
  np.testing.assert_allclose(osac.actor_loss(q, q, np.full(2, 10, f32), 0.0), 6.0, rtol=1e-6)
  # BC: DummyActorNet emits an unsquashed Normal(loc, scale) = obs @ [[2, 1], [1, 1]] + 5
  head = (OBS @ np.array([[2, 1], [1, 1]], f32) + 5).astype(f32)
  logp_data = torch.distributions.Normal(torch.tensor(head[:, 0]), torch.tensor(head[:, 1])).log_prob(
      torch.tensor(ACT[:, 0])).numpy()
  np.testing.assert_allclose(ocql.bc_actor_loss(np.full(2, 10, f32), logp_data, 0.0), 13.404237,
                             rtol=1e-6)


def test_cql_loss_closed_form_and_scaling():  # :237-267
  zero = np.zeros((2, 10), f32)
  want = np.mean([np.logaddexp(np.log(10) + 3 - 10, np.log(10) + 2 + np.log(2)) - 7,
                  np.logaddexp(np.log(10) + 5 - 10, np.log(10) + 4 + np.log(2)) - 10])
  np.testing.assert_allclose(_mock_cql_loss(zero), want, rtol=1e-6)
  np.testing.assert_allclose(_mock_cql_loss(zero), -2.5042, atol=1e-4)
  rng = np.random.RandomState(3)
  a = (rng.rand(2, 10) * 2 - 1).astype(f32)
  np.testing.assert_allclose(_mock_cql_loss(a, 10.0), 10 * _mock_cql_loss(a, 1.0), rtol=1e-6)
  np.testing.assert_allclose(-23.073713, 10 * -2.307371, rtol=1e-6)   # the reference pair


def test_cql_loss_reference_value_inside_monte_carlo_spread():
  """The reference's -2.307371 comes from TF's uniform stream, which is not reproduced here; it
  must be a plausible draw of the same estimator."""
  rng = np.random.RandomState(0)
  draws = np.array([_mock_cql_loss(ocql.uniform_actions(rng.rand(2, 10).astype(f32)[..., None],
                                                        -1.0, 1.0)[..., 0])
                    for _ in range(20000)])
  mean, sd = draws.mean(), draws.std()
  assert abs(mean - -2.359) < 0.005 and abs(sd - 0.127) < 0.005, (mean, sd)
  assert abs(-2.307371 - mean) < 1.0 * sd


@pytest.mark.parametrize('lo, hi', [(-1.0, 1.0), ([-1.0, -2.0, 0.0], [1.0, 2.0, 3.0]),
                                    ([-1.0, -1.0, -1.0], [1.0, 1.0, 1.0])])
def test_uniform_log_density_bound_layouts(lo, hi):  # :624-631 quirk
  A = 3
  want = -A * np.sum(np.log(np.asarray(hi, np.float64) - np.asarray(lo, np.float64)))
  got = ocql.uniform_log_prob(lo, hi, A)
  np.testing.assert_allclose(got, want, rtol=1e-6)
  spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, lo, hi)
  assert cql_sac_agent.uniform_log_prob(spec) == float(got)
  if np.ndim(lo) == 0:
    np.testing.assert_allclose(got, -A * np.log(2.0), rtol=1e-6)      # -A log(range)
  elif np.all(np.asarray(lo) == -1) and np.all(np.asarray(hi) == 1):
    np.testing.assert_allclose(got, -A * A * np.log(2.0), rtol=1e-6)  # per-dim bounds: A * sum


def test_lagrange_golden():  # :531-654: cql_alpha 5 -> 5 e^-0.5 after one Adam step at lr 0.5
  la = np.array([np.log(f32(5.0))], f32)
  opt = ooptim.AdamTF(0.5, eps=1e-7)
  alpha, loss, g = ocql.lagrange_step(la[0], 2.904868, 10.0, (-1, 10.0))
  np.testing.assert_allclose(alpha, 5.0, rtol=1e-6)
  assert loss > 0 and g == loss
  opt.apply([la], [np.array([g], f32)])
  np.testing.assert_allclose(np.exp(la[0]), 3.032653, rtol=1e-5)
  # clip_by_value: gradient inside [lo, hi] including the bounds, none outside
  for x, passes in ((0.0, True), (-1.0, True), (2.0, True), (2.5, False), (-1.5, False)):
    _, l, g = ocql.lagrange_step(x, 3.0, 10.0, (-1.0, 2.0))
    assert (g == l) if passes else (g == 0)


def _mlp(rng, n_in, hidden, n_out):
  layers = []
  for h in hidden:
    layers.append(dict(kind='dense', w=(rng.randn(n_in, h) * .3).astype(f32),
                       b=(rng.randn(h) * .05).astype(f32), act='relu'))
    n_in = h
  layers.append(dict(kind='dense', w=(rng.randn(n_in, n_out) * .3).astype(f32),
                     b=np.zeros(n_out, f32), act=None))
  return onn.Sequential(layers)


def _oracle(rng, D=2, A=1, **kw):
  return ocql.CqlSacOracle(_mlp(rng, D, (16,), 2 * A), _mlp(rng, D + A, (16,), 1),
                           _mlp(rng, D + A, (16,), 1), -np.ones(A, f32), np.ones(A, f32),
                           ooptim.AdamTF(1e-3), ooptim.AdamTF(1e-3), ooptim.AdamTF(1e-3), **kw)


def _exp(rng, B, D, A):
  return dict(observation=rng.randn(B, 2, D).astype(f32),
              action=(rng.rand(B, 2, A) * 2 - 1).astype(f32), reward=rng.rand(B, 2).astype(f32),
              discount=np.ones((B, 2), f32))


@pytest.mark.parametrize('lagrange, variable, want1, want2', [(True, False, 5.0, 3.032653),
                                                              (False, False, 5.0, 5.0),
                                                              (False, True, 5.0, 6.0)])
def test_train_lagrange_and_variable_cql_alpha(lagrange, variable, want1, want2):
  rng = np.random.RandomState(4)
  B, N = 5, 5
  orc = _oracle(rng, use_lagrange_cql_alpha=lagrange, cql_alpha=5.0, num_cql_samples=N,
                cql_alpha_learning_rate=0.5, cql_tau=10, log_cql_alpha_clipping=(-1, 10.0))
  e = _exp(rng, B, 2, 1)
  draws = lambda: [rng.randn(B, 1).astype(f32) for _ in range(3)] + [
      rng.randn(B * N, 1).astype(f32), rng.rand(B * N, 1).astype(f32)]
  out = orc.train(e, *draws())
  np.testing.assert_allclose(out['cql_alpha'], want1, rtol=1e-6)
  assert (out['cql_alpha_loss'] > 0) if lagrange else (out['cql_alpha_loss'] == 0)
  if variable:
    orc.cql_alpha = f32(orc.cql_alpha + 1)
  out = orc.train(e, *draws())
  np.testing.assert_allclose(out['cql_alpha'], want2, rtol=2e-5)
  assert orc.train_step_counter == 2


def test_cql_loss_gradient_matches_autograd():
  rng = np.random.RandomState(5)
  B, N, tau = 7, 4, 0.7
  t = lambda a: torch.tensor(a.astype(np.float64), requires_grad=True)
  arrs = dict(q1=rng.randn(B), q2=rng.randn(B), q1_pi=rng.randn(B, N) * 3, q2_pi=rng.randn(B, N) * 3,
              q1_unif=rng.randn(B, N) * 3, q2_unif=rng.randn(B, N) * 3)
  logp = (rng.randn(B, N) * 2).astype(f32)
  ulogp = ocql.uniform_log_prob([-1, -2], [1, 3], 2)
  loss, grads = ocql.cql_loss(*[arrs[k].astype(f32) for k in ('q1', 'q2', 'q1_pi', 'q2_pi')], logp,
                              arrs['q1_unif'].astype(f32), arrs['q2_unif'].astype(f32), ulogp, tau)
  T = {k: t(v.astype(f32)) for k, v in arrs.items()}
  lp = torch.tensor(logp.astype(np.float64))
  terms = []
  for i in ('1', '2'):
    z = torch.cat([T['q' + i + '_pi'] * tau - lp, T['q' + i + '_unif'] * tau - float(ulogp)], 1)
    terms.append(torch.logsumexp(z, 1) / tau - T['q' + i])
  ref = (terms[0] + terms[1]).mean() / 2
  np.testing.assert_allclose(loss, ref.item(), rtol=1e-5)
  g = torch.autograd.grad(ref, list(T.values()))
  for k, gr in zip(T, g):
    R.assert_grad_close('cql_loss/' + k, grads[k], gr, 1e-5, 1e-5)


def test_squashed_log_prob_and_gradient_match_autograd():
  rng = np.random.RandomState(6)
  B, A = 64, 3
  amin, amax = np.array([-2, 0, -1], f32), np.array([1, 4, 1], f32)
  head = (rng.randn(B, 2 * A) * .5).astype(f32)
  act = (amin + (amax - amin) * rng.rand(B, A)).astype(f32)
  act[:4] = amin
  act[4:8] = amax                                   # dataset actions at the bounds stay finite
  logp, dhead = ocql.squashed_log_prob(head, act, amin, amax)
  assert np.isfinite(logp).all() and np.isfinite(dhead).all()
  h = torch.tensor(head.astype(np.float64), requires_grad=True)
  half, shift = R.t64((amax - amin) / 2), R.t64((amax + amin) / 2)
  y = torch.clamp((R.t64(act) - shift) / half, -float(ocql.TANH_CLIP), float(ocql.TANH_CLIP))
  u = torch.atanh(y)
  base = torch.distributions.Normal(h[:, :A], torch.exp(h[:, A:])).log_prob(u)
  ref = (base - torch.log(half) - 2 * (R.LOG2 - u - R.softplus(-2 * u))).sum(1)
  np.testing.assert_allclose(logp, ref.detach().numpy(), rtol=1e-5, atol=1e-4)
  (g,) = torch.autograd.grad(ref.sum(), h)
  R.assert_grad_close('bc_logp_dhead', dhead, g, 1e-5, 1e-5)


@pytest.mark.parametrize('num_bc_steps, bc_debug, entropy', [(0, False, False), (2, False, True),
                                                             (0, True, False)])
def test_train_runs_and_counts(num_bc_steps, bc_debug, entropy):
  rng = np.random.RandomState(7)
  B, N, D, A = 6, 3, 4, 2
  orc = _oracle(rng, D, A, cql_alpha=2.0, num_cql_samples=N, num_bc_steps=num_bc_steps,
                bc_debug_mode=bc_debug, include_critic_entropy_term=entropy,
                reward_noise_variance=0.1)
  for step in range(3):
    out = orc.train(_exp(rng, B, D, A), *[rng.randn(B, A).astype(f32) for _ in range(3)],
                    rng.randn(B * N, A).astype(f32), rng.rand(B * N, A).astype(f32),
                    rng.randn(B).astype(f32))
    assert all(np.isfinite(v) for v in out.values())
    crit = out['cql_loss'] * out['cql_alpha'] + (0 if bc_debug else out['critic_loss'])
    np.testing.assert_allclose(out['loss'], crit + out['actor_loss'] + out['alpha_loss'], rtol=1e-5)
  assert orc.train_step_counter == 3
