"""The gradient metric of the gradient tests rejects the errors Adam hides.

Adam's first step moves every element by about lr·g/|g|, so a gradient that is off by a constant
factor trains the same as the correct one.  These float64 problems show that the metric the GPU
gradient tests use (grad_refs.assert_grad_close, at the loosest bound any of them may use) fails a
gradient scaled by 1.01, a SAC actor gradient without the action half-range, one with α replaced
by 1, a PPO gradient without its l2 term and a loss divided by B instead of the global batch, and
that it accepts the reference rounded to float32.  Host only: no CUDA device needed.
"""
import numpy as np
import pytest
import torch

import grad_refs as R

BOUND = R.MAX_BOUND


def _layers(rng, sizes, act):
  out = []
  for i, (a, b) in enumerate(zip(sizes[:-1], sizes[1:])):
    w = torch.tensor(rng.randn(a, b) / np.sqrt(a), dtype=R.F64, requires_grad=True)
    bias = torch.tensor(rng.randn(b) * 0.1, dtype=R.F64, requires_grad=True)
    out.append((w, bias, act if i < len(sizes) - 2 else None))
  return out


def _params(layers):
  return [p for w, b, _ in layers for p in (w, b)]


def _sac_actor_grads(amin, amax, log_alpha, global_batch):
  """Actor-parameter gradient of the SAC actor loss through the tanh-Normal sample and twin
  critics (fixed seed: every call sees the same networks and data)."""
  rng = np.random.RandomState(0)
  B, D, A = 64, 7, 3
  actor = _layers(rng, [D, 32, 2 * A], 'relu')
  c1, c2 = _layers(rng, [D + A, 32, 1], 'relu'), _layers(rng, [D + A, 32, 1], 'relu')
  obs = torch.tensor(rng.randn(B, D), dtype=R.F64)
  eps = torch.tensor(rng.randn(B, A), dtype=R.F64)
  w = torch.tensor((rng.rand(B) > 0.2) * rng.rand(B), dtype=R.F64)
  a, _, logp = R.sac_sample(R.mlp(actor, obs), eps, amin, amax)
  x = torch.cat([obs, a], dim=1)
  q1, q2 = R.mlp(c1, x)[:, 0], R.mlp(c2, x)[:, 0]
  loss = R.sac_actor_loss(q1, q2, logp, log_alpha, 0.7, global_batch, w)
  return torch.autograd.grad(loss, _params(actor))


def _ppo_grads(policy_l2):
  rng = np.random.RandomState(1)
  N, D, A = 96, 5, 2
  actor = _layers(rng, [D, 16, A], 'tanh')
  value = _layers(rng, [D, 16, 1], 'tanh')
  std_bias = torch.tensor(rng.randn(A) * 0.3, dtype=R.F64, requires_grad=True)
  amin, amax = torch.tensor([-2.0, 0.0], dtype=R.F64), torch.tensor([1.0, 10.0], dtype=R.F64)
  obs = torch.tensor(rng.randn(N, D), dtype=R.F64)
  loc, scale = R.normal_projection(R.mlp(actor, obs), std_bias, amin, amax)
  action = (loc + scale * torch.tensor(rng.randn(N, A))).detach()
  old_logp = R.normal_log_prob(loc, scale, action).detach() + torch.tensor(rng.randn(N) * 0.2)
  v = R.mlp(value, obs)[:, 0]
  w = torch.tensor((rng.rand(N) > 0.1).astype(np.float64))
  loss = R.ppo_loss(R.normal_log_prob(loc, scale, action), R.normal_entropy(scale), old_logp,
                    torch.tensor(rng.randn(N)), torch.tensor(rng.randn(N)), v, v.detach(), w,
                    float(N), 0.2, 0.2, 0.5, 0.01)
  loss = loss + R.l2_loss([k for k, _, _ in actor], policy_l2)
  params = _params(actor) + [std_bias] + _params(value)
  return torch.autograd.grad(loss, params)


AMIN = torch.tensor([-2.0, 0.0, -0.5], dtype=R.F64)
AMAX = torch.tensor([1.0, 10.0, 0.5], dtype=R.F64)


def _reference():
  return _sac_actor_grads(AMIN, AMAX, 0.7, 128.0)


def _rejected(got, ref):
  return any(not R.grad_close(g, r, BOUND, BOUND) for g, r in zip(got, ref))


def test_metric_accepts_the_reference_rounded_to_float32():
  ref = _reference()
  assert not _rejected([g.float() for g in ref], ref)
  ref = _ppo_grads(0.01)
  assert not _rejected([g.float() for g in ref], ref)


def test_metric_rejects_a_constant_factor():
  ref = _reference()
  assert _rejected([1.01 * g for g in ref], ref)


def test_metric_rejects_a_missing_half_range():
  # same shift, half-range 1: a = shift + tanh(u) (what a backward that drops `half` computes)
  shift = (AMAX + AMIN) / 2
  assert _rejected(_sac_actor_grads(shift - 1, shift + 1, 0.7, 128.0), _reference())


def test_metric_rejects_alpha_replaced_by_one():
  assert _rejected(_sac_actor_grads(AMIN, AMAX, 0.0, 128.0), _reference())


def test_metric_rejects_dividing_by_the_local_batch():
  # the reference uses global_batch = 2B; the mutant divides by B = 64
  assert _rejected(_sac_actor_grads(AMIN, AMAX, 0.7, 64.0), _reference())


def test_metric_rejects_a_missing_l2_term():
  assert _rejected(_ppo_grads(0.0), _ppo_grads(0.01))


def test_metric_errors_report_the_measured_size():
  ref = _reference()
  rel, mx = R.grad_errors([1.01 * g for g in ref][0], ref[0])
  assert rel == pytest.approx(0.01, rel=1e-9) and mx == pytest.approx(0.01, rel=1e-9)
  with pytest.raises(AssertionError, match='relative L2 error'):
    R.assert_grad_close('scaled', 1.01 * ref[0], ref[0], BOUND, BOUND)
  with pytest.raises(AssertionError, match='bound above'):
    R.assert_grad_close('loose', ref[0], ref[0], 2e-3, BOUND)
