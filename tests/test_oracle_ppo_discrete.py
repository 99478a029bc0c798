"""Host checks of discrete-action PPO: the categorical oracle against torch CPU autograd and
torch.distributions, the policy's recorded distribution parameters and the spec validation."""
import numpy as np
import pytest
import torch

from agents_b200.agents.ppo import ppo_policy
from agents_b200.networks import actor_distribution_network as adn
from agents_b200.networks import layers as L
from agents_b200.networks import value_network
from agents_b200.specs import tensor_spec
from agents_b200.trajectories import time_step as ts
from oracle import nn as onn
from oracle import optim as ooptim
from oracle import ppo_discrete as opd

f32 = np.float32


@pytest.mark.parametrize('A', [2, 6, 18, 300])
def test_log_prob_entropy_kl_match_torch(A):
  rng = np.random.RandomState(A)
  N = 257
  z, zo = (rng.randn(N, A) * 3).astype(f32), (rng.randn(N, A) * 3).astype(f32)
  a = rng.randint(0, A, N)
  p, q = torch.distributions.Categorical(logits=torch.tensor(z)), torch.distributions.Categorical(
      logits=torch.tensor(zo))
  np.testing.assert_allclose(opd.categorical_log_prob(z, a), p.log_prob(torch.tensor(a)).numpy(),
                             rtol=1e-5, atol=1e-5)
  np.testing.assert_allclose(opd.categorical_entropy(z), p.entropy().numpy(), rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(opd.categorical_kl(zo, z),
                             torch.distributions.kl_divergence(q, p).numpy(), rtol=1e-4, atol=1e-5)


def _identity_oracle(A, **kw):
  """Actor = identity dense layer (logits = observation), value = first column: the oracle's
  gradients w.r.t. logits / values can then be compared with autograd on the raw tensors."""
  actor = onn.Sequential([dict(kind='dense', w=np.eye(A, dtype=f32), b=np.zeros(A, f32))])
  wv = np.zeros((A, 1), f32)
  wv[0, 0] = 1
  value = onn.Sequential([dict(kind='dense', w=wv, b=np.zeros(1, f32))])
  return opd.CategoricalPPOOracle(actor, value, ooptim.AdamTF(1e-3), **kw)


@pytest.mark.parametrize('cfg', [
    dict(clip_eps=0.2),
    dict(clip_eps=0.2, value_clip=0.3, ent_coef=0.01, logp_clip=1.5),
    dict(clip_eps=0.0, ent_coef=0.05, kl_cutoff_factor=2.0, kl_cutoff_coef=1000.0,
         initial_adaptive_kl_beta=0.7, adaptive_kl_target=0.01, adaptive_kl_tolerance=0.3),
])
def test_loss_backward_matches_autograd(cfg):
  rng = np.random.RandomState(3)
  B, T, A = 9, 7, 6
  N = B * T
  kw = dict(clip_eps=0.2, vf_coef=0.5, ent_coef=0.0, value_clip=0.0, logp_clip=0.0)
  kw.update(cfg)
  orc = _identity_oracle(A, **kw)
  z = (rng.randn(N, A) * 1.5).astype(f32)
  zo = (z + rng.randn(N, A) * 0.3).astype(f32)
  a = rng.randint(0, A, N)
  old_logp = (opd.categorical_log_prob(zo, a)).astype(f32)
  adv, ret = rng.randn(N).astype(f32), rng.randn(N).astype(f32)
  v_old = (z[:, 0] + rng.randn(N) * 0.3).astype(f32)
  w = (rng.rand(N) > 0.2).astype(f32)
  info, _, dlogits, dv = orc.loss_and_grads(z, a, old_logp, ret, adv, v_old, w, B, T,
                                            old_logits=zo)
  tz = torch.tensor(z, dtype=torch.float64, requires_grad=True)
  tv = torch.tensor(z[:, 0], dtype=torch.float64, requires_grad=True)
  d = lambda x: torch.tensor(x, dtype=torch.float64)
  dist = torch.distributions.Categorical(logits=tz)
  lp = dist.log_prob(torch.tensor(a))
  if kw['logp_clip'] > 0:
    lp = torch.clamp(lp, -kw['logp_clip'], kw['logp_clip'])
  ratio = torch.exp(lp - d(old_logp))
  obj = ratio * d(adv)
  if kw['clip_eps'] > 0:
    obj = torch.minimum(obj, torch.clamp(ratio, 1 - kw['clip_eps'], 1 + kw['clip_eps']) * d(adv))
  err = (d(ret) - tv) ** 2
  if kw['value_clip'] > 0:
    vo = d(v_old)
    err = torch.maximum(err, (d(ret) - (vo + torch.clamp(tv - vo, -kw['value_clip'], kw['value_clip']))) ** 2)
  total = ((-obj * d(w)).sum() + kw['vf_coef'] * (err * d(w)).sum()
           + kw['ent_coef'] * (-dist.entropy() * d(w)).sum()) / (T * B)
  if cfg.get('initial_adaptive_kl_beta'):
    q = torch.distributions.Categorical(logits=d(zo))
    mean_kl = (torch.distributions.kl_divergence(q, dist) * d(w)).mean()
    over = torch.clamp(mean_kl - cfg['kl_cutoff_factor'] * cfg['adaptive_kl_target'], min=0)
    total = total + cfg['kl_cutoff_coef'] * over ** 2 + cfg['initial_adaptive_kl_beta'] * mean_kl
  total.backward()
  np.testing.assert_allclose(info['loss'], total.item(), rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(dlogits, tz.grad.numpy(), rtol=1e-4, atol=1e-7)
  np.testing.assert_allclose(dv, tv.grad.numpy(), rtol=1e-4, atol=1e-8)


def test_sampling_oracle_frequencies():
  rng = np.random.RandomState(0)
  A, N = 6, 200000
  z = np.tile((rng.randn(1, A) * 1.2).astype(f32), (N, 1))
  draws, u = opd.categorical_sample(z, seed=1234, call=0)
  assert draws.dtype == np.int32 and draws.min() >= 0 and draws.max() < A
  p = torch.softmax(torch.tensor(z[0], dtype=torch.float64), 0).numpy()
  counts = np.bincount(draws, minlength=A)
  from scipy import stats
  assert stats.chisquare(counts, p * N).pvalue > 1e-4
  again, _ = opd.categorical_sample(z[:10], seed=1234, call=0)
  np.testing.assert_array_equal(again, draws[:10])
  other, _ = opd.categorical_sample(z, seed=1234, call=1)
  assert (other != draws).mean() > 0.3


def _specs():
  obs = tensor_spec.TensorSpec((5,), torch.float32, 'observation')
  act = tensor_spec.BoundedTensorSpec((), torch.int64, 0, 3, 'action')
  return obs, act


def test_dist_params_are_logits():
  # ppo_utils_test.py:102-113: a Categorical policy records {'logits'}
  obs, act = _specs()
  actor = adn.ActorDistributionNetwork(obs, act, fc_layer_params=(8,), device='cpu')
  value = value_network.ValueNetwork(obs, fc_layer_params=(8,), device='cpu')
  assert actor.discrete and actor.num_actions == 4
  pol = ppo_policy.PPOPolicy(ts.time_step_spec(obs), act, actor, value, collect=True)
  assert set(pol.info_spec) == {'dist_params'}
  assert set(pol.info_spec['dist_params']) == {'logits'}
  assert pol.info_spec['dist_params']['logits'].shape == (4,)
  pol = ppo_policy.PPOPolicy(ts.time_step_spec(obs), act, actor, value, collect=True,
                             compute_value_and_advantage_in_train=False)
  assert set(pol.info_spec) == {'dist_params', 'value_prediction'}
  # the continuous head keeps {'loc', 'scale'}
  cont = tensor_spec.BoundedTensorSpec((2,), torch.float32, -1.0, 1.0, 'action')
  cactor = adn.ActorDistributionNetwork(obs, cont, fc_layer_params=(8,), device='cpu')
  assert not cactor.discrete
  assert set(ppo_policy.PPOPolicy(ts.time_step_spec(obs), cont, cactor, value).info_spec[
      'dist_params']) == {'loc', 'scale'}


def test_conv_torso_layers():
  obs = tensor_spec.TensorSpec((84, 84, 4), torch.uint8, 'observation')
  act = tensor_spec.BoundedTensorSpec((1,), torch.int32, 0, 5, 'action')
  conv = ((32, 8, 4), (64, 4, 2), (64, 3, 1))
  actor = adn.ActorDistributionNetwork(obs, act, fc_layer_params=(512,), device='cpu',
                                       preprocessing_layers=L.CastScale(255.), conv_layer_params=conv)
  kinds = [type(l).__name__ for l in actor.layers]
  assert kinds == ['CastScale', 'Conv2D', 'Conv2D', 'Conv2D', 'Flatten', 'Dense', 'Dense']
  assert actor.layers[-1].units == 6
  value = value_network.ValueNetwork(obs, fc_layer_params=(512,), device='cpu',
                                     preprocessing_layers=L.CastScale(255.), conv_layer_params=conv)
  assert [type(l).__name__ for l in value.layers][-3:] == ['Flatten', 'Dense', 'Dense']
  # without a conv front the MLP nets keep their plain Dense stacks
  mlp = adn.ActorDistributionNetwork(tensor_spec.TensorSpec((5,), torch.float32), act,
                                     fc_layer_params=(8,), device='cpu')
  assert [type(l).__name__ for l in mlp.layers] == ['Dense', 'Dense']


@pytest.mark.parametrize('spec, match', [
    (tensor_spec.BoundedTensorSpec((2,), torch.int32, 0, 3), r'shape \(\) or \(1,\)'),
    (tensor_spec.BoundedTensorSpec((), torch.int32, 1, 3), 'minimum == 0'),
    (tensor_spec.TensorSpec((), torch.int32), 'BoundedTensorSpec'),
    ([tensor_spec.BoundedTensorSpec((), torch.int32, 0, 3)] * 2, 'nested or multiple'),
    ({'a': tensor_spec.BoundedTensorSpec((), torch.int32, 0, 3),
      'b': tensor_spec.BoundedTensorSpec((1,), torch.float32, -1.0, 1.0)}, 'nested or multiple'),
])
def test_bad_discrete_specs_are_rejected(spec, match):
  obs = tensor_spec.TensorSpec((5,), torch.float32)
  with pytest.raises(ValueError, match=match):
    adn.ActorDistributionNetwork(obs, spec, device='cpu')
