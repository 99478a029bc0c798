"""PPO on the GPU: reference scalar-loss goldens through the fused kernel, kernel parity vs
oracle/ppo.py, and PPOClipAgent.train parity (losses within 1e-5 relative)."""
import numpy as np
import pytest
import torch

from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.agents.ppo import ppo_clip_agent
from agents_b200.networks import actor_distribution_network
from agents_b200.networks import layers as L
from agents_b200.networks import value_network
from agents_b200.specs import tensor_spec
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory
from agents_b200.utils import tensor_normalizer
from agents_b200.utils import workspace
from oracle import nn as onn
from oracle import optim as ooptim
from oracle import ppo as oppo

from conftest import record_parity

pytestmark = pytest.mark.gpu
f32 = np.float32


def _ppo_loss(cuda, loc, scale, action, old_logp, adv, ret, v, v_old, w, T, **kw):
  N, A = action.shape
  d = lambda a: None if a is None else torch.as_tensor(np.ascontiguousarray(a, dtype=f32), device=cuda)
  t = dict(loc=d(loc), scale=d(scale), action=d(action), old=d(old_logp), adv=d(adv), ret=d(ret),
           v=d(v), vo=d(v_old), w=d(w))
  losses = torch.empty(6, device=cuda)
  dloc = torch.empty(N, A, device=cuda); dscale = torch.empty(N, A, device=cuda); dv = torch.empty(N, device=cuda)
  flag = torch.zeros(1, dtype=torch.int32, device=cuda)
  ws, nb = workspace.get(cuda)
  _lib.call('b200rl_ppo_loss', _lib.ptr(t['loc']), _lib.ptr(t['scale']), A, _lib.ptr(t['action']),
            _lib.ptr(t['old']), _lib.ptr(t['adv']), _lib.ptr(t['ret']), _lib.ptr(t['v']), _lib.ptr(t['vo']),
            _lib.ptr(t['w']), N, A, T, float(kw.get('global_batch', N // T)), kw.get('clip_eps', 0.2),
            kw.get('value_clip', 0.0), kw.get('vf_coef', 0.5), kw.get('ent_coef', 0.0),
            kw.get('logp_clip', 0.0), _lib.ptr(losses), _lib.ptr(dloc), _lib.ptr(dscale), A, _lib.ptr(dv),
            _lib.ptr(flag), None, _lib.ptr(ws), nb, _lib.stream())
  return losses.cpu().numpy(), dloc.cpu().numpy(), dscale.cpu().numpy(), dv.cpu().numpy()


def test_reference_loss_goldens_through_kernel(cuda):
  # agents/ppo/ppo_agent_test.py:919-985 (DummyActorNet -> loc [9,15], scale [8,12]; value [9,15])
  loc, scale = np.array([[9.], [15.]], f32), np.array([[8.], [12.]], f32)
  losses, _, _, _ = _ppo_loss(cuda, loc, scale, np.array([[0.], [1.]], f32), [.9, .3], [1.9, 1.], [1.9, 1.],
                              [9., 15.], None, [1., 1.], T=1, clip_eps=10.0, vf_coef=1.0, ent_coef=0.1)
  np.testing.assert_allclose(losses[0], -0.0164646133, rtol=1e-5)   # policy gradient
  np.testing.assert_allclose(losses[1], 123.205, rtol=1e-6)          # value estimation
  np.testing.assert_allclose(losses[2], -0.370111, rtol=1e-5)        # entropy regularisation
  assert losses[3] == 0.0                                            # clip fraction
  # :644-727: with a time dimension of 2 and half of the weights zero every term is x 2/4
  rep = lambda a: np.repeat(np.asarray(a, f32), 2, axis=0)
  losses, _, _, _ = _ppo_loss(cuda, rep(loc), rep(scale), rep([[0.], [1.]]), rep([.9, .3]), rep([1.9, 1.]),
                              rep([1.9, 1.]), rep([9., 15.]), None, [1., 0., 1., 0.], T=2, clip_eps=10.0,
                              vf_coef=1.0, ent_coef=0.1)
  np.testing.assert_allclose(losses[:3], np.array([-0.0164646133, 123.205, -0.370111]) * 2 / 4, rtol=1e-5)


@pytest.mark.parametrize('cfg', [dict(clip_eps=0.2), dict(clip_eps=0.2, value_clip=0.3, ent_coef=0.01, logp_clip=6.0),
                                 dict(clip_eps=0.0, vf_coef=1.0)])
def test_ppo_loss_kernel_parity(cuda, cfg):
  rng = np.random.RandomState(0)
  B, T, A = 37, 9, 6
  N = B * T
  loc, scale = rng.randn(N, A).astype(f32), (rng.rand(N, A) + .3).astype(f32)
  action = (loc + rng.randn(N, A) * scale).astype(f32)
  old_logp = (oppo.normal_log_prob(loc, scale, action) + rng.randn(N) * .3).astype(f32)
  adv, ret, v = rng.randn(N).astype(f32), rng.randn(N).astype(f32), rng.randn(N).astype(f32)
  v_old = (v + rng.randn(N) * .3).astype(f32)
  w = (rng.rand(N) > .15).astype(f32)
  kw = dict(clip_eps=0.2, value_clip=0.0, vf_coef=0.5, ent_coef=0.0, logp_clip=0.0)
  kw.update(cfg)
  losses, dloc, dscale, dv = _ppo_loss(cuda, loc, scale, action, old_logp, adv, ret, v, v_old, w, T, **kw)
  sh = (B, T)
  logp = oppo.normal_log_prob(loc, scale, action)
  pg, cf = oppo.policy_gradient_loss(logp.reshape(sh), old_logp.reshape(sh), adv.reshape(sh), w.reshape(sh),
                                     kw['clip_eps'], kw['logp_clip'])
  ve = oppo.value_estimation_loss(v.reshape(sh), ret.reshape(sh), w.reshape(sh), kw['vf_coef'],
                                  kw['value_clip'], v_old.reshape(sh))
  en = oppo.entropy_regularization_loss(oppo.normal_entropy(scale).reshape(sh), w.reshape(sh), kw['ent_coef'])
  np.testing.assert_allclose(losses[0], pg, rtol=1e-5, atol=1e-7)
  np.testing.assert_allclose(losses[1], ve, rtol=1e-5)
  np.testing.assert_allclose(losses[2], en, rtol=1e-5, atol=1e-9)
  np.testing.assert_allclose(losses[3], cf, rtol=1e-6)
  # gradients vs torch autograd of the same expression
  tl, tsc, tv = [torch.tensor(x, requires_grad=True) for x in (loc, scale, v)]
  dist = torch.distributions.Normal(tl, tsc)
  lp = dist.log_prob(torch.tensor(action)).sum(-1)
  if kw['logp_clip'] > 0:
    lp = torch.clamp(lp, -kw['logp_clip'], kw['logp_clip'])
  ratio = torch.exp(lp - torch.tensor(old_logp))
  a_t, w_t, r_t = torch.tensor(adv), torch.tensor(w), torch.tensor(ret)
  obj = ratio * a_t
  if kw['clip_eps'] > 0:
    obj = torch.minimum(obj, torch.clamp(ratio, 1 - kw['clip_eps'], 1 + kw['clip_eps']) * a_t)
  err = (r_t - tv) ** 2
  if kw['value_clip'] > 0:
    vo = torch.tensor(v_old)
    err = torch.maximum(err, (r_t - (vo + torch.clamp(tv - vo, -kw['value_clip'], kw['value_clip']))) ** 2)
  total = ((-obj * w_t).sum() + kw['vf_coef'] * (err * w_t).sum()
           + kw['ent_coef'] * (-dist.entropy().sum(-1) * w_t).sum()) / (T * B)
  total.backward()
  # per-element gradients: the kernel's ratio = expf(lp - old_lp) (CUDA libm, <= 2 ulp) vs torch
  # CPU's vectorised exp, and z = (a - loc) / scale squared in a different association, give
  # elements that agree to ~1e-5..1e-4 of their own value (the losses above hold 1e-5); the
  # measured error relative to the largest gradient is recorded (ppo_loss_grads_err_rel_to_max)
  for name, g_, w_ in (('dloc', dloc, tl.grad.numpy()), ('dscale', dscale, tsc.grad.numpy()),
                       ('dv', dv, tv.grad.numpy())):
    record_parity('ppo_loss_grads_err_rel_to_max', **{
        name: float(np.abs(g_ - w_).max()) / max(float(np.abs(w_).max()), 1e-30)})
  np.testing.assert_allclose(dloc, tl.grad.numpy(), rtol=2e-4, atol=1e-8)
  np.testing.assert_allclose(dscale, tsc.grad.numpy(), rtol=2e-4, atol=1e-8)
  np.testing.assert_allclose(dv, tv.grad.numpy(), rtol=2e-4, atol=1e-9)


def test_normalizer_and_moments_parity(cuda):
  rng = np.random.RandomState(1)
  spec = tensor_spec.TensorSpec((17,), torch.float32)
  n = tensor_normalizer.StreamingTensorNormalizer(spec, device=cuda)
  o = oppo.StreamingNormalizer((17,))
  for i in range(4):
    x = (rng.randn(64, 33, 17) * (1 + i) + i).astype(f32)
    n.update(torch.as_tensor(x, device=cuda))
    o.update(x.reshape(-1, 17))
    cnt, avg, m2, carry = [t.cpu().numpy() for t in n.variables]
    np.testing.assert_allclose(cnt, o.count, rtol=1e-6)
    np.testing.assert_allclose(avg, o.avg, rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(m2, o.m2, rtol=1e-4)
  y = rng.randn(50, 17).astype(f32) * 3
  np.testing.assert_allclose(n.normalize(torch.as_tensor(y, device=cuda)).cpu().numpy(), o.normalize(y),
                             rtol=1e-4, atol=1e-5)
  np.testing.assert_allclose(
      n.normalize(torch.as_tensor(y, device=cuda), clip_value=0, center_mean=False).cpu().numpy(),
      o.normalize(y, clip_value=0, center_mean=False), rtol=1e-4, atol=1e-5)


def _build(cuda, D=17, A=6, hidden=(200, 100), **kw):
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, -1.0, 1.0, 'action')
  actor = actor_distribution_network.ActorDistributionNetwork(obs_spec, act_spec, fc_layer_params=hidden,
                                                              activation_fn='tanh', device=cuda).set_seed(1)
  value = value_network.ValueNetwork(obs_spec, fc_layer_params=hidden, activation_fn='tanh',
                                     device=cuda).set_seed(2)
  agent = ppo_clip_agent.PPOClipAgent(ts.time_step_spec(obs_spec), act_spec,
                                      optimizer=optimizers.Adam(1e-3), actor_net=actor, value_net=value, **kw)
  agent.initialize()
  return agent, actor, value


def _mirror(net):
  layers = []
  for l in net.layers:
    if isinstance(l, L.Dense):
      layers.append(dict(kind='dense', w=l.kernel.cpu().numpy().copy(), b=l.bias.cpu().numpy().copy(),
                         act=l.activation))
  return onn.Sequential(layers)


def _experience(rng, B, T, D, A):
  e = dict(observation=rng.randn(B, T, D).astype(f32), action=np.clip(rng.randn(B, T, A) * .5, -1, 1).astype(f32),
           loc=(rng.randn(B, T, A) * .2).astype(f32), scale=(rng.rand(B, T, A) * .3 + .5).astype(f32),
           reward=rng.rand(B, T).astype(f32), discount=np.ones((B, T), f32),
           step_type=np.ones((B, T), np.int32), next_step_type=np.ones((B, T), np.int32))
  ends = rng.rand(B, T) < 0.05
  e['next_step_type'][ends] = 2
  e['discount'][ends] = 0
  e['step_type'][:, 1:][ends[:, :-1]] = 2        # the step after a LAST is a boundary step
  return e


def _to_traj(cuda, e):
  d = lambda a: torch.as_tensor(a, device=cuda)
  return trajectory.Trajectory(d(e['step_type']), d(e['observation']), d(e['action']),
                               {'dist_params': {'loc': d(e['loc']), 'scale': d(e['scale'])}},
                               d(e['next_step_type']), d(e['reward']), d(e['discount']))


@pytest.mark.parametrize('cfg', [
    dict(num_epochs=1, normalize_rewards=False, normalize_observations=False),
    dict(num_epochs=3, normalize_rewards=True, normalize_observations=False, entropy_regularization=0.01,
         gradient_clipping=0.5, value_clipping=0.2),
])
def test_ppo_clip_agent_train_parity(cuda, cfg):
  rng = np.random.RandomState(7)
  B, T, D, A = 64, 33, 17, 6
  kw = dict(importance_ratio_clipping=0.2, use_gae=True, lambda_value=0.95, discount_factor=0.99)
  kw.update(cfg)
  agent, actor, value = _build(cuda, D, A, hidden=(64, 32), **kw)
  orc = oppo.PPOOracle(_mirror(actor), actor._std.bias.cpu().numpy().copy(), _mirror(value), -np.ones(A, f32),
                       np.ones(A, f32), ooptim.AdamTF(1e-3, eps=1e-7), num_epochs=kw['num_epochs'],
                       clip_eps=0.2, vf_coef=0.5, ent_coef=kw.get('entropy_regularization', 0.0),
                       gamma=0.99, lam=0.95, value_clip=kw.get('value_clipping') or 0.0,
                       gradient_clipping=kw.get('gradient_clipping'),
                       normalize_rewards=kw['normalize_rewards'])
  for it in range(3):
    e = _experience(rng, B, T, D, A)
    infos = orc.train(e)
    got = agent.train(_to_traj(cuda, e))
    want = infos[-1]
    # north-star bound 1e-5 relative on every loss term (the policy-gradient loss is a mean of
    # ratio * advantage terms of both signs, hence an absolute floor as well).
    record_parity('ppo_train_b64_t33', loss_rel=abs(got.loss.item() - want['loss']) / max(abs(want['loss']), 1e-30),
                  pg_abs=abs(got.extra.policy_gradient_loss.item() - want['pg']),
                  pg_rel=abs(got.extra.policy_gradient_loss.item() - want['pg']) / max(abs(want['pg']), 1e-30))
    np.testing.assert_allclose(got.loss.item(), want['loss'], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(got.extra.policy_gradient_loss.item(), want['pg'], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(got.extra.value_estimation_loss.item(), want['ve'], rtol=1e-5)
    np.testing.assert_allclose(got.extra.clip_fraction.item(), want['clip_fraction'], atol=2.0 / (B * T))
  assert int(agent.train_step_counter.item()) == 3 * kw['num_epochs']
  # post-Adam parameters: Adam divides by sqrt(v) + eps, so a 1e-7 gradient difference on a
  # near-zero gradient moves a parameter by up to lr = 1e-3 x O(1); bound = a few % of one step
  for v, w in zip(actor.variables + value.variables, orc.actor.params() + [orc.std_bias] + orc.value.params()):
    record_parity('ppo_train_b64_t33', param_max_abs=float(np.abs(v.cpu().numpy() - w).max()))
    np.testing.assert_allclose(v.cpu().numpy(), w, rtol=2e-3, atol=2e-5)
  agent.check_numerics()


def test_ppo_preprocess_structure(cuda):
  """agents/ppo/ppo_agent_test.py:352-455: returns/advantages are [B,T] with a zero-padded last
  step and equal the agent's own compute_return_and_advantage on the first T-1 steps."""
  rng = np.random.RandomState(3)
  B, T, D, A = 5, 9, 17, 6
  agent, actor, value = _build(cuda, D, A, hidden=(16,), importance_ratio_clipping=0.2, use_gae=True,
                               normalize_rewards=False, normalize_observations=False)
  e = _experience(rng, B, T, D, A)
  vp, ret, adv = agent._preprocess(_to_traj(cuda, e))
  assert tuple(ret.shape) == tuple(adv.shape) == (B, T)
  assert float(ret[:, -1].abs().sum()) == 0 and float(adv[:, -1].abs().sum()) == 0
  wret, wadv = oppo.compute_return_and_advantage(e['reward'][:, :-1], e['discount'][:, :-1],
                                                 e['next_step_type'][:, :-1], vp.cpu().numpy(), 0.99, 0.95)
  np.testing.assert_allclose(ret[:, :-1].cpu().numpy(), wret, rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(adv[:, :-1].cpu().numpy(), wadv, rtol=1e-5, atol=1e-5)


def test_ppo_collect_policy(cuda):
  agent, actor, value = _build(cuda, 17, 6, hidden=(16,), importance_ratio_clipping=0.2, use_gae=True,
                               normalize_observations=False)
  obs = torch.randn(4096, 17, device=cuda)
  step = agent.collect_policy.action(ts.restart(obs, batch_size=4096))
  loc, scale = step.info['dist_params']['loc'], step.info['dist_params']['scale']
  assert tuple(step.action.shape) == (4096, 6)
  z = ((step.action - loc) / scale).cpu().numpy()
  assert abs(z.mean()) < 0.02 and abs(z.std() - 1) < 0.02          # N(0,1) draws
  np.testing.assert_allclose(scale.cpu().numpy(), np.log(2.0), rtol=1e-5)   # softplus(0)
  step2 = agent.collect_policy.action(ts.restart(obs, batch_size=4096))
  assert not torch.equal(step.action, step2.action)
  greedy = agent.policy.action(ts.restart(obs, batch_size=4096))
  assert torch.equal(greedy.action, loc)


# ---- KL penalty (ppo_agent.py:1514-1690) ---------------------------------------------------------
def _kl_agent(cuda, **kw):
  from agents_b200.agents.ppo import ppo_agent
  obs_spec = tensor_spec.TensorSpec((2,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((1,), torch.float32, -1.0, 1.0, 'action')
  actor = actor_distribution_network.ActorDistributionNetwork(obs_spec, act_spec, fc_layer_params=None,
                                                              device=cuda).set_seed(1)
  value = value_network.ValueNetwork(obs_spec, fc_layer_params=None, device=cuda).set_seed(2)
  agent = ppo_agent.PPOAgent(ts.time_step_spec(obs_spec), act_spec, optimizers.Adam(1e-3), actor_net=actor,
                             value_net=value, use_gae=True, **kw)
  agent.initialize()
  return agent


def test_kl_reference_goldens_through_the_agent(cuda):
  """ppo_agent_test.py:1045-1078 (kl_cutoff_loss = coef * 0.24^2), :1080-1124 (adaptive loss moves
  with beta), :1126-1164 (beta 1.0 -> 1.0 -> 1.5 -> 1.0)."""
  kl = torch.tensor([[1.5, -0.5, 6.5, -1.5, -2.3]], device=cuda)
  for coef in (0.0, 30.0):
    agent = _kl_agent(cuda, kl_cutoff_factor=5.0, adaptive_kl_target=0.1, kl_cutoff_coef=coef)
    np.testing.assert_allclose(agent.kl_cutoff_loss(kl).item(), coef * 0.24 ** 2, rtol=1e-5)
  agent = _kl_agent(cuda, initial_adaptive_kl_beta=1.0, adaptive_kl_target=10.0, adaptive_kl_tolerance=0.5)
  t = lambda v: torch.tensor([v], device=cuda)
  assert agent.adaptive_kl_loss(t(10.0)).item() == agent.adaptive_kl_loss(t(10.0)).item()
  l1 = agent.adaptive_kl_loss(t(1.0)).item()
  agent.update_adaptive_kl_beta(t(1.0))
  assert l1 > agent.adaptive_kl_loss(t(1.0)).item()
  l1 = agent.adaptive_kl_loss(t(100.0)).item()
  agent.update_adaptive_kl_beta(t(100.0))
  assert l1 < agent.adaptive_kl_loss(t(100.0)).item()
  agent = _kl_agent(cuda, initial_adaptive_kl_beta=1.0, adaptive_kl_target=10.0, adaptive_kl_tolerance=0.5)
  assert agent.update_adaptive_kl_beta(t(10.0)).item() == 1.0
  assert agent.update_adaptive_kl_beta(t(100.0)).item() == 1.5
  np.testing.assert_allclose(agent.update_adaptive_kl_beta(t(1.0)).item(), 1.0, rtol=1e-6)
  # PPOAgent with the reference's default KL settings constructs (it used to raise)
  _kl_agent(cuda)


def test_kl_kernel_parity(cuda):
  rng = np.random.RandomState(4)
  N, A = 777, 6
  la, lb = (rng.randn(N, A) * .4).astype(f32), (rng.randn(N, A) * .4).astype(f32)
  sa, sb = (rng.rand(N, A) * .5 + .4).astype(f32), (rng.rand(N, A) * .5 + .4).astype(f32)
  w = (rng.rand(N) > .3).astype(f32)
  d = lambda a: torch.as_tensor(a, device=cuda)
  out_kl = torch.empty(N, device=cuda)
  s = torch.empty(1, device=cuda)
  ws, nb = workspace.get(cuda)
  t = [d(x) for x in (lb, sb, la, sa, w)]      # keep the device tensors alive across the launch
  _lib.call('b200rl_ppo_kl', _lib.ptr(t[0]), _lib.ptr(t[1]), A, _lib.ptr(t[2]), _lib.ptr(t[3]), A,
            _lib.ptr(t[4]), N, A, 1.0 / N, _lib.ptr(out_kl), _lib.ptr(s), _lib.ptr(ws), nb, _lib.stream())
  want = oppo.normal_kl(la, sa, lb, sb) * w
  np.testing.assert_allclose(out_kl.cpu().numpy(), want, rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(s.item(), want.mean(dtype=f32), rtol=1e-5)


@pytest.mark.parametrize('cfg', [
    dict(kl_cutoff_factor=2.0, kl_cutoff_coef=1000.0, initial_adaptive_kl_beta=1.0, adaptive_kl_target=0.01,
         adaptive_kl_tolerance=0.3, importance_ratio_clipping=0.0),          # reference defaults (:140-144)
    dict(kl_cutoff_factor=0.0, kl_cutoff_coef=0.0, initial_adaptive_kl_beta=0.7, adaptive_kl_target=0.05,
         adaptive_kl_tolerance=0.5, importance_ratio_clipping=0.2),
])
def test_ppo_agent_kl_train_parity(cuda, cfg):
  """PPOAgent (KL-penalty form) with BOTH normalisers on, 3 train calls x 2 epochs vs the oracle:
  losses, kl_penalty_loss, adaptive beta and parameters."""
  from agents_b200.agents.ppo import ppo_agent
  rng = np.random.RandomState(9)
  B, T, D, A = 64, 33, 17, 6
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, -1.0, 1.0, 'action')
  actor = actor_distribution_network.ActorDistributionNetwork(obs_spec, act_spec, fc_layer_params=(64, 32),
                                                              activation_fn='tanh', device=cuda).set_seed(1)
  value = value_network.ValueNetwork(obs_spec, fc_layer_params=(64, 32), activation_fn='tanh',
                                     device=cuda).set_seed(2)
  agent = ppo_agent.PPOAgent(ts.time_step_spec(obs_spec), act_spec, optimizers.Adam(1e-3), actor_net=actor,
                             value_net=value, use_gae=True, num_epochs=2, normalize_rewards=True,
                             normalize_observations=True, **cfg)
  agent.initialize()
  orc = oppo.PPOOracle(_mirror(actor), actor._std.bias.cpu().numpy().copy(), _mirror(value), -np.ones(A, f32),
                       np.ones(A, f32), ooptim.AdamTF(1e-3, eps=1e-7), num_epochs=2,
                       clip_eps=cfg['importance_ratio_clipping'], vf_coef=0.5, gamma=0.99, lam=0.95,
                       normalize_rewards=True, normalize_observations=True, obs_dim=D,
                       kl_cutoff_factor=cfg['kl_cutoff_factor'], kl_cutoff_coef=cfg['kl_cutoff_coef'],
                       initial_adaptive_kl_beta=cfg['initial_adaptive_kl_beta'],
                       adaptive_kl_target=cfg['adaptive_kl_target'],
                       adaptive_kl_tolerance=cfg['adaptive_kl_tolerance'])
  for it in range(3):
    e = _experience(rng, B, T, D, A)
    want = orc.train(e)[-1]
    got = agent.train(_to_traj(cuda, e))
    np.testing.assert_allclose(got.loss.item(), want['loss'], rtol=2e-5, atol=1e-7)
    np.testing.assert_allclose(got.extra.kl_penalty_loss.item(), want['kl'], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(got.extra.value_estimation_loss.item(), want['ve'], rtol=2e-5)
    np.testing.assert_allclose(agent._adaptive_kl_beta.item(), orc.beta, rtol=1e-6)
  # post-Adam parameters: Adam divides by sqrt(v) + eps, so a 1e-7 gradient difference on a
  # near-zero gradient moves a parameter by up to lr = 1e-3 x O(1); bound = a few % of one step
  for v, w in zip(actor.variables + value.variables, orc.actor.params() + [orc.std_bias] + orc.value.params()):
    record_parity('ppo_train_b64_t33', param_max_abs=float(np.abs(v.cpu().numpy() - w).max()))
    np.testing.assert_allclose(v.cpu().numpy(), w, rtol=2e-3, atol=2e-5)
  agent.check_numerics()
