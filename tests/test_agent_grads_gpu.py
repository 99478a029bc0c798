"""Each agent's whole pre-optimizer gradient against float64 autograd.

Every agent-level parity test elsewhere compares parameters after an Adam or RMSProp step, and
both divide by a running gradient magnitude: a constant factor in a gradient (a wrong
1/global_batch, a missing loss weight or action half-range) leaves the update almost unchanged.
Here the agents train with a RecordingOptimizer that keeps a copy of every gradient it is handed
and leaves the parameters alone.  The recorded gradients are compared, per parameter tensor, with
float64 autograd of the loss restated in tests/grad_refs.py on float64 copies of the networks.

Bounds (relative L2 error and max error over max|g_ref|, per tensor) are at least 4x the largest
error measured on an H100 80GB HBM3 at a 400 W power limit; record_parity keeps the measured
values.  The PPO rows run with both the default tensor-core GEMMs and the FFMA GEMMs.
"""
import os

import numpy as np
import pytest
import torch

import grad_refs as R
from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.agents.dqn import dqn_agent
from agents_b200.agents.ppo import ppo_agent
from agents_b200.agents.ppo import ppo_clip_agent
from agents_b200.agents.sac import sac_agent
from agents_b200.networks import actor_distribution_network
from agents_b200.networks import critic_network
from agents_b200.networks import layers as L
from agents_b200.networks import sequential
from agents_b200.networks import tanh_normal_projection_network as tnp
from agents_b200.networks import value_network
from agents_b200.specs import tensor_spec
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory
from conftest import record_parity
from oracle import nn as onn
from oracle import ppo as oppo
from oracle import ppo_discrete as oppod

pytestmark = pytest.mark.gpu
f32 = np.float32

TOL_REL_L2 = 1e-4
TOL_MAX = 1e-4
TOL_SCALE = 1e-5      # recorded global-norm clip scale against clip / max(‖g_ref‖, clip)
TOL_EPOCH = 1e-5      # epoch 2 against epoch 1 of one train call (tensor-core GEMMs)
AMIN = np.array([-2.0, 0.0, -0.5, 0.1, -7.0], f32)
AMAX = np.array([1.0, 10.0, 0.5, 0.7, -3.0], f32)


class RecordingOptimizer(optimizers.Optimizer):
  """Keeps a copy of every gradient (and global-norm clip scale) it is handed; the parameters do
  not move, so every later step of a train call sees the networks the reference sees."""

  def __init__(self):
    super().__init__()
    self.calls = []

  def apply_flat(self, params, grads, grad_scale=None):
    self.calls.append(dict(base=grads.data_ptr(), grads=grads.clone(),
                           grad_scale=None if grad_scale is None else grad_scale.clone()))


def _grad_views(net):
  """The network's gradient views in the order of net.variables."""
  out = []
  for l in net.layers:
    if getattr(l, 'has_params', False):
      out += [g for g in (getattr(l, 'd_kernel', None), getattr(l, 'd_bias', None)) if g is not None]
  return out


def _recorded(call, views):
  """The recorded flat gradient cut into the tensors `views` occupy in the live buffer."""
  out = []
  for v in views:
    off = (v.data_ptr() - call['base']) // 4
    assert 0 <= off and off + v.numel() <= call['grads'].numel()
    out.append(call['grads'][off:off + v.numel()].view(v.shape))
  return out


def _layers64(net):
  """float64 leaf copies [(kernel, bias, activation)] of the network's Dense layers."""
  return [(R.t64(l.kernel).requires_grad_(), R.t64(l.bias).requires_grad_(), l.activation)
          for l in net.layers if isinstance(l, L.Dense)]


def _params(layers):
  return [p for w, b, _ in layers for p in (w, b)]


def _compare(family, names, got, ref, rel_l2=TOL_REL_L2, rel_max=TOL_MAX):
  assert len(got) == len(ref) == len(names)
  for name, g, r in zip(names, got, ref):
    e = R.grad_errors(g, r)
    record_parity(family, **{name + '_rel_l2': e[0], name + '_max': e[1]})
  for name, g, r in zip(names, got, ref):
    R.assert_grad_close(f'{family}/{name}', g, r, rel_l2, rel_max)


def _names(prefix, layers, extra=()):
  out = []
  for i in range(len(layers)):
    out += [f'{prefix}{i}_kernel', f'{prefix}{i}_bias']
  return out + list(extra)


# ---- SAC ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('use_log_alpha', [True, False])
def test_sac_agent_gradients(cuda, use_log_alpha):
  rng = np.random.RandomState(21 + use_log_alpha)
  D, A, B = 11, 5, 300
  gamma, reward_scale, lw_actor, lw_critic, lw_alpha = 0.93, 2.5, 0.7, 1.3, 0.6
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, AMIN, AMAX, 'action')
  actor = tnp.TanhNormalActorNetwork(obs_spec, act_spec, fc_layer_params=(64, 64), device=cuda).set_seed(1)
  critic = critic_network.CriticNetwork((obs_spec, act_spec), joint_fc_layer_params=(64, 64),
                                        device=cuda).set_seed(2)
  opt_actor, opt_critic, opt_alpha = RecordingOptimizer(), RecordingOptimizer(), RecordingOptimizer()
  agent = sac_agent.SacAgent(
      ts.time_step_spec(obs_spec), act_spec, critic_network=critic, actor_network=actor,
      actor_optimizer=opt_actor, critic_optimizer=opt_critic, alpha_optimizer=opt_alpha,
      actor_loss_weight=lw_actor, critic_loss_weight=lw_critic, alpha_loss_weight=lw_alpha,
      target_update_tau=0.005, gamma=gamma, reward_scale_factor=reward_scale, initial_log_alpha=0.7,
      use_log_alpha_in_alpha_loss=use_log_alpha)
  agent.initialize()
  c1, c2 = agent._critic_network_1, agent._critic_network_2
  # float64 copies before train(): the target update moves the target critics at its end
  A64, C1, C2 = _layers64(actor), _layers64(c1), _layers64(c2)
  T1 = _layers64(agent._target_critic_network_1)
  T2 = _layers64(agent._target_critic_network_2)
  log_alpha = float(agent.log_alpha.item())
  obs = rng.randn(B, 2, D).astype(f32)
  action = (AMIN + (AMAX - AMIN) * rng.rand(B, 2, A)).astype(f32)
  reward, discount = rng.randn(B, 2).astype(f32), (rng.rand(B, 2) > 0.1).astype(f32)
  weights = (rng.rand(B) * 2).astype(f32)
  weights[rng.rand(B) < 0.2] = 0.0
  noise = [(rng.randn(B, A) * 1.5).astype(f32) for _ in range(3)]
  d = lambda a: torch.as_tensor(a, device=cuda)
  ones = torch.ones(B, 2, dtype=torch.int32, device=cuda)
  traj = trajectory.Trajectory(ones, d(obs), d(action), (), ones, d(reward), d(discount))
  agent.train(traj, weights=d(weights), noise=noise)
  agent.check_numerics()
  assert len(opt_critic.calls) == len(opt_actor.calls) == len(opt_alpha.calls) == 1

  lo, hi = R.t64(AMIN), R.t64(AMAX)
  o0, o1 = R.t64(obs[:, 0]), R.t64(obs[:, 1])
  w = R.t64(weights)
  eps_next, eps_actor, eps_alpha = (R.t64(n) for n in noise)
  # critic step (sac_agent.py:341-362)
  with torch.no_grad():
    a2, _, logp2 = R.sac_sample(R.mlp(A64, o1), eps_next, lo, hi)
    x2 = torch.cat([o1, a2], dim=1)
    tq1, tq2 = R.mlp(T1, x2)[:, 0], R.mlp(T2, x2)[:, 0]
  x = torch.cat([o0, R.t64(action[:, 0])], dim=1)
  q1, q2 = R.mlp(C1, x)[:, 0], R.mlp(C2, x)[:, 0]
  closs, _ = R.sac_critic_loss(q1, q2, tq1, tq2, logp2, R.t64(reward[:, 0]), R.t64(discount[:, 0]),
                               log_alpha, gamma, reward_scale, lw_critic, float(B), w)
  g_critic = torch.autograd.grad(closs, _params(C1) + _params(C2))
  got = _recorded(opt_critic.calls[0], _grad_views(c1) + _grad_views(c2))
  _compare('agent_grads_sac_critic', _names('c1_', C1) + _names('c2_', C2), got, g_critic)
  # actor step (:364-377); the critics have not moved
  a, _, logp = R.sac_sample(R.mlp(A64, o0), eps_actor, lo, hi)
  xa = torch.cat([o0, a], dim=1)
  aloss = R.sac_actor_loss(R.mlp(C1, xa)[:, 0], R.mlp(C2, xa)[:, 0], logp, log_alpha, lw_actor, float(B), w)
  g_actor = torch.autograd.grad(aloss, _params(A64))
  got = _recorded(opt_actor.calls[0], _grad_views(actor))
  _compare('agent_grads_sac_actor', _names('actor', A64), got, g_actor)
  # alpha step (:379-390); the actor has not moved
  with torch.no_grad():
    _, _, logp3 = R.sac_sample(R.mlp(A64, o0), eps_alpha, lo, hi)
  la = torch.tensor(log_alpha, dtype=R.F64, requires_grad=True)
  alloss = R.sac_alpha_loss(logp3, la, -A / 2.0, use_log_alpha, lw_alpha, float(B), w)
  (g_la,) = torch.autograd.grad(alloss, la)
  _compare('agent_grads_sac_alpha', ['log_alpha'], [opt_alpha.calls[0]['grads'][:1]], [g_la.reshape(1)])


# ---- PPO ------------------------------------------------------------------------------------------
PPO_KW = dict(importance_ratio_clipping=0.2, lambda_value=0.95, discount_factor=0.99,
              entropy_regularization=0.01, policy_l2_reg=0.01, value_function_l2_reg=0.02,
              value_pred_loss_coef=0.5, num_epochs=2, use_gae=True, normalize_rewards=False,
              normalize_observations=False, gradient_clipping=0.05, value_clipping=0.2)
KL_KW = dict(kl_cutoff_factor=2.0, kl_cutoff_coef=50.0, initial_adaptive_kl_beta=0.7,
             adaptive_kl_target=0.05, adaptive_kl_tolerance=0.3)


def _mirror(net):
  return onn.Sequential([dict(kind='dense', w=l.kernel.cpu().numpy().copy(), b=l.bias.cpu().numpy().copy(),
                              act=l.activation) for l in net.layers if isinstance(l, L.Dense)])


def _episodes(rng, B, T):
  step_type, next_step_type = np.ones((B, T), np.int32), np.ones((B, T), np.int32)
  discount = np.ones((B, T), f32)
  ends = rng.rand(B, T) < 0.05
  next_step_type[ends], discount[ends] = 2, 0
  step_type[:, 1:][ends[:, :-1]] = 2          # the step after a LAST is a boundary step
  return step_type, next_step_type, discount


def _ppo_targets(value, e, old_logp):
  """Advantages, returns, old log-probs and weights as oracle.ppo computes them."""
  orc = oppo.PPOOracle(None, np.zeros(1, f32), _mirror(value), np.zeros(1, f32), np.ones(1, f32), None,
                       gamma=PPO_KW['discount_factor'], lam=PPO_KW['lambda_value'])
  vp, ret, adv = orc.preprocess(e)
  w = oppo.make_trajectory_mask(e['step_type'], ret, adv) * e['weights']
  return dict(vp=vp.reshape(-1), ret=ret.reshape(-1), adv_n=oppo.normalize_advantages(adv).reshape(-1),
              old_logp=old_logp.reshape(-1), w=w.reshape(-1).astype(f32))


@pytest.fixture(params=['tf32x3', 'ffma'])
def gemm_mode(request):
  """The default 3xTF32 tensor-core GEMMs, and the FP32 FFMA GEMMs (b200rl_set_gemm_mode(0)),
  whose deterministic split-K makes weight gradients bit-reproducible."""
  if request.param == 'ffma':
    _lib.call('b200rl_set_gemm_mode', 0)
  try:
    yield request.param
  finally:
    _lib.call('b200rl_set_gemm_mode', int(os.environ.get('B200RL_GEMM_MODE', '1')))


def _check_ppo(family, agent, opt, nets, ref_params, loss, clip, gemm_mode):
  actor, value = nets
  assert len(opt.calls) == 2
  # The parameters do not move, so both epochs must hand the optimizer the same gradient.  With
  # the FFMA GEMMs that holds bit for bit; the tensor-core weight-gradient GEMMs add their split-K
  # partials with floating-point atomics (DESIGN.md §4), so there the summation order may differ.
  g0, g1 = opt.calls[0]['grads'], opt.calls[1]['grads']
  if gemm_mode == 'ffma':
    assert torch.equal(g0, g1), 'the two epochs differ'
    assert torch.equal(opt.calls[0]['grad_scale'], opt.calls[1]['grad_scale'])
  else:
    e = R.grad_errors(g1, g0)
    record_parity(family, epoch_rel_l2=e[0], epoch_max=e[1])
    R.assert_grad_close(f'{family}/epoch 2 vs epoch 1', g1, g0, TOL_EPOCH, TOL_EPOCH)
  family = f'{family}_{gemm_mode}'
  g_ref = torch.autograd.grad(loss, ref_params)
  views = _grad_views(actor) + _grad_views(value)
  names = ([f'actor_{i}' for i in range(len(_grad_views(actor)))] +
           [f'value_{i}' for i in range(len(_grad_views(value)))])
  _compare(family, names, _recorded(opt.calls[0], views), g_ref)
  norm = float(torch.sqrt(sum((g * g).sum() for g in g_ref)))
  scale_ref = clip / max(norm, clip)
  assert scale_ref < 0.5, 'global-norm clipping does not engage'
  scale = float(opt.calls[0]['grad_scale'][0])
  err = abs(scale - scale_ref) / scale_ref
  record_parity(family, grad_scale=err)
  assert err <= TOL_SCALE, (scale, scale_ref)
  agent.check_numerics()


@pytest.mark.parametrize('kind', ['clip', 'kl'])
def test_ppo_continuous_gradients(cuda, kind, gemm_mode):
  rng = np.random.RandomState(31 + (kind == 'kl'))
  B, T, D, A = 24, 17, 13, 5
  N = B * T
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, AMIN, AMAX, 'action')
  actor = actor_distribution_network.ActorDistributionNetwork(
      obs_spec, act_spec, fc_layer_params=(64, 32), activation_fn='tanh', device=cuda).set_seed(1)
  value = value_network.ValueNetwork(obs_spec, fc_layer_params=(64, 32), activation_fn='tanh',
                                     device=cuda).set_seed(2)
  opt = RecordingOptimizer()
  if kind == 'kl':
    agent = ppo_agent.PPOAgent(ts.time_step_spec(obs_spec), act_spec, opt, actor_net=actor, value_net=value,
                               **PPO_KW, **KL_KW)
  else:
    agent = ppo_clip_agent.PPOClipAgent(ts.time_step_spec(obs_spec), act_spec, opt, actor_net=actor,
                                        value_net=value, **PPO_KW)
  agent.initialize()
  with torch.no_grad():   # a non-zero std bias, so softplus / sigmoid are not at 0
    actor._std.bias.copy_(torch.as_tensor(rng.randn(A) * 0.5, dtype=torch.float32))
  obs = rng.randn(B, T, D).astype(f32)
  loc, scale = actor.distribution_params(torch.as_tensor(obs.reshape(N, D), device=cuda))
  loc, scale = loc.cpu().numpy(), scale.cpu().numpy()
  old_loc = (loc + 0.1 * (AMAX - AMIN) / 2 * rng.randn(N, A)).astype(f32)
  old_scale = (scale * np.exp(0.2 * rng.randn(N, A))).astype(f32)
  action = np.clip(old_loc + old_scale * rng.randn(N, A), AMIN, AMAX).astype(f32)
  step_type, next_step_type, discount = _episodes(rng, B, T)
  weights = (rng.rand(B, T) * 2).astype(f32)
  weights[rng.rand(B, T) < 0.2] = 0.0
  e = dict(observation=obs, reward=rng.rand(B, T).astype(f32), discount=discount, step_type=step_type,
           next_step_type=next_step_type, weights=weights)
  d = lambda a: torch.as_tensor(a, device=cuda)
  traj = trajectory.Trajectory(
      d(step_type), d(obs), d(action.reshape(B, T, A)),
      {'dist_params': {'loc': d(old_loc.reshape(B, T, A)), 'scale': d(old_scale.reshape(B, T, A))}},
      d(next_step_type), d(e['reward']), d(discount))
  agent.train(traj, weights=d(weights))

  p = _ppo_targets(value, e, oppo.normal_log_prob(old_loc, old_scale, action))
  A64, V64 = _layers64(actor), _layers64(value)
  std64 = R.t64(actor._std.bias).requires_grad_()
  o64 = R.t64(obs.reshape(N, D))
  loc64, scale64 = R.normal_projection(R.mlp(A64, o64), std64, R.t64(AMIN), R.t64(AMAX))
  v = R.mlp(V64, o64)[:, 0]
  w = R.t64(p['w'])
  loss = R.ppo_loss(R.normal_log_prob(loc64, scale64, R.t64(action)), R.normal_entropy(scale64),
                    R.t64(p['old_logp']), R.t64(p['adv_n']), R.t64(p['ret']), v, R.t64(p['vp']), w, float(N),
                    PPO_KW['importance_ratio_clipping'], PPO_KW['value_clipping'],
                    PPO_KW['value_pred_loss_coef'], PPO_KW['entropy_regularization'])
  if kind == 'kl':
    kl = R.normal_kl(R.t64(old_loc), R.t64(old_scale), loc64, scale64)
    loss = loss + R.kl_penalty(kl, w, float(N), KL_KW['kl_cutoff_factor'], KL_KW['adaptive_kl_target'],
                               KL_KW['kl_cutoff_coef'], KL_KW['initial_adaptive_kl_beta'])
  loss = (loss + R.l2_loss([k for k, _, _ in A64], PPO_KW['policy_l2_reg'])
          + R.l2_loss([k for k, _, _ in V64], PPO_KW['value_function_l2_reg']))
  _check_ppo(f'agent_grads_ppo_{kind}', agent, opt, (actor, value),
             _params(A64) + [std64] + _params(V64), loss, PPO_KW['gradient_clipping'], gemm_mode)


def test_ppo_discrete_gradients(cuda, gemm_mode):
  rng = np.random.RandomState(41)
  B, T, D, A = 24, 17, 13, 7
  N = B * T
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int64, 0, A - 1, 'action')
  actor = actor_distribution_network.ActorDistributionNetwork(
      obs_spec, act_spec, fc_layer_params=(64, 32), activation_fn='tanh', device=cuda).set_seed(3)
  value = value_network.ValueNetwork(obs_spec, fc_layer_params=(64, 32), activation_fn='tanh',
                                     device=cuda).set_seed(4)
  opt = RecordingOptimizer()
  agent = ppo_agent.PPOAgent(ts.time_step_spec(obs_spec), act_spec, opt, actor_net=actor, value_net=value,
                             **PPO_KW, **KL_KW)
  agent.initialize()
  obs = rng.randn(B, T, D).astype(f32)
  logits = actor.distribution_params(torch.as_tensor(obs.reshape(N, D), device=cuda)).cpu().numpy()
  old_logits = (logits + 0.3 * rng.randn(N, A)).astype(f32)
  action = rng.randint(0, A, N).astype(np.int64)
  step_type, next_step_type, discount = _episodes(rng, B, T)
  weights = (rng.rand(B, T) * 2).astype(f32)
  weights[rng.rand(B, T) < 0.2] = 0.0
  e = dict(observation=obs, reward=rng.rand(B, T).astype(f32), discount=discount, step_type=step_type,
           next_step_type=next_step_type, weights=weights)
  d = lambda a: torch.as_tensor(a, device=cuda)
  traj = trajectory.Trajectory(d(step_type), d(obs), d(action.reshape(B, T)),
                               {'dist_params': {'logits': d(old_logits.reshape(B, T, A))}},
                               d(next_step_type), d(e['reward']), d(discount))
  agent.train(traj, weights=d(weights))

  p = _ppo_targets(value, e, oppod.categorical_log_prob(old_logits, action))
  A64, V64 = _layers64(actor), _layers64(value)
  o64 = R.t64(obs.reshape(N, D))
  lg = R.mlp(A64, o64)
  v = R.mlp(V64, o64)[:, 0]
  w = R.t64(p['w'])
  loss = R.ppo_loss(R.categorical_log_prob(lg, torch.as_tensor(action)), R.categorical_entropy(lg),
                    R.t64(p['old_logp']), R.t64(p['adv_n']), R.t64(p['ret']), v, R.t64(p['vp']), w, float(N),
                    PPO_KW['importance_ratio_clipping'], PPO_KW['value_clipping'],
                    PPO_KW['value_pred_loss_coef'], PPO_KW['entropy_regularization'])
  kl = R.categorical_kl(R.t64(old_logits), lg)
  loss = loss + R.kl_penalty(kl, w, float(N), KL_KW['kl_cutoff_factor'], KL_KW['adaptive_kl_target'],
                             KL_KW['kl_cutoff_coef'], KL_KW['initial_adaptive_kl_beta'])
  loss = (loss + R.l2_loss([k for k, _, _ in A64], PPO_KW['policy_l2_reg'])
          + R.l2_loss([k for k, _, _ in V64], PPO_KW['value_function_l2_reg']))
  _check_ppo('agent_grads_ppo_discrete', agent, opt, (actor, value), _params(A64) + _params(V64), loss,
             PPO_KW['gradient_clipping'], gemm_mode)


# ---- DQN ------------------------------------------------------------------------------------------
def test_dqn_agent_gradients(cuda):
  rng = np.random.RandomState(51)
  B, D, A, n = 300, 9, 4, 2
  T = n + 1
  gamma, reward_scale, clip = 0.97, 1.7, 0.1
  l2 = (0.01, 0.02, 0.005)
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, A - 1, 'action')
  net = sequential.Sequential([L.Dense(64, activation='relu', kernel_regularizer_l2=l2[0]),
                               L.Dense(32, activation='relu', kernel_regularizer_l2=l2[1]),
                               L.Dense(A, kernel_regularizer_l2=l2[2])],
                              input_spec=obs_spec, device=cuda).set_seed(5)
  opt = RecordingOptimizer()
  agent = dqn_agent.DqnAgent(ts.time_step_spec(obs_spec), act_spec, q_network=net, optimizer=opt,
                             n_step_update=n, gamma=gamma, reward_scale_factor=reward_scale,
                             gradient_clipping=clip, target_update_tau=1.0, target_update_period=1)
  agent.initialize()
  Q64, TQ64 = _layers64(net), _layers64(agent._target_q_network)
  obs = rng.randn(B, T, D).astype(f32)
  step_type = rng.randint(0, 3, (B, T)).astype(np.int32)
  action = rng.randint(0, A, (B, T)).astype(np.int32)
  reward, discount = rng.randn(B, T).astype(f32), (rng.rand(B, T) > 0.1).astype(f32)
  weights = (rng.rand(B) * 2).astype(f32)
  weights[rng.rand(B) < 0.2] = 0.0
  d = lambda a: torch.as_tensor(a, device=cuda)
  traj = trajectory.Trajectory(d(step_type), d(obs), d(action), (), d(np.ones((B, T), np.int32)),
                               d(reward), d(discount))
  agent.train(traj, weights=d(weights))
  agent.check_numerics()
  assert len(opt.calls) == 1

  q = R.mlp(Q64, R.t64(obs[:, 0]))
  qsa = q.gather(1, torch.as_tensor(action[:, 0], dtype=torch.int64).reshape(-1, 1))[:, 0]
  with torch.no_grad():
    nt = R.mlp(TQ64, R.t64(obs[:, T - 1]))
    nq = nt.gather(1, nt.argmax(dim=1, keepdim=True))[:, 0]
    target = R.n_step_targets(R.t64(reward), R.t64(discount), nq, gamma, reward_scale)
  valid = R.t64(step_type[:, 0] != 2)
  loss = R.aggregate(valid * R.huber(target - qsa), R.t64(weights), float(B))
  for (k, _, _), c in zip(Q64, l2):
    loss = loss + R.l2_loss([k], c)
  g_raw = torch.autograd.grad(loss, _params(Q64))
  # eager_utils.clip_gradient_norms: tf.clip_by_norm per variable
  g_ref = [R.clip_by_norm(g, clip) for g in g_raw]
  clipped = [float(g.norm()) > clip for g in g_raw]
  assert any(clipped) and not all(clipped), 'per-variable clipping should engage for some variables only'
  _compare('agent_grads_dqn', _names('q', Q64), _recorded(opt.calls[0], _grad_views(net)), g_ref)
