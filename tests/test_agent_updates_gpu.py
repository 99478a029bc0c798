"""Each agent's real update step against update_refs.py: the optimizer step with the clip scale
it is handed, the target-network update, the Periodically counters, train_step_counter and the
optimizers' iterations.

The agents train with their real optimizers wrapped in a CheckedOptimizer.  On every apply_flat
it keeps copies of the parameters, the gradient, the slots, the step counter and *grad_scale,
runs the real update, and keeps copies of the new state.  After each train() every recorded step
is compared with the reference stepped from the recorded pre-step state.  The gradients
themselves are checked in test_agent_grads_gpu.py; here they are only inputs.
"""
import numpy as np
import pytest
import torch

import update_refs as U
from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.agents.dqn import dqn_agent
from agents_b200.agents.ppo import ppo_agent
from agents_b200.agents.ppo import ppo_clip_agent
from agents_b200.agents.sac import sac_agent
from agents_b200.networks import actor_distribution_network
from agents_b200.networks import critic_network
from agents_b200.networks import layers as L
from agents_b200.networks import q_network
from agents_b200.networks import tanh_normal_projection_network as tnp
from agents_b200.networks import value_network
from agents_b200.specs import tensor_spec
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory
from conftest import record_parity
from test_agent_grads_gpu import AMAX, AMIN, KL_KW, PPO_KW, _episodes

pytestmark = pytest.mark.gpu
f32 = np.float32
TRAIN_CALLS = 3


class CheckedOptimizer(optimizers.Optimizer):
  """Runs `inner`'s real update and keeps device copies of the state before and after it."""

  def __init__(self, inner):
    super().__init__()
    self.inner = inner
    self.records = []
    self.steps = 0

  def iterations(self, params):
    return self.inner.iterations(params)

  def variables(self):
    return self.inner.variables()

  def apply_flat(self, params, grads, grad_scale=None):
    slots = self.inner._get_slots(params)
    pre = dict(p=params.clone(), g=grads.clone(), scale=None if grad_scale is None else grad_scale.clone(),
               **{k: s.clone() for k, s in slots.items()})
    self.inner.apply_flat(params, grads, grad_scale)
    post = dict(p=params.clone(), **{k: s.clone() for k, s in slots.items()})
    self.records.append((pre, post))
    self.steps += 1

  def check(self, family):
    """Compares every recorded step with the reference and forgets them."""
    opt = self.inner
    for i, (pre, post) in enumerate(self.records):
      scale = None if pre['scale'] is None else float(pre['scale'][0])
      n = lambda k, d: d[k].cpu().numpy()
      where = f'{family} step {i + 1}'
      if isinstance(opt, optimizers.AdamOptimizer):
        step = int(pre['step'][0])
        ref = U.adam(n('p', pre), n('g', pre), n('m', pre), n('v', pre), step, opt.learning_rate,
                     opt.beta1, opt.beta2, opt.epsilon, scale=scale)
        slots = {k: U.slot_errors(n(k, post), ref[k]) for k in ('m', 'v')}
        assert post['step'].cpu().tolist() == [ref['step'], 0], where
      else:
        ref = U.rmsprop(n('p', pre), n('g', pre), n('ms', pre), n('mg', pre), n('mom', pre),
                        opt.learning_rate, opt.decay, opt.momentum, opt.epsilon, opt.centered,
                        scale=scale)
        slots = {k: U.slot_errors(n(k, post), ref[k]) for k in (('ms', 'mg') if opt.centered else ('ms',))}
        mraw, mratio = U.cond_error(n('mom', post), ref['mom'], ref['cond'])
        record_parity(family, mom=mraw, mom_over_bound=mratio)
        assert mratio <= 1.0, f'{where}: mom error {mraw:.3g}'
      raw, ratio = U.update_error(n('p', post), n('p', pre), ref['u'], np.asarray(ref['cond']))
      record_parity(family, update=raw, update_over_bound=ratio,
                    **{k: max(e) for k, e in slots.items()})
      assert ratio <= 1.0, f'{where}: update error {raw:.3g}'
      for k, e in slots.items():
        assert max(e) <= U.TOL_SLOT, f'{where}: slot {k} {e}'
    self.records = []


def _check_target(family, target, online, before, tau, gate):
  """The target after train() against the Periodically-gated blend of `before` (the target at
  the start of train()) with the online parameters after their optimizer step."""
  ref, fired = U.polyak_step(gate, before, online.cpu().numpy(), tau)
  got = target.cpu().numpy()
  if not fired:
    assert np.array_equal(got.view(np.int32), before.view(np.int32)), f'{family}: target moved'
  elif tau == 1.0:
    assert np.array_equal(got.view(np.int32), online.cpu().numpy().view(np.int32)), family
  else:
    e = U.polyak_error(got, before, online.cpu().numpy(), ref)
    record_parity(family, polyak=e)
    assert e <= U.TOL_POLYAK, f'{family}: target error {e:.3g}'


def _check_counters(agent, opts, train_steps, gate=None, counter=None):
  assert int(agent.train_step_counter) == train_steps
  for opt, params in opts:
    if isinstance(opt.inner, optimizers.AdamOptimizer):
      assert int(opt.iterations(params)) == opt.steps
  if gate is not None and gate.period != 1:
    assert counter.cpu().tolist() == [gate.counter, 0]


# ---- SAC ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('tau,period', [(0.005, 1), (0.5, 2)])
def test_sac_agent_updates(cuda, tau, period):
  rng = np.random.RandomState(61 + period)
  D, A, B = 11, 5, 256
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, AMIN, AMAX, 'action')
  actor = tnp.TanhNormalActorNetwork(obs_spec, act_spec, fc_layer_params=(64, 64), device=cuda).set_seed(1)
  critic = critic_network.CriticNetwork((obs_spec, act_spec), joint_fc_layer_params=(64, 64),
                                        device=cuda).set_seed(2)
  opts = [CheckedOptimizer(optimizers.Adam(3e-4)), CheckedOptimizer(optimizers.Adam(3e-4)),
          CheckedOptimizer(optimizers.AdamOptimizer(1e-3))]
  agent = sac_agent.SacAgent(
      ts.time_step_spec(obs_spec), act_spec, critic_network=critic, actor_network=actor,
      actor_optimizer=opts[0], critic_optimizer=opts[1], alpha_optimizer=opts[2],
      target_update_tau=tau, target_update_period=period, gamma=0.99, reward_scale_factor=1.5,
      initial_log_alpha=0.3)
  agent.initialize()
  gate = U.Periodically(period)
  d = lambda a: torch.as_tensor(a, device=cuda)
  for call in range(TRAIN_CALLS):
    obs = rng.randn(B, 2, D).astype(f32)
    action = (AMIN + (AMAX - AMIN) * rng.rand(B, 2, A)).astype(f32)
    ones = torch.ones(B, 2, dtype=torch.int32, device=cuda)
    traj = trajectory.Trajectory(ones, d(obs), d(action), (), ones, d(rng.randn(B, 2).astype(f32)),
                                 d((rng.rand(B, 2) > 0.1).astype(f32)))
    before = agent._target_params.cpu().numpy()
    agent.train(traj, noise=[(rng.randn(B, A)).astype(f32) for _ in range(3)])
    agent.check_numerics()
    for opt, name in zip(opts, ('actor', 'critic', 'alpha')):
      assert len(opt.records) == 1
      opt.check(f'agent_updates_sac_{name}')
    _check_target('agent_updates_sac_target', agent._target_params, agent._critic_params, before,
                  tau, gate)
    _check_counters(agent, [(opts[0], actor.flat_params), (opts[1], agent._critic_params),
                            (opts[2], agent._log_alpha)], call + 1, gate, agent._update_target._counter)


# ---- PPO ------------------------------------------------------------------------------------------
def _ppo_experience(rng, cuda, actor, B, T, D, A, discrete):
  N = B * T
  obs = rng.randn(B, T, D).astype(f32)
  step_type, next_step_type, discount = _episodes(rng, B, T)
  d = lambda a: torch.as_tensor(a, device=cuda)
  params = actor.distribution_params(torch.as_tensor(obs.reshape(N, D), device=cuda))
  if discrete:
    old_logits = (params.cpu().numpy() + 0.3 * rng.randn(N, A)).astype(f32)
    action = rng.randint(0, A, N).astype(np.int64).reshape(B, T)
    info = {'dist_params': {'logits': d(old_logits.reshape(B, T, A))}}
  else:
    loc, scale = (x.cpu().numpy() for x in params)
    old_loc = (loc + 0.1 * (AMAX - AMIN) / 2 * rng.randn(N, A)).astype(f32)
    old_scale = (scale * np.exp(0.2 * rng.randn(N, A))).astype(f32)
    action = np.clip(old_loc + old_scale * rng.randn(N, A), AMIN, AMAX).astype(f32).reshape(B, T, A)
    info = {'dist_params': {'loc': d(old_loc.reshape(B, T, A)), 'scale': d(old_scale.reshape(B, T, A))}}
  return trajectory.Trajectory(d(step_type), d(obs), d(action), info, d(next_step_type),
                               d(rng.rand(B, T).astype(f32)), d(discount))


@pytest.mark.parametrize('kind,clip', [('clip', 0.05), ('clip', 1e6), ('kl', 0.05), ('discrete', 0.05)])
def test_ppo_agent_updates(cuda, kind, clip):
  """num_epochs = 3: three Adam steps per train(), each with the global-norm clip scale of its
  own gradient (binding at 0.05, exactly 1 at 1e6)."""
  rng = np.random.RandomState(71 + len(kind))
  B, T, D = 16, 9, 13
  A = 7 if kind == 'discrete' else 5
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = (tensor_spec.BoundedTensorSpec((), torch.int64, 0, A - 1, 'action') if kind == 'discrete'
              else tensor_spec.BoundedTensorSpec((A,), torch.float32, AMIN, AMAX, 'action'))
  actor = actor_distribution_network.ActorDistributionNetwork(
      obs_spec, act_spec, fc_layer_params=(64, 32), activation_fn='tanh', device=cuda).set_seed(5)
  value = value_network.ValueNetwork(obs_spec, fc_layer_params=(64, 32), activation_fn='tanh',
                                     device=cuda).set_seed(6)
  opt = CheckedOptimizer(optimizers.Adam(3e-4) if kind == 'clip' else optimizers.AdamOptimizer(1e-3))
  kw = dict(PPO_KW, num_epochs=3, gradient_clipping=clip)
  if kind == 'clip':
    agent = ppo_clip_agent.PPOClipAgent(ts.time_step_spec(obs_spec), act_spec, opt, actor_net=actor,
                                        value_net=value, **kw)
  else:
    agent = ppo_agent.PPOAgent(ts.time_step_spec(obs_spec), act_spec, opt, actor_net=actor,
                               value_net=value, **kw, **KL_KW)
  agent.initialize()
  family = f'agent_updates_ppo_{kind}'
  for call in range(TRAIN_CALLS):
    traj = _ppo_experience(rng, cuda, actor, B, T, D, A, kind == 'discrete')
    agent.train(traj)
    agent.check_numerics()
    assert len(opt.records) == 3
    for pre, _ in opt.records:   # the clip scale the optimizer was handed
      scale_ref, _ = U.global_norm_scale(pre['g'].cpu().numpy(), clip)
      scale = float(pre['scale'][0])
      if clip > 1e3:
        assert scale == 1.0
      else:
        assert scale_ref < 0.9, 'global-norm clipping does not engage'
        e = U.rel_error(scale, scale_ref)
        record_parity(family, clip_scale=e)
        assert e <= U.TOL_CLIP, (scale, scale_ref)
    opt.check(family)
    _check_counters(agent, [(opt, agent._flat_params)], 3 * (call + 1))


# ---- DQN ------------------------------------------------------------------------------------------
DQN_OPTS = {
    'bench_rmsprop': lambda: optimizers.RMSPropOptimizer(2.5e-4, decay=0.95, momentum=0.0, epsilon=1e-5,
                                                         centered=True),
    'keras_mnih15_rmsprop': lambda: optimizers.RMSprop(2.5e-4, rho=0.95, momentum=0.95, epsilon=0.01,
                                                       centered=True),
    'adam': lambda: optimizers.AdamOptimizer(1e-3),
}


def _mnih_agent(cuda, cls, opt, tau, period, clip):
  obs_spec = tensor_spec.TensorSpec((84, 84, 4), torch.uint8, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 5, 'action')
  net = q_network.QNetwork(obs_spec, act_spec, preprocessing_layers=L.CastScale(255.),
                           conv_layer_params=((32, 8, 4), (64, 4, 2), (64, 3, 1)),
                           fc_layer_params=(512,), device=cuda).set_seed(9)
  agent = cls(ts.time_step_spec(obs_spec), act_spec, q_network=net, optimizer=opt, n_step_update=1,
              gamma=0.99, gradient_clipping=clip, target_update_tau=tau, target_update_period=period)
  agent.initialize()
  return agent, net


def _atari_batch(rng, cuda, B):
  d = lambda a: torch.as_tensor(a, device=cuda)
  ones = np.ones((B, 2), np.int32)
  return trajectory.Trajectory(d(ones), d(rng.randint(0, 256, (B, 2, 84, 84, 4)).astype(np.uint8)),
                               d(rng.randint(0, 6, (B, 2)).astype(np.int32)), (), d(ones),
                               d(rng.randn(B, 2).astype(f32)), d((rng.rand(B, 2) > 0.1).astype(f32)))


@pytest.mark.parametrize('tau,period', [(1.0, 3), (0.5, 2)])
@pytest.mark.parametrize('opt_name', sorted(DQN_OPTS))
@pytest.mark.parametrize('cls', [dqn_agent.DqnAgent, dqn_agent.DdqnAgent], ids=['dqn', 'ddqn'])
def test_dqn_agent_updates(cuda, cls, opt_name, tau, period):
  """The Mnih'15 Q-network (1.69 M parameters).  The per-variable clip is the median of the
  variables' gradient norms on the first batch, so it binds on about half of them."""
  B = 32
  probe_rng = np.random.RandomState(81)
  probe = CheckedOptimizer(optimizers.AdamOptimizer(1e-3))
  agent, net = _mnih_agent(cuda, cls, probe, tau, period, None)
  agent.train(_atari_batch(probe_rng, cuda, B))
  g = probe.records[0][0]['g'].cpu().numpy().astype(np.float64)
  offs = net.param_offsets
  clip = float(np.median([np.sqrt((g[a:b] ** 2).sum()) for a, b in zip(offs, offs[1:])]))

  rng = np.random.RandomState(81)
  opt = CheckedOptimizer(DQN_OPTS[opt_name]())
  agent, net = _mnih_agent(cuda, cls, opt, tau, period, clip)
  gate = U.Periodically(period)
  family = f'agent_updates_dqn_{opt_name}'
  for call in range(TRAIN_CALLS):
    before = agent._target_q_network.flat_params.cpu().numpy()
    agent.train(_atari_batch(rng, cuda, B))
    agent.check_numerics()
    assert len(opt.records) == 1
    g = opt.records[0][0]['g'].cpu().numpy().astype(np.float64)
    norms = np.array([np.sqrt((g[a:b] ** 2).sum()) for a, b in zip(offs, offs[1:])])
    assert (norms <= clip * (1 + U.TOL_CLIP)).all(), 'a variable above the clip reached the optimizer'
    if call == 0:
      binding = np.abs(norms / clip - 1) <= U.TOL_CLIP
      assert binding.any() and not binding.all(), norms / clip
    opt.check(family)
    _check_target(f'agent_updates_dqn_target_tau_{tau}', agent._target_q_network.flat_params,
                  net.flat_params, before, tau, gate)
    _check_counters(agent, [(opt, net.flat_params)], call + 1, gate, agent._update_target._counter)
