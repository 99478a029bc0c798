"""ReinforceAgent, b200rl_reinforce_loss, ActorPolicy and DynamicEpisodeDriver on the GPU:
the loss kernel against float64 autograd and oracle/reinforce.py, the reference's goldens
(agents/reinforce/reinforce_agent_test.py, drivers/dynamic_episode_driver_test.py), the
empty-batch contract, train parity with ReinforceOracle, graph replay, restore, policy draws and a
CartPole run that must learn."""
import numpy as np
import pytest
import torch

from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.agents.reinforce import reinforce_agent
from agents_b200.drivers import dynamic_episode_driver
from agents_b200.environments import tf_environment
from agents_b200.networks import actor_distribution_network
from agents_b200.networks import layers as L
from agents_b200.networks import value_network
from agents_b200.policies import actor_policy
from agents_b200.policies import tf_policy
from agents_b200.replay_buffers import tf_uniform_replay_buffer as rb_mod
from agents_b200.specs import tensor_spec
from agents_b200.train import learner as learner_lib
from agents_b200.trajectories import policy_step
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory
from agents_b200.utils import common
from oracle import nn as onn
from oracle import optim as ooptim
from oracle import philox
from oracle import ppo_discrete as opd
from oracle import reinforce as R

import test_oracle_reinforce as host
from conftest import record_parity

pytestmark = pytest.mark.gpu
f32 = np.float32
CANARY = 12345.0


# ---- the loss kernel ----------------------------------------------------------------------------
def _rows(cuda, x, ld):
  """[N, A] host array -> (base tensor [N, ld], view [N, A]) on the device (row stride ld)."""
  N, A = x.shape
  base = torch.full((N, ld), -777.0, dtype=torch.float32, device=cuda)
  base[:, :A] = torch.as_tensor(x, device=cuda)
  return base


def _grad_buf(cuda, N, A, ld):
  return torch.full((N * ld + 64,), CANARY, dtype=torch.float32, device=cuda)


def _kernel(cuda, case, cfg, discrete, value_coef=0.3, ld_pad=0):
  B, T = case['ret'].shape
  N = B * T
  d = lambda a, dt=torch.float32: None if a is None else torch.as_tensor(a, dtype=dt, device=cuda).contiguous()
  if discrete:
    A = case['params'].shape[1]
    ld = A + ld_pad
    p0, p1 = _rows(cuda, case['params'], ld), None
    action = d(case['action'], torch.int32)
    g0, g1 = _grad_buf(cuda, N, A, ld), None
  else:
    A = case['params'][0].shape[1]
    ld = A + ld_pad
    p0, p1 = _rows(cuda, case['params'][0], ld), _rows(cuda, case['params'][1], ld)
    action = d(case['action'])
    g0, g1 = _grad_buf(cuda, N, A, ld), _grad_buf(cuda, N, A, ld)
  V = d(case['V'])
  # every input stays referenced until the launch has been enqueued
  ret, st, nst, w = d(case['ret']), d(case['st'], torch.int32), d(case['nst'], torch.int32), d(case['w'])
  dv = torch.full((N + 64,), CANARY, dtype=torch.float32, device=cuda) if V is not None else None
  losses = torch.empty(6, dtype=torch.float32, device=cuda)
  ne = torch.zeros(1, dtype=torch.float32, device=cuda)
  flag = torch.zeros(1, dtype=torch.int32, device=cuda)
  ws = torch.empty(4 * (4096 + (B + 3) // 4 * 4 + N), dtype=torch.uint8, device=cuda)
  use_adv = bool(cfg['use_advantage']) and V is not None
  _lib.call('b200rl_reinforce_loss', p0.data_ptr(), None if p1 is None else p1.data_ptr(), ld,
            _lib.ptr(action), A, _lib.ptr(ret), _lib.ptr(V), _lib.ptr(st), _lib.ptr(nst), _lib.ptr(w),
            B, T, int(use_adv),
            int(cfg['normalize']), float(cfg['entropy'] or 0.0), float(value_coef), _lib.ptr(losses),
            g0.data_ptr(), None if g1 is None else g1.data_ptr(), ld, None if dv is None else dv.data_ptr(),
            _lib.ptr(ne), _lib.ptr(flag), _lib.ptr(ws), ws.numel(), _lib.stream())
  torch.cuda.synchronize()
  grads = []
  for g in (g0, g1):
    if g is None:
      continue
    assert torch.all(g[N * ld:] == CANARY), 'gradient written past its end'
    grads.append(g[:N * ld].reshape(N, ld)[:, :A].cpu().numpy())
    if ld_pad:
      assert torch.all(g[:N * ld].reshape(N, ld)[:, A:] == CANARY), 'gradient written in the row pad'
  if dv is not None:
    assert torch.all(dv[N:] == CANARY)
    dv = dv[:N].cpu().numpy().reshape(B, T)
  return losses.cpu().numpy(), grads, dv, float(ne.item()), int(flag.item())


KERNEL_CASES = [(False, 1), (False, 6), (True, 2), (True, 6), (True, 18), (True, 300)]


@pytest.mark.parametrize('discrete,A', KERNEL_CASES, ids=[f"{'cat' if c else 'normal'}{a}" for c, a in KERNEL_CASES])
@pytest.mark.parametrize('name', sorted(host.CONFIGS))
def test_loss_kernel_matches_float64_and_oracle(cuda, discrete, A, name):
  cfg = host.CONFIGS[name]
  rng = np.random.default_rng(11 + A)
  case = host.make_case(rng, 24, 60, A, discrete, cfg)
  losses, grads, dv, ne, flag = _kernel(cuda, case, cfg, discrete, ld_pad=3 if A == 6 else 0)
  assert flag == 0
  info, _, _ = host.oracle_grads(case, cfg, discrete)
  total, want_params, want_dv = host.autograd_grads(case, cfg, discrete)
  assert ne == info['num_episodes']
  rel = abs(losses[5] - total) / max(abs(total), 1e-6)
  record_parity(f'reinforce_loss_{name}_{"cat" if discrete else "normal"}{A}', loss_rel=rel)
  assert rel <= 1e-5, (losses, total)
  np.testing.assert_allclose(losses[0], info['policy_gradient_loss'], rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(losses[2], info['entropy_regularization_loss'], rtol=1e-5, atol=1e-7)
  np.testing.assert_allclose(losses[3], info['value_estimation_loss'], rtol=1e-5, atol=1e-7)
  assert losses[1] == 0 and losses[4] == 0
  for got, want in zip(grads, want_params):
    host._close(got, want, 1e-4)
  if want_dv is not None:
    host._close(dv, want_dv, 1e-4)


def test_out_of_range_actions_raise_the_flag_and_stay_in_bounds(cuda):
  cfg = host.CONFIGS['no_baseline_norm']
  rng = np.random.default_rng(2)
  case = host.make_case(rng, 4, 8, 5, True, cfg)
  case['action'][3], case['action'][9] = -1, 5
  losses, grads, _, _, flag = _kernel(cuda, case, cfg, True)
  assert flag & 1
  assert np.all(np.isfinite(losses)) and np.all(np.isfinite(grads[0]))


def test_no_complete_episode_zeroes_gradients_and_sets_the_flag(cuda):
  cfg = host.CONFIGS['baseline_adv_norm_ent_weights']
  rng = np.random.default_rng(4)
  case = host.make_case(rng, 3, 6, 6, True, cfg)
  case['st'][:] = R.STEP_MID
  case['nst'][:] = R.STEP_MID
  losses, grads, dv, ne, flag = _kernel(cuda, case, cfg, True)
  assert flag == 2 and ne == 0
  assert np.all(losses == 0) and np.all(grads[0] == 0) and np.all(dv == 0)


def test_loss_kernel_graph_replay_is_bitwise_equal_to_eager(cuda):
  cfg = host.CONFIGS['baseline_adv_norm_ent_weights']
  rng = np.random.default_rng(5)
  case = host.make_case(rng, 64, 512, 6, False, cfg)       # N = 32768: many CTAs per stage
  B, T, N, A = 64, 512, 64 * 512, 6
  d = lambda a, dt=torch.float32: torch.as_tensor(a, dtype=dt, device=cuda).contiguous()
  loc, scale, act = d(case['params'][0]), d(case['params'][1]), d(case['action'])
  ret, V, w = d(case['ret']), d(case['V']), d(case['w'])
  st, nst = d(case['st'], torch.int32), d(case['nst'], torch.int32)
  outs = [torch.empty(6, device=cuda), torch.empty(N, A, device=cuda), torch.empty(N, A, device=cuda),
          torch.empty(N, device=cuda)]
  flag = torch.zeros(1, dtype=torch.int32, device=cuda)
  ws = torch.empty(4 * (4096 + B + N), dtype=torch.uint8, device=cuda)

  def launch():
    _lib.call('b200rl_reinforce_loss', _lib.ptr(loc), _lib.ptr(scale), A, _lib.ptr(act), A, _lib.ptr(ret),
              _lib.ptr(V), _lib.ptr(st), _lib.ptr(nst), _lib.ptr(w), B, T, 1, 1, 0.01, 0.2,
              _lib.ptr(outs[0]), _lib.ptr(outs[1]), _lib.ptr(outs[2]), A, _lib.ptr(outs[3]), None,
              _lib.ptr(flag), _lib.ptr(ws), ws.numel(), _lib.stream())

  launch()
  eager = [o.clone() for o in outs]
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  g = torch.cuda.CUDAGraph()
  with torch.cuda.stream(s):
    with torch.cuda.graph(g, stream=s):
      launch()
  torch.cuda.current_stream().wait_stream(s)
  for o in outs:
    o.zero_()
  g.replay()
  torch.cuda.synchronize()
  for a, b in zip(outs, eager):
    assert torch.equal(a, b)


# ---- goldens through the kernel and the agent's public losses -----------------------------------
def _agent(cuda, act_spec=None, **kw):
  obs_spec = tensor_spec.TensorSpec([2], torch.float32)
  act_spec = act_spec or tensor_spec.BoundedTensorSpec([1], torch.float32, -1, 1)
  actor = actor_distribution_network.ActorDistributionNetwork(obs_spec, act_spec, fc_layer_params=(4,),
                                                              device=cuda)
  return reinforce_agent.ReinforceAgent(ts.time_step_spec(obs_spec), act_spec, actor,
                                        optimizers.Adam(1e-3), **kw)


@pytest.mark.parametrize('name', sorted(host.TRAIN_GOLDENS))
def test_train_goldens_through_the_kernel(cuda, name):
  exp, expected = host.golden_experience(name)
  T = exp['reward'].shape[1]
  loc, scale = host._dummy_actor(exp['observation'].reshape(-1, 2))
  case = dict(st=exp['step_type'], nst=exp['next_step_type'], V=None, w=None, params=(loc, scale),
              action=exp['action'].reshape(T, 1),
              ret=R.compute_returns(exp['reward'], exp['discount'], exp['next_step_type'], 1.0))
  cfg = dict(use_advantage=False, normalize=False, entropy=None)
  losses, _, _, _, flag = _kernel(cuda, case, cfg, False)
  assert flag == 0
  np.testing.assert_allclose(losses[5], expected, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize('obs,actions,is_boundary,returns,num_episodes,expected', [
    ([[1, 2], [3, 4]], [[0], [1]], [0, 0], [1.9, 1.0], 1, 10.983667373657227),
    ([[1, 2]] * 4, [[0], [1], [2], [3]], [0, 1, 0, 1], [1.9, 1.9, 1.0, 1.0], 2, 5.140229225158691),
    ([[1, 2]] * 2, [[0], [1]], [0, 1], [3.0, 0.0], 1, 10.8935775757),
    ([[1, 2]] * 2, [[0], [1]], [0, 1], [0.0, 3.0], 1, 0.0),
    ([[1, 2]] * 4, [[0], [1], [2], [3]], [0, 1, 0, 1], [3.0, 0.0, 4.0, 0.0], 2, 12.2091741562),
    ([[1, 2]] * 4, [[0], [1], [2], [3]], [0, 1, 0, 1], [0.0, 3.0, 0.0, 4.0], 2, 0.0),
])
def test_policy_gradient_loss_goldens_through_the_agent(cuda, obs, actions, is_boundary, returns,
                                                        num_episodes, expected):
  agent = _agent(cuda)
  loc, scale = host._dummy_actor(obs)
  dist = (torch.as_tensor(loc, device=cuda), torch.as_tensor(scale, device=cuda))
  got = agent.policy_gradient_loss(dist, torch.tensor(actions, dtype=torch.float32, device=cuda),
                                   torch.tensor(is_boundary, device=cuda), returns, num_episodes)
  np.testing.assert_allclose(got.item(), expected, rtol=1e-6, atol=1e-6)


def test_value_and_entropy_goldens_through_the_agent(cuda):
  obs_spec = tensor_spec.TensorSpec([2], torch.float32)
  agent = _agent(cuda, value_network=value_network.ValueNetwork(obs_spec, device=cuda),
                 value_estimation_loss_coef=0.5)
  v = torch.tensor([9.0, 15.0], device=cuda)                        # DummyValueNet on [[1,2],[3,4]]
  np.testing.assert_allclose(agent.value_estimation_loss(v, [1.9, 1.0], 1).item(), 123.205, rtol=1e-6)
  act = tensor_spec.BoundedTensorSpec([], torch.int32, 0, 1)
  for probs, weights in (([[0.8, 0.2]], [1.0]), ([[0.8, 0.2], [0.3, 0.7]], [0.5, 0.5])):
    cat = _agent(cuda, act_spec=act, entropy_regularization=1.0)
    logits = torch.log(torch.tensor(probs, device=cuda))
    H = torch.distributions.Categorical(probs=torch.tensor(probs, dtype=torch.float64)).entropy()
    want = float(torch.mean(-H.mean() * torch.tensor(weights, dtype=torch.float64)))
    got = cat.entropy_regularization_loss(logits, torch.tensor(weights, device=cuda))
    assert abs(got.item() - want) < 1e-4
    assert _agent(cuda, act_spec=act).entropy_regularization_loss(logits).item() == 0.0


# ---- train: parity, empty batch, graph replay, restore ------------------------------------------
def _nets(cuda, obs_spec, act_spec, baseline, l2=0.0):
  actor = actor_distribution_network.ActorDistributionNetwork(
      obs_spec, act_spec, fc_layer_params=(32, 16), activation_fn='tanh', device=cuda).set_seed(1)
  value = None
  if baseline:
    value = value_network.ValueNetwork(obs_spec, fc_layer_params=(32, 16), activation_fn='tanh',
                                       device=cuda).set_seed(2)
  if l2:
    for net in (actor, value):
      if net is not None:
        net.create_variables()
        net.layers[0].l2 = l2
  return actor, value


def _mirror(net):
  layers = []
  for l in net.layers:
    if isinstance(l, L.Dense):
      layers.append(dict(kind='dense', w=l.kernel.cpu().numpy().copy(), b=l.bias.cpu().numpy().copy(),
                         act=l.activation, l2=getattr(l, 'l2', 0.0)))
  return onn.Sequential(layers)


def _experience(rng, B, T, D, A, discrete):
  st, nst = host.random_steps(rng, B, T)
  e = dict(step_type=st, next_step_type=nst, observation=rng.normal(size=(B, T, D)).astype(f32),
           reward=rng.normal(size=(B, T)).astype(f32),
           discount=np.where(nst == R.STEP_LAST, 0.0, 1.0).astype(f32))
  if discrete:
    e['action'] = rng.integers(0, A, size=(B, T)).astype(np.int64)
  else:
    e['action'] = rng.uniform(-1, 1, size=(B, T, A)).astype(f32)
  return e


def _traj(cuda, e):
  d = lambda a: torch.as_tensor(a, device=cuda)
  return trajectory.Trajectory(d(e['step_type']), d(e['observation']), d(e['action']), (),
                               d(e['next_step_type']), d(e['reward']), d(e['discount']))


TRAIN_CONFIGS = {
    'normal_baseline_clip_l2': dict(discrete=False, baseline=True, clip=0.5, l2=1e-3, entropy=None,
                                    normalize=True),
    'normal_no_baseline_entropy': dict(discrete=False, baseline=False, clip=None, l2=0.0, entropy=0.01,
                                       normalize=True),
    'categorical_baseline_clip_l2_entropy': dict(discrete=True, baseline=True, clip=0.5, l2=1e-3,
                                                 entropy=0.01, normalize=True),
    'categorical_no_baseline_raw': dict(discrete=True, baseline=False, clip=None, l2=0.0, entropy=None,
                                        normalize=False),
}


def _make_pair(cuda, cfg, D=17, A=6, lr=1e-3):
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  if cfg['discrete']:
    act_spec = tensor_spec.BoundedTensorSpec((), torch.int64, 0, A - 1, 'action')
  else:
    act_spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, -1, 1, 'action')
  actor, value = _nets(cuda, obs_spec, act_spec, cfg['baseline'], cfg['l2'])
  agent = reinforce_agent.ReinforceAgent(
      ts.time_step_spec(obs_spec), act_spec, actor, optimizers.Adam(lr), value_network=value,
      gamma=0.99, normalize_returns=cfg['normalize'], gradient_clipping=cfg['clip'],
      entropy_regularization=cfg['entropy'])
  agent.initialize()
  kw = {}
  if not cfg['discrete']:
    kw = dict(std_bias=actor._std.bias.cpu().numpy().copy(), amin=-np.ones(A, f32), amax=np.ones(A, f32))
  orc = R.ReinforceOracle(_mirror(actor), _mirror(value) if value is not None else None,
                          ooptim.AdamTF(lr, eps=1e-7), discrete=cfg['discrete'], gamma=0.99,
                          normalize_returns=cfg['normalize'], gradient_clipping=cfg['clip'],
                          entropy_regularization=cfg['entropy'], **kw)
  return agent, orc, [n for n in (actor, value) if n is not None]


@pytest.mark.parametrize('name', sorted(TRAIN_CONFIGS))
def test_agent_train_matches_oracle(cuda, name):
  cfg = TRAIN_CONFIGS[name]
  rng = np.random.default_rng(21)
  B, T, D, A = 16, 40, 17, 6
  agent, orc, nets = _make_pair(cuda, cfg, D, A)
  for _ in range(5):
    e = _experience(rng, B, T, D, A, cfg['discrete'])
    w = rng.uniform(0.5, 1.5, size=(B, T)).astype(f32)
    want = orc.train(e, weights=w)
    got = agent.train(_traj(cuda, e), weights=torch.as_tensor(w, device=cuda))
    rel = abs(got.loss.item() - want['loss']) / max(abs(want['loss']), 1e-30)
    record_parity('reinforce_train_' + name, loss_rel=rel)
    np.testing.assert_allclose(got.loss.item(), want['loss'], rtol=1e-5, atol=1e-6)
    x = got.extra
    np.testing.assert_allclose(x.policy_gradient_loss.item(), want['policy_gradient_loss'], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(x.entropy_regularization_loss.item(), want['entropy_regularization_loss'],
                               rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(x.value_estimation_loss.item(), want['value_estimation_loss'], rtol=1e-5,
                               atol=1e-7)
    np.testing.assert_allclose(x.policy_network_regularization_loss.item(),
                               want['policy_network_regularization_loss'], rtol=1e-5, atol=1e-8)
    np.testing.assert_allclose(x.value_network_regularization_loss.item(),
                               want['value_network_regularization_loss'], rtol=1e-5, atol=1e-8)
  assert int(agent.train_step_counter.item()) == 5
  got = np.concatenate([v.cpu().numpy().reshape(-1) for n in nets for v in n.variables])
  want = np.concatenate([p.reshape(-1) for p in orc.params()])
  err = np.abs(got - want)
  record_parity('reinforce_train_' + name, param_max_abs=float(err.max()))
  assert float((err > 2e-3 * np.abs(want) + 2e-5).mean()) <= 1e-3
  assert err.max() <= 5 * 1e-3
  agent.check_numerics()


def _empty(cuda, B=4, T=8, D=17, A=6):
  rng = np.random.default_rng(1)
  e = _experience(rng, B, T, D, A, True)
  e['step_type'][:] = R.STEP_MID
  e['next_step_type'][:] = R.STEP_MID
  return _traj(cuda, e), _traj(cuda, _experience(rng, B, T, D, A, True))


def test_empty_batch_raises_before_the_update(cuda):
  cfg = TRAIN_CONFIGS['categorical_baseline_clip_l2_entropy']
  agent, _, _ = _make_pair(cuda, cfg)
  empty, good = _empty(cuda)
  before = agent._flat_params.clone()
  with pytest.raises(ValueError, match='No complete episode found. REINFORCE requires full episodes'):
    agent.train(empty)
  assert torch.equal(agent._flat_params, before)
  assert int(agent.train_step_counter.item()) == 0
  agent.train(good)                              # the flag bit was consumed by the raise
  agent.check_numerics()


def test_empty_batch_under_graph_replay_sets_the_flag(cuda):
  # without L2 terms every gradient of the replayed step is the loss kernel's, hence zero
  cfg = dict(TRAIN_CONFIGS['categorical_baseline_clip_l2_entropy'], l2=0.0)
  agent, _, _ = _make_pair(cuda, cfg)
  empty, good = _empty(cuda)
  train_fn = common.function(agent.train)
  for _ in range(3):
    train_fn(good)
  agent.check_numerics()
  grads_before = agent._flat_grads.clone()
  train_fn(empty)
  torch.cuda.synchronize()
  assert torch.all(agent._flat_grads == 0) and not torch.all(grads_before == 0)
  with pytest.raises(FloatingPointError, match='No complete episode found'):
    agent.check_numerics()


def test_graph_replay_matches_eager_and_restore_reproduces_the_next_loss(cuda):
  cfg = TRAIN_CONFIGS['normal_baseline_clip_l2']
  rng = np.random.default_rng(9)
  eager, _, _ = _make_pair(cuda, cfg)
  graphed, _, _ = _make_pair(cuda, cfg)
  train_fn = common.function(graphed.train)
  batches = [_traj(cuda, _experience(rng, 8, 32, 17, 6, False)) for _ in range(6)]
  for i, b in enumerate(batches[:5]):
    l1 = eager.train(b).loss.item()
    l2 = train_fn(b).loss.item()
    if i == 0:
      assert l1 == l2                                  # same parameters: the same bits
    np.testing.assert_allclose(l2, l1, rtol=1e-6)
  # inside a captured graph the weight gradients run on a side stream (network.backward), so the
  # parameters agree to fp32 rounding
  torch.testing.assert_close(graphed._flat_params, eager._flat_params, rtol=1e-5, atol=1e-6)
  # restore: the checkpointed tensors of `eager` into a fresh agent reproduce its next loss
  restored, _, _ = _make_pair(cuda, cfg)
  dst = learner_lib._agent_state_tensors(restored)
  for k, v in learner_lib._agent_state_tensors(eager).items():
    dst[k].copy_(v)
  restored.train_step_counter.fill_(int(eager.train_step_counter.item()))
  assert restored.train(batches[5]).loss.item() == eager.train(batches[5]).loss.item()
  # the weight gradients accumulate split-K partials with atomic adds: equal to fp32 rounding
  torch.testing.assert_close(restored._flat_params, eager._flat_params, rtol=1e-5, atol=1e-6)
  assert int(restored.train_step_counter.item()) == int(eager.train_step_counter.item()) == 6


# ---- ActorPolicy draws ----------------------------------------------------------------------------
def test_actor_policy_draws_match_philox_and_clip(cuda):
  obs_spec = tensor_spec.TensorSpec((5,), torch.float32)
  act_spec = tensor_spec.BoundedTensorSpec((3,), torch.float32, -0.5, 0.5)
  actor = actor_distribution_network.ActorDistributionNetwork(obs_spec, act_spec, fc_layer_params=(8,),
                                                              std_bias_initializer_value=1.0, device=cuda)
  pol = actor_policy.ActorPolicy(ts.time_step_spec(obs_spec), act_spec, actor, seed=3)
  obs = torch.randn(1000, 5, device=cuda)
  loc, scale = [t.cpu().numpy() for t in actor.distribution_params(obs)]
  seed = (3 ^ actor_policy._ACTOR_SEED_TAG) & 0xFFFFFFFFFFFFFFFF
  for call in range(2):
    act = pol.action(ts.restart(obs, batch_size=1000)).action.cpu().numpy()
    r = philox.philox(np.arange(3000, dtype=np.uint64), call, seed)
    u1 = ((r[0] >> 8).astype(np.float64) + 1.0) / 16777216.0
    u2 = (r[1] >> 8).astype(np.float64) / 16777216.0
    z = (np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)).reshape(1000, 3)
    want = np.clip(loc + scale * z, -0.5, 0.5)
    np.testing.assert_allclose(act, want, rtol=0, atol=2e-5)
    assert act.min() >= -0.5 and act.max() <= 0.5
    assert (np.abs(loc + scale * z) > 0.5).any()       # the clip was exercised
  greedy = actor_policy.ActorPolicy(ts.time_step_spec(obs_spec), act_spec, actor, collect=False)
  np.testing.assert_array_equal(greedy.action(ts.restart(obs, batch_size=1000)).action.cpu().numpy(), loc)
  # Categorical head
  cat_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 6)
  cat = actor_distribution_network.ActorDistributionNetwork(obs_spec, cat_spec, fc_layer_params=(8,),
                                                            device=cuda)
  pol = actor_policy.ActorPolicy(ts.time_step_spec(obs_spec), cat_spec, cat, seed=3)
  logits = cat.distribution_params(obs).cpu().numpy() * 1.0
  act = pol.action(ts.restart(obs, batch_size=1000)).action.cpu().numpy()
  want, u = opd.categorical_sample(logits, seed, 0)
  near = (np.abs(opd.categorical_cdf(logits) - u[:, None]) < 1e-6).any(axis=1)
  np.testing.assert_array_equal(act[~near], want[~near])
  assert pol.info_spec == () and pol.action(ts.restart(obs, batch_size=1000)).info == ()


# ---- DynamicEpisodeDriver -----------------------------------------------------------------------
class EnvMock(tf_environment.TFEnvironment):
  """drivers/test_utils.py PyEnvironmentMock (state += action, the episode ends at state >= 3),
  batched to [1] on the device."""

  def __init__(self, device, final_state=3):
    obs = tensor_spec.TensorSpec([], torch.int32, 'observation')
    act = tensor_spec.BoundedTensorSpec([], torch.int32, 1, 2, 'action')
    super().__init__(ts.time_step_spec(obs), act, batch_size=1)
    self._dev, self._final = device, final_state
    self._state = 0
    self._cur = None

  def _current_time_step(self):
    return self._cur if self._cur is not None else self._reset()

  def _reset(self):
    self._state = 0
    self._cur = ts.restart(torch.zeros(1, dtype=torch.int32, device=self._dev), batch_size=1)
    return self._cur

  def _step(self, action):
    if self._cur is None or self._state >= self._final:
      return self._reset()
    self._state += int(action.item())
    obs = torch.full((1,), self._state, dtype=torch.int32, device=self._dev)
    rew = torch.ones(1, device=self._dev)
    self._cur = ts.transition(obs, rew) if self._state < self._final else ts.termination(obs, rew)
    return self._cur


class PolicyMock(tf_policy.TFPolicy):
  """drivers/test_utils.py TFPolicyMock: actions alternate 1, 2 within an episode; info = 2 * action."""

  def __init__(self, time_step_spec, action_spec, device):
    super().__init__(time_step_spec, action_spec,
                     policy_state_spec=tensor_spec.BoundedTensorSpec((), torch.int32, 1, 2),
                     info_spec=action_spec)
    self._dev = device

  def get_initial_state(self, batch_size=None):
    return torch.zeros(batch_size or 1, dtype=torch.int32, device=self._dev)

  def _action(self, time_step, policy_state, seed):
    policy_state = torch.where(time_step.is_first(), torch.zeros_like(policy_state), policy_state)
    action = (policy_state % 2 + 1).to(torch.int32)
    return policy_step.PolicyStep(action, policy_state + 1, (action * 2).to(torch.int32))


def _counters():
  c = {'episodes': 0, 'steps': 0, 'transitions': 0}

  def episodes(traj):                  # NumEpisodesObserver: boundary transitions
    c['episodes'] += int((traj.step_type == ts.StepType.LAST).sum())

  def steps(traj):                     # NumStepsObserver: non-boundary transitions
    c['steps'] += int((traj.step_type != ts.StepType.LAST).sum())

  def transitions(t):                  # NumStepsTransitionObserver
    c['transitions'] += int((t[0].step_type != ts.StepType.LAST).sum())
  return c, [episodes, steps], [transitions]


def test_episode_driver_observer_goldens(cuda):
  # dynamic_episode_driver_test.py:83-172: 5 runs of 1 episode, one run of 5, num_episodes=5
  for how in ('five_runs', 'run_arg', 'ctor'):
    env = EnvMock(cuda)
    policy = PolicyMock(env.time_step_spec(), env.action_spec(), cuda)
    c, obs, tobs = _counters()
    kw = dict(num_episodes=5) if how == 'ctor' else {}
    driver = dynamic_episode_driver.DynamicEpisodeDriver(env, policy, observers=obs,
                                                         transition_observers=tobs, **kw)
    if how == 'five_runs':
      for _ in range(5):
        driver.run()
    elif how == 'run_arg':
      driver.run(num_episodes=5)
    else:
      driver.run()
    assert c == {'episodes': 5, 'steps': 10, 'transitions': 10}, (how, c)


def test_episode_driver_replay_buffer_goldens(cuda):
  # :174-240: three runs of one episode, and one run of three
  for num_episodes, runs in ((1, 3), (3, 1)):
    env = EnvMock(cuda)
    policy = PolicyMock(env.time_step_spec(), env.action_spec(), cuda)
    rb = rb_mod.TFUniformReplayBuffer(policy.trajectory_spec, batch_size=1, max_length=1000, device=cuda)
    driver = dynamic_episode_driver.DynamicEpisodeDriver(env, policy, num_episodes=num_episodes,
                                                         observers=[rb.add_batch])
    for _ in range(runs):
      driver.run()
    tr = rb.gather_all()
    assert tr.step_type.cpu().tolist() == [[0, 1, 2, 0, 1, 2, 0, 1, 2]]
    assert tr.action.cpu().tolist() == [[1, 2, 1, 1, 2, 1, 1, 2, 1]]
    assert tr.observation.cpu().tolist() == [[0, 1, 3, 0, 1, 3, 0, 1, 3]]
    assert tr.policy_info.cpu().tolist() == [[2, 4, 2, 2, 4, 2, 2, 4, 2]]
    assert tr.next_step_type.cpu().tolist() == [[1, 2, 0, 1, 2, 0, 1, 2, 0]]
    assert tr.reward.cpu().tolist() == [[1.0, 1.0, 0.0, 1.0, 1.0, 0.0, 1.0, 1.0, 0.0]]
    assert tr.discount.cpu().tolist() == [[1.0, 0.0, 1.0, 1.0, 0.0, 1.0, 1.0, 0.0, 1.0]]
  env = EnvMock(cuda)
  policy = PolicyMock(env.time_step_spec(), env.action_spec(), cuda)
  c, obs, tobs = _counters()
  dynamic_episode_driver.DynamicEpisodeDriver(env, policy, observers=obs, num_episodes=5).run(
      maximum_iterations=4)
  assert c['episodes'] + c['steps'] == 4                # bounded: no counter read past the bound


# ---- CartPole end to end --------------------------------------------------------------------------
CARTPOLE_THRESHOLD = 80.0


def test_cartpole_end_to_end_learns(cuda):
  """Device CartPole (8 envs) -> DynamicEpisodeDriver(collect policy, 8 episodes, at most 600
  iterations) -> TFUniformReplayBuffer -> gather_all -> ReinforceAgent.train (value baseline,
  normalised advantages, gamma 0.99, Adam 3e-3) -> clear, 30 iterations; then the greedy policy's
  mean first-episode length over 16 evaluation envs must reach CARTPOLE_THRESHOLD.
  Threshold: the same configuration run on the CPU through oracle/reinforce.py (oracle CartPole,
  oracle categorical draws, (64,) relu nets) gave 192, 134, 143, 325, 179, 245, 204 and 295 for
  seeds 0-7 (median ~198); an untrained policy lasts ~20 steps.  80 sits below the smallest of
  those with margin and is ~4x the untrained length."""
  from agents_b200.environments import random_tf_environment
  B, NE, TMAX, iters = 8, 8, 600, 30
  env = random_tf_environment.CartPoleTFEnvironment(batch_size=B, seed=0, device=cuda)
  tss, act_spec = env.time_step_spec(), env.action_spec()
  actor = actor_distribution_network.ActorDistributionNetwork(tss.observation, act_spec,
                                                              fc_layer_params=(64,), device=cuda).set_seed(0)
  value = value_network.ValueNetwork(tss.observation, fc_layer_params=(64,), device=cuda).set_seed(1)
  agent = reinforce_agent.ReinforceAgent(tss, act_spec, actor, optimizers.Adam(3e-3), value_network=value,
                                         gamma=0.99, normalize_returns=True)
  agent.initialize()
  assert agent.collect_data_spec.policy_info == ()
  rb = rb_mod.TFUniformReplayBuffer(agent.collect_data_spec, batch_size=B, max_length=TMAX, device=cuda)
  driver = dynamic_episode_driver.DynamicEpisodeDriver(env, agent.collect_policy, observers=[rb.add_batch],
                                                       num_episodes=NE)
  for _ in range(iters):
    driver.run(maximum_iterations=TMAX)
    exp = rb.gather_all()
    assert exp.action.shape[0] == B
    agent.train(exp)
    rb.clear()
  agent.check_numerics()
  ev = random_tf_environment.CartPoleTFEnvironment(batch_size=16, seed=7, device=cuda)
  step = ev.reset()
  length = torch.zeros(16, dtype=torch.int32, device=cuda)
  alive = torch.ones(16, dtype=torch.bool, device=cuda)
  for _ in range(500):
    step = ev.step(agent.policy.action(step).action)
    length += alive.to(torch.int32)
    alive &= step.step_type != ts.StepType.LAST
    if not bool(alive.any()):
      break
  mean_len = float(length.float().mean())
  record_parity('reinforce_cartpole', mean_episode_length=mean_len)
  assert mean_len >= CARTPOLE_THRESHOLD, mean_len
