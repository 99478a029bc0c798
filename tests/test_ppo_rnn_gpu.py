"""Recurrent PPO on the GPU: PPOAgent.train with ActorDistributionRnnNetwork / ValueRnnNetwork
against PPOOracle on oracle/lstm.py networks, the stateful collect policy, the guards of the agents
that do not train recurrent networks, and a cue-recall task only a recurrent policy can solve."""
import numpy as np
import pytest
import torch

from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.drivers import dynamic_episode_driver
from agents_b200.drivers import dynamic_step_driver
from agents_b200.environments import random_tf_environment
from agents_b200.replay_buffers import tf_uniform_replay_buffer as rb_mod
from agents_b200.train import learner as learner_lib
from agents_b200.train import ppo_learner
from agents_b200.utils import common
from agents_b200.agents.dqn import dqn_agent
from agents_b200.agents.ppo import ppo_agent
from agents_b200.agents.ppo import ppo_clip_agent
from agents_b200.agents.sac import sac_agent
from agents_b200.agents.cql import cql_sac_agent
from agents_b200.networks import actor_distribution_rnn_network as adrn
from agents_b200.networks import layers as L
from agents_b200.networks import lstm_encoding_network as len_
from agents_b200.networks import value_network
from agents_b200.networks import value_rnn_network as vrn
from agents_b200.specs import tensor_spec
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory
from oracle import lstm as olstm
from oracle import nn as onn
from oracle import optim as ooptim
from oracle import ppo as oppo
from oracle import ppo_discrete as oppod

import grad_refs as R

from conftest import record_parity

pytestmark = pytest.mark.gpu
f32 = np.float32


def _dense(l):
  return dict(kind='dense', w=l.kernel.cpu().numpy().copy(), b=l.bias.cpu().numpy().copy(),
              act=l.activation)


def _mirror(net):
  """oracle copy of a network: RnnNet for a recurrent one (Dense / StdBias layers after the LSTMs
  go to `post`), Sequential otherwise."""
  if not net.state_spec:
    return onn.Sequential([_dense(l) for l in net.layers if isinstance(l, L.Dense)])
  pre = [_dense(l) for l in net._pre]
  cells = [[c.kernel.cpu().numpy().copy(), c.recurrent_kernel.cpu().numpy().copy(),
            c.bias.cpu().numpy().copy()] for c in net._cells]
  post = [_dense(l) for l in net._post if isinstance(l, L.Dense)]
  return olstm.RnnNet(pre, cells, post)


def _experience(rng, B, T, D, A, discrete=False):
  e = dict(observation=rng.randn(B, T, D).astype(f32), reward=rng.rand(B, T).astype(f32),
           discount=np.ones((B, T), f32), step_type=np.ones((B, T), np.int32),
           next_step_type=np.ones((B, T), np.int32),
           value_prediction=rng.randn(B, T).astype(f32))
  if discrete:
    e['action'] = rng.randint(0, A, size=(B, T)).astype(np.int32)
    e['logits'] = rng.randn(B, T, A).astype(f32)
  else:
    e['action'] = np.clip(rng.randn(B, T, A) * .5, -1, 1).astype(f32)
    e['loc'] = (rng.randn(B, T, A) * .2).astype(f32)
    e['scale'] = (rng.rand(B, T, A) * .3 + .5).astype(f32)
  e['step_type'][:, 0] = 0
  ends = rng.rand(B, T) < 0.08
  e['next_step_type'][ends] = 2
  e['discount'][ends] = 0
  e['step_type'][:, 1:][ends[:, :-1]] = 0            # the step after a LAST starts an episode
  return e


def _to_traj(cuda, e, with_value=False):
  d = lambda a: torch.as_tensor(a, device=cuda)
  if 'logits' in e:
    info = {'dist_params': {'logits': d(e['logits'])}}
  else:
    info = {'dist_params': {'loc': d(e['loc']), 'scale': d(e['scale'])}}
  if with_value:
    info['value_prediction'] = d(e['value_prediction'])
  return trajectory.Trajectory(d(e['step_type']), d(e['observation']), d(e['action']), info,
                               d(e['next_step_type']), d(e['reward']), d(e['discount']))


def _specs(D, A, discrete):
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  if discrete:
    act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, A - 1, 'action')
  else:
    act_spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, -1.0, 1.0, 'action')
  return obs_spec, act_spec


def _build(cuda, D, A, rnn_value, discrete=False, optimizer=None, **kw):
  obs_spec, act_spec = _specs(D, A, discrete)
  actor = adrn.ActorDistributionRnnNetwork(obs_spec, act_spec, input_fc_layer_params=(32,),
                                           lstm_size=(20,), output_fc_layer_params=(16,),
                                           activation_fn='tanh', device=cuda).set_seed(1)
  if rnn_value:
    value = vrn.ValueRnnNetwork(obs_spec, input_fc_layer_params=(32,), lstm_size=(7, 5),
                                output_fc_layer_params=(16,), activation_fn='tanh',
                                device=cuda).set_seed(2)
  else:
    value = value_network.ValueNetwork(obs_spec, fc_layer_params=(32,), activation_fn='tanh',
                                       device=cuda).set_seed(2)
  agent = ppo_agent.PPOAgent(ts.time_step_spec(obs_spec), act_spec,
                             optimizer=optimizer or optimizers.Adam(1e-3), actor_net=actor,
                             value_net=value, **kw)
  agent.initialize()
  return agent, actor, value


KL_KW = dict(kl_cutoff_factor=2.0, kl_cutoff_coef=1000.0, initial_adaptive_kl_beta=1.0,
             adaptive_kl_target=0.01, adaptive_kl_tolerance=0.3)
NO_KL_KW = dict(kl_cutoff_factor=0.0, initial_adaptive_kl_beta=0.0)


@pytest.mark.parametrize('discrete', [False, True])
@pytest.mark.parametrize('rnn_value', [True, False])
@pytest.mark.parametrize('kl', [False, True])
@pytest.mark.parametrize('value_in_train', [True, False])
def test_recurrent_ppo_train_matches_oracle(cuda, discrete, rnn_value, kl, value_in_train):
  rng = np.random.RandomState(3 + 2 * discrete + kl)
  B, T, D, A = 6, 21, 9, 3
  kl_kw = KL_KW if kl else NO_KL_KW
  agent, actor, value = _build(cuda, D, A, rnn_value, discrete, importance_ratio_clipping=0.2,
                               use_gae=True, lambda_value=0.95, discount_factor=0.99,
                               num_epochs=3, normalize_rewards=False,
                               normalize_observations=False,
                               compute_value_and_advantage_in_train=value_in_train, **kl_kw)
  oa, ov = _mirror(actor), _mirror(value)
  okw = dict(num_epochs=3, clip_eps=0.2, vf_coef=0.5, gamma=0.99, lam=0.95, **kl_kw)
  opt = ooptim.AdamTF(1e-3, eps=1e-7)
  if discrete:
    orc = oppod.CategoricalPPOOracle(oa, ov, opt, **okw)
  else:
    orc = oppo.PPOOracle(oa, actor._std.bias.cpu().numpy().copy(), ov, -np.ones(A, f32),
                         np.ones(A, f32), opt, **okw)
  tag = 'ppo_rnn_train_%s' % ('discrete' if discrete else 'normal')
  for it in range(2):
    e = _experience(rng, B, T, D, A, discrete)
    oa.step_type = e['step_type']
    if rnn_value:
      ov.step_type = e['step_type']
    if value_in_train:
      want = orc.train(e)[-1]
      got = agent.train(_to_traj(cuda, e))
    else:
      want = orc.train(orc.preprocess_sequence(e), preprocessed=True)[-1]
      got = agent.train(agent.preprocess_sequence(_to_traj(cuda, e, with_value=True)))
    record_parity(tag, loss_rel=abs(got.loss.item() - want['loss']) / abs(want['loss']))
    np.testing.assert_allclose(got.loss.item(), want['loss'], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(got.extra.policy_gradient_loss.item(), want['pg'], rtol=1e-5,
                               atol=1e-6)
    np.testing.assert_allclose(got.extra.value_estimation_loss.item(), want['ve'], rtol=1e-5)
    np.testing.assert_allclose(got.extra.kl_penalty_loss.item(), want['kl'], rtol=1e-5, atol=1e-7)
    if kl:
      np.testing.assert_allclose(agent._adaptive_kl_beta.item(), orc.beta, rtol=1e-6)
  for v, w in zip(actor.variables + value.variables, orc.params()):
    np.testing.assert_allclose(v.cpu().numpy(), w, rtol=2e-3, atol=2e-5)
  assert int(agent.train_step_counter.item()) == 6
  agent.check_numerics()


# ---- gradients before the optimiser against float64 ---------------------------------------------
class RecordingOptimizer(optimizers.Optimizer):
  """Keeps a copy of every gradient it is handed; the parameters do not move."""

  def __init__(self):
    super().__init__()
    self.calls = []

  def apply_flat(self, params, grads, grad_scale=None):
    self.calls.append(grads.clone())


def _views(net):
  out = []
  for l in net.layers:
    for n in ('d_kernel', 'd_recurrent_kernel', 'd_bias'):
      g = getattr(l, n, None)
      if g is not None:
        out.append(g)
  return out


def _rnn64(net, x, step_type):
  """float64 torch forward of an LSTMEncodingNetwork-based net over [B*T, D] rows; returns
  (output of the last Dense, leaf parameters in net.variables order)."""
  B, T = step_type.shape
  leaves = []
  p = lambda t: leaves.append(R.t64(t).requires_grad_()) or leaves[-1]
  for l in net._pre:
    x = R.activate(x @ p(l.kernel) + p(l.bias), l.activation)
  for c in net._cells:
    W, U, b = p(c.kernel), p(c.recurrent_kernel), p(c.bias)
    H = c.units
    xw = (x @ W + b).reshape(B, T, 4 * H)
    h = torch.zeros(B, H, dtype=torch.float64)
    cc = torch.zeros(B, H, dtype=torch.float64)
    hs = []
    for t in range(T):
      keep = torch.as_tensor(step_type[:, t] != 0, dtype=torch.float64)[:, None]
      h, cc = h * keep, cc * keep
      z = xw[:, t] + h @ U
      i, f = torch.sigmoid(z[:, :H]), torch.sigmoid(z[:, H:2 * H])
      g, o = torch.tanh(z[:, 2 * H:3 * H]), torch.sigmoid(z[:, 3 * H:])
      cc = f * cc + i * g
      h = o * torch.tanh(cc)
      hs.append(h)
    x = torch.stack(hs, 1).reshape(B * T, H)
  for l in net._post:
    if isinstance(l, L.Dense):
      x = R.activate(x @ p(l.kernel) + p(l.bias), l.activation)
  return x, leaves


@pytest.mark.parametrize('kl', [False, True])
def test_recurrent_ppo_gradients_match_float64(cuda, kl):
  rng = np.random.RandomState(41 + kl)
  B, T, D, A = 5, 19, 7, 3
  N = B * T
  opt = RecordingOptimizer()
  kl_kw = KL_KW if kl else NO_KL_KW
  ent, l2a, l2v = 0.01, 0.01, 0.02
  agent, actor, value = _build(cuda, D, A, True, optimizer=opt, importance_ratio_clipping=0.2,
                               use_gae=True, lambda_value=0.95, discount_factor=0.99,
                               num_epochs=1, normalize_rewards=False,
                               normalize_observations=False, entropy_regularization=ent,
                               policy_l2_reg=l2a, value_function_l2_reg=l2v, **kl_kw)
  with torch.no_grad():
    actor._std.bias.copy_(torch.as_tensor(rng.randn(A) * 0.5, dtype=torch.float32))
  e = _experience(rng, B, T, D, A)
  agent.train(_to_traj(cuda, e))
  assert len(opt.calls) == 1
  # targets as the oracle computes them (the value pass of preprocessing is covered above)
  ov = _mirror(value)
  ov.step_type = e['step_type']
  orc = oppo.PPOOracle(None, np.zeros(1, f32), ov, np.zeros(1, f32), np.ones(1, f32), None,
                       gamma=0.99, lam=0.95)
  vp, ret, adv = orc.preprocess(e)
  w = oppo.make_trajectory_mask(e['step_type'], ret, adv).reshape(-1)
  old_loc, old_scale = e['loc'].reshape(N, A), e['scale'].reshape(N, A)
  action = e['action'].reshape(N, A)
  old_logp = oppo.normal_log_prob(old_loc, old_scale, action)
  adv_n = oppo.normalize_advantages(adv).reshape(-1)
  o64 = R.t64(e['observation'].reshape(N, D))
  m_raw, a_leaves = _rnn64(actor, o64, e['step_type'])
  std64 = R.t64(actor._std.bias).requires_grad_()
  v, v_leaves = _rnn64(value, o64, e['step_type'])
  amin, amax = R.t64(-np.ones(A)), R.t64(np.ones(A))
  loc64, scale64 = R.normal_projection(m_raw, std64, amin, amax)
  loss = R.ppo_loss(R.normal_log_prob(loc64, scale64, R.t64(action)), R.normal_entropy(scale64),
                    R.t64(old_logp), R.t64(adv_n), R.t64(ret.reshape(-1)), v[:, 0],
                    R.t64(vp.reshape(-1)), R.t64(w), float(N), 0.2, 0.0, 0.5, ent)
  if kl:
    kl64 = R.normal_kl(R.t64(old_loc), R.t64(old_scale), loc64, scale64)
    loss = loss + R.kl_penalty(kl64, R.t64(w), float(N), KL_KW['kl_cutoff_factor'],
                               KL_KW['adaptive_kl_target'], KL_KW['kl_cutoff_coef'],
                               KL_KW['initial_adaptive_kl_beta'])
  loss = (loss + R.l2_loss([t for t in a_leaves if t.dim() == 2], l2a)
          + R.l2_loss([t for t in v_leaves if t.dim() == 2], l2v))
  a_ref = a_leaves + [std64]
  g_ref = torch.autograd.grad(loss, a_ref + v_leaves)
  views = _views(actor) + _views(value)
  base = agent._flat_grads.data_ptr()
  rec = opt.calls[0]
  for k, (view, ref) in enumerate(zip(views, g_ref)):
    off = (view.data_ptr() - base) // 4
    got = rec[off:off + view.numel()].reshape(view.shape)
    err = R.grad_errors(got, ref)
    record_parity('ppo_rnn_grads_float64', rel_l2=err[0], rel_max=err[1])
    R.assert_grad_close(f'variable {k}', got, ref, 1e-4, 1e-4)


def test_recurrent_collect_policy_state_and_reset(cuda):
  agent, actor, value = _build(cuda, 5, 2, True, importance_ratio_clipping=0.2, use_gae=True,
                               compute_value_and_advantage_in_train=False)
  pol = agent.collect_policy
  assert set(pol.policy_state_spec) == {'actor_network_state', 'value_network_state'}
  assert set(agent.policy.policy_state_spec) == {'actor_network_state'}
  B = 4
  state = pol.get_initial_state(B)
  obs = torch.randn(B, 5, device=cuda)
  mid = torch.ones(B, dtype=torch.int32, device=cuda)
  first = torch.zeros(B, dtype=torch.int32, device=cuda)
  step = lambda st, s: pol.action(ts.TimeStep(st, torch.zeros(B, device=cuda),
                                              torch.ones(B, device=cuda), obs), s)
  a1 = step(first, state)
  a2 = step(mid, a1.state)
  assert not torch.equal(a1.info['dist_params']['loc'], a2.info['dist_params']['loc'])
  # FIRST resets: the step from a non-zero state equals the step from the initial state
  a3 = step(first, a2.state)
  assert torch.equal(a3.info['dist_params']['loc'], a1.info['dist_params']['loc'])
  assert torch.equal(a3.info['value_prediction'], a1.info['value_prediction'])
  for x, y in zip(torch.utils._pytree.tree_leaves(a3.state), torch.utils._pytree.tree_leaves(a1.state)):
    assert torch.equal(x, y)


def test_learner_rejects_minibatches_for_recurrent_networks(cuda):
  from agents_b200.train import ppo_learner
  agent, _, _ = _build(cuda, 5, 2, False, importance_ratio_clipping=0.2, use_gae=True,
                       compute_value_and_advantage_in_train=False, update_normalizers_in_train=False)
  with pytest.raises(ValueError, match='RNN'):
    ppo_learner.PPOLearner('/nonexistent', None, agent, lambda: None, lambda: None, 1,
                           minibatch_size=4, shuffle_buffer_size=4)


def _stateful_net(cuda, spec):
  return len_.LSTMEncodingNetwork(spec, input_fc_layer_params=(8,), lstm_size=(4,),
                                  output_fc_layer_params=(), device=cuda)


def test_dqn_agent_rejects_stateful_network(cuda):
  spec = tensor_spec.TensorSpec((3,), torch.float32)
  act = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 1)
  with pytest.raises(NotImplementedError, match='feed-forward'):
    dqn_agent.DqnAgent(ts.time_step_spec(spec), act, q_network=_stateful_net(cuda, spec),
                       optimizer=optimizers.Adam(1e-3))


def test_sac_agent_rejects_stateful_network(cuda):
  spec = tensor_spec.TensorSpec((3,), torch.float32)
  act = tensor_spec.BoundedTensorSpec((2,), torch.float32, -1.0, 1.0)
  with pytest.raises(NotImplementedError, match='feed-forward'):
    sac_agent.SacAgent(ts.time_step_spec(spec), act, critic_network=_stateful_net(cuda, spec),
                       actor_network=_stateful_net(cuda, spec), actor_optimizer=None,
                       critic_optimizer=None, alpha_optimizer=None)


def test_cql_sac_agent_rejects_stateful_network(cuda):
  spec = tensor_spec.TensorSpec((3,), torch.float32)
  act = tensor_spec.BoundedTensorSpec((2,), torch.float32, -1.0, 1.0)
  with pytest.raises(NotImplementedError, match='feed-forward'):
    cql_sac_agent.CqlSacAgent(ts.time_step_spec(spec), act,
                              critic_network=_stateful_net(cuda, spec),
                              actor_network=_stateful_net(cuda, spec), actor_optimizer=None,
                              critic_optimizer=None, alpha_optimizer=None, cql_alpha=1.0,
                              num_cql_samples=1, include_critic_entropy_term=False,
                              use_lagrange_cql_alpha=False)


# ---- capture, restore and the reference's RNN train flow ------------------------------------------
def _leaves(x):
  return torch.utils._pytree.tree_leaves(x)


@pytest.fixture
def ffma():
  """FP32 FFMA GEMMs, whose deterministic split-K makes weight gradients bit-reproducible (the
  tensor-core weight-gradient GEMMs add split-K partials with floating-point atomics)."""
  _lib.call('b200rl_set_gemm_mode', 0)
  try:
    yield
  finally:
    _lib.call('b200rl_set_gemm_mode', 1)


def _collect_setup(cuda, B, value_in_train):
  obs_spec, act_spec = _specs(4, 2, False)
  agent, _, _ = _build(cuda, 4, 2, True, importance_ratio_clipping=0.2, use_gae=True,
                       compute_value_and_advantage_in_train=value_in_train)
  env = random_tf_environment.RandomTFEnvironment(ts.time_step_spec(obs_spec), act_spec,
                                                  batch_size=B, episode_end_probability=0.2,
                                                  seed=3, device=cuda)
  rb = rb_mod.TFUniformReplayBuffer(agent.collect_data_spec, batch_size=B, max_length=64,
                                    device=cuda)
  driver = dynamic_step_driver.DynamicStepDriver(env, agent.collect_policy,
                                                 observers=[rb.add_batch], num_steps=B * 4)
  return agent, env, rb, driver


@pytest.mark.parametrize('value_in_train', [True, False])
def test_stateful_collect_graph_replays_bit_for_bit(cuda, value_in_train):
  """DynamicStepDriver with the recurrent collect policy (its state threaded through the driver,
  resets at FIRST): 12 runs of 4 steps captured into one CUDA graph store the same trajectories,
  bit for bit, as 12 eager runs."""
  B = 8
  out = []
  for graphed in (False, True):
    agent, env, rb, driver = _collect_setup(cuda, B, value_in_train)
    run = lambda t, s: driver.run(t, s, maximum_iterations=4)
    if graphed:
      run = common.function(run)
    time_step, state = env.reset(), agent.collect_policy.get_initial_state(B)
    for _ in range(12):
      time_step, state = run(time_step, state)
    exp = rb.gather_all()
    out.append([t.clone() for t in _leaves(exp)] + [t.clone() for t in _leaves(state)])
  assert int((out[0][0] == 0).sum()) > B          # several episodes started inside the window
  for a, b in zip(*out):
    assert torch.equal(a, b)


def test_train_graph_replays_bit_for_bit(cuda, ffma):
  rng = np.random.RandomState(6)
  B, T, D, A = 4, 16, 5, 3
  make = lambda: _build(cuda, D, A, True, importance_ratio_clipping=0.2, use_gae=True,
                        num_epochs=2, normalize_observations=False, normalize_rewards=False,
                        **KL_KW)[0]
  eager, graphed = make(), make()
  train_fn = common.function(graphed.train)
  for _ in range(5):
    traj = _to_traj(cuda, _experience(rng, B, T, D, A))
    l1 = eager.train(traj).loss.item()
    l2 = train_fn(traj).loss.item()
    assert l1 == l2
  assert torch.equal(graphed._flat_params, eager._flat_params)
  assert torch.equal(graphed._adaptive_kl_beta, eager._adaptive_kl_beta)


def test_ppo_learner_restores_bit_for_bit_with_full_sequences(cuda, tmp_path, ffma):
  """PPOLearner over full [B, T] sequences checkpoints after every train step; a learner built
  over a fresh agent restores it and reproduces the original's next run bit for bit."""
  rng = np.random.RandomState(8)
  B, T, D, A = 4, 12, 5, 2
  make = lambda seed: _build(cuda, D, A, True, importance_ratio_clipping=0.2, use_gae=True,
                             num_epochs=1, normalize_observations=False, normalize_rewards=False,
                             update_normalizers_in_train=False, **KL_KW)[0]
  exps = [_to_traj(cuda, _experience(rng, B, T, D, A)) for _ in range(2)]
  ds_of = lambda agent: (lambda: iter([(e, ()) for e in exps]))
  a1 = make(0)
  l1 = ppo_learner.PPOLearner(str(tmp_path / 'run'), a1.train_step_counter, a1, ds_of(a1),
                              ds_of(a1), num_samples=2, num_epochs=2, checkpoint_interval=1)
  l1.run()
  a2 = make(1)
  with torch.no_grad():
    a2._flat_params.add_(1.0)                      # differs until restored
  l2 = ppo_learner.PPOLearner(str(tmp_path / 'run'), a2.train_step_counter, a2, ds_of(a2),
                              ds_of(a2), num_samples=2, num_epochs=2, checkpoint_interval=0)
  assert int(a2.train_step_counter.item()) == int(a1.train_step_counter.item()) == 4
  for k, v in learner_lib._agent_state_tensors(a1).items():
    assert torch.equal(learner_lib._agent_state_tensors(a2)[k], v), k
  i1, i2 = l1.run(), l2.run()
  assert i1.loss.item() == i2.loss.item()
  assert torch.equal(a1._flat_params, a2._flat_params)


def test_reference_rnn_train_flow(cuda):
  """ppo_agent_test.py testRNNTrain: recurrent actor (LSTM 20) and value (LSTM 10) without fc
  layers, one episode of a RandomTFEnvironment through DynamicEpisodeDriver into a
  TFUniformReplayBuffer(max_length=7), train, and the step counter is 1.  The episode is
  collected with the agent's recurrent collect policy (the reference uses a RandomTFPolicy that
  fills the collect policy's info_spec)."""
  obs_spec = tensor_spec.TensorSpec((2,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((1,), torch.float32, -1.0, 1.0, 'action')
  tss = ts.time_step_spec(obs_spec)
  actor = adrn.ActorDistributionRnnNetwork(obs_spec, act_spec, input_fc_layer_params=None,
                                           output_fc_layer_params=None, lstm_size=(20,),
                                           device=cuda)
  value = vrn.ValueRnnNetwork(obs_spec, input_fc_layer_params=None, output_fc_layer_params=None,
                              lstm_size=(10,), device=cuda)
  agent = ppo_agent.PPOAgent(tss, act_spec, optimizer=optimizers.Adam(1e-3), actor_net=actor,
                             value_net=value, num_epochs=1, use_gae=True)
  agent.initialize()
  env = random_tf_environment.RandomTFEnvironment(tss, act_spec, batch_size=1, seed=2,
                                                  device=cuda)
  rb = rb_mod.TFUniformReplayBuffer(agent.collect_policy.trajectory_spec, batch_size=1,
                                    max_length=7, device=cuda)
  driver = dynamic_episode_driver.DynamicEpisodeDriver(env, agent.collect_policy,
                                                       observers=[rb.add_batch], num_episodes=1)
  assert int(agent.train_step_counter.item()) == 0
  driver.run()
  agent.train(rb.gather_all())
  assert int(agent.train_step_counter.item()) == 1
  agent.check_numerics()


# ---- learning: a task that needs memory -----------------------------------------------------------
CUE_STEPS = 3          # decisions per episode; the cue is visible at the first only


def _cue_episode(policy, cuda, cue):
  """One batch of cue-recall episodes: observation (cue, 1) at the FIRST step and (0, 0) after;
  reward 1 when the action of the last decision equals (cue > 0).  Returns the [B, CUE_STEPS + 1]
  trajectory (its last column the LAST boundary step) and the last decision's actions."""
  B = cue.shape[0]
  state = policy.get_initial_state(B)
  zeros = torch.zeros(B, 2, device=cuda)
  obs0 = torch.stack([cue, torch.ones_like(cue)], 1)
  cols = dict(step_type=[], observation=[], action=[], info=[], reward=[], discount=[],
              next_step_type=[])
  last = None
  for t in range(CUE_STEPS + 1):
    st = 0 if t == 0 else (2 if t == CUE_STEPS else 1)
    step_type = torch.full((B,), st, dtype=torch.int32, device=cuda)
    obs = obs0 if t == 0 else zeros
    step = policy.action(ts.TimeStep(step_type, torch.zeros(B, device=cuda),
                                     torch.ones(B, device=cuda), obs), state)
    state = step.state
    if t == CUE_STEPS - 1:
      last = step.action
    done = t == CUE_STEPS - 1
    reward = (step.action == (cue > 0).to(step.action.dtype)).float() if done else \
        torch.zeros(B, device=cuda)
    cols['step_type'].append(step_type)
    cols['observation'].append(obs)
    cols['action'].append(step.action)
    cols['info'].append(step.info)
    cols['reward'].append(reward)
    cols['discount'].append(torch.zeros(B, device=cuda) if done else torch.ones(B, device=cuda))
    nxt = 2 if t == CUE_STEPS - 1 else (0 if t == CUE_STEPS else 1)
    cols['next_step_type'].append(torch.full((B,), nxt, dtype=torch.int32, device=cuda))
  stk = lambda xs: torch.stack(xs, 1)
  info = {'dist_params': {'logits': stk([i['dist_params']['logits'] for i in cols['info']])}} \
      if cols['info'][0] else ()
  traj = trajectory.Trajectory(stk(cols['step_type']), stk(cols['observation']),
                               stk(cols['action']), info, stk(cols['next_step_type']),
                               stk(cols['reward']), stk(cols['discount']))
  return traj, last


def _cue_accuracy(recurrent, seed):
  cuda = torch.device('cuda')
  torch.manual_seed(seed)
  obs_spec = tensor_spec.TensorSpec((2,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 1, 'action')
  if recurrent:
    actor = adrn.ActorDistributionRnnNetwork(obs_spec, act_spec, input_fc_layer_params=(32,),
                                             lstm_size=(16,), output_fc_layer_params=(32,),
                                             device=cuda).set_seed(seed)
    value = vrn.ValueRnnNetwork(obs_spec, input_fc_layer_params=(32,), lstm_size=(16,),
                                output_fc_layer_params=(32,), device=cuda).set_seed(seed + 1)
  else:
    from agents_b200.networks import actor_distribution_network as adn
    actor = adn.ActorDistributionNetwork(obs_spec, act_spec, fc_layer_params=(32, 32),
                                         device=cuda).set_seed(seed)
    value = value_network.ValueNetwork(obs_spec, fc_layer_params=(32, 32),
                                       device=cuda).set_seed(seed + 1)
  agent = ppo_clip_agent.PPOClipAgent(ts.time_step_spec(obs_spec), act_spec,
                                      optimizer=optimizers.Adam(3e-3), actor_net=actor,
                                      value_net=value, importance_ratio_clipping=0.2,
                                      use_gae=True, num_epochs=4, discount_factor=1.0,
                                      lambda_value=0.95, normalize_observations=False,
                                      normalize_rewards=False, seed=seed)
  agent.initialize()
  gen = torch.Generator(device='cpu').manual_seed(seed)
  cue_of = lambda n: (torch.randint(0, 2, (n,), generator=gen).float() * 2 - 1).to(cuda)
  for _ in range(200):
    traj, _ = _cue_episode(agent.collect_policy, cuda, cue_of(64))
    agent.train(traj)
  agent.check_numerics()
  cue = cue_of(1024)
  _, last = _cue_episode(agent.policy, cuda, cue)
  return float((last == (cue > 0).to(last.dtype)).float().mean())


def test_cue_recall_needs_memory(cuda):
  """A +-1 cue at the first step, zeros after it, and a reward for matching the cue's sign at the
  last of three decisions: recurrent PPO learns it, feed-forward PPO cannot do better than
  chance (its observation at the last decision carries no information)."""
  rnn = _cue_accuracy(True, 0)
  ff = _cue_accuracy(False, 0)
  record_parity('ppo_rnn_cue_recall', recurrent_accuracy=rnn, feed_forward_accuracy=ff)
  assert rnn > 0.9, rnn
  assert abs(ff - 0.5) < 0.1, ff
