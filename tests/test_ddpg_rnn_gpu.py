"""Recurrent DDPG on the GPU: the b200rl_ddpg_seq_critic_loss / b200rl_ddpg_seq_actor_loss kernels
against float64, ActorRnnNetwork and CriticRnnNetwork (structure, state, sequence vs chained steps,
copies, gradients and the input-only dQ/da against float64 autograd), DdpgAgent on them against the
numpy oracle (tests/ddpg_rnn_oracle.py) and float64 autograd, CUDA-graph replays, a Learner restore,
the stateful actor policies, the reference train_eval_rnn flow, and a cue-recall task only a
recurrent agent can solve."""
import numpy as np
import pytest
import torch

from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.agents.ddpg import ddpg_agent
from agents_b200.agents.sac import sac_agent
from agents_b200.agents.td3 import td3_agent
from agents_b200.drivers import dynamic_episode_driver
from agents_b200.drivers import dynamic_step_driver
from agents_b200.environments import random_tf_environment
from agents_b200.networks import actor_network
from agents_b200.networks import actor_rnn_network
from agents_b200.networks import critic_network
from agents_b200.networks import critic_rnn_network
from agents_b200.networks import lstm_encoding_network
from agents_b200.replay_buffers import tf_uniform_replay_buffer as rb_mod
from agents_b200.specs import tensor_spec
from agents_b200.train import learner as learner_lib
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory
from agents_b200.utils import common
from oracle import ddpg as oddpg
from oracle import lstm as olstm
from oracle import optim as ooptim

import ddpg_rnn_oracle as O
import test_oracle_ddpg_rnn as H

from conftest import record_parity

pytestmark = pytest.mark.gpu
f32 = np.float32
FIRST, MID, LAST = 0, 1, 2


@pytest.fixture
def ffma():
  """FP32 FFMA GEMMs, whose deterministic split-K makes weight gradients bit-reproducible (the
  tensor-core weight-gradient GEMMs add split-K partials with floating-point atomics)."""
  _lib.call('b200rl_set_gemm_mode', 0)
  try:
    yield
  finally:
    _lib.call('b200rl_set_gemm_mode', 1)


def _leaves(x):
  return torch.utils._pytree.tree_leaves(x)


def _rel(got, ref):
  got, ref = np.asarray(got, np.float64).reshape(-1), np.asarray(ref, np.float64).reshape(-1)
  m, d = np.abs(ref).max(), np.abs(got - ref).max()
  return d / m if m > 0 else d


# ---- the kernels --------------------------------------------------------------------------------
class Scratch(object):
  def __init__(self, cuda):
    self.partials = torch.empty(_lib.DDPG_SEQ_MAX_BLOCKS, dtype=torch.float32, device=cuda)
    self.ticket = torch.zeros(1, dtype=torch.int32, device=cuda)
    self.nan_flag = torch.zeros(1, dtype=torch.int32, device=cuda)


def _critic_call(s, q, tq, r, d, w, w_stride, B, T, gamma, scale, kind):
  loss, dq = torch.empty(1, device=q.device), torch.empty_like(q)
  _lib.call('b200rl_ddpg_seq_critic_loss', _lib.ptr(q), _lib.ptr(tq), _lib.dptr(r), _lib.dptr(d),
            r.stride(0), r.stride(1), _lib.ptr(w), w_stride, B, T, gamma, scale, kind,
            _lib.ptr(loss), _lib.ptr(dq), _lib.ptr(s.nan_flag), _lib.ptr(s.partials),
            _lib.ptr(s.ticket), _lib.stream())
  return loss, dq


def _actor_call(s, dqda, w, w_stride, B, T, A, clip, amin, amax):
  loss, dy = torch.empty(1, device=dqda.device), torch.empty((B * (T - 1), A), device=dqda.device)
  _lib.call('b200rl_ddpg_seq_actor_loss', _lib.dptr(dqda), dqda.stride(0), _lib.ptr(w), w_stride,
            B, T, A, int(clip is not None), 0.0 if clip is None else float(clip), _lib.ptr(amin),
            _lib.ptr(amax), _lib.ptr(loss), _lib.ptr(dy), _lib.ptr(s.nan_flag),
            _lib.ptr(s.partials), _lib.ptr(s.ticket), _lib.stream())
  return loss, dy


KERNEL_SHAPES = [(1, 1, 1), (3, 7, 6), (64, 10, 1), (64, 33, 21), (1000, 7, 6), (1000, 1000, 1),
                 (5000, 10, 6), (5000, 33, 1), (3, 1000, 21), (5000, 1, 21), (1, 33, 6)]
VARIANTS = [(_lib.LOSS_HUBER, None, None), (_lib.LOSS_SQUARED, 'scalar', 0.0),
            (_lib.LOSS_HUBER, 'row', 0.5), (_lib.LOSS_SQUARED, 'row', None)]


@pytest.mark.parametrize('B,Tm,A', KERNEL_SHAPES)
@pytest.mark.parametrize('variant', range(len(VARIANTS)))
def test_seq_kernels_match_float64(cuda, B, Tm, A, variant):
  kind, wmode, clip = VARIANTS[variant]
  rng = np.random.default_rng(B * 131 + Tm * 7 + A + variant)
  T, N = Tm + 1, B * Tm
  q = rng.normal(size=N).astype(f32) * 2
  tq = rng.normal(size=N).astype(f32) * 2
  # reward / discount read in place from [B, T] columns of a wider buffer
  rd = rng.normal(size=(B, T + 3)).astype(f32)
  dd = rng.uniform(0, 1, (B, T + 3)).astype(f32)
  w = {None: None, 'scalar': np.array([0.7], f32), 'row': rng.uniform(0, 2, B).astype(f32)}[wmode]
  dqda = rng.normal(size=(N, A + 2)).astype(f32)
  amin = rng.uniform(-2, 0, A).astype(f32)
  amax = amin + rng.uniform(0.5, 2, A).astype(f32)
  s = Scratch(cuda)
  d = lambda a: torch.as_tensor(a, device=cuda)   # noqa: E731
  r_t, d_t = d(rd)[:, :T], d(dd)[:, :T]
  w_t, ws = (None, 0) if w is None else (d(w), int(w.size > 1))
  runs = [(_critic_call(s, d(q), d(tq), r_t, d_t, w_t, ws, B, T, 0.9, 1.5, kind),
           _actor_call(s, d(dqda)[:, 1:1 + A], w_t, ws, B, T, A, clip, d(amin), d(amax)))
          for _ in range(2)]
  (closs, dq), (aloss, dy) = runs[0]
  for x, y in zip(_leaves(runs[0]), _leaves(runs[1])):
    assert torch.equal(x, y)
  assert int(s.ticket.item()) == 0 and int(s.nan_flag.item()) == 0
  # float64
  wb = np.ones(B) if w is None else np.broadcast_to(w.astype(np.float64), (B,))
  y = 1.5 * rd[:, :Tm].astype(np.float64).reshape(-1) + 0.9 * dd[:, :Tm].reshape(-1) * tq
  e = y - q
  l = np.where(np.abs(e) <= 1, 0.5 * e * e, np.abs(e) - 0.5) if kind == _lib.LOSS_HUBER else e * e
  g = -np.clip(e, -1, 1) if kind == _lib.LOSS_HUBER else -2 * e
  closs64 = (l.reshape(B, Tm).sum(1) * wb).sum() / B
  dq64 = g * np.repeat(wb, Tm) / B
  c = dqda[:, 1:1 + A].astype(np.float64)
  if clip is not None:
    c = np.clip(c, -clip, clip)
  wr = np.repeat(wb, Tm)[:, None]
  aloss64 = (wr * c * c).sum() / (B * A)
  dy64 = 0.5 * (amax - amin).astype(np.float64) * (-2 * wr * c / (B * A))
  errs = dict(critic_loss=abs(closs.item() - closs64) / max(abs(closs64), 1e-30),
              dq=_rel(dq.cpu(), dq64),
              actor_loss=abs(aloss.item() - aloss64) / max(abs(aloss64), 1e-30) if aloss64 else
              abs(aloss.item()), dy=_rel(dy.cpu(), dy64))
  record_parity('ddpg_seq_loss_float64', **errs)
  for k, v in errs.items():
    assert v <= 1e-6, (k, v)


@pytest.mark.parametrize('B,A', [(7, 6), (256, 1), (5000, 21)])
@pytest.mark.parametrize('kind', [_lib.LOSS_HUBER, _lib.LOSS_SQUARED])
def test_one_transition_matches_feed_forward_kernels(cuda, B, A, kind):
  """At T-1 = 1, dq and dy are the feed-forward kernels' bits; the losses agree to a few ulps."""
  rng = np.random.default_rng(B + A)
  d = lambda a: torch.as_tensor(a, device=cuda)   # noqa: E731
  q, tq = d(rng.normal(size=B).astype(f32) * 2), d(rng.normal(size=B).astype(f32) * 2)
  r2, d2 = d(rng.normal(size=(B, 2)).astype(f32)), d(rng.uniform(0, 1, (B, 2)).astype(f32))
  w = d(rng.uniform(0, 2, B).astype(f32))
  dqda = d(rng.normal(size=(B, A)).astype(f32))
  amin, amax = d(np.full(A, -2, f32)), d(np.full(A, 1, f32))
  s = Scratch(cuda)
  closs, dq = _critic_call(s, q, tq, r2, d2, w, 1, B, 2, 0.99, 0.5, kind)
  aloss, dy = _actor_call(s, dqda, w, 1, B, 2, A, 0.5, amin, amax)
  fl, fdq = torch.empty(1, device=cuda), torch.empty(B, device=cuda)
  r, dc = r2[:, 0].contiguous(), d2[:, 0].contiguous()
  _lib.call('b200rl_ddpg_critic_loss', _lib.ptr(q), _lib.ptr(tq), _lib.ptr(r), _lib.ptr(dc),
            _lib.ptr(w), B, 0.99, 0.5, kind, _lib.ptr(fl), _lib.ptr(fdq), None, None, _lib.stream())
  fa, fdy = torch.empty(1, device=cuda), torch.empty(B, A, device=cuda)
  _lib.call('b200rl_ddpg_actor_loss', _lib.ptr(dqda), A, _lib.ptr(w), B, A, 1, 0.5,
            _lib.ptr(amin), _lib.ptr(amax), _lib.ptr(fa), _lib.ptr(fdy), None, _lib.stream())
  assert torch.equal(dq, fdq) and torch.equal(dy, fdy)
  for a, b in ((closs, fl), (aloss, fa)):
    assert abs(a.item() - b.item()) <= 8 * np.spacing(np.float32(abs(b.item())))


# ---- networks -----------------------------------------------------------------------------------
def _img_specs():
  return (tensor_spec.BoundedTensorSpec((8, 8, 3), torch.float32, 0, 1),
          tensor_spec.BoundedTensorSpec((2,), torch.float32, 2, 3))


def test_critic_rnn_network_builds_like_the_reference(cuda):
  """critic_rnn_network_test.py testBuilds: 15 variables with conv, observation, action, joint,
  LSTM and output layers; the [h, c] state named network_state_0 / _1."""
  obs_spec, act_spec = _img_specs()
  net = critic_rnn_network.CriticRnnNetwork(
      (obs_spec, act_spec), observation_conv_layer_params=[(4, 2, 2)],
      observation_fc_layer_params=(4,), action_fc_layer_params=(5,), joint_fc_layer_params=(5,),
      lstm_size=(3,), output_fc_layer_params=(5,), device=cuda)
  obs = torch.rand(1, 8, 8, 3, device=cuda)
  act = 2 + torch.rand(1, 2, device=cuda)
  q, state = net((obs, act), torch.zeros(1, dtype=torch.int32, device=cuda),
                 net.get_initial_state(batch_size=1))
  assert tuple(q.shape) == (1,)
  assert [tuple(v.shape) for v in net.variables] == [
      (2, 2, 3, 4), (4,), (64, 4), (4,), (2, 5), (5,), (9, 5), (5,), (5, 12), (3, 12), (12,),
      (3, 5), (5,), (5, 1), (1,)]
  assert isinstance(state, list) and [tuple(s.shape) for s in state] == [(1, 3), (1, 3)]
  assert [s.name for s in net.state_spec] == ['network_state_0', 'network_state_1']
  assert float(net._post[-1].kernel.abs().max()) <= 0.003
  with pytest.raises(ValueError):
    critic_rnn_network.CriticRnnNetwork((obs_spec, act_spec), device=cuda)
  with pytest.raises(NotImplementedError):
    critic_rnn_network.CriticRnnNetwork((obs_spec, act_spec), rnn_construction_fn=lambda: None,
                                        device=cuda)
  # the reference's default init (testInit) and the example's action_fc None
  critic_rnn_network.CriticRnnNetwork((obs_spec, act_spec), observation_conv_layer_params=[
      (4, 2, 2)], lstm_size=(3,), device=cuda).create_variables()
  n = critic_rnn_network.CriticRnnNetwork((tensor_spec.TensorSpec((3,), torch.float32), act_spec),
                                          action_fc_layer_params=None, lstm_size=(3, 4),
                                          device=cuda)
  q, state = n((torch.rand(2, 3, device=cuda), act.expand(2, 2)), None, n.get_initial_state(2))
  assert tuple(q.shape) == (2,) and isinstance(state, tuple) and len(state) == 2
  assert [s.name for s in _leaves(n.state_spec)] == ['network_state_%d' % i for i in range(4)]


def test_actor_rnn_network_builds_like_the_reference(cuda):
  """actor_rnn_network_test.py testBuilds / testActionsWithinRange with one action: 11 variables,
  the [h, c] state, actions inside the spec."""
  obs_spec, act_spec = _img_specs()
  net = actor_rnn_network.ActorRnnNetwork(obs_spec, act_spec, conv_layer_params=[(4, 2, 2)],
                                          input_fc_layer_params=(5,), lstm_size=(3,),
                                          output_fc_layer_params=(5,), device=cuda)
  obs = torch.rand(1, 8, 8, 3, device=cuda)
  actions, state = net(obs, torch.zeros(1, dtype=torch.int32, device=cuda),
                       net.get_initial_state(batch_size=1))
  assert tuple(actions.shape) == (1, 2)
  assert [tuple(v.shape) for v in net.variables] == [
      (2, 2, 3, 4), (4,), (64, 5), (5,), (5, 12), (3, 12), (12,), (3, 5), (5,), (5, 2), (2,)]
  assert isinstance(state, list) and [tuple(s.shape) for s in state] == [(1, 3), (1, 3)]
  assert [s.name for s in net.state_spec] == ['network_state_spec'] * 2
  big = actor_rnn_network.ActorRnnNetwork(obs_spec, act_spec, conv_layer_params=[(4, 2, 2)],
                                          input_fc_layer_params=(5,), lstm_size=(3,),
                                          output_fc_layer_params=(5,), device=cuda).set_seed(3)
  with torch.no_grad():
    big.create_variables()
    big._post[-1].kernel.mul_(3000.0)     # saturate the tanh
  a, _ = big(torch.rand(64, 5, 8, 8, 3, device=cuda) * 4)
  assert float(a.min()) >= 2.0 and float(a.max()) <= 3.0
  assert float(net._post[-1].kernel.abs().max()) <= 0.003


def _seq_inputs(cuda, rng, B, T, D, A):
  st = np.ones((B, T), np.int32)
  st[:, 0] = FIRST
  st[1, 5] = FIRST
  st[2, 3] = LAST
  st[2, 4] = FIRST
  d = lambda a: torch.as_tensor(a, device=cuda)   # noqa: E731
  return (d(rng.normal(size=(B, T, D)).astype(f32)), d(rng.uniform(-1, 1, (B, T, A)).astype(f32)),
          d(st))


def _small_nets(cuda, D, A, action_fc=(6,), seed=0):
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, -1.0, 2.0, 'action')
  actor = actor_rnn_network.ActorRnnNetwork(obs_spec, act_spec, input_fc_layer_params=(16,),
                                            lstm_size=(8,), output_fc_layer_params=(12,),
                                            device=cuda).set_seed(seed + 1)
  critic = critic_rnn_network.CriticRnnNetwork(
      (obs_spec, act_spec), observation_fc_layer_params=(10,), action_fc_layer_params=action_fc,
      joint_fc_layer_params=(12,), lstm_size=(8,), output_fc_layer_params=(9,),
      device=cuda).set_seed(seed + 2)
  actor.create_variables()
  critic.create_variables()
  return obs_spec, act_spec, actor, critic


def test_sequence_equals_chained_steps(cuda):
  rng = np.random.default_rng(5)
  B, T, D, A = 3, 12, 4, 2
  _, _, actor, critic = _small_nets(cuda, D, A)
  obs, act, st = _seq_inputs(cuda, rng, B, T, D, A)
  for net, inputs, step in ((actor, obs, lambda t: obs[:, t]),
                            (critic, (obs, act), lambda t: (obs[:, t], act[:, t]))):
    full, fstate = net(inputs, st, net.get_initial_state(B))
    state, outs = net.get_initial_state(B), []
    for t in range(T):
      o, state = net(step(t), st[:, t], state)
      outs.append(o)
    chained = torch.stack(outs, 1)
    assert chained.shape == full.shape
    rel = (chained - full).abs().max().item() / full.abs().max().item()
    record_parity('ddpg_rnn_network_chained_' + net.name, rel=rel)
    assert rel <= 1e-5
    for a, b in zip(_leaves(fstate), _leaves(state)):
      assert (a - b).abs().max().item() <= 1e-5 * max(1.0, b.abs().max().item())


def test_copy_is_independent(cuda):
  rng = np.random.default_rng(1)
  _, _, actor, critic = _small_nets(cuda, 4, 2)
  obs, act, st = _seq_inputs(cuda, rng, 3, 7, 4, 2)
  for net, inputs in ((actor, obs), (critic, (obs, act))):
    before = net(inputs, st)[0].clone()
    cp = net.copy(name='Target')
    with torch.no_grad():
      cp.flat_params.copy_(net.flat_params)
    assert torch.equal(cp(inputs, st)[0], before)
    assert all(a is not b for a, b in zip(cp.layers, net.layers))
    with torch.no_grad():
      cp.flat_params.add_(torch.randn_like(cp.flat_params) * 0.1)
    assert not torch.allclose(cp(inputs, st)[0], before)
    assert torch.equal(net(inputs, st)[0], before)


def _oracle_actor(net):
  dense = lambda l: dict(w=l.kernel.cpu().numpy().copy(), b=l.bias.cpu().numpy().copy(),  # noqa
                         act=l.activation)
  cells = [[c.kernel.cpu().numpy().copy(), c.recurrent_kernel.cpu().numpy().copy(),
            c.bias.cpu().numpy().copy()] for c in net._cells]
  return olstm.RnnNet([dense(l) for l in net._pre], cells, [dense(l) for l in net._post])


def _oracle_critic(net):
  dense = lambda ls: [dict(w=l.kernel.cpu().numpy().copy(), b=l.bias.cpu().numpy().copy(),  # noqa
                           act=l.activation) for l in ls]
  cells = [[c.kernel.cpu().numpy().copy(), c.recurrent_kernel.cpu().numpy().copy(),
            c.bias.cpu().numpy().copy()] for c in net._cells]
  return O.RnnCritic(dense(net._obs_layers), dense(net._act_layers), dense(net._joint_layers),
                     cells, dense(net._post))


@pytest.mark.parametrize('action_fc', [(6,), None])
def test_network_gradients_and_input_only_dqda_match_float64(cuda, action_fc):
  rng = np.random.default_rng(11)
  B, T, D, A = 4, 9, 5, 2
  _, _, actor, critic = _small_nets(cuda, D, A, action_fc)
  obs, act, st = _seq_inputs(cuda, rng, B, T, D, A)
  st_np = st.cpu().numpy()
  oc, oa = _oracle_critic(critic), _oracle_actor(actor)
  x64, a64 = H._t(obs.cpu().numpy().reshape(B * T, D)), H._t(act.cpu().numpy().reshape(B * T, A))
  dq_np = rng.normal(size=B * T).astype(f32)
  # critic parameter gradients
  q, tape = critic.forward_train((obs, act), st)
  grads = critic.backward(tape, torch.as_tensor(dq_np, device=cuda))
  cp = [H._t(p, True) for p in oc.params()]
  q64 = H._critic64(oc, cp, x64, a64, st_np)
  assert _rel(q.cpu(), q64.detach().numpy()) <= 1e-5
  ref = torch.autograd.grad(q64, cp, grad_outputs=H._t(dq_np))
  for view, r in zip(critic._grad_views, ref):
    err = _rel(view.cpu(), r.numpy())
    record_parity('ddpg_rnn_layer_grads_float64_critic', rel=err)
    assert err <= 1e-4
  # the input-only dQ/da: flat_grads bit-unchanged
  before = critic.flat_grads.clone()
  q, tape = critic.forward_train((obs, act), st)
  da = critic.action_gradient(tape, torch.as_tensor(dq_np, device=cuda))
  torch.cuda.synchronize()
  assert torch.equal(critic.flat_grads, before)
  a_in = a64.clone().requires_grad_(True)
  da64, = torch.autograd.grad(H._critic64(oc, [H._t(p) for p in oc.params()], x64, a_in, st_np),
                              a_in, grad_outputs=H._t(dq_np))
  err = _rel(da.cpu(), da64.numpy())
  record_parity('ddpg_rnn_dqda_float64', rel=err)
  assert err <= 1e-4
  # actor parameter gradients
  dy_np = rng.normal(size=(B * T, A)).astype(f32)
  y, atape = actor.forward_train(obs, st)
  agrads = actor.backward(atape, torch.as_tensor(dy_np, device=cuda))
  ap = [H._t(p, True) for p in oa.params()]
  y64 = H._actor64(oa, ap, x64, st_np)
  assert _rel(y.cpu(), y64.detach().numpy()) <= 1e-5
  ref = torch.autograd.grad(y64, ap, grad_outputs=H._t(dy_np))
  for view, r in zip(actor._grad_views, ref):
    err = _rel(view.cpu(), r.numpy())
    record_parity('ddpg_rnn_layer_grads_float64_actor', rel=err)
    assert err <= 1e-4
  assert agrads.data_ptr() == actor.flat_grads.data_ptr()


# ---- the agent ----------------------------------------------------------------------------------
def _build(cuda, D=5, A=2, action_fc=(6,), seed=0, actor_opt=None, critic_opt=None, **kw):
  obs_spec, act_spec, actor, critic = _small_nets(cuda, D, A, action_fc, seed)
  agent = ddpg_agent.DdpgAgent(ts.time_step_spec(obs_spec), act_spec, actor_network=actor,
                               critic_network=critic,
                               actor_optimizer=actor_opt or optimizers.Adam(1e-3),
                               critic_optimizer=critic_opt or optimizers.Adam(2e-3), **kw)
  agent.initialize()
  return agent


def _experience(rng, B, T, D, A):
  st = rng.choice([FIRST, MID, LAST], (B, T), p=[0.15, 0.7, 0.15]).astype(np.int32)
  st[:, 0] = FIRST
  return dict(step_type=st, next_step_type=np.roll(st, -1, 1),
              observation=rng.normal(size=(B, T, D)).astype(f32),
              action=rng.uniform(-1, 2, (B, T, A)).astype(f32),
              reward=rng.normal(size=(B, T)).astype(f32),
              discount=(st != LAST).astype(f32))


def _to_traj(cuda, e):
  d = lambda k: torch.as_tensor(e[k], device=cuda)   # noqa: E731
  return trajectory.Trajectory(d('step_type'), d('observation'), d('action'), (),
                               d('next_step_type'), d('reward'), d('discount'))


TRAIN_CASES = [  # (loss, weights, dqda_clipping, gradient_clipping, tau, period, action_fc)
    ('huber', None, None, None, 1.0, 1, (6,)),
    ('squared', 'row', 0.5, 0.5, 0.5, 2, None),
    ('huber', 'scalar', 0.0, None, 0.1, 3, (6,)),
    ('squared', 'row', None, 1.0, 0.3, 1, (6,)),
]


@pytest.mark.parametrize('case', range(len(TRAIN_CASES)))
def test_recurrent_train_matches_oracle(cuda, case):
  kind, wmode, dqc, gclip, tau, period, action_fc = TRAIN_CASES[case]
  rng = np.random.default_rng(20 + case)
  B, T, D, A = 6, 9, 5, 2
  loss_fn = common.element_wise_huber_loss if kind == 'huber' else \
      common.element_wise_squared_loss
  agent = _build(cuda, D, A, action_fc, td_errors_loss_fn=loss_fn, dqda_clipping=dqc,
                 gradient_clipping=gclip, target_update_tau=tau, target_update_period=period,
                 gamma=0.9, reward_scale_factor=1.5)
  orc = O.RecurrentDdpgOracle(_oracle_actor(agent._actor_network),
                              _oracle_critic(agent._critic_network), [-1.0] * A, [2.0] * A,
                              ooptim.AdamTF(1e-3, eps=1e-7), ooptim.AdamTF(2e-3, eps=1e-7),
                              gamma=0.9, reward_scale=1.5, tau=tau, target_update_period=period,
                              loss=oddpg.HUBER if kind == 'huber' else oddpg.SQUARED,
                              dqda_clipping=dqc, gradient_clipping=gclip)
  for step in range(4):
    e = _experience(rng, B, T, D, A)
    w = {None: None, 'scalar': f32(0.6), 'row': rng.uniform(0, 2, B).astype(f32)}[wmode]
    got = agent.train(_to_traj(cuda, e), weights=None if w is None else torch.as_tensor(
        w, device=cuda))
    want = orc.train(e, w)
    for k in ('critic_loss', 'actor_loss'):
      g, r = getattr(got.extra, k).item(), float(want[k])
      rel = abs(g - r) / max(abs(r), 1e-6)
      record_parity('ddpg_rnn_train_oracle', **{k + '_rel': rel})
      assert rel <= 1e-5, (step, k, g, r)
    for net, params in ((agent._critic_network, orc.critic.params()),
                        (agent._actor_network, orc.actor.params()),
                        (agent._target_critic_network, orc.tc.params()),
                        (agent._target_actor_network, orc.ta.params())):
      for v, p in zip(net.variables, params):
        err = _rel(v.detach().cpu(), p)
        record_parity('ddpg_rnn_train_params', rel=err)
        assert err <= 1e-5, (step, net.name, err)
  agent.check_numerics()
  assert int(agent.train_step_counter.item()) == 4
  assert int(agent._seq_ticket.item()) == 0


class RecordingOptimizer(optimizers.Optimizer):
  """Keeps a copy of every gradient it is handed; the parameters do not move."""

  def __init__(self):
    super().__init__()
    self.calls = []

  def apply_flat(self, params, grads, grad_scale=None):
    self.calls.append(grads.clone())


@pytest.mark.parametrize('action_fc', [(6,), None])
def test_optimizer_gradients_match_float64(cuda, action_fc):
  rng = np.random.default_rng(31)
  B, T, D, A = 5, 10, 5, 2
  ao, co = RecordingOptimizer(), RecordingOptimizer()
  w = rng.uniform(0, 2, B).astype(f32)
  agent = _build(cuda, D, A, action_fc, actor_opt=ao, critic_opt=co, dqda_clipping=0.05,
                 gamma=0.95, target_update_period=1000)
  with torch.no_grad():          # targets that differ from the online networks
    agent._target_params.mul_(0.9)
  e = _experience(rng, B, T, D, A)
  agent.train(_to_traj(cuda, e), weights=torch.as_tensor(w, device=cuda))
  oa, oc = _oracle_actor(agent._actor_network), _oracle_critic(agent._critic_network)
  ota, otc = _oracle_actor(agent._target_actor_network), \
      _oracle_critic(agent._target_critic_network)
  win = O.RecurrentDdpgOracle.windows(e)
  x0, x1, st0, st1 = H._t(win['x0']), H._t(win['x1']), win['st0'], win['st1']
  scale = lambda y: 0.5 + 1.5 * y   # noqa: E731   spec [-1, 2]
  wt = H._t(w)
  a2 = scale(H._actor64(ota, [H._t(p) for p in ota.params()], x1, st1))
  tq = H._critic64(otc, [H._t(p) for p in otc.params()], x1, a2, st1)
  y = H._t(win['r'].reshape(-1)) + 0.95 * H._t(win['d'].reshape(-1)) * tq
  cp = [H._t(p, True) for p in oc.params()]
  err = y - H._critic64(oc, cp, x0, H._t(win['act']), st0)
  el = torch.where(err.abs() <= 1, 0.5 * err * err, err.abs() - 0.5)
  cref = torch.autograd.grad((el.reshape(B, T - 1).sum(1) * wt).mean(), cp)
  ap = [H._t(p, True) for p in oa.params()]
  a = scale(H._actor64(oa, ap, x0, st0))
  a_in = a.detach().requires_grad_(True)
  dqda, = torch.autograd.grad(H._critic64(oc, [H._t(p) for p in oc.params()], x0, a_in,
                                          st0).sum(), a_in)
  c = dqda.clamp(-0.05, 0.05)
  aloss = ((((a.detach() + c) - a) ** 2).reshape(B, T - 1, A).sum(1) * wt[:, None]).mean()
  aref = torch.autograd.grad(aloss, ap)
  for net, rec, refs in ((agent._critic_network, co.calls[0], cref),
                         (agent._actor_network, ao.calls[0], aref)):
    base = net.flat_grads.data_ptr()
    for view, r in zip(net._grad_views, refs):
      off = (view.data_ptr() - base) // 4
      got = rec[off:off + view.numel()].reshape(view.shape).cpu().numpy()
      e_ = _rel(got, r.numpy())
      record_parity('ddpg_rnn_grads_float64_' + net.name, rel=e_)
      assert e_ <= 1e-4, (net.name, e_)


def test_constructor_and_replica_errors(cuda):
  obs_spec, act_spec, actor, critic = _small_nets(cuda, 4, 2)
  ff_actor = actor_network.ActorNetwork(obs_spec, act_spec, fc_layer_params=(8,), device=cuda)
  ff_critic = critic_network.CriticNetwork((obs_spec, act_spec), joint_fc_layer_params=(8,),
                                           device=cuda)
  mk = lambda a, c: ddpg_agent.DdpgAgent(ts.time_step_spec(obs_spec), act_spec, a, c)  # noqa
  with pytest.raises(NotImplementedError, match='both networks recurrent'):
    mk(actor, ff_critic)
  with pytest.raises(NotImplementedError, match='both networks recurrent'):
    mk(ff_actor, critic)
  enc = lstm_encoding_network.LSTMEncodingNetwork(obs_spec, lstm_size=(4,), device=cuda)
  with pytest.raises(NotImplementedError, match='ActorRnnNetwork'):
    mk(enc, critic)
  with pytest.raises(NotImplementedError):
    td3_agent.Td3Agent(ts.time_step_spec(obs_spec), act_spec, actor, critic,
                       optimizers.Adam(1e-3), optimizers.Adam(1e-3))
  with pytest.raises(NotImplementedError):
    sac_agent.SacAgent(ts.time_step_spec(obs_spec), act_spec, critic_network=critic,
                       actor_network=actor, actor_optimizer=optimizers.Adam(1e-3),
                       critic_optimizer=optimizers.Adam(1e-3),
                       alpha_optimizer=optimizers.Adam(1e-3))
  agent = _build(cuda, 4, 2)
  assert agent.train_sequence_length is None
  e = _experience(np.random.default_rng(0), 2, 1, 4, 2)
  with pytest.raises(ValueError, match='at least 2'):
    agent.train(_to_traj(cuda, e))
  agent.replicas = 2
  with pytest.raises(NotImplementedError):
    agent.train(_to_traj(cuda, _experience(np.random.default_rng(0), 2, 4, 4, 2)))


# ---- policies -----------------------------------------------------------------------------------
def _time_step(cuda, step_type, obs):
  B = obs.shape[0]
  return ts.TimeStep(torch.full((B,), step_type, dtype=torch.int32, device=cuda),
                     torch.zeros(B, device=cuda), torch.ones(B, device=cuda), obs)


def test_stateful_actor_policies(cuda):
  agent = _build(cuda, 4, 2)
  B = 6
  obs = torch.randn(B, 4, device=cuda)
  greedy, collect = agent.policy, agent.collect_policy
  assert greedy.policy_state_spec == agent._actor_network.state_spec == collect.policy_state_spec
  s0 = greedy.get_initial_state(B)
  assert isinstance(s0, list) and isinstance(collect.get_initial_state(B), list)
  a1 = greedy.action(_time_step(cuda, FIRST, obs), s0)
  a2 = greedy.action(_time_step(cuda, MID, obs), a1.state)
  assert not torch.equal(a1.state[0], a2.state[0])
  a3 = greedy.action(_time_step(cuda, FIRST, obs), a2.state)     # FIRST resets
  assert all(torch.equal(x, y) for x, y in zip(a3.state, a1.state))
  want, _ = agent._actor_network(obs, torch.zeros(B, dtype=torch.int32, device=cuda), s0)
  assert torch.equal(a1.action, want)
  assert float(a1.action.min()) >= -1 and float(a1.action.max()) <= 2
  c1 = collect.action(_time_step(cuda, FIRST, obs), s0)
  assert all(torch.equal(x, y) for x, y in zip(c1.state, a1.state))
  for pol in (greedy, collect):
    with pytest.raises(ValueError, match='stateful'):
      pol.action(_time_step(cuda, FIRST, obs))


# Launches of the feed-forward DDPG policies and train() before the recurrent path was added,
# counted with _lib.launch_count() on the configuration of _ff_agent: the feed-forward path must
# keep issuing exactly these.
PARENT_FF_LAUNCHES = dict(policy=4, collect=5, train=42)


def _ff_agent(cuda):
  obs_spec = tensor_spec.TensorSpec((5,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((2,), torch.float32, -1.0, 2.0, 'action')
  actor = actor_network.ActorNetwork(obs_spec, act_spec, fc_layer_params=(16, 8),
                                     device=cuda).set_seed(1)
  critic = critic_network.CriticNetwork((obs_spec, act_spec), observation_fc_layer_params=(12,),
                                        joint_fc_layer_params=(10,), device=cuda).set_seed(2)
  agent = ddpg_agent.DdpgAgent(ts.time_step_spec(obs_spec), act_spec, actor_network=actor,
                               critic_network=critic, actor_optimizer=optimizers.Adam(1e-3),
                               critic_optimizer=optimizers.Adam(1e-3), gradient_clipping=1.0,
                               dqda_clipping=0.5)
  agent.initialize()
  return agent


def ff_launch_counts(cuda):
  agent = _ff_agent(cuda)
  rng = np.random.default_rng(0)
  obs = torch.randn(8, 5, device=cuda)
  out = {}
  for k, pol in (('policy', agent.policy), ('collect', agent.collect_policy)):
    n0 = _lib.launch_count()
    step = pol.action(_time_step(cuda, MID, obs))
    out[k] = _lib.launch_count() - n0
    assert step.state == () and pol.get_initial_state(8) == ()
  traj = _to_traj(cuda, _experience(rng, 8, 2, 5, 2))
  agent.train(traj)
  n0 = _lib.launch_count()
  agent.train(traj)
  out['train'] = _lib.launch_count() - n0
  return out


def test_feed_forward_launches_unchanged(cuda):
  assert ff_launch_counts(cuda) == PARENT_FF_LAUNCHES


# ---- graphs and restore -------------------------------------------------------------------------
def test_train_graph_replays_bit_for_bit(cuda, ffma):
  rng = np.random.default_rng(6)
  B, T, D, A = 4, 11, 5, 2
  make = lambda: _build(cuda, D, A, gradient_clipping=1.0, target_update_tau=0.5,  # noqa: E731
                        target_update_period=2, dqda_clipping=0.5)
  eager, graphed = make(), make()
  train_fn = common.function(graphed.train)
  for _ in range(5):
    traj = _to_traj(cuda, _experience(rng, B, T, D, A))
    w = torch.as_tensor(rng.uniform(0, 2, B).astype(f32), device=cuda)
    l1 = eager.train(traj, weights=w).loss.item()
    l2 = train_fn(traj, weights=w).loss.item()
    assert l1 == l2
  assert torch.equal(graphed._online_params, eager._online_params)
  assert torch.equal(graphed._target_params, eager._target_params)
  assert int(graphed._seq_ticket.item()) == 0


def test_stateful_ou_collect_graph_replays_bit_for_bit(cuda):
  """12 runs of 4 OU-noise collect steps with the actor state threaded through DynamicStepDriver:
  captured into one CUDA graph they store the same trajectories and end in the same network and OU
  state, bit for bit, as 12 eager runs."""
  B = 8
  out = []
  for graphed in (False, True):
    agent = _build(cuda, 4, 2, ou_stddev=0.3, ou_damping=0.15)
    obs_spec = tensor_spec.TensorSpec((4,), torch.float32, 'observation')
    act_spec = tensor_spec.BoundedTensorSpec((2,), torch.float32, -1.0, 2.0, 'action')
    env = random_tf_environment.RandomTFEnvironment(ts.time_step_spec(obs_spec), act_spec,
                                                    batch_size=B, episode_end_probability=0.2,
                                                    seed=3, device=cuda)
    rb = rb_mod.TFUniformReplayBuffer(agent.collect_data_spec, batch_size=B, max_length=64,
                                      device=cuda)
    driver = dynamic_step_driver.DynamicStepDriver(env, agent.collect_policy,
                                                   observers=[rb.add_batch], num_steps=B * 4)
    run = lambda t, s: driver.run(t, s, maximum_iterations=4)   # noqa: E731
    if graphed:
      run = common.function(run)
    time_step, state = env.reset(), agent.collect_policy.get_initial_state(B)
    for _ in range(12):
      time_step, state = run(time_step, state)
    exp = rb.gather_all()
    out.append([t.clone() for t in _leaves(exp)] + [t.clone() for t in _leaves(state)] +
               [agent.collect_policy.ou_state.clone()])
  assert int((out[0][0] == FIRST).sum()) > B
  for a, b in zip(*out):
    assert torch.equal(a, b)


def test_learner_restores_bit_for_bit(cuda, tmp_path, ffma):
  rng = np.random.default_rng(8)
  B, T, D, A = 4, 9, 5, 2
  exps = [_to_traj(cuda, _experience(rng, B, T, D, A)) for _ in range(4)]
  a1 = _build(cuda, D, A, target_update_tau=0.3, seed=0)
  l1 = learner_lib.Learner(str(tmp_path / 'run'), a1.train_step_counter, a1,
                           experience_dataset_fn=lambda: iter([(e, ()) for e in exps]),
                           checkpoint_interval=1)
  l1.run(iterations=2)
  a2 = _build(cuda, D, A, target_update_tau=0.3, seed=5)
  l2 = learner_lib.Learner(str(tmp_path / 'run'), a2.train_step_counter, a2,
                           experience_dataset_fn=lambda: iter([(e, ()) for e in exps[2:]]),
                           checkpoint_interval=0)
  assert int(a2.train_step_counter.item()) == 2
  for k, v in learner_lib._agent_state_tensors(a1).items():
    assert torch.equal(learner_lib._agent_state_tensors(a2)[k], v), k
  i1, i2 = l1.run(iterations=2), l2.run(iterations=2)
  assert i1.loss.item() == i2.loss.item()
  assert torch.equal(a1._online_params, a2._online_params)
  assert torch.equal(a1._target_params, a2._target_params)


# ---- the reference example's wiring -------------------------------------------------------------
def test_train_eval_rnn_flow(cuda):
  """ddpg/examples/v2/train_eval_rnn.py at a small size: DynamicEpisodeDriver collection with the
  OU collect policy, TFUniformReplayBuffer.as_dataset(num_steps=11), then train."""
  obs_spec = tensor_spec.TensorSpec((3,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((1,), torch.float32, -1.0, 1.0, 'action')
  env = random_tf_environment.RandomTFEnvironment(ts.time_step_spec(obs_spec), act_spec,
                                                  batch_size=1, episode_end_probability=0.05,
                                                  seed=1, device=cuda)
  actor = actor_rnn_network.ActorRnnNetwork(obs_spec, act_spec, input_fc_layer_params=(40, 30),
                                            lstm_size=(8,), output_fc_layer_params=(10,),
                                            device=cuda)
  critic = critic_rnn_network.CriticRnnNetwork(
      (obs_spec, act_spec), observation_fc_layer_params=(40,), action_fc_layer_params=None,
      joint_fc_layer_params=(30,), lstm_size=(8,), output_fc_layer_params=(10,), device=cuda)
  agent = ddpg_agent.DdpgAgent(ts.time_step_spec(obs_spec), act_spec, actor_network=actor,
                               critic_network=critic, actor_optimizer=optimizers.Adam(1e-4),
                               critic_optimizer=optimizers.Adam(1e-3), ou_stddev=0.2,
                               ou_damping=0.15, target_update_tau=0.05, target_update_period=5,
                               gamma=0.995)
  agent.initialize()
  rb = rb_mod.TFUniformReplayBuffer(agent.collect_data_spec, batch_size=1, max_length=1000,
                                    device=cuda)
  driver = dynamic_episode_driver.DynamicEpisodeDriver(env, agent.collect_policy,
                                                       observers=[rb.add_batch], num_episodes=2)
  time_step, state = driver.run()
  it = iter(rb.as_dataset(sample_batch_size=8, num_steps=11))
  for _ in range(3):
    time_step, state = driver.run(time_step=time_step, policy_state=state)
    for _ in range(4):
      exp, _ = next(it)
      loss = agent.train(exp)
  agent.check_numerics()
  assert np.isfinite(loss.loss.item())
  assert int(agent.train_step_counter.item()) == 12


# ---- learning: a task that needs memory ---------------------------------------------------------
CUE_STEPS = 3      # decisions per episode; the cue is visible at the first only


def _cue_batch(rng, B):
  """Random-action cue-recall episodes as [B, CUE_STEPS + 1] sequences: observation (cue, 1) at
  FIRST and (0, 0) after, reward -(a - cue)^2 at the last decision, a LAST boundary step."""
  T = CUE_STEPS + 1
  cue = rng.choice([-1.0, 1.0], B).astype(f32)
  obs = np.zeros((B, T, 2), f32)
  obs[:, 0] = np.stack([cue, np.ones(B, f32)], 1)
  act = rng.uniform(-1.5, 1.5, (B, T, 1)).astype(f32)
  rew = np.zeros((B, T), f32)
  rew[:, CUE_STEPS - 1] = -(act[:, CUE_STEPS - 1, 0] - cue) ** 2
  st = np.full((B, T), MID, np.int32)
  st[:, 0], st[:, -1] = FIRST, LAST
  nst = np.roll(st, -1, 1)
  nst[:, -1] = FIRST
  disc = np.ones((B, T), f32)
  disc[:, CUE_STEPS - 1] = 0
  return dict(step_type=st, next_step_type=nst, observation=obs, action=act, reward=rew,
              discount=disc)


def _cue_error(cuda, recurrent, seed, steps=2000, B=64):
  obs_spec = tensor_spec.TensorSpec((2,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((1,), torch.float32, -1.5, 1.5, 'action')
  if recurrent:
    actor = actor_rnn_network.ActorRnnNetwork(obs_spec, act_spec, input_fc_layer_params=(32,),
                                              lstm_size=(16,), output_fc_layer_params=(32,),
                                              device=cuda).set_seed(seed)
    critic = critic_rnn_network.CriticRnnNetwork(
        (obs_spec, act_spec), observation_fc_layer_params=(32,), action_fc_layer_params=None,
        joint_fc_layer_params=(32,), lstm_size=(16,), output_fc_layer_params=(32,),
        device=cuda).set_seed(seed + 1)
  else:
    actor = actor_network.ActorNetwork(obs_spec, act_spec, fc_layer_params=(32, 32),
                                       device=cuda).set_seed(seed)
    critic = critic_network.CriticNetwork((obs_spec, act_spec), observation_fc_layer_params=(32,),
                                          joint_fc_layer_params=(32,), device=cuda).set_seed(
                                              seed + 1)
  agent = ddpg_agent.DdpgAgent(ts.time_step_spec(obs_spec), act_spec, actor_network=actor,
                               critic_network=critic, actor_optimizer=optimizers.Adam(1e-3),
                               critic_optimizer=optimizers.Adam(3e-3), target_update_tau=0.05,
                               gamma=0.0)
  agent.initialize()
  rng = np.random.default_rng(seed)
  for _ in range(steps):
    e = _cue_batch(rng, B)
    if not recurrent:       # the feed-forward agent trains on the episodes' [*, 2] transitions
      e = {k: np.stack([v[:, :-1], v[:, 1:]], 2).reshape((-1, 2) + v.shape[2:])
           for k, v in e.items()}
    agent.train(_to_traj(cuda, e))
  agent.check_numerics()
  cue = torch.as_tensor(rng.choice([-1.0, 1.0], 1024).astype(f32), device=cuda)
  state = agent.policy.get_initial_state(1024)
  for t in range(CUE_STEPS):
    obs = torch.stack([cue, torch.ones_like(cue)], 1) if t == 0 else torch.zeros(1024, 2,
                                                                                 device=cuda)
    step = agent.policy.action(_time_step(cuda, FIRST if t == 0 else MID, obs), state)
    state = step.state
  return float((step.action[:, 0] - cue).abs().mean())


def test_cue_recall_needs_memory(cuda):
  """A +-1 cue at the first step, zeros after it, and reward -(a - cue)^2 at the last of three
  decisions, learnt offline from random-action episodes: recurrent DDPG recalls the cue; the
  feed-forward agent cannot beat |a - cue| = 1 in expectation (its last observation carries no
  information)."""
  rnn = _cue_error(cuda, True, 0)
  ff = _cue_error(cuda, False, 0)
  record_parity('ddpg_rnn_cue_recall', recurrent_error=rnn, feed_forward_error=ff)
  assert rnn <= 0.5, rnn
  assert ff >= 0.9, ff
