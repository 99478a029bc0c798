"""Recurrent DQN on the GPU: the b200rl_dqn_seq_td_loss kernel against float64, DqnAgent /
DdqnAgent on QRnnNetwork against the numpy oracle (tests/dqn_rnn_oracle.py) and float64 autograd,
the reference's RNN smoke loss, QRnnNetwork, the stateful Q policies, CUDA-graph replays, a Learner
restore, and a cue-recall task only a recurrent Q network can solve."""
import numpy as np
import pytest
import torch

from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.agents.categorical_dqn import categorical_dqn_agent
from agents_b200.agents.dqn import dqn_agent
from agents_b200.drivers import dynamic_step_driver
from agents_b200.environments import random_tf_environment
from agents_b200.networks import lstm_encoding_network as len_
from agents_b200.networks import q_network
from agents_b200.networks import q_rnn_network
from agents_b200.policies import q_policy
from agents_b200.replay_buffers import tf_uniform_replay_buffer as rb_mod
from agents_b200.specs import tensor_spec
from agents_b200.train import learner as learner_lib
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory
from agents_b200.utils import common
from oracle import lstm as olstm
from oracle import optim as ooptim

import dqn_rnn_oracle as O
import grad_refs as R

from conftest import record_parity

pytestmark = pytest.mark.gpu
f32 = np.float32
LAST = 2


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
  """||got - ref|| / ||ref|| (the absolute error when ref is 0)."""
  got, ref = np.asarray(got, np.float64).reshape(-1), np.asarray(ref, np.float64).reshape(-1)
  m, d = np.linalg.norm(ref), np.linalg.norm(got - ref)
  return d / m if m > 0 else d


def _rel_max(got, ref):
  """max |got - ref| / max |ref| (the absolute error when ref is 0)."""
  got, ref = np.asarray(got, np.float64).reshape(-1), np.asarray(ref, np.float64).reshape(-1)
  m, d = np.abs(ref).max(), np.abs(got - ref).max()
  return d / m if m > 0 else d


# ---- the kernel ---------------------------------------------------------------------------------
class SeqLoss(object):
  """One b200rl_dqn_seq_td_loss launch with its own scratch."""

  def __init__(self, cuda):
    self.partials = torch.empty(_lib.DQN_SEQ_MAX_BLOCKS, dtype=torch.float32, device=cuda)
    self.ticket = torch.zeros(1, dtype=torch.int32, device=cuda)
    self.nan_flag = torch.zeros(1, dtype=torch.int32, device=cuda)

  def __call__(self, q, nt, ns, mask, act, st, rew, disc, w, w_stride, B, A, T, gamma, scale,
               kind, gb=None):
    dev = q.device
    loss = torch.empty(1, device=dev)
    td_loss = torch.empty(B, device=dev)
    td_error = torch.empty((B, T - 1), device=dev)
    dq = torch.empty_like(q)
    _lib.call('b200rl_dqn_seq_td_loss', _lib.ptr(q), _lib.ptr(nt), _lib.ptr(ns), _lib.ptr(mask),
              _lib.dptr(act), act.stride(0), act.stride(1), _lib.dptr(st), st.stride(0),
              st.stride(1), _lib.ptr(rew), _lib.ptr(disc), _lib.ptr(w), w_stride, B, A, T,
              gamma, scale, kind, float(gb or B), _lib.ptr(loss), _lib.ptr(td_loss),
              _lib.ptr(td_error), _lib.ptr(dq), _lib.ptr(self.nan_flag), _lib.ptr(self.partials),
              _lib.ptr(self.ticket), _lib.stream())
    return loss, td_loss, td_error, dq


def _strided(x, cuda, strided):
  """[B, T] int32 on the device; strided: a column view of a wider [B, T, 3] tensor."""
  t = torch.as_tensor(x, device=cuda)
  if not strided:
    return t.contiguous()
  wide = torch.full(tuple(t.shape) + (3,), 77, dtype=t.dtype, device=cuda)
  wide[..., 1] = t
  return wide[..., 1]


def _case(rng, B, Tm, A, last, masked, clamp):
  T = Tm + 1
  N = B * Tm
  q, nt, ns = (rng.randn(N, A).astype(f32) * 2 for _ in range(3))
  act = rng.randint(0, A, (B, T)).astype(np.int32)
  if clamp:
    act[0, 0], act[-1, Tm - 1] = -3, A + 2
  st = np.ones((B, T), np.int32)
  st[:, 0] = 0
  if last == 'first':
    st[:, 0] = LAST
  elif last == 'middle':
    st[:, Tm // 2] = LAST
  elif last == 'last':
    st[:, Tm - 1] = LAST
  elif last == 'all':
    st[:] = LAST
  else:
    st = rng.choice([0, 1, 2], (B, T), p=[0.2, 0.6, 0.2]).astype(np.int32)
  rew = rng.randn(B, T).astype(f32)
  disc = (rng.rand(B, T) > 0.2).astype(f32) * rng.rand(B, T).astype(f32)
  mask = None
  if masked:
    mask = (rng.rand(N, A) > 0.3).astype(np.int32)
    mask[:, -1] = 1
  return q, nt, ns, mask, act, st, rew, disc


KERNEL_SHAPES = [(1, 1, 1), (1, 1000, 2), (7, 1, 18), (7, 2, 6), (7, 80, 1), (256, 1, 2),
                 (256, 10, 6), (256, 80, 18), (5000, 1, 6), (5000, 2, 2), (5000, 10, 18),
                 (256, 1000, 2), (5000, 80, 1)]
VARIANTS = [  # (loss, last, masked, weights, strided, clamp)
    ('huber', 'random', False, 'none', False, False),
    ('squared', 'random', True, 'row', True, False),
    ('huber', 'first', True, 'scalar', False, True),
    ('huber', 'middle', False, 'zero', True, False),
    ('squared', 'last', False, 'row', False, True),
    ('huber', 'all', True, 'row', True, False),
]


@pytest.mark.parametrize('B,Tm,A', KERNEL_SHAPES)
@pytest.mark.parametrize('variant', range(len(VARIANTS)))
def test_seq_kernel_matches_float64(cuda, B, Tm, A, variant):
  kind, last, masked, wkind, strided, clamp = VARIANTS[variant]
  rng = np.random.RandomState(B + 7 * Tm + 31 * A + variant)
  q, nt, ns, mask, act, st, rew, disc = _case(rng, B, Tm, A, last, masked, clamp)
  T = Tm + 1
  if wkind == 'none':
    w, w_stride = None, 0
  elif wkind == 'scalar':
    w, w_stride = np.array(0.7, f32), 0
  elif wkind == 'zero':
    w, w_stride = np.zeros(B, f32), 1
  else:
    w, w_stride = np.where(rng.rand(B) < 0.3, 0, rng.rand(B)).astype(f32), 1
  d = lambda x: None if x is None else torch.as_tensor(x, device=cuda)
  run = SeqLoss(cuda)
  kcode = _lib.LOSS_HUBER if kind == 'huber' else _lib.LOSS_SQUARED
  args = (d(q), d(nt), d(ns), d(mask), _strided(act, cuda, strided),
          _strided(st, cuda, strided), d(rew), d(disc), d(w), w_stride, B, A, T, 0.9, 1.5, kcode)
  got = run(*args)
  got = [t.clone() for t in got]
  again = run(*args)
  for a, b in zip(got, again):                    # fixed-order sums: the same bits
    assert torch.equal(a, b)
  assert int(run.ticket.item()) == 0
  assert int(run.nan_flag.item()) == int(clamp)
  want = O.seq_loss_float64(q, nt, ns, act[:, :-1], st[:, :-1], rew[:, :-1], disc[:, :-1], 0.9,
                            1.5, kind, w, mask)
  # relative to float64 of the same float32 inputs; a single element of td_error / dq carries the
  # float32 rounding of y - q, which is relative to |y| and |q| rather than to the difference
  errs = dict(loss=_rel(got[0].item(), want[0]), td_loss=_rel(got[1].cpu(), want[1]),
              td_error=_rel(got[2].cpu(), want[2]), dq=_rel(got[3].cpu(), want[3]))
  record_parity('dqn_seq_td_loss_float64', **errs,
                **{k + '_max': _rel_max(g.cpu(), w) for k, g, w in
                   (('td_loss', got[1], want[1]), ('td_error', got[2], want[2]),
                    ('dq', got[3], want[3]))})
  for k, e in errs.items():
    assert e <= 1e-6, (k, e)


@pytest.mark.parametrize('B,A', [(7, 6), (256, 2), (5000, 18)])
@pytest.mark.parametrize('kind', [_lib.LOSS_HUBER, _lib.LOSS_SQUARED])
def test_one_transition_matches_feed_forward_kernel(cuda, B, A, kind):
  rng = np.random.RandomState(B + A + kind)
  q, nt, ns, mask, act, st, rew, disc = _case(rng, B, 1, A, 'random', True, False)
  q, nt, ns, mask, act, st, rew, disc = (torch.as_tensor(x, device=cuda) for x in
                                          (q, nt, ns, mask, act, st, rew, disc))
  w = torch.as_tensor(rng.rand(B).astype(f32), device=cuda)
  seq = SeqLoss(cuda)(q, nt, ns, mask, act, st, rew, disc, w, 1, B, A, 2, 0.95, 1.5, kind)
  loss = torch.empty(1, device=cuda)
  td_loss, td_error, dq = torch.empty(B, device=cuda), torch.empty(B, device=cuda), q * 0
  _lib.call('b200rl_dqn_td_loss', _lib.ptr(q), _lib.ptr(nt), _lib.ptr(ns), _lib.ptr(mask),
            _lib.ptr(act), _lib.ptr(st), _lib.ptr(rew), _lib.ptr(disc),
            _lib.ptr(w), 2, 2, B, A, 2, 0.95, 1.5, kind, float(B), _lib.ptr(loss),
            _lib.ptr(td_loss), _lib.ptr(td_error), _lib.ptr(dq), None, _lib.stream())
  assert torch.equal(seq[1], td_loss)
  assert torch.equal(seq[2].reshape(-1), td_error)
  assert torch.equal(seq[3], dq)
  if B <= 256:                                   # one block in both: the same sum order
    assert torch.equal(seq[0], loss)
  else:
    assert abs(seq[0].item() - loss.item()) <= 1e-6 * abs(loss.item())


# ---- agents -------------------------------------------------------------------------------------
def _smoke_agent(cuda, agent_class):
  exp, (W, U, b) = O.reference_smoke_case()
  obs_spec = tensor_spec.TensorSpec((2,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 1, 'action')
  net = len_.LSTMEncodingNetwork(obs_spec, input_fc_layer_params=(), lstm_size=(2,),
                                 output_fc_layer_params=(), device=cuda)
  net.create_variables()
  cell = net._cells[0]
  with torch.no_grad():
    cell.kernel.copy_(torch.as_tensor(W))
    cell.recurrent_kernel.copy_(torch.as_tensor(U))
    cell.bias.copy_(torch.as_tensor(b))
  agent = agent_class(ts.time_step_spec(obs_spec), act_spec, q_network=net, optimizer=None,
                      gamma=1.0)
  agent.initialize()
  return agent, _to_traj(cuda, exp)


def _to_traj(cuda, e):
  d = lambda k: torch.as_tensor(e[k], device=cuda)
  obs = d('observation')
  if 'mask' in e:
    obs = {'obs': obs, 'mask': d('mask')}
  return trajectory.Trajectory(d('step_type'), obs, d('action'), (), d('next_step_type'),
                               d('reward'), d('discount'))


@pytest.mark.parametrize('agent_class', [dqn_agent.DqnAgent, dqn_agent.DdqnAgent])
def test_reference_rnn_smoke_loss(cuda, agent_class):
  """dqn_agent_test.py testLossRNNSmokeTest: 28.722265 (the reference's _loss runs at gamma 1)."""
  agent, traj = _smoke_agent(cuda, agent_class)
  info = agent.loss(traj)
  got = info.loss.item()
  record_parity('dqn_rnn_reference_smoke', rel=abs(got - O.REFERENCE_SMOKE_LOSS) /
                O.REFERENCE_SMOKE_LOSS)
  assert abs(got - O.REFERENCE_SMOKE_LOSS) <= 1e-6 * O.REFERENCE_SMOKE_LOSS, got
  assert tuple(info.extra.td_loss.shape) == (2,)
  assert tuple(info.extra.td_error.shape) == (2, 2)
  assert agent.train_sequence_length is None


def _dense(l):
  return dict(w=l.kernel.cpu().numpy().copy(), b=l.bias.cpu().numpy().copy(), act=l.activation)


def _mirror(net):
  cells = [[c.kernel.cpu().numpy().copy(), c.recurrent_kernel.cpu().numpy().copy(),
            c.bias.cpu().numpy().copy()] for c in net._cells]
  return olstm.RnnNet([_dense(l) for l in net._pre], cells, [_dense(l) for l in net._post])


def _specs(D, A, masked):
  obs = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act = tensor_spec.BoundedTensorSpec((), torch.int32, 0, A - 1, 'action')
  if masked:
    return {'obs': obs, 'mask': tensor_spec.TensorSpec((A,), torch.int32, 'mask')}, obs, act
  return obs, obs, act


def _experience(rng, B, T, D, A, masked):
  st = rng.choice([0, 1, 2], (B, T), p=[0.15, 0.7, 0.15]).astype(np.int32)
  st[:, 0] = 0
  e = dict(step_type=st, next_step_type=np.roll(st, -1, 1),
           observation=rng.randn(B, T, D).astype(f32),
           action=rng.randint(0, A, (B, T)).astype(np.int32),
           reward=rng.randn(B, T).astype(f32),
           discount=(st != LAST).astype(f32) * f32(1.0))
  if masked:
    m = (rng.rand(B, T, A) > 0.3).astype(np.int32)
    m[..., 0] = 1
    e['mask'] = m
  return e


def _build(cuda, D, A, agent_class=dqn_agent.DqnAgent, masked=False, optimizer=None, l2=0.0,
           seed=0, **kw):
  spec, obs_spec, act_spec = _specs(D, A, masked)
  net = q_rnn_network.QRnnNetwork(obs_spec, act_spec, input_fc_layer_params=(16,),
                                  lstm_size=(8, 6), output_fc_layer_params=(12,),
                                  device=cuda).set_seed(seed)
  if l2:
    net._post[0].l2 = l2
  splitter = (lambda o: (o['obs'], o['mask'])) if masked else None
  agent = agent_class(ts.time_step_spec(spec), act_spec, q_network=net,
                      optimizer=optimizer or optimizers.AdamOptimizer(1e-2),
                      observation_and_action_constraint_splitter=splitter, **kw)
  agent.initialize()
  return agent, net


TRAIN_CASES = [  # (agent, loss, masked, weights, clipping, l2, tau, period)
    (dqn_agent.DqnAgent, 'huber', False, False, None, 0.0, 1.0, 1),
    (dqn_agent.DdqnAgent, 'squared', True, True, 0.5, 0.01, 0.5, 2),
    (dqn_agent.DqnAgent, 'squared', True, False, 1.0, 0.02, 0.1, 1),
    (dqn_agent.DdqnAgent, 'huber', False, True, None, 0.0, 1.0, 3),
]


@pytest.mark.parametrize('case', range(len(TRAIN_CASES)))
def test_recurrent_train_matches_oracle(cuda, case):
  cls, kind, masked, weighted, clip, l2, tau, period = TRAIN_CASES[case]
  rng = np.random.RandomState(10 + case)
  B, T, D, A = 6, 9, 5, 3
  loss_fn = common.element_wise_huber_loss if kind == 'huber' else \
      common.element_wise_squared_loss
  agent, net = _build(cuda, D, A, cls, masked, l2=l2, td_errors_loss_fn=loss_fn,
                      gradient_clipping=clip, target_update_tau=tau,
                      target_update_period=period, gamma=0.9, reward_scale_factor=1.5)
  onet = _mirror(net)
  n_pre = 2 * len(net._pre) + 3 * len(net._cells)
  orc = O.RecurrentDqnOracle(onet, ooptim.AdamTF(1e-2, eps=1e-8), gamma=0.9, reward_scale=1.5,
                             loss_fn=kind, target_update_tau=tau, target_update_period=period,
                             gradient_clipping=clip, ddqn=cls is dqn_agent.DdqnAgent,
                             l2=[(n_pre, l2)] if l2 else ())
  for step in range(4):
    e = _experience(rng, B, T, D, A, masked)
    w = rng.rand(B).astype(f32) if weighted else None
    got = agent.train(_to_traj(cuda, e), weights=None if w is None else torch.as_tensor(
        w, device=cuda))
    want = orc.train(e, w)
    rel = abs(got.loss.item() - float(want['loss'])) / max(1.0, abs(float(want['loss'])))
    record_parity('dqn_rnn_train_oracle', loss_rel=rel,
                  td_loss=_rel(got.extra.td_loss.cpu(), want['td_loss']))
    assert rel <= 1e-5, (step, got.loss.item(), want['loss'])
    np.testing.assert_allclose(got.extra.td_loss.cpu().numpy(), want['td_loss'], rtol=1e-5,
                               atol=1e-5)
  agent.check_numerics()
  assert int(agent.train_step_counter.item()) == 4


class RecordingOptimizer(optimizers.Optimizer):
  """Keeps a copy of every gradient it is handed; the parameters do not move."""

  def __init__(self):
    super().__init__()
    self.calls = []

  def apply_flat(self, params, grads, grad_scale=None):
    self.calls.append(grads.clone())


def _rnn64(net, x, step_type):
  """float64 torch forward of a QRnnNetwork over [B*T, D] rows; returns (q [B*T, A], leaves in
  net.variables order)."""
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
    x = R.activate(x @ p(l.kernel) + p(l.bias), l.activation)
  return x, leaves


@pytest.mark.parametrize('agent_class', [dqn_agent.DqnAgent, dqn_agent.DdqnAgent])
def test_recurrent_gradients_match_float64(cuda, agent_class):
  rng = np.random.RandomState(21)
  B, T, D, A = 5, 13, 4, 3
  l2 = 0.01
  opt = RecordingOptimizer()
  # the target update fires at step 1000, so the target after train() is the one train() used
  agent, net = _build(cuda, D, A, agent_class, optimizer=opt, l2=l2, gamma=0.95,
                      target_update_period=1000)
  with torch.no_grad():     # a target that differs from the online net
    agent._target_q_network.flat_params.mul_(0.9)
  e = _experience(rng, B, T, D, A, False)
  agent.train(_to_traj(cuda, e))
  N = B * (T - 1)
  x0 = R.t64(e['observation'][:, :-1].reshape(N, D))
  x1 = R.t64(e['observation'][:, 1:].reshape(N, D))
  st0, st1 = e['step_type'][:, :-1], e['next_step_type'][:, :-1]
  q64, leaves = _rnn64(net, x0, st0)
  nt64, _ = _rnn64(agent._target_q_network, x1, st1)
  ns64 = _rnn64(net, x1, st1)[0] if agent_class is dqn_agent.DdqnAgent else nt64
  _, _, _, dq = O.seq_loss_float64(q64.detach().numpy(), nt64.detach().numpy(),
                                   ns64.detach().numpy(), e['action'][:, :-1], st0,
                                   e['reward'][:, :-1], e['discount'][:, :-1], 0.95, 1.0,
                                   'huber', None, None)
  g_ref = list(torch.autograd.grad(q64, leaves, grad_outputs=torch.as_tensor(dq)))
  k = 2 * len(net._pre) + 3 * len(net._cells)       # the first output Dense kernel carries l2
  g_ref[k] = g_ref[k] + 2 * l2 * leaves[k].detach()
  base = net.flat_grads.data_ptr()
  rec = opt.calls[0]
  for i, (view, ref) in enumerate(zip(net._grad_views, g_ref)):
    off = (view.data_ptr() - base) // 4
    got = rec[off:off + view.numel()].reshape(view.shape)
    err = R.grad_errors(got, ref)
    record_parity('dqn_rnn_grads_float64', rel_l2=err[0], rel_max=err[1])
    R.assert_grad_close(f'variable {i}', got, ref, 1e-4, 1e-4)


def test_constructor_and_replica_errors(cuda):
  spec, obs_spec, act_spec = _specs(3, 2, False)
  net = lambda: q_rnn_network.QRnnNetwork(obs_spec, act_spec, lstm_size=(4,), device=cuda)
  with pytest.raises(NotImplementedError, match='n_step_update = 2'):
    dqn_agent.DqnAgent(ts.time_step_spec(spec), act_spec, q_network=net(),
                       optimizer=optimizers.AdamOptimizer(1e-3), n_step_update=2)
  c51_net = net()
  c51_net.num_atoms = 51
  with pytest.raises(NotImplementedError, match='stateless'):
    categorical_dqn_agent.CategoricalDqnAgent(ts.time_step_spec(spec), act_spec,
                                              categorical_q_network=c51_net,
                                              optimizer=optimizers.AdamOptimizer(1e-3))
  agent, _ = _build(cuda, 3, 2)
  agent.replicas = 2
  e = _experience(np.random.RandomState(0), 2, 4, 3, 2, False)
  with pytest.raises(NotImplementedError, match='one replica'):
    agent.train(_to_traj(cuda, e))


# ---- network ------------------------------------------------------------------------------------
def test_q_rnn_network_structure_and_state(cuda):
  """q_rnn_network_test.py: one LSTM(40) and stacked (10, 5) cells on CartPole's spec."""
  obs_spec = tensor_spec.TensorSpec((4,), torch.float32)
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int64, 0, 1)
  first = torch.zeros(1, dtype=torch.int32, device=cuda)
  obs = torch.randn(1, 4, device=cuda)
  net = q_rnn_network.QRnnNetwork(obs_spec, act_spec, lstm_size=(40,), device=cuda)
  q, state = net(obs, first, network_state=net.get_initial_state(batch_size=1))
  assert tuple(q.shape) == (1, 2)
  assert tuple(state[0].shape) == (1, 40) and tuple(state[1].shape) == (1, 40)
  # input fc (75, 40), the LSTM, output fc (75, 40) and the Q head: 4 + 3 + 4 + 2 variables
  assert len(net.trainable_variables) == 13
  head = net._post[-1]
  assert bool((head.bias == -0.2).all())
  assert float(head.kernel.abs().max()) <= 0.03
  stacked = q_rnn_network.QRnnNetwork(obs_spec, act_spec, lstm_size=(10, 5), device=cuda)
  q, state = stacked(obs, first, network_state=stacked.get_initial_state(batch_size=1))
  assert tuple(q.shape) == (1, 2) and len(state) == 2
  assert [tuple(s.shape) for s in state[0]] == [(1, 10), (1, 10)]
  assert [tuple(s.shape) for s in state[1]] == [(1, 5), (1, 5)]
  with pytest.raises(ValueError):
    q_rnn_network.QRnnNetwork(obs_spec, act_spec, device=cuda)          # no lstm_size
  with pytest.raises(ValueError):
    q_rnn_network.QRnnNetwork(obs_spec, tensor_spec.BoundedTensorSpec((2,), torch.int32, 0, 1),
                              lstm_size=(4,), device=cuda)


def test_q_rnn_network_sequence_equals_chained_steps(cuda):
  rng = np.random.RandomState(5)
  B, T, D = 3, 12, 4
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32)
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 5)
  net = q_rnn_network.QRnnNetwork(obs_spec, act_spec, lstm_size=(10, 5), device=cuda).set_seed(2)
  obs = torch.as_tensor(rng.randn(B, T, D).astype(f32), device=cuda)
  st = np.ones((B, T), np.int32)
  st[:, 0] = 0
  st[2, 6] = 0
  st = torch.as_tensor(st, device=cuda)
  full, fstate = net(obs, st, net.get_initial_state(B))
  state = net.get_initial_state(B)
  outs = []
  for t in range(T):
    o, state = net(obs[:, t], st[:, t], state)
    outs.append(o)
  step = torch.stack(outs, 1)
  assert tuple(full.shape) == (B, T, 6)
  rel = (step - full).abs().max().item() / full.abs().max().item()
  record_parity('q_rnn_network_chained', rel=rel)
  # the B*T-row and B-row GEMMs of the fc layers may take different routes
  assert rel <= 1e-5
  for a, b in zip(_leaves(fstate), _leaves(state)):
    assert (a - b).abs().max().item() <= 1e-5 * max(1.0, b.abs().max().item())


def test_copy_is_independent(cuda):
  obs_spec = tensor_spec.TensorSpec((4,), torch.float32)
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 2)
  net = q_rnn_network.QRnnNetwork(obs_spec, act_spec, input_fc_layer_params=(8,), lstm_size=(6,),
                                  output_fc_layer_params=(8,), device=cuda).set_seed(1)
  net.create_variables()
  obs = torch.randn(5, 7, 4, device=cuda)
  st = torch.ones(5, 7, dtype=torch.int32, device=cuda)
  st[:, 0] = 0
  before, _ = net(obs, st)
  before = before.clone()
  cp = net.copy(name='Target')
  with torch.no_grad():
    cp.flat_params.copy_(net.flat_params)
  same, _ = cp(obs, st)
  assert torch.equal(same, before)
  for layers in ('_pre', '_cells', '_post'):
    for a, b in zip(getattr(cp, layers), getattr(net, layers)):
      assert a is not b
  with torch.no_grad():
    cp.flat_params.add_(torch.randn_like(cp.flat_params) * 0.1)
  after, _ = cp(obs, st)
  assert not torch.allclose(after, before)
  orig, _ = net(obs, st)
  assert torch.equal(orig, before)


# ---- policies -----------------------------------------------------------------------------------
def _time_step(cuda, step_type, obs):
  B = obs.shape[0]
  return ts.TimeStep(torch.full((B,), step_type, dtype=torch.int32, device=cuda),
                     torch.zeros(B, device=cuda), torch.ones(B, device=cuda), obs)


def test_stateful_q_policies(cuda):
  agent, net = _build(cuda, 4, 3)
  B = 6
  obs = torch.randn(B, 4, device=cuda)
  greedy, collect = agent.policy, agent.collect_policy
  assert greedy.policy_state_spec == net.state_spec == collect.policy_state_spec
  s0 = greedy.get_initial_state(B)
  a1 = greedy.action(_time_step(cuda, 0, obs), s0)
  a2 = greedy.action(_time_step(cuda, 1, obs), a1.state)
  assert not all(torch.equal(x, y) for x, y in zip(_leaves(a1.state), _leaves(a2.state)))
  a3 = greedy.action(_time_step(cuda, 0, obs), a2.state)        # FIRST resets
  for x, y in zip(_leaves(a3.state), _leaves(a1.state)):
    assert torch.equal(x, y)
  q1, _ = net(obs, torch.zeros(B, dtype=torch.int32, device=cuda), s0)
  assert torch.equal(a1.action.long(), q1.argmax(1))
  # epsilon 1: every action is random, the state is still the greedy branch's
  rand = q_policy.EpsilonGreedyPolicy(agent.policy.wrapped_policy, epsilon=1.0, seed=3)
  r1 = rand.action(_time_step(cuda, 0, obs), s0)
  r2 = rand.action(_time_step(cuda, 1, obs), r1.state)
  for x, y in zip(_leaves(r2.state), _leaves(a2.state)):
    assert torch.equal(x, y)
  for pol in (greedy, collect):
    with pytest.raises(ValueError, match='stateful'):
      pol.action(_time_step(cuda, 0, obs))


def test_feed_forward_policy_launches_unchanged(cuda):
  """A feed-forward greedy or epsilon-greedy action is the Q network's launches plus the one
  selection launch, and keeps the empty state."""
  obs_spec = tensor_spec.TensorSpec((4,), torch.float32)
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 2)
  net = q_network.QNetwork(obs_spec, act_spec, fc_layer_params=(16,), device=cuda)
  agent = dqn_agent.DqnAgent(ts.time_step_spec(obs_spec), act_spec, q_network=net,
                             optimizer=optimizers.AdamOptimizer(1e-3))
  agent.initialize()
  obs = torch.randn(8, 4, device=cuda)
  n0 = _lib.launch_count()
  net(obs)
  per_net = _lib.launch_count() - n0
  for pol in (agent.policy, agent.collect_policy):
    assert pol.policy_state_spec == () and pol.get_initial_state(8) == ()
    n0 = _lib.launch_count()
    step = pol.action(_time_step(cuda, 1, obs))
    assert _lib.launch_count() - n0 == per_net + 1
    assert step.state == ()


# ---- graphs and restore ---------------------------------------------------------------------------
def _collect_setup(cuda, B):
  agent, _ = _build(cuda, 4, 2, epsilon_greedy=0.3, seed=0)
  obs_spec = tensor_spec.TensorSpec((4,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 1, 'action')
  env = random_tf_environment.RandomTFEnvironment(ts.time_step_spec(obs_spec), act_spec,
                                                  batch_size=B, episode_end_probability=0.2,
                                                  seed=3, device=cuda)
  rb = rb_mod.TFUniformReplayBuffer(agent.collect_data_spec, batch_size=B, max_length=64,
                                    device=cuda)
  driver = dynamic_step_driver.DynamicStepDriver(env, agent.collect_policy,
                                                 observers=[rb.add_batch], num_steps=B * 4)
  return agent, env, rb, driver


def test_stateful_collect_graph_replays_bit_for_bit(cuda):
  """12 runs of 4 epsilon-greedy steps with the recurrent state threaded through the driver:
  captured into one CUDA graph, they store the same trajectories and end in the same state, bit
  for bit, as 12 eager runs."""
  B = 8
  out = []
  for graphed in (False, True):
    agent, env, rb, driver = _collect_setup(cuda, B)
    run = lambda t, s: driver.run(t, s, maximum_iterations=4)
    if graphed:
      run = common.function(run)
    time_step, state = env.reset(), agent.collect_policy.get_initial_state(B)
    for _ in range(12):
      time_step, state = run(time_step, state)
    exp = rb.gather_all()
    out.append([t.clone() for t in _leaves(exp)] + [t.clone() for t in _leaves(state)])
  assert int((out[0][0] == 0).sum()) > B
  for a, b in zip(*out):
    assert torch.equal(a, b)


def test_train_graph_replays_bit_for_bit(cuda, ffma):
  rng = np.random.RandomState(6)
  B, T, D, A = 4, 11, 5, 3
  make = lambda: _build(cuda, D, A, dqn_agent.DdqnAgent, masked=True, gradient_clipping=1.0,
                        target_update_tau=0.5, l2=0.01)[0]
  eager, graphed = make(), make()
  train_fn = common.function(graphed.train)
  for _ in range(5):
    traj = _to_traj(cuda, _experience(rng, B, T, D, A, True))
    l1 = eager.train(traj).loss.item()
    l2 = train_fn(traj).loss.item()
    assert l1 == l2
  assert torch.equal(graphed._q_network.flat_params, eager._q_network.flat_params)
  assert torch.equal(graphed._target_q_network.flat_params, eager._target_q_network.flat_params)
  assert int(graphed._seq_ticket.item()) == 0


def test_learner_restores_bit_for_bit(cuda, tmp_path, ffma):
  rng = np.random.RandomState(8)
  B, T, D, A = 4, 9, 5, 2
  exps = [_to_traj(cuda, _experience(rng, B, T, D, A, False)) for _ in range(4)]
  ds = lambda: iter([(e, ()) for e in exps])
  a1, _ = _build(cuda, D, A, target_update_tau=0.3, seed=0)
  l1 = learner_lib.Learner(str(tmp_path / 'run'), a1.train_step_counter, a1,
                           experience_dataset_fn=ds, checkpoint_interval=1)
  l1.run(iterations=2)
  a2, _ = _build(cuda, D, A, target_update_tau=0.3, seed=1)
  l2 = learner_lib.Learner(str(tmp_path / 'run'), a2.train_step_counter, a2,
                           experience_dataset_fn=lambda: iter([(e, ()) for e in exps[2:]]),
                           checkpoint_interval=0)
  assert int(a2.train_step_counter.item()) == 2
  for k, v in learner_lib._agent_state_tensors(a1).items():
    assert torch.equal(learner_lib._agent_state_tensors(a2)[k], v), k
  i1, i2 = l1.run(iterations=2), l2.run(iterations=2)
  assert i1.loss.item() == i2.loss.item()
  assert torch.equal(a1._q_network.flat_params, a2._q_network.flat_params)
  assert torch.equal(a1._target_q_network.flat_params, a2._target_q_network.flat_params)


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
  cols = dict(step_type=[], observation=[], action=[], reward=[], discount=[], next_step_type=[])
  last = None
  for t in range(CUE_STEPS + 1):
    st = 0 if t == 0 else (LAST if t == CUE_STEPS else 1)
    step_type = torch.full((B,), st, dtype=torch.int32, device=cuda)
    obs = obs0 if t == 0 else zeros
    step = policy.action(ts.TimeStep(step_type, torch.zeros(B, device=cuda),
                                     torch.ones(B, device=cuda), obs), state)
    state = step.state
    done = t == CUE_STEPS - 1
    if done:
      last = step.action
    reward = (step.action == (cue > 0).to(step.action.dtype)).float() if done else \
        torch.zeros(B, device=cuda)
    cols['step_type'].append(step_type)
    cols['observation'].append(obs)
    cols['action'].append(step.action)
    cols['reward'].append(reward)
    cols['discount'].append(torch.zeros(B, device=cuda) if done else torch.ones(B, device=cuda))
    nxt = LAST if done else (0 if t == CUE_STEPS else 1)
    cols['next_step_type'].append(torch.full((B,), nxt, dtype=torch.int32, device=cuda))
  stk = lambda k: torch.stack(cols[k], 1)
  traj = trajectory.Trajectory(stk('step_type'), stk('observation'), stk('action'), (),
                               stk('next_step_type'), stk('reward'), stk('discount'))
  return traj, last


def _cue_accuracy(recurrent, seed):
  cuda = torch.device('cuda')
  obs_spec = tensor_spec.TensorSpec((2,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 1, 'action')
  if recurrent:
    net = q_rnn_network.QRnnNetwork(obs_spec, act_spec, input_fc_layer_params=(32,),
                                    lstm_size=(16,), output_fc_layer_params=(32,),
                                    device=cuda).set_seed(seed)
  else:
    net = q_network.QNetwork(obs_spec, act_spec, fc_layer_params=(32, 32),
                             device=cuda).set_seed(seed)
  agent = dqn_agent.DqnAgent(ts.time_step_spec(obs_spec), act_spec, q_network=net,
                             optimizer=optimizers.AdamOptimizer(3e-3), epsilon_greedy=0.3,
                             target_update_tau=0.05, gamma=1.0, seed=seed)
  agent.initialize()
  gen = torch.Generator(device='cpu').manual_seed(seed)
  cue_of = lambda n: (torch.randint(0, 2, (n,), generator=gen).float() * 2 - 1).to(cuda)
  for _ in range(300):
    traj, _ = _cue_episode(agent.collect_policy, cuda, cue_of(64))
    if recurrent:
      agent.train(traj)
    else:                       # the feed-forward agent trains on the episode's transitions
      agent.train(trajectory.Trajectory(*[
          t.unfold(1, 2, 1).reshape(-1, 2) if isinstance(t, torch.Tensor) and t.dim() == 2 else
          (t.unfold(1, 2, 1).permute(0, 1, 3, 2).reshape(-1, 2, t.shape[-1])
           if isinstance(t, torch.Tensor) else t) for t in traj]))
  agent.check_numerics()
  cue = cue_of(1024)
  _, last = _cue_episode(agent.policy, cuda, cue)
  return float((last == (cue > 0).to(last.dtype)).float().mean())


def test_cue_recall_needs_memory(cuda):
  """A +-1 cue at the first step, zeros after it, and a reward for matching the cue's sign at the
  last of three decisions: recurrent DQN learns it from whole-episode [B, 4] sequences;
  feed-forward DQN cannot do better than chance (its observation at the last decision carries no
  information)."""
  rnn = _cue_accuracy(True, 0)
  ff = _cue_accuracy(False, 0)
  record_parity('dqn_rnn_cue_recall', recurrent_accuracy=rnn, feed_forward_accuracy=ff)
  assert rnn > 0.9, rnn
  assert abs(ff - 0.5) < 0.1, ff
