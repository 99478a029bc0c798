"""CategoricalDqnAgent (C51) on the GPU: the fused loss and expected-Q kernels against float64
autograd and the numpy oracle, the reference's goldens through the kernel and the agent, train
parity against CategoricalDqnOracle, graph replay, checkpoints and the constructor errors."""
import tempfile

import numpy as np
import pytest
import torch

from conftest import record_parity
from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.agents.categorical_dqn import categorical_dqn_agent as c51
from agents_b200.networks import categorical_q_network
from agents_b200.networks import layers as L
from agents_b200.networks import sequential
from agents_b200.policies import categorical_q_policy
from agents_b200.policies import epsilon_greedy_policy
from agents_b200.policies import greedy_policy
from agents_b200.specs import tensor_spec
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory
from agents_b200.train import learner as learner_lib
from agents_b200.train.utils import train_utils
from agents_b200.utils import common
from oracle import categorical_dqn as oc51
from oracle import nn as onn
from oracle import optim as ooptim
from oracle import philox
from test_oracle_categorical_dqn import _torch_loss

pytestmark = pytest.mark.gpu
f32 = np.float32
CANARY = 12345.0


# ---- the loss kernel ------------------------------------------------------------------------------
def _call_loss(cuda, q, nxt, actions, reward, discount, z, gamma, scale, mask=None, stride=1,
               zsel=None):
  B, A, N = q.shape
  T = reward.shape[1]
  d = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=cuda)
  act_store = np.zeros((B, stride), np.int32)
  act_store[:, 0] = actions
  act_store[:, 1:] = -7                                   # other columns must not be read
  t_act = d(act_store)
  canary = lambda n: torch.full((n + 8,), CANARY, dtype=torch.float32, device=cuda)
  loss, dq, rows = canary(1), canary(B * A * N), canary(B)
  flag = torch.zeros(1, dtype=torch.int32, device=cuda)
  tq, tn, tr, td_, tz = d(q.reshape(B, -1)), d(nxt.reshape(B, -1)), d(reward), d(discount), d(z)
  tm = d(mask.astype(np.int32)) if mask is not None else None
  tzs = d(zsel) if zsel is not None else None
  _lib.call('b200rl_c51_loss', _lib.ptr(tq), _lib.ptr(tn), _lib.ptr(tm), _lib.dptr(t_act), stride,
            _lib.ptr(tr), _lib.ptr(td_), _lib.ptr(tz), _lib.ptr(tzs), B, A, N, T, float(gamma), float(scale),
            float(B), _lib.ptr(loss), _lib.ptr(dq), _lib.ptr(flag), _lib.ptr(rows), 4 * B,
            _lib.stream())
  for buf, n in ((loss, 1), (dq, B * A * N), (rows, B)):
    assert torch.all(buf[n:] == CANARY), 'write past the end of an output'
  return loss[0].item(), dq[:B * A * N].cpu().numpy().reshape(B, A, N), int(flag.item())


def _case(A, N, T, masked, seed):
  rng = np.random.RandomState(seed)
  B = 37
  q = (rng.randn(B, A, N) * 2).astype(f32)
  nxt = (rng.randn(B, A, N) * 2).astype(f32)
  actions = rng.randint(0, A, size=B).astype(np.int32)
  reward = (rng.randn(B, T) * 3).astype(f32)
  reward[0], reward[1] = 40.0, -40.0                      # Tz clipped at both ends
  z = oc51.tf_linspace(-10.0, 10.0, N)
  reward[2] = 0.0                                         # with gamma = scale = 1 these two rows
  reward[3] = z[-2]                                       # put every Tz_j exactly on an atom
  discount = (rng.rand(B, T) > 0.2).astype(f32)
  discount[2] = 1.0
  discount[3] = 0.0
  mask = None
  if masked:
    mask = (rng.rand(B, A) > 0.4).astype(np.int32)
    mask[:, rng.randint(A)] = 1
    # rows where the unmasked greedy action is masked
    qv = oc51.convert_q_logits_to_values(nxt, z)
    best = qv.argmax(1)
    if A > 1:
      mask[:8][np.arange(8), best[:8]] = 0
      mask[:8][np.arange(8), (best[:8] + 1) % A] = 1
  return q, nxt, actions, reward, discount, z, mask


@pytest.mark.parametrize('A', [1, 2, 6, 18])
@pytest.mark.parametrize('N', [2, 5, 51, 201])
def test_loss_kernel_parity(cuda, A, N):
  for T in (2, 3, 4):
    for masked in (False, True):
      q, nxt, actions, reward, discount, z, mask = _case(A, N, T, masked, A * 1000 + N * 10 + T)
      gamma, scale = (1.0, 1.0) if masked else (0.95, 0.7)
      stride = 3 if masked else 1
      got, dq, flag = _call_loss(cuda, q, nxt, actions, reward, discount, z, gamma, scale, mask,
                                 stride)
      assert flag == 0
      want = oc51.c51_loss(q, nxt, actions, reward, discount, z, gamma, scale, next_mask=mask)
      ref, ref_dq, _ = _torch_loss(q, nxt, actions, reward, discount, z, gamma, scale, mask)
      rel = abs(got - ref) / abs(ref)
      dq_err = float(np.abs(dq - ref_dq).max() / np.abs(ref_dq).max())
      record_parity('c51_loss_kernel', loss_rel=rel, dq_rel_max=dq_err)
      assert rel <= 1e-5, (T, masked, got, ref)
      np.testing.assert_allclose(got, want['loss'], rtol=1e-5)
      assert dq_err <= 1e-4, (T, masked, dq_err)
      np.testing.assert_allclose(dq, want['dlogits'], rtol=0, atol=1e-4 * np.abs(want['dlogits']).max())
      other = np.ones_like(dq, dtype=bool)
      other[np.arange(len(actions)), actions] = False
      assert np.all(dq[other] == 0)


def test_loss_kernel_selects_with_the_policy_support(cuda):
  """The greedy action at s_n comes from select_support (the target policy's own atoms), the
  projection from support: with a reversed selection support the argmax flips."""
  q, nxt, actions, reward, discount, z, mask = _case(6, 51, 3, True, 11)
  for zsel in (oc51.policy_support(-10.0, 10.0, 51), -z):
    got, dq, flag = _call_loss(cuda, q, nxt, actions, reward, discount, z, 0.9, 0.5, mask,
                               zsel=zsel)
    want = oc51.c51_loss(q, nxt, actions, reward, discount, z, 0.9, 0.5, next_mask=mask,
                         select_support=zsel)
    assert flag == 0
    np.testing.assert_allclose(got, want['loss'], rtol=1e-5)
    np.testing.assert_allclose(dq, want['dlogits'], rtol=0, atol=1e-4 * np.abs(want['dlogits']).max())
  flipped = oc51.c51_loss(q, nxt, actions, reward, discount, z, 0.9, 0.5, next_mask=mask,
                          select_support=-z)
  same = oc51.c51_loss(q, nxt, actions, reward, discount, z, 0.9, 0.5, next_mask=mask)
  assert (flipped['best'] != same['best']).any()


@pytest.mark.parametrize('B,A,N', [(5000, 6, 51), (400, 2, 1024)])
def test_loss_kernel_launch_shapes(cuda, B, A, N):
  """B = 5000: more rows than the grid has warps (the row loop strides); N = 1024 at B = 400:
  the atom cap, three warps and 36 KB of shared memory per block.  The float64 reference runs in
  row chunks."""
  rng = np.random.RandomState(B + N)
  q = (rng.randn(B, A, N) * 2).astype(f32)
  nxt = (rng.randn(B, A, N) * 2).astype(f32)
  actions = rng.randint(0, A, size=B).astype(np.int32)
  reward = (rng.randn(B, 3) * 4).astype(f32)
  discount = (rng.rand(B, 3) > 0.2).astype(f32)
  z = oc51.tf_linspace(-10.0, 10.0, N)
  got, dq, flag = _call_loss(cuda, q, nxt, actions, reward, discount, z, 0.97, 0.8)
  assert flag == 0
  chunk = 25 if N > 256 else 1000
  total, ref_dq = 0.0, np.zeros((B, A, N))
  for lo in range(0, B, chunk):
    s = slice(lo, lo + chunk)
    n = len(actions[s])
    l, g, _ = _torch_loss(q[s], nxt[s], actions[s], reward[s], discount[s], z, 0.97, 0.8, None)
    total += l * n / B
    ref_dq[s] = g * n / B
  rel = abs(got - total) / abs(total)
  dq_err = float(np.abs(dq - ref_dq).max() / np.abs(ref_dq).max())
  record_parity('c51_loss_kernel', loss_rel=rel, dq_rel_max=dq_err)
  assert rel <= 1e-5 and dq_err <= 1e-4, (rel, dq_err)


def test_loss_kernel_deterministic_and_flags(cuda):
  q, nxt, actions, reward, discount, z, mask = _case(6, 51, 3, True, 7)
  a = _call_loss(cuda, q, nxt, actions, reward, discount, z, 0.99, 1.0, mask)
  b = _call_loss(cuda, q, nxt, actions, reward, discount, z, 0.99, 1.0, mask)
  assert a[0] == b[0] and np.array_equal(a[1], b[1])
  bad = actions.copy()
  bad[0], bad[1] = -1, 6                                  # clamped to 0 and 5, flag raised
  got, dq, flag = _call_loss(cuda, q, nxt, bad, reward, discount, z, 0.99, 1.0, mask)
  assert flag == 1
  want = oc51.c51_loss(q, nxt, np.clip(bad, 0, 5), reward, discount, z, 0.99, 1.0, next_mask=mask)
  np.testing.assert_allclose(got, want['loss'], rtol=1e-5)
  q2 = q.copy()
  q2[0, actions[0], 0] = np.inf
  assert _call_loss(cuda, q2, nxt, actions, reward, discount, z, 0.99, 1.0, mask)[2] == 1
  with pytest.raises(ValueError, match='num_atoms'):
    _call_loss(cuda, q[:, :, :1], nxt[:, :, :1], actions, reward, discount, z[:1], 0.99, 1.0)
  with pytest.raises(ValueError, match='at least 2'):
    _call_loss(cuda, q, nxt, actions, reward[:, :1], discount[:, :1], z, 0.99, 1.0)


# ---- goldens (categorical_dqn_agent_test.py) ----------------------------------------------------
class _CatNet(sequential.Sequential):
  """A Sequential read as [B, A, N] logits (the reference test's DummyCategoricalNet shape)."""

  def __init__(self, layers, num_actions, num_atoms, input_spec=None, device='cuda'):
    super(_CatNet, self).__init__(layers, input_spec=input_spec, device=device)
    self._num_actions, self.num_atoms = num_actions, num_atoms

  def create_variables(self, input_tensor_spec=None, **kwargs):
    super(_CatNet, self).create_variables(input_tensor_spec, **kwargs)
    return tensor_spec.TensorSpec((self._num_actions, self.num_atoms), torch.float32)


def _dummy_net(cuda):
  w = np.array([np.concatenate((np.arange(51), np.ones(51))), np.ones(102)], f32)
  return _CatNet([L.Dense(102, kernel_initializer=w, bias_initializer=1.0)], 2, 51, device=cuda)


def _specs(with_mask=False):
  obs = tensor_spec.TensorSpec([2], torch.float32)
  if with_mask:
    obs = (obs, tensor_spec.BoundedTensorSpec([2], torch.int32, 0, 1))
  return ts.time_step_spec(obs), tensor_spec.BoundedTensorSpec((), torch.int32, 0, 1)


def _exp(cuda, obs_seq, masks=None):
  T = len(obs_seq)
  t = lambda a, dt: torch.as_tensor(np.stack(a, axis=1), device=cuda).to(dt)
  obs = t([np.asarray(o, f32) for o in obs_seq], torch.float32)
  if masks is not None:
    obs = (obs, t([np.asarray(m, np.int32) for m in masks], torch.int32))
  return trajectory.Trajectory(
      step_type=t([np.zeros(2)] + [np.ones(2)] * (T - 1), torch.int32), observation=obs,
      action=t([np.array([0, 1])] * T, torch.int32), policy_info=(),
      next_step_type=t([np.ones(2)] * T, torch.int32),
      reward=t([np.array([10, 20])] * T, torch.float32),
      discount=t([np.array([.9, .9])] * T, torch.float32))


TWO = [[[1, 2], [3, 4]], [[5, 6], [7, 8]]]


def test_goldens_through_the_agent(cuda):
  """testCriticLoss 2.19525, testCriticLossWithMaskedActions 5.062895, testCriticLossNStep
  2.19525, testTrain 2.19525; `weights` does not change the loss (:463-466)."""
  tss, acts = _specs()
  agent = c51.CategoricalDqnAgent(tss, acts, _dummy_net(cuda), None)
  agent.initialize()
  info = agent._loss(_exp(cuda, TWO))
  np.testing.assert_allclose(info.loss.item(), 2.19525, atol=1e-4)
  assert info.extra.td_loss == () and info.extra.td_error == ()
  w = torch.tensor([0.0, 3.0], device=cuda)
  assert agent.loss(_exp(cuda, TWO), weights=w).loss.item() == info.loss.item()
  tss_m, _ = _specs(with_mask=True)
  agent = c51.CategoricalDqnAgent(tss_m, acts, _dummy_net(cuda), None,
                                  observation_and_action_constraint_splitter=lambda x: (x[0], x[1]))
  agent.initialize()
  loss = agent._loss(_exp(cuda, TWO, masks=[[[1, 0], [0, 1]], [[0, 1], [1, 0]]])).loss
  np.testing.assert_allclose(loss.item(), 5.062895, atol=1e-4)
  agent = c51.CategoricalDqnAgent(tss, acts, _dummy_net(cuda), None, n_step_update=2)
  agent.initialize()
  loss = agent._loss(_exp(cuda, TWO + [[[9, 10], [11, 12]]])).loss
  np.testing.assert_allclose(loss.item(), 2.19525, atol=1e-4)
  agent = c51.CategoricalDqnAgent(tss, acts, _dummy_net(cuda), optimizers.AdamOptimizer(0.01))
  agent.initialize()
  info = agent.train(_exp(cuda, TWO), weights=None)
  np.testing.assert_allclose(info.loss.item(), 2.19525, atol=1e-4)
  assert int(agent.train_step_counter.item()) == 1
  agent.check_numerics()


def test_goldens_through_the_kernel(cuda):
  net = oc51.CategoricalDqnOracle(onn.Sequential([dict(
      kind='dense', w=np.array([np.concatenate((np.arange(51), np.ones(51))), np.ones(102)], f32),
      b=np.ones(102, f32), act=None)]), None, 51).q_net
  z = oc51.tf_linspace(-10.0, 10.0, 51)
  q = net.forward(np.array([[1, 2], [3, 4]], f32)).reshape(2, 2, 51)
  for obs_n, T, mask, want in ((TWO[1], 2, None, 2.19525), (TWO[1], 2, [[0, 1], [1, 0]], 5.062895),
                               ([[9, 10], [11, 12]], 3, None, 2.19525)):
    nxt = net.forward(np.array(obs_n, f32)).reshape(2, 2, 51)
    rew = np.tile(np.array([[10], [20]], f32), (1, T))
    got = _call_loss(cuda, q, nxt, np.array([0, 1], np.int32), rew, np.full((2, T), 0.9, f32), z,
                     1.0, 1.0, None if mask is None else np.array(mask))[0]
    np.testing.assert_allclose(got, want, atol=1e-4)


# ---- q values / policies ------------------------------------------------------------------------
@pytest.mark.parametrize('B,A,N', [(1, 6, 51), (256, 6, 51), (33, 18, 201), (5, 2, 2)])
def test_q_values_kernel_and_greedy(cuda, B, A, N):
  rng = np.random.RandomState(B + A + N)
  logits = (rng.randn(B, A, N) * 2).astype(f32)
  logits[:, 1 % A] = logits[:, 0]                         # ties: the first action must win
  z = oc51.policy_support(-10.0, 10.0, N)
  tl, tz = torch.as_tensor(logits, device=cuda), torch.as_tensor(z, device=cuda)
  q = torch.empty(B, A, device=cuda)
  _lib.call('b200rl_c51_q_values', _lib.ptr(tl), _lib.ptr(tz), B, A, N, _lib.ptr(q), _lib.stream())
  p64 = torch.softmax(torch.as_tensor(logits, dtype=torch.float64), -1)
  ref = (p64 * torch.as_tensor(z, dtype=torch.float64)).sum(-1).numpy()
  err = float(np.abs(q.cpu().numpy() - ref).max())
  record_parity('c51_q_values', abs_max=err)
  assert err <= 1e-5
  np.testing.assert_allclose(q.cpu().numpy(), oc51.convert_q_logits_to_values(logits, z), atol=2e-6)
  # the policy stack: greedy == the oracle's first argmax, epsilon-greedy == the Philox oracle
  obs_spec = tensor_spec.TensorSpec([N], torch.float32)
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, A - 1)

  class _Id(_CatNet):
    def __call__(self, observation, step_type=None, network_state=(), training=False):
      return observation, network_state

  net = _Id([L.Dense(1)], A, N, input_spec=tensor_spec.TensorSpec([A * N], torch.float32),
            device=cuda)
  pol = categorical_q_policy.CategoricalQPolicy(ts.time_step_spec(obs_spec), act_spec, net,
                                                -10.0, 10.0)
  step = ts.restart(tl.reshape(B, A * N), batch_size=B)
  qq = q.cpu().numpy()
  best = oc51.greedy_action(qq)
  np.testing.assert_array_equal(greedy_policy.GreedyPolicy(pol).action(step).action.cpu().numpy(),
                                best)
  eps = epsilon_greedy_policy.EpsilonGreedyPolicy(pol, epsilon=0.5, seed=11)
  seed = (11 ^ greedy_policy._POLICY_SEED_TAG) & 0xFFFFFFFFFFFFFFFF
  for call in range(2):
    got = eps.action(step).action.cpu().numpy()
    r = philox.philox(np.arange(B, dtype=np.uint64), call, seed)
    u = philox.uniform_f32(r[0])
    want = np.where(u >= f32(0.5), best, (r[1] % np.uint32(A)).astype(np.int64))
    np.testing.assert_array_equal(got, want)


# ---- train parity -------------------------------------------------------------------------------
def _mirror(net, l2=None):
  out = []
  for l in net.layers:
    if isinstance(l, L.CastScale): out.append(dict(kind='cast_scale', divisor=l.divisor))
    elif isinstance(l, L.Conv2D): out.append(dict(kind='conv', w=l.kernel.cpu().numpy().copy(), b=l.bias.cpu().numpy().copy(), stride=l.stride, act=l.activation))
    elif isinstance(l, L.Flatten): out.append(dict(kind='flatten'))
    else: out.append(dict(kind='dense', w=l.kernel.cpu().numpy().copy(), b=l.bias.cpu().numpy().copy(), act=l.activation, l2=l.l2))
  return onn.Sequential(out)


def _random_exp(rng, B, T, obs_shape, A, u8):
  obs = (rng.randint(0, 256, size=(B, T) + obs_shape).astype(np.uint8) if u8
         else rng.randn(B, T, *obs_shape).astype(f32))
  return dict(observation=obs, step_type=rng.randint(0, 3, size=(B, T)).astype(np.int32),
              action=rng.randint(0, A, size=(B, T)).astype(np.int32),
              next_step_type=rng.randint(0, 3, size=(B, T)).astype(np.int32),
              reward=(rng.randn(B, T) * 3).astype(f32), discount=(rng.rand(B, T) > 0.1).astype(f32))


def _to_traj(cuda, e):
  d = lambda a: torch.as_tensor(a, device=cuda)
  return trajectory.Trajectory(d(e['step_type']), d(e['observation']), d(e['action']), (),
                               d(e['next_step_type']), d(e['reward']), d(e['discount']))


def test_train_parity_atari_config(cuda):
  """The Atari example's net on 84x84x4 uint8 (conv (32,8,4)(64,4,2)(64,3,1), fc 512, A = 6,
  N = 51), B = 32, n_step 2, gamma 0.99, centered RMSProp: 5 steps against the oracle."""
  rng = np.random.RandomState(0)
  A, B, n = 6, 32, 2
  obs_spec = tensor_spec.TensorSpec((84, 84, 4), torch.uint8)
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, A - 1)
  net = categorical_q_network.CategoricalQNetwork(
      obs_spec, act_spec, preprocessing_layers=L.CastScale(255.),
      conv_layer_params=((32, 8, 4), (64, 4, 2), (64, 3, 1)), fc_layer_params=(512,),
      device=cuda).set_seed(1)
  opt = optimizers.RMSPropOptimizer(2.5e-4, decay=0.95, momentum=0.0, epsilon=1e-5, centered=True)
  agent = c51.CategoricalDqnAgent(ts.time_step_spec(obs_spec), act_spec, net, opt,
                                  n_step_update=n, gamma=0.99, target_update_period=2)
  agent.initialize()
  orc = oc51.CategoricalDqnOracle(_mirror(net), ooptim.RMSPropTF(
      2.5e-4, decay=0.95, momentum=0.0, eps=1e-5, centered=True, ms_init=1.0), 51, gamma=0.99,
      target_update_period=2)
  for _ in range(5):
    e = _random_exp(rng, B, n + 1, (84, 84, 4), A, True)
    want = orc.train(e)
    got = agent.train(_to_traj(cuda, e)).loss.item()
    record_parity('c51_train_atari', loss_rel=abs(got - want['loss']) / abs(want['loss']))
    np.testing.assert_allclose(got, want['loss'], rtol=1e-5)
  agent.check_numerics()


def _mlp_agent(cuda, seed, l2=1e-3, **kw):
  obs_spec = tensor_spec.TensorSpec((6,), torch.float32)
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 2)
  net = _CatNet([L.Dense(32, activation='relu', kernel_regularizer_l2=l2),
                 L.Dense(3 * 21, kernel_regularizer_l2=l2)], 3, 21, input_spec=obs_spec,
                device=cuda).set_seed(seed)
  agent = c51.CategoricalDqnAgent(ts.time_step_spec(obs_spec), act_spec, net,
                                  optimizers.AdamOptimizer(1e-2), min_q_value=-5.0,
                                  max_q_value=5.0, gamma=0.9, reward_scale_factor=0.5,
                                  gradient_clipping=0.5, target_update_tau=0.3,
                                  target_update_period=2, **kw)
  agent.initialize()
  return agent, net


def test_train_parity_mlp_adam_clip_l2_polyak(cuda):
  rng = np.random.RandomState(1)
  agent, net = _mlp_agent(cuda, 3)
  orc = oc51.CategoricalDqnOracle(_mirror(net), ooptim.AdamTF(1e-2, eps=1e-8), 21, -5.0, 5.0,
                                  gamma=0.9, reward_scale=0.5, target_update_tau=0.3,
                                  target_update_period=2, gradient_clipping=0.5)
  for step in range(5):
    e = _random_exp(rng, 64, 2, (6,), 3, False)
    if step == 0:                 # pre-optimiser gradients against float64 autograd
      params = [torch.as_tensor(p, dtype=torch.float64).requires_grad_(True)
                for p in orc.q_net.params()]
      tparams = [torch.as_tensor(p, dtype=torch.float64) for p in orc.target_net.params()]
    want = orc.train(e)
    got = agent.train(_to_traj(cuda, e)).loss.item()
    np.testing.assert_allclose(got, want['loss'], rtol=1e-5)
    if step == 0:
      _check_grads_float64(net, params, tparams, e)
  for v, w in zip(agent._target_q_network.variables, orc.target_net.params()):
    np.testing.assert_allclose(v.cpu().numpy(), w, rtol=1e-3, atol=1e-5)


def _check_grads_float64(net, params, tparams, e):
  from grad_refs import assert_grad_close
  w1, b1, w2, b2 = params

  def fwd(x, p):
    h = torch.relu(torch.as_tensor(x, dtype=torch.float64) @ p[0] + p[1])
    return (h @ p[2] + p[3]).reshape(-1, 3, 21)

  z = torch.as_tensor(oc51.tf_linspace(-5.0, 5.0, 21), dtype=torch.float64)
  q = fwd(e['observation'][:, 0], params)
  with torch.no_grad():
    nxt = fwd(e['observation'][:, -1], tparams)
    p = torch.softmax(nxt, -1)
    best = (p * z).sum(-1).argmax(-1)
    pb = p[torch.arange(len(best)), best]
    tz = (0.5 * torch.as_tensor(e['reward'][:, 0], dtype=torch.float64)[:, None] +
          0.9 * torch.as_tensor(e['discount'][:, 0], dtype=torch.float64)[:, None] * z)
    tz = tz.clamp(z[0], z[-1])
    m = ((1 - (tz[:, None, :] - z[None, :, None]).abs() / (z[1] - z[0])).clamp(0, 1) *
         pb[:, None, :]).sum(-1)
  l = q[torch.arange(len(best)), torch.as_tensor(e['action'][:, 0], dtype=torch.int64)]
  loss = (m * (torch.logsumexp(l, -1, keepdim=True) - l)).sum(-1).mean()
  loss = loss + 1e-3 * (w1 * w1).sum() + 1e-3 * (w2 * w2).sum()
  loss.backward()
  got = [g.cpu() for g in net._grad_views]
  for name, g, p in zip(('w1', 'b1', 'w2', 'b2'), got, params):
    ref = p.grad * (0.5 / torch.clamp(p.grad.norm(), min=0.5))          # clip_by_norm per variable
    assert_grad_close(f'c51 mlp {name}', g, ref, 1e-4, 1e-4)


def test_graph_replay_matches_eager_bit_for_bit(cuda):
  rng = np.random.RandomState(4)
  eager, _ = _mlp_agent(cuda, 5)
  graphed, _ = _mlp_agent(cuda, 5)
  train_fn = common.function(graphed.train)
  for _ in range(6):
    e = _random_exp(rng, 8, 2, (6,), 3, False)               # 8 rows: one CTA
    l1 = eager.train(_to_traj(cuda, e)).loss.item()
    l2 = train_fn(_to_traj(cuda, e)).loss.item()
    assert l1 == l2
  assert torch.equal(eager._q_network.flat_params, graphed._q_network.flat_params)
  assert torch.equal(eager._target_q_network.flat_params, graphed._target_q_network.flat_params)


def test_learner_checkpoint_restore_reproduces_losses(cuda):
  rng = np.random.RandomState(6)
  batches = [_random_exp(rng, 32, 2, (6,), 3, False) for _ in range(7)]
  root = tempfile.mkdtemp()

  def make(seed):
    step = train_utils.create_train_step(cuda)
    agent, _ = _mlp_agent(cuda, seed, train_step_counter=step)
    it = iter([_to_traj(cuda, e) for e in batches])
    return agent, step, learner_lib.Learner(root, step, agent, experience_dataset_fn=lambda: it,
                                            checkpoint_interval=4)

  agent, step, lrn = make(7)
  lrn.run(iterations=4)
  want = [agent.train(_to_traj(cuda, e)).loss.item() for e in batches[4:]]
  agent2, step2, _ = make(8)                                 # other weights, then restored
  assert int(step2.item()) == 4
  got = [agent2.train(_to_traj(cuda, e)).loss.item() for e in batches[4:]]
  assert got == want


def test_constructor_errors(cuda):
  tss, acts = _specs()
  plain = sequential.Sequential([L.Dense(102)], input_spec=tss.observation, device=cuda)
  with pytest.raises(TypeError, match='num_atoms'):
    c51.CategoricalDqnAgent(tss, acts, plain, None)
  other = _CatNet([L.Dense(10)], 2, 5, device=cuda)
  with pytest.raises(ValueError, match='different numbers of atoms'):
    c51.CategoricalDqnAgent(tss, acts, _dummy_net(cuda), None, target_categorical_q_network=other)
  with pytest.raises(ValueError, match='inner dims'):
    c51.CategoricalDqnAgent(tss, acts, _CatNet([L.Dense(102)], 3, 34, device=cuda), None)
  with pytest.raises(ValueError, match='Only scalar actions'):
    c51.CategoricalDqnAgent(tss, tensor_spec.BoundedTensorSpec([1, 2], torch.int32, 0, 1),
                            _dummy_net(cuda), None)
  with pytest.raises(ValueError, match='minimum of 0'):
    c51.CategoricalDqnAgent(tss, tensor_spec.BoundedTensorSpec((), torch.int32, 1, 2),
                            _dummy_net(cuda), None)
  with pytest.raises(NotImplementedError):
    c51.CategoricalDqnAgent(tss, acts, _dummy_net(cuda), None, epsilon_greedy=None,
                            boltzmann_temperature=1.0)
  rnn = _dummy_net(cuda)
  rnn._state_spec = (tensor_spec.TensorSpec([4], torch.float32),)
  with pytest.raises(NotImplementedError):
    c51.CategoricalDqnAgent(tss, acts, rnn, None)
  agent = c51.CategoricalDqnAgent(tss, acts, _dummy_net(cuda), None)
  agent.replicas = 2
  with pytest.raises(NotImplementedError):
    agent.loss(_exp(cuda, TWO))
  with pytest.raises(TypeError, match='BoundedTensorSpec'):
    categorical_q_network.CategoricalQNetwork(tss.observation,
                                              tensor_spec.TensorSpec((), torch.int32), device=cuda)
  net = categorical_q_network.CategoricalQNetwork(tss.observation, acts, num_atoms=7,
                                                  fc_layer_params=(4,), device=cuda)
  assert net.num_atoms == 7
  out, _ = net(torch.zeros(3, 2, device=cuda))
  assert tuple(out.shape) == (3, 2, 7)
  head = net.layers[-1]
  assert head.units == 14 and torch.all(head.bias == -0.2) and head.kernel.abs().max() <= 0.03


# ---- CartPole end to end ----------------------------------------------------------------------------
CARTPOLE_THRESHOLD = 150.0


def test_cartpole_end_to_end_learns(cuda):
  """Device CartPole (8 envs) -> DynamicStepDriver(epsilon-greedy collect policy, one step per
  iteration) -> TFUniformReplayBuffer -> get_next(64, 3) -> CategoricalDqnAgent.train, for 100
  collect-only iterations and then 6000 iterations (the C51 tutorial's agent: Dense(100), 51
  atoms on [-20, 20], n_step_update 2, gamma 0.99, Adam 1e-3, epsilon 0.1).  Then the greedy
  policy's mean first-episode length over 16 evaluation envs must reach CARTPOLE_THRESHOLD.
  Threshold: the same configuration run on the CPU through oracle/categorical_dqn.py (with the
  oracle CartPole, epsilon-greedy and uniform replay of oracle/env.py and oracle/replay.py) gave
  281.6, 289.7, 401.3, 335.5, 411.5, 303.9, 319.7 and 271.2 for seeds 0-7 (median ~311); an
  untrained greedy policy lasts about 9 steps.  150 sits well below the smallest of those."""
  from agents_b200.drivers import dynamic_step_driver
  from agents_b200.environments import random_tf_environment
  from agents_b200.replay_buffers import tf_uniform_replay_buffer as rb_mod
  envs, iters = 8, 6000
  env = random_tf_environment.CartPoleTFEnvironment(batch_size=envs, seed=0, device=cuda,
                                                    action_dtype=torch.int32)
  tss, act_spec = env.time_step_spec(), env.action_spec()
  net = categorical_q_network.CategoricalQNetwork(tss.observation, act_spec,
                                                  fc_layer_params=(100,), device=cuda).set_seed(0)
  agent = c51.CategoricalDqnAgent(tss, act_spec, net, optimizers.AdamOptimizer(1e-3),
                                  min_q_value=-20.0, max_q_value=20.0, n_step_update=2,
                                  gamma=0.99, epsilon_greedy=0.1)
  agent.initialize()
  rb = rb_mod.TFUniformReplayBuffer(agent.collect_data_spec, batch_size=envs, max_length=2000,
                                    device=cuda, seed=0)
  driver = dynamic_step_driver.DynamicStepDriver(env, agent.collect_policy,
                                                 observers=[rb.add_batch], num_steps=envs)
  time_step, policy_state = env.reset(), None
  for _ in range(100):
    time_step, policy_state = driver.run(time_step, policy_state, maximum_iterations=1)
  for _ in range(iters):
    time_step, policy_state = driver.run(time_step, policy_state, maximum_iterations=1)
    exp, _ = rb.get_next(sample_batch_size=64, num_steps=3)
    agent.train(exp)
  agent.check_numerics()
  ev = random_tf_environment.CartPoleTFEnvironment(batch_size=16, seed=7, device=cuda,
                                                   action_dtype=torch.int32)
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
  record_parity('c51_cartpole', mean_episode_length=mean_len)
  assert mean_len >= CARTPOLE_THRESHOLD, mean_len
