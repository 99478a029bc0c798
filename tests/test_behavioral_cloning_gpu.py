"""Behavioral cloning on the GPU: the behavioral_cloning.cu kernels against float64 across the
lane-group boundaries and past the grid cap, the Normal draws (supplied and device), the reference
golden through the agent, BehavioralCloningAgent.train against the numpy oracle, gradients before
the optimiser, graph replay of train and of the collect step, Learner checkpoints, the policies,
unsupported options and an offline learning check."""
import tempfile

import numpy as np
import pytest
import torch

import grad_refs as R
from conftest import record_parity
from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.agents.behavioral_cloning import behavioral_cloning_agent as bca
from agents_b200.networks import actor_distribution_network as adn
from agents_b200.networks import actor_network
from agents_b200.networks import layers as L
from agents_b200.networks import q_network
from agents_b200.networks import sequential
from agents_b200.networks import tanh_normal_projection_network as tnpn
from agents_b200.specs import tensor_spec
from agents_b200.train import learner as learner_lib
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory
from agents_b200.utils import common
from oracle import behavioral_cloning as obc
from oracle import nn as onn
from oracle import optim as ooptim

pytestmark = pytest.mark.gpu
f32 = np.float32
F64 = torch.float64


def _d(cuda, a):
  return torch.as_tensor(np.ascontiguousarray(a), device=cuda)


def _ws(cuda):
  return torch.empty(512, dtype=torch.float32, device=cuda)


# ---- 1. kernels against float64 -----------------------------------------------------------------
def _discrete(cuda, z, ld, act, a_stride, minimum, w, w_div, N, A):
  loss, pe = torch.empty(1, device=cuda), torch.empty(N, device=cuda)
  ld_g = A + 2
  g = torch.full((N, ld_g), 7.0, device=cuda)                     # canary columns
  flag, ws = torch.zeros(1, dtype=torch.int32, device=cuda), _ws(cuda)
  tz, ta = _d(cuda, z), _d(cuda, act)
  tw = None if w is None else _d(cuda, w)
  _lib.call('b200rl_bc_discrete_loss', _lib.ptr(tz), ld, _lib.ptr(ta), a_stride, minimum,
            _lib.ptr(tw), w_div, N, A, _lib.ptr(loss), _lib.ptr(pe), _lib.ptr(g), ld_g,
            _lib.ptr(flag), _lib.ptr(ws), ws.numel() * 4, _lib.stream())
  g = g.cpu()
  assert bool((g[:, A:] == 7).all())
  return loss.item(), pe.cpu(), g[:, :A], int(flag.item())


def _w_rows(w, w_div, N):
  return torch.ones(N, dtype=F64) if w is None else R.t64(np.repeat(w, w_div))


# (A, N): A on both sides of the lane-group boundaries; N past the 512-block cap of each group
# (131072 rows at G = 1, 16384 at G = 8, 4096 at G = 32)
_DISC = [(1, 300), (2, 140000), (8, 1000), (9, 17000), (64, 3000), (65, 5000), (1000, 4500)]


@pytest.mark.parametrize('A,N', _DISC)
def test_discrete_kernel_matches_float64(cuda, A, N):
  rng = np.random.RandomState(A * 7 + N)
  ld, a_stride, minimum = A + 3, 2, 3
  z = (rng.randn(N, ld) * 2).astype(f32)
  labels = rng.randint(0, A, N)
  act = np.zeros(N * a_stride, np.int32)
  act[::a_stride] = labels + minimum
  act[1::a_stride] = -77                                          # never read
  Z = R.t64(z[:, :A])
  ce = torch.logsumexp(Z, 1) - Z[torch.arange(N), torch.as_tensor(labels)]
  p = torch.softmax(Z, 1)
  onehot = torch.zeros_like(Z)
  onehot[torch.arange(N), torch.as_tensor(labels)] = 1
  for wkind in ('none', 'rows', 'batch', 'scalar'):
    w, w_div = None, 1
    zz = z
    if wkind == 'rows':
      w = rng.rand(N).astype(f32)
      w[0] = 0.0
      zz = z.copy()
      zz[0, 0] = np.nan                                           # zero weight on a NaN row
    elif wkind == 'batch':
      w_div = 4 if N % 4 == 0 else 1
      w = rng.rand(N // w_div).astype(f32)
    elif wkind == 'scalar':
      w, w_div = np.array([0.37], f32), N
    loss, pe, g, flag = _discrete(cuda, zz, ld, act, a_stride, minimum, w, w_div, N, A)
    W = _w_rows(w, w_div, N)
    keep = W != 0
    ref = (ce[keep] * W[keep]).sum() / N
    cond = (ce.abs() * W).sum() / N
    err = abs(loss - ref.item()) / max(cond.item(), 1e-30)
    record_parity(f'bc_discrete_A{A}_N{N}', **{f'{wkind}_loss_rel': err})
    assert err < 2e-5, (wkind, loss, ref.item())
    torch.testing.assert_close(pe[keep].double(), ce[keep], rtol=2e-6, atol=2e-5)
    want = (W / N)[:, None] * (p - onehot)
    torch.testing.assert_close(g[keep].double(), want[keep], rtol=1e-5, atol=1e-6 / N)
    assert flag == 0
    if wkind == 'rows':
      assert not bool(g[0].any()) and bool(torch.isnan(pe[0]))


def test_discrete_kernel_flags_out_of_range_label(cuda):
  N, A = 50, 5
  z = np.random.RandomState(0).randn(N, A).astype(f32)
  act = np.random.RandomState(1).randint(1, 1 + A, N).astype(np.int32)
  act[7] = 1 + A                                                  # label A: outside [0, A)
  w = np.ones(N, f32)
  loss, pe, _, flag = _discrete(cuda, z, A, act, 1, 1, w, 1, N, A)
  assert flag == 1 and bool(torch.isnan(pe[7])) and np.isnan(loss)
  assert bool(torch.isfinite(pe[torch.arange(N) != 7]).all())
  w[7] = 0.0                                                      # multiply_no_nan drops the row
  loss, pe, g, flag = _discrete(cuda, z, A, act, 1, 1, w, 1, N, A)
  assert flag == 1 and np.isfinite(loss) and not bool(g[7].any())


def _continuous(cuda, pred, scale, ld, target, ld_t, lo, hi, z, w, w_div, N, A, rng_ctr=None,
                advance=0, seed=5):
  loss, pe = torch.empty(1, device=cuda), torch.empty(N, device=cuda)
  ld_g = A + 1
  dp = torch.full((N, ld_g), 7.0, device=cuda)
  ds = torch.full((N, ld_g), 7.0, device=cuda) if scale is not None else None
  ts_ = [None if a is None else _d(cuda, a) for a in (pred, scale, target, lo, hi, z, w)]
  flag, ws = torch.zeros(1, dtype=torch.int32, device=cuda), _ws(cuda)
  p_, s_, t_, lo_, hi_, z_, w_ = [_lib.ptr(t) for t in ts_]
  _lib.call('b200rl_bc_continuous_loss', p_, s_, ld, t_, ld_t, lo_, hi_, z_, seed,
            _lib.ptr(rng_ctr), advance, w_, w_div, N, A, _lib.ptr(loss), _lib.ptr(pe),
            _lib.ptr(dp), _lib.ptr(ds), ld_g, _lib.ptr(flag), _lib.ptr(ws), ws.numel() * 4,
            _lib.stream())
  dp = dp.cpu()
  assert bool((dp[:, A:] == 7).all())
  if ds is not None:
    ds = ds.cpu()
    assert bool((ds[:, A:] == 7).all())
    ds = ds[:, :A]
  return loss.item(), pe.cpu(), dp[:, :A], ds, int(flag.item())


def _close_rows(what, got, want, cond, keep, name):
  """|got - want| <= 1e-5 |want| + 8u cond on the kept rows (u = 2^-24)."""
  err = ((got.double() - want).abs() - 1e-5 * want.abs())[keep]
  floor = (8 * 2.0 ** -24 * cond)[keep]
  record_parity(name, **{what + '_err_over_floor': float((err / floor.clamp_min(1e-300)).max())})
  assert bool((err <= floor).all()), (what, float(err.max()))


_CONT = [(1, 140000), (6, 4096), (8, 1000), (9, 17000), (65, 5000)]


@pytest.mark.parametrize('A,N', _CONT)
@pytest.mark.parametrize('mode', ['deterministic', 'normal'])
def test_continuous_kernel_matches_float64(cuda, A, N, mode):
  rng = np.random.RandomState(A * 3 + N)
  ld, ld_t = A + 2, A + 3
  pred = rng.uniform(-1, 1, (N, ld)).astype(f32)
  scale = rng.uniform(0.1, 1, (N, ld)).astype(f32) if mode == 'normal' else None
  target = rng.uniform(-2, 2, (N, ld_t)).astype(f32)
  lo, hi = rng.uniform(-3, -0.5, A).astype(f32), rng.uniform(0.5, 2, A).astype(f32)
  z = rng.randn(N, A).astype(f32) if mode == 'normal' else None
  Y, T = R.t64(pred[:, :A]), R.t64(target[:, :A])
  LO, HI = R.t64(lo), R.t64(hi)
  if mode == 'normal':
    Z = R.t64(z)
    a, dmul = Y + R.t64(scale[:, :A]) * Z, 1.0
    mag_a = Y.abs() + (R.t64(scale[:, :A]) * Z).abs()
  else:
    a, dmul = (HI + LO) / 2 + (HI - LO) / 2 * Y, (HI - LO) / 2
    mag_a = ((HI + LO) / 2).abs() + ((HI - LO) / 2 * Y).abs()
  d = a - T
  mse = (d * d).mean(1)
  for wkind in ('none', 'rows'):
    w = None
    pp = pred
    if wkind == 'rows':
      w = rng.rand(N).astype(f32)
      w[0] = 0.0
      pp = pred.copy()
      pp[0, 0] = np.inf
    loss, pe, dp, ds, flag = _continuous(cuda, pp, scale, ld, target, ld_t, lo, hi, z, w, 1, N, A)
    W = _w_rows(w, 1, N)
    keep = W != 0
    ref = (mse[keep] * W[keep]).sum() / N
    err = abs(loss - ref.item()) / max(((mse * W).sum() / N).item(), 1e-30)
    record_parity(f'bc_continuous_{mode}_A{A}_N{N}', **{f'{wkind}_loss_rel': err})
    assert err < 2e-5, (wkind, loss, ref.item())
    torch.testing.assert_close(pe[keep].double(), mse[keep], rtol=2e-6, atol=1e-6)
    gd = (2 * W / (N * A))[:, None] * d
    # a - t cancels: the float32 a - t carries an error of a few u times the magnitudes of the
    # terms that form it, so that is the floor
    cond = (2 * W / (N * A))[:, None] * (mag_a + T.abs())
    _close_rows('dpred', dp, dmul * gd, dmul * cond, keep, f'bc_continuous_{mode}_A{A}_N{N}')
    if mode == 'normal':
      _close_rows('dscale', ds, gd * Z, cond * Z.abs(), keep, f'bc_continuous_{mode}_A{A}_N{N}')
    if wkind == 'rows':
      assert not bool(dp[0].any()) and (ds is None or not bool(ds[0].any()))
    assert flag == 0


# ---- 2. Normal draws ----------------------------------------------------------------------------
def test_normal_supplied_draws_match_the_oracle(cuda):
  rng = np.random.RandomState(4)
  N, A = 700, 6
  loc, scale = rng.uniform(-1, 1, (N, A)).astype(f32), rng.uniform(.1, 1, (N, A)).astype(f32)
  t, z, w = rng.uniform(-1, 1, (N, A)).astype(f32), rng.randn(N, A).astype(f32), rng.rand(N).astype(f32)
  ctr = torch.zeros(2, dtype=torch.int64, device=cuda)
  loss, pe, dl, ds, _ = _continuous(cuda, loc, scale, A, t, A, None, None, z, w, 1, N, A, ctr)
  wl, wpe, wdl, wds = obc.continuous_loss(loc, t, w, scale=scale, z=z)
  np.testing.assert_allclose(loss, wl, rtol=1e-6)
  np.testing.assert_allclose(pe.numpy(), wpe, rtol=1e-6, atol=1e-7)
  cond = R.t64((2 * w / (N * A))[:, None] * (np.abs(loc) + np.abs(scale * z) + np.abs(t)))
  keep = torch.ones(N, dtype=torch.bool)
  _close_rows('dloc', dl, R.t64(wdl), cond, keep, 'bc_normal_supplied')
  _close_rows('dscale', ds, R.t64(wds), cond * R.t64(np.abs(z)), keep, 'bc_normal_supplied')
  assert ctr.cpu().tolist() == [0, 0]                             # supplied draws: no advance


def test_normal_device_draws_have_standard_moments(cuda):
  N, A = 200000, 5
  loc, scale = np.zeros((N, A), f32), np.ones((N, A), f32)
  t = np.full((N, A), -1.0, f32)                                  # a - t = z + 1, never 0
  ctr = torch.zeros(2, dtype=torch.int64, device=cuda)
  zs = []
  for call in range(2):
    _, _, dl, ds, _ = _continuous(cuda, loc, scale, A, t, A, None, None, None, None, 1, N, A, ctr,
                                  advance=1)
    zs.append((ds / dl).double().reshape(-1))                     # dscale = dloc * z
    assert ctr.cpu().tolist() == [call + 1, 0]
  for z in zs:
    n = z.numel()
    m, v = float(z.mean()), float(z.var())
    k4 = float(((z - m) ** 4).mean())
    record_parity('bc_normal_device_moments', mean_sigmas=abs(m) * n ** .5,
                  var_sigmas=abs(v - 1) / (2 / n) ** .5, kurtosis=k4)
    assert abs(m) < 5 / n ** .5 and abs(v - 1) < 5 * (2 / n) ** .5 and abs(k4 - 3) < 0.05
  assert not torch.equal(zs[0], zs[1])
  _, _, dl, ds, _ = _continuous(cuda, loc, scale, A, t, A, None, None, None, None, 1, N, A, ctr)
  _, _, dl2, ds2, _ = _continuous(cuda, loc, scale, A, t, A, None, None, None, None, 1, N, A, ctr)
  assert torch.equal(ds, ds2) and ctr.cpu().tolist() == [2, 0]    # advance=0 leaves the counter


# ---- 3. the reference golden through the agent --------------------------------------------------
def _traj(cuda, obs, act, outer):
  one = torch.ones(outer, dtype=torch.int32, device=cuda)
  zero = torch.zeros(outer, dtype=torch.float32, device=cuda)
  return trajectory.Trajectory(one, _d(cuda, obs), _d(cuda, act), (), one, zero, zero + 1)


def test_reference_golden_through_agent(cuda):
  obs_spec = tensor_spec.TensorSpec((2,), torch.float32)
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 1)
  net = sequential.Sequential([L.Dense(2)], input_spec=obs_spec, device=cuda)
  agent = bca.BehavioralCloningAgent(ts.time_step_spec(obs_spec), act_spec, cloning_network=net,
                                     optimizer=optimizers.AdamOptimizer(1e-3))
  net.layers[0].kernel.copy_(torch.tensor([[2., 1.], [1., 1.]]))
  net.layers[0].bias.copy_(torch.tensor([1., 1.]))
  exp = _traj(cuda, np.array([[1, 2], [3, 4]], f32), np.array([0, 1], np.int32), (2,))
  before = agent.loss(exp)
  np.testing.assert_allclose(before.loss.item(), 1.6809245, rtol=1e-6)
  got = agent.train(exp)
  np.testing.assert_allclose(got.loss.item(), 1.6809245, rtol=1e-6)
  assert tuple(got.extra.loss.shape) == (2,)
  after = agent.loss(exp).loss.item()
  assert after < 1.6809245 and agent.loss(exp).loss.item() == after
  agent.check_numerics()


# ---- 4. train against the oracle -----------------------------------------------------------------
def _mirror(net):
  """(oracle Sequential of the layer stack, std bias or None, indices of kernels with L2)."""
  layers, l2, k = [], [], 0
  std = None
  for l in net.layers:
    if isinstance(l, L.Dense):
      layers.append(dict(kind='dense', w=l.kernel.cpu().numpy().copy(),
                         b=l.bias.cpu().numpy().copy(), act=l.activation))
      if l.l2:
        l2.append((l.l2, k))
      k += 2
    elif isinstance(l, L.Flatten):
      layers.append(dict(kind='flatten'))
    elif isinstance(l, adn.StdBias):
      std = l.bias.cpu().numpy().copy()
  return onn.Sequential(layers), std, l2


def _net(cuda, kind, D, A, l2):
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32)
  if kind == 'q':
    act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 1, A)
    net = q_network.QNetwork(obs_spec, act_spec, fc_layer_params=(32, 16), device=cuda)
  elif kind == 'seq':
    act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 1, A)
    net = sequential.Sequential([L.Dense(32, activation='relu', kernel_regularizer_l2=l2),
                                 L.Dense(A, kernel_regularizer_l2=l2)], input_spec=obs_spec,
                                device=cuda)
  elif kind == 'cat':
    act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, A - 1)
    net = adn.ActorDistributionNetwork(obs_spec, act_spec, fc_layer_params=(32,), device=cuda)
  elif kind == 'actor':
    act_spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, -2.0, 1.0)
    net = actor_network.ActorNetwork(obs_spec, act_spec, fc_layer_params=(32, 16), device=cuda)
  else:
    act_spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, -2.0, 1.0)
    net = adn.ActorDistributionNetwork(obs_spec, act_spec, fc_layer_params=(32,), device=cuda)
  return obs_spec, act_spec, net.set_seed(3)


_KIND = {'q': obc.LOGITS, 'seq': obc.LOGITS, 'cat': obc.LOGITS, 'actor': obc.DETERMINISTIC,
         'normal': obc.NORMAL}


def _make(cuda, kind, D=7, A=4, l2=0.0, clip=None, outer_dims=1, lr=1e-3, seed=0):
  obs_spec, act_spec, net = _net(cuda, kind, D, A, l2)
  agent = bca.BehavioralCloningAgent(ts.time_step_spec(obs_spec), act_spec, cloning_network=net,
                                     optimizer=optimizers.Adam(lr), num_outer_dims=outer_dims,
                                     gradient_clipping=clip, seed=seed)
  return agent, act_spec


def _data(rng, kind, outer, D, A, act_spec):
  obs = rng.randn(*outer, D).astype(f32)
  if _KIND[kind] == obc.LOGITS:
    act = rng.randint(int(act_spec.minimum), int(act_spec.maximum) + 1, outer).astype(np.int32)
  else:
    act = rng.uniform(-2, 1, (*outer, A)).astype(f32)
  return obs, act


_TRAIN = [('q', 1, 'rows', 0.0, None), ('q', 2, 'batch', 0.0, 0.05), ('seq', 2, 'rows', 0.01, None),
          ('cat', 1, None, 0.0, 0.05), ('cat', 2, 'scalar', 0.0, None),
          ('actor', 1, 'rows', 0.0, 0.01), ('actor', 2, 'batch', 0.0, None),
          ('normal', 1, None, 0.0, None), ('normal', 2, 'rows', 0.0, 0.05)]


@pytest.mark.parametrize('cfg', _TRAIN, ids=lambda c: '-'.join(str(x) for x in c))
def test_agent_train_matches_oracle(cuda, cfg):
  kind, outer_dims, wkind, l2, clip = cfg
  D, A, B, T = 7, 4, 64, 3
  agent, act_spec = _make(cuda, kind, D, A, l2=l2, clip=clip, outer_dims=outer_dims)
  net = agent.cloning_network
  seq, std, l2s = _mirror(net)
  orc = obc.BcOracle(seq, _KIND[kind], amin=np.full(A, -2, f32), amax=np.full(A, 1, f32),
                     std_bias=std, minimum=int(getattr(act_spec, 'minimum', 0)),
                     optimizer=ooptim.AdamTF(1e-3, eps=1e-7), gradient_clipping=clip, l2=l2s)
  rng = np.random.RandomState(17)
  outer = (B,) if outer_dims == 1 else (B, T)
  n = int(np.prod(outer))
  name = 'bc_train_' + '_'.join(str(c) for c in cfg)
  for step in range(6):
    obs, act = _data(rng, kind, outer, D, A, act_spec)
    w = {None: None, 'rows': rng.rand(*outer).astype(f32), 'batch': rng.rand(B).astype(f32),
         'scalar': np.array(0.6, f32)}[wkind]
    z = rng.randn(n, A).astype(f32) if kind == 'normal' else None
    wl, wpe = orc.train(obs.reshape(n, D), act.reshape(n, -1) if act.ndim > len(outer) else
                        act.reshape(n), w, z, outer)
    got = agent.train(_traj(cuda, obs, act, outer), weights=None if w is None else _d(cuda, w),
                      **({} if z is None else {'noise': _d(cuda, z)}))
    assert tuple(got.extra.loss.shape) == outer
    rel = abs(got.loss.item() - wl) / abs(wl)
    record_parity(name, loss_rel=rel)
    np.testing.assert_allclose(got.loss.item(), wl, rtol=2e-5, err_msg=f'step {step}')
    np.testing.assert_allclose(got.extra.loss.cpu().numpy().reshape(n), wpe, rtol=5e-5, atol=1e-6)
  assert int(agent.train_step_counter.item()) == 6
  got = np.concatenate([v.cpu().numpy().ravel() for v in net.variables])
  want = np.concatenate([p.ravel() for p in orc.params()])
  diff = np.abs(got - want)
  out = diff > 1e-5 + 1e-3 * np.abs(want)
  record_parity(name, outlier_frac=out.mean(), max_abs=diff.max())
  assert out.mean() <= 1e-3 and diff.max() <= 6 * 1e-3, (out.mean(), diff.max())
  assert agent._sample_rng.cpu().tolist() == [0, 0]               # supplied draws
  agent.check_numerics()


# ---- 5. gradients before the optimiser ----------------------------------------------------------
@pytest.mark.parametrize('kind', ['seq', 'cat', 'actor', 'normal'])
def test_gradients_before_the_optimizer_match_float64(cuda, kind):
  D, A, B, T = 7, 4, 128, 2
  agent, act_spec = _make(cuda, kind, D, A, l2=0.01 if kind == 'seq' else 0.0, outer_dims=2,
                          lr=0.0)
  net = agent.cloning_network
  rng = np.random.RandomState(23)
  obs, act = _data(rng, kind, (B, T), D, A, act_spec)
  w = rng.rand(B).astype(f32)
  z = rng.randn(B * T, A).astype(f32)
  dense = [l for l in net.layers if isinstance(l, L.Dense)]
  P = [(R.t64(l.kernel).requires_grad_(), R.t64(l.bias).requires_grad_(), l.activation)
       for l in dense]
  params = [t for p in P for t in p[:2]]
  std = None
  if kind == 'normal':
    std = R.t64(net.layers[-1].bias).requires_grad_()
    params.append(std)
  agent.train(_traj(cuda, obs, act, (B, T)), weights=_d(cuda, w),
              **({'noise': _d(cuda, z)} if kind == 'normal' else {}))
  out = R.mlp(P, R.t64(obs.reshape(B * T, D)))
  W = R.t64(np.repeat(w, T))
  if _KIND[kind] == obc.LOGITS:
    lab = torch.as_tensor(act.reshape(-1).astype(np.int64) - int(act_spec.minimum))
    pe = torch.nn.functional.cross_entropy(out, lab, reduction='none')
  else:
    lo, hi = -2.0, 1.0
    if kind == 'actor':
      a = (hi + lo) / 2 + (hi - lo) / 2 * out
    else:
      a = (hi + lo) / 2 + (hi - lo) / 2 * torch.tanh(out) + R.softplus(std) * R.t64(z)
    pe = ((a - R.t64(act.reshape(B * T, A))) ** 2).mean(1)
  loss = (pe * W).sum() / (B * T)
  for l, p in zip(dense, P):
    if l.l2:
      loss = loss + l.l2 * (p[0] ** 2).sum()
  ref = torch.autograd.grad(loss, params)
  for i, (g, rf) in enumerate(zip(net._grad_views, ref)):
    e = R.grad_errors(g, rf)
    record_parity(f'bc_grads_{kind}', **{f'{i}_rel_l2': e[0], f'{i}_max': e[1]})
    R.assert_grad_close(f'bc {kind}/{i}', g, rf, 1e-4, 1e-4)


# ---- 6. graph replay -------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', ['q', 'normal'])
def test_graph_replay_matches_eager_bit_for_bit(cuda, kind):
  (eager, spec), (graphed, _) = _make(cuda, kind, clip=0.05), _make(cuda, kind, clip=0.05)
  train_fn = common.function(graphed.train)
  rng = np.random.RandomState(11)
  for step in range(6):
    obs, act = _data(rng, kind, (8,), 7, 4, spec)
    traj = _traj(cuda, obs, act, (8,))
    w = _d(cuda, rng.rand(8).astype(f32))
    l1, l2 = eager.train(traj, weights=w), train_fn(traj, weights=w)
    assert l1.loss.item() == l2.loss.item(), step
    assert torch.equal(l1.extra.loss, l2.extra.loss), step
  assert int(graphed.train_step_counter.item()) == 6 and graphed._train_step_host == 6
  assert torch.equal(eager.cloning_network.flat_params, graphed.cloning_network.flat_params)
  if kind == 'normal':                                            # train advances the draw counter
    assert graphed._sample_rng.cpu().tolist() == [6, 0] == eager._sample_rng.cpu().tolist()


def test_captured_collect_step_matches_eager_calls(cuda):
  (eager, _), (graphed, _) = _make(cuda, 'q', seed=4), _make(cuda, 'q', seed=4)
  step = ts.restart(torch.randn(64, 7, device=cuda), batch_size=64)
  act_fn = common.function(lambda t: graphed.collect_policy.action(t).action)
  for call in range(6):
    a1 = eager.collect_policy.action(step).action
    a2 = act_fn(step)
    assert torch.equal(a1, a2), call


# ---- 7. Learner checkpoints -----------------------------------------------------------------------
def test_learner_checkpoint_restore_reproduces_losses_and_draws(cuda):
  rng = np.random.RandomState(12)
  spec = tensor_spec.BoundedTensorSpec((4,), torch.float32, -2.0, 1.0)
  batches = [_data(rng, 'normal', (8,), 7, 4, spec) for _ in range(7)]
  root = tempfile.mkdtemp()

  def make(perturb):
    from agents_b200.train.utils import train_utils
    step = train_utils.create_train_step(cuda)
    obs_spec, act_spec, net = _net(cuda, 'normal', 7, 4, 0.0)
    agent = bca.BehavioralCloningAgent(ts.time_step_spec(obs_spec), act_spec, net,
                                       optimizers.Adam(1e-3), train_step_counter=step)
    if perturb:
      net.flat_params.mul_(0.5)
      agent._sample_rng.fill_(9)
    it = iter([_traj(cuda, o, a, (8,)) for o, a in batches])
    return agent, step, learner_lib.Learner(root, step, agent, experience_dataset_fn=lambda: it,
                                            checkpoint_interval=4)

  agent, _, lrn = make(False)
  lrn.run(iterations=4)
  want = [agent.train(_traj(cuda, o, a, (8,))).loss.item() for o, a in batches[4:]]
  agent2, step2, _ = make(True)
  assert int(step2.item()) == 4 and agent2._sample_rng.cpu().tolist() == [4, 0]
  got = [agent2.train(_traj(cuda, o, a, (8,))).loss.item() for o, a in batches[4:]]
  assert got == want


# ---- 8. policies -----------------------------------------------------------------------------------
def test_policies_respect_the_action_minimum(cuda):
  agent, _ = _make(cuda, 'q', A=5)
  N = 20000
  step = ts.restart(torch.randn(N, 7, device=cuda), batch_size=N)
  q = agent.cloning_network(step.observation)[0]
  greedy = agent.policy.action(step).action
  assert torch.equal(greedy.long(), q.argmax(1) + 1)
  col = agent.collect_policy.action(step).action.long()
  assert int(col.min()) >= 1 and int(col.max()) <= 5
  # epsilon 0.1: a random action differs from the greedy one with probability 0.1 * 4/5
  frac = float((col != greedy.long()).double().mean())
  sd = (0.08 * 0.92 / N) ** .5
  record_parity('bc_epsilon_greedy', sigmas=abs(frac - 0.08) / sd)
  assert abs(frac - 0.08) < 5 * sd, frac
  cont, _ = _make(cuda, 'normal')
  a = cont.collect_policy.action(step).action
  assert float(a.min()) >= -2.0 and float(a.max()) <= 1.0
  loc = cont.cloning_network(step.observation)[0][0]
  assert torch.equal(cont.policy.action(step).action, loc)


# ---- 9. unsupported options -------------------------------------------------------------------------
def test_unsupported_options_raise(cuda):
  obs_spec = tensor_spec.TensorSpec((3,), torch.float32)
  cont = tensor_spec.BoundedTensorSpec((2,), torch.float32, -1.0, 1.0)
  disc = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 2)
  tss = ts.time_step_spec(obs_spec)
  with pytest.raises(NotImplementedError, match='loss_fn'):
    bca.BehavioralCloningAgent(tss, disc, sequential.Sequential([L.Dense(3)], device=cuda), None,
                               loss_fn=lambda e, training=False: None)
  with pytest.raises(NotImplementedError, match='TanhNormalActorNetwork'):
    bca.BehavioralCloningAgent(tss, cont, tnpn.TanhNormalActorNetwork(obs_spec, cont, device=cuda),
                               None)
  rnn = sequential.Sequential([L.Dense(3)], device=cuda)
  rnn._state_spec = (tensor_spec.TensorSpec((4,), torch.float32),)
  with pytest.raises(NotImplementedError, match='non-RNN'):
    bca.BehavioralCloningAgent(tss, disc, rnn, None)
  with pytest.raises(NotImplementedError, match='continuous action'):
    bca.BehavioralCloningAgent(tss, cont, sequential.Sequential([L.Dense(2)], device=cuda), None)
  with pytest.raises(NotImplementedError, match='logits'):
    bca.BehavioralCloningAgent(tss, disc, sequential.Sequential([L.Dense(4)], device=cuda), None)
  agent, spec = _make(cuda, 'q')
  obs, act = _data(np.random.RandomState(0), 'q', (4,), 7, 4, spec)
  agent.replicas = 2
  with pytest.raises(NotImplementedError, match='data-parallel'):
    agent.train(_traj(cuda, obs, act, (4,)))
  agent.replicas = 1
  agent._optimizer = None
  with pytest.raises(ValueError, match='Optimizer is undefined'):
    agent.train(_traj(cuda, obs, act, (4,)))


# ---- 10. offline learning ----------------------------------------------------------------------------
def test_offline_learning_clones_a_linear_teacher(cuda):
  D, A, n_train, B = 8, 4, 8192, 256
  rng = np.random.RandomState(5)
  teacher = rng.randn(D, A).astype(f32)
  obs = rng.randn(n_train + 2048, D).astype(f32)
  labels = (obs @ teacher).argmax(1).astype(np.int32) + 1
  agent, _ = _make(cuda, 'q', D=D, A=A, lr=3e-3)
  held = torch.as_tensor(obs[n_train:], device=cuda)

  def agreement():
    step = ts.restart(held, batch_size=held.shape[0])
    return float((agent.policy.action(step).action.cpu().numpy() == labels[n_train:]).mean())

  a0 = agreement()
  train_fn = common.function(agent.train)
  for i in range(400):
    idx = rng.randint(0, n_train, B)
    train_fn(_traj(cuda, obs[idx], labels[idx], (B,)))
  a1 = agreement()
  record_parity('bc_offline_learning', initial=a0, final=a1)
  assert a1 > 0.9, (a0, a1)
