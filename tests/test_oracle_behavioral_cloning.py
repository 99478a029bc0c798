"""Host checks of the behavioral-cloning oracle (oracle/behavioral_cloning.py) and of the agent's
action-spec checks: the reference golden of testLoss, the losses and a train step's gradients
against float64 torch autograd (both continuous modes, with and without weights, a zero weight on
a row whose loss is inf or NaN), and the reference's spec-check parametrisation."""
import numpy as np
import pytest
import torch

from agents_b200 import optimizers
from agents_b200.agents.behavioral_cloning import behavioral_cloning_agent as bca
from agents_b200.networks import layers as L
from agents_b200.networks import sequential
from agents_b200.specs import tensor_spec
from agents_b200.trajectories import time_step as ts
from oracle import behavioral_cloning as obc
from oracle import nn as onn

f32 = np.float32
F64 = torch.float64


def test_reference_golden_testLoss():
  # agents/behavioral_cloning/behavioral_cloning_agent_test.py testLoss: Dense kernel
  # [[2, 1], [1, 1]], bias [1, 1]; the mean cross-entropy of the first train step's loss
  net = onn.Sequential([dict(kind='dense', w=np.array([[2, 1], [1, 1]], f32),
                             b=np.array([1, 1], f32), act=None)])
  o = obc.BcOracle(net, obc.LOGITS)
  loss, pe = o.train(np.array([[1, 2], [3, 4]], f32), np.array([0, 1], np.int32))
  np.testing.assert_allclose(loss, 1.6809245, rtol=1e-6)
  np.testing.assert_allclose(pe, [np.log1p(np.exp(-1.0)), 3 + np.log1p(np.exp(-3.0))], rtol=1e-6)


def _weights(rng, n, kind):
  if kind is None:
    return None
  w = rng.rand(n)
  w[1] = 0.0
  return w


@pytest.mark.parametrize('weighted', [None, 'rows'])
@pytest.mark.parametrize('A', [1, 5, 70])
def test_discrete_loss_matches_autograd(weighted, A):
  rng = np.random.RandomState(A)
  n = 9
  z = (rng.randn(n, A) * 3).astype(f32)
  lab = rng.randint(0, A, n)
  w = _weights(rng, n, weighted)
  if w is not None:
    z[1, 0] = np.nan                                  # zero weight on a NaN row
    z[1, -1] = np.inf
  loss, pe, g = obc.discrete_loss(z, lab, w)
  Z = torch.tensor(z, dtype=F64, requires_grad=True)
  W = torch.ones(n, dtype=F64) if w is None else torch.tensor(w, dtype=F64)
  ce = torch.nn.functional.cross_entropy(Z, torch.tensor(lab), reduction='none')
  keep = W != 0
  ref = (ce[keep] * W[keep]).sum() / n
  np.testing.assert_allclose(loss, ref.item(), rtol=1e-6)
  np.testing.assert_allclose(pe[keep.numpy()], ce[keep].detach().numpy(), rtol=1e-6)
  want = torch.autograd.grad(ref, Z)[0].numpy()     # NaN * 0 on the dropped rows
  k = keep.numpy()
  np.testing.assert_allclose(g[k], want[k], rtol=1e-5, atol=1e-9)
  if w is not None:
    assert not g[1].any() and np.isnan(pe[1])


def test_discrete_out_of_range_label_is_nan():
  loss, pe, _ = obc.discrete_loss(np.zeros((3, 4), f32), np.array([0, 4, -1]))
  assert np.isnan(loss) and np.isnan(pe[1]) and np.isnan(pe[2]) and pe[0] == np.float32(np.log(4))


@pytest.mark.parametrize('weighted', [None, 'rows'])
@pytest.mark.parametrize('mode', ['deterministic', 'normal'])
def test_continuous_loss_matches_autograd(weighted, mode):
  rng = np.random.RandomState(7)
  n, A = 11, 6
  y = rng.uniform(-1, 1, (n, A)).astype(f32)
  t = rng.uniform(-2, 2, (n, A)).astype(f32)
  lo, hi = rng.uniform(-3, -0.5, A).astype(f32), rng.uniform(0.5, 2, A).astype(f32)
  s = rng.uniform(0.1, 1, (n, A)).astype(f32)
  z = rng.randn(n, A).astype(f32)
  w = _weights(rng, n, weighted)
  if w is not None:
    y[1, 2] = np.inf if mode == 'normal' else np.nan
  Y = torch.tensor(y, dtype=F64, requires_grad=True)
  S = torch.tensor(s, dtype=F64, requires_grad=True)
  if mode == 'deterministic':
    loss, pe, dy, ds = obc.continuous_loss(y, t, w, lo, hi)
    LO, HI = torch.tensor(lo, dtype=F64), torch.tensor(hi, dtype=F64)
    act = (HI + LO) / 2 + (HI - LO) / 2 * Y
  else:
    loss, pe, dy, ds = obc.continuous_loss(y, t, w, scale=s, z=z)
    act = Y + S * torch.tensor(z, dtype=F64)
  W = torch.ones(n, dtype=F64) if w is None else torch.tensor(w, dtype=F64)
  mse = ((act - torch.tensor(t, dtype=F64)) ** 2).mean(1)
  keep = W != 0
  ref = (mse[keep] * W[keep]).sum() / n
  np.testing.assert_allclose(loss, ref.item(), rtol=1e-6)
  np.testing.assert_allclose(pe[keep.numpy()], mse[keep].detach().numpy(), rtol=1e-6)
  gy, gs = torch.autograd.grad(ref, (Y, S), allow_unused=True)
  k = keep.numpy()
  np.testing.assert_allclose(dy[k], gy.numpy()[k], rtol=1e-5, atol=1e-9)
  if mode == 'normal':
    np.testing.assert_allclose(ds[k], gs.numpy()[k], rtol=1e-5, atol=1e-9)
  if w is not None:
    assert not dy[1].any()


def _torch_dense(x, layers):
  for l in layers:
    x = x @ l['W'] + l['B']
    if l['act'] == 'relu':
      x = torch.relu(x)
    elif l['act'] == 'tanh':
      x = torch.tanh(x)
  return x


@pytest.mark.parametrize('kind', [obc.LOGITS, obc.DETERMINISTIC, obc.NORMAL])
def test_train_gradients_match_autograd(kind):
  """Gradients of the total loss (with an L2 term, [B, T] weights) through a two-layer stack."""
  rng = np.random.RandomState(3)
  B, T, D, H, A = 4, 3, 5, 8, 3
  n = B * T
  last = 'tanh' if kind == obc.DETERMINISTIC else None
  layers = [dict(kind='dense', w=(rng.randn(D, H) * .5).astype(f32), b=(rng.randn(H) * .1).astype(f32),
                 act='relu'),
            dict(kind='dense', w=(rng.randn(H, A) * .5).astype(f32), b=(rng.randn(A) * .1).astype(f32),
                 act=last)]
  lo, hi = np.array([-1, -2, 0], f32), np.array([1, 1, 3], f32)
  std = rng.randn(A).astype(f32) * .3
  o = obc.BcOracle(onn.Sequential(layers), kind, amin=lo, amax=hi, std_bias=std, minimum=2,
                   l2=[(0.01, 0)])
  obs = rng.randn(n, D).astype(f32)
  act = rng.randint(2, 2 + A, n) if kind == obc.LOGITS else rng.uniform(-1, 1, (n, A)).astype(f32)
  w = rng.rand(B).astype(f32)
  z = rng.randn(n, A).astype(f32)
  loss, _, grads = o.loss_and_grads(obs, act, w, z, outer=(B, T))
  P = [torch.tensor(p, dtype=F64, requires_grad=True) for p in o.params()]
  tl = [dict(W=P[0], B=P[1], act='relu'), dict(W=P[2], B=P[3], act=last)]
  out = _torch_dense(torch.tensor(obs, dtype=F64), tl)
  W = torch.tensor(np.repeat(w, T), dtype=F64)
  if kind == obc.LOGITS:
    pe = torch.nn.functional.cross_entropy(out, torch.tensor(act - 2), reduction='none')
  else:
    LO, HI = torch.tensor(lo, dtype=F64), torch.tensor(hi, dtype=F64)
    if kind == obc.DETERMINISTIC:
      a = (HI + LO) / 2 + (HI - LO) / 2 * out
    else:
      loc = (HI + LO) / 2 + (HI - LO) / 2 * torch.tanh(out)
      a = loc + torch.nn.functional.softplus(P[4]) * torch.tensor(z, dtype=F64)
    pe = ((a - torch.tensor(act, dtype=F64)) ** 2).mean(1)
  ref = (pe * W).sum() / n + 0.01 * (P[0] ** 2).sum()
  np.testing.assert_allclose(loss, ref.item(), rtol=2e-5)
  for g, want in zip(grads, torch.autograd.grad(ref, P)):
    np.testing.assert_allclose(g, want.numpy(), rtol=2e-4, atol=2e-6)


# ---- the reference's testCreateAgentNestSizeChecks --------------------------------------------
_MSG = '.* single, scalar discrete.*'


@pytest.mark.parametrize('action_spec,expected_error', [
    ([tensor_spec.BoundedTensorSpec((), torch.int32, 0, 1),
      tensor_spec.BoundedTensorSpec((), torch.int32, 0, 1)], _MSG),            # MultipleActions
    ([tensor_spec.BoundedTensorSpec((1,), torch.int32, 0, 1)], _MSG),          # NonScalarAction
    ([tensor_spec.BoundedTensorSpec((), torch.int32, 0, 1)], None),            # ScalarDiscreteAction
    (tensor_spec.BoundedTensorSpec((3, 2), torch.float32, 0, 1), 'rank'),      # SingleNonScalarFloat
    ([tensor_spec.BoundedTensorSpec((), torch.float32, 0, 1),
      tensor_spec.BoundedTensorSpec((), torch.float32, 0, 1)], _MSG),          # MultipleContinuous
    ([tensor_spec.BoundedTensorSpec((), torch.int32, 0, 1),
      tensor_spec.BoundedTensorSpec((), torch.float32, 0, 1)], _MSG),          # MixedDiscreteAndCont.
], ids=['MultipleActions', 'NonScalarAction', 'ScalarDiscreteAction', 'SingleNonScalarFloatAction',
        'MultipleContinuous', 'MixedDiscreteAndContinuous'])
def test_create_agent_nest_size_checks(action_spec, expected_error):
  obs_spec = tensor_spec.TensorSpec((2,), torch.float32)
  net = sequential.Sequential([L.Dense(2)], input_spec=obs_spec, device='cpu')
  make = lambda: bca.BehavioralCloningAgent(ts.time_step_spec(obs_spec), action_spec,
                                            cloning_network=net, optimizer=None)
  if expected_error == 'rank':
    # departure: the reference accepts a continuous action of rank > 1
    with pytest.raises(NotImplementedError, match='rank 0 or 1'):
      make()
  elif expected_error is not None:
    with pytest.raises(ValueError, match=expected_error):
      make()
  else:
    assert make().policy is not None


def test_custom_loss_fn_is_rejected():
  obs_spec = tensor_spec.TensorSpec((2,), torch.float32)
  net = sequential.Sequential([L.Dense(2)], input_spec=obs_spec, device='cpu')
  with pytest.raises(NotImplementedError, match='loss_fn'):
    bca.BehavioralCloningAgent(ts.time_step_spec(obs_spec),
                               tensor_spec.BoundedTensorSpec((), torch.int32, 0, 1), net,
                               optimizers.Adam(1e-3), loss_fn=lambda e, training=False: None)
