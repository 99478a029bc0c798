"""The C51 oracle against the reference's own numbers (agents/categorical_dqn/
categorical_dqn_agent.py docstring, categorical_dqn_agent_test.py) and float64 autograd (no GPU)."""
import numpy as np
import pytest
import torch

from oracle import categorical_dqn as oc51
from oracle import nn as onn

f32 = np.float32
N_ATOMS = 51


def _dummy_net():
  # categorical_dqn_agent_test.py:36-82 DummyCategoricalNet: Dense(2 -> 2*51), the stated constant
  # kernel, ones bias
  w = np.array([np.concatenate((np.arange(N_ATOMS), np.ones(N_ATOMS))),
                np.concatenate((np.ones(N_ATOMS), np.ones(N_ATOMS)))], dtype=f32)
  return onn.Sequential([dict(kind='dense', w=w, b=np.ones(2 * N_ATOMS, f32), act=None)])


def _exp(obs_seq, masks=None, T=2):
  B = 2
  e = dict(observation=np.stack([np.asarray(o, f32) for o in obs_seq], axis=1),
           action=np.tile(np.array([[0], [1]], np.int32), (1, T)),
           reward=np.tile(np.array([[10], [20]], f32), (1, T)),
           discount=np.full((B, T), 0.9, f32))
  if masks is not None:
    e['mask'] = np.stack([np.asarray(m, np.int32) for m in masks], axis=1)
  return e


def test_project_distribution_docstring_example():
  # categorical_dqn_agent.py:577-581, :727-728
  got = oc51.project_distribution([[0, 2, 4, 6, 8], [1, 3, 4, 5, 6]],
                                  [[0.1, 0.6, 0.1, 0.1, 0.1], [0.1, 0.2, 0.5, 0.1, 0.1]],
                                  [4, 5, 6, 7, 8])
  np.testing.assert_allclose(got, [[0.8, 0, 0.1, 0, 0.1], [0.8, 0.1, 0.1, 0, 0]], atol=1e-7)


def test_supports():
  z = oc51.tf_linspace(-10.0, 10.0, 51)
  assert z.dtype == f32 and z[0] == -10 and z[-1] == 10
  np.testing.assert_allclose(z, np.linspace(-10, 10, 51), atol=2e-6)
  np.testing.assert_allclose(oc51.policy_support(-10.0, 10.0, 51), z, atol=2e-6)


@pytest.mark.parametrize('masked', [False, True])
def test_critic_loss_goldens(masked):
  """testCriticLoss :255-285 -> 2.19525; testCriticLossWithMaskedActions :287-337 -> 5.062895;
  testTrain :476-506 -> 2.19525 (the loss of the first step)."""
  orc = oc51.CategoricalDqnOracle(_dummy_net(), None, N_ATOMS)
  masks = [[[1, 0], [0, 1]], [[0, 1], [1, 0]]] if masked else None
  out = orc.loss(_exp([[[1, 2], [3, 4]], [[5, 6], [7, 8]]], masks))
  np.testing.assert_allclose(out['loss'], 5.062895 if masked else 2.19525, atol=1e-4)


def test_train_golden():
  class Sgd(object):
    def apply(self, params, grads):
      for p, g in zip(params, grads):
        p -= f32(0.01) * g
  orc = oc51.CategoricalDqnOracle(_dummy_net(), Sgd(), N_ATOMS)
  out = orc.train(_exp([[[1, 2], [3, 4]], [[5, 6], [7, 8]]]))
  np.testing.assert_allclose(out['loss'], 2.19525, atol=1e-4)
  assert orc.train_step_counter == 1


def test_critic_loss_n_step_golden():
  """testCriticLossNStep :339-397: returns [[19], [38]], final discount [[0.81], [0.81]], 2.19525."""
  orc = oc51.CategoricalDqnOracle(_dummy_net(), None, N_ATOMS)
  out = orc.loss(_exp([[[1, 2], [3, 4]], [[5, 6], [7, 8]], [[9, 10], [11, 12]]], T=3))
  np.testing.assert_allclose(out['returns'], [19, 38], atol=1e-4)
  np.testing.assert_allclose(out['final_discount'], [0.81, 0.81], atol=1e-4)
  np.testing.assert_allclose(out['loss'], 2.19525, atol=1e-4)


def _torch_loss(q, nxt, actions, reward, discount, z, gamma, scale, mask):
  """float64 restatement for autograd: the target distribution is a constant (stop_gradient)."""
  q = torch.as_tensor(q, dtype=torch.float64).requires_grad_(True)
  nxt = torch.as_tensor(nxt, dtype=torch.float64)
  z64 = torch.as_tensor(z, dtype=torch.float64)
  B = q.shape[0]
  p = torch.softmax(nxt, -1)
  qv = (p * z64).sum(-1)
  if mask is not None:
    qv = torch.where(torch.as_tensor(mask, dtype=torch.bool), qv, torch.tensor(-np.inf, dtype=torch.float64))
  best = qv.argmax(-1)
  pb = p[torch.arange(B), best]
  r = torch.as_tensor(reward, dtype=torch.float64)[:, :-1] * scale
  d = torch.as_tensor(discount, dtype=torch.float64)[:, :-1] * gamma
  R = torch.zeros(B, dtype=torch.float64)
  for t in range(r.shape[1] - 1, -1, -1):
    R = r[:, t] + d[:, t] * R
  tz = (R[:, None] + d.prod(1)[:, None] * z64).clamp(z64[0], z64[-1])
  quot = (1 - (tz[:, None, :] - z64[None, :, None]).abs() / (z64[1] - z64[0])).clamp(0, 1)
  m = (quot * pb[:, None, :]).sum(-1)
  l = q[torch.arange(B), torch.as_tensor(actions, dtype=torch.int64)]
  loss = (m * (torch.logsumexp(l, -1, keepdim=True) - l)).sum(-1).mean()
  loss.backward()
  return loss.item(), q.grad.numpy(), m.detach().numpy()


@pytest.mark.parametrize('A,N,T,masked', [(1, 2, 2, False), (2, 5, 3, True), (6, 51, 2, True),
                                          (18, 51, 4, False), (3, 201, 3, True)])
def test_loss_and_dlogits_against_float64_autograd(A, N, T, masked):
  rng = np.random.RandomState(A * 100 + N + T)
  B = 16
  q = (rng.randn(B, A, N) * 2).astype(f32)
  nxt = (rng.randn(B, A, N) * 2).astype(f32)
  actions = rng.randint(0, A, size=B)
  reward = (rng.randn(B, T) * 4).astype(f32)
  reward[0] = 50.0                                  # beyond v_max
  reward[1] = -50.0                                 # below v_min
  discount = (rng.rand(B, T) > 0.2).astype(f32)
  mask = (rng.rand(B, A) > 0.4).astype(np.int32) if masked else None
  if masked:
    mask[:, -1] = 1
  z = oc51.tf_linspace(-10.0, 10.0, N)
  out = oc51.c51_loss(q, nxt, actions, reward, discount, z, gamma=0.97, reward_scale=0.5,
                      next_mask=mask)
  want, dq, m = _torch_loss(q, nxt, actions, reward, discount, z, 0.97, 0.5, mask)
  np.testing.assert_allclose(out['loss'], want, rtol=1e-5)
  np.testing.assert_allclose(out['target'], m, atol=2e-6)
  np.testing.assert_allclose(out['dlogits'], dq, atol=1e-6, rtol=1e-4)


def test_projection_conserves_mass():
  """Tz on atoms (l == u: the floor/ceil form drops that mass), between atoms and beyond both
  ends of the support: every row's projected mass equals its input mass."""
  N = 11
  z = oc51.tf_linspace(-5.0, 5.0, N)
  rng = np.random.RandomState(0)
  p = rng.rand(6, N).astype(f32)
  p /= p.sum(1, keepdims=True)
  rows = [z.copy(), z + f32(0.37), z * f32(3), z - f32(20), z + f32(20),
          np.round(rng.randn(N) * 3).astype(f32)]
  m = oc51.project_distribution(np.stack(rows), p, z)
  np.testing.assert_allclose(m.sum(1), p.sum(1), atol=1e-6)
  np.testing.assert_allclose(m[0], p[0], atol=1e-7)          # exactly on atoms: identity
  np.testing.assert_allclose(m[3], np.eye(N)[0] * p[3].sum(), atol=1e-6)
  np.testing.assert_allclose(m[4], np.eye(N)[-1] * p[4].sum(), atol=1e-6)
  assert (m >= 0).all()
