"""Optimiser / target-update / clip kernels, epsilon-greedy and environment kernels vs oracle."""
import numpy as np
import pytest
import torch

from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.utils import common
from agents_b200.utils import workspace
from oracle import env as oenv
from oracle import optim as ooptim

pytestmark = pytest.mark.gpu
f32 = np.float32


@pytest.mark.parametrize('n', [1, 1000, 70001])
def test_adam_parity(cuda, n):
  rng = np.random.RandomState(n)
  p = rng.randn(n).astype(f32)
  opt, oopt = optimizers.AdamOptimizer(1e-3), ooptim.AdamTF(1e-3, eps=1e-8)
  tp = torch.as_tensor(p.copy(), device=cuda)
  wp = [p.copy()]
  for _ in range(4):
    g = rng.randn(n).astype(f32)
    opt.apply_flat(tp, torch.as_tensor(g, device=cuda))
    oopt.apply(wp, [g])
  np.testing.assert_allclose(tp.cpu().numpy(), wp[0], rtol=1e-5, atol=1e-7)
  assert int(opt.iterations(tp).item()) == 4


@pytest.mark.parametrize('centered', [False, True])
def test_rmsprop_parity(cuda, centered):
  rng = np.random.RandomState(1)
  n = 5000
  p = rng.randn(n).astype(f32)
  opt = optimizers.RMSPropOptimizer(2.5e-4, decay=0.95, momentum=0.9, epsilon=1e-5, centered=centered)
  oopt = ooptim.RMSPropTF(2.5e-4, decay=0.95, momentum=0.9, eps=1e-5, centered=centered)
  tp, wp = torch.as_tensor(p.copy(), device=cuda), [p.copy()]
  for _ in range(4):
    g = rng.randn(n).astype(f32)
    opt.apply_flat(tp, torch.as_tensor(g, device=cuda))
    oopt.apply(wp, [g])
  np.testing.assert_allclose(tp.cpu().numpy(), wp[0], rtol=1e-5, atol=1e-7)


def test_soft_update_and_periodically(cuda):  # utils/common_test.py:83-143, :230-331
  s = torch.tensor([1., 2., 3.], device=cuda)
  t = torch.tensor([3., 5., 7.], device=cuda)
  common.soft_variables_update(s, t, tau=0.1)
  np.testing.assert_allclose(t.cpu().numpy(), [2.8, 4.7, 6.6], rtol=1e-6)
  common.soft_variables_update(s, t, tau=1.0)
  assert t.cpu().tolist() == [1., 2., 3.]
  with pytest.raises(ValueError, match=r'Input `tau` should be in \[0, 1\]'):
    common.soft_variables_update(s, t, tau=1.5)
  t.zero_()
  fired = []
  p = common.Periodically(lambda period, ctr: common.soft_variables_update(s, t, 1.0, period=period, counter=ctr), 3, device=cuda)
  for i in range(7):
    t.zero_()
    p()
    fired.append(bool(t.sum().item() > 0))
  assert fired == [False, False, True, False, False, True, False]
  assert p._counter.cpu().tolist() == [7, 0]


def test_clip_kernels(cuda):
  rng = np.random.RandomState(2)
  sizes = [5, 1000, 1, 4097]
  offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
  g = (rng.randn(offs[-1]) * 3).astype(f32)
  tg = torch.as_tensor(g.copy(), device=cuda)
  toffs = torch.as_tensor(offs, device=cuda)
  _lib.call('b200rl_clip_by_norm_segments', _lib.ptr(tg), _lib.ptr(toffs),
            len(sizes), 2.0, _lib.stream())
  want = np.concatenate([ooptim.clip_by_norm(g[offs[i]:offs[i + 1]], 2.0) for i in range(len(sizes))])
  np.testing.assert_allclose(tg.cpu().numpy(), want, rtol=1e-5, atol=1e-7)
  ws, nb = workspace.get(cuda)
  scale = torch.empty(1, device=cuda); norm = torch.empty(1, device=cuda)
  tg = torch.as_tensor(g, device=cuda)
  _lib.call('b200rl_global_norm_scale', _lib.ptr(tg), tg.numel(), 0.5, _lib.ptr(scale), _lib.ptr(norm),
            _lib.ptr(ws), nb, _lib.stream())
  _, wn = ooptim.clip_by_global_norm([g], 0.5)
  np.testing.assert_allclose(norm.item(), wn, rtol=1e-5)
  np.testing.assert_allclose(scale.item(), 0.5 / max(wn, 0.5), rtol=1e-5)


@pytest.mark.parametrize('B,A,use_mask', [(1, 2, False), (300, 6, False), (513, 5, True)])
def test_epsilon_greedy_bit_exact(cuda, B, A, use_mask):
  rng = np.random.RandomState(B)
  q = rng.randn(B, A).astype(f32)
  mask = None
  if use_mask:
    mask = (rng.rand(B, A) > 0.4).astype(np.int32)
    mask[np.arange(B), rng.randint(0, A, B)] = 1
  rngs = torch.zeros(2, dtype=torch.int64, device=cuda)
  out = torch.empty(B, dtype=torch.int32, device=cuda)
  tq = torch.as_tensor(q, device=cuda)
  tm = None if mask is None else torch.as_tensor(mask, device=cuda)
  for call, eps in enumerate([0.1, 0.5, 1.0, -1.0]):
    _lib.call('b200rl_epsilon_greedy', _lib.ptr(tq), _lib.ptr(tm), B, A, eps, 77, _lib.ptr(rngs),
              None, None, _lib.ptr(out), _lib.stream())
    want = oenv.epsilon_greedy(q, eps, 77, call, mask)
    np.testing.assert_array_equal(out.cpu().numpy(), want)
  assert rngs.cpu().tolist() == [4, 0]


@pytest.mark.parametrize('obs_elems,u8', [(28224, True), (17, False), (33, True)])
def test_random_env_step_bit_exact(cuda, obs_elems, u8):
  B = 37
  st = torch.full((B,), 2, dtype=torch.int32, device=cuda)      # all LAST -> first call resets
  obs = torch.empty((B, obs_elems), dtype=torch.uint8 if u8 else torch.float32, device=cuda)
  rew = torch.empty(B, device=cuda); disc = torch.empty(B, device=cuda)
  rngs = torch.zeros(2, dtype=torch.int64, device=cuda)
  wst = np.full(B, 2, np.int32)
  seen_last = False
  for call in range(12):
    _lib.call('b200rl_env_random_step', _lib.ptr(st), None, _lib.ptr(obs), obs_elems, int(u8), _lib.ptr(rew),
              _lib.ptr(disc), B, 0.3, 5, _lib.ptr(rngs), _lib.stream())
    wst, wobs, wrew, wdisc = oenv.random_env_step(wst, obs_elems, u8, 0.3, 5, call)
    np.testing.assert_array_equal(st.cpu().numpy(), wst)
    np.testing.assert_array_equal(obs.cpu().numpy(), wobs)
    np.testing.assert_array_equal(rew.cpu().numpy(), wrew)
    np.testing.assert_array_equal(disc.cpu().numpy(), wdisc)
    seen_last |= bool((wst == 2).any())
  assert seen_last and (wst == 0).sum() < B
  assert rngs.cpu().tolist() == [12, 0]     # 2-D grid: one advance per launch, ticket back to 0


def test_cartpole_step_parity(cuda):
  B = 64
  rng = np.random.RandomState(0)
  state = torch.zeros(B, 4, device=cuda); steps = torch.zeros(B, dtype=torch.int32, device=cuda)
  st = torch.full((B,), 2, dtype=torch.int32, device=cuda)
  obs = torch.empty(B, 4, device=cuda); rew = torch.empty(B, device=cuda); disc = torch.empty(B, device=cuda)
  rngs = torch.zeros(2, dtype=torch.int64, device=cuda)
  wstate, wsteps, wst = np.zeros((B, 4), f32), np.zeros(B, np.int32), np.full(B, 2, np.int32)
  for call in range(60):
    act = rng.randint(0, 2, size=B).astype(np.int32)
    tact = torch.as_tensor(act, device=cuda)
    _lib.call('b200rl_env_cartpole_step', _lib.ptr(state), _lib.ptr(steps), _lib.ptr(st),
              _lib.ptr(tact), _lib.ptr(obs), _lib.ptr(rew), _lib.ptr(disc), B, 25,
              11, _lib.ptr(rngs), _lib.stream())
    # step the oracle from the device state so 1-ulp sin/cos differences cannot accumulate
    wstate, wsteps, wst2, wobs, wrew, wdisc = oenv.cartpole_step(wstate, wsteps, wst, act, 25, 11, call)
    np.testing.assert_allclose(state.cpu().numpy(), wstate, rtol=1e-5, atol=1e-6)
    near = np.isclose(np.abs(wstate[:, 2]), 0.20943951, atol=1e-5) | np.isclose(np.abs(wstate[:, 0]), 2.4, atol=1e-5)
    got_st = st.cpu().numpy()
    assert ((got_st == wst2) | near).all()
    np.testing.assert_array_equal(steps.cpu().numpy(), wsteps)
    np.testing.assert_array_equal(rew.cpu().numpy(), wrew)
    wstate, wst = state.cpu().numpy(), got_st
    assert ((disc.cpu().numpy() == wdisc) | near).all()
  assert (wsteps <= 25).all()
  assert rngs.cpu().tolist() == [60, 0]
  # several blocks: the resets draw from the launch's call, which advances once per launch
  B = 600
  state = torch.zeros(B, 4, device=cuda); steps = torch.zeros(B, dtype=torch.int32, device=cuda)
  st = torch.full((B,), 2, dtype=torch.int32, device=cuda)
  tact = torch.zeros(B, dtype=torch.int32, device=cuda)
  obs = torch.empty(B, 4, device=cuda); rew = torch.empty(B, device=cuda); disc = torch.empty(B, device=cuda)
  rngs = torch.zeros(2, dtype=torch.int64, device=cuda)
  for call in range(2):
    _lib.call('b200rl_env_cartpole_step', _lib.ptr(state), _lib.ptr(steps), _lib.ptr(st),
              _lib.ptr(tact), _lib.ptr(obs), _lib.ptr(rew), _lib.ptr(disc), B, 25,
              11, _lib.ptr(rngs), _lib.stream())
    assert rngs.cpu().tolist() == [call + 1, 0]
    if call == 0:
      wstate = oenv.cartpole_step(np.zeros((B, 4), f32), np.zeros(B, np.int32), np.full(B, 2, np.int32),
                                  np.zeros(B, np.int32), 25, 11, 0)[0]
      np.testing.assert_allclose(state.cpu().numpy(), wstate, rtol=1e-5, atol=1e-6)
