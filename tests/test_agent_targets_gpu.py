"""The targets the agents actually train against, against float64 (tests/target_refs.py).

PPOAgent._preprocess: returns and advantages from the value predictions it computed itself,
with and without the TD(λ) return and the reward normaliser, at config 3's 4096 x 128 and at odd
shapes; then the train-time weights and normalised advantages rebuilt with b200rl_ppo_weights,
tensor_normalizer.batch_moments and b200rl_normalize the way PPOAgent._train calls them.
ReinforceAgent._returns with γ = 1 and 0.99, episodes ending inside a 32-step tile.

Bounds are those of target_refs.py (at least 4x the largest error measured on an H100 80GB HBM3
at a 700 W power limit); each comparison records its error with record_parity.
"""
import numpy as np
import pytest
import torch

import target_refs as R
from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.agents.ppo import ppo_agent
from agents_b200.agents.reinforce import reinforce_agent
from agents_b200.networks import actor_distribution_network
from agents_b200.networks import value_network
from agents_b200.specs import tensor_spec
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory
from agents_b200.utils import tensor_normalizer
from conftest import record_parity

pytestmark = pytest.mark.gpu
f32 = np.float32
D, A = 5, 2


def _specs():
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, -1.0, 1.0, 'action')
  return obs_spec, act_spec


def _experience(rng, B, T, p_last=0.05):
  """Episodes end at random steps (inside tiles too); half of the LAST steps are terminations
  (discount 0), the other half time limits that keep their discount."""
  nst = np.ones((B, T), np.int32)
  last = rng.rand(B, T) < p_last
  nst[last] = R.STEP_LAST
  st = np.ones((B, T), np.int32)
  st[:, 1:][last[:, :-1]] = R.STEP_FIRST
  st[:, 0] = R.STEP_FIRST
  disc = np.ones((B, T), f32)
  disc[last & (rng.rand(B, T) < 0.5)] = 0
  return dict(observation=rng.randn(B, T, D).astype(f32),
              action=np.clip(rng.randn(B, T, A) * .5, -1, 1).astype(f32),
              reward=(rng.randn(B, T) * 3 + 2).astype(f32), discount=disc, step_type=st, next_step_type=nst)


def _traj(cuda, e):
  d = lambda a: torch.as_tensor(a, device=cuda)
  B, T = e['reward'].shape
  info = {'dist_params': {'loc': torch.zeros(B, T, A, device=cuda), 'scale': torch.ones(B, T, A, device=cuda)}}
  return trajectory.Trajectory(d(e['step_type']), d(e['observation']), d(e['action']), info,
                               d(e['next_step_type']), d(e['reward']), d(e['discount']))


# ---- PPO -----------------------------------------------------------------------------------------
def _ppo(cuda, **kw):
  obs_spec, act_spec = _specs()
  actor = actor_distribution_network.ActorDistributionNetwork(obs_spec, act_spec, fc_layer_params=(16,),
                                                              device=cuda).set_seed(1)
  value = value_network.ValueNetwork(obs_spec, fc_layer_params=(16,), device=cuda).set_seed(2)
  agent = ppo_agent.PPOAgent(ts.time_step_spec(obs_spec), act_spec, optimizers.Adam(1e-3), actor_net=actor,
                             value_net=value, use_gae=True, lambda_value=0.95, discount_factor=0.99,
                             normalize_observations=False, reward_norm_clipping=10.0, **kw)
  agent.initialize()
  return agent


def _ppo_reference(reward, d_eff, vp, lam, norm):
  """float64 returns / advantages over the first T-1 steps, and their condition sums.  With the
  reward normaliser the kernels see r·inv (uncentred, clipped to ±10) from the normaliser's state;
  its rounding, TOL_NORMALIZE·u·|r|·inv per step, is one more term of each S."""
  B, T = vp.shape
  h = T - 1
  r = R.f64(reward[:, :h])
  rmag = np.abs(r)
  if norm is not None:
    cnt, m2 = norm
    r, rmag = R.normalize(r.reshape(-1, 1), None, m2, cnt, 1e-3, 10.0)
    r, rmag = r.reshape(B, h), rmag.reshape(B, h)
  d = R.f64(d_eff[:, :h])
  ret, Sr = R.recurrence(d, r, vp[:, T - 1], np.maximum(rmag, np.abs(r)))
  a, b, bmag = R.gae_terms(vp[:, :h], vp[:, T - 2], d, r, lam)
  adv, Sa = R.recurrence(a, b, None, bmag - np.abs(r) + np.maximum(rmag, np.abs(r)))
  return ret, Sr, adv, Sa


@pytest.mark.parametrize('B,T', [(4096, 128), (9, 34), (1, 2), (3, 65)])
@pytest.mark.parametrize('td_lambda_return', [False, True])
@pytest.mark.parametrize('normalize_rewards', [False, True])
def test_ppo_preprocess_and_train_targets(cuda, B, T, td_lambda_return, normalize_rewards):
  rng = np.random.RandomState(B + T)
  agent = _ppo(cuda, use_td_lambda_return=td_lambda_return, normalize_rewards=normalize_rewards)
  norm = None
  if normalize_rewards:
    for _ in range(3):
      agent.update_reward_normalizer(torch.as_tensor((rng.randn(64, 33) * 3 + 2).astype(f32), device=cuda))
    cnt, _, m2, _ = agent._reward_normalizer.variables
    norm = (cnt.cpu().numpy(), m2.cpu().numpy())
  e = _experience(rng, B, T)
  vp, ret, adv = agent._preprocess(_traj(cuda, e))
  vp, got_ret, got_adv = vp.cpu().numpy(), ret.cpu().numpy(), adv.cpu().numpy()
  assert (R.bits(got_ret[:, -1]) == 0).all() and (R.bits(got_adv[:, -1]) == 0).all()
  d_eff = R.ppo_discounts(e['discount'], e['next_step_type'], 0.99)
  wret, Sr, wadv, Sa = _ppo_reference(e['reward'], d_eff, vp, 0.95, norm)
  tol = R.TOL_SCAN + (R.TOL_NORMALIZE if normalize_rewards else 0.0)
  ea = R.scan_error(got_adv[:, :-1], wadv, Sa)
  if td_lambda_return:                      # returns = fp32(adv + vp): one more rounding of |ret|
    wret, Sr, tol_r = wadv + vp[:, :-1], Sa + np.abs(vp[:, :-1]), tol + 1.0
  else:
    tol_r = tol
  er = R.scan_error(got_ret[:, :-1], wret, Sr)
  key = f'agent_targets_ppo{"_tdl" if td_lambda_return else ""}{"_norm" if normalize_rewards else ""}'
  record_parity(key, returns=er, advantages=ea)
  assert er <= tol_r and ea <= tol, (er, ea)
  if not normalize_rewards:                  # the kernels saw exactly these inputs: kernel order, bit for bit
    h = T - 1
    assert np.array_equal(R.bits(got_adv[:, :-1]), R.bits(R.gae_kernel_order(
        vp[:, :h], vp[:, T - 2], d_eff[:, :h], e['reward'][:, :h], 0.95)))
    if not td_lambda_return:
      assert np.array_equal(R.bits(got_ret[:, :-1]), R.bits(R.discounted_return_kernel_order(
          e['reward'][:, :h], d_eff[:, :h], vp[:, T - 1])))

  # the train-time weights and normalised advantages, as PPOAgent._train builds them
  N = B * T
  st = _lib.stream()
  w = torch.empty(N, device=cuda)
  step_type = torch.as_tensor(e['step_type'], device=cuda)
  _lib.call('b200rl_ppo_weights', _lib.ptr(step_type), _lib.ptr(ret), _lib.ptr(adv), None, N, _lib.ptr(w), st)
  assert np.array_equal(R.bits(w.cpu().numpy()),
                        R.bits(R.ppo_weights(e['step_type'].reshape(-1), got_ret.reshape(-1),
                                             got_adv.reshape(-1))))
  mean = torch.empty(1, device=cuda)
  var = torch.empty(1, device=cuda)
  tensor_normalizer.batch_moments(adv.reshape(N, 1), 1, mean, var)
  var.mul_(1.0 / N)
  adv_n = torch.empty(N, device=cuda)
  _lib.call('b200rl_normalize', _lib.ptr(adv), _lib.ptr(adv_n), N, 1, _lib.ptr(mean), _lib.ptr(var), None,
            1e-8, 0.0, st)
  mu, m2, absmean = R.column_moments(got_adv.reshape(N, 1))
  em = R.mean_error(mean, mu, absmean)
  ev = R.m2_error(R.f64(var) * N, m2, R.moments_slack(N, absmean))
  want, M = R.normalize(got_adv.reshape(N, 1), mean, var, None, 1e-8, 0.0)
  en = R.normalize_error(adv_n.cpu().numpy().reshape(N, 1), want, M)
  record_parity('agent_targets_ppo_adv_norm', mean=em, m2=ev, normalize=en)
  assert em <= R.TOL_MEAN and ev <= R.TOL_M2 and en <= R.TOL_NORMALIZE, (em, ev, en)


# ---- REINFORCE -----------------------------------------------------------------------------------
def _reinforce(cuda, gamma):
  obs_spec, act_spec = _specs()
  actor = actor_distribution_network.ActorDistributionNetwork(obs_spec, act_spec, fc_layer_params=(4,),
                                                              device=cuda)
  return reinforce_agent.ReinforceAgent(ts.time_step_spec(obs_spec), act_spec, actor, optimizers.Adam(1e-3),
                                        gamma=gamma)


@pytest.mark.parametrize('B,T', [(1, 1), (7, 33), (64, 500)])
@pytest.mark.parametrize('gamma', [1.0, 0.99])
def test_reinforce_returns(cuda, B, T, gamma):
  rng = np.random.RandomState(B * T)
  e = _experience(rng, B, T, p_last=0.02)
  if T > 20:
    e['next_step_type'][0, [13, 20]] = R.STEP_LAST        # episodes that end mid-tile
    e['discount'][0, 13] = 0
    e['next_step_type'][1] = R.STEP_MID                   # one episode as long as the batch
    e['discount'][1] = 1
  got = _reinforce(cuda, gamma)._returns(_traj(cuda, e)).cpu().numpy()
  d_eff = R.ppo_discounts(e['discount'], e['next_step_type'], gamma)
  want, S = R.discounted_return(e['reward'], d_eff, None)
  err = R.scan_error(got, want, S)
  record_parity('agent_targets_reinforce', **{f'gamma{gamma}': err})
  assert err <= R.TOL_SCAN
  assert np.array_equal(R.bits(got), R.bits(R.discounted_return_kernel_order(e['reward'], d_eff, None)))
