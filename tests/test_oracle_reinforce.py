"""oracle/reinforce.py against the reference's ReinforceAgent goldens
(agents/reinforce/reinforce_agent_test.py) and its hand-written backward against float64 torch
autograd; ReinforceAgent's rejected configurations (no GPU)."""
import numpy as np
import pytest
import torch

from oracle import ppo
from oracle import ppo_discrete
from oracle import reinforce as R

f32 = np.float32
F, M, L = R.STEP_FIRST, R.STEP_MID, R.STEP_LAST


def _dummy_actor(obs):
  """DummyActorNet(unbounded_actions=True) (reinforce_agent_test.py:38-94): Dense(2) with kernel
  [[2, 1], [1, 1]] and bias 5; loc = obs . [2, 1] + 5, scale = obs . [1, 1] + 5."""
  obs = np.asarray(obs, f32)
  out = obs @ np.array([[2, 1], [1, 1]], f32) + f32(5)
  return out[:, :1], out[:, 1:]


def _pg_golden(obs, actions, is_boundary, returns, num_episodes):
  loc, scale = _dummy_actor(obs)
  logp = ppo.normal_log_prob(loc, scale, np.asarray(actions, f32))
  return R.policy_gradient_loss(logp, np.asarray(is_boundary), np.asarray(returns, f32),
                                num_episodes)


@pytest.mark.parametrize('obs,actions,is_boundary,returns,num_episodes,expected', [
    ([[1, 2], [3, 4]], [[0], [1]], [0, 0], [1.9, 1.0], 1, 10.983667373657227),        # :152-175
    ([[1, 2]] * 4, [[0], [1], [2], [3]], [0, 1, 0, 1], [1.9, 1.9, 1.0, 1.0], 2,
     5.140229225158691),                                                              # :177-211
    ([[1, 2]] * 2, [[0], [1]], [0, 1], [3.0, 0.0], 1, 10.8935775757),                 # :213-260
    ([[1, 2]] * 2, [[0], [1]], [0, 1], [0.0, 3.0], 1, 0.0),                           # :262-309
    ([[1, 2]] * 4, [[0], [1], [2], [3]], [0, 1, 0, 1], [3.0, 0.0, 4.0, 0.0], 2,
     12.2091741562),                                                                  # :311-365
    ([[1, 2]] * 4, [[0], [1], [2], [3]], [0, 1, 0, 1], [0.0, 3.0, 0.0, 4.0], 2, 0.0),  # :367-421
])
def test_policy_gradient_loss_goldens(obs, actions, is_boundary, returns, num_episodes, expected):
  got = _pg_golden(obs, actions, is_boundary, returns, num_episodes)
  np.testing.assert_allclose(got, expected, rtol=1e-6, atol=1e-6)


def test_value_estimation_loss_golden():
  # :444-468: DummyValueNet V = obs . [2, 1] + 5, coef 0.5, num_episodes 1
  obs = np.array([[1, 2], [3, 4]], f32)
  v = obs @ np.array([2, 1], f32) + f32(5)
  got = R.value_estimation_loss(v, np.array([1.9, 1.0], f32), 1, None, 0.5)
  np.testing.assert_allclose(got, 123.205, rtol=1e-6)


@pytest.mark.parametrize('probs,weights', [([[[0.8, 0.2]]], [1]),
                                           ([[[0.8, 0.2]], [[0.3, 0.7]]], [0.5, 0.5])])
def test_entropy_loss_golden(probs, weights):
  # :423-442: mean(-mean(H) * weights)
  logits = np.log(np.asarray(probs, f32)).reshape(-1, 2)
  ent = ppo_discrete.categorical_entropy(logits)
  expected = np.mean(-np.mean(ent) * np.asarray(weights, f32))
  w = np.broadcast_to(np.asarray(weights, f32)[:, None], (len(weights), 1)).reshape(-1)
  got = R.entropy_regularization_loss(ent, w, 1.0)
  np.testing.assert_allclose(got, expected, atol=1e-4)


# reinforce_agent_test.py:470-969: train() of one [1, T] experience, use_advantage_loss=False,
# normalize_returns=False, DummyActorNet, gamma 1.
TRAIN_GOLDENS = {
    'single_bandit': ([F], [L], [3], [0], [0], 10.8935775757),
    'multiple_bandits': ([F, F], [L, L], [3, 4], [0, 0], [0, 2], 12.2091741562),
    'single_episode_reward_on_first': ([F, L], [L, F], [3, 4], [1, 0], [0, 1], 10.8935775757),
    'single_episode_reward_on_last': ([F, L], [L, F], [0, 3], [1, 0], [0, 1], 0.0),
    'multiple_episodes_reward_on_first': ([F, L, F, L], [L, F, L, F], [3, 0, 4, 0], [1, 0, 1, 0],
                                          [0, 1, 2, 3], 12.2091741562),
    'partial_episode': ([F, L, F, M], [L, F, M, M], [3, 0, 4, 0], [1, 0, 1, 0], [0, 1, 2, 3],
                        10.8935775757),
    'multiple_episodes_reward_on_last': ([F, L, F, L], [L, F, L, F], [0, 3, 0, 4], [1, 0, 1, 0],
                                         [0, 1, 2, 3], 0.0),
}


def golden_experience(name):
  st, nst, rew, disc, act, expected = TRAIN_GOLDENS[name]
  T = len(st)
  exp = dict(step_type=np.array([st], np.int32), next_step_type=np.array([nst], np.int32),
             reward=np.array([rew], f32), discount=np.array([disc], f32),
             observation=np.tile(np.array([1, 2], f32), (1, T, 1)),
             action=np.array(act, f32).reshape(1, T, 1))
  return exp, expected


@pytest.mark.parametrize('name', sorted(TRAIN_GOLDENS))
def test_train_loss_goldens(name):
  exp, expected = golden_experience(name)
  ret = R.compute_returns(exp['reward'], exp['discount'], exp['next_step_type'], 1.0)
  loc, scale = _dummy_actor(exp['observation'].reshape(-1, 2))
  T = exp['reward'].shape[1]
  logp = ppo.normal_log_prob(loc, scale, exp['action'].reshape(-1, 1)).reshape(1, T)
  ent = ppo.normal_entropy(scale).reshape(1, T)
  info, _ = R.loss_and_grads(logp, ent, ret, None, exp['step_type'], exp['next_step_type'],
                             use_advantage=False, normalize=False)
  np.testing.assert_allclose(info['total'], expected, rtol=1e-6, atol=1e-6)
  assert info['entropy_regularization_loss'] == 0 and info['value_estimation_loss'] == 0


def test_masks_and_returns():
  nst = np.array([[M, L, F, M, M], [L, F, L, F, M]], np.int32)
  np.testing.assert_array_equal(R.valid_mask(nst), [[1, 1, 0, 0, 0], [1, 1, 1, 0, 0]])
  assert R.num_episodes(nst) == 3
  ret = R.compute_returns(np.ones((1, 4), f32), np.ones((1, 4), f32),
                          np.array([[M, L, M, M]], np.int32), 0.5)
  np.testing.assert_allclose(ret, [[1.5, 1.0, 1.5, 1.0]])
  x = np.array([1.0, 2.0, 3.0, 6.0], f32)
  np.testing.assert_allclose(R.standard_normalize(x),
                             (x - x.mean()) / (x.std() + np.finfo(np.float32).eps), rtol=1e-6)


def test_no_complete_episode_raises():
  z = np.zeros((1, 3), f32)
  with pytest.raises(ValueError, match='No complete episode found'):
    R.loss_and_grads(z, z, z, None, np.array([[F, M, M]]), np.array([[M, M, M]]))


# ---- the hand-written backward against float64 autograd ----------------------------------------
def random_steps(rng, B, T):
  """Consistent step types: FIRST starts every row, LAST w.p. 0.3, FIRST after LAST; rows end
  mid-episode (partial episodes at the row ends) and at least one LAST exists."""
  st = np.zeros((B, T + 1), np.int32)
  for b in range(B):
    for t in range(1, T + 1):
      prev = st[b, t - 1]
      st[b, t] = F if prev == L else (L if rng.random() < 0.3 else M)
  st[0, 2] = L
  st[0, 3] = F
  return st[:, :T].copy(), st[:, 1:].copy()


def torch_total(params, action, V, ret, st, nst, w, cfg, discrete):
  d = torch.float64
  if discrete:
    lp = torch.log_softmax(params, -1)
    logp = lp.gather(1, torch.as_tensor(action, dtype=torch.int64)[:, None])[:, 0]
    H = -(lp.exp() * lp).sum(-1)
  else:
    loc, scale = params
    a = torch.as_tensor(action, dtype=d)
    logp = (-0.5 * ((a - loc) / scale) ** 2 - torch.log(scale) - 0.5 * np.log(2 * np.pi)).sum(-1)
    H = (0.5 + 0.5 * np.log(2 * np.pi) + torch.log(scale)).sum(-1)
  B, T = ret.shape
  logp, H = logp.reshape(B, T), H.reshape(B, T)
  is_last = torch.as_tensor(nst == L, dtype=d)
  ne = is_last.sum()
  valid = (torch.flip(torch.cumsum(torch.flip(is_last, [1]), 1), [1]) > 0).to(d)
  wt = valid * (torch.as_tensor(w, dtype=d) if w is not None else 1.0)
  r = torch.as_tensor(ret, dtype=d)
  adv = r - V if (cfg['use_advantage'] and V is not None) else r
  if cfg['normalize']:
    mean = adv.mean()
    adv = (adv - mean) / (torch.sqrt(((adv - mean) ** 2).mean()) + float(R.EPS))
  c = torch.as_tensor(st != L, dtype=d)
  total = -(logp * c * adv * wt).sum() / ne
  if cfg['entropy']:
    total = total + cfg['entropy'] * (-H * wt).mean()
  if V is not None:
    total = total + cfg['value_coef'] * ((r - V) ** 2 * wt).sum() / ne
  return total


CONFIGS = {
    'baseline_adv_norm': dict(baseline=True, use_advantage=True, normalize=True, entropy=None),
    'baseline_adv_raw': dict(baseline=True, use_advantage=True, normalize=False, entropy=None),
    'baseline_no_adv_norm_ent': dict(baseline=True, use_advantage=False, normalize=True,
                                     entropy=0.01),
    'no_baseline_norm': dict(baseline=False, use_advantage=True, normalize=True, entropy=None),
    'no_baseline_raw_ent_weights': dict(baseline=False, use_advantage=True, normalize=False,
                                        entropy=0.05, weights=True),
    'baseline_adv_norm_ent_weights': dict(baseline=True, use_advantage=True, normalize=True,
                                          entropy=0.02, weights=True),
}


def make_case(rng, B, T, A, discrete, cfg):
  N = B * T
  st, nst = random_steps(rng, B, T)
  ret = rng.normal(size=(B, T)).astype(f32)
  V = rng.normal(size=(B, T)).astype(f32) if cfg['baseline'] else None
  w = rng.uniform(0.2, 1.5, size=(B, T)).astype(f32) if cfg.get('weights') else None
  if discrete:
    params = (rng.normal(size=(N, A)) * 1.5).astype(f32)
    action = rng.integers(0, A, size=N).astype(np.int32)
  else:
    params = (rng.normal(size=(N, A)).astype(f32), rng.uniform(0.4, 1.6, size=(N, A)).astype(f32))
    action = rng.normal(size=(N, A)).astype(f32)
  return dict(st=st, nst=nst, ret=ret, V=V, w=w, params=params, action=action)


def oracle_grads(case, cfg, discrete, value_coef=0.3):
  B, T = case['ret'].shape
  if discrete:
    logp = ppo_discrete.categorical_log_prob(case['params'], case['action'])
    ent = ppo_discrete.categorical_entropy(case['params'])
  else:
    loc, scale = case['params']
    logp = ppo.normal_log_prob(loc, scale, case['action'])
    ent = ppo.normal_entropy(scale)
  info, (g_logp, g_ent, dv) = R.loss_and_grads(
      logp.reshape(B, T), ent.reshape(B, T), case['ret'], case['V'], case['st'], case['nst'],
      case['w'], cfg['use_advantage'], cfg['normalize'], cfg['entropy'], value_coef)
  g_logp, g_ent = g_logp.reshape(-1), g_ent.reshape(-1)
  if discrete:
    dparams = (ppo_discrete.categorical_loss_grad(case['params'], case['action'], g_logp, g_ent),)
  else:
    dparams = R.normal_param_grads(case['params'][0], case['params'][1], case['action'], g_logp,
                                   g_ent)
  return info, dparams, dv


def autograd_grads(case, cfg, discrete, value_coef=0.3):
  d = torch.float64
  if discrete:
    params = torch.tensor(case['params'], dtype=d, requires_grad=True)
    leaves = [params]
  else:
    leaves = [torch.tensor(p, dtype=d, requires_grad=True) for p in case['params']]
    params = tuple(leaves)
  V = None
  if case['V'] is not None:
    V = torch.tensor(case['V'], dtype=d, requires_grad=True)
  total = torch_total(params, case['action'], V, case['ret'], case['st'], case['nst'], case['w'],
                      dict(cfg, value_coef=value_coef), discrete)
  total.backward()
  return total.item(), [l.grad.numpy() for l in leaves], (V.grad.numpy() if V is not None else None)


def _close(got, want, tol):
  scale = max(float(np.abs(want).max()), 1e-3)
  assert float(np.abs(np.asarray(got, np.float64) - want).max()) <= tol * scale


@pytest.mark.parametrize('discrete', [False, True], ids=['normal', 'categorical'])
@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_oracle_backward_matches_float64_autograd(name, discrete):
  cfg = CONFIGS[name]
  rng = np.random.default_rng(7)
  case = make_case(rng, 3, 9, 4 if discrete else 2, discrete, cfg)
  info, dparams, dv = oracle_grads(case, cfg, discrete)
  total, want_params, want_dv = autograd_grads(case, cfg, discrete)
  np.testing.assert_allclose(info['total'], total, rtol=1e-5, atol=1e-6)
  for got, want in zip(dparams, want_params):
    _close(got, want, 1e-4)
  if want_dv is not None:
    _close(dv, want_dv, 1e-4)
  else:
    assert dv is None


def test_zero_spread_advantages_give_a_finite_value_gradient():
  """adv = returns - V constant: the reference's 0 * inf = NaN term is defined as 0 here."""
  cfg = dict(baseline=True, use_advantage=True, normalize=True, entropy=None)
  rng = np.random.default_rng(3)
  case = make_case(rng, 2, 5, 2, True, cfg)
  case['V'] = (case['ret'] - f32(0.5)).astype(f32)
  _, _, dv = oracle_grads(case, cfg, True)
  assert np.all(np.isfinite(dv))


# ---- rejected configurations (host-only construction) ------------------------------------------
def _specs():
  from agents_b200.specs import tensor_spec
  from agents_b200.trajectories import time_step as ts
  obs = tensor_spec.TensorSpec([3], torch.float32)
  act = tensor_spec.BoundedTensorSpec([], torch.int32, 0, 1)
  return ts.time_step_spec(obs), obs, act


def _actor(obs, act):
  from agents_b200.networks import actor_distribution_network
  return actor_distribution_network.ActorDistributionNetwork(obs, act, fc_layer_params=(4,),
                                                             device='cpu')


def test_custom_advantage_fn_is_rejected():
  from agents_b200.agents.reinforce import reinforce_agent
  tss, obs, act = _specs()
  with pytest.raises(NotImplementedError, match='advantage_fn'):
    reinforce_agent.ReinforceAgent(tss, act, _actor(obs, act), None,
                                   advantage_fn=lambda r, v: r)


def test_stateful_actor_is_rejected():
  from agents_b200.agents.reinforce import reinforce_agent
  tss, obs, act = _specs()
  net = _actor(obs, act)
  net._state_spec = (obs,)
  with pytest.raises(NotImplementedError, match='stateless'):
    reinforce_agent.ReinforceAgent(tss, act, net, None)


def test_non_distribution_actor_is_rejected():
  from agents_b200.agents.reinforce import reinforce_agent
  from agents_b200.networks import value_network
  tss, obs, act = _specs()
  with pytest.raises(TypeError, match='distribution'):
    reinforce_agent.ReinforceAgent(tss, act, value_network.ValueNetwork(obs, device='cpu'), None)


def test_multi_replica_training_is_rejected():
  from agents_b200.agents.reinforce import reinforce_agent
  from agents_b200.networks import value_network
  tss, obs, act = _specs()
  agent = reinforce_agent.ReinforceAgent(tss, act, _actor(obs, act), None,
                                         value_network=value_network.ValueNetwork(obs, device='cpu'))
  assert agent.collect_data_spec.policy_info == ()
  assert agent.train_sequence_length is None
  agent.replicas = 2
  with pytest.raises(NotImplementedError, match='one replica'):
    agent.train(None)
