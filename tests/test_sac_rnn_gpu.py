"""Recurrent SAC on the GPU: the b200rl_sac_seq_{critic,actor,alpha}_loss kernels against float64,
the tanh-Normal ActorDistributionRnnNetwork (variables, sequence vs chained steps, copies,
gradients against float64 autograd), SacAgent on it with CriticRnnNetwork critics against the numpy
oracle (tests/sac_rnn_oracle.py) and float64 autograd, CUDA-graph replays, a Learner restore, the
stateful SAC policies, the feed-forward launch counts, the reference train_eval_rnn flow, and a
cue-recall task only a recurrent agent can solve."""
import numpy as np
import pytest
import torch

from agents_b200 import _lib
from agents_b200 import optimizers
from agents_b200.agents.cql import cql_sac_agent
from agents_b200.agents.ppo import ppo_agent
from agents_b200.agents.ppo import ppo_policy
from agents_b200.agents.sac import sac_agent
from agents_b200.drivers import dynamic_episode_driver
from agents_b200.drivers import dynamic_step_driver
from agents_b200.environments import random_tf_environment
from agents_b200.networks import actor_distribution_rnn_network as adrn
from agents_b200.networks import actor_rnn_network
from agents_b200.networks import critic_network
from agents_b200.networks import critic_rnn_network
from agents_b200.networks import lstm_encoding_network
from agents_b200.networks import tanh_normal_projection_network as tnp
from agents_b200.networks import value_rnn_network
from agents_b200.policies import actor_policy
from agents_b200.replay_buffers import tf_uniform_replay_buffer as rb_mod
from agents_b200.specs import tensor_spec
from agents_b200.train import learner as learner_lib
from agents_b200.trajectories import time_step as ts
from agents_b200.utils import common
from oracle import optim as ooptim
from oracle import philox
from oracle import sac as osac

import sac_rnn_oracle as O
import test_ddpg_rnn_gpu as D
import test_oracle_ddpg_rnn as H
import test_oracle_sac_rnn as S

from conftest import record_parity

pytestmark = pytest.mark.gpu
f32 = np.float32
FIRST, MID, LAST = 0, 1, 2
ffma = D.ffma
_leaves, _rel = D._leaves, D._rel


# ---- the kernels --------------------------------------------------------------------------------
class Scratch(object):
  def __init__(self, cuda):
    self.partials = torch.empty(_lib.SAC_SEQ_MAX_BLOCKS, dtype=torch.float32, device=cuda)
    self.ticket = torch.zeros(1, dtype=torch.int32, device=cuda)
    self.nan_flag = torch.zeros(1, dtype=torch.int32, device=cuda)

  def args(self):
    return _lib.ptr(self.nan_flag), _lib.ptr(self.partials), _lib.ptr(self.ticket)


def _seq_calls(s, B, T, q1, q2, tq1, tq2, lp, r, d, w, ws, la, gamma, rs, cw, aw, alw, te, use_la):
  dev, N = q1.device, q1.numel()
  out = dict(closs=torch.empty(1, device=dev), dq1=torch.empty(N, device=dev),
             dq2=torch.empty(N, device=dev), aloss=torch.empty(1, device=dev),
             dlogp=torch.empty(N, device=dev), da1=torch.empty(N, device=dev),
             da2=torch.empty(N, device=dev), alloss=torch.empty(1, device=dev),
             dla=torch.empty(1, device=dev))
  _lib.call('b200rl_sac_seq_critic_loss', _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(tq1), _lib.ptr(tq2),
            _lib.ptr(lp), _lib.dptr(r), _lib.dptr(d), r.stride(0), r.stride(1), _lib.ptr(w), ws,
            _lib.ptr(la), B, T, gamma, rs, cw, _lib.ptr(out['closs']), _lib.ptr(out['dq1']),
            _lib.ptr(out['dq2']), *s.args(), _lib.stream())
  _lib.call('b200rl_sac_seq_actor_loss', _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(lp), _lib.ptr(w), ws,
            _lib.ptr(la), B, T, aw, _lib.ptr(out['aloss']), _lib.ptr(out['dlogp']),
            _lib.ptr(out['da1']), _lib.ptr(out['da2']), *s.args(), _lib.stream())
  _lib.call('b200rl_sac_seq_alpha_loss', _lib.ptr(lp), _lib.ptr(w), ws, _lib.ptr(la), B, T, te,
            int(use_la), alw, _lib.ptr(out['alloss']), _lib.ptr(out['dla']), *s.args(),
            _lib.stream())
  return out


KERNEL_SHAPES = [(1, 1), (7, 8), (64, 9), (33, 64), (1000, 65), (5, 1000), (5000, 8), (300000, 2)]
VARIANTS = [  # weights, gamma, reward scale, critic / actor / alpha loss weights, use_log_alpha
    (None, 0.99, 1.0, 0.5, 1.0, 1.0, True), ('scalar', 0.9, 0.1, 1.5, 0.7, 2.0, False),
    ('row_zeros', 0.5, 2.0, 0.5, 1.0, 0.3, True)]


@pytest.mark.parametrize('B,Tm', KERNEL_SHAPES)
@pytest.mark.parametrize('variant', range(len(VARIANTS)))
def test_seq_kernels_match_float64(cuda, B, Tm, variant):
  wmode, gamma, rs, cw, aw, alw, use_la = VARIANTS[variant]
  rng = np.random.default_rng(B * 31 + Tm * 7 + variant)
  T, N = Tm + 1, B * Tm
  q1, q2, tq1, tq2 = (rng.normal(size=N).astype(f32) * 2 for _ in range(4))
  lp = rng.normal(size=N).astype(f32)
  rd = rng.normal(size=(B, T + 3)).astype(f32)          # [B, T] column views of wider buffers
  dd = rng.uniform(0, 1, (B, T + 3)).astype(f32)
  w = {None: None, 'scalar': np.array([0.7], f32),
       'row_zeros': np.where(rng.uniform(size=B) < 0.2, 0, rng.uniform(0, 2, B)).astype(f32)}[wmode]
  if wmode == 'row_zeros':
    w[-1] = 1.25
    if B > 1:                # a zero-weight row with a nan reward and an inf log-prob adds 0
      w[0] = 0
      rd[0, 0], lp[0] = np.nan, np.inf
  la = np.array([-0.4], f32)
  s = Scratch(cuda)
  d = lambda a: torch.as_tensor(a, device=cuda)   # noqa: E731
  w_t, ws = (None, 0) if w is None else (d(w), int(w.size > 1))
  args = (B, T, d(q1), d(q2), d(tq1), d(tq2), d(lp), d(rd)[:, :T], d(dd)[:, :T], w_t, ws, d(la),
          gamma, rs, cw, aw, alw, -0.6, use_la)
  runs = [_seq_calls(s, *args) for _ in range(2)]
  for k in runs[0]:
    assert torch.equal(runs[0][k], runs[1][k]) or k in ('dq1', 'dq2') and wmode == 'row_zeros'
  assert int(s.ticket.item()) == 0 and int(s.nan_flag.item()) == 0
  got = {k: v.cpu().numpy().astype(np.float64) for k, v in runs[0].items()}
  # float64
  wb = np.ones(B) if w is None else np.broadcast_to(w.astype(np.float64), (B,))
  live = np.repeat(wb != 0, Tm)
  alpha = np.exp(np.float64(la[0]))
  r, dc = rd[:, :Tm].astype(np.float64).reshape(-1), dd[:, :Tm].astype(np.float64).reshape(-1)
  y = rs * r + gamma * dc * (np.minimum(tq1, tq2) - alpha * lp.astype(np.float64))
  e1, e2 = y - q1, y - q2
  rows = lambda per: np.where(wb == 0, 0, per.reshape(B, Tm).sum(1) * wb).sum() / B   # noqa: E731
  with np.errstate(invalid='ignore'):
    closs = cw * rows(np.where(live, e1 * e1 + e2 * e2, 0))
    aloss = aw * rows(np.where(live, alpha * lp - np.minimum(q1, q2), 0))
    S64 = rows(np.where(live, -lp.astype(np.float64) + 0.6, 0))
  k = np.repeat(wb / B, Tm)
  coef, dcoef = (la[0], 1.0) if use_la else (alpha, alpha)
  ref = dict(closs=closs, aloss=aloss, alloss=alw * coef * S64, dla=alw * dcoef * S64,
             dq1=(-2 * e1 * cw * k)[live], dq2=(-2 * e2 * cw * k)[live], dlogp=alpha * aw * k,
             da1=np.where(q1 <= q2, -aw * k, 0), da2=np.where(q1 <= q2, 0, -aw * k))
  errs = {}
  for key, want in ref.items():
    g = got[key][live] if key in ('dq1', 'dq2') else got[key]
    errs[key] = _rel(g, want)
  record_parity('sac_seq_loss_float64', **errs)
  for key, v in errs.items():
    # the TD error y - q cancels: y rounded to fp32 before the subtraction dominates the critic's
    # error, so its loss and dq get more room than the sums alone need
    assert v <= (1e-5 if key in ('closs', 'dq1', 'dq2') else 1e-6), (key, v)


@pytest.mark.parametrize('B', [7, 256, 5000])
def test_one_transition_matches_feed_forward_kernels(cuda, B):
  """At T-1 = 1, dq1, dq2, dlogp and the actor's dq1 / dq2 are the feed-forward kernels' bits; the
  losses agree to fp32 reordering."""
  rng = np.random.default_rng(B)
  d = lambda a: torch.as_tensor(a, device=cuda)   # noqa: E731
  q1, q2, tq1, tq2, lp = (d(rng.normal(size=B).astype(f32) * 2) for _ in range(5))
  r2, d2 = d(rng.normal(size=(B, 2)).astype(f32)), d(rng.uniform(0, 1, (B, 2)).astype(f32))
  w = d(rng.uniform(0, 2, B).astype(f32))
  la = d(np.array([0.3, 0, 0, 0], f32))
  s = Scratch(cuda)
  seq = _seq_calls(s, B, 2, q1, q2, tq1, tq2, lp, r2, d2, w, 1, la, 0.99, 0.5, 0.5, 1.0, 1.0,
                   -1.0, True)
  r, dc = r2[:, 0].contiguous(), d2[:, 0].contiguous()
  ff = {k: torch.empty(B, device=cuda) for k in ('dq1', 'dq2', 'dlogp', 'da1', 'da2')}
  ff.update({k: torch.empty(1, device=cuda) for k in ('closs', 'aloss', 'alloss', 'dla')})
  _lib.call('b200rl_sac_critic_loss', _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(tq1), _lib.ptr(tq2),
            _lib.ptr(lp), _lib.ptr(r), _lib.ptr(dc), _lib.ptr(w), _lib.ptr(la), B, 0.99, 0.5, 0.5,
            float(B), _lib.ptr(ff['closs']), _lib.ptr(ff['dq1']), _lib.ptr(ff['dq2']), None, None,
            _lib.stream())
  _lib.call('b200rl_sac_actor_loss', _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(lp), _lib.ptr(w),
            _lib.ptr(la), B, 1.0, float(B), _lib.ptr(ff['aloss']), _lib.ptr(ff['dlogp']),
            _lib.ptr(ff['da1']), _lib.ptr(ff['da2']), None, _lib.stream())
  _lib.call('b200rl_sac_alpha_loss', _lib.ptr(lp), _lib.ptr(w), _lib.ptr(la), B, -1.0, 1, 1.0,
            float(B), _lib.ptr(ff['alloss']), _lib.ptr(ff['dla']), None, _lib.stream())
  for k in ('dq1', 'dq2', 'dlogp', 'da1', 'da2'):
    assert torch.equal(seq[k], ff[k]), k
  for k in ('closs', 'aloss', 'alloss', 'dla'):
    a, b = seq[k].item(), ff[k].item()
    assert abs(a - b) <= 1e-6 * max(abs(b), 1e-3), (k, a, b)


# ---- the tanh-Normal recurrent actor ------------------------------------------------------------
def _specs(D_=5, A=2):
  return (tensor_spec.TensorSpec((D_,), torch.float32, 'observation'),
          tensor_spec.BoundedTensorSpec((A,), torch.float32, -1.0, 2.0, 'action'))


def _actor(cuda, obs_spec, act_spec, seed=1, fc=(16,), lstm=(8,), out=(12,)):
  return adrn.ActorDistributionRnnNetwork(
      obs_spec, act_spec, input_fc_layer_params=fc, lstm_size=lstm, output_fc_layer_params=out,
      continuous_projection_net=tnp.TanhNormalProjectionNetwork, device=cuda).set_seed(seed)


def _critic(cuda, obs_spec, act_spec, seed=2, action_fc=(6,)):
  return critic_rnn_network.CriticRnnNetwork(
      (obs_spec, act_spec), observation_fc_layer_params=(10,), action_fc_layer_params=action_fc,
      joint_fc_layer_params=(12,), lstm_size=(8,), output_fc_layer_params=(9,),
      device=cuda).set_seed(seed)


def test_tanh_actor_variables_and_errors(cuda):
  """input_fc, LSTM, output_fc, projection Dense(2A) in the reference's order; a glorot_uniform
  head with a zero bias; unsupported projection arguments raise."""
  obs_spec, act_spec = _specs(5, 3)
  net = _actor(cuda, obs_spec, act_spec)
  net.create_variables()
  assert [tuple(v.shape) for v in net.variables] == [
      (5, 16), (16,), (16, 32), (8, 32), (32,), (8, 12), (12,), (12, 6), (6,)]
  head = net._post[-1]
  assert head.activation is None and float(head.bias.abs().max()) == 0.0
  assert float(head.kernel.abs().max()) <= np.sqrt(6.0 / (12 + 6)) + 1e-6
  assert net.num_actions == 3 and net.tanh_normal
  assert torch.equal(net.action_min, torch.full((3,), -1.0, device=cuda))
  h, state = net(torch.randn(4, 7, 5, device=cuda), torch.ones(4, 7, dtype=torch.int32,
                                                                   device=cuda))
  assert tuple(h.shape) == (4, 7, 6) and [tuple(x.shape) for x in state] == [(4, 8), (4, 8)]
  with pytest.raises(NotImplementedError):
    tnp.TanhNormalProjectionNetwork(act_spec, std_transform=torch.nn.functional.softplus)
  with pytest.raises(NotImplementedError):
    tnp.TanhNormalProjectionNetwork(act_spec, activation_fn='relu')
  normal = adrn.ActorDistributionRnnNetwork(obs_spec, act_spec, lstm_size=(4,), device=cuda)
  assert not normal.tanh_normal
  # PPO and ActorPolicy must not misread the [N, 2A] head
  value = value_rnn_network.ValueRnnNetwork(obs_spec, lstm_size=(4,), device=cuda)
  tss = ts.time_step_spec(obs_spec)
  with pytest.raises(NotImplementedError):
    ppo_agent.PPOAgent(tss, act_spec, optimizer=optimizers.Adam(1e-3), actor_net=net,
                       value_net=value, use_gae=True)
  with pytest.raises(NotImplementedError):
    ppo_policy.PPOPolicy(tss, act_spec, net, value)
  with pytest.raises(NotImplementedError):
    actor_policy.ActorPolicy(tss, act_spec, net)


def _seq_inputs(cuda, rng, B, T, D_, A):
  st = np.ones((B, T), np.int32)
  st[:, 0] = FIRST
  st[1, 5] = FIRST
  st[2, 4] = FIRST
  d = lambda a: torch.as_tensor(a, device=cuda)   # noqa: E731
  return d(rng.normal(size=(B, T, D_)).astype(f32)), d(st)


def test_sequence_equals_chained_steps_and_copy_is_independent(cuda):
  rng = np.random.default_rng(5)
  B, T, D_, A = 3, 12, 4, 2
  net = _actor(cuda, *_specs(D_, A))
  obs, st = _seq_inputs(cuda, rng, B, T, D_, A)
  full, fstate = net(obs, st, net.get_initial_state(B))
  state, outs = net.get_initial_state(B), []
  for t in range(T):
    o, state = net(obs[:, t], st[:, t], state)
    outs.append(o)
  chained = torch.stack(outs, 1)
  rel = (chained - full).abs().max().item() / full.abs().max().item()
  record_parity('sac_rnn_actor_chained', rel=rel)
  assert rel <= 1e-5
  for a, b in zip(_leaves(fstate), _leaves(state)):
    assert (a - b).abs().max().item() <= 1e-5 * max(1.0, b.abs().max().item())
  cp = net.copy(name='Copy')
  with torch.no_grad():
    cp.flat_params.copy_(net.flat_params)
  assert torch.equal(cp(obs, st)[0], full)
  assert all(a is not b for a, b in zip(cp.layers, net.layers))
  with torch.no_grad():
    cp.flat_params.add_(torch.randn_like(cp.flat_params) * 0.1)
  assert not torch.allclose(cp(obs, st)[0], full)
  assert torch.equal(net(obs, st)[0], full)


def test_tanh_actor_gradients_match_float64(cuda):
  rng = np.random.default_rng(11)
  B, T, D_, A = 4, 9, 5, 2
  net = _actor(cuda, *_specs(D_, A))
  net.create_variables()
  obs, st = _seq_inputs(cuda, rng, B, T, D_, A)
  oa = D._oracle_actor(net)
  dh = rng.normal(size=(B * T, 2 * A)).astype(f32)
  h, ctx = net.forward_train(obs, st)
  grads = net.backward(ctx, torch.as_tensor(dh, device=cuda))
  ap = [H._t(p, True) for p in oa.params()]
  h64 = H._actor64(oa, ap, H._t(obs.cpu().numpy().reshape(B * T, D_)), st.cpu().numpy())
  assert _rel(h.cpu(), h64.detach().numpy()) <= 1e-5
  for view, r in zip(net._grad_views, torch.autograd.grad(h64, ap, grad_outputs=H._t(dh))):
    err = _rel(view.cpu(), r.numpy())
    record_parity('sac_rnn_actor_grads_float64', rel=err)
    assert err <= 1e-4
  assert grads.data_ptr() == net.flat_grads.data_ptr()


# ---- the agent ----------------------------------------------------------------------------------
def _build(cuda, D_=5, A=2, seed=0, action_fc=(6,), critic2=False, actor_opt=None,
           critic_opt=None, alpha_opt=None, **kw):
  obs_spec, act_spec = _specs(D_, A)
  actor = _actor(cuda, obs_spec, act_spec, seed + 1)
  c2 = _critic(cuda, obs_spec, act_spec, seed + 7, action_fc) if critic2 else None
  agent = sac_agent.SacAgent(
      ts.time_step_spec(obs_spec), act_spec, critic_network=_critic(cuda, obs_spec, act_spec,
                                                                    seed + 2, action_fc),
      actor_network=actor, actor_optimizer=actor_opt or optimizers.Adam(1e-3),
      critic_optimizer=critic_opt or optimizers.Adam(2e-3),
      alpha_optimizer=alpha_opt or optimizers.Adam(3e-3), critic_network_2=c2, seed=seed, **kw)
  agent.initialize()
  return agent


def _experience(rng, B, T, D_, A):
  e = D._experience(rng, B, T, D_, A)
  e['reward'] = e['reward'] * 2
  return e


def _oracle(agent, tau=1.0, period=1, **kw):
  A = agent._actor_network.num_actions
  return O.RecurrentSacOracle(
      D._oracle_actor(agent._actor_network), D._oracle_critic(agent._critic_network_1),
      D._oracle_critic(agent._critic_network_2), [-1.0] * A, [2.0] * A,
      ooptim.AdamTF(1e-3, eps=1e-7), ooptim.AdamTF(2e-3, eps=1e-7), ooptim.AdamTF(3e-3, eps=1e-7),
      tau=tau, period=period, **kw)


TRAIN_CASES = [  # (weights, tau, period, gamma, reward scale, target_entropy, use_log_alpha, c2)
    (None, 1.0, 1, 1.0, 1.0, None, True, False),
    ('row_zeros', 0.5, 2, 0.9, 1.5, -1.3, True, False),
    ('scalar', 0.1, 3, 0.99, 0.1, None, False, True),
    ('row', 0.3, 1, 0.95, 2.0, 0.4, False, False),
]


@pytest.mark.parametrize('case', range(len(TRAIN_CASES)))
def test_recurrent_train_matches_oracle(cuda, case):
  wmode, tau, period, gamma, rs, te, use_la, c2 = TRAIN_CASES[case]
  rng = np.random.default_rng(40 + case)
  B, T, D_, A = 6, 9, 5, 2
  agent = _build(cuda, D_, A, critic2=c2, target_update_tau=tau, target_update_period=period,
                 gamma=gamma, reward_scale_factor=rs, target_entropy=te,
                 use_log_alpha_in_alpha_loss=use_la, initial_log_alpha=-0.2,
                 actor_loss_weight=1.3, critic_loss_weight=0.7, alpha_loss_weight=0.9)
  assert agent.train_sequence_length is None
  orc = _oracle(agent, tau, period, gamma=gamma, reward_scale=rs, target_entropy=te,
                initial_log_alpha=-0.2, actor_loss_weight=1.3, critic_loss_weight=0.7,
                alpha_loss_weight=0.9, use_log_alpha=use_la)
  for step in range(4):
    e = _experience(rng, B, T, D_, A)
    w = {None: None, 'scalar': f32(0.6), 'row': rng.uniform(0, 2, B).astype(f32),
         'row_zeros': np.array([0, 1.5, 0.3, 0, 2.0, 1.0], f32)}[wmode]
    eps = [rng.normal(size=(B, T - 1, A)).astype(f32) for _ in range(3)]
    got = agent.train(D._to_traj(cuda, e), weights=None if w is None else torch.as_tensor(
        w, device=cuda), noise=tuple(torch.as_tensor(x, device=cuda) for x in eps))
    want = orc.train(e, *eps, weights=w)
    for k in ('critic_loss', 'actor_loss', 'alpha_loss'):
      g, r = getattr(got.extra, k).item(), float(want[k])
      rel = abs(g - r) / max(abs(r), 1e-6)
      record_parity('sac_rnn_train_oracle', **{k + '_rel': rel})
      assert rel <= 1e-5, (step, k, g, r)
    la_err = abs(agent.log_alpha.item() - float(orc.log_alpha[0]))
    record_parity('sac_rnn_train_log_alpha', abs=la_err)
    assert la_err <= 1e-6
    for net, params in ((agent._critic_network_1, orc.c1.params()),
                        (agent._critic_network_2, orc.c2.params()),
                        (agent._actor_network, orc.actor.params()),
                        (agent._target_critic_network_1, orc.t1.params()),
                        (agent._target_critic_network_2, orc.t2.params())):
      for v, p in zip(net.variables, params):
        err = _rel(v.detach().cpu(), p)
        record_parity('sac_rnn_train_params', rel=err)
        assert err <= 1e-5, (step, net.name, err)
  agent.check_numerics()
  assert int(agent.train_step_counter.item()) == 4
  assert int(agent._seq_ticket.item()) == 0


@pytest.mark.parametrize('action_fc,use_la', [((6,), True), (None, False)])
def test_optimizer_gradients_match_float64(cuda, action_fc, use_la):
  rng = np.random.default_rng(31)
  B, T, D_, A = 5, 10, 5, 2
  ao, co, alo = D.RecordingOptimizer(), D.RecordingOptimizer(), D.RecordingOptimizer()
  w = np.array([1.2, 0.0, 0.5, 2.0, 0.9], f32)
  agent = _build(cuda, D_, A, action_fc=action_fc, actor_opt=ao, critic_opt=co, alpha_opt=alo,
                 gamma=0.95, reward_scale_factor=1.5, target_update_period=1000,
                 initial_log_alpha=0.3, use_log_alpha_in_alpha_loss=use_la)
  with torch.no_grad():          # targets that differ from the online critics
    agent._target_params.mul_(0.9)
  e = _experience(rng, B, T, D_, A)
  eps = [rng.normal(size=(B, T - 1, A)).astype(f32) for _ in range(3)]
  agent.train(D._to_traj(cuda, e), weights=torch.as_tensor(w, device=cuda),
              noise=tuple(torch.as_tensor(x, device=cuda) for x in eps))
  c1, c2 = D._oracle_critic(agent._critic_network_1), D._oracle_critic(agent._critic_network_2)
  t1, t2 = (D._oracle_critic(agent._target_critic_network_1),
            D._oracle_critic(agent._target_critic_network_2))
  win = O.RecurrentSacOracle.windows(e)
  ref = S.float64_reference(D._oracle_actor(agent._actor_network), c1, c2, t1, t2, win,
                            [x.reshape(-1, A) for x in eps], 0.3, np.full(A, -1, f32),
                            np.full(A, 2, f32), w, 0.95, 1.5, -A / 2.0, use_la)
  views = [(agent._critic_network_1, co.calls[0], ref['critic_grads'][:len(c1.params())]),
           (agent._critic_network_2, co.calls[0], ref['critic_grads'][len(c1.params()):]),
           (agent._actor_network, ao.calls[0], ref['actor_grads'])]
  base = agent._critic_grads.data_ptr()
  for net, rec, refs in views:
    b0 = base if net is not agent._actor_network else net.flat_grads.data_ptr()
    for view, r in zip(net._grad_views, refs):
      off = (view.data_ptr() - b0) // 4
      got = rec[off:off + view.numel()].reshape(view.shape).cpu().numpy()
      err = _rel(got, r)
      record_parity('sac_rnn_grads_float64_' + net.name, rel=err)
      assert err <= 1e-4, (net.name, err)
  dla = alo.calls[0][0].item()
  err = abs(dla - ref['dlog_alpha']) / max(abs(ref['dlog_alpha']), 1e-6)
  record_parity('sac_rnn_dlog_alpha_float64', rel=err)
  assert err <= 1e-5


def test_constructor_and_replica_errors(cuda):
  obs_spec, act_spec = _specs(4, 2)
  actor, critic = _actor(cuda, obs_spec, act_spec), _critic(cuda, obs_spec, act_spec)
  ff_critic = critic_network.CriticNetwork((obs_spec, act_spec), joint_fc_layer_params=(8,),
                                           device=cuda)
  ff_actor = tnp.TanhNormalActorNetwork(obs_spec, act_spec, fc_layer_params=(8,), device=cuda)
  normal = adrn.ActorDistributionRnnNetwork(obs_spec, act_spec, lstm_size=(4,), device=cuda)
  det = actor_rnn_network.ActorRnnNetwork(obs_spec, act_spec, lstm_size=(4,), device=cuda)
  enc = lstm_encoding_network.LSTMEncodingNetwork(obs_spec, lstm_size=(4,), device=cuda)
  tss = ts.time_step_spec(obs_spec)
  mk = lambda a, c, **kw: sac_agent.SacAgent(tss, act_spec, critic_network=c, actor_network=a,  # noqa
                                             actor_optimizer=None, critic_optimizer=None,
                                             alpha_optimizer=None, **kw)
  for a, c, kw in ((actor, ff_critic, {}), (ff_actor, critic, {}), (normal, critic, {}),
                   (det, critic, {}), (enc, enc, {}), (actor, critic, dict(
                       critic_network_2=ff_critic))):
    with pytest.raises(NotImplementedError, match='feed-forward'):
      mk(a, c, **kw)
  with pytest.raises(NotImplementedError):
    mk(actor, critic, gradient_clipping=1.0)
  with pytest.raises(ValueError):
    mk(actor, critic, td_errors_loss_fn=common.element_wise_huber_loss)
  with pytest.raises(NotImplementedError, match='feed-forward'):
    cql_sac_agent.CqlSacAgent(tss, act_spec, critic_network=critic, actor_network=actor,
                              actor_optimizer=None, critic_optimizer=None, alpha_optimizer=None,
                              cql_alpha=1.0, num_cql_samples=1, include_critic_entropy_term=False,
                              use_lagrange_cql_alpha=False)
  agent = _build(cuda, 4, 2)
  with pytest.raises(ValueError, match='at least 2'):
    agent.train(D._to_traj(cuda, _experience(np.random.default_rng(0), 2, 1, 4, 2)))
  traj = D._to_traj(cuda, _experience(np.random.default_rng(0), 2, 4, 4, 2))
  agent.replicas = 2
  with pytest.raises(NotImplementedError):
    agent.train(traj)
  agent.replicas, agent._grad_sync = 1, lambda g: None
  with pytest.raises(NotImplementedError):
    agent.train(traj)


# ---- policies -----------------------------------------------------------------------------------
def test_stateful_sac_policies(cuda):
  agent = _build(cuda, 4, 2)
  B = 6
  obs = torch.randn(B, 4, device=cuda)
  greedy, collect = agent.policy, agent.collect_policy
  assert greedy.policy_state_spec == agent._actor_network.state_spec == collect.policy_state_spec
  s0 = greedy.get_initial_state(B)
  assert all(float(x.abs().max()) == 0 for x in _leaves(s0))
  a1 = greedy.action(D._time_step(cuda, FIRST, obs), s0)
  a2 = greedy.action(D._time_step(cuda, MID, obs), a1.state)
  assert not torch.equal(a1.state[0], a2.state[0])
  a3 = greedy.action(D._time_step(cuda, FIRST, obs), a2.state)     # FIRST resets
  assert all(torch.equal(x, y) for x, y in zip(a3.state, a1.state))
  assert torch.equal(a3.action, a1.action)
  head, _ = agent._actor_network.distribution_params(obs, torch.zeros(B, dtype=torch.int32,
                                                                      device=cuda), s0)
  h = head.cpu().numpy()
  amin, amax = np.full(2, -1, f32), np.full(2, 2, f32)
  want, _, _ = osac.sample_and_log_prob(h, np.zeros((B, 2), f32), amin, amax)
  assert _rel(a1.action.cpu(), want) <= 1e-6               # tanh(loc) scaled to the spec
  # collect: Philox draws through b200rl_sac_sample, element n*A + k of call 0
  c1 = collect.action(D._time_step(cuda, FIRST, obs), s0)
  assert all(torch.equal(x, y) for x, y in zip(c1.state, a1.state))
  r = philox.philox(np.arange(B * 2, dtype=np.uint64), 0, collect._seed)
  u1 = ((r[0] >> np.uint32(8)).astype(np.float64) + 1) / 16777216.0
  z = (np.sqrt(-2 * np.log(u1)) * np.cos(2 * np.pi * philox.uniform_f32(r[1]))).astype(f32)
  z = z.reshape(B, 2)
  want_c, _, _ = osac.sample_and_log_prob(h, z, amin, amax)
  err = _rel(c1.action.cpu(), want_c)
  record_parity('sac_rnn_collect_philox', rel=err)
  assert err <= 1e-5
  for act in (a1.action, c1.action):
    assert float(act.min()) >= -1 and float(act.max()) <= 2
  for pol in (greedy, collect):
    with pytest.raises(ValueError, match='stateful'):
      pol.action(D._time_step(cuda, FIRST, obs))


# Launches of the feed-forward SacAgent policies and train(), and of CqlSacAgent.train(), before
# the recurrent path was added, counted with _lib.launch_count() on the configurations of
# ff_launch_counts: the feed-forward paths must keep issuing exactly these.
PARENT_FF_LAUNCHES = dict(policy=4, collect=4, train=52, cql_train=59)


def ff_launch_counts(cuda):
  obs_spec, act_spec = _specs(5, 2)
  mk_nets = lambda: (  # noqa: E731
      tnp.TanhNormalActorNetwork(obs_spec, act_spec, fc_layer_params=(16, 8),
                                 device=cuda).set_seed(1),
      critic_network.CriticNetwork((obs_spec, act_spec), joint_fc_layer_params=(10,),
                                   device=cuda).set_seed(2))
  actor, critic = mk_nets()
  tss = ts.time_step_spec(obs_spec)
  agent = sac_agent.SacAgent(tss, act_spec, critic_network=critic, actor_network=actor,
                             actor_optimizer=optimizers.Adam(1e-3),
                             critic_optimizer=optimizers.Adam(1e-3),
                             alpha_optimizer=optimizers.Adam(1e-3))
  agent.initialize()
  obs = torch.randn(8, 5, device=cuda)
  out = {}
  for k, pol in (('policy', agent.policy), ('collect', agent.collect_policy)):
    n0 = _lib.launch_count()
    step = pol.action(D._time_step(cuda, MID, obs))
    out[k] = _lib.launch_count() - n0
    assert step.state == () and pol.get_initial_state(8) == ()
  traj = D._to_traj(cuda, D._experience(np.random.default_rng(0), 8, 2, 5, 2))
  agent.train(traj)
  n0 = _lib.launch_count()
  agent.train(traj)
  out['train'] = _lib.launch_count() - n0
  actor, critic = mk_nets()
  cql = cql_sac_agent.CqlSacAgent(tss, act_spec, critic_network=critic, actor_network=actor,
                                  actor_optimizer=optimizers.Adam(1e-3),
                                  critic_optimizer=optimizers.Adam(1e-3),
                                  alpha_optimizer=optimizers.Adam(1e-3), cql_alpha=1.0,
                                  num_cql_samples=4, include_critic_entropy_term=True,
                                  use_lagrange_cql_alpha=False)
  cql.initialize()
  cql.train(traj)
  n0 = _lib.launch_count()
  cql.train(traj)
  out['cql_train'] = _lib.launch_count() - n0
  return out


def test_feed_forward_launches_unchanged(cuda):
  assert ff_launch_counts(cuda) == PARENT_FF_LAUNCHES


# ---- graphs and restore -------------------------------------------------------------------------
def test_train_graph_replays_bit_for_bit(cuda, ffma):
  rng = np.random.default_rng(6)
  B, T, D_, A = 4, 11, 5, 2
  make = lambda: _build(cuda, D_, A, target_update_tau=0.5, target_update_period=2)  # noqa: E731
  eager, graphed = make(), make()
  train_fn = common.function(graphed.train)
  for _ in range(5):
    traj = D._to_traj(cuda, _experience(rng, B, T, D_, A))
    w = torch.as_tensor(rng.uniform(0, 2, B).astype(f32), device=cuda)
    l1 = eager.train(traj, weights=w).loss.item()
    l2 = train_fn(traj, weights=w).loss.item()
    assert l1 == l2
  for a, b in ((graphed._critic_params, eager._critic_params),
               (graphed._target_params, eager._target_params),
               (graphed._actor_network.flat_params, eager._actor_network.flat_params),
               (graphed._log_alpha, eager._log_alpha)):
    assert torch.equal(a, b)
  assert int(graphed._seq_ticket.item()) == 0


def test_stateful_collect_graph_replays_bit_for_bit(cuda):
  """12 runs of 4 collect steps with the actor state threaded through DynamicStepDriver: captured
  into one CUDA graph they store the same trajectories and end in the same state, bit for bit, as
  12 eager runs."""
  B = 8
  out = []
  obs_spec, act_spec = _specs(4, 2)
  for graphed in (False, True):
    agent = _build(cuda, 4, 2)
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
    out.append([t.clone() for t in _leaves(exp)] + [t.clone() for t in _leaves(state)])
  assert int((out[0][0] == FIRST).sum()) > B
  for a, b in zip(*out):
    assert torch.equal(a, b)


def test_learner_restores_bit_for_bit(cuda, tmp_path, ffma):
  rng = np.random.default_rng(8)
  B, T, D_, A = 4, 9, 5, 2
  exps = [D._to_traj(cuda, _experience(rng, B, T, D_, A)) for _ in range(4)]
  a1 = _build(cuda, D_, A, target_update_tau=0.3, seed=0)
  l1 = learner_lib.Learner(str(tmp_path / 'run'), a1.train_step_counter, a1,
                           experience_dataset_fn=lambda: iter([(e, ()) for e in exps]),
                           checkpoint_interval=1)
  l1.run(iterations=2)
  a2 = _build(cuda, D_, A, target_update_tau=0.3, seed=5)
  l2 = learner_lib.Learner(str(tmp_path / 'run'), a2.train_step_counter, a2,
                           experience_dataset_fn=lambda: iter([(e, ()) for e in exps[2:]]),
                           checkpoint_interval=0)
  assert int(a2.train_step_counter.item()) == 2
  for k, v in learner_lib._agent_state_tensors(a1).items():
    assert torch.equal(learner_lib._agent_state_tensors(a2)[k], v), k
  # the train-step draws are not agent state: give the second agent the first one's stream
  a2._train_policy._seed = a1._train_policy._seed
  a2._train_policy._rng = a1._train_policy._rng.clone()
  i1, i2 = l1.run(iterations=2), l2.run(iterations=2)
  assert i1.loss.item() == i2.loss.item()
  assert torch.equal(a1._critic_params, a2._critic_params)
  assert torch.equal(a1._target_params, a2._target_params)
  assert torch.equal(a1._log_alpha, a2._log_alpha)


# ---- the reference example's wiring -------------------------------------------------------------
def test_train_eval_rnn_flow(cuda):
  """sac/examples/v2/train_eval_rnn.py at a small size: DynamicEpisodeDriver collection with the
  stateful collect policy, TFUniformReplayBuffer.as_dataset(num_steps=T), then train."""
  obs_spec = tensor_spec.TensorSpec((3,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((1,), torch.float32, -1.0, 1.0, 'action')
  env = random_tf_environment.RandomTFEnvironment(ts.time_step_spec(obs_spec), act_spec,
                                                  batch_size=1, episode_end_probability=0.05,
                                                  seed=1, device=cuda)
  actor = adrn.ActorDistributionRnnNetwork(
      obs_spec, act_spec, input_fc_layer_params=(40, 30), lstm_size=(8,),
      output_fc_layer_params=(10,), continuous_projection_net=tnp.TanhNormalProjectionNetwork,
      device=cuda)
  critic = critic_rnn_network.CriticRnnNetwork(
      (obs_spec, act_spec), observation_fc_layer_params=None, action_fc_layer_params=None,
      joint_fc_layer_params=(30,), lstm_size=(8,), output_fc_layer_params=(10,),
      kernel_initializer=None, device=cuda)
  agent = sac_agent.SacAgent(ts.time_step_spec(obs_spec), act_spec, actor_network=actor,
                             critic_network=critic, actor_optimizer=optimizers.Adam(3e-4),
                             critic_optimizer=optimizers.Adam(3e-4),
                             alpha_optimizer=optimizers.Adam(3e-4), target_update_tau=0.05,
                             target_update_period=5,
                             td_errors_loss_fn=common.element_wise_squared_loss, gamma=0.99,
                             reward_scale_factor=0.1)
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
def _cue_error(cuda, recurrent, seed, steps=1500, B=64):
  obs_spec = tensor_spec.TensorSpec((2,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((1,), torch.float32, -1.5, 1.5, 'action')
  if recurrent:
    actor = adrn.ActorDistributionRnnNetwork(
        obs_spec, act_spec, input_fc_layer_params=(32,), lstm_size=(16,),
        output_fc_layer_params=(32,), continuous_projection_net=tnp.TanhNormalProjectionNetwork,
        device=cuda).set_seed(seed)
    critic = critic_rnn_network.CriticRnnNetwork(
        (obs_spec, act_spec), observation_fc_layer_params=(32,), action_fc_layer_params=None,
        joint_fc_layer_params=(32,), lstm_size=(16,), output_fc_layer_params=(32,),
        device=cuda).set_seed(seed + 1)
  else:
    actor = tnp.TanhNormalActorNetwork(obs_spec, act_spec, fc_layer_params=(32, 32),
                                       device=cuda).set_seed(seed)
    critic = critic_network.CriticNetwork((obs_spec, act_spec), observation_fc_layer_params=(32,),
                                          joint_fc_layer_params=(32,), device=cuda).set_seed(
                                              seed + 1)
  agent = sac_agent.SacAgent(ts.time_step_spec(obs_spec), act_spec, actor_network=actor,
                             critic_network=critic, actor_optimizer=optimizers.Adam(1e-3),
                             critic_optimizer=optimizers.Adam(3e-3),
                             alpha_optimizer=optimizers.Adam(1e-3), target_update_tau=0.05,
                             gamma=0.0)
  agent.initialize()
  rng = np.random.default_rng(seed)
  for _ in range(steps):
    e = D._cue_batch(rng, B)
    if not recurrent:       # the feed-forward agent trains on the episodes' [*, 2] transitions
      e = {k: np.stack([v[:, :-1], v[:, 1:]], 2).reshape((-1, 2) + v.shape[2:])
           for k, v in e.items()}
    agent.train(D._to_traj(cuda, e))
  agent.check_numerics()
  cue = torch.as_tensor(rng.choice([-1.0, 1.0], 1024).astype(f32), device=cuda)
  state = agent.policy.get_initial_state(1024)
  for t in range(D.CUE_STEPS):
    obs = torch.stack([cue, torch.ones_like(cue)], 1) if t == 0 else torch.zeros(1024, 2,
                                                                                 device=cuda)
    step = agent.policy.action(D._time_step(cuda, FIRST if t == 0 else MID, obs), state)
    state = step.state
  return float((step.action[:, 0] - cue).abs().mean())


def test_cue_recall_needs_memory(cuda):
  """The cue-recall task of test_ddpg_rnn_gpu: recurrent SAC's greedy policy recalls the cue; the
  feed-forward agent cannot beat |a - cue| = 1 in expectation."""
  rnn = _cue_error(cuda, True, 0)
  ff = _cue_error(cuda, False, 0)
  record_parity('sac_rnn_cue_recall', recurrent_error=rnn, feed_forward_error=ff)
  assert rnn <= 0.5, rnn
  assert ff >= 0.9, ff
