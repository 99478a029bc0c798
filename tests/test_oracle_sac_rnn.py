"""Host checks of tests/sac_rnn_oracle.py against float64 torch autograd of the reference formulas
(agents/sac/sac_agent.py critic_loss / actor_loss / alpha_loss on [B, T] sequences through a
recurrent tanh-Normal actor and recurrent critics): the losses, the critic, actor and log-alpha
gradients, and the actor gradient through the tanh-Normal sample and both critics' recurrence,
under four reset patterns, three weight modes and both alpha-loss coefficients."""
import math

import numpy as np
import pytest
import torch

from oracle import lstm as olstm
from oracle import optim
import sac_rnn_oracle as oracle
import test_oracle_ddpg_rnn as H

f32 = np.float32
FIRST, MID, LAST = 0, 1, 2


def _nets(rng, D, A):
  actor = olstm.RnnNet([H._dense(rng, D, 6, 'relu')], [H._cell(rng, 6, 5)],
                       [H._dense(rng, 5, 7, 'relu'), H._dense(rng, 7, 2 * A, None)])
  critics = [oracle.RnnCritic([H._dense(rng, D, 5, 'relu')], act,
                              [H._dense(rng, 5 + (4 if act else A), 6, 'relu')],
                              [H._cell(rng, 6, 4)],
                              [H._dense(rng, 4, 5, 'relu'), H._dense(rng, 5, 1, None)])
             for act in ([H._dense(rng, A, 4, 'relu')], [])]
  return actor, critics[0], critics[1]


def sample64(head, eps, amin, amax):
  """(a, logp) of the tanh-squashed Normal in float64 (oracle.sac.sample_and_log_prob)."""
  A = head.shape[1] // 2
  loc, ls = head[:, :A], head[:, A:]
  u = loc + torch.exp(ls) * eps
  half, shift = 0.5 * (amax - amin), 0.5 * (amax + amin)
  lp = (-0.5 * eps * eps - ls - 0.5 * math.log(2 * math.pi) - torch.log(half) -
        2.0 * (math.log(2.0) - u - torch.nn.functional.softplus(-2.0 * u))).sum(1)
  return shift + half * torch.tanh(u), lp


def _rowsum(per, B, wt):
  return (per.reshape(B, -1).sum(1) * wt).sum() / B


def float64_reference(actor, c1, c2, t1, t2, win, eps, log_alpha, amin, amax, weights=None,
                      gamma=1.0, reward_scale=1.0, target_entropy=-0.5, use_log_alpha=True,
                      cw=0.5, aw=1.0, alw=1.0):
  """Float64 autograd of the three losses at the same parameters (no updates in between).
  eps = (eps_next, eps_actor, eps_alpha), each [N, A].  Returns dict of losses and gradients
  (critic: c1 then c2 params; actor params; log alpha)."""
  B = win['B']
  st0, st1 = win['st0'], win['st1']
  x0, x1 = H._t(win['x0']), H._t(win['x1'])
  lo, hi = H._t(amin), H._t(amax)
  wt = torch.ones(B, dtype=torch.float64) if weights is None else \
      H._t(np.broadcast_to(np.asarray(weights, f32), (B,)))
  alpha = math.exp(float(log_alpha))
  fixed = lambda net: [H._t(p) for p in net.params()]   # noqa: E731
  # critic loss
  a2, lp2 = sample64(H._actor64(actor, fixed(actor), x1, st1), H._t(eps[0]), lo, hi)
  tq = torch.minimum(H._critic64(t1, fixed(t1), x1, a2, st1), H._critic64(t2, fixed(t2), x1, a2,
                                                                           st1)) - alpha * lp2
  y = reward_scale * H._t(win['r'].reshape(-1)) + gamma * H._t(win['d'].reshape(-1)) * tq
  p1, p2 = [H._t(p, True) for p in c1.params()], [H._t(p, True) for p in c2.params()]
  act = H._t(win['act'])
  e1, e2 = y - H._critic64(c1, p1, x0, act, st0), y - H._critic64(c2, p2, x0, act, st0)
  closs = cw * _rowsum(e1 * e1 + e2 * e2, B, wt)
  cgrads = torch.autograd.grad(closs, p1 + p2)
  # actor loss: through the sample and both critics' recurrence
  ap = [H._t(p, True) for p in actor.params()]
  a, lp = sample64(H._actor64(actor, ap, x0, st0), H._t(eps[1]), lo, hi)
  qmin = torch.minimum(H._critic64(c1, fixed(c1), x0, a, st0), H._critic64(c2, fixed(c2), x0, a,
                                                                            st0))
  aloss = aw * _rowsum(alpha * lp - qmin, B, wt)
  agrads = torch.autograd.grad(aloss, ap)
  # alpha loss
  _, lp3 = sample64(H._actor64(actor, fixed(actor), x0, st0), H._t(eps[2]), lo, hi)
  la = torch.tensor(float(log_alpha), dtype=torch.float64, requires_grad=True)
  coef = la if use_log_alpha else torch.exp(la)
  alloss = alw * coef * _rowsum(-lp3 - target_entropy, B, wt)
  dla, = torch.autograd.grad(alloss, la)
  return dict(critic_loss=closs.item(), actor_loss=aloss.item(), alpha_loss=alloss.item(),
              critic_grads=[g.numpy() for g in cgrads], actor_grads=[g.numpy() for g in agrads],
              dlog_alpha=float(dla))


PATTERNS = {
    'none': lambda B, T: np.ones((B, T), np.int32),
    'first_mid': lambda B, T: np.array([[MID, MID, MID, FIRST, MID, MID][:T]] * B, np.int32),
    'first_at_0': lambda B, T: np.pad(np.ones((B, T - 1), np.int32), ((0, 0), (1, 0))),
    'every_first': lambda B, T: np.zeros((B, T), np.int32),
}


def _experience(rng, B, T, D, A, st):
  nst = np.roll(st, -1, 1)
  nst[:, -1] = MID
  return dict(observation=rng.normal(size=(B, T, D)).astype(f32),
              action=rng.uniform(-1, 2, (B, T, A)).astype(f32),
              reward=rng.normal(size=(B, T)).astype(f32) * 3,
              discount=rng.uniform(0, 1, (B, T)).astype(f32), step_type=st, next_step_type=nst)


@pytest.mark.parametrize('pattern', sorted(PATTERNS))
@pytest.mark.parametrize('weights,use_log_alpha', [(None, True), ('scalar', False),
                                                   ('row_zeros', True)])
def test_recurrent_losses_and_gradients_match_float64(pattern, weights, use_log_alpha):
  rng = np.random.default_rng(17)
  B, T, D, A = 3, 6, 4, 2
  actor, c1, c2 = _nets(rng, D, A)
  st = PATTERNS[pattern](B, T)
  exp = _experience(rng, B, T, D, A, st)
  w = {None: None, 'scalar': f32(0.7),
       'row_zeros': np.array([1.3, 0.0, 0.6], f32)}[weights]
  amin, amax = np.array([-1, 0], f32), np.array([2, 1], f32)
  orc = oracle.RecurrentSacOracle(actor, c1, c2, amin, amax, optim.AdamTF(), optim.AdamTF(),
                                  optim.AdamTF(), gamma=0.9, reward_scale=1.5,
                                  target_entropy=-0.8, initial_log_alpha=-0.3,
                                  critic_loss_weight=0.5, actor_loss_weight=1.2,
                                  alpha_loss_weight=0.7, use_log_alpha=use_log_alpha)
  for p in orc.t1.params() + orc.t2.params():   # targets that differ from the online critics
    p *= f32(0.9)
  win = orc.windows(exp)
  N = B * (T - 1)
  eps = [rng.normal(size=(N, A)).astype(f32) for _ in range(3)]
  closs, cgrads = orc.critic_grads(win, eps[0], w)
  aloss, agrads, _ = orc.actor_grads(win, eps[1], w)
  alloss, dla = orc.alpha_grad(win, eps[2], w)
  ref = float64_reference(actor, c1, c2, orc.t1, orc.t2, win, eps, -0.3, amin, amax, w, 0.9, 1.5,
                          -0.8, use_log_alpha, 0.5, 1.2, 0.7)
  for got, k in ((closs, 'critic_loss'), (aloss, 'actor_loss'), (alloss, 'alpha_loss'),
                 (dla, 'dlog_alpha')):
    np.testing.assert_allclose(got, ref[k], rtol=2e-5, atol=1e-6, err_msg=k)
  for g, r in zip(cgrads + agrads, ref['critic_grads'] + ref['actor_grads']):
    np.testing.assert_allclose(g, r, rtol=1e-4, atol=2e-6)


def test_zero_weight_row_adds_exactly_zero():
  """A row of weight 0 whose loss is inf or nan adds 0 to all three losses."""
  B, Tm = 3, 4
  q = np.zeros(B * Tm, f32)
  logp = np.zeros(B * Tm, f32)
  logp[Tm:2 * Tm] = np.inf
  r = np.zeros((B, Tm), f32)
  r[1] = np.nan
  w = np.array([1, 0, 1], f32)
  with np.errstate(invalid='ignore'):
    assert np.isfinite(oracle.seq_critic_loss(q, q, q, q, q, r, np.ones((B, Tm), f32), 0.0,
                                              weights=w)[0])
    assert np.isfinite(oracle.seq_actor_loss(q, q, logp, 0.0, B, w)[0])
    assert np.isfinite(oracle.seq_alpha_loss(logp, 0.0, B, -1.0, True, w)[0])
