"""Host checks of tests/ddpg_rnn_oracle.py against float64 torch autograd of the reference
formulas (agents/ddpg/ddpg_agent.py critic_loss / actor_loss on [B, T] sequences through recurrent
networks): the losses, the critic and actor gradients, and dQ/da through the critic's LSTM, for
several reset patterns."""
import numpy as np
import pytest
import torch

from oracle import ddpg as oddpg
from oracle import optim
import ddpg_rnn_oracle as oracle

f32 = np.float32
FIRST, MID, LAST = 0, 1, 2


def _dense(rng, i, o, act):
  return {'w': rng.uniform(-0.5, 0.5, (i, o)).astype(f32), 'b': rng.uniform(-0.1, 0.1, o).astype(f32),
          'act': act}


def _cell(rng, i, h):
  return [rng.uniform(-0.5, 0.5, (i, 4 * h)).astype(f32), rng.uniform(-0.5, 0.5, (h, 4 * h)).astype(f32),
          rng.uniform(-0.1, 0.1, 4 * h).astype(f32)]


def _nets(rng, D, A, action_branch):
  actor = oracle.olstm.RnnNet([_dense(rng, D, 6, 'relu')], [_cell(rng, 6, 5)],
                              [_dense(rng, 5, 7, 'relu'), _dense(rng, 7, A, 'tanh')])
  act = [_dense(rng, A, 4, 'relu')] if action_branch else []
  critic = oracle.RnnCritic([_dense(rng, D, 5, 'relu')], act,
                            [_dense(rng, 5 + (4 if action_branch else A), 6, 'relu')],
                            [_cell(rng, 6, 4)], [_dense(rng, 4, 5, 'relu'), _dense(rng, 5, 1, None)])
  return actor, critic


def _t(a, grad=False):
  return torch.tensor(np.asarray(a), dtype=torch.float64, requires_grad=grad)


def _lstm64(x, W, U, b, st):
  B, T, _ = x.shape
  H = U.shape[0]
  h = torch.zeros(B, H, dtype=torch.float64)
  c = torch.zeros(B, H, dtype=torch.float64)
  out = []
  for t in range(T):
    keep = torch.tensor(st[:, t] != FIRST, dtype=torch.float64)[:, None]
    h, c = h * keep, c * keep
    z = x[:, t] @ W + b + h @ U
    i, f, g, o = torch.sigmoid(z[:, :H]), torch.sigmoid(z[:, H:2 * H]), torch.tanh(
        z[:, 2 * H:3 * H]), torch.sigmoid(z[:, 3 * H:])
    c = f * c + i * g
    h = o * torch.tanh(c)
    out.append(h)
  return torch.stack(out, 1)


def _stack64(layers, x, params):
  for l, (w, b) in zip(layers, params):
    x = x @ w + b
    x = torch.relu(x) if l['act'] == 'relu' else torch.tanh(x) if l['act'] == 'tanh' else x
  return x


def _actor64(actor, p, x, st):
  B, T = st.shape
  pre, post = 2 * len(actor.pre), 2 * len(actor.post)
  pairs = lambda ps: list(zip(ps[0::2], ps[1::2]))   # noqa: E731
  y = _stack64(actor.pre, x, pairs(p[:pre]))
  h = _lstm64(y.reshape(B, T, -1), *p[pre:pre + 3], st).reshape(B * T, -1)
  return _stack64(actor.post, h, pairs(p[len(p) - post:]))


def _critic64(critic, p, x, a, st):
  B, T = st.shape
  pairs = lambda ps: list(zip(ps[0::2], ps[1::2]))   # noqa: E731
  no, na, nj = 2 * len(critic.obs), 2 * len(critic.act), 2 * len(critic.joint)
  h = _stack64(critic.obs, x, pairs(p[:no]))
  ab = _stack64(critic.act, a, pairs(p[no:no + na]))
  j = _stack64(critic.joint, torch.cat([h, ab], 1), pairs(p[no + na:no + na + nj]))
  k = no + na + nj
  hs = _lstm64(j.reshape(B, T, -1), *p[k:k + 3], st).reshape(B * T, -1)
  return _stack64(critic.post, hs, pairs(p[k + 3:])).reshape(-1)


PATTERNS = {
    'mid': lambda B, T: np.ones((B, T), np.int32),
    'first_at_0': lambda B, T: np.pad(np.ones((B, T - 1), np.int32), ((0, 0), (1, 0))),
    'mid_first_last': lambda B, T: np.array([[FIRST, MID, LAST, FIRST, MID, MID][:T]] * B, np.int32),
    'staggered': lambda B, T: np.array([[MID if (t + b) % 3 else FIRST for t in range(T)]
                                        for b in range(B)], np.int32),
}


@pytest.mark.parametrize('pattern', sorted(PATTERNS))
@pytest.mark.parametrize('kind,clip,weights,action_branch', [
    (oddpg.HUBER, None, None, True), (oddpg.SQUARED, 0.5, 'row', False),
    (oddpg.HUBER, 0.0, 'scalar', True)])
def test_recurrent_losses_and_gradients_match_float64(pattern, kind, clip, weights, action_branch):
  rng = np.random.default_rng(7)
  B, T, D, A = 3, 6, 4, 2
  actor, critic = _nets(rng, D, A, action_branch)
  st = PATTERNS[pattern](B, T)
  nst = np.roll(st, -1, 1)
  nst[:, -1] = MID
  exp = dict(observation=rng.normal(size=(B, T, D)).astype(f32),
             action=rng.uniform(-1, 2, (B, T, A)).astype(f32),
             reward=rng.normal(size=(B, T)).astype(f32) * 3,
             discount=rng.uniform(0, 1, (B, T)).astype(f32), step_type=st, next_step_type=nst)
  w = {None: None, 'scalar': f32(0.7), 'row': rng.uniform(0, 2, B).astype(f32)}[weights]
  amin, amax = np.array([-1, 0], f32), np.array([2, 1], f32)
  orc = oracle.RecurrentDdpgOracle(actor, critic, amin, amax, optim.AdamTF(), optim.AdamTF(),
                                   gamma=0.9, reward_scale=1.5, loss=kind, dqda_clipping=clip)
  win = orc.windows(exp)
  closs, cgrads, _ = orc.critic_grads(win, w)
  aloss, agrads, dqda = orc.actor_grads(win, w)

  Tm = T - 1
  st0, st1 = win['st0'], win['st1']
  wt = torch.ones(B, dtype=torch.float64) if w is None else _t(np.broadcast_to(w, (B,)))
  scale = lambda y: _t(0.5 * (amax + amin)) + _t(0.5 * (amax - amin)) * y   # noqa: E731
  # critic_loss
  tap = [_t(p) for p in orc.ta.params()]
  tcp = [_t(p) for p in orc.tc.params()]
  a2 = scale(_actor64(actor, tap, _t(win['x1']), st1))
  tq = _critic64(critic, tcp, _t(win['x1']), a2, st1)
  y = 1.5 * _t(win['r'].reshape(-1)) + 0.9 * _t(win['d'].reshape(-1)) * tq
  cp = [_t(p, True) for p in critic.params()]
  e = y - _critic64(critic, cp, _t(win['x0']), _t(win['act']), st0)
  el = torch.where(e.abs() <= 1, 0.5 * e * e, e.abs() - 0.5) if kind == oddpg.HUBER else e * e
  loss64 = (el.reshape(B, Tm).sum(1) * wt).mean()
  g64 = torch.autograd.grad(loss64, cp)
  np.testing.assert_allclose(closs, float(loss64.detach()), rtol=1e-5)
  for g, r in zip(cgrads, g64):
    np.testing.assert_allclose(g, r.numpy(), rtol=1e-4, atol=1e-5)
  # actor_loss: dqda through the critic's recurrence
  ap = [_t(p, True) for p in actor.params()]
  a = scale(_actor64(actor, ap, _t(win['x0']), st0))
  cp = [_t(p) for p in critic.params()]
  a_in = a.detach().requires_grad_(True)
  q = _critic64(critic, cp, _t(win['x0']), a_in, st0)
  dqda64, = torch.autograd.grad(q.sum(), a_in)
  np.testing.assert_allclose(dqda, dqda64.numpy(), rtol=1e-4, atol=1e-6)
  c = dqda64 if clip is None else dqda64.clamp(-clip, clip)
  l = ((a.detach() + c) - a) ** 2
  aloss64 = (l.reshape(B, Tm, A).sum(1) * wt[:, None]).mean()
  ga64 = torch.autograd.grad(aloss64, ap)
  np.testing.assert_allclose(aloss, float(aloss64.detach()), rtol=1e-5, atol=1e-12)
  for g, r in zip(agrads, ga64):
    np.testing.assert_allclose(g, r.numpy(), rtol=1e-4, atol=1e-6)


def test_dqda_sees_later_steps_and_stops_at_reset():
  """dqda[b, t] includes dQ_t'/da_t for later t' of the same episode, and nothing across a FIRST."""
  rng = np.random.default_rng(3)
  B, T, D, A = 2, 5, 3, 1
  _, critic = _nets(rng, D, A, True)
  st = np.array([[FIRST, MID, MID, FIRST, MID]] * B, np.int32)
  critic.step_type = st
  x = rng.normal(size=(B * T, D)).astype(f32)
  a = rng.uniform(-1, 1, (B * T, A)).astype(f32)
  q, tape = critic.forward(x, a, keep=True)
  local = np.zeros(B * T, f32)
  local[1::T] = 1.0                     # only Q at t = 1
  _, da = critic.backward(tape, local)
  da = da.reshape(B, T)
  assert np.all(da[:, 0] != 0) and np.all(da[:, 1] != 0)     # a_0 moves Q_1 through the LSTM
  assert np.all(da[:, 2:] == 0)                               # nothing flows backward in time
  local = np.zeros(B * T, f32)
  local[4::T] = 1.0                     # Q at t = 4, after the reset at t = 3
  _, da = critic.backward(tape, local)
  da = da.reshape(B, T)
  assert np.all(da[:, :3] == 0) and np.all(da[:, 3:] != 0)
