"""The kernels between the losses and the optimizer, through the C ABI, against float64 torch.

Covers b200rl_sac_sample / _sac_sample_bwd / _sac_critic_loss / _sac_actor_loss /
_sac_alpha_loss, b200rl_normal_proj_fwd / _normal_proj_bwd chained with b200rl_colsum the way
ActorDistributionNetwork.backward chains them, b200rl_normal_logp, b200rl_normal_sample,
b200rl_colsum with a centre / squares (the normaliser moments), b200rl_concat2, b200rl_l2_sum and
b200rl_add_scaled.  Gradients are float64 autograd of the restated forward (tests/grad_refs.py).

Every output is NaN-filled before the call and carries a canary tail; strided outputs also carry
canary columns past A.  Both must come back untouched.  Each comparison records its measured
error with record_parity; the bounds below are at least 4x the largest value measured on an
H100 80GB HBM3 at a 400 W power limit.
"""
import math

import numpy as np
import pytest
import torch

import grad_refs as R
from agents_b200 import _lib
from agents_b200.utils import workspace
from conftest import record_parity

pytestmark = pytest.mark.gpu
f32 = np.float32
TAIL = 64
# asymmetric per-dimension bounds, cycled over the action dimensions
BOUNDS = [(-2.0, 1.0), (0.0, 10.0), (-0.5, 0.5), (0.1, 0.7), (-7.0, -3.0)]

# bounds, each at least 4x the largest error measured on the H100 (see the module docstring)
TOL_U = 1e-6          # |u - u_ref| / (|loc| + |std·eps|)
TOL_ACTION = 2e-6     # |a - a_ref| / (|shift| + half)
TOL_LOGP = 1e-6       # |logp - logp_ref| / Σ_k |terms_k|
TOL_GRAD = 1e-5       # relative L2 and max-error-over-max of every gradient tensor
TOL_LOSS = 1e-5       # |loss - ref| / (Σ_b |w_b·term_b| · scale)
# The critic's TD error y - q is a difference of fp32 values, so rows with y ≈ q carry the
# rounding of y at a much larger relative size (measured: dq 3.7e-6, loss 7.4e-6).
TOL_CRITIC_GRAD = 2e-5
TOL_CRITIC_LOSS = 4e-5
TOL_SUM = 1e-5        # column sums / l2 sums, error / Σ|term|
TOL_AXPY = 5e-7       # add_scaled, error / (|dst| + |alpha·src|)


def _canary(n, offset=0.0):
  return torch.arange(n, dtype=torch.float32) * 0.25 - 9.75 + offset


class Out(object):
  """A NaN-filled [rows, ld] float32 output with canary columns [cols, ld) and a canary tail."""

  def __init__(self, cuda, rows, cols, ld=None):
    ld = cols if ld is None else ld
    self.rows, self.cols, self.ld = rows, cols, ld
    self.buf = torch.full((rows * ld + TAIL,), float('nan'), device=cuda)
    self.want = self.buf.clone()
    self.want[rows * ld:] = _canary(TAIL).to(cuda)
    if ld > cols:
      grid = self.want[:rows * ld].view(rows, ld)
      grid[:, cols:] = _canary(ld - cols, 100.0).to(cuda)
    self.buf.copy_(self.want)

  def ptr(self):
    return self.buf.data_ptr()

  def value(self):
    return self.buf[:self.rows * self.ld].view(self.rows, self.ld)[:, :self.cols]

  def check_canaries(self, what):
    tail = self.buf[self.rows * self.ld:]
    assert torch.equal(tail, self.want[self.rows * self.ld:]), f'{what}: canary tail overwritten'
    if self.ld > self.cols:
      got = self.buf[:self.rows * self.ld].view(self.rows, self.ld)[:, self.cols:]
      want = self.want[:self.rows * self.ld].view(self.rows, self.ld)[:, self.cols:]
      assert torch.equal(got, want), f'{what}: canary columns past A overwritten'


def _dev(cuda, a):
  return torch.as_tensor(np.ascontiguousarray(a, dtype=f32), device=cuda)


def _bounds(A):
  amin = np.array([BOUNDS[k % len(BOUNDS)][0] for k in range(A)], f32)
  amax = np.array([BOUNDS[k % len(BOUNDS)][1] for k in range(A)], f32)
  return amin, amax


def _rel(err, mag):
  """max over elements of |err| / magnitude."""
  return float((R.t64(err).abs() / R.t64(mag).clamp(min=1e-30)).max())


# ---- tanh-Normal sampling (SAC) -------------------------------------------------------------------
def _sac_inputs(rng, N, A):
  loc = rng.uniform(-6, 6, (N, A)).astype(f32)
  log_std = rng.uniform(-5, 2, (N, A)).astype(f32)
  eps = rng.randn(N, A).astype(f32)
  # pin |u| > 10 on both sides (tanh saturation, softplus(-2u) on both sides of 20)
  pinned = [(6.0, 2.0, 1.0), (-6.0, 2.0, -1.0), (5.0, 1.2, 2.0), (0.1, -5.0, 0.3)]
  flat = [(i // A, i % A) for i in range(min(N * A, len(pinned)))]
  for (n, k), (l, s, e) in zip(flat, pinned):
    loc[n, k], log_std[n, k], eps[n, k] = l, s, e
  return np.concatenate([loc, log_std], axis=1), eps


def _sac_sample(cuda, head, eps, amin, amax, ld):
  N, A = eps.shape
  th, te, tmin, tmax = (_dev(cuda, x) for x in (head, eps, amin, amax))
  act, logp, u, e = Out(cuda, N, A, ld), Out(cuda, N, 1), Out(cuda, N, A), Out(cuda, N, A)
  _lib.call('b200rl_sac_sample', _lib.ptr(th), N, A, _lib.ptr(tmin), _lib.ptr(tmax), _lib.ptr(te), 0,
            None, act.ptr(), ld, logp.ptr(), u.ptr(), e.ptr(), _lib.stream())
  torch.cuda.synchronize()
  for o, what in ((act, 'action'), (logp, 'logp'), (u, 'u'), (e, 'eps')):
    o.check_canaries(what)
  return act.value(), logp.value()[:, 0], u.value(), e.value()


@pytest.mark.parametrize('A', [1, 6, 17])
@pytest.mark.parametrize('N', [1, 257, 4099])
def test_sac_sample(cuda, N, A):
  rng = np.random.RandomState(N * 31 + A)
  head, eps = _sac_inputs(rng, N, A)
  amin, amax = _bounds(A)
  act, logp, u, e = _sac_sample(cuda, head, eps, amin, amax, A + 3)
  assert torch.equal(e.cpu(), torch.as_tensor(eps))
  h64, e64, lo, hi = (R.t64(x) for x in (head, eps, amin, amax))
  a_ref, u_ref, logp_ref = R.sac_sample(h64, e64, lo, hi)
  assert bool((u_ref > 10).any()) and (N * A < 2 or bool((u_ref < -10).any()))
  std_e = torch.exp(h64[:, A:]) * e64
  err_u = _rel(R.t64(u) - u_ref, h64[:, :A].abs() + std_e.abs())
  half, shift = (hi - lo) / 2, (hi + lo) / 2
  err_a = _rel(R.t64(act) - a_ref, (shift.abs() + half).expand_as(a_ref))
  terms = (0.5 * e64 * e64 + h64[:, A:].abs() + 0.5 * R.LOG2PI + torch.log(half).abs()
           + 2 * (R.LOG2 + u_ref.abs() + R.softplus(-2 * u_ref))).sum(dim=1)
  err_lp = _rel(R.t64(logp) - logp_ref, terms)
  record_parity('grad_kernels_sac_sample', u=err_u, action=err_a, logp=err_lp)
  assert err_u <= TOL_U and err_a <= TOL_ACTION and err_lp <= TOL_LOGP, (err_u, err_a, err_lp)
  a = act.cpu()
  assert bool((a >= torch.as_tensor(amin)).all() and (a <= torch.as_tensor(amax)).all()), \
      'an action left [amin, amax]'


@pytest.mark.parametrize('which', ['da1', 'da2', 'both'])
@pytest.mark.parametrize('A', [1, 6, 17])
@pytest.mark.parametrize('N', [1, 257, 4099])
def test_sac_sample_bwd(cuda, N, A, which):
  """dL/dhead for L = Σ da·a + Σ dlogp·logp, eps fixed; da read from [N, o_dim + A] critic
  input-gradient rows at a pointer offset of o_dim, as SacAgent passes them."""
  rng = np.random.RandomState(N * 7 + A)
  o_dim = 5
  head, eps = _sac_inputs(rng, N, A)
  amin, amax = _bounds(A)
  _, _, u, e = _sac_sample(cuda, head, eps, amin, amax, A)
  dx1 = _dev(cuda, rng.randn(N * (o_dim + A) + TAIL))
  dx2 = _dev(cuda, rng.randn(N * (o_dim + A) + TAIL))
  dlogp = _dev(cuda, rng.randn(N))
  th, tmin, tmax = _dev(cuda, head), _dev(cuda, amin), _dev(cuda, amax)
  u, e = u.contiguous(), e.contiguous()
  p1 = dx1.data_ptr() + 4 * o_dim if which in ('da1', 'both') else None
  p2 = dx2.data_ptr() + 4 * o_dim if which in ('da2', 'both') else None
  dhead = Out(cuda, N, 2 * A)
  _lib.call('b200rl_sac_sample_bwd', _lib.ptr(th), _lib.ptr(u), _lib.ptr(e), _lib.ptr(tmin),
            _lib.ptr(tmax), p1, p2, o_dim + A, _lib.ptr(dlogp), N, A, dhead.ptr(), _lib.stream())
  torch.cuda.synchronize()
  dhead.check_canaries('dhead')
  rows = lambda t: R.t64(t[:N * (o_dim + A)].view(N, o_dim + A)[:, o_dim:])
  da = torch.zeros(N, A, dtype=R.F64)
  if p1 is not None:
    da = da + rows(dx1)
  if p2 is not None:
    da = da + rows(dx2)
  h64 = R.t64(head).requires_grad_()
  a, _, logp = R.sac_sample(h64, R.t64(eps), R.t64(amin), R.t64(amax))
  (g_ref,) = torch.autograd.grad((da * a).sum() + (R.t64(dlogp) * logp).sum(), h64)
  got = dhead.value()
  for name, gs, rs in (('dloc', got[:, :A], g_ref[:, :A]), ('dlog_std', got[:, A:], g_ref[:, A:])):
    rel, mx = R.grad_errors(gs, rs)
    record_parity('grad_kernels_sac_sample_bwd', **{name + '_rel_l2': rel, name + '_max': mx})
    R.assert_grad_close(f'{name} N={N} A={A} {which}', gs, rs, TOL_GRAD, TOL_GRAD)


# ---- SAC losses -----------------------------------------------------------------------------------
def _ties(rng, B, frac=0.1):
  a, b = rng.randn(B).astype(f32) * 3, rng.randn(B).astype(f32) * 3
  tie = rng.rand(B) < frac
  tie[0] = True
  b[tie] = a[tie]
  return a, b


def _weights(rng, B):
  w = rng.rand(B).astype(f32) * 2
  w[rng.rand(B) < 0.2] = 0.0
  return w


@pytest.mark.parametrize('gb_factor', [1, 2])
@pytest.mark.parametrize('use_weights', [False, True])
@pytest.mark.parametrize('B', [1, 255, 256, 257, 4096])
def test_sac_losses(cuda, B, use_weights, gb_factor):
  rng = np.random.RandomState(B * 4 + 2 * use_weights + gb_factor)
  gb = float(gb_factor * B)
  q1, q2 = _ties(rng, B)
  tq1, tq2 = _ties(rng, B)
  qa1, qa2 = _ties(rng, B)
  next_logp, logp = rng.randn(B).astype(f32) * 4, rng.randn(B).astype(f32) * 4
  reward, discount = rng.randn(B).astype(f32), (rng.rand(B) > 0.1).astype(f32)
  w = _weights(rng, B) if use_weights else None
  gamma, reward_scale, lw_c, lw_a, lw_al, target_entropy = 0.93, 2.5, 0.7, 1.3, 0.6, -3.0
  t = {k: _dev(cuda, v) for k, v in dict(q1=q1, q2=q2, tq1=tq1, tq2=tq2, nl=next_logp, lp=logp,
                                          r=reward, d=discount, qa1=qa1, qa2=qa2).items()}
  tw = _dev(cuda, w) if use_weights else None
  w64 = R.t64(w) if use_weights else None
  wabs = w64.abs() if use_weights else torch.ones(B, dtype=R.F64)
  flag = torch.zeros(1, dtype=torch.int32, device=cuda)
  for log_alpha in (0.0, 0.7, -1.3):
    la = torch.full((4,), log_alpha, dtype=torch.float32, device=cuda)
    la32 = float(la[0])
    alpha = math.exp(la32)
    # critic
    loss, dq1, dq2, td = Out(cuda, 1, 1), Out(cuda, B, 1), Out(cuda, B, 1), Out(cuda, B, 1)
    _lib.call('b200rl_sac_critic_loss', _lib.ptr(t['q1']), _lib.ptr(t['q2']), _lib.ptr(t['tq1']),
              _lib.ptr(t['tq2']), _lib.ptr(t['nl']), _lib.ptr(t['r']), _lib.ptr(t['d']), _lib.ptr(tw),
              _lib.ptr(la), B, gamma, reward_scale, lw_c, gb, loss.ptr(), dq1.ptr(), dq2.ptr(), td.ptr(),
              _lib.ptr(flag), _lib.stream())
    q64 = [R.t64(x).requires_grad_() for x in (q1, q2)]
    ref, y = R.sac_critic_loss(q64[0], q64[1], R.t64(tq1), R.t64(tq2), R.t64(next_logp), R.t64(reward),
                               R.t64(discount), la32, gamma, reward_scale, lw_c, gb, w64)
    g1, g2 = torch.autograd.grad(ref, q64)
    y_mag = (reward_scale * R.t64(reward).abs() + gamma * R.t64(discount) *
             (torch.minimum(R.t64(tq1), R.t64(tq2)).abs() + alpha * R.t64(next_logp).abs()))
    err_y = _rel(R.t64(td.value()[:, 0]) - y, y_mag)
    per_abs = ((y - q64[0].detach()) ** 2 + (y - q64[1].detach()) ** 2) * wabs
    err_l = abs(float(loss.value()[0, 0]) - float(ref.detach())) / max(lw_c * float(per_abs.sum()) / gb, 1e-30)
    # actor
    aloss, dlogp, dqa1, dqa2 = Out(cuda, 1, 1), Out(cuda, B, 1), Out(cuda, B, 1), Out(cuda, B, 1)
    _lib.call('b200rl_sac_actor_loss', _lib.ptr(t['qa1']), _lib.ptr(t['qa2']), _lib.ptr(t['lp']), _lib.ptr(tw),
              _lib.ptr(la), B, lw_a, gb, aloss.ptr(), dlogp.ptr(), dqa1.ptr(), dqa2.ptr(), _lib.ptr(flag),
              _lib.stream())
    a64 = [R.t64(x).requires_grad_() for x in (qa1, qa2, logp)]
    aref = R.sac_actor_loss(a64[0], a64[1], a64[2], la32, lw_a, gb, w64)
    ga1, ga2, glp = torch.autograd.grad(aref, a64)
    a_abs = (alpha * R.t64(logp).abs() + torch.minimum(R.t64(qa1), R.t64(qa2)).abs()) * wabs
    err_al = abs(float(aloss.value()[0, 0]) - float(aref.detach())) / max(lw_a * float(a_abs.sum()) / gb, 1e-30)
    grads = [('dq1', dq1, g1), ('dq2', dq2, g2), ('dqa1', dqa1, ga1), ('dqa2', dqa2, ga2),
             ('dlogp', dlogp, glp)]
    for use_log_alpha in (1, 0):
      lal, dla = Out(cuda, 1, 1), Out(cuda, 1, 4)
      _lib.call('b200rl_sac_alpha_loss', _lib.ptr(t['lp']), _lib.ptr(tw), _lib.ptr(la), B, target_entropy,
                use_log_alpha, lw_al, gb, lal.ptr(), dla.ptr(), _lib.ptr(flag), _lib.stream())
      la64 = torch.tensor(la32, dtype=R.F64, requires_grad=True)
      lref = R.sac_alpha_loss(R.t64(logp), la64, target_entropy, bool(use_log_alpha), lw_al, gb, w64)
      (gla,) = torch.autograd.grad(lref, la64)
      coef, dcoef = (abs(la32), 1.0) if use_log_alpha else (alpha, alpha)
      s_abs = float(((-R.t64(logp) - target_entropy).abs() * wabs).sum()) * lw_al / gb
      err_all = abs(float(lal.value()[0, 0]) - float(lref.detach())) / max(coef * s_abs, 1e-30)
      err_dla = abs(float(dla.value()[0, 0]) - float(gla)) / max(dcoef * s_abs, 1e-30)
      record_parity('grad_kernels_sac_losses', alpha_loss=err_all, dlog_alpha=err_dla)
      assert err_all <= TOL_LOSS, (use_log_alpha, log_alpha, err_all)
      assert err_dla <= TOL_LOSS, (use_log_alpha, log_alpha, err_dla)
      lal.check_canaries('alpha loss')
      assert torch.isnan(dla.value()[0, 1:]).all(), 'dlog_alpha wrote past element 0'
      dla.check_canaries('dlog_alpha')
    torch.cuda.synchronize()
    record_parity('grad_kernels_sac_losses', td_targets=err_y, critic_loss=err_l, actor_loss=err_al)
    assert err_y <= TOL_LOSS and err_l <= TOL_CRITIC_LOSS and err_al <= TOL_LOSS, (err_y, err_l, err_al)
    for name, o, g in grads:
      rel, mx = R.grad_errors(o.value()[:, 0], g)
      record_parity('grad_kernels_sac_losses', **{name + '_rel_l2': rel, name + '_max': mx})
      tol = TOL_CRITIC_GRAD if name in ('dq1', 'dq2') else TOL_GRAD
      R.assert_grad_close(f'{name} B={B} log_alpha={log_alpha}', o.value()[:, 0], g, tol, tol)
    for o, what in ((loss, 'critic loss'), (dq1, 'dq1'), (dq2, 'dq2'), (td, 'td_targets'),
                    (aloss, 'actor loss'), (dlogp, 'dlogp'), (dqa1, 'dqa1'), (dqa2, 'dqa2')):
      o.check_canaries(what)
  assert flag.item() == 0


# ---- Normal projection head + std-bias column sum ------------------------------------------------
@pytest.mark.parametrize('A', [1, 6, 63, 64])
@pytest.mark.parametrize('N', [1, 300, 70000])
def test_normal_projection_fwd_bwd_colsum(cuda, N, A):
  """The chain of ActorDistributionNetwork._head and .backward: proj_fwd -> (loss) -> proj_bwd ->
  colsum of the per-row std-bias gradient."""
  rng = np.random.RandomState(N + A)
  amin, amax = _bounds(A)
  m_raw = (rng.randn(N, A) * 2).astype(f32)
  s_raw = np.array([(-30.0, 0.0, 19.9, 20.1, 25.0)[k % 5] for k in range(A)], f32)
  dloc, dscale = rng.randn(N, A).astype(f32), rng.randn(N, A).astype(f32)
  tm, ts_, tmin, tmax, tdl, tds = (_dev(cuda, x) for x in (m_raw, s_raw, amin, amax, dloc, dscale))
  loc, scale, dm, dsp, ds = Out(cuda, N, A), Out(cuda, N, A), Out(cuda, N, A), Out(cuda, N, A), Out(cuda, 1, A)
  st = _lib.stream()
  _lib.call('b200rl_normal_proj_fwd', _lib.ptr(tm), _lib.ptr(ts_), _lib.ptr(tmin), _lib.ptr(tmax), N, A,
            loc.ptr(), scale.ptr(), st)
  _lib.call('b200rl_normal_proj_bwd', _lib.ptr(tm), _lib.ptr(ts_), _lib.ptr(tmin), _lib.ptr(tmax),
            _lib.ptr(tdl), _lib.ptr(tds), N, A, dm.ptr(), dsp.ptr(), st)
  ws, nb = workspace.get(cuda)
  part = dsp.value().contiguous()
  _lib.call('b200rl_colsum', _lib.ptr(part), None, 0, N, A, 1.0, ds.ptr(), _lib.ptr(ws), nb, st)
  torch.cuda.synchronize()
  for o, what in ((loc, 'loc'), (scale, 'scale'), (dm, 'dm_raw'), (dsp, 'ds_part'), (ds, 'ds')):
    o.check_canaries(what)
  m64, s64 = R.t64(m_raw).requires_grad_(), R.t64(s_raw).requires_grad_()
  lo, hi = R.t64(amin), R.t64(amax)
  loc_ref, scale_ref = R.normal_projection(m64, s64, lo, hi)
  L = (R.t64(dloc) * loc_ref).sum() + (R.t64(dscale) * scale_ref).sum()
  gm, gs = torch.autograd.grad(L, [m64, s64])
  half, shift = (hi - lo) / 2, (hi + lo) / 2
  err_loc = _rel(R.t64(loc.value()) - loc_ref.detach(), (shift.abs() + half).expand(N, A))
  err_scale = _rel(R.t64(scale.value()) - scale_ref.detach(), scale_ref.detach())
  # the reduced std-bias gradient, per column against Σ_n |dscale_n · sigmoid(s)|
  col_mag = R.t64(dscale).abs().sum(0) * torch.sigmoid(R.t64(s_raw))
  err_ds = _rel(R.t64(ds.value()[0]) - gs, col_mag)
  rel, mx = R.grad_errors(dm.value(), gm)
  record_parity('grad_kernels_normal_projection', loc=err_loc, scale=err_scale, ds_col=err_ds,
                dm_raw_rel_l2=rel, dm_raw_max=mx)
  assert err_loc <= TOL_ACTION and err_scale <= TOL_U, (err_loc, err_scale)
  assert err_ds <= TOL_SUM, err_ds
  R.assert_grad_close(f'dm_raw N={N} A={A}', dm.value(), gm, TOL_GRAD, TOL_GRAD)


# ---- Normal log-prob and sampling (PPO) ----------------------------------------------------------
def test_normal_logp_strided(cuda):
  rng = np.random.RandomState(11)
  N, A, ld = 1031, 6, 9
  loc = np.full((N, ld), np.nan, f32)
  scale = np.full((N, ld), np.nan, f32)
  loc[:, :A] = rng.randn(N, A) * 2
  scale[:, :A] = rng.rand(N, A) * 2 + 0.05
  action = (loc[:, :A] + scale[:, :A] * rng.randn(N, A) * 2).astype(f32)
  tl, tsc, ta = _dev(cuda, loc), _dev(cuda, scale), _dev(cuda, action)
  out = Out(cuda, N, 1)
  _lib.call('b200rl_normal_logp', _lib.ptr(tl), _lib.ptr(tsc), ld, _lib.ptr(ta), N, A, out.ptr(), _lib.stream())
  torch.cuda.synchronize()
  out.check_canaries('logp')
  l64, s64, a64 = R.t64(loc[:, :A]), R.t64(scale[:, :A]), R.t64(action)
  ref = R.normal_log_prob(l64, s64, a64)
  z = (a64 - l64) / s64
  mag = (0.5 * z * z + torch.log(s64).abs() + 0.5 * R.LOG2PI).sum(1)
  err = _rel(R.t64(out.value()[:, 0]) - ref, mag)
  record_parity('grad_kernels_normal_logp', logp=err)
  assert err <= TOL_LOGP, err


def _normal_sample(cuda, loc, scale, ld, N, A, amin, amax, rng_call, seed=5):
  out = Out(cuda, N, A)
  _lib.call('b200rl_normal_sample', _lib.ptr(loc), _lib.ptr(scale), ld, N, A, _lib.ptr(amin), _lib.ptr(amax),
            seed, _lib.ptr(rng_call), out.ptr(), _lib.stream())
  torch.cuda.synchronize()
  out.check_canaries('normal_sample')
  return out.value().clone()


def test_normal_sample_clips_to_bounds(cuda):
  rng = np.random.RandomState(12)
  N, A, ld = 4099, 5, 8
  amin, amax = _bounds(A)
  loc = np.full((N, ld), np.nan, f32)
  scale = np.full((N, ld), np.nan, f32)
  # loc at or near a bound, so that clipping engages on both sides
  near = np.where(rng.rand(N, A) < 0.5, amin, amax)
  loc[:, :A] = near + (rng.rand(N, A) - 0.5) * 0.1 * (amax - amin)
  scale[:, :A] = 0.2 * (amax - amin)
  tl, tsc, tmin, tmax = (_dev(cuda, x) for x in (loc, scale, amin, amax))
  rng_call = torch.zeros(2, dtype=torch.int64, device=cuda)
  x = _normal_sample(cuda, tl, tsc, ld, N, A, tmin, tmax, rng_call)
  lo, hi = torch.as_tensor(amin, device=cuda), torch.as_tensor(amax, device=cuda)
  assert bool(torch.isfinite(x).all()), 'a draw read past A (NaN padding) or is not finite'
  assert bool(((x >= lo) & (x <= hi)).all()), 'a draw left [amin, amax]'
  assert bool((x == lo).any(0).all() and (x == hi).any(0).all()), 'clipping never engaged'
  assert rng_call.cpu().tolist() == [1, 0]


def test_normal_sample_moments_and_counter(cuda):
  rng = np.random.RandomState(13)
  N, A, ld = 1 << 17, 8, 11            # about 1 M draws
  loc = (rng.randn(N, ld) * 3).astype(f32)
  scale = (rng.rand(N, ld) + 0.5).astype(f32)
  tl, tsc = _dev(cuda, loc), _dev(cuda, scale)
  rng_call = torch.zeros(2, dtype=torch.int64, device=cuda)
  out = Out(cuda, N, A)
  _lib.call('b200rl_normal_sample', _lib.ptr(tl), _lib.ptr(tsc), ld, N, A, None, None, 9,
            _lib.ptr(rng_call), out.ptr(), _lib.stream())
  torch.cuda.synchronize()
  out.check_canaries('normal_sample')
  x = R.t64(out.value())
  z = (x - R.t64(loc[:, :A])) / R.t64(scale[:, :A])
  n = z.numel()
  mean, std = float(z.mean()), float(z.std())
  record_parity('grad_kernels_normal_sample', mean_sigmas=abs(mean) * math.sqrt(n),
                std_sigmas=abs(std - 1) * math.sqrt(2 * n))
  assert abs(mean) <= 5 / math.sqrt(n), mean
  assert abs(std - 1) <= 5 / math.sqrt(2 * n), std
  assert rng_call.cpu().tolist() == [1, 0]
  # one advance per call, also when the grid is not a whole number of blocks; fresh draws each call
  small_loc, small_scale = _dev(cuda, loc[:1001, :3]), _dev(cuda, scale[:1001, :3])
  o1, o2 = Out(cuda, 1001, 3), Out(cuda, 1001, 3)
  for o in (o1, o2):
    _lib.call('b200rl_normal_sample', _lib.ptr(small_loc), _lib.ptr(small_scale), 3, 1001, 3, None, None, 9,
              _lib.ptr(rng_call), o.ptr(), _lib.stream())
  torch.cuda.synchronize()
  assert rng_call.cpu().tolist() == [3, 0]
  assert not torch.equal(o1.value(), o2.value())


# ---- colsum with centre / squares (normaliser moments) -------------------------------------------
@pytest.mark.parametrize('mode', ['sum', 'centered', 'centered_squared'])
@pytest.mark.parametrize('cols', [1, 17, 64, 65])
@pytest.mark.parametrize('rows', [1, 255, 4097, 100000])
def test_colsum_moments(cuda, rows, cols, mode):
  rng = np.random.RandomState(rows + cols)
  x = (rng.randn(rows, cols) * 3 + 5).astype(f32)
  center = x.mean(0).astype(f32) + rng.randn(cols).astype(f32) * 0.01
  squared = int(mode == 'centered_squared')
  tc = _dev(cuda, center) if mode != 'sum' else None
  scale = 1.0 / rows
  tx = _dev(cuda, x)
  out = Out(cuda, 1, cols)
  ws, nb = workspace.get(cuda)
  _lib.call('b200rl_colsum', _lib.ptr(tx), _lib.ptr(tc), squared, rows, cols, scale, out.ptr(), _lib.ptr(ws), nb,
            _lib.stream())
  torch.cuda.synchronize()
  out.check_canaries('colsum')
  v = R.t64(x) - (R.t64(center) if tc is not None else 0.0)
  term = v * v if squared else v
  ref = term.sum(0) * scale
  err = _rel(R.t64(out.value()[0]) - ref, term.abs().sum(0) * scale)
  record_parity('grad_kernels_colsum', **{mode: err})
  assert err <= TOL_SUM, err


# ---- concat2, l2_sum, add_scaled -------------------------------------------------------------------
@pytest.mark.parametrize('N,da,lda,db,ldb', [(1, 1, 1, 1, 1), (257, 17, 20, 6, 6), (4099, 17, 17, 6, 9),
                                             (1000, 11, 16, 3, 7)])
def test_concat2_strided(cuda, N, da, lda, db, ldb):
  rng = np.random.RandomState(N + da + db)
  a = np.full((N, lda), np.nan, f32)
  b = np.full((N, ldb), np.nan, f32)
  a[:, :da], b[:, :db] = rng.randn(N, da), rng.randn(N, db)
  ta, tb = _dev(cuda, a), _dev(cuda, b)
  out = Out(cuda, N, da + db)
  _lib.call('b200rl_concat2', _lib.ptr(ta), lda, da, _lib.ptr(tb), ldb, db, N, out.ptr(), _lib.stream())
  torch.cuda.synchronize()
  out.check_canaries('concat2')
  want = torch.cat([ta[:, :da], tb[:, :db]], dim=1)
  assert torch.equal(out.value(), want), 'concat2 is not bit-exact'


SIZES = [1, 1023, 1025, 3136 * 512]


@pytest.mark.parametrize('n', SIZES)
def test_l2_sum_accumulates(cuda, n):
  rng = np.random.RandomState(n % 1000)
  x = (rng.randn(n) * 0.05).astype(f32)
  tx = _dev(cuda, x)
  out = Out(cuda, 1, 1)
  out.buf[0] = 0.75
  coef = 0.37
  _lib.call('b200rl_l2_sum', _lib.ptr(tx), n, coef, out.ptr(), _lib.stream())
  torch.cuda.synchronize()
  out.check_canaries('l2_sum')
  x64 = R.t64(x)
  ref = 0.75 + coef * float((x64 * x64).sum())
  err = abs(float(out.value()[0, 0]) - ref) / ref
  record_parity('grad_kernels_l2_sum', rel=err)
  assert err <= TOL_SUM, err


@pytest.mark.parametrize('n', SIZES)
def test_add_scaled(cuda, n):
  rng = np.random.RandomState(n % 997)
  dst0, src = rng.randn(n).astype(f32), rng.randn(n).astype(f32)
  alpha = 0.3
  out = Out(cuda, n, 1)
  out.buf[:n] = _dev(cuda, dst0)
  ts_ = _dev(cuda, src)
  _lib.call('b200rl_add_scaled', out.ptr(), _lib.ptr(ts_), n, alpha, _lib.stream())
  torch.cuda.synchronize()
  out.check_canaries('add_scaled')
  d64, s64 = R.t64(dst0), R.t64(src)
  err = _rel(R.t64(out.value()[:, 0]) - (d64 + alpha * s64), d64.abs() + alpha * s64.abs())
  record_parity('grad_kernels_add_scaled', rel=err)
  assert err <= TOL_AXPY, err
