"""The loss metrics of loss_refs.py, at the bounds the GPU tests use, accept the kernels' own fp32
association orders and the rounded float64 reference, and reject the mistakes a loss test must
catch.  The float64 references' analytic gradients are checked against float64 autograd.  No GPU.

Each mutant is the fp32 kernel-order restatement with one deliberate mistake (loss_refs
*_fp32(mutant=...)).  All listed mutants are rejected, two of them only on inputs built for it:
- `>=` in the clip-fraction test differs from `>` only on a ratio exactly at 1 ± eps, so it is
  shown on such rows.  The GPU inputs keep a 1e-4 margin from the clip range (so fp32 and float64
  agree on every branch), so there the count is checked exactly but a tie is never drawn.
- A Bessel-corrected σ moves the normalised advantages by a relative 1/(2N): ≈ 35 000 u at the
  N = 240 used here, but only ≈ 20 u at N = 400 000, inside TOL_ELEM, so large GPU batches alone
  would not catch it.
"""
import math

import numpy as np
import pytest
import torch

import loss_refs as R

f32 = np.float32


def _ppo_normal_case(seed, N, A, T=4, gb=None, clip_eps=0.2, value_clip=0.3, logp_clip=0.0, kl=False):
  rng = np.random.RandomState(seed)
  loc, scale, action = R.normal_params(rng, N, A)
  logp = R.normal_terms(loc, scale, action)['logp']
  if logp_clip == 'auto':
    logp_clip = R.logp_clip_for(logp, 0.7)
  rows = R.ppo_rows(rng, logp, clip_eps, value_clip, logp_clip)
  kw = dict(loc=loc, scale=scale, action=action, T=T, global_batch=gb or N / T, clip_eps=clip_eps,
            value_clip=value_clip, vf_coef=0.5, ent_coef=0.01, logp_clip=logp_clip, **rows)
  if kl:
    kw['kl'] = dict(old_loc=(loc + rng.randn(N, A) * scale * 0.3).astype(f32),
                    old_scale=(scale * np.exp(rng.randn(N, A) * 0.2)).astype(f32),
                    terms=[0.013, 0.021, 0.7], grad_scale=1.0 / N)
  return kw


def _ppo_cat_case(seed, N, A, T=4, clip_eps=0.2, value_clip=0.3, logp_clip=0.0, kl=False):
  rng = np.random.RandomState(seed)
  z, act = R.logits_rows(rng, N, A)
  logp, _ = R.categorical_logp(z, act)
  if logp_clip == 'auto':
    logp_clip = R.logp_clip_for(logp, 0.6)
  rows = R.ppo_rows(rng, logp, clip_eps, value_clip, logp_clip)
  kw = dict(logits=z, action=act, T=T, global_batch=N / T, clip_eps=clip_eps, value_clip=value_clip,
            vf_coef=0.5, ent_coef=0.01, logp_clip=logp_clip, **rows)
  if kl:
    kw['kl'] = dict(old_logits=R.old_logits_like(rng, z), terms=[0.013, 0.021, 0.7], grad_scale=1.0 / N)
  return kw


def _ppo_errors(ref, got, grads):
  e = {'loss%d' % i: R.sum_error(got['losses'][i], ref['losses'][i], ref['c_losses'][i])
       for i in (0, 1, 2, 4, 5)}
  e['clip_fraction_exact'] = 0.0 if f32(got['losses'][3]) == f32(ref['losses'][3]) else math.inf
  for g in grads:
    e[g] = R.elem_error(got[g], ref[g], ref['c_' + g])
  e['dv'] = R.elem_error(got['dv'], ref['dv'], ref['c_dv'])
  return e


def _bounded(e):
  return all(v <= (R.TOL_SUM if k.startswith('loss') else R.TOL_ELEM) for k, v in e.items())


NORMAL_CASES = [(300, 1, 0.0, False), (257, 6, 'auto', True), (70000, 3, 'auto', False), (203000, 2, 0.0, True)]


@pytest.mark.parametrize('N,A,logp_clip,kl', NORMAL_CASES)
def test_ppo_normal_kernel_order_and_rounded_reference_are_accepted(N, A, logp_clip, kl):
  kw = _ppo_normal_case(N + A, N, A, logp_clip=logp_clip, kl=kl)
  ref = R.ppo_loss(**kw)
  emu = R.ppo_loss_fp32(**kw)
  e = _ppo_errors(ref, emu, ('dloc', 'dscale'))
  assert _bounded(e), e
  rounded = dict(losses=ref['losses'].astype(f32), dloc=ref['dloc'].astype(f32),
                 dscale=ref['dscale'].astype(f32), dv=ref['dv'].astype(f32))
  assert _bounded(_ppo_errors(ref, rounded, ('dloc', 'dscale')))


CAT_CASES = [(300, 2, 0.0, True), (333, 9, 'auto', False), (200, 65, 0.0, True), (150, 300, 'auto', True),
             (140000, 8, 0.0, False)]


@pytest.mark.parametrize('N,A,logp_clip,kl', CAT_CASES)
def test_ppo_categorical_kernel_order_and_rounded_reference_are_accepted(N, A, logp_clip, kl):
  kw = _ppo_cat_case(N + A, N, A, logp_clip=logp_clip, kl=kl)
  ref = R.ppo_loss_categorical(**kw)
  emu = R.ppo_loss_categorical_fp32(**kw)
  e = _ppo_errors(ref, emu, ('dlogits',))
  e['logp'] = R.elem_error(emu['logp'], ref['logp'], ref['c_logp'])
  assert _bounded(e), e
  rounded = dict(losses=ref['losses'].astype(f32), dlogits=ref['dlogits'].astype(f32), dv=ref['dv'].astype(f32))
  assert _bounded(_ppo_errors(ref, rounded, ('dlogits',)))


# ---- mutants -------------------------------------------------------------------------------------
def _rejected(ref, got, grads):
  return not _bounded(_ppo_errors(ref, got, grads))


@pytest.mark.parametrize('mutant', ['second_pass_dropped', 'last_partial_block_dropped',
                                    'unclipped_gradient_outside_clip', 'logp_clip_derivative_kept',
                                    'value_clip_min', 'kl_scale_grad_without_so2', 'denom_N'])
def test_ppo_normal_mutants_are_rejected(mutant):
  """On 70 000 rows (two grid-stride passes, 264 partials, the last block partly filled)."""
  kw = _ppo_normal_case(5, 70000, 3, gb=52000.0, logp_clip='auto', kl=True)
  ref = R.ppo_loss(**kw)
  assert not _rejected(ref, R.ppo_loss_fp32(**kw), ('dloc', 'dscale'))
  assert _rejected(ref, R.ppo_loss_fp32(**kw, mutant=mutant), ('dloc', 'dscale'))


@pytest.mark.parametrize('A', [9, 63, 65, 300])
@pytest.mark.parametrize('mutant', ['last_strided_column_dropped', 'entropy_grad_without_ent', 'second_pass_dropped'])
def test_ppo_categorical_mutants_are_rejected(A, mutant):
  """G = 8 and 32 rows, the last strided column on lane 0 (A = 9, 65), G − 1 (A = 63) and 11
  (A = 300); 40 000 rows take more than one pass for G = 8 and 32."""
  kw = _ppo_cat_case(A, 40000 if mutant == 'second_pass_dropped' else 500, A, logp_clip='auto', kl=True)
  ref = R.ppo_loss_categorical(**kw)
  assert not _rejected(ref, R.ppo_loss_categorical_fp32(**kw), ('dlogits',))
  assert _rejected(ref, R.ppo_loss_categorical_fp32(**kw, mutant=mutant), ('dlogits',))


def tie_old_logps(lp, eps=0.25, span=400):
  """fp32 old_logp values for a row of clipped log-prob lp (exactly ±logp_clip) whose fp32 ratio
  exp(lp − old) is exactly 1 + eps and 1 − eps while the float64 ratio lies just inside the clip
  range (correctly rounded; the GPU test reads the kernel's own ratios back instead)."""
  out = []
  for r in (1 + eps, 1 - eps):
    x = f32(f32(lp) - f32(math.log(r)))
    for k in range(-span, span + 1):
      old = f32(x + f32(k) * np.spacing(x))
      d = f32(f32(lp) - old)
      if abs(float(R.exp32(d)) - 1) == eps and abs(math.exp(lp - float(old)) - 1) < eps:
        out.append(old)
        break
  return out


def test_clip_fraction_ge_is_rejected_on_a_tie():
  """Rows whose fp32 ratio is exactly 1 ± eps while the float64 ratio lies just inside the clip
  range: neither the reference nor the kernel counts them, `>=` does, and the clip fraction is
  compared exactly.  The rows' logp is clipped to −0.125, so lp − old is exact in fp32."""
  kw = _ppo_normal_case(6, 64, 2, clip_eps=0.25, logp_clip=0.125)
  rows = tie_old_logps(-0.125)
  assert len(rows) == 2, rows
  for i, old in enumerate(rows):
    kw['loc'][i], kw['scale'][i], kw['action'][i] = 0, 1, 0
    kw['old_logp'][i] = old
  ref = R.ppo_loss(**kw)
  got, bad = R.ppo_loss_fp32(**kw), R.ppo_loss_fp32(**kw, mutant='clip_count_ge')
  assert f32(got['losses'][3]) == f32(ref['losses'][3])
  assert f32(bad['losses'][3]) != f32(ref['losses'][3])


# ---- REINFORCE -----------------------------------------------------------------------------------
def reinforce_case(seed, B, T, A, discrete, cfg, const_adv=None):
  rng = np.random.RandomState(seed)
  st, nst = R.reinforce_steps(rng, B, T)
  N = B * T
  ret = (rng.randn(B, T) * 10.0 ** rng.uniform(-1, 1, (B, 1))).astype(f32)
  V = rng.randn(B, T).astype(f32) if cfg['baseline'] else None
  if const_adv is not None:
    ret[:] = const_adv
    if V is not None:
      V[:] = 0
  w = np.where(rng.rand(B, T) < 0.5, 1.0, rng.uniform(0, 2, (B, T))).astype(f32) if cfg.get('weights') else None
  if discrete:
    params, action = R.logits_rows(rng, N, A)
  else:
    loc, scale, action = R.normal_params(rng, N, A)
    params = (loc, scale)
  return dict(params=params, action=action, ret=ret, value=V, step_type=st, next_step_type=nst,
              weights=w, use_advantage=cfg['use_advantage'], normalize=cfg['normalize'],
              entropy_coef=cfg['entropy'], value_coef=0.3, discrete=discrete)


def reinforce_errors(ref, got):
  e = {'loss%d' % i: R.sum_error(got['losses'][i], ref['losses'][i], ref['c_losses'][i]) for i in range(6)}
  for i, (g, w, c) in enumerate(zip(got['grads'], ref['grads'], ref['c_grads'])):
    e['grad%d' % i] = R.elem_error(g, w, c)
  if ref['dv'] is not None:
    e['dv'] = R.elem_error(got['dv'], ref['dv'], ref['c_dv'])
  return e


def reinforce_bounded(e):
  tol = lambda k: R.TOL_SUM if k.startswith('loss') else (R.TOL_DV_NORM if k == 'dv' else R.TOL_ELEM)
  return all(v <= tol(k) for k, v in e.items())


import test_oracle_reinforce as host   # noqa: E402  (CONFIGS, make_case, autograd_grads)


@pytest.mark.parametrize('discrete,A', [(False, 3), (True, 6), (True, 65)])
@pytest.mark.parametrize('name', sorted(host.CONFIGS))
def test_reinforce_kernel_order_and_rounded_reference_are_accepted(discrete, A, name):
  cfg = host.CONFIGS[name]
  kw = reinforce_case(A, 40, 37, A, discrete, cfg)
  ref = R.reinforce_loss(**kw)
  assert reinforce_bounded(reinforce_errors(ref, R.reinforce_loss_fp32(**kw))), reinforce_errors(
      ref, R.reinforce_loss_fp32(**kw))
  rounded = dict(losses=ref['losses'].astype(f32), grads=[g.astype(f32) for g in ref['grads']],
                 dv=None if ref['dv'] is None else ref['dv'].astype(f32))
  assert reinforce_bounded(reinforce_errors(ref, rounded))


def test_reinforce_large_batch_is_accepted():
  """2113 trajectories (past the stats cap) and 4 loss-stage passes."""
  cfg = host.CONFIGS['baseline_adv_norm_ent_weights']
  kw = reinforce_case(1, 2113, 190, 2, False, cfg)
  ref = R.reinforce_loss(**kw)
  e = reinforce_errors(ref, R.reinforce_loss_fp32(**kw))
  assert reinforce_bounded(e), e


@pytest.mark.parametrize('mutant', ['bessel_sigma', 'stage5_dv_omitted'])
def test_reinforce_mutants_are_rejected(mutant):
  cfg = host.CONFIGS['baseline_adv_norm']
  kw = reinforce_case(2, 8, 30, 3, False, cfg)
  ref = R.reinforce_loss(**kw)
  assert reinforce_bounded(reinforce_errors(ref, R.reinforce_loss_fp32(**kw)))
  assert not reinforce_bounded(reinforce_errors(ref, R.reinforce_loss_fp32(**kw, mutant=mutant)))


@pytest.mark.parametrize('const', [0.0, 0.37])
def test_reinforce_zero_sigma(const):
  """Constant advantages: σ = 0, D = eps, the σ-derivative term of dV is 0."""
  cfg = host.CONFIGS['baseline_adv_norm']
  kw = reinforce_case(3, 6, 20, 2, False, cfg, const_adv=const)
  ref = R.reinforce_loss(**kw)
  assert ref['sigma'] == 0 and ref['k6'] == 0
  e = reinforce_errors(ref, R.reinforce_loss_fp32(**kw))
  assert reinforce_bounded(e), e


@pytest.mark.parametrize('discrete', [False, True])
@pytest.mark.parametrize('name', sorted(host.CONFIGS))
def test_reinforce_reference_matches_float64_autograd(discrete, name):
  cfg = host.CONFIGS[name]
  rng = np.random.default_rng(7)
  case = host.make_case(rng, 3, 9, 4 if discrete else 2, discrete, cfg)
  cfg = dict(cfg, entropy=cfg['entropy'] and R.h32(cfg['entropy']))   # coefficients as fp32 values
  total, want_params, want_dv = host.autograd_grads(case, cfg, discrete, value_coef=R.h32(0.3))
  ref = R.reinforce_loss(case['params'], case['action'], case['ret'], case['V'], case['st'], case['nst'],
                         case['w'], cfg['use_advantage'], cfg['normalize'], cfg['entropy'], 0.3, discrete)
  np.testing.assert_allclose(ref['losses'][5], total, rtol=1e-12, atol=1e-14)
  for got, want in zip(ref['grads'], want_params):
    np.testing.assert_allclose(got, want, rtol=1e-10, atol=1e-13)
  if want_dv is not None:
    np.testing.assert_allclose(ref['dv'], want_dv, rtol=1e-10, atol=1e-13)


# ---- PPO and CQL references against float64 autograd ----------------------------------------------
def _t(a, grad=False):
  return torch.tensor(np.asarray(a, np.float64), requires_grad=grad)


def _ppo_autograd(kw, logp_fn, params, ent_fn, kl_fn):
  old, adv, ret, v, vo, w = (_t(kw[k]) for k in ('old_logp', 'adv', 'ret', 'v', 'v_old', 'w'))
  V = _t(kw['v'], True)
  den = float(f32(kw['T']) * f32(kw['global_batch']))
  eps, vcl, L = R.h32(kw['clip_eps']), R.h32(kw['value_clip']), R.h32(kw['logp_clip'])
  logp = logp_fn()
  lp = torch.clamp(logp, -L, L) if L > 0 else logp
  ratio = torch.exp(lp - old)
  pg = -torch.minimum(ratio * adv, torch.clamp(ratio, 1 - eps, 1 + eps) * adv)
  err = (ret - V) ** 2
  if vcl > 0:
    vc = vo + torch.clamp(V - vo, -vcl, vcl)
    err = torch.maximum(err, (ret - vc) ** 2)
  total = ((pg * w).sum() + R.h32(kw['vf_coef']) * (err * w).sum() -
           R.h32(kw['ent_coef']) * (ent_fn() * w).sum()) / den
  if 'kl' in kw:
    total = total + R.h32(kw['kl']['terms'][2]) * R.h32(kw['kl']['grad_scale']) * (kl_fn() * w).sum()
  return torch.autograd.grad(total, params + [V])


@pytest.mark.parametrize('logp_clip,kl', [(0.0, False), ('auto', True)])
def test_ppo_normal_reference_matches_float64_autograd(logp_clip, kl):
  kw = _ppo_normal_case(11, 40, 3, logp_clip=logp_clip, kl=kl)
  loc, scale = _t(kw['loc'], True), _t(kw['scale'], True)
  a = _t(kw['action'])
  c = 0.5 * R.LOG2PI
  logp = lambda: (-0.5 * ((a - loc) / scale) ** 2 - torch.log(scale) - c).sum(1)
  ent = lambda: (0.5 + c + torch.log(scale)).sum(1)

  def kl_fn():
    mo, so = _t(kw['kl']['old_loc']), _t(kw['kl']['old_scale'])
    d = torch.log(so) - torch.log(scale)
    z = (mo - loc) / scale
    return (0.5 * z * z + 0.5 * torch.expm1(2 * d) - d).sum(1)

  gl, gs, gv = _ppo_autograd(kw, logp, [loc, scale], ent, kl_fn)
  ref = R.ppo_loss(**kw)
  assert (ref['dobj'] == 0).any() and (ref['dobj'] != 0).any()
  np.testing.assert_allclose(ref['dloc'], gl.numpy(), rtol=1e-9, atol=1e-14)
  np.testing.assert_allclose(ref['dscale'], gs.numpy(), rtol=1e-9, atol=1e-14)
  np.testing.assert_allclose(ref['dv'], gv.numpy(), rtol=1e-9, atol=1e-14)


@pytest.mark.parametrize('A,logp_clip,kl', [(5, 0.0, True), (12, 'auto', False), (70, 0.0, True)])
def test_ppo_categorical_reference_matches_float64_autograd(A, logp_clip, kl):
  kw = _ppo_cat_case(A, 48, A, logp_clip=logp_clip, kl=kl)
  z = _t(kw['logits'], True)
  act = torch.tensor(kw['action'].astype(np.int64))
  lsm = lambda: torch.log_softmax(z, 1)
  logp = lambda: lsm().gather(1, act[:, None])[:, 0]
  ent = lambda: -(torch.softmax(z, 1) * torch.where(torch.softmax(z, 1) > 0, lsm(), torch.zeros(()))).sum(1)

  def kl_fn():
    lq = torch.log_softmax(_t(kw['kl']['old_logits']), 1)
    q = lq.exp()
    return (q * torch.where(q > 0, lq - lsm(), torch.zeros(()))).sum(1)

  gz, gv = _ppo_autograd(kw, logp, [z], ent, kl_fn)
  ref = R.ppo_loss_categorical(**kw)
  np.testing.assert_allclose(ref['dlogits'], gz.numpy(), rtol=1e-9, atol=1e-14)
  np.testing.assert_allclose(ref['dv'], gv.numpy(), rtol=1e-9, atol=1e-14)


@pytest.mark.parametrize('N', [4, 33])
@pytest.mark.parametrize('lagrange', [False, True])
def test_cql_reference_matches_float64_autograd_and_kernel_order(N, lagrange):
  rng = np.random.RandomState(N)
  B, temp = 50, 0.8
  R_ = B + 2 * B * N
  q1, q2 = (rng.randn(R_) * 4).astype(f32), (rng.randn(R_) * 4).astype(f32)
  logp = (rng.randn(B * N) * 3).astype(f32)
  td = [(rng.randn(B) * .1).astype(f32) for _ in range(2)]
  ul = -3.2
  kw = dict(log_alpha=1.2, clip=(-1.0, 2.0)) if lagrange else dict(alpha=2.5, clip=(0, 0))
  ref = R.cql_loss(q1, q2, logp, B, N, ul, temp, kw.get('alpha'), kw['clip'], 5.0, False, 0.75, td,
                   log_alpha=kw.get('log_alpha'))
  Q1, Q2 = _t(q1, True), _t(q2, True)
  lp = _t(logp).reshape(B, N)
  terms = []
  for Q in (Q1, Q2):
    x = torch.cat([Q[B:B + B * N].reshape(B, N) * R.h32(temp) - lp,
                   Q[B + B * N:].reshape(B, N) * R.h32(temp) - R.h32(ul)], 1)
    terms.append(torch.logsumexp(x, 1) / R.h32(temp) - Q[:B])
  cql = (terms[0] + terms[1]).mean() / 2
  a = ref['out'][1]
  g1, g2 = torch.autograd.grad(a * cql, (Q1, Q2))
  np.testing.assert_allclose(ref['out'][0], cql.item(), rtol=1e-12)
  np.testing.assert_allclose(ref['dq1'], g1.numpy() + np.r_[td[0], np.zeros(2 * B * N)], rtol=1e-10, atol=1e-15)
  np.testing.assert_allclose(ref['dq2'], g2.numpy() + np.r_[td[1], np.zeros(2 * B * N)], rtol=1e-10, atol=1e-15)
  if not lagrange:
    emu = R.cql_loss_fp32(q1, q2, logp, B, N, ul, temp, 2.5, 5.0, False, 0.75, td)
    for i in range(3):
      assert R.sum_error(emu['out'][i], ref['out'][i], ref['c_out'][i]) <= R.TOL_SUM
    for k in ('dq1', 'dq2'):
      assert R.elem_error(emu[k], ref[k], ref['c_' + k]) <= R.TOL_ELEM
    # the last partial block dropped from the final sum
    assert R.sum_error(ref['out'][0] * (1 - 1.0 / B), ref['out'][0], ref['c_out'][0]) > R.TOL_SUM


def test_categorical_kl_and_logp_kernel_order_are_accepted():
  rng = np.random.RandomState(3)
  for A in (2, 9, 65, 300):
    z, act = R.logits_rows(rng, 400, A)
    zo = R.old_logits_like(rng, z)
    w = rng.uniform(0, 2, 400).astype(f32)
    ref = R.ppo_kl_categorical(z, zo, w, 1.0 / 400)
    G = R.cat_group(A)
    m, s, _ = R.group_stats(z, G)
    mo, so, _ = R.group_stats(zo, G)
    ls, lso = np.log(s).astype(f32), np.log(so).astype(f32)
    lq = ((zo - mo[:, None]).astype(f32) - lso[:, None]).astype(f32)
    q = np.exp(lq).astype(f32)
    lpn = ((z - m[:, None]).astype(f32) - ls[:, None]).astype(f32)
    with np.errstate(invalid='ignore', over='ignore'):
      terms = np.where(q > 0, (q * (lq - lpn).astype(f32)).astype(f32), f32(0))
    kl = (terms.sum(axis=1, dtype=f32) * w).astype(f32)
    assert R.elem_error(kl, ref['kl'], ref['c_kl']) <= R.TOL_ELEM
    lp, clp = R.categorical_logp(z, act)
    assert R.elem_error(lp.astype(f32), lp, clp) <= R.TOL_ELEM
    # the last column dropped from the stats
    m2, s2, _ = R.group_stats(z, G, drop_last_col=True)
    bad = ((z[np.arange(400), act] - m2).astype(f32) - np.log(s2).astype(f32)).astype(f32)
    assert R.elem_error(bad, lp, clp) > R.TOL_ELEM
