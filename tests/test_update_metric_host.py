"""The update metrics of update_refs.py, at the bounds the GPU tests use, reject the mistakes an
optimizer, clip or target-update test has to catch, and accept the float64 reference rounded to
fp32.  No GPU needed.

Each mutant below is the reference with one deliberate mistake, computed in float64 and rounded
to fp32 the way a kernel would store it.  A mutant is rejected when its updated parameters, any
of its slots, its clipped gradient / scale or its blended target falls outside the bound.
"""
import numpy as np
import pytest

import update_refs as U

f32 = np.float32
N = 4099
SCALE = 0.37


def _state(seed, n=N, warm=True):
  rng = np.random.RandomState(seed)
  p = rng.randn(n).astype(f32)
  g = U.gradients(rng, n)
  if not warm:
    return rng, p, g, np.zeros(n, f32), np.zeros(n, f32)
  m = (U.gradients(rng, n) * 0.3).astype(f32)
  v = (m.astype(np.float64) ** 2 * (1 + rng.rand(n))).astype(f32)
  return rng, p, g, m, v


def _adam_ok(got, ref, pre_p):
  """(accepted, details) of an fp32 Adam result `got` = dict(p, m, v) against the reference."""
  _, ratio = U.update_error(got['p'], pre_p, ref['u'], ref['cond'])
  slots = [max(U.slot_errors(got[k], ref[k])) for k in ('m', 'v')]
  return ratio <= 1.0 and all(e <= U.TOL_SLOT for e in slots), (ratio, slots)


def _rms_ok(got, ref, pre_p, centered):
  _, ratio = U.update_error(got['p'], pre_p, ref['u'], ref['cond'])
  _, mom_ratio = U.cond_error(got['mom'], ref['mom'], ref['cond'])
  slots = [max(U.slot_errors(got[k], ref[k])) for k in (('ms', 'mg') if centered else ('ms',))]
  ok = ratio <= 1.0 and mom_ratio <= 1.0 and all(e <= U.TOL_SLOT for e in slots)
  return ok, (ratio, mom_ratio, slots)


def _fp32(d):
  return {k: (v.astype(f32) if isinstance(v, np.ndarray) else v) for k, v in d.items()}


# ---- Adam -----------------------------------------------------------------------------------------
ADAM = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8)


@pytest.mark.parametrize('step', [0, 1, 4, 10 ** 6])
@pytest.mark.parametrize('scale', [None, SCALE])
def test_adam_reference_rounded_to_fp32_is_accepted(step, scale):
  _, p, g, m, v = _state(1, warm=step > 0)
  ref = U.adam(p, g, m, v, step, scale=scale, **ADAM)
  ok, info = _adam_ok(_fp32(ref), ref, p)
  assert ok, info


def _adam_mutant(kind, p, g, m, v, step, scale):
  lr, b1, b2, eps = (U.h32(ADAM[k]) for k in ('lr', 'beta1', 'beta2', 'eps'))
  g = g.astype(np.float64)
  gm = gv = g * U.h32(scale)
  if kind == 'scale_m_only':
    gv = g
  elif kind == 'scale_twice':
    gm = gv = g * U.h32(scale) ** 2
  t = step + 1
  lr_t = lr if kind == 'no_bias_correction' else lr * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
  m = m + (gm - m) * (1 - b1)
  v = v + (gv * gv - v) * (1 - b2)
  return _fp32(dict(p=p - m * lr_t / (np.sqrt(v) + eps), m=m, v=v))


@pytest.mark.parametrize('kind,step', [('no_bias_correction', 0), ('no_bias_correction', 4),
                                       ('scale_m_only', 0), ('scale_m_only', 4),
                                       ('scale_twice', 0), ('scale_twice', 4)])
def test_adam_mutants_are_rejected(kind, step):
  _, p, g, m, v = _state(2, warm=step > 0)
  ref = U.adam(p, g, m, v, step, scale=SCALE, **ADAM)
  ok, info = _adam_ok(_adam_mutant(kind, p, g, m, v, step, SCALE), ref, p)
  assert not ok, info


def test_scale_twice_is_invisible_in_the_parameters_after_one_step():
  """Why the slots are compared: Adam's first update is ≈ lr·sign(g) whatever g's scale."""
  _, p, g, m, v = _state(3, warm=False)
  ref = U.adam(p, g, m, v, 0, scale=SCALE, **ADAM)
  bad = _adam_mutant('scale_twice', p, g, m, v, 0, SCALE)
  assert U.update_error(bad['p'], p, ref['u'], ref['cond'])[1] < 1e3
  assert max(U.slot_errors(bad['v'], ref['v'])) > 100 * U.TOL_SLOT


# ---- RMSProp --------------------------------------------------------------------------------------
RMS = {
    'tf1_bench': (dict(lr=2.5e-4, decay=0.95, momentum=0.0, eps=1e-5, centered=True), 1.0),
    'keras_mnih15': (dict(lr=2.5e-4, decay=0.95, momentum=0.95, eps=0.01, centered=True), 0.0),
    'plain_momentum': (dict(lr=1e-3, decay=0.9, momentum=0.9, eps=1e-7, centered=False), 0.0),
}


def _rms_state(seed, ms_init, steps=3):
  """A state after `steps` reference steps from the optimizer's initial slots."""
  rng = np.random.RandomState(seed)
  p = rng.randn(N).astype(f32)
  ms, mg, mom = np.full(N, ms_init, f32), np.zeros(N, f32), np.zeros(N, f32)
  return rng, p, ms, mg, mom


@pytest.mark.parametrize('cfg', sorted(RMS))
def test_rmsprop_reference_rounded_to_fp32_is_accepted(cfg):
  kw, ms_init = RMS[cfg]
  rng, p, ms, mg, mom = _rms_state(4, ms_init)
  for _ in range(4):
    g = U.gradients(rng, N)
    ref = U.rmsprop(p, g, ms, mg, mom, scale=SCALE, **kw)
    got = _fp32(ref)
    ok, info = _rms_ok(got, ref, p, kw['centered'])
    assert ok, info
    p, ms, mom = got['p'], got['ms'], got['mom']
    mg = got['mg'] if kw['centered'] else mg


def _rms_mutant(kind, p, g, ms, mg, mom, lr, decay, momentum, eps, centered):
  lr, rho, mu, eps = (U.h32(x) for x in (lr, decay, momentum, eps))
  g = g.astype(np.float64) * U.h32(SCALE)
  ms = ms + (g * g - ms) * (1 - rho)
  var = ms
  if centered:
    mg = mg + (g - mg) * (1 - rho)
    var = ms - mg * mg
  step = lr * g / (np.sqrt(var) + eps) if kind == 'eps_outside_sqrt' else lr * g / np.sqrt(var + eps)
  mom = step if kind == 'no_momentum' else mom * mu + step
  return _fp32(dict(p=p - mom, ms=ms, mg=mg, mom=mom))


@pytest.mark.parametrize('kind,cfg', [('eps_outside_sqrt', 'keras_mnih15'),
                                      ('eps_outside_sqrt', 'plain_momentum'),
                                      ('no_momentum', 'keras_mnih15'),
                                      ('no_momentum', 'plain_momentum')])
def test_rmsprop_mutants_are_rejected(kind, cfg):
  kw, ms_init = RMS[cfg]
  rng, p, ms, mg, mom = _rms_state(5, ms_init)
  for _ in range(3):                       # warm up the slots (momentum must be non-zero)
    r = _fp32(U.rmsprop(p, U.gradients(rng, N), ms, mg, mom, scale=SCALE, **kw))
    p, ms, mom = r['p'], r['ms'], r['mom']
    mg = r['mg'] if kw['centered'] else mg
  g = U.gradients(rng, N)
  ref = U.rmsprop(p, g, ms, mg, mom, scale=SCALE, **kw)
  ok, info = _rms_ok(_rms_mutant(kind, p, g, ms, mg, mom, **kw), ref, p, kw['centered'])
  assert not ok, info


@pytest.mark.parametrize('cfg,wrong_init', [('keras_mnih15', 1.0), ('tf1_bench', 0.0)])
def test_rmsprop_wrong_ms_init_is_rejected(cfg, wrong_init):
  kw, ms_init = RMS[cfg]
  rng = np.random.RandomState(6)
  p, g = rng.randn(N).astype(f32), U.gradients(rng, N)
  z = np.zeros(N, f32)
  ref = U.rmsprop(p, g, np.full(N, ms_init, f32), z, z, **kw)
  bad = _fp32(U.rmsprop(p, g, np.full(N, wrong_init, f32), z, z, **kw))
  ok, info = _rms_ok(bad, ref, p, kw['centered'])
  assert not ok, info


def test_centered_bound_follows_kappa():
  """Near-constant gradients drive ms − mg² towards ε; the bound widens with κ, and a flat 1e-3
  error is still rejected where κ is small."""
  kw, _ = RMS['tf1_bench']
  rng = np.random.RandomState(7)
  g = (1.0 + 1e-3 * rng.randn(N)).astype(f32)
  mg = g.copy()
  ms = (g.astype(np.float64) ** 2 * (1 + 1e-4)).astype(f32)
  p, mom = rng.randn(N).astype(f32), np.zeros(N, f32)
  ref = U.rmsprop(p, g, ms, mg, mom, **kw)
  assert ref['cond'].max() > 1e3
  ok, info = _rms_ok(_fp32(ref), ref, p, True)
  assert ok, info
  _, p2, ms2, mg2, mom2 = _rms_state(8, 1.0)
  g2 = U.gradients(rng, N)
  ref2 = U.rmsprop(p2, g2, ms2, mg2, mom2, **kw)
  assert ref2['cond'].max() < 10
  bad = _fp32(dict(ref2, p=p2 - ref2['u'] * (1 + 1e-3)))
  assert U.update_error(bad['p'], p2, ref2['u'], ref2['cond'])[1] > 1.0


# ---- clipping -------------------------------------------------------------------------------------
def test_clip_uses_norm_not_squared_norm():
  rng = np.random.RandomState(9)
  offs = [0, 1024, 1024, 2049, 2052, 6000]
  g = (rng.randn(offs[-1]) * 0.2).astype(f32)
  g[2049:2052] = 0                              # padding
  clip = 1.5
  ref, norms = U.clip_by_norm_segments(g, offs, clip)
  assert (norms[[0, 2, 4]] > clip).all() and norms[3] == 0
  assert max(U.slot_errors(ref.astype(f32), ref)) <= U.TOL_CLIP
  bad = g.astype(np.float64).copy()
  for b, e, nrm in zip(offs[:-1], offs[1:], norms):
    bad[b:e] *= clip / max(nrm * nrm, clip)
  assert max(U.slot_errors(bad.astype(f32), ref)) > U.TOL_CLIP
  scale, nrm = U.global_norm_scale(g, 3.0)
  assert nrm > 3.0
  assert U.rel_error(f32(scale), scale) <= U.TOL_CLIP
  assert U.rel_error(f32(3.0 / max(nrm * nrm, 3.0)), scale) > U.TOL_CLIP
  assert U.global_norm_scale(g, 0.0)[0] == 1.0 and U.global_norm_scale(g, 1e4)[0] == 1.0


# ---- target updates -------------------------------------------------------------------------------
@pytest.mark.parametrize('tau', [0.005, 0.5 + 2 ** -10])
def test_polyak_tau_swapped_is_rejected(tau):
  rng = np.random.RandomState(10)
  t, s = rng.randn(N).astype(f32), rng.randn(N).astype(f32)
  ref = U.polyak(t, s, tau)
  assert U.polyak_error(ref.astype(f32), t, s, ref) <= U.TOL_POLYAK
  bad = (U.h32(tau) * t + (1 - U.h32(tau)) * s.astype(np.float64)).astype(f32)
  assert U.polyak_error(bad, t, s, ref) > U.TOL_POLYAK


@pytest.mark.parametrize('period', [2, 5])
def test_periodically_firing_early_is_rejected(period):
  rng = np.random.RandomState(11)
  s = rng.randn(N).astype(f32)
  gate = U.Periodically(period)
  tgt_ref = tgt_bad = rng.randn(N).astype(f32)
  fired, worst = [], 0.0
  for c in range(1, 2 * period + 1):
    new_ref, f = U.polyak_step(gate, tgt_ref, s, 0.5)
    fired.append(f)
    early = c % period == period - 1                  # the mutant fires one call early
    new_bad = U.polyak(tgt_bad, s, 0.5).astype(f32) if early else tgt_bad
    worst = max(worst, U.polyak_error(new_bad, tgt_ref, s, new_ref))
    tgt_ref, tgt_bad = new_ref.astype(f32), new_bad
  assert fired == [c % period == 0 for c in range(1, 2 * period + 1)]
  assert gate.counter == 2 * period
  assert worst > U.TOL_POLYAK


def test_periodically_counts_calls_that_do_nothing():
  """tau = 0 makes the body a no-op, but the counter still advances on every call."""
  gate = U.Periodically(3)
  t = np.arange(5, dtype=f32)
  for _ in range(4):
    out, _ = U.polyak_step(gate, t, t + 1, 0.0)
    assert (out == t).all()
  assert gate.counter == 4
  one = U.Periodically(1)
  assert all(one() for _ in range(3)) and one.counter == 0
  assert not U.Periodically(None)()
