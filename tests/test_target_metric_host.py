"""The target metrics of target_refs.py, at the bounds the GPU tests use, accept the kernels' own
fp32 association orders and reject the mistakes a returns / advantages / normaliser test has to
catch.  No GPU needed.

Each mutant is the reference or the kernel-order emulation with one deliberate mistake.

Not rejected, so not listed: dropping the Kahan carry of normalizer_update.  The carry only
recovers the rounding of each m2 += value step, at most ½ulp(m2) per update, while the fp32
column sums feeding each update err by more.  Over 50 updates of 1 .. 30k rows, with and without
the carry, oracle/ppo.StreamingNormalizer's worst m2_error was the same (11.3, against TOL_M2 = 32),
so no bound that accepts the kernel can reject the mutant.
"""
import numpy as np
import pytest

import target_refs as R
from oracle import value_ops as ovo

f32 = np.float32


def _scan_inputs(seed, B, T, gamma, p_end=0.05):
  rng = np.random.RandomState(seed)
  r = (rng.randn(B, T) * 10.0 ** rng.uniform(-3, 3, (B, 1))).astype(f32)
  d = (gamma * (rng.rand(B, T) > p_end)).astype(f32)
  v = (rng.randn(B, T) * 10.0 ** rng.uniform(-2, 2, (B, 1))).astype(f32)
  fv = rng.randn(B).astype(f32)
  return r, d, v, fv


SHAPES = [(5, 1), (5, 31), (5, 32), (5, 33), (9, 127), (4, 1000)]


@pytest.mark.parametrize('B,T', SHAPES)
@pytest.mark.parametrize('gamma', [0.99, 1.0])
def test_kernel_order_and_serial_oracle_are_accepted(B, T, gamma):
  r, d, v, fv = _scan_inputs(B * 7 + T, B, T, gamma)
  ref, S = R.discounted_return(r, d, fv)
  for got in (R.discounted_return_kernel_order(r, d, fv),
              ovo.discounted_return(r, d, fv, time_major=False), ref.astype(f32)):
    assert R.scan_error(got, ref, S) <= R.TOL_SCAN
  for lam in (0.0, 0.95, 1.0):
    ref, S = R.gae(v, fv, d, r, lam)
    for got in (R.gae_kernel_order(v, fv, d, r, lam),
                ovo.generalized_advantage_estimation(v, fv, d, r, lam, time_major=False),
                ref.astype(f32)):
      assert R.scan_error(got, ref, S) <= R.TOL_SCAN


def test_kernel_order_emulation_is_not_the_serial_order():
  """The emulation is a distinct association order: it differs from the serial oracle in the
  last bits somewhere, so the bit-equality check on the GPU pins the kernel's order."""
  r, d, v, fv = _scan_inputs(1, 64, 200, 1.0)
  assert not np.array_equal(R.discounted_return_kernel_order(r, d, fv),
                            ovo.discounted_return(r, d, fv, time_major=False))


@pytest.mark.parametrize('lane,T', [(31, 65), (1, 40)])
def test_carry_from_the_wrong_lane_is_rejected(lane, T):
  r, d, _, fv = _scan_inputs(2, 8, T, 0.99, p_end=0.0)
  ref, S = R.discounted_return(r, d, fv)
  assert R.scan_error(R.scan_kernel_order(d, r, fv, carry_lane=lane), ref, S) > R.TOL_SCAN


@pytest.mark.parametrize('T', [33, 127])
def test_partial_tile_dropped_is_rejected(T):
  """Tile count T // 32 instead of ceil(T / 32): the last, partial tile is never scanned."""
  r, d, _, fv = _scan_inputs(3, 8, T, 0.99)
  ref, S = R.discounted_return(r, d, fv)
  assert R.scan_error(R.scan_kernel_order(d, r, fv, ntiles=T // 32), ref, S) > R.TOL_SCAN


def _ppo_case(seed, B, T):
  """A PPO batch whose time-limit LAST steps keep their discount (only terminations zero it)."""
  rng = np.random.RandomState(seed)
  r = rng.randn(B, T).astype(f32)
  disc = np.ones((B, T), f32)
  nst = np.ones((B, T), np.int32)
  last = rng.rand(B, T) < 0.1
  nst[last] = R.STEP_LAST
  disc[last & (rng.rand(B, T) < 0.5)] = 0
  vp = rng.randn(B, T).astype(f32)
  return r, disc, nst, vp


def _ppo_targets(r, d_eff, vp, lam):
  T = vp.shape[1]
  ret = R.discounted_return(r[:, :T - 1], d_eff[:, :T - 1], vp[:, T - 1])
  adv = R.gae(vp[:, :T - 1], vp[:, T - 2], d_eff[:, :T - 1], r[:, :T - 1], lam)
  return ret, adv


def test_last_mask_ignored_is_rejected():
  r, disc, nst, vp = _ppo_case(4, 9, 34)
  d_eff = R.ppo_discounts(disc, nst, 0.99)
  no_mask = (disc * f32(0.99)).astype(f32)
  assert not np.array_equal(R.bits(d_eff), R.bits(no_mask))
  (ret, S), _ = _ppo_targets(r, d_eff, vp, 0.95)
  bad = R.discounted_return_kernel_order(r[:, :-1], no_mask[:, :-1], vp[:, -1])
  assert R.scan_error(bad, ret, S) > R.TOL_SCAN


def test_gae_bootstrapped_from_the_last_value_is_rejected():
  """PPO's GAE takes V[:, T-2] as its final value (the reference's own quirk), not V[:, T-1]."""
  r, disc, nst, vp = _ppo_case(5, 9, 34)
  d_eff = R.ppo_discounts(disc, nst, 0.99)
  _, (adv, S) = _ppo_targets(r, d_eff, vp, 0.95)
  ok = R.gae_kernel_order(vp[:, :-1], vp[:, -2], d_eff[:, :-1], r[:, :-1], 0.95)
  assert R.scan_error(ok, adv, S) <= R.TOL_SCAN
  bad = R.gae_kernel_order(vp[:, :-1], vp[:, -1], d_eff[:, :-1], r[:, :-1], 0.95)
  assert R.scan_error(bad, adv, S) > R.TOL_SCAN


def test_lambda_applied_to_delta_is_rejected():
  r, d, v, fv = _scan_inputs(6, 8, 65, 0.99)
  ref, S = R.gae(v, fv, d, r, 0.95)
  a, delta = R.gae_terms_fp32(v, fv, d, r, 0.95)
  bad = R.scan_kernel_order(a, (delta * f32(0.95)).astype(f32), None)
  assert R.scan_error(bad, ref, S) > R.TOL_SCAN


def test_fv_stride_ignored_is_rejected():
  """PPO reads row b's final value at vp[b, T-1] (stride T); a stride of 1 reads vp[0, T-1+b]."""
  r, disc, nst, vp = _ppo_case(7, 9, 34)
  d_eff = R.ppo_discounts(disc, nst, 0.99)
  (ret, S), _ = _ppo_targets(r, d_eff, vp, 0.95)
  T = vp.shape[1]
  wrong_fv = vp.reshape(-1)[T - 1:T - 1 + vp.shape[0]]
  bad = R.discounted_return_kernel_order(r[:, :-1], d_eff[:, :-1], wrong_fv)
  assert R.scan_error(bad, ret, S) > R.TOL_SCAN


# ---- n-step --------------------------------------------------------------------------------------
@pytest.mark.parametrize('T', [2, 3, 5, 33])
def test_nstep_oracle_is_accepted(T):
  rng = np.random.RandomState(T)
  rew = rng.randn(40, T).astype(f32)
  disc = ((rng.rand(40, T) > 0.2) * 0.9).astype(f32)
  disc[20:] = 0.9                                    # rows without an episode end
  wr, S, wd = R.nstep_reduce(rew, disc, 0.97)
  gr, gd = ovo.n_step_reduce(rew, disc, 0.97)
  assert R.scan_error(gr, wr, S) <= R.TOL_SCAN
  assert R.rel_error_u(gd, wd) <= R.TOL_NSTEP_DISC * (T + 1)
  # γ^(T−1) instead of γ^(T−2)
  if T > 2:
    assert R.rel_error_u((gd * f32(0.97)).astype(f32), wd) > R.TOL_NSTEP_DISC * (T + 1)


# ---- masks and weights ---------------------------------------------------------------------------
def test_ppo_weights_zero_rule_and_signed_zeros():
  st = np.array([0, 1, 2, 1, 1, 1, 0, 2], np.int32)
  ret = np.array([0.0, -0.0, 1.0, 0.0, 2.0, -0.0, 0.0, 0.0], f32)
  adv = np.array([0.0, 0.0, 1.0, 3.0, 0.0, -0.0, -0.0, 0.0], f32)
  w = np.array([2.0, 3.0, 4.0, -0.0, 5.0, 6.0, 7.0, 8.0], f32)
  assert R.ppo_weights(st, ret, adv).tolist() == [0, 0, 0, 1, 1, 0, 0, 0]
  got = R.ppo_weights(st, ret, adv, w)
  assert got.tolist() == [0, 0, 0, 0, 5, 0, 0, 0]
  assert R.bits(got)[3] == R.bits(f32(-0.0))         # a valid -0 weight is passed through
  assert R.bits(got)[0] == 0                         # masked entries are +0
  dropped = np.where(st != R.STEP_LAST, w, f32(0)).astype(f32)    # the ret == adv == 0 rule dropped
  assert not np.array_equal(R.bits(got), R.bits(dropped))


def test_ppo_discounts_signed_zeros():
  d = np.array([-0.0, 0.0, 1.0, -0.0, 0.5], f32)
  nst = np.array([1, 1, 2, 2, 0], np.int32)
  got = R.ppo_discounts(d, nst, 0.99)
  assert R.bits(got).tolist() == R.bits(np.array([-0.0, 0.0, 0.0, -0.0, f32(0.5) * f32(0.99)], f32)).tolist()


# ---- KL beta -------------------------------------------------------------------------------------
def test_beta_update_uses_strict_comparisons():
  target, tol = 0.01, 0.3
  hi = f32(f32(target) * f32(f32(1) + f32(tol)))
  lo = f32(f32(target) * f32(f32(1) - f32(tol)))
  assert R.kl_beta_update(hi, 1.0, target, tol) == f32(1.0)
  assert R.kl_beta_update(np.nextafter(hi, f32(1)), 1.0, target, tol) == f32(1.5)
  assert R.kl_beta_update(lo, 1.0, target, tol) == f32(1.0)
  assert R.kl_beta_update(np.nextafter(lo, f32(0)), 1.0, target, tol) == f32(f32(1) / f32(1.5))
  # the mutant with >= / <= fires at m == hi / m == lo, where the kernel leaves beta alone
  def mutant(m, beta):
    f = f32(f32(1) / f32(1.5)) if m <= lo else (f32(1.5) if m >= hi else f32(1))
    return f32(min(max(f32(f32(beta) * f), f32(10e-16)), f32(10e16)))
  for m in (lo, hi):
    assert mutant(m, 1.0) != R.kl_beta_update(m, 1.0, target, tol)
  for m in (np.nextafter(lo, f32(0)), np.nextafter(hi, f32(1)), f32(target)):
    assert mutant(m, 1.0) == R.kl_beta_update(m, 1.0, target, tol)
  assert R.kl_beta_update(1.0, 10e16, target, tol) == f32(10e16)
  assert R.kl_beta_update(0.0, 10e-16, target, tol) == f32(10e-16)


# ---- moments and normalize -----------------------------------------------------------------------
def test_normalize_rounded_reference_is_accepted_and_eps_outside_sqrt_rejected():
  rng = np.random.RandomState(8)
  x = (rng.randn(500, 17) * 3 + 1e3 * rng.uniform(-1, 1, 17)).astype(f32)
  mu, m2, _ = R.column_moments(x)
  cnt = np.full(17, 500.0, f32)
  mu32, m232 = mu.astype(f32), m2.astype(f32)
  for clip in (0.0, 5.0):
    ref, M = R.normalize(x, mu32, m232, cnt, 1e-3, clip)
    assert R.normalize_error(ref.astype(f32), ref, M) <= R.TOL_NORMALIZE
  ref, M = R.normalize(x, mu32, m232, cnt, 1e-3, 0.0)
  var = m232.astype(np.float64) / cnt
  bad = ((x - mu32.astype(np.float64)) / (np.sqrt(var) + R.h32(1e-3))).astype(f32)
  assert R.normalize_error(bad, ref, M) > R.TOL_NORMALIZE


def test_bessel_corrected_variance_is_rejected():
  """_train normalises advantages by the population variance m2/N (tf.nn.moments)."""
  rng = np.random.RandomState(9)
  adv = (rng.randn(1000, 1) * 2 + 0.5).astype(f32)
  mu, m2, absmean = R.column_moments(adv)
  ref, M = R.normalize(adv, mu, m2 / 1000, None, 1e-8, 0.0)
  assert R.normalize_error(ref.astype(f32), ref, M) <= R.TOL_NORMALIZE
  bad, _ = R.normalize(adv, mu, m2 / 999, None, 1e-8, 0.0)
  assert R.normalize_error(bad.astype(f32), ref, M) > R.TOL_NORMALIZE
  # and as a second moment: m2·N/(N−1) is outside the m2 bound
  assert R.m2_error(m2 * 1000 / 999, m2, R.moments_slack(1000, absmean)) > R.TOL_M2


def test_chan_merge_matches_one_pass_over_the_concatenation():
  rng = np.random.RandomState(10)
  parts = [(rng.randn(n, 3) * (1 + i) + 5 * i).astype(f32) for i, n in enumerate((1, 7, 300, 2))]
  m = R.ChanMerge(3)
  for p in parts:
    m.update(p)
  mu, m2, absmean = R.column_moments(np.concatenate(parts))
  np.testing.assert_allclose(m.avg, mu, rtol=1e-12)
  np.testing.assert_allclose(m.m2, m2, rtol=1e-9)    # the 1e-10 initial count
  np.testing.assert_allclose(m.count, 310 + 1e-10, rtol=1e-15)
  np.testing.assert_allclose(m.absmean, absmean, rtol=1e-12)


def test_fp32_streaming_oracle_is_accepted_and_wrong_count_init_rejected():
  """oracle/ppo.StreamingNormalizer (fp32, the kernel's formulas) stays inside the bounds over
  many merges; a merge that starts the count at 0 instead of 1e-10 gives the same state, but
  one that starts it at 1 does not."""
  from oracle import ppo as oppo
  rng = np.random.RandomState(11)
  o, m = oppo.StreamingNormalizer((5,)), R.ChanMerge(5)
  bad = oppo.StreamingNormalizer((5,))
  bad.count[:] = 1.0
  worst_bad = 0.0
  for k in range(30):
    x = (rng.randn(int(10 ** rng.uniform(0, 3.5)), 5) * (1 + 0.1 * k) + 0.3 * k).astype(f32)
    o.update(x)
    bad.update(x)
    m.update(x)
    assert R.mean_error(o.avg, m.avg, m.absmean) <= R.TOL_MEAN
    assert R.m2_error(o.m2, m.m2, m.slack) <= R.TOL_M2
    assert R.rel_error_u(o.count, m.count) <= R.TOL_COUNT
    worst_bad = max(worst_bad, R.mean_error(bad.avg, m.avg, m.absmean))
  assert worst_bad > R.TOL_MEAN
