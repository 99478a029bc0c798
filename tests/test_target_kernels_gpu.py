"""The training-target kernels through the C ABI, against float64 (tests/target_refs.py).

Covers b200rl_discounted_return / _gae in both layouts, their batch-major _ld variants (PPO's
strided call), b200rl_nstep_reduce, b200rl_ppo_discounts / _ppo_weights (bit for bit),
b200rl_normalize, b200rl_normalizer_update through StreamingTensorNormalizer, and
b200rl_ppo_kl_beta_update (bit for bit).

Every output is NaN-filled before the call and carries a canary tail; strided outputs also carry
canary columns.  Both must come back untouched.  Strided inputs carry NaN in their padding, and
final values are read through a pointer into a NaN-filled array, so a read of anything else
shows.  Each comparison records its measured error with record_parity; the bounds in
target_refs.py are at least 4x the largest value measured on an H100 80GB HBM3 at a 700 W power
limit.
"""
import numpy as np
import pytest
import torch

import target_refs as R
from agents_b200 import _lib
from agents_b200.specs import tensor_spec
from agents_b200.utils import tensor_normalizer
from conftest import record_parity
from oracle import value_ops as ovo

pytestmark = pytest.mark.gpu
f32 = np.float32


def _dev(cuda, a):
  """A device copy of `a`.  Keep it in a variable for as long as a launch may read it: a
  temporary passed as _lib.ptr(_dev(...)) is freed before the call, and its block is handed to
  the next allocation."""
  return torch.as_tensor(np.ascontiguousarray(a), device=cuda)


def _scan_inputs(seed, B, T):
  """Rewards and values with per-row scales spanning 1e-3 .. 1e3 (a per-element metric must not
  let a large row hide a small one); discounts 0.99 on even rows and 1 on odd ones, with random
  episode ends except on rows b % 4 == 3, zeros at lanes 0 and 31 of every tile on rows b % 3 == 1, and at t = T-1 on rows
  b % 3 == 2."""
  rng = np.random.RandomState(seed)
  r = (rng.randn(B, T) * 10.0 ** rng.uniform(-3, 3, (B, 1))).astype(f32)
  v = (rng.randn(B, T) * 10.0 ** rng.uniform(-2, 2, (B, 1))).astype(f32)
  fv = (rng.randn(B) * 3).astype(f32)
  gamma = np.where(np.arange(B) % 2 == 0, 0.99, 1.0)[:, None]
  d = (gamma * (rng.rand(B, T) > 0.03)).astype(f32)
  d[3::4] = gamma[3::4]                             # whole-length episodes (γ = 1 on odd rows)
  t = np.arange(T)
  d[1::3][:, (t % 32 == 0) | (t % 32 == 31)] = 0
  d[2::3, T - 1] = 0
  return r, d, v, fv


def _nan_padded(cuda, x, ld):
  """[B, ld] device copy of x [B, T] with NaN in columns T..ld."""
  B, T = x.shape
  p = np.full((B, ld), np.nan, f32)
  p[:, :T] = x
  return _dev(cuda, p)


def _final_in(cuda, fv, stride, offset=5):
  """(holder, pointer) with fv[b] at holder[offset + b*stride] and NaN everywhere else."""
  B = fv.shape[0]
  h = torch.full((offset + B * stride + 8,), float('nan'), device=cuda)
  h[offset:offset + B * stride:stride] = _dev(cuda, fv)
  return h, h.data_ptr() + 4 * offset


# ---- discounted return / GAE, both layouts ---------------------------------------------------------
BS = [1, 7, 8, 9, 129, 4097]
TS = [1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 1000]


@pytest.mark.parametrize('T', TS)
@pytest.mark.parametrize('B', BS)
def test_scans_both_layouts(cuda, B, T):
  r, d, v, fv = _scan_inputs(B * 1009 + T, B, T)
  st = _lib.stream()
  worst = {}

  def check(name, out, ref, S, exact, time_major=False):
    out.check_canaries(name)
    got = out.numpy().T if time_major else out.numpy()
    err = R.scan_error(got, ref, S)
    worst[name] = max(worst.get(name, 0.0), err)
    assert err <= R.TOL_SCAN, (name, err)
    if exact is not None:
      assert np.array_equal(R.bits(got), R.bits(exact)), f'{name}: not the kernel order bit for bit'

  for tm in (False, True):
    lay = 'time_major' if tm else 'batch_major'
    io = (lambda x: x.T.copy()) if tm else (lambda x: x)
    shape = (T, B) if tm else (B, T)
    tr, td, tv, tfv = _dev(cuda, io(r)), _dev(cuda, io(d)), _dev(cuda, io(v)), _dev(cuda, fv)
    for final in (None, fv):
      ref, S = R.discounted_return(r, d, final)
      out = R.Out(cuda, *shape)
      _lib.call('b200rl_discounted_return', _lib.ptr(tr), _lib.ptr(td),
                None if final is None else _lib.ptr(tfv), out.ptr(), B, T, int(tm), 1, st)
      exact = (io(ovo.discounted_return(io(r), io(d), final, time_major=True)) if tm
               else R.discounted_return_kernel_order(r, d, final))
      check(f'return_{lay}', out, ref, S, exact, tm)
      # provide_all = 0: one return per trajectory, out[b]
      one = R.Out(cuda, 1, B)
      _lib.call('b200rl_discounted_return', _lib.ptr(tr), _lib.ptr(td),
                None if final is None else _lib.ptr(tfv), one.ptr(), B, T, int(tm), 0, st)
      check(f'return0_{lay}', one, ref[:, :1].T, S[:, :1].T, exact[:, :1].T)
    for lam in (0.0, 0.95, 1.0):
      ref, S = R.gae(v, fv, d, r, lam)
      out = R.Out(cuda, *shape)
      _lib.call('b200rl_gae', _lib.ptr(tv), _lib.ptr(tfv), _lib.ptr(td), _lib.ptr(tr), lam,
                out.ptr(), B, T, int(tm), st)
      exact = (io(ovo.generalized_advantage_estimation(io(v), fv, io(d), io(r), lam, True)) if tm
               else R.gae_kernel_order(v, fv, d, r, lam))
      check(f'gae_{lay}', out, ref, S, exact, tm)
  record_parity('target_kernels_scans', **worst)


def test_scans_empty_batch(cuda):
  x = torch.zeros(4, device=cuda)
  for tm in (0, 1):
    out = R.Out(cuda, 1, 0)
    _lib.call('b200rl_discounted_return', _lib.ptr(x), _lib.ptr(x), _lib.ptr(x), out.ptr(), 0, 4, tm, 1,
              _lib.stream())
    _lib.call('b200rl_gae', _lib.ptr(x), _lib.ptr(x), _lib.ptr(x), _lib.ptr(x), 0.95, out.ptr(), 0, 4, tm,
              _lib.stream())
    out.check_canaries('B = 0')


# ---- the strided batch-major variants -------------------------------------------------------------
@pytest.mark.parametrize('B,T', [(1, 1), (9, 2), (7, 31), (8, 33), (129, 64), (9, 65), (33, 127), (5, 1000)])
def test_ld_variants(cuda, B, T):
  r, d, v, fv = _scan_inputs(B * 31 + T, B, T)
  ld_in = T + 5
  tr, td, tv = (_nan_padded(cuda, x, ld_in) for x in (r, d, v))
  st = _lib.stream()
  worst = {}
  for ld_out in (T, T + 3):
    for fv_stride in (1, ld_in):
      hold, fvp = _final_in(cuda, fv, fv_stride)
      ref, S = R.discounted_return(r, d, fv)
      out = R.Out(cuda, B, T, ld_out)
      _lib.call('b200rl_discounted_return_ld', _lib.ptr(tr), _lib.ptr(td), fvp, out.ptr(), B, T, ld_in,
                ld_out, fv_stride, st)
      out.check_canaries('discounted_return_ld')
      got = out.numpy()
      worst['return_ld'] = max(worst.get('return_ld', 0.0), R.scan_error(got, ref, S))
      assert R.scan_error(got, ref, S) <= R.TOL_SCAN
      assert np.array_equal(R.bits(got), R.bits(R.discounted_return_kernel_order(r, d, fv)))
      for lam in (0.0, 0.95, 1.0):
        ref, S = R.gae(v, fv, d, r, lam)
        out = R.Out(cuda, B, T, ld_out)
        _lib.call('b200rl_gae_ld', _lib.ptr(tv), fvp, _lib.ptr(td), _lib.ptr(tr), lam, out.ptr(), B, T,
                  ld_in, ld_out, fv_stride, st)
        out.check_canaries('gae_ld')
        got = out.numpy()
        worst['gae_ld'] = max(worst.get('gae_ld', 0.0), R.scan_error(got, ref, S))
        assert R.scan_error(got, ref, S) <= R.TOL_SCAN
        assert np.array_equal(R.bits(got), R.bits(R.gae_kernel_order(v, fv, d, r, lam)))
      del hold
  record_parity('target_kernels_scans_ld', **worst)


@pytest.mark.parametrize('B,T', [(1, 2), (9, 34), (5, 33), (64, 129), (4096, 128)])
def test_ppo_call(cuda, B, T):
  """PPOAgent._preprocess's exact calls: a scan of length T-1 over [B, T] rows, returns
  bootstrapped from vp + (T-1) and GAE from vp + (T-2), both with stride T; column T-1 of the
  outputs is never written."""
  r, d, vp, _ = _scan_inputs(B + 7 * T, B, T)
  tr, td, tvp = _dev(cuda, r), _dev(cuda, d), _dev(cuda, vp)
  st = _lib.stream()
  ret = R.Out(cuda, B, T - 1, T)
  adv = R.Out(cuda, B, T - 1, T)
  _lib.call('b200rl_discounted_return_ld', _lib.ptr(tr), _lib.ptr(td), tvp.data_ptr() + 4 * (T - 1),
            ret.ptr(), B, T - 1, T, T, T, st)
  _lib.call('b200rl_gae_ld', _lib.ptr(tvp), tvp.data_ptr() + 4 * (T - 2), _lib.ptr(td), _lib.ptr(tr), 0.95,
            adv.ptr(), B, T - 1, T, T, T, st)
  ret.check_canaries('ppo returns')
  adv.check_canaries('ppo advantages')
  h = T - 1
  wret, Sr = R.discounted_return(r[:, :h], d[:, :h], vp[:, T - 1])
  wadv, Sa = R.gae(vp[:, :h], vp[:, T - 2], d[:, :h], r[:, :h], 0.95)
  er, ea = R.scan_error(ret.numpy(), wret, Sr), R.scan_error(adv.numpy(), wadv, Sa)
  record_parity('target_kernels_ppo_call', returns=er, advantages=ea)
  assert er <= R.TOL_SCAN and ea <= R.TOL_SCAN
  assert np.array_equal(R.bits(ret.numpy()), R.bits(R.discounted_return_kernel_order(r[:, :h], d[:, :h],
                                                                                      vp[:, T - 1])))
  assert np.array_equal(R.bits(adv.numpy()), R.bits(R.gae_kernel_order(vp[:, :h], vp[:, T - 2], d[:, :h],
                                                                       r[:, :h], 0.95)))


# ---- n-step --------------------------------------------------------------------------------------
@pytest.mark.parametrize('T', [2, 3, 5, 33])
def test_nstep_reduce(cuda, T):
  rng = np.random.RandomState(T)
  B = 300
  rew = (rng.randn(B, T) * 10.0 ** rng.uniform(-2, 2, (B, 1))).astype(f32)
  disc = ((rng.rand(B, T) > 0.2) * 0.9).astype(f32)
  disc[::2] = 0.95                                  # rows without an episode end
  gamma = 0.97
  outr, outd = R.Out(cuda, 1, B), R.Out(cuda, 1, B)
  trew, tdisc = _dev(cuda, rew), _dev(cuda, disc)
  _lib.call('b200rl_nstep_reduce', _lib.ptr(trew), _lib.ptr(tdisc), gamma, outr.ptr(), outd.ptr(), B, T,
            _lib.stream())
  outr.check_canaries('nstep reward')
  outd.check_canaries('nstep discount')
  wr, S, wd = R.nstep_reduce(rew, disc, gamma)
  er = R.scan_error(outr.numpy()[0], wr, S)
  ed = R.rel_error_u(outd.numpy()[0], wd) / (T + 1)
  record_parity('target_kernels_nstep', reward=er, discount_per_factor=ed)
  assert er <= R.TOL_SCAN and ed <= R.TOL_NSTEP_DISC
  assert (outd.numpy()[0][1::2][(disc[1::2, :T - 1] == 0).any(axis=1)] == 0).all()


# ---- PPO / REINFORCE masks and weights, bit for bit --------------------------------------------------
@pytest.mark.parametrize('n', [1, 255, 256, 257, 524288])
def test_ppo_discounts_and_weights(cuda, n):
  rng = np.random.RandomState(n % 1000)
  special = np.array([0.0, -0.0, 1.0, 0.5], f32)
  disc = np.where(rng.rand(n) < 0.5, special[rng.randint(0, 4, n)], rng.rand(n)).astype(f32)
  nst = rng.randint(0, 3, n).astype(np.int32)
  st = rng.randint(0, 3, n).astype(np.int32)
  ret = np.where(rng.rand(n) < 0.3, special[rng.randint(0, 2, n)], rng.randn(n)).astype(f32)
  adv = np.where(rng.rand(n) < 0.3, special[rng.randint(0, 2, n)], rng.randn(n)).astype(f32)
  w = np.where(rng.rand(n) < 0.2, special[rng.randint(0, 2, n)], rng.rand(n) * 3).astype(f32)
  s = _lib.stream()
  tdisc, tnst, tst, tret, tadv, tw = (_dev(cuda, a) for a in (disc, nst, st, ret, adv, w))
  for gamma in (0.99, 1.0):
    out = R.Out(cuda, 1, n)
    _lib.call('b200rl_ppo_discounts', _lib.ptr(tdisc), _lib.ptr(tnst), gamma, n, out.ptr(), s)
    out.check_canaries('ppo_discounts')
    assert np.array_equal(R.bits(out.numpy()[0]), R.bits(R.ppo_discounts(disc, nst, gamma)))
  for weights, tweights in ((None, None), (w, tw)):
    out = R.Out(cuda, 1, n)
    _lib.call('b200rl_ppo_weights', _lib.ptr(tst), _lib.ptr(tret), _lib.ptr(tadv), _lib.ptr(tweights), n,
              out.ptr(), s)
    out.check_canaries('ppo_weights')
    assert np.array_equal(R.bits(out.numpy()[0]), R.bits(R.ppo_weights(st, ret, adv, weights)))


# ---- normalize -----------------------------------------------------------------------------------
@pytest.mark.parametrize('rows,cols', [(1, 1), (7, 17), (129, 65), (1000, 3), (4097, 1)])
def test_normalize(cuda, rows, cols):
  rng = np.random.RandomState(rows * 7 + cols)
  mu = (1e3 * rng.uniform(-1, 1, cols) * (rng.rand(cols) < 0.7)).astype(f32)
  sd = (10.0 ** rng.uniform(-2, 1, cols)).astype(f32)
  x = (mu + sd * rng.randn(rows, cols) * 3).astype(f32)
  cnt = (rng.uniform(1, 1e5, cols)).astype(f32)
  var = (sd.astype(np.float64) ** 2 * rng.uniform(0.5, 2, cols))
  m2_cnt = (var * cnt).astype(f32)
  var32 = var.astype(f32)
  tx, tmu, tm2_cnt, tcnt, tvar = (_dev(cuda, a) for a in (x, mu, m2_cnt, cnt, var32))
  worst = 0.0
  for centred in (True, False):
    for with_count in (True, False):
      m2, count = (m2_cnt, cnt) if with_count else (var32, None)
      tm2, tcount = (tm2_cnt, tcnt) if with_count else (tvar, None)
      for clip in (0.0, 5.0):
        for eps in (1e-3, 1e-8):
          out = R.Out(cuda, rows, cols)
          _lib.call('b200rl_normalize', _lib.ptr(tx), out.ptr(), rows, cols, _lib.ptr(tmu) if centred else None,
                    _lib.ptr(tm2), _lib.ptr(tcount), eps, clip, _lib.stream())
          out.check_canaries('normalize')
          ref, M = R.normalize(x, mu if centred else None, m2, count, eps, clip)
          err = R.normalize_error(out.numpy(), ref, M)
          worst = max(worst, err)
          assert err <= R.TOL_NORMALIZE, (centred, with_count, clip, eps, err)
          if clip > 0:
            assert np.abs(out.numpy()).max() <= clip
  record_parity('target_kernels_normalize', err=worst)


# ---- the streaming normaliser --------------------------------------------------------------------
def _schedule(max_rows, n=50):
  """n batch sizes, log-spaced from 1 row to max_rows, shuffled so big and small ones alternate."""
  rows = np.unique(np.round(np.logspace(0, np.log10(max_rows), n)).astype(int))
  rows = np.concatenate([rows, np.full(n - rows.size, 3)])
  return np.random.RandomState(max_rows).permutation(rows)


@pytest.mark.parametrize('cols,max_rows,mean0,std0,drift', [
    (1, 524288, 0.0, 1.0, 0.02), (17, 524288, 5.0, 2.0, 0.02), (64, 65536, -3.0, 0.5, 0.02),
    (65, 65536, 1.0, 10.0, 0.02), (17, 65536, 1e4, 1e-2, 1e-7)])
def test_streaming_normalizer(cuda, cols, max_rows, mean0, std0, drift):
  """About 50 updates of 1 .. max_rows rows whose mean and scale drift by `drift` per update
  (columns 64 and 65 straddle b200rl_colsum's block caps); count / avg / m2 against the float64
  merge after every update."""
  rng = np.random.RandomState(cols)
  spec = tensor_spec.TensorSpec((cols,), torch.float32)
  n = tensor_normalizer.StreamingTensorNormalizer(spec, device=cuda)
  ref = R.ChanMerge(cols)
  col_mean = mean0 + rng.uniform(-1, 1, cols) * max(abs(mean0), 1.0) * 0.1
  col_std = std0 * 10.0 ** rng.uniform(-0.5, 0.5, cols)
  worst = dict(count=0.0, mean=0.0, m2=0.0, normalize=0.0)
  for k, rows in enumerate(_schedule(max_rows)):
    g = 1.0 + drift * k
    x = (col_mean * g + col_std * g * rng.randn(rows, cols)).astype(f32)
    n.update(_dev(cuda, x))
    ref.update(x)
    cnt, avg, m2, _ = n.variables
    e = dict(count=R.rel_error_u(cnt, ref.count), mean=R.mean_error(avg, ref.avg, ref.absmean),
             m2=R.m2_error(m2, ref.m2, ref.slack))
    for key, v in e.items():
      worst[key] = max(worst[key], v)
    assert e['count'] <= R.TOL_COUNT and e['mean'] <= R.TOL_MEAN and e['m2'] <= R.TOL_M2, (k, rows, e)
    if k % 10 == 9:
      # normalize from the kernel's own state, against float64 on that state
      y = x[:min(rows, 4096)]
      got = n.normalize(_dev(cuda, y), clip_value=5.0).cpu().numpy()
      want, M = R.normalize(y, avg, m2, cnt, 1e-3, 5.0)
      worst['normalize'] = max(worst['normalize'], R.normalize_error(got, want, M))
      assert R.normalize_error(got, want, M) <= R.TOL_NORMALIZE
  record_parity(f'target_kernels_streaming_normalizer_cols{cols}', **worst)


# ---- adaptive KL beta, bit for bit -------------------------------------------------------------------
def test_kl_beta_update(cuda):
  probes = []
  for target, tol in ((0.01, 0.3), (10.0, 0.5), (0.3, 0.0), (1e-3, 0.25)):
    t32, tl32 = f32(target), f32(tol)
    lo, hi = f32(t32 * f32(f32(1) - tl32)), f32(t32 * f32(f32(1) + tl32))
    ms = [lo, np.nextafter(lo, f32(-1)), np.nextafter(lo, f32(1)), hi, np.nextafter(hi, f32(-1)),
          np.nextafter(hi, f32(1)), f32(0), f32(1e30)]
    for m in ms:
      for beta in (1.0, 10e-16, 1.5e-15, 10e16, 7e16, 0.37):
        probes.append((m, beta, target, tol))
  n = len(probes)
  mk = _dev(cuda, np.array([p[0] for p in probes], f32))
  beta = _dev(cuda, np.array([p[1] for p in probes], f32))
  for i, (_, _, target, tol) in enumerate(probes):
    _lib.call('b200rl_ppo_kl_beta_update', mk.data_ptr() + 4 * i, beta.data_ptr() + 4 * i, target, tol,
              _lib.stream())
  want = np.array([R.kl_beta_update(*p) for p in probes], f32)
  got = beta.cpu().numpy()
  bad = np.nonzero(R.bits(got) != R.bits(want))[0]
  assert bad.size == 0, [(probes[i], got[i], want[i]) for i in bad[:5]]
  assert n > 100
