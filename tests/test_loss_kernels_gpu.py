"""The policy / value loss kernels through the C ABI, against float64 (tests/loss_refs.py), below,
at and beyond their grid caps and across their lane-group boundaries.

Covers b200rl_ppo_loss and b200rl_ppo_kl (Normal head), b200rl_ppo_loss_categorical,
b200rl_ppo_kl_categorical and b200rl_categorical_logp, b200rl_reinforce_loss (both heads, all
five stages) and b200rl_cql_loss.  The launch geometry is restated here (nb per kernel, G from
A) and test_every_kernel_and_group_crosses_its_grid_cap asserts that the parametrisation runs
every (kernel, G) pair below its cap, at it with every partial populated, and at least three
grid-stride passes deep with the last warp (G = 32: the last block) only partly valid.

Every output is NaN-filled with a canary tail (and canary columns when strided); every strided
input carries NaN in its padding; every call gets a private NaN-filled workspace of exactly the
size the ABI checks, followed by a canary tail, so a final kernel that reads a partial past nb
returns NaN.  Each call is repeated and must match bit for bit (all reductions are fixed-order).
Inputs keep a relative margin of 1e-4 from every branch threshold (loss_refs.MARGIN), asserted
when they are drawn, so no row takes another branch in fp32 than in float64.
"""
import ctypes

import numpy as np
import pytest
import torch

import loss_refs as R
import target_refs as TR
import test_oracle_reinforce as host
from agents_b200 import _lib
from conftest import record_parity

pytestmark = pytest.mark.gpu
f32 = np.float32

# launch geometry (csrc/ppo.cu, reinforce.cu, cql.cu)
K_RED = 264          # kRedBlocks = 2 * kNumSMs: ppo_loss, ppo_kl
K_CAT = 512          # kCatRedBlocks: ppo_loss_categorical, ppo_kl_categorical
K_RF_STAT = 264      # kRfStatBlocks (8 trajectories per block)
K_RF_LOSS = 512      # kRfLossBlocks
K_CQL = 256          # kCqlRedBlocks


def _cdiv(a, b):
  return -(-a // b)


def geometry(rows, G, cap, per_block=256):
  """(nb, passes, last warp partly valid) of a grid-stride kernel over `rows` rows of G lanes."""
  want = _cdiv(rows * G, per_block)
  nb = min(want, cap)
  passes = _cdiv(rows * G, nb * per_block)
  rows_per_warp = max(32 // G, 1)
  partial = (rows % rows_per_warp != 0) if G < 32 else (rows * G) % per_block != 0
  return nb, passes, partial, want


COVERED = {}


def _covered(kernel, G, rows, cap, per_block=256):
  nb, passes, partial, want = geometry(rows, G, cap, per_block)
  s = COVERED.setdefault((kernel, G), set())
  if want < cap:
    s.add('below')
  if want == cap and rows * G == cap * per_block:
    s.add('at')
  if passes >= 3 and partial:
    s.add('beyond')
  return nb


def _dev(cuda, a, dtype=None):
  t = torch.as_tensor(np.ascontiguousarray(a), device=cuda)
  return t if dtype is None else t.to(dtype)


def _padded(cuda, x, ld):
  """[N, ld] device copy of x [N, A] with NaN in columns A..ld."""
  N, A = x.shape
  p = np.full((N, ld), np.nan, f32)
  p[:, :A] = x
  return _dev(cuda, p)


class Ws(object):
  """A NaN-filled workspace of exactly `nbytes` bytes followed by a canary tail."""

  def __init__(self, cuda, nbytes):
    self.n = nbytes // 4
    self.buf = torch.full((self.n + TR.TAIL,), float('nan'), device=cuda)
    self.buf[self.n:] = TR._canary(TR.TAIL).to(cuda)
    self.tail = self.buf[self.n:].clone()
    self.nbytes = nbytes

  def ptr(self):
    return self.buf.data_ptr()

  def check(self, what):
    assert torch.equal(self.buf[self.n:], self.tail), f'{what}: workspace overrun'


def _twice(run, outs):
  """Runs `run` twice; the second run's outputs must equal the first bit for bit."""
  run()
  torch.cuda.synchronize()
  first = [TR.bits(o.value()).copy() for o in outs]
  run()
  torch.cuda.synchronize()
  for o, b in zip(outs, first):
    assert np.array_equal(TR.bits(o.value()), b), 'repeated call differs'


# ---- PPO, Normal head ------------------------------------------------------------------------------
PPO_N = [1, 255, 257, 67584, 67585, 202759, 524288]


# T only scales denom; the two largest N run at T = 128 (4096 x 128 is the production batch)
PPO_CASES = [(N, A, T) for N in PPO_N for A in (1, 6, 17) for T in (1, 128) if T == 128 or N < 202759]


@pytest.mark.parametrize('N,A,T', PPO_CASES)
def test_ppo_loss_and_kl(cuda, N, A, T):
  idx = PPO_N.index(N) * 6 + [1, 6, 17].index(A) * 2 + (T == 128)
  rng = np.random.RandomState(idx)
  loc, scale, action = R.normal_params(rng, N, A)
  logp = R.normal_terms(loc, scale, action)['logp']
  logp_clip = R.logp_clip_for(logp, 0.7) if idx % 3 else 0.0
  value_clip = 0.3 if idx % 4 != 1 else 0.0
  rows = R.ppo_rows(rng, logp, 0.2, value_clip, logp_clip)
  gb = N / T if idx % 2 else 2.5 * N / T                        # the data-parallel shard case
  use_kl = idx % 2 == 0
  ld_ls, ld_g = (A + 3, A + 2) if idx % 3 != 2 else (A, A)
  kw = dict(loc=loc, scale=scale, action=action, T=T, global_batch=gb, clip_eps=0.2,
            value_clip=value_clip, vf_coef=0.5, ent_coef=0.01, logp_clip=logp_clip, **rows)
  old_loc = (loc + rng.randn(N, A) * scale * 0.3).astype(f32)
  old_scale = (scale * np.exp(rng.randn(N, A) * 0.2)).astype(f32)
  terms = np.array([0.013, 0.021, 0.7], f32)
  if use_kl:
    kw['kl'] = dict(old_loc=old_loc, old_scale=old_scale, terms=terms, grad_scale=1.0 / N)
  ref = R.ppo_loss(**kw)
  nb = _covered('ppo_loss', 1, N, K_RED)
  _covered('ppo_kl', 1, N, K_RED)

  t_loc, t_scale = _padded(cuda, loc, ld_ls), _padded(cuda, scale, ld_ls)
  t_ol, t_os = _padded(cuda, old_loc, ld_ls), _padded(cuda, old_scale, ld_ls)
  t_act = _dev(cuda, action)
  t = {k: _dev(cuda, rows[k]) for k in ('old_logp', 'adv', 'ret', 'v', 'v_old', 'w')}
  t_terms = _dev(cuda, terms)
  losses = TR.Out(cuda, 1, 6)
  dloc, dscale = TR.Out(cuda, N, A, ld_g), TR.Out(cuda, N, A, ld_g)
  dv = TR.Out(cuda, 1, N)
  flag = torch.zeros(1, dtype=torch.int32, device=cuda)
  ws = Ws(cuda, K_RED * 4 * 4)
  kl_arg = _lib.PpoKl(t_ol.data_ptr(), t_os.data_ptr(), ld_ls, t_terms.data_ptr(), 1.0 / N) if use_kl else None

  def run():
    _lib.call('b200rl_ppo_loss', t_loc.data_ptr(), t_scale.data_ptr(), ld_ls, _lib.ptr(t_act),
              _lib.ptr(t['old_logp']), _lib.ptr(t['adv']), _lib.ptr(t['ret']), _lib.ptr(t['v']),
              _lib.ptr(t['v_old']), _lib.ptr(t['w']), N, A, T, gb, 0.2, value_clip, 0.5, 0.01, logp_clip,
              losses.ptr(), dloc.ptr(), dscale.ptr(), ld_g, dv.ptr(), _lib.ptr(flag),
              ctypes.byref(kl_arg) if use_kl else None, ws.ptr(), ws.nbytes, _lib.stream())

  _twice(run, [losses, dloc, dscale, dv])
  for o, name in ((losses, 'losses'), (dloc, 'dloc'), (dscale, 'dscale'), (dv, 'dv')):
    o.check_canaries(name)
  ws.check('ppo_loss')
  assert flag.item() == 0
  got = losses.numpy()[0]
  e = {f'loss{i}': R.sum_error(got[i], ref['losses'][i], ref['c_losses'][i]) for i in (0, 1, 2, 4, 5)}
  e['dloc'] = R.elem_error(dloc.numpy(), ref['dloc'], ref['c_dloc'])
  e['dscale'] = R.elem_error(dscale.numpy(), ref['dscale'], ref['c_dscale'])
  e['dv'] = R.elem_error(dv.numpy()[0], ref['dv'], ref['c_dv'])
  # the clip fraction is an exact count over N
  assert got[3] == f32(ref['sums'][3]) / f32(N), (got[3], ref['sums'][3], N)
  assert (ref['dobj'] == 0).any() or N < 300

  # ppo_kl on the same pair, weighted and unweighted
  kl_1 = R.ppo_kl(loc, scale, old_loc, old_scale, None, 1.0 / N)
  kl_w = dict(kl=kl_1['kl'] * rows['w'], c_kl=kl_1['c_kl'] * rows['w'])
  kl_w.update(total=kl_w['kl'].sum() * R.h32(1.0 / N), c_total=kl_w['c_kl'].sum() * R.h32(1.0 / N))
  for weighted in (True, False):
    out_kl, out_sum = TR.Out(cuda, 1, N), TR.Out(cuda, 1, 1)
    ws2 = Ws(cuda, K_RED * 4)

    def run_kl():
      _lib.call('b200rl_ppo_kl', t_loc.data_ptr(), t_scale.data_ptr(), ld_ls, t_ol.data_ptr(), t_os.data_ptr(),
                ld_ls, _lib.ptr(t['w']) if weighted else None, N, A, 1.0 / N, out_kl.ptr(), out_sum.ptr(),
                ws2.ptr(), ws2.nbytes, _lib.stream())

    _twice(run_kl, [out_kl, out_sum])
    out_kl.check_canaries('ppo_kl')
    out_sum.check_canaries('ppo_kl sum')
    ws2.check('ppo_kl')
    kref = kl_w if weighted else kl_1
    e['kl_rows'] = max(e.get('kl_rows', 0.0), R.elem_error(out_kl.numpy()[0], kref['kl'], kref['c_kl']))
    e['kl_sum'] = max(e.get('kl_sum', 0.0), R.sum_error(out_sum.numpy()[0, 0], kref['total'], kref['c_total']))
  record_parity('loss_kernels_ppo_normal', **e)
  for k, v in e.items():
    assert v <= (R.TOL_SUM if k.startswith('loss') or k == 'kl_sum' else R.TOL_ELEM), (k, v, nb)


# ---- PPO, Categorical head ---------------------------------------------------------------------------
def _cat_ns(A):
  G = R.cat_group(A)
  at = K_CAT * 256 // G
  extra = {1: 17, 8: 3, 32: 5}[G]
  return [333, at, 3 * at + extra]


CAT_CASES = [(A, N) for A in (1, 2, 8, 9, 64, 65, 300) for N in _cat_ns(A)]


@pytest.mark.parametrize('A,N', CAT_CASES)
def test_ppo_loss_categorical_kl_and_logp(cuda, A, N):
  idx = CAT_CASES.index((A, N))
  rng = np.random.RandomState(100 + idx)
  G = R.cat_group(A)
  z, act = R.logits_rows(rng, N, A)
  zo = R.old_logits_like(rng, z)
  logp, c_logp = R.categorical_logp(z, act)
  logp_clip = R.logp_clip_for(logp, 0.6) if idx % 2 and A > 1 else 0.0
  value_clip = 0.3 if idx % 3 else 0.0
  rows = R.ppo_rows(rng, logp, 0.2, value_clip, logp_clip)
  T = 128 if idx % 2 else 1
  gb = N / T if idx % 4 < 2 else 3.0 * N / T
  use_kl = idx % 2 == 0
  ld, ld_g = A + 3, A + 1
  terms = np.array([0.013, 0.021, 0.7], f32)
  kw = dict(logits=z, action=act, T=T, global_batch=gb, clip_eps=0.2, value_clip=value_clip,
            vf_coef=0.5, ent_coef=0.01, logp_clip=logp_clip, **rows)
  if use_kl:
    kw['kl'] = dict(old_logits=zo, terms=terms, grad_scale=1.0 / N)
  ref = R.ppo_loss_categorical(**kw)
  _covered('ppo_loss_categorical', G, N, K_CAT)
  _covered('ppo_kl_categorical', G, N, K_CAT)

  tz, tzo = _padded(cuda, z, ld), _padded(cuda, zo, ld)
  tact = _dev(cuda, act)
  t = {k: _dev(cuda, rows[k]) for k in ('old_logp', 'adv', 'ret', 'v', 'v_old', 'w')}
  t_terms = _dev(cuda, terms)
  losses, dz, dv = TR.Out(cuda, 1, 6), TR.Out(cuda, N, A, ld_g), TR.Out(cuda, 1, N)
  flag = torch.zeros(1, dtype=torch.int32, device=cuda)
  ws = Ws(cuda, K_CAT * 4 * 4)
  kl_arg = _lib.PpoKlLogits(tzo.data_ptr(), ld, t_terms.data_ptr(), 1.0 / N) if use_kl else None

  def run():
    _lib.call('b200rl_ppo_loss_categorical', tz.data_ptr(), ld, _lib.ptr(tact), _lib.ptr(t['old_logp']),
              _lib.ptr(t['adv']), _lib.ptr(t['ret']), _lib.ptr(t['v']), _lib.ptr(t['v_old']), _lib.ptr(t['w']),
              N, A, T, gb, 0.2, value_clip, 0.5, 0.01, logp_clip, losses.ptr(), dz.ptr(), ld_g, dv.ptr(),
              _lib.ptr(flag), ctypes.byref(kl_arg) if use_kl else None, ws.ptr(), ws.nbytes, _lib.stream())

  _twice(run, [losses, dz, dv])
  for o, name in ((losses, 'losses'), (dz, 'dlogits'), (dv, 'dv')):
    o.check_canaries(name)
  ws.check('ppo_loss_categorical')
  assert flag.item() == 0
  got = losses.numpy()[0]
  e = {f'loss{i}': R.sum_error(got[i], ref['losses'][i], ref['c_losses'][i]) for i in (0, 1, 2, 4, 5)}
  assert got[3] == f32(ref['sums'][3]) / f32(N)
  e['dlogits'] = R.elem_error(dz.numpy(), ref['dlogits'], ref['c_dlogits'])
  e['dv'] = R.elem_error(dv.numpy()[0], ref['dv'], ref['c_dv'])

  out = TR.Out(cuda, 1, N)
  _twice(lambda: _lib.call('b200rl_categorical_logp', tz.data_ptr(), ld, _lib.ptr(tact), N, A, out.ptr(),
                           _lib.ptr(flag), _lib.stream()), [out])
  out.check_canaries('categorical_logp')
  e['logp'] = R.elem_error(out.numpy()[0], logp, c_logp)
  for weighted in (True, False):
    out_kl, out_sum = TR.Out(cuda, 1, N), TR.Out(cuda, 1, 1)
    ws2 = Ws(cuda, K_CAT * 4)

    def run_kl():
      _lib.call('b200rl_ppo_kl_categorical', tz.data_ptr(), ld, tzo.data_ptr(), ld,
                _lib.ptr(t['w']) if weighted else None, N, A, 1.0 / N, out_kl.ptr(), out_sum.ptr(), ws2.ptr(),
                ws2.nbytes, _lib.stream())

    _twice(run_kl, [out_kl, out_sum])
    out_kl.check_canaries('ppo_kl_categorical')
    ws2.check('ppo_kl_categorical')
    kref = R.ppo_kl_categorical(z, zo, rows['w'] if weighted else None, 1.0 / N)
    e['kl_rows'] = max(e.get('kl_rows', 0.0), R.elem_error(out_kl.numpy()[0], kref['kl'], kref['c_kl']))
    e['kl_sum'] = max(e.get('kl_sum', 0.0), R.sum_error(out_sum.numpy()[0, 0], kref['total'], kref['c_total']))
  assert flag.item() == 0
  record_parity(f'loss_kernels_ppo_categorical_G{G}', **e)
  for k, v in e.items():
    assert v <= (R.TOL_SUM if k.startswith('loss') or k == 'kl_sum' else R.TOL_ELEM), (k, v)


def test_categorical_numeric_edges_have_reference_semantics():
  """The edge rows logits_rows mixes in, in float64: masked columns get p = 0 exactly, a
  dominant row has p = 1 and H = 0 to fp32 precision, equal logits have H = log A."""
  rng = np.random.RandomState(0)
  z, act = R.logits_rows(rng, 64, 9)
  st = R.softmax_terms(z)
  kind = np.arange(64) % 8
  assert (st['p'][z == f32(R.MASKED)] == 0).all() and (z == f32(R.MASKED)).any()
  assert (np.abs(st['ent'][kind == 3]) < 1e-40).all()
  np.testing.assert_allclose(st['ent'][kind == 4], np.log(9), rtol=1e-15)
  assert (act[kind == 1] == 0).all() and (act[kind == 2] == 8).all()


# ---- REINFORCE -------------------------------------------------------------------------------------
RF_SHAPES = {1: [(1, 5), (7, 33), (2112, 3), (2113, 40), (4096, 32), (6341, 63)],
             8: [(1, 5), (7, 33), (2112, 3), (2113, 40), (4096, 4), (6341, 9)],
             32: [(1, 5), (7, 33), (2112, 3), (2113, 40), (4096, 1), (6341, 2)]}
RF_HEADS = [(False, 3), (True, 6), (True, 9), (True, 65)]
RF_CASES = [(d, A, B, T) for d, A in RF_HEADS for B, T in RF_SHAPES[1 if not d else R.cat_group(A)]]
CFG_NAMES = sorted(host.CONFIGS)


def _rf_inputs(rng, B, T, A, discrete, cfg, const_adv=None):
  N = B * T
  st, nst = R.reinforce_steps(rng, B, T)
  ret = (rng.randn(B, T) * 10.0 ** rng.uniform(-1, 1, (B, 1))).astype(f32)
  V = rng.randn(B, T).astype(f32) if cfg['baseline'] else None
  if const_adv is not None:
    ret[:] = const_adv
    if V is not None:
      V[:] = 0
  w = None
  if cfg.get('weights'):
    w = np.where(rng.rand(B, T) < 0.5, 1.0, rng.uniform(0, 2, (B, T))).astype(f32)
    w[rng.rand(B, T) < 0.05] = 0
  if discrete:
    params, action = R.logits_rows(rng, N, A)
  else:
    loc, scale, action = R.normal_params(rng, N, A)
    params = (loc, scale)
  return dict(params=params, action=action, ret=ret, value=V, step_type=st, next_step_type=nst, weights=w,
              use_advantage=cfg['use_advantage'], normalize=cfg['normalize'], entropy_coef=cfg['entropy'],
              value_coef=0.3, discrete=discrete)


def _rf_run(cuda, kw):
  ret = kw['ret']
  B, T = ret.shape
  N = B * T
  discrete = kw['discrete']
  A = (kw['params'].shape[1] if discrete else kw['params'][0].shape[1])
  ld, ld_g = A + 2, A + 1
  if discrete:
    p0, p1 = _padded(cuda, kw['params'], ld), None
    act = _dev(cuda, kw['action'])
  else:
    p0, p1 = _padded(cuda, kw['params'][0], ld), _padded(cuda, kw['params'][1], ld)
    act = _dev(cuda, kw['action'])
  V = None if kw['value'] is None else _dev(cuda, kw['value'])
  tret, tst, tnst = _dev(cuda, ret), _dev(cuda, kw['step_type']), _dev(cuda, kw['next_step_type'])
  tw = None if kw['weights'] is None else _dev(cuda, kw['weights'])
  use_adv = bool(kw['use_advantage']) and V is not None
  losses, ne = TR.Out(cuda, 1, 6), TR.Out(cuda, 1, 1)
  g0 = TR.Out(cuda, N, A, ld_g)
  g1 = None if discrete else TR.Out(cuda, N, A, ld_g)
  dv = None if V is None else TR.Out(cuda, 1, N)
  flag = torch.zeros(1, dtype=torch.int32, device=cuda)
  ws = Ws(cuda, 4 * (4096 + (B + 3) // 4 * 4 + N))

  def run():
    flag.zero_()
    _lib.call('b200rl_reinforce_loss', p0.data_ptr(), None if p1 is None else p1.data_ptr(), ld, _lib.ptr(act), A,
              _lib.ptr(tret), _lib.ptr(V), _lib.ptr(tst), _lib.ptr(tnst), _lib.ptr(tw), B, T, int(use_adv),
              int(kw['normalize']), float(kw['entropy_coef'] or 0.0), 0.3, losses.ptr(), g0.ptr(),
              None if g1 is None else g1.ptr(), ld_g, None if dv is None else dv.ptr(), ne.ptr(), _lib.ptr(flag),
              ws.ptr(), ws.nbytes, _lib.stream())

  outs = [o for o in (losses, ne, g0, g1, dv) if o is not None]
  _twice(run, outs)
  for o in outs:
    o.check_canaries('reinforce_loss')
  ws.check('reinforce_loss')
  return dict(losses=losses.numpy()[0], grads=[g.numpy() for g in (g0, g1) if g is not None],
              dv=None if dv is None else dv.numpy()[0].reshape(B, T), episodes=ne.numpy()[0, 0],
              flag=int(flag.item()))


def _rf_check(got, ref, kw, tag):
  assert got['episodes'] == ref['episodes']
  assert got['flag'] == (2 if ref['episodes'] == 0 else 0), (got['flag'], ref['episodes'])
  e = {f'loss{i}': R.sum_error(got['losses'][i], ref['losses'][i], ref['c_losses'][i]) for i in range(6)}
  for i, (g, w, c) in enumerate(zip(got['grads'], ref['grads'], ref['c_grads'])):
    e[f'grad{i}'] = R.elem_error(g, w, c)
  stage5 = kw['value'] is not None and kw['use_advantage'] and kw['normalize']
  if ref['dv'] is not None:
    e['dv_stage5' if stage5 else 'dv'] = R.elem_error(got['dv'], ref['dv'], ref['c_dv'])
  record_parity(f'loss_kernels_reinforce_{tag}', **e)
  for k, v in e.items():
    tol = R.TOL_SUM if k.startswith('loss') else (R.TOL_DV_NORM if k == 'dv_stage5' else R.TOL_ELEM)
    assert v <= tol, (k, v)


@pytest.mark.parametrize('discrete,A,B,T', RF_CASES)
def test_reinforce_loss(cuda, discrete, A, B, T):
  idx = RF_CASES.index((discrete, A, B, T))
  G = R.cat_group(A) if discrete else 1
  _covered('reinforce_stats', 32, B, K_RF_STAT)    # a warp (32 lanes) per trajectory
  _covered('reinforce_loss_' + ('cat' if discrete else 'normal'), G, B * T, K_RF_LOSS)
  for name in {'baseline_adv_norm_ent_weights', CFG_NAMES[idx % len(CFG_NAMES)]}:
    cfg = host.CONFIGS[name]
    kw = _rf_inputs(np.random.RandomState(idx * 7 + len(name)), B, T, A, discrete, cfg)
    ref = R.reinforce_loss(**kw)
    got = _rf_run(cuda, kw)
    _rf_check(got, ref, kw, ('cat' if discrete else 'normal') + f'_G{G}')


@pytest.mark.parametrize('discrete', [False, True])
@pytest.mark.parametrize('const', [0.0, 0.37])
def test_reinforce_zero_sigma(cuda, discrete, const):
  """Constant advantages (zero advantages at const = 0): σ = 0, the σ-derivative term of dV is 0."""
  for name in ('baseline_adv_norm', 'no_baseline_norm'):
    kw = _rf_inputs(np.random.RandomState(5), 40, 30, 9 if discrete else 2, discrete, host.CONFIGS[name], const)
    ref = R.reinforce_loss(**kw)
    assert ref['sigma'] == 0
    got = _rf_run(cuda, kw)
    _rf_check(got, ref, kw, 'zero_sigma')


# ---- CQL -------------------------------------------------------------------------------------------
def _cql_bs(N):
  G = R.cat_group(2 * N)
  at = K_CQL * 256 // G
  return [300, at, 3 * at + 5]


CQL_CASES = [(N, B) for N in (4, 5, 32, 33) for B in _cql_bs(N)]


@pytest.mark.parametrize('N,B', CQL_CASES)
def test_cql_loss(cuda, N, B):
  idx = CQL_CASES.index((N, B))
  rng = np.random.RandomState(200 + idx)
  G = R.cat_group(2 * N)
  _covered('cql_loss', G, B, K_CQL)
  R_ = B + 2 * B * N
  q1, q2 = (rng.randn(R_) * 4).astype(f32), (rng.randn(R_) * 4).astype(f32)
  logp = (rng.randn(B * N) * 3).astype(f32)
  td = [(rng.randn(B) * 0.1).astype(f32) for _ in range(2)]
  temp, ul, tau = 0.8, -4.1, 5.0
  lagrange, bc_debug = idx % 2 == 1, idx % 3 == 2
  clip = (-1.0, 2.0) if idx % 4 == 1 else (-1.0, 0.5)
  ref = R.cql_loss(q1, q2, logp, B, N, ul, temp, None if lagrange else 2.5, clip, tau, bc_debug, 0.75, td,
                   log_alpha=1.2 if lagrange else None)
  tq1, tq2, tlp = _dev(cuda, q1), _dev(cuda, q2), _dev(cuda, logp)
  alpha = None if lagrange else _dev(cuda, np.array([2.5], f32))
  la = _dev(cuda, np.array([1.2], f32)) if lagrange else None
  cl = _dev(cuda, np.array([0.75], f32))
  dq = [TR.Out(cuda, 1, R_), TR.Out(cuda, 1, R_)]
  out, dla = TR.Out(cuda, 1, 4), TR.Out(cuda, 1, 1)
  nan = torch.zeros(1, dtype=torch.int32, device=cuda)
  ws = Ws(cuda, K_CQL * 4)

  def run():
    for d, t in zip(dq, td):
      d.buf[:B] = _dev(cuda, t)
    _lib.call('b200rl_cql_loss', _lib.ptr(tq1), _lib.ptr(tq2), _lib.ptr(tlp), B, N, ul, temp, _lib.ptr(alpha),
              _lib.ptr(la), clip[0], clip[1], tau, int(bc_debug), _lib.ptr(cl), dq[0].ptr(), dq[1].ptr(), out.ptr(),
              dla.ptr(), _lib.ptr(nan), ws.ptr(), ws.nbytes, _lib.stream())

  _twice(run, dq + [out] + ([dla] if lagrange else []))
  for o in dq + [out]:
    o.check_canaries('cql_loss')
  ws.check('cql_loss')
  assert nan.item() == 0
  got = out.numpy()[0]
  e = {f'out{i}': R.sum_error(got[i], ref['out'][i], ref['c_out'][i]) for i in range(4)}
  for i in range(2):
    e[f'dq{i + 1}'] = R.elem_error(dq[i].numpy()[0], ref[f'dq{i + 1}'], ref[f'c_dq{i + 1}'])
  if lagrange:
    e['dlog_alpha'] = R.sum_error(dla.numpy()[0, 0], ref['dla'], ref['c_out'][3])
  record_parity(f'loss_kernels_cql_G{G}', **e)
  for k, v in e.items():
    assert v <= (R.TOL_ELEM if k.startswith('dq') else R.TOL_SUM), (k, v)


# ---- coverage ---------------------------------------------------------------------------------------
def test_every_kernel_and_group_crosses_its_grid_cap():
  """Restates the parametrisation above through `geometry` (independent of test order)."""
  COVERED.clear()
  for N in PPO_N:
    _covered('ppo_loss', 1, N, K_RED)
    _covered('ppo_kl', 1, N, K_RED)
  for A, N in CAT_CASES:
    _covered('ppo_loss_categorical', R.cat_group(A), N, K_CAT)
    _covered('ppo_kl_categorical', R.cat_group(A), N, K_CAT)
  for d, A, B, T in RF_CASES:
    _covered('reinforce_stats', 32, B, K_RF_STAT)
    _covered('reinforce_loss_' + ('cat' if d else 'normal'), R.cat_group(A) if d else 1, B * T, K_RF_LOSS)
  for N, B in CQL_CASES:
    _covered('cql_loss', R.cat_group(2 * N), B, K_CQL)
  want = {('ppo_loss', 1), ('ppo_kl', 1), ('reinforce_stats', 32), ('reinforce_loss_normal', 1)}
  want |= {(k, G) for k in ('ppo_loss_categorical', 'ppo_kl_categorical', 'reinforce_loss_cat', 'cql_loss')
           for G in (1, 8, 32)}
  assert set(COVERED) == want, set(COVERED) ^ want
  for key, s in sorted(COVERED.items()):
    assert s == {'below', 'at', 'beyond'}, (key, s)
  # every group width meets its lane boundaries: A = 8 / 9 and 64 / 65
  assert {8, 9, 64, 65} <= {A for A, _ in CAT_CASES}
