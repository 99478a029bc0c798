"""The update kernels of csrc/optim.cu through the C ABI, against the float64 restatements in
update_refs.py: Adam, RMSProp (plain / centered, float4 and scalar paths), per-segment and global
clip-by-norm, the Periodically-gated Polyak update and the step counters.

Every step is checked against the reference stepped from the state the device held before the
launch, so rounding cannot accumulate across steps.  Sizes run from 1 element to the Mnih'15
Q-network's flat buffer (~1.69 M floats), which takes the grid-stride loop's second pass (the
grid holds 132 × 8 blocks of 256 threads).  Every array a kernel writes carries a canary tail
that must come back untouched.  Bounds are in update_refs.py; record_parity keeps the largest
measured error of each family.
"""
import functools

import numpy as np
import pytest
import torch

import update_refs as U
from agents_b200 import _lib
from agents_b200.networks import layers as L
from agents_b200.networks import q_network
from agents_b200.specs import tensor_spec
from agents_b200.utils import workspace
from conftest import record_parity

pytestmark = pytest.mark.gpu
f32 = np.float32
CANARY = 16
CANARY_VALUE = -777.25
SCALES = [None, 0.37, 1.0, 0.0]
SIZES = [1, 3, 4, 4097, 270337, 'mnih']


@functools.lru_cache(maxsize=None)
def _mnih_net():
  obs_spec = tensor_spec.TensorSpec((84, 84, 4), torch.uint8)
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 5)
  net = q_network.QNetwork(obs_spec, act_spec, preprocessing_layers=L.CastScale(255.),
                           conv_layer_params=((32, 8, 4), (64, 4, 2), (64, 3, 1)),
                           fc_layer_params=(512,), device='cuda').set_seed(0)
  net.create_variables()
  return net


def _size(n):
  return _mnih_net().flat_params.numel() if n == 'mnih' else n


class Buf(object):
  """A device fp32 array at element `offset` of a buffer padded with canaries on both sides."""

  def __init__(self, a, offset=0):
    a = np.asarray(a, f32)
    self.n, self.offset = a.size, offset
    self.full = torch.full((offset + a.size + CANARY,), CANARY_VALUE, dtype=torch.float32,
                           device='cuda')
    self.t = self.full[offset:offset + a.size]
    self.t.copy_(torch.as_tensor(a))

  def np(self):
    return self.t.cpu().numpy()

  def check_canary(self, what):
    c = torch.cat([self.full[:self.offset], self.full[self.offset + self.n:]])
    assert bool((c == CANARY_VALUE).all()), f'{what}: canary overwritten'


def _scale_dev(scale):
  return None if scale is None else torch.tensor([scale, CANARY_VALUE], dtype=torch.float32,
                                                 device='cuda')


def _counter(value):
  return torch.tensor([value, 0, 12345], dtype=torch.int64, device='cuda')


# ---- Adam -----------------------------------------------------------------------------------------
ADAM = {'tf1': dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8),   # tf.compat.v1.train.AdamOptimizer
        'keras': dict(lr=3e-4, beta1=0.9, beta2=0.999, eps=1e-7)}  # tf.keras.optimizers.Adam


def _adam_launch(p, g, m, v, step, scale_dev, kw):
  _lib.call('b200rl_adam_tf', _lib.ptr(p.t), _lib.ptr(g), _lib.ptr(m.t), _lib.ptr(v.t), p.n,
            kw['lr'], kw['beta1'], kw['beta2'], kw['eps'], _lib.ptr(step), _lib.ptr(scale_dev),
            _lib.stream())


@pytest.mark.parametrize('start', ['fresh', 'warm'])
@pytest.mark.parametrize('cfg', sorted(ADAM))
@pytest.mark.parametrize('n', SIZES)
def test_adam_kernel(cuda, n, cfg, start):
  """fresh: p = m = v = 0 and step 0, five steps (the first measures u with no p to round
  against).  warm: random p and slots, step preset to 10⁶ (β^t = 0), two steps."""
  n = _size(n)
  kw = ADAM[cfg]
  rng = np.random.RandomState(n % 1000 + (cfg == 'keras') + 7 * (start == 'warm'))
  for scale in SCALES:
    if start == 'fresh':
      p0, m0, v0, t0, steps = np.zeros(n, f32), np.zeros(n, f32), np.zeros(n, f32), 0, 5
    else:
      p0 = rng.randn(n).astype(f32)
      m0 = (U.gradients(rng, n) * 0.3).astype(f32)
      v0 = (m0.astype(np.float64) ** 2 * (1 + rng.rand(n))).astype(f32)
      t0, steps = 10 ** 6, 2
    p, m, v = Buf(p0), Buf(m0), Buf(v0)
    step, sdev = _counter(t0), _scale_dev(scale)
    for k in range(steps):
      g = torch.as_tensor(U.gradients(rng, n), device=cuda)
      pre = dict(p=p.np(), m=m.np(), v=v.np(), step=int(step[0]))
      _adam_launch(p, g, m, v, step, sdev, kw)
      ref = U.adam(pre['p'], g.cpu().numpy(), pre['m'], pre['v'], pre['step'], scale=scale, **kw)
      raw, ratio = U.update_error(p.np(), pre['p'], ref['u'], ref['cond'])
      em, ev = U.slot_errors(m.np(), ref['m']), U.slot_errors(v.np(), ref['v'])
      family = f'update_kernels_adam_{start}'
      record_parity(family, update=raw, update_over_bound=ratio, m=max(em), v=max(ev))
      where = f'n={n} {cfg} {start} scale={scale} step {k + 1}'
      assert ratio <= 1.0, f'{where}: update error {raw:.3g} (cond {ref["cond"]:.3g})'
      assert max(em) <= U.TOL_SLOT and max(ev) <= U.TOL_SLOT, f'{where}: m {em}, v {ev}'
      assert step.cpu().tolist() == [ref['step'], 0, 12345], where
      for b, name in ((p, 'p'), (m, 'm'), (v, 'v')):
        b.check_canary(f'{where} {name}')
      if sdev is not None:
        assert float(sdev[1]) == CANARY_VALUE


# ---- RMSProp --------------------------------------------------------------------------------------
# (hyperparameters, ms initial value)
RMS = {
    'tf1_bench': (dict(lr=2.5e-4, decay=0.95, momentum=0.0, eps=1e-5, centered=True), 1.0),
    'keras_mnih15': (dict(lr=2.5e-4, decay=0.95, momentum=0.95, eps=0.01, centered=True), 0.0),
    'plain_mu0': (dict(lr=1e-3, decay=0.9, momentum=0.0, eps=1e-10, centered=False), 1.0),
    'plain_mu09': (dict(lr=1e-3, decay=0.9, momentum=0.9, eps=1e-7, centered=False), 0.0),
    'centered_mu09': (dict(lr=1e-3, decay=0.9, momentum=0.9, eps=1e-10, centered=True), 1.0),
}


def _rms_launch(p, g, ms, mg, mom, scale_dev, kw):
  _lib.call('b200rl_rmsprop_tf', _lib.ptr(p.t), _lib.ptr(g.t), _lib.ptr(ms.t), _lib.ptr(mg.t),
            _lib.ptr(mom.t), p.n, kw['lr'], kw['decay'], kw['momentum'], kw['eps'],
            int(kw['centered']), _lib.ptr(scale_dev), _lib.stream())


def _rms_check(family, where, bufs, pre, g, scale, kw):
  p, ms, mg, mom = bufs
  ref = U.rmsprop(pre['p'], g, pre['ms'], pre['mg'], pre['mom'], scale=scale, **kw)
  raw, ratio = U.update_error(p.np(), pre['p'], ref['u'], ref['cond'])
  mraw, mratio = U.cond_error(mom.np(), ref['mom'], ref['cond'])
  ems = U.slot_errors(ms.np(), ref['ms'])
  emg = U.slot_errors(mg.np(), ref['mg']) if kw['centered'] else (0.0, 0.0)
  record_parity(family, update=raw, update_over_bound=ratio, mom=mraw, mom_over_bound=mratio,
                ms=max(ems), mg=max(emg), max_kappa=float(ref['cond'].max()))
  assert ratio <= 1.0, f'{where}: update error {raw:.3g}, max κ {ref["cond"].max():.3g}'
  assert mratio <= 1.0, f'{where}: mom error {mraw:.3g}'
  assert max(ems) <= U.TOL_SLOT and max(emg) <= U.TOL_SLOT, f'{where}: ms {ems}, mg {emg}'
  if not kw['centered']:
    assert (mg.np() == pre['mg']).all(), f'{where}: mg written by the plain form'
  for b, name in zip(bufs, ('p', 'ms', 'mg', 'mom')):
    b.check_canary(f'{where} {name}')


@pytest.mark.parametrize('cfg', sorted(RMS))
@pytest.mark.parametrize('n', SIZES[:4] + [4098, 4099] + SIZES[4:])
def test_rmsprop_kernel(cuda, n, cfg):
  """Four steps from the optimizer's initial slots; n % 4 ≠ 0 takes the scalar path."""
  n = _size(n)
  kw, ms_init = RMS[cfg]
  rng = np.random.RandomState(n % 1000 + 3)
  for scale in SCALES:
    bufs = p, ms, mg, mom = (Buf(rng.randn(n)), Buf(np.full(n, ms_init)), Buf(np.zeros(n)),
                             Buf(np.zeros(n)))
    sdev = _scale_dev(scale)
    for k in range(4):
      g = Buf(U.gradients(rng, n))
      pre = dict(p=p.np(), ms=ms.np(), mg=mg.np(), mom=mom.np())
      _rms_launch(p, g, ms, mg, mom, sdev, kw)
      _rms_check(f'update_kernels_rmsprop_{cfg}', f'n={n} {cfg} scale={scale} step {k + 1}', bufs,
                 pre, g.np(), scale, kw)
      g.check_canary('g')


@pytest.mark.parametrize('cfg', ['tf1_bench', 'keras_mnih15', 'plain_mu09'])
def test_rmsprop_scalar_path_matches_float4_path(cuda, cfg):
  """Offsetting any one of p / g / ms / mg / mom by one float sends the launch down the scalar
  path; it must store the same bits as the float4 path on the same data."""
  kw, ms_init = RMS[cfg]
  n = 4096
  rng = np.random.RandomState(17)
  # a warmed-up state: non-zero momentum and mg
  state = dict(p=rng.randn(n).astype(f32), ms=(np.abs(rng.randn(n)) + ms_init).astype(f32),
               mg=(rng.randn(n) * 0.1).astype(f32), mom=(rng.randn(n) * 1e-4).astype(f32))
  state['ms'] = np.maximum(state['ms'], state['mg'] ** 2 * 1.5).astype(f32)
  g = U.gradients(rng, n)
  outs = {}
  for shifted in [None, 'p', 'g', 'ms', 'mg', 'mom']:
    off = lambda k: 1 if k == shifted else 0
    bufs = tuple(Buf(state[k], off(k)) for k in ('p', 'ms', 'mg', 'mom'))
    gb = Buf(g, off('g'))
    sdev = _scale_dev(0.37)
    pre = {k: state[k] for k in ('p', 'ms', 'mg', 'mom')}
    _rms_launch(bufs[0], gb, bufs[1], bufs[2], bufs[3], sdev, kw)
    _rms_check(f'update_kernels_rmsprop_{cfg}', f'{cfg} shifted {shifted}', bufs, pre, g, 0.37, kw)
    outs[shifted] = [b.np() for b in bufs]
  for shifted in ['p', 'g', 'ms', 'mg', 'mom']:
    for name, a, b in zip(('p', 'ms', 'mg', 'mom'), outs[None], outs[shifted]):
      assert np.array_equal(a.view(np.int32), b.view(np.int32)), f'{shifted} shifted: {name} differs'


# ---- global-norm scale ----------------------------------------------------------------------------
@pytest.mark.parametrize('n', [1, 75776, 75777, 5 * 2 ** 20 + 3])
def test_global_norm_scale(cuda, n):
  """n = 75 776 is one element per thread of the 296 × 256 partial-sum grid."""
  rng = np.random.RandomState(n % 1000)
  g = U.gradients(rng, n, zeros=0.01 if n > 1 else 0.0)
  g = Buf(g)
  ws, nb = workspace.get(cuda)
  _, nrm_ref = U.global_norm_scale(g.np(), 1.0)
  for clip in [0.0, 0.5 * nrm_ref, 2.0 * nrm_ref]:
    for outputs in ['both', 'scale', 'norm']:
      out = torch.full((4,), CANARY_VALUE, dtype=torch.float32, device=cuda)
      sc = out[0:1] if outputs in ('both', 'scale') else None
      nr = out[2:3] if outputs in ('both', 'norm') else None
      _lib.call('b200rl_global_norm_scale', _lib.ptr(g.t), n, float(clip), _lib.ptr(sc),
                _lib.ptr(nr), _lib.ptr(ws), nb, _lib.stream())
      got = out.cpu().numpy()
      scale_ref, _ = U.global_norm_scale(g.np(), clip)
      where = f'n={n} clip={clip:.3g} {outputs}'
      assert got[1] == CANARY_VALUE and got[3] == CANARY_VALUE, where
      if nr is None:
        assert got[2] == CANARY_VALUE, f'{where}: NULL norm written'
      else:
        e = U.rel_error(got[2], nrm_ref)
        record_parity('update_kernels_global_norm', norm=e)
        assert e <= U.TOL_NORM, f'{where}: norm {got[2]} vs {nrm_ref}'
      if sc is None:
        assert got[0] == CANARY_VALUE, f'{where}: NULL scale written'
      elif clip == 0.0 or clip > nrm_ref:
        assert got[0] == 1.0, f'{where}: scale {got[0]} where the clip does not bind'
      else:
        e = U.rel_error(got[0], scale_ref)
        record_parity('update_kernels_global_norm', scale=e)
        assert e <= U.TOL_CLIP, f'{where}: scale {got[0]} vs {scale_ref}'
  g.check_canary('g')


# ---- per-variable clip ----------------------------------------------------------------------------
def test_clip_by_norm_segments_on_network_offsets(cuda):
  """The padded offsets of the Mnih'15 Q-network (its 6-float head bias is padded to 8, its fc
  kernel holds 1.6 M floats), then a 0-length segment and segments of 1 024 and 1 025 floats."""
  net = _mnih_net()
  offs = list(net.param_offsets)
  end = offs[-1]
  offs += [end, end + 1024, end + 2049]
  sizes = [v.numel() for v in net.variables] + [0, 1024, 1025]
  assert 1605632 in sizes and any(b - a > s for a, b, s in zip(offs, offs[1:], sizes))
  rng = np.random.RandomState(23)
  g = U.gradients(rng, offs[-1])
  pad = np.zeros(offs[-1], bool)
  for a, b, s in zip(offs, offs[1:], sizes):
    pad[a + s:b] = True
  g[pad] = 0.0
  clip = 200.0
  ref, norms = U.clip_by_norm_segments(g, offs, clip)
  assert (norms > clip).any() and ((norms < clip) & (norms > 0)).any()
  gb = Buf(g)
  toffs = torch.tensor(offs, dtype=torch.int64, device=cuda)
  _lib.call('b200rl_clip_by_norm_segments', _lib.ptr(gb.t), _lib.ptr(toffs), len(offs) - 1,
            clip, _lib.stream())
  got = gb.np()
  gb.check_canary('g')
  assert (got[pad] == 0).all(), 'padding written'
  for i, (a, b) in enumerate(zip(offs, offs[1:])):
    if norms[i] <= clip:
      assert np.array_equal(got[a:b].view(np.int32), g[a:b].view(np.int32)), f'segment {i} moved'
    else:
      e = U.slot_errors(got[a:b], ref[a:b])
      record_parity('update_kernels_clip_segments', rel_l2=e[0], max=e[1])
      assert max(e) <= U.TOL_CLIP, f'segment {i} ({b - a} floats): {e}'


# ---- Polyak / Periodically ------------------------------------------------------------------------
@pytest.mark.parametrize('period', [1, 2, 5])
@pytest.mark.parametrize('tau', [0.0, 0.005, 0.5, 1.0])
@pytest.mark.parametrize('n', [3, 270337, 'mnih'])
def test_soft_update(cuda, n, tau, period):
  """2 × period calls with a fresh source each time.  τ = 1 copies bit for bit, a call that does
  not fire leaves the target bit for bit, and the counter follows Periodically, which advances
  on every call even when τ = 0 makes the body a no-op."""
  n = _size(n)
  rng = np.random.RandomState(n % 1000 + period)
  tgt = Buf(rng.randn(n))
  counter = _counter(0)
  gate = U.Periodically(period)
  for c in range(2 * period):
    src = Buf(rng.randn(n))
    before = tgt.np()
    _lib.call('b200rl_soft_update', _lib.ptr(tgt.t), _lib.ptr(src.t), n, tau, period,
              _lib.ptr(counter), _lib.stream())
    ref, fired = U.polyak_step(gate, before, src.np(), tau)
    got = tgt.np()
    where = f'n={n} tau={tau} period={period} call {c + 1}'
    if not fired or tau == 0.0:
      assert np.array_equal(got.view(np.int32), before.view(np.int32)), f'{where}: target moved'
    elif tau == 1.0:
      assert np.array_equal(got.view(np.int32), src.np().view(np.int32)), f'{where}: not a copy'
    else:
      e = U.polyak_error(got, before, src.np(), ref)
      record_parity('update_kernels_polyak', **{f'tau_{tau}': e})
      assert e <= U.TOL_POLYAK, f'{where}: error {e:.3g}'
    assert counter.cpu().tolist() == [gate.counter, 0, 12345], where
    tgt.check_canary(where)
    src.check_canary(where)


def test_counter_add(cuda):
  c = _counter(10 ** 6)
  for inc, want in [(1, 10 ** 6 + 1), (3, 10 ** 6 + 4), (0, 10 ** 6 + 4), (2 ** 40, 10 ** 6 + 4 + 2 ** 40)]:
    _lib.call('b200rl_counter_add', _lib.ptr(c), inc, _lib.stream())
    assert c.cpu().tolist() == [want, 0, 12345]
