"""b200rl_lstm_plan on the host (no GPU): the launch shape of the LSTM sequence kernels for every H
and a spread of B, a kernel case in tests/test_lstm_gpu.py for every launch class the planner can
pick, and the gridDim.y limit on the batch of the three LSTM entry points."""
import ctypes

import pytest
import torch

from agents_b200 import _lib

from test_lstm_gpu import CASES

BATCHES = (1, 2, 3, 4, 5, 8, 9, 12, 13, 16, 17, 24, 33, 40, 64, 4099)
U_BYTES = 128 * 1024          # resident U slice per CTA
SMEM_MAX = 227 * 1024         # opt-in shared memory per block on sm_90
MAX_THREADS = 384
MAX_TILES = 65535             # gridDim.y


def _plan(B, H):
  """(cluster, rows_fwd, rows_bwd, depth_fwd, depth_bwd, smem_fwd, smem_bwd)."""
  out = [ctypes.c_int() for _ in range(5)] + [ctypes.c_int64() for _ in range(2)]
  _lib.call('b200rl_lstm_plan', B, H, *[ctypes.byref(o) for o in out])
  return tuple(o.value for o in out)


def _launch_class(B, H):
  """(cs, forward rows, forward ring depth, backward rows, backward ring depth, ragged, padded):
  each entry selects different indexing in the kernels.  Ragged: the last CTA of the cluster owns
  fewer units than the others; padded: H is rounded up to Hp = ceil(H/4)*4."""
  cs, bf, bb, df, db, _, _ = _plan(B, H)
  hc = -(-H // cs)
  return (cs, bf, df, bb, db, cs > 1 and H % hc != 0, H % 4 != 0)


def test_plan_shapes_fit_the_kernels():
  for H in range(1, 257):
    hp = -(-H // 4) * 4
    for B in BATCHES:
      cs, bf, bb, df, db, sf, sb = _plan(B, H)
      fits = [c for c in (1, 2, 4, 8) if 16 * hp * -(-H // c) <= U_BYTES]
      assert cs == fits[0], (B, H, cs)
      hc = -(-H // cs)
      for rows, depth in ((bf, df), (bb, db)):
        assert rows % 4 == 0 and 4 <= rows <= min(16, -(-B // 4) * 4), (B, H, rows)
        assert depth in (2, 4), (B, H, depth)
        assert hc * rows // 4 <= MAX_THREADS, (B, H, rows)
      assert sf == 4 * (4 * hp * hc + 2 * bf * hp + df * bf * 4 * hc), (B, H)
      assert sb == 4 * (4 * H * hc + 2 * bb * 4 * H + db * bb * 7 * hc), (B, H)
      assert max(sf, sb) <= SMEM_MAX, (B, H, sf, sb)
  for B in (1, 4099):
    with pytest.raises(ValueError, match='units must be in'):
      _plan(B, 257)


def test_kernel_cases_cover_every_launch_class():
  """Every launch class the planner picks for H = 1..256 has a case in test_lstm_gpu.CASES, so a
  planner change that opens a new class fails here until a kernel case is added for it."""
  classes = {}
  for H in range(1, 257):
    for B in BATCHES:
      classes.setdefault(_launch_class(B, H), (B, H))
  covered = {_launch_class(B, H) for B, _, H in CASES}
  missing = sorted((k, classes[k]) for k in set(classes) - covered)
  assert not missing, '%d of %d launch classes have no kernel case, e.g. (B, H):\n%s' % (
      len(missing), len(classes), '\n'.join('%s %s' % m for m in missing))


def _entry_call(name, B, H):
  """One call of b200rl_lstm_seq_fwd / _bwd at [B, T = 1] with dummy 16-byte aligned addresses."""
  a = [0x10000 * (i + 1) for i in range(10)]
  if name == 'b200rl_lstm_seq_fwd':
    _lib.call(name, a[0], a[1], a[2], None, None, B, 1, H, a[3], a[4], a[5], a[6], a[7], a[8],
              None)
  else:
    _lib.call(name, a[0], a[1], a[2], None, a[3], a[4], B, 1, H, a[5], None)


def _limits(H):
  _, bf, bb, _, _, _, _ = _plan(4099, H)        # B >= 16: the rows of every larger batch
  return MAX_TILES * bf, MAX_TILES * bb


@pytest.mark.parametrize('H', [20, 256])
def test_batch_past_the_grid_limit_is_rejected(H):
  """Each direction launches ceil(B / rows) tiles along gridDim.y, at most 65535: one row past
  that is a ValueError naming the largest batch, raised before any CUDA call."""
  lim_f, lim_b = _limits(H)
  for name, lim in (('b200rl_lstm_seq_fwd', lim_f), ('b200rl_lstm_seq_bwd', lim_b)):
    with pytest.raises(ValueError, match=r'B must be <= %d for %d units' % (lim, H)):
      _entry_call(name, lim + 1, H)
  lim = min(lim_f, lim_b)
  _plan(lim, H)
  for B in (lim + 1, lim_f + 1, lim_b + 1):
    with pytest.raises(ValueError, match=r'B must be <= %d for %d units' % (lim, H)):
      _plan(B, H)


def _device_present():
  if torch.cuda.is_available():
    return True
  try:
    cu = ctypes.CDLL('libcuda.so.1')
  except OSError:
    return False
  n = ctypes.c_int(0)
  return cu.cuInit(0) == 0 and cu.cuDeviceGetCount(ctypes.byref(n)) == 0 and n.value > 0


@pytest.mark.parametrize('H', [20, 256])
def test_batch_at_the_grid_limit_passes_the_argument_checks(H):
  """At the largest batch every argument check passes and the call goes on to the launch, which
  fails for want of a device.  Where a device exists the dummy addresses would reach a kernel, so
  this is skipped there; test_lstm_gpu runs the largest grid (B = 1 048 560, H = 1) on real
  buffers instead."""
  if _device_present():
    pytest.skip('a CUDA device is present: the call would launch on dummy addresses')
  for name, lim in zip(('b200rl_lstm_seq_fwd', 'b200rl_lstm_seq_bwd'), _limits(H)):
    with pytest.raises(_lib.B200RLError, match='CUDA launch failed'):
      _entry_call(name, lim, H)
