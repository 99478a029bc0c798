"""The raw-uint8 first-layer GEMMs, whose A operand goes to wgmma from registers.

tc_gemm_kernel with an exact A view (AConvU8Raw for the conv forward, AConvTU8Raw for the filter
gradient) loads each thread's m64k8 fragments straight from the raw uint8 ring slot, converts
them to fp32 and issues both TF32 passes (a * b_lo, a * b_hi) from two register sets.  The K-
contiguous forward view reorders the reduction index inside each K block and the split of B
stores B in the same order.  The rows below cover the Atari geometry (84x84x4, 8x8 filters,
stride 4) at batch 1, 3, 32 and 256, filter counts that select BN = 32 with an N tail, 64 and
128, an M tail, K ranges whose last split is short, [B, 2, 84, 84, 4] observation slices passed
through the image stride, and (through the route tests' off = 1 variants) a uint8 base that is
not 4-byte aligned, which takes the byte copies.  The filter gradient also runs with
accumulate = 1 and no bias gradient.

Each row runs through the route tests' own numeric checks (test_gemm_routes_gpu): both data
families, float64 references, NaN canaries and the 1e-5 BOUND.  The kernel check asks that the
exact-view tensor-core GEMM ran.  test_atari_dw_grid checks that the filter-gradient grid at the
benchmark's batch is the one the split-K planner makes for two CTAs per SM.
"""
import json
import os
import re
import tempfile

import numpy as np
import pytest
import torch

import test_gemm_routes_gpu as R
from test_gemm_routes_gpu import gemm  # noqa: F401  (fixture)

Conv = R.Conv
U8 = (r'tc_gemm_kernel<\d+,3,[02],AConvT?U8Raw,BRow,(true|false)>|splitk_reduce_kernel',)
ATARI = (84, 84, 4, 32, 8, 4)
OBS = 2 * 84 * 84 * 4          # image stride of one [2, 84, 84, 4] observation pair


@pytest.fixture
def u8(gemm, monkeypatch):  # noqa: F811
  """The route tests' workspace fixture; the kernel check asks for an exact-view GEMM, and the
  gradient modes add accumulate = 1 without a bias gradient."""

  def exact_only(table, row, fn):
    names = R._kernel_names(fn)
    if names is None:          # the profiler saw no kernel: the numeric checks still run
      return
    other = sorted({n for n in names if not any(re.fullmatch(p, n) for p in row.kernels)})
    assert not other and any('U8Raw' in n for n in names), \
        f'{table} {row.id}: launched {sorted(set(names))}, expected the raw-uint8 tensor-core GEMM'

  monkeypatch.setattr(R, 'check_route', exact_only)
  monkeypatch.setattr(R, 'GRAD_MODES', R.GRAD_MODES + ((1, False),))
  return gemm


ROWS = [
    Conv(1, *ATARI, U8, u8=True),                  # M = 400: a 16-row tail tile
    Conv(3, *ATARI, U8, u8=True),                  # dW: K = 1200 in 160-wide splits, the last 80
    Conv(32, *ATARI, U8, u8=True),
    Conv(256, *ATARI, U8, u8=True),                # the benchmark's batch
    Conv(3, *ATARI, U8, u8=True, xbs=OBS),         # frame 0 of [3, 2, 84, 84, 4]
    Conv(32, *ATARI, U8, u8=True, xbs=OBS),
    Conv(2, 45, 45, 4, 32, 9, 4, U8, u8=True),     # K = 324: forward splits 192 + 132
    Conv(3, 84, 84, 4, 20, 8, 4, U8, u8=True),     # BN = 32 with 12 empty columns
    Conv(3, 84, 84, 4, 64, 8, 4, U8, u8=True),     # BN = 64
    Conv(2, 84, 84, 4, 128, 8, 4, U8, u8=True),    # BN = 128
]


@pytest.mark.gpu
@pytest.mark.parametrize('row', ROWS, ids=R._ids(ROWS))
def test_u8_conv_fwd(u8, row):
  R.test_conv_fwd_route(u8, row)


@pytest.mark.gpu
@pytest.mark.parametrize('row', ROWS, ids=R._ids(ROWS))
def test_u8_conv_bwd(u8, row):
  R.test_conv_bwd_route(u8, row)


def plan_splits(tiles, K, target, bk=32):
  """Split count of nn.cu's plan_split_k (round down, no workspace cap)."""
  s = 1
  if tiles < target and K >= 8 * bk:
    s = min(target // tiles, K // (4 * bk), 65535)
    s = 1 if s < 2 else s
  kps = -(-K // s)
  kps = -(-kps // bk) * bk
  return -(-K // kps)


def _kernel_grids(fn):
  """(name, grid) of every kernel `fn` launches, from the profiler trace's kernel args."""
  from torch.profiler import ProfilerActivity, profile
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    fn()
    torch.cuda.synchronize()
  with tempfile.TemporaryDirectory() as d:
    path = os.path.join(d, 'trace.json')
    prof.export_chrome_trace(path)
    with open(path) as f:
      events = json.load(f).get('traceEvents', [])
  return [(R._normalise(e['name']), e.get('args', {}).get('grid'))
          for e in events if e.get('cat') == 'kernel' and 'name' in e]


@pytest.mark.gpu
def test_atari_dw_grid(u8):
  """conv1 dW at batch 256 (M = 256 x 400 positions) is a 256 x 32 output, 2 tiles of 128 x 32:
  the planner splits K for 2 x 132 CTAs, 128 splits of 800 positions."""
  row = Conv(256, *ATARI, U8, u8=True)
  K, M = row.k * row.k * row.C, row.N * row.oh * row.ow
  rng = np.random.RandomState(0)
  x = R.pixels(rng, 'gauss', (row.N, row.H, row.W, row.C))
  w, dy = R.data(rng, 'gauss', (K, row.F)), R.data(rng, 'gauss', (M, row.F))
  prefill = (np.zeros((K, row.F), np.float32), np.zeros(row.F, np.float32))
  got = _kernel_grids(lambda: R._conv_bwd(row, u8, x, w, dy, 0, True, prefill, R.NONE, 0))
  grids = [g for n, g in got if n.startswith('tc_gemm_kernel<32,3,2,AConvTU8Raw')]
  if not got:
    pytest.skip('kernel events unavailable: the CUDA profiler recorded none')
  assert len(grids) == 1 and grids[0] is not None, f'launched {got}'
  splits = plan_splits(2, M, 2 * 132)
  assert splits == 128
  assert list(grids[0]) == [1, 2, splits], f'dW grid {grids[0]}, planned [1, 2, {splits}]'
