"""Edges of the tensor-core GEMM's cp.async operand ring that the route table does not reach.

tc_gemm_kernel copies raw operand tiles global -> shared several K blocks ahead with cp.async and
zero-fills every chunk (or the part of a chunk) that lies past a K tail, a row end or an image.
The rows below put those edges where the ring can get them wrong: a K tail that is not a multiple
of 4 inside a 16-byte aligned row stride (with NaN in the stride gap), M and N tails inside a
partial tile (including a partial 4-row group of an MN-contiguous view), K ranges of one and two
blocks (shorter than the ring), split-K ranges whose last split is shorter than the others, and
uint8 conv inputs whose 32-byte (kx, c) runs are 16-byte aligned, only 4-byte aligned, or at an
odd image stride (byte copies).

Each row runs through the route tests' own numeric checks (test_gemm_routes_gpu): both data
families, every activation / accumulate / alignment variant, float64 references, NaN canaries
and the 1e-5 BOUND.  The kernel check is this file's own: it asks only that the tensor-core GEMM
(and the split-K reduce, where the planner splits) ran, so that each edge really goes through the
ring, and it leaves the route table's bookkeeping of observed kernels and profiler sessions alone.
"""
import re

import pytest

import test_gemm_routes_gpu as R
from test_gemm_routes_gpu import gemm  # noqa: F401  (fixture)

Dense, Conv = R.Dense, R.Conv
TC = (r'tc_gemm_kernel<.*>|splitk_reduce_kernel',)


@pytest.fixture
def ring(gemm, monkeypatch):  # noqa: F811
  """The route tests' workspace fixture, with their kernel check replaced by `tc_only`."""

  def tc_only(table, row, fn):
    names = R._kernel_names(fn)
    if names is None:          # the profiler saw no kernel: the numeric checks still run
      return
    other = sorted({n for n in names if not any(re.fullmatch(p, n) for p in row.kernels)})
    assert not other and any(n.startswith('tc_gemm_kernel<') for n in names), \
        f'{table} {row.id}: launched {sorted(set(names))}, expected the tensor-core GEMM only'

  monkeypatch.setattr(R, 'check_route', tc_only)
  return gemm


DENSE_FWD = [
    Dense(129, 38, 64, TC, ldx=40),    # K tail 38 in 16-byte rows, NaN gap: 2 K blocks
    Dense(129, 38, 64, TC, ldx=41),    # the same with 4-byte copies
    Dense(130, 60, 50, TC),            # M tail, N = 50: scalar copies of the weights
    Dense(200, 72, 100, TC),           # BN = 128 with 28 empty columns, M tail
    Dense(256, 1300, 64, TC),          # split-K: 5-block splits, the last one 1 block with a tail
    Dense(256, 1000, 32, TC),          # BN = 32: 5-block splits, the last one 2 blocks
]
DENSE_BWD = [
    Dense(129, 38, 64, TC, ldx=40),    # dW: X^T rows end mid 4-row group (partial 16-byte copy)
    Dense(130, 70, 20, TC),            # dX: one K block (K = 20)
    Dense(96, 40, 36, TC),             # dX: two K blocks (K = 36)
    Dense(129, 38, 64, TC, ldx=41, out_off=1),
]
CONV_FWD = [
    Conv(2, 36, 36, 4, 32, 8, 4, TC, u8=True),                      # (kx, c) runs 16-byte aligned
    Conv(2, 20, 21, 4, 32, 8, 2, TC, u8=True),                      # runs 4-byte aligned, M tail
    Conv(2, 20, 20, 4, 32, 8, 2, TC, u8=True, xbs=20 * 20 * 4 + 1),  # odd image stride: byte copies
    Conv(2, 11, 11, 8, 48, 3, 2, TC, xbs=11 * 11 * 8 + 4),          # fp32, N tail, strided images
]
CONV_BWD = CONV_FWD


@pytest.mark.gpu
@pytest.mark.parametrize('row', DENSE_FWD, ids=R._ids(DENSE_FWD))
def test_ring_dense_fwd(ring, row):
  R.test_dense_fwd_route(ring, row)


@pytest.mark.gpu
@pytest.mark.parametrize('row', DENSE_BWD, ids=R._ids(DENSE_BWD))
def test_ring_dense_bwd(ring, row):
  R.test_dense_bwd_route(ring, row)


@pytest.mark.gpu
@pytest.mark.parametrize('row', CONV_FWD, ids=R._ids(CONV_FWD))
def test_ring_conv_fwd(ring, row):
  R.test_conv_fwd_route(ring, row)


@pytest.mark.gpu
@pytest.mark.parametrize('row', CONV_BWD, ids=R._ids(CONV_BWD))
def test_ring_conv_bwd(ring, row):
  R.test_conv_bwd_route(ring, row)
