"""Every dense / conv GEMM route of agents_b200/csrc/nn.cu against a float64 reference.

The dispatch in nn.cu picks one of about twenty kernels and epilogues for a dense or conv layer
from its shape: skinny heads, thin inputs, the wgmma tensor-core GEMM with BN 32/64/128 and the
STORE / COL2IM / ATOMIC epilogues, split-K with and without the reduce pass, the fp32 FFMA
GEMM, raw-u8 operands, the fused act' mask and bias gradient, accumulation, and 16-byte or scalar
gathers and stores.  Each row of the tables below gives an entry point, a shape and the kernel
instantiations that shape must launch.  The tests drive the C ABI directly, so every pointer,
stride and flag is under their control, check the launched kernel names under torch.profiler,
and compare every output with float64 numpy computed from the same fp32 inputs.

Metric: each element's error is normalised by the magnitude of its own dot product,
    e = max |got - ref| / (|A| @ |B| + |bias|),
with two absolute allowances: 4 ulp of 1.0 after tanhf, and 2^-23 |unmasked gradient| for the
fp32 (1 - y*y) of a tanh mask.  Masked gradients scale the magnitude by |act'(X)|, and
accumulated outputs allow two fp32 roundings of the prefill.  A correct 3xTF32 or fp32 kernel
measures well below 1e-5 on any data.  Dropping one TF32 cross term costs >= 3.3e-4 on positive
data, and a single TF32 pass ~7e-4 (numpy emulation, test_adversarial_data_defeats_single_pass_tf32).
So BOUND = 1e-5 separates a correct kernel from a degraded one, and
test_single_pass_tf32_exceeds_bound shows that it does on the GPU.  The rows with one long
unsplit reduction (K = 3136 or 2304 in a single CTA) pin the accumulation itself: the tensor
cores' fp32 accumulator does not round to nearest, and tc_gemm_kernel has to keep its chains
of wgmma accumulates short for these rows to stay within BOUND.

Every case runs on two data families: Gaussian, and "TF32-adversarial" values uniform in [1, 2)
(all 23 mantissa bits populated, all products positive, so a missing lo pass cannot hide behind
cancellation).  Every output array is followed by 64 canary floats that must stay untouched,
and inputs are followed by NaN canaries, so an over-read surfaces as a NaN output.
"""
import ctypes
import itertools
import json
import os
import re
import tempfile
import zlib
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from agents_b200 import _lib
from oracle import nn as onn
from conftest import record_parity

f32, f64 = np.float32, np.float64
BOUND = 1e-5
ULP1 = 2.0 ** -23                 # ulp of 1.0 in fp32
TINY = 1e-30
CANARY = 64                       # canary elements after every device array
CANARY_F32 = 0x7FC5A5A5           # a quiet NaN whose payload no arithmetic produces
CANARY_U8 = 0xA5
WS_BYTES = 32 << 20
U8_SCALE = 255.0
NONE, RELU, TANH = _lib.ACT_NONE, _lib.ACT_RELU, _lib.ACT_TANH
ACTS = (NONE, RELU, TANH)
FAMILIES = ('gauss', 'adversarial')
# (accumulate, db requested): dW / db overwritten, db skipped, and dW / db added to a random prefill
GRAD_MODES = ((0, True), (0, False), (1, True))


# ---- the route table ------------------------------------------------------------------------
# Kernel names are matched (re.fullmatch) against the demangled name with the b200rl:: / tc::
# namespaces, the parameter list and the blanks after commas removed.
def tc(bn, epi, a, b, passes=3, chains=False):
  """tc_gemm_kernel<BN, PASSES, EPI, A view, B view, CHAINS>; EPI 0 = STORE, 1 = COL2IM,
  2 = ATOMIC; CHAINS: a CTA's K range is longer than 256, so its accumulation is chained."""
  return f'tc_gemm_kernel<{bn},{passes},{epi},{a},{b},{str(chains).lower()}>'


def sg(bm, bn, tm, tn, a, b):
  return f'sgemm_kernel<{bm},{bn},{tm},{tn},{a},{b}>'


REDUCE = 'splitk_reduce_kernel'
COLSUM = ('colsum_partial_kernel', 'colsum_final_kernel')


@dataclass(frozen=True)
class Dense:
  M: int
  K: int
  N: int
  kernels: tuple
  ldx: int = 0          # row stride of X (0: K)
  ws: bool = True       # pass the workspace (split-K allowed)
  dw: bool = True       # backward: compute dW (db alone otherwise)
  out_off: int = 0      # outputs start this many floats past a 16-byte boundary

  @property
  def id(self):
    s = f'{self.M}x{self.K}x{self.N}'
    s += f'_ldx{self.ldx}' if self.ldx else ''
    s += '' if self.ws else '_nows'
    s += '' if self.dw else '_nodW'
    return s + (f'_outoff{self.out_off}' if self.out_off else '')


@dataclass(frozen=True)
class Conv:
  N: int
  H: int
  W: int
  C: int
  F: int
  k: int
  s: int
  kernels: tuple
  u8: bool = False
  xbs: int = 0          # x_batch_stride in elements (0: H*W*C)
  out_off: int = 0

  @property
  def id(self):
    s = f'{self.N}x{self.H}x{self.W}x{self.C}_F{self.F}k{self.k}s{self.s}'
    s += '_u8' if self.u8 else ''
    s += f'_xbs{self.xbs}' if self.xbs else ''
    return s + (f'_outoff{self.out_off}' if self.out_off else '')

  @property
  def oh(self):
    return (self.H - self.k) // self.s + 1

  @property
  def ow(self):
    return (self.W - self.k) // self.s + 1


TC_FWD128 = tc(128, 0, 'ARow', 'BRow')
TC_FWD128_LONG = tc(128, 0, 'ARow', 'BRow', chains=True)
DENSE_FWD = [
    Dense(1, 4, 1, ('skinny_fwd_kernel<4>',)),
    Dense(300, 768, 16, ('skinny_fwd_kernel<16>',)),          # W is exactly 48 KiB: still skinny
    Dense(300, 769, 16, (tc(32, 0, 'ARow', 'BRow'), REDUCE)),   # one row more: tensor cores, split 5
    Dense(33, 1, 20, ('thin_fwd_kernel',)),
    Dense(64, 32, 256, ('thin_fwd_kernel',)),
    Dense(64, 33, 256, (TC_FWD128,)),
    Dense(129, 40, 64, (tc(64, 0, 'ARow', 'BRow'),), ldx=40),  # 16-byte gathers
    Dense(129, 40, 64, (tc(64, 0, 'ARow', 'BRow'),), ldx=41),  # odd row stride: scalar gathers
    Dense(32, 65, 65, (TC_FWD128,)),
    Dense(31, 65, 65, (sg(64, 64, 4, 4, 'ARow', 'BRow'),)),    # M < 32: FFMA
    Dense(256, 3136, 512, (TC_FWD128, REDUCE)),                # split 14
    Dense(256, 3136, 512, (TC_FWD128_LONG,), ws=False),        # no workspace: one K pass
    Dense(4096, 3136, 512, (TC_FWD128_LONG,)),                 # 128 tiles: no split either
    Dense(256, 3136, 6, (sg(128, 32, 4, 4, 'ARow', 'BRow'), REDUCE)),   # N < 16, K > 1024
    Dense(8, 3136, 512, (sg(64, 64, 4, 4, 'ARow', 'BRow'), REDUCE)),
    Dense(5000, 7, 62, (sg(128, 64, 8, 4, 'ARow', 'BRow'),)),  # K < 8, N % 4 != 0
    Dense(20000, 7, 130, (sg(128, 128, 8, 8, 'ARow', 'BRow'),)),
]

TC_DX = lambda bn, chains=False: tc(bn, 0, 'ARow', 'BCol', chains=chains)   # noqa: E731  dY @ W^T
TC_DW = lambda bn, chains=False: tc(bn, 2, 'ACol', 'BRow', chains=chains)   # noqa: E731  X^T @ dY
DENSE_BWD = [
    Dense(1, 4, 1, ('skinny_dx_kernel<4>', 'skinny_dw_kernel<4,1>')),
    Dense(300, 768, 16, ('skinny_dx_kernel<16>', 'skinny_dw_kernel<16,4>')),
    Dense(300, 769, 16, (TC_DX(128), TC_DW(32))),
    Dense(33, 1, 20, (sg(128, 32, 4, 4, 'ARow', 'BCol'), 'thin_dw_kernel<8>')),
    Dense(64, 32, 256, (TC_DX(32), REDUCE, 'thin_dw_kernel<32>')),
    Dense(64, 33, 256, (TC_DX(64), REDUCE, TC_DW(128))),
    Dense(129, 40, 64, (TC_DX(64), TC_DW(64)), ldx=40),
    Dense(129, 40, 64, (TC_DX(64), TC_DW(64)), ldx=41),
    Dense(32, 65, 65, (TC_DX(128), TC_DW(128))),
    Dense(31, 65, 65, (sg(64, 64, 4, 4, 'ARow', 'BCol'), TC_DW(128))),
    Dense(256, 3136, 512, (TC_DX(128), REDUCE, TC_DW(128))),
    Dense(256, 3136, 512, (TC_DX(128, True), TC_DW(128)), ws=False),
    Dense(2304, 3136, 512, (TC_DX(128, True), TC_DW(128, True))),   # unsplit: dX 512, dW 2304
    Dense(256, 3136, 6, (sg(64, 64, 4, 4, 'ARow', 'BCol'), sg(128, 32, 4, 4, 'ACol', 'BRow'), REDUCE)
          + COLSUM),
    Dense(8, 3136, 512, (sg(64, 64, 4, 4, 'ARow', 'BCol'), REDUCE, TC_DW(128))),
    Dense(5000, 7, 62, (sg(128, 32, 4, 4, 'ARow', 'BCol'), sg(64, 64, 4, 4, 'ACol', 'BRow'), REDUCE)
          + COLSUM),
    Dense(20000, 7, 130, (sg(128, 32, 4, 4, 'ARow', 'BCol'), sg(64, 64, 4, 4, 'ACol', 'BRow'), REDUCE)
          + COLSUM),
    Dense(257, 300, 5, ('skinny_dx_kernel<8>', 'skinny_dw_kernel<8,2>')),
    Dense(257, 300, 5, ('skinny_dx_kernel<8>',) + COLSUM, dw=False),
    # outputs one float past a 16-byte boundary: the vector stores must fall back to scalar ones
    Dense(257, 300, 5, ('skinny_dx_kernel<8>', 'skinny_dw_kernel<8,2>'), out_off=1),
    Dense(129, 40, 64, (TC_DX(64), TC_DW(64)), ldx=40, out_off=1),
]

C_U8 = (3, 84, 84, 4, 32, 8, 4)       # the Atari first layer
C_U8_SMALL = (1, 12, 12, 4, 16, 8, 4)  # M = 4 output positions
C_F32 = (3, 20, 20, 32, 64, 4, 2)
C_ODD = (1, 7, 9, 5, 3, 3, 2)         # C % 4 != 0
C_WIDE = (2, 7, 7, 8, 256, 3, 1)      # F = 256 reduction, one output tile
AF, ATF = 'AConv<float>', 'AConvT<float>'
CONV_FWD = [
    Conv(*C_U8, (tc(32, 0, 'AConvU8Raw', 'BRow'), REDUCE), u8=True),
    Conv(*C_U8_SMALL, (sg(128, 32, 4, 4, 'AConv<unsigned char>', 'BRow'), REDUCE), u8=True),
    Conv(*C_F32, (tc(64, 0, AF, 'BRow'), REDUCE)),
    Conv(*C_F32, (tc(64, 0, AF, 'BRow'), REDUCE), xbs=2 * 20 * 20 * 32),
    Conv(*C_ODD, (sg(128, 32, 4, 4, AF, 'BRow'),)),
    Conv(*C_WIDE, (tc(128, 0, AF, 'BRow'),)),
]
COL2IM = tc(128, 1, 'ARow', 'BCol')
CONV_BWD = [
    Conv(*C_U8, (tc(32, 2, 'AConvTU8Raw', 'BRow'),), u8=True),
    Conv(*C_U8_SMALL, (sg(128, 32, 4, 4, 'AConvT<unsigned char>', 'BRow'),) + COLSUM, u8=True),
    Conv(*C_F32, (tc(64, 2, ATF, 'BRow'), COL2IM)),
    Conv(*C_F32, (tc(64, 2, ATF, 'BRow'), COL2IM), xbs=2 * 20 * 20 * 32),   # a [B,2,H,W,C] slice
    Conv(*C_ODD, (sg(128, 32, 4, 4, ATF, 'BRow'), sg(64, 64, 4, 4, 'ARow', 'BCol'), 'col2im_kernel')
         + COLSUM),
    Conv(*C_WIDE, (tc(128, 2, ATF, 'BRow'), COL2IM)),           # the col2im GEMM splits K in two
    # misaligned dX / dW / db, and an image stride that misaligns the mask input X
    Conv(*C_F32, (tc(64, 2, ATF, 'BRow'), COL2IM), out_off=1),
    Conv(*C_F32, (tc(64, 2, ATF, 'BRow'), COL2IM), xbs=20 * 20 * 32 + 1),
]

TABLES = dict(dense_fwd=DENSE_FWD, dense_bwd=DENSE_BWD, conv_fwd=CONV_FWD, conv_bwd=CONV_BWD)


# ---- float64 reference and metric -------------------------------------------------------------
def route_err(got, ref, scale, absolute=0.0):
  """max over elements of (|got - ref| - absolute)+ / scale, in float64."""
  got = np.asarray(got, f64)
  excess = np.maximum(np.abs(got - ref) - absolute, 0.0)
  return float(np.max(excess / (scale + TINY))) if got.size else 0.0


def mm(a, b):
  """A @ B and |A| @ |B| in float64."""
  a, b = np.asarray(a, f64), np.asarray(b, f64)
  return a @ b, np.abs(a) @ np.abs(b)


def act_out(z, s, bias, act):
  """Forward epilogue: (reference, magnitude, absolute allowance) of act(z + bias)."""
  if bias is not None:
    z, s = z + np.asarray(bias, f64), s + np.abs(np.asarray(bias, f64))
  if act == RELU:
    return np.maximum(z, 0.0), s, 0.0
  if act == TANH:
    return np.tanh(z), s, 4 * ULP1
  return z, s, 0.0


def act_input(raw, x_act):
  """X as the layer with activation x_act would have produced it."""
  if x_act == RELU:
    return np.maximum(raw, f32(0))
  if x_act == TANH:
    return np.tanh(raw).astype(f32)
  return raw


def masked(g, s, x, x_act):
  """Input gradient times act'(X): (reference, magnitude, absolute allowance)."""
  if x_act == NONE:
    return g, s, 0.0
  x = np.asarray(x, f64)
  d = (x > 0).astype(f64) if x_act == RELU else 1.0 - x * x
  absolute = ULP1 * np.abs(g) if x_act == TANH else 0.0
  return d * g, np.abs(d) * s, absolute


def im2col(x, k, s):
  return onn.im2col(np.ascontiguousarray(x, f64), k, k, s)[0]


def col2im(dcol, shape, k, s):
  """The scatter loop of oracle.nn.conv2d_bwd in float64: dcol [N*OH*OW, k*k*C] -> [N,H,W,C]."""
  n, h, w, c = shape
  oh, ow = (h - k) // s + 1, (w - k) // s + 1
  d = np.asarray(dcol, f64).reshape(n, oh, ow, k, k, c)
  dx = np.zeros(shape, f64)
  for ky in range(k):
    for kx in range(k):
      dx[:, ky:ky + oh * s:s, kx:kx + ow * s:s, :] += d[:, :, :, ky, kx, :]
  return dx


def tf32(x):
  """x with the low 13 mantissa bits cleared: the value a TF32 tensor-core operand keeps."""
  return (np.asarray(x, f32).view(np.uint32) & np.uint32(0xFFFFE000)).view(f32)


def data(rng, family, shape):
  if family == 'gauss':
    return rng.standard_normal(shape).astype(f32)
  return rng.uniform(1.0, 2.0, shape).astype(f32)


def pixels(rng, family, shape):
  lo = 0 if family == 'gauss' else 128
  return rng.randint(lo, 256, size=shape).astype(np.uint8)


def rng_for(key, family):
  return np.random.RandomState(zlib.crc32(f'{key}:{family}'.encode()))


# ---- device buffers with canaries -------------------------------------------------------------
def _canary(dtype, n):
  if dtype == np.uint8:
    return np.full(n, CANARY_U8, np.uint8)
  return np.full(n, CANARY_F32, np.uint32).view(f32)


class DevBuf(object):
  """`arr` on the device `off` elements past a 16-byte aligned allocation, canaries before (the
  `off` slack) and CANARY elements after."""

  def __init__(self, arr, off=0):
    arr = np.ascontiguousarray(arr)
    self.shape, self.off, self.n = arr.shape, off, arr.size
    host = np.concatenate([_canary(arr.dtype, off), arr.reshape(-1), _canary(arr.dtype, CANARY)])
    self.t = torch.from_numpy(host).to('cuda')
    assert self.t.data_ptr() % 16 == 0
    self.ptr = self.t.data_ptr() + off * arr.itemsize

  def fetch(self, what):
    """The array; asserts that the canaries are intact and every element is finite."""
    h = self.t.cpu().numpy()
    bits = h.view(np.uint8 if h.dtype == np.uint8 else np.uint32)
    c = CANARY_U8 if h.dtype == np.uint8 else CANARY_F32
    assert (bits[:self.off] == c).all() and (bits[self.off + self.n:] == c).all(), \
        f'{what}: a kernel wrote outside the {self.shape} output'
    got = h[self.off:self.off + self.n].reshape(self.shape)
    bad = int((~np.isfinite(got)).sum())
    assert bad == 0, f'{what}: {bad} of {got.size} elements not finite (unwritten or NaN read)'
    return got


def ptr(buf):
  return None if buf is None else buf.ptr


def nans(shape):
  return np.full(shape, np.nan, f32)


def strided_rows(x, ld):
  """[M, K] rows at stride ld; the gap columns hold NaN."""
  out = nans((x.shape[0], ld))
  out[:, :x.shape[1]] = x
  return out


def strided_images(x, xbs):
  """[N, H, W, C] images `xbs` elements apart; the gaps hold NaN (canary bytes for u8)."""
  if not xbs:
    return x
  n = x.shape[0]
  out = np.full((n, xbs), np.nan, f32) if x.dtype == f32 else np.full((n, xbs), CANARY_U8, np.uint8)
  out[:, :x[0].size] = x.reshape(n, -1)
  return out


# ---- route check ------------------------------------------------------------------------------
_OBSERVED = set()     # normalised kernel names seen by the route checks
_CHECKED = set()      # table rows whose route check ran
_PROFILER = {'empty': False}


def _normalise(name):
  name = re.sub(r'^void ', '', name).split('(')[0]
  name = name.replace('b200rl::', '').replace('tc::', '')
  return re.sub(r',\s+', ',', name).strip()


def _kernel_names(fn):
  """Normalised names of the kernels `fn` launches, or None if the profiler saw no kernel.
  Read from the exported trace: the library's kernels have no PyTorch op to hang from."""
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
  names = [e['name'] for e in events if e.get('cat') == 'kernel' and 'name' in e]
  return [_normalise(n) for n in names] or None


def check_route(table, row, fn):
  """Runs fn once under the profiler; the set of launched kernels must be exactly row.kernels."""
  names = _kernel_names(fn)
  _CHECKED.add((table, row.id))
  if names is None:
    _PROFILER['empty'] = True
    return
  _OBSERVED.update(names)
  unexpected = sorted({n for n in names if not any(re.fullmatch(p, n) for p in row.kernels)})
  missing = [p for p in row.kernels if not any(re.fullmatch(p, n) for n in names)]
  assert not unexpected and not missing, \
      f'{table} {row.id}: launched {sorted(set(names))}, the table expects {list(row.kernels)}'


class Errors(object):
  """Largest e per output of one row; recorded, then asserted against BOUND."""

  def __init__(self, table, row):
    self.key, self.worst, self.fails = f'{table}:{row.id}', {}, []

  def add(self, label, out, buf, ref, scale, absolute=0.0):
    got = buf.fetch(f'{self.key} {label} {out}')
    e = route_err(got, ref, scale, absolute)
    k = f'{self.key}:{out}'
    self.worst[k] = max(self.worst.get(k, 0.0), e)
    if not e <= BOUND:
      self.fails.append(f'{label} {out}: e={e:.3g}')

  def finish(self):
    record_parity('gemm_route_err', **self.worst)
    assert not self.fails, f'{self.key} exceeds {BOUND}: ' + '; '.join(self.fails[:8])


def _default_mode():
  return int(os.environ.get('B200RL_GEMM_MODE', '1'))


@pytest.fixture
def gemm(cuda):
  """Pins the 3xTF32 tensor-core mode the table is written for; yields the workspace."""
  _lib.call('b200rl_set_gemm_mode', 1)
  ws = torch.empty(WS_BYTES // 4, dtype=torch.float32, device=cuda)
  try:
    yield lambda use=True: (ws.data_ptr(), WS_BYTES) if use else (None, 0)
  finally:
    _lib.call('b200rl_set_gemm_mode', _default_mode())


def _ids(rows):
  return [r.id for r in rows]


# ---- dense ------------------------------------------------------------------------------------
def _dense_fwd(row, ws, x, w, b, act, off):
  ldx = row.ldx or row.K
  X, W = DevBuf(strided_rows(x, ldx), off), DevBuf(w, off)
  B = DevBuf(b, off) if b is not None else None
  Y = DevBuf(nans((row.M, row.N)), row.out_off)
  _lib.call('b200rl_dense_fwd', X.ptr, ldx, W.ptr, ptr(B), Y.ptr, row.M, row.K, row.N, act,
            *ws(row.ws), _lib.stream())
  return Y


@pytest.mark.gpu
@pytest.mark.parametrize('row', DENSE_FWD, ids=_ids(DENSE_FWD))
def test_dense_fwd_route(gemm, row):
  errs = Errors('dense_fwd', row)
  for fam in FAMILIES:
    rng = rng_for(row.id, fam)
    x, w, b = data(rng, fam, (row.M, row.K)), data(rng, fam, (row.K, row.N)), data(rng, fam, (row.N,))
    z, s = mm(x, w)
    if fam == FAMILIES[0]:
      check_route('dense_fwd', row, lambda: _dense_fwd(row, gemm, x, w, b, NONE, 0))
    for off, bias, act in itertools.product((0, 1), (True, False), ACTS):
      bb = b if bias else None
      Y = _dense_fwd(row, gemm, x, w, bb, act, off)
      errs.add(f'{fam} off={off} bias={bias} act={act}', 'Y', Y, *act_out(z, s, bb, act))
  errs.finish()


def _dense_bwd(row, ws, x, w, dy, acc, want_db, prefill, x_act, off):
  ldx = row.ldx or row.K
  X, W, dY = DevBuf(strided_rows(x, ldx), off), DevBuf(w, off), DevBuf(dy, off)
  init = (lambda a: a) if acc else (lambda a: nans(a.shape))
  dX = DevBuf(nans((row.M, row.K)), row.out_off)
  dW = DevBuf(init(prefill[0]), row.out_off) if row.dw else None
  db = DevBuf(init(prefill[1]), row.out_off) if want_db else None
  _lib.call('b200rl_dense_bwd', X.ptr, ldx, W.ptr, dY.ptr, dX.ptr, ptr(dW), ptr(db), row.M, row.K,
            row.N, acc, x_act, *ws(row.ws), _lib.stream())
  return dX, dW, db


def _grad_checks(errs, label, acc, prefill, outs, refs):
  """outs: (dW, db) buffers or None; refs: ((ref, magnitude) of dW, of db)."""
  for name, buf, (ref, s), p in zip(('dW', 'db'), outs, refs, prefill):
    if buf is None:
      continue
    if acc:
      p = np.asarray(p, f64)
      errs.add(label, name, buf, p + ref, s, 2 * 2.0 ** -23 * np.abs(p))
    else:
      errs.add(label, name, buf, ref, s)


@pytest.mark.gpu
@pytest.mark.parametrize('row', DENSE_BWD, ids=_ids(DENSE_BWD))
def test_dense_bwd_route(gemm, row):
  M, K, N = row.M, row.K, row.N
  errs = Errors('dense_bwd', row)
  for fam in FAMILIES:
    rng = rng_for(row.id, fam)
    raw, w, dy = data(rng, fam, (M, K)), data(rng, fam, (K, N)), data(rng, fam, (M, N))
    prefill = (rng.standard_normal((K, N)).astype(f32), rng.standard_normal(N).astype(f32))
    gx, sx = mm(dy, w.T)
    db_ref = (np.asarray(dy, f64).sum(0), np.abs(np.asarray(dy, f64)).sum(0))
    if fam == FAMILIES[0]:
      check_route('dense_bwd', row, lambda: _dense_bwd(row, gemm, raw, w, dy, 0, True, prefill, NONE, 0))
    for x_act in ACTS:
      x = act_input(raw, x_act)
      dw_ref = mm(x.T, dy)
      dx_ref = masked(gx, sx, x, x_act)
      for (acc, want_db), off in itertools.product(GRAD_MODES, (0, 1)):
        label = f'{fam} x_act={x_act} acc={acc} db={want_db} off={off}'
        dX, dW, db = _dense_bwd(row, gemm, x, w, dy, acc, want_db, prefill, x_act, off)
        errs.add(label, 'dX', dX, *dx_ref)
        _grad_checks(errs, label, acc, prefill, (dW, db), (dw_ref, db_ref))
  errs.finish()


# ---- conv -------------------------------------------------------------------------------------
def _geom(row):
  return _lib.ConvGeom(row.N, row.H, row.W, row.C, row.k, row.k, row.F, row.s, row.xbs)


def _conv_input(rng, fam, row, x_act=NONE):
  shape = (row.N, row.H, row.W, row.C)
  if row.u8:
    return pixels(rng, fam, shape)
  return act_input(data(rng, fam, shape), x_act)


def _as_f64(x):
  return x.astype(f64) / U8_SCALE if x.dtype == np.uint8 else x.astype(f64)


def _conv_fwd(row, ws, x, w, b, act, off):
  X, W = DevBuf(strided_images(x, row.xbs), off), DevBuf(w, off)
  B = DevBuf(b, off) if b is not None else None
  Y = DevBuf(nans((row.N * row.oh * row.ow, row.F)), row.out_off)
  g = _geom(row)
  _lib.call('b200rl_conv2d_fwd', X.ptr, int(row.u8), U8_SCALE, W.ptr, ptr(B), Y.ptr, ctypes.byref(g),
            act, *ws(), _lib.stream())
  return Y


@pytest.mark.gpu
@pytest.mark.parametrize('row', CONV_FWD, ids=_ids(CONV_FWD))
def test_conv_fwd_route(gemm, row):
  errs = Errors('conv_fwd', row)
  K = row.k * row.k * row.C
  for fam in FAMILIES:
    rng = rng_for(row.id, fam)
    x, w, b = _conv_input(rng, fam, row), data(rng, fam, (K, row.F)), data(rng, fam, (row.F,))
    z, s = mm(im2col(_as_f64(x), row.k, row.s), w)
    if fam == FAMILIES[0]:
      check_route('conv_fwd', row, lambda: _conv_fwd(row, gemm, x, w, b, NONE, 0))
    for off, bias, act in itertools.product((0, 1), (True, False), ACTS):
      bb = b if bias else None
      Y = _conv_fwd(row, gemm, x, w, bb, act, off)
      errs.add(f'{fam} off={off} bias={bias} act={act}', 'Y', Y, *act_out(z, s, bb, act))
  errs.finish()


def _conv_bwd(row, ws, x, w, dy, acc, want_db, prefill, x_act, off):
  X, W, dY = DevBuf(strided_images(x, row.xbs), off), DevBuf(w, off), DevBuf(dy, off)
  init = (lambda a: a) if acc else (lambda a: nans(a.shape))
  dX = None if row.u8 else DevBuf(nans((row.N, row.H, row.W, row.C)), row.out_off)
  dW = DevBuf(init(prefill[0]), row.out_off)
  db = DevBuf(init(prefill[1]), row.out_off) if want_db else None
  g = _geom(row)
  _lib.call('b200rl_conv2d_bwd', X.ptr, int(row.u8), U8_SCALE, W.ptr, dY.ptr, ptr(dX), dW.ptr, ptr(db),
            ctypes.byref(g), acc, x_act, *ws(), _lib.stream())
  return dX, dW, db


@pytest.mark.gpu
@pytest.mark.parametrize('row', CONV_BWD, ids=_ids(CONV_BWD))
def test_conv_bwd_route(gemm, row):
  errs = Errors('conv_bwd', row)
  K, M = row.k * row.k * row.C, row.N * row.oh * row.ow
  shape = (row.N, row.H, row.W, row.C)
  for fam in FAMILIES:
    rng = rng_for(row.id, fam)
    raw = pixels(rng, fam, shape) if row.u8 else data(rng, fam, shape)
    w, dy = data(rng, fam, (K, row.F)), data(rng, fam, (M, row.F))
    prefill = (rng.standard_normal((K, row.F)).astype(f32), rng.standard_normal(row.F).astype(f32))
    gcol, scol = mm(dy, w.T)
    gx, sx = col2im(gcol, shape, row.k, row.s), col2im(scol, shape, row.k, row.s)
    db_ref = (np.asarray(dy, f64).sum(0), np.abs(np.asarray(dy, f64)).sum(0))
    if fam == FAMILIES[0]:
      check_route('conv_bwd', row, lambda: _conv_bwd(row, gemm, raw, w, dy, 0, True, prefill, NONE, 0))
    for x_act in ((NONE,) if row.u8 else ACTS):
      x = raw if row.u8 else act_input(raw, x_act)
      dw_ref = mm(im2col(_as_f64(x), row.k, row.s).T, dy)
      dx_ref = masked(gx, sx, x, x_act)
      for (acc, want_db), off in itertools.product(GRAD_MODES, (0, 1)):
        label = f'{fam} x_act={x_act} acc={acc} db={want_db} off={off}'
        dX, dW, db = _conv_bwd(row, gemm, x, w, dy, acc, want_db, prefill, x_act, off)
        if dX is not None:
          errs.add(label, 'dX', dX, *dx_ref)
        _grad_checks(errs, label, acc, prefill, (dW, db), (dw_ref, db_ref))
  errs.finish()


# ---- the bound can fail -----------------------------------------------------------------------
@pytest.mark.gpu
def test_single_pass_tf32_exceeds_bound(gemm):
  """Mode 2 (one TF32 pass) on a tensor-core row with adversarial data must exceed BOUND: the
  metric and data above really detect a missing lo pass."""
  row = Dense(64, 33, 256, (tc(128, 0, 'ARow', 'BRow', passes=1),))
  rng = rng_for('single_pass', 'adversarial')
  x, w = data(rng, 'adversarial', (row.M, row.K)), data(rng, 'adversarial', (row.K, row.N))
  z, s = mm(x, w)
  _lib.call('b200rl_set_gemm_mode', 2)
  try:
    Y = _dense_fwd(row, gemm, x, w, None, NONE, 0)
    e = route_err(Y.fetch('mode 2'), z, s)
  finally:
    _lib.call('b200rl_set_gemm_mode', _default_mode())
  record_parity('gemm_route_err', **{'single_pass_tf32_control': e})
  assert e > BOUND, f'single-pass TF32 measured e={e:.3g}, within the 3xTF32 bound {BOUND}'


def _run_route_test(gemm, table, row):
  dict(dense_fwd=test_dense_fwd_route, dense_bwd=test_dense_bwd_route, conv_fwd=test_conv_fwd_route,
       conv_bwd=test_conv_bwd_route)[table](gemm, row)


@pytest.mark.gpu
def test_every_listed_kernel_was_observed(gemm):
  """Every kernel instantiation named in the tables was launched by some row.  A dispatch change
  then has to update the table instead of silently leaving a kernel untested.

  The verdict does not depend on what else ran in this process: rows whose route test did not run
  here (a -k selection, or a suite split across processes) run now, and if the profiler saw no
  kernel events earlier, every row runs again under a fresh profiler session."""
  if _PROFILER['empty']:
    _PROFILER['empty'] = False
    todo = [(t, r) for t, tab in TABLES.items() for r in tab]
  else:
    todo = [(t, r) for t, tab in TABLES.items() for r in tab if (t, r.id) not in _CHECKED]
  for t, r in todo:
    _run_route_test(gemm, t, r)
  if _PROFILER['empty']:
    pytest.skip('kernel names unavailable: the CUDA profiler recorded no kernel events')
  listed = {p for tab in TABLES.values() for r in tab for p in r.kernels}
  missing = sorted(p for p in listed if not any(re.fullmatch(p, n) for n in _OBSERVED))
  assert not missing, f'listed but never launched: {missing}'


# ---- host-only checks of the reference, the metric and the data -------------------------------
def test_reference_matches_oracle():
  """The float64 reference agrees with oracle/nn.py (float32) and col2im is im2col's adjoint."""
  rng = np.random.RandomState(0)
  x, w, b = rng.randn(5, 7).astype(f32), rng.randn(7, 3).astype(f32), rng.randn(3).astype(f32)
  z, s = mm(x, w)
  ref, _, _ = act_out(z, s, b, TANH)
  np.testing.assert_allclose(ref, onn.dense_fwd(x, w, b, 'tanh'), rtol=1e-5, atol=1e-6)
  assert np.all(s >= np.abs(z))
  n, h, wd, c, f, k, st = C_ODD
  xi = rng.randn(n, h, wd, c).astype(f32)
  wt = rng.randn(k, k, c, f).astype(f32)
  oh, ow = (h - k) // st + 1, (wd - k) // st + 1
  dz = rng.randn(n, oh, ow, f).astype(f32)
  zc, _ = mm(im2col(xi, k, st), wt.reshape(-1, f))
  np.testing.assert_allclose(zc.reshape(n, oh, ow, f), onn.conv2d_fwd(xi, wt, None, st), rtol=1e-5,
                             atol=1e-5)
  gcol, _ = mm(dz.reshape(-1, f), wt.reshape(-1, f).T)
  dx, dw, db = onn.conv2d_bwd(xi, wt, dz, st)
  np.testing.assert_allclose(col2im(gcol, xi.shape, k, st), dx, rtol=1e-5, atol=1e-5)
  np.testing.assert_allclose(mm(im2col(xi, k, st).T, dz.reshape(-1, f))[0], dw.reshape(-1, f),
                             rtol=1e-5, atol=1e-5)
  # adjoint: <im2col(x), d> == <x, col2im(d)> exactly up to float64 rounding
  d = rng.randn(*gcol.shape)
  lhs = float(np.sum(im2col(xi, k, st) * d))
  rhs = float(np.sum(np.asarray(xi, f64) * col2im(d, xi.shape, k, st)))
  assert abs(lhs - rhs) <= 1e-12 * np.abs(d).sum() * np.abs(xi).max()


def test_metric():
  rng = np.random.RandomState(1)
  a, b = rng.randn(16, 40), rng.randn(40, 8)
  z, s = mm(a, b)
  assert route_err(z, z, s) == 0.0
  assert route_err(z + 1e-4 * s, z, s) == pytest.approx(1e-4)
  assert route_err(z + 1e-6, z, s, absolute=2e-6) == 0.0          # absolute allowance
  g, gs, absolute = masked(z, s, np.zeros_like(z), RELU)          # relu mask 0: result must be 0
  assert route_err(np.zeros_like(z), g, gs, absolute) == 0.0
  assert route_err(np.full_like(z, 1e-20), g, gs, absolute) > 1e6
  y = np.tanh(rng.randn(*z.shape)).astype(f32)
  g, gs, absolute = masked(z, s, y, TANH)
  fp32 = np.asarray(z, f32) * (f32(1) - y * y)                     # what the kernels compute
  assert route_err(fp32, g, gs, absolute) < BOUND


def test_adversarial_data_defeats_single_pass_tf32():
  """numpy emulation of the tensor-core arithmetic (TF32 operands, exact products): the
  adversarial family pushes one TF32 pass above 16x BOUND and one dropped cross term above BOUND,
  while the 3-pass split (lo parts TF32-truncated as the hardware reads them) stays below it."""
  for K in (8, 65, 3136):
    rng = rng_for(f'emulation{K}', 'adversarial')
    a, b = data(rng, 'adversarial', (64, K)), data(rng, 'adversarial', (K, 16))
    z, s = mm(a, b)
    ah, bh = tf32(a), tf32(b)
    al, bl = tf32(a - ah), tf32(b - bh)
    hh, hl, lh = mm(ah, bh)[0], mm(ah, bl)[0], mm(al, bh)[0]
    assert route_err(hh, z, s) > 16 * BOUND, K
    assert route_err(hh + hl, z, s) > BOUND, K
    assert route_err(hh + hl + lh, z, s) < BOUND / 4, K
  rng = rng_for('emulation_gauss', 'gauss')
  a, b = data(rng, 'gauss', (64, 3136)), data(rng, 'gauss', (3136, 16))
  z, s = mm(a, b)
  assert route_err(mm(tf32(a), tf32(b))[0], z, s) > BOUND
