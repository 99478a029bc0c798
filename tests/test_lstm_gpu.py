"""LSTM sequence kernels (csrc/lstm.cu) and the recurrent networks against float64.

Kernels: the forward (outputs, gates, c, consumed h, final state) within 2e-5 relative of
oracle/lstm.py in float64, and the backward (dG) plus the layer's dW, dU, db and dx within 1e-4,
over a case for every launch class b200rl_lstm_plan picks (tests/test_lstm_plan_host.py checks
that), T up to 1001, B across the tile boundary up to the largest grid, and four reset patterns.
Networks: the reference's structure tests, a stacked network against float64 and [B, T] == T
chained [B, 1] calls."""
import os

import numpy as np
import pytest
import torch

from agents_b200 import _lib
from agents_b200.networks import actor_distribution_rnn_network as adrn
from agents_b200.networks import lstm_encoding_network as len_
from agents_b200.networks import value_rnn_network as vrn
from agents_b200.specs import tensor_spec
from oracle import lstm as olstm

from conftest import record_parity

pytestmark = pytest.mark.gpu
f32 = np.float32


def _plan(B, H):
  """(cluster, rows forward / backward, ring depth forward / backward)."""
  import ctypes
  out = [ctypes.c_int() for _ in range(5)]
  _lib.call('b200rl_lstm_plan', B, H, *[ctypes.byref(o) for o in out], None, None)
  return tuple(o.value for o in out)


def _steps(rng, B, T, pattern):
  st = np.ones((B, T), np.int32)
  if pattern == 'first':
    st[:, 0] = 0
  elif pattern == 'random':
    st[rng.rand(B, T) < 0.1] = 0
  elif pattern == 'every':
    st[:] = 0
  return st


def _layer(cuda, In, H, seed):
  net = len_.LSTMEncodingNetwork(tensor_spec.TensorSpec((In,), torch.float32),
                                 input_fc_layer_params=(), lstm_size=(H,),
                                 output_fc_layer_params=(), device=cuda).set_seed(seed)
  net.create_variables()
  return net, net.layers[0]


def _rel(got, want):
  return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


def _run(cuda, B, T, In, H, pattern, seed=0, init_state=False):
  rng = np.random.RandomState(seed)
  net, cell = _layer(cuda, In, H, seed)
  # a larger recurrent kernel than the orthogonal init, so that the recurrence matters
  with torch.no_grad():
    cell.recurrent_kernel.mul_(1.5)
    cell.bias.uniform_(-0.5, 0.5)
  x = rng.randn(B, T, In).astype(f32)
  st = _steps(rng, B, T, pattern)
  dh = rng.randn(B, T, H).astype(f32)
  h0 = c0 = None
  if init_state:
    h0, c0 = rng.randn(B, H).astype(f32) * 0.5, rng.randn(B, H).astype(f32) * 0.5
  d = lambda a: torch.as_tensor(a, device=cuda)
  st_d = d(st)
  state = None if h0 is None else (d(h0), d(c0))
  h, (hT, cT), ctx = cell.forward_seq(d(x.reshape(B * T, In)), st_d, B, T, state)
  net.flat_grads.zero_()
  dx = cell.backward_seq(ctx, d(dh.reshape(B * T, H)), need_dx=True)
  W, U, b = (t.detach().cpu().numpy().astype(np.float64) for t in
             (cell.kernel, cell.recurrent_kernel, cell.bias))
  wh, (whT, wcT), cache = olstm.lstm_forward(
      x.astype(np.float64), W, U, b, st, None if h0 is None else h0.astype(np.float64),
      None if c0 is None else c0.astype(np.float64))
  wdx, wdW, wdU, wdb, wdG = olstm.lstm_backward(cache, dh.astype(np.float64))
  g = lambda t: t.detach().cpu().numpy()
  fwd = dict(h=_rel(g(h).reshape(B, T, H), wh), hT=_rel(g(hT), whT), cT=_rel(g(cT), wcT),
             gates=_rel(g(ctx[1]).reshape(B, T, 4 * H), cache['gates']),
             c=_rel(g(ctx[2]).reshape(B, T, H), cache['c']),
             h_used=_rel(g(ctx[3]).reshape(B, T, H), cache['h_used']))
  bwd = dict(dx=_rel(g(dx).reshape(B, T, In), wdx), dW=_rel(g(cell.d_kernel), wdW),
             dU=_rel(g(cell.d_recurrent_kernel), wdU), db=_rel(g(cell.d_bias), wdb))
  return fwd, bwd


CASES = [(B, T, H) for H in (1, 5, 7, 20, 40, 64, 96, 128, 160, 256)
         for (B, T) in ((1, 33), (17, 33), (40, 2))] + [
    (30, 1001, 20), (30, 1001, 40), (5, 1001, 256), (3, 1, 7), (33, 1001, 128), (9, 1001, 160)]
# One case per launch class (cluster size, rows and ring depth of each direction, ragged last
# slice, padded H) that the cases above leave out.  By cluster size:
CLASS_CASES = [
    # cs 1: 8- and 12-row tiles, backward ring of 2, 8-row backward, forward ring of 2 (H = 89)
    (12, 33, 39), (9, 33, 40), (24, 33, 76), (33, 33, 77), (9, 33, 84), (12, 33, 85),
    (17, 33, 87), (5, 33, 88), (16, 33, 88), (8, 33, 89), (13, 33, 89),
    # cs 2: ragged (odd H) and padded slices, 12-row tiles
    (4, 33, 90), (1, 33, 91), (24, 33, 98), (33, 33, 99), (9, 33, 102), (12, 33, 104),
    (12, 33, 105), (5, 33, 110), (8, 33, 112), (17, 33, 113), (16, 33, 114), (13, 33, 116),
    (9, 33, 117), (12, 33, 122), (40, 33, 123), (9, 33, 124), (33, 33, 126), (8, 33, 127),
    # cs 4: 38/38/38/36 units at H = 150
    (8, 33, 129), (24, 33, 139), (17, 33, 140), (2, 33, 150), (5, 33, 156), (16, 33, 157),
    (9, 33, 165), (40, 33, 172), (13, 33, 173), (12, 33, 174), (9, 33, 176),
    # cs 8: a 26-unit last slice at H = 250, 12-row tiles, backward ring of 2
    (9, 33, 181), (1, 33, 188), (13, 33, 191), (33, 33, 192), (40, 33, 196), (24, 33, 201),
    (12, 33, 204), (9, 33, 208), (17, 33, 212), (16, 33, 216), (40, 33, 220), (12, 33, 229),
    (13, 33, 235), (5, 33, 236), (9, 33, 236), (12, 33, 240), (9, 33, 241), (2, 33, 250),
    (12, 33, 252), (8, 33, 255), (9, 33, 256)]
# Long sequences through the ragged and depth-2 paths; 257 clusters of 4 and 513 clusters of 8
# CTAs, more than fit on the GPU at once; and the largest grid, 65535 tiles of 16 rows.
WIDE_CASES = [(13, 1001, 255), (17, 1001, 89), (9, 1001, 150), (4099, 5, 150), (4099, 5, 255),
              (65535 * 16, 2, 1)]
CASES += CLASS_CASES + WIDE_CASES


def _parity_group(B, T, H):
  """Suffix of the parity record of an added case: the path it was added for."""
  if (B, T, H) in WIDE_CASES:
    return '_long' if T == 1001 else '_many_tiles'
  if (B, T, H) not in CLASS_CASES:
    return ''
  cs, _, _, df, db = _plan(B, H)
  hc = -(-H // cs)
  if cs > 1 and H % hc:
    return '_ragged'
  if cs > 1 and H % 4:
    return '_padded'
  return '_ring2' if 2 in (df, db) else '_tiles'


@pytest.mark.parametrize('B,T,H', CASES)
@pytest.mark.parametrize('pattern', ['none', 'first', 'random', 'every'])
def test_lstm_seq_kernels_match_float64(cuda, B, T, H, pattern):
  if pattern in ('none', 'every') and (T == 1001 or (B, T, H) in CLASS_CASES + WIDE_CASES):
    pytest.skip('long sequences and added launch classes run the first-step and random resets')
  fwd, bwd = _run(cuda, B, T, 11, H, pattern, seed=B * 1000 + H + T)
  group = _parity_group(B, T, H)
  record_parity('lstm_seq_fwd' + group, **{k + '_rel': v for k, v in fwd.items()})
  record_parity('lstm_seq_bwd' + group, **{k + '_rel': v for k, v in bwd.items()})
  for k, v in fwd.items():
    assert v <= 2e-5, (k, v, _plan(B, H))
  for k, v in bwd.items():
    assert v <= 1e-4, (k, v, _plan(B, H))


def test_lstm_plan_covers_every_cluster_size():
  seen = {_plan(B, H)[0] for H in (1, 5, 7, 20, 40, 64, 96, 128, 160, 256) for B in (1, 17)}
  assert seen == {1, 2, 4, 8}
  with pytest.raises(ValueError):
    _plan(4, 257)
  with pytest.raises(ValueError):
    len_.LSTM(257)


@pytest.mark.parametrize('H', [7, 128])
def test_lstm_given_initial_state(cuda, H):
  fwd, bwd = _run(cuda, 6, 33, 5, H, 'random', seed=11, init_state=True)
  record_parity('lstm_seq_fwd_initial_state', **{k + '_rel': v for k, v in fwd.items()})
  record_parity('lstm_seq_bwd_initial_state', **{k + '_rel': v for k, v in bwd.items()})
  for k, v in fwd.items():
    assert v <= 2e-5, (k, v)
  for k, v in bwd.items():
    assert v <= 1e-4, (k, v)


def _bwd(cuda, cell, ctx, dh, B, T, H):
  dG = torch.empty((B * T, 4 * H), device=cuda)
  _lib.call('b200rl_lstm_seq_bwd', _lib.ptr(dh), _lib.ptr(ctx[1]), _lib.ptr(ctx[2]), None,
            _lib.ptr(cell.recurrent_kernel), _lib.ptr(ctx[5]), B, T, H, _lib.ptr(dG),
            _lib.stream())
  return dG.reshape(B, T, 4 * H)


@pytest.mark.parametrize('H', [20, 256])
def test_nothing_crosses_a_reset(cuda, H):
  """Forward: perturbing every input before a FIRST leaves every output after it bit-identical.
  Backward: perturbing every output gradient from the FIRST on leaves the gate gradients before
  it bit-identical (the recurrent carries are cut at the reset)."""
  rng = np.random.RandomState(5)
  B, T, In, t0 = 3, 40, 6, 17
  net, cell = _layer(cuda, In, H, 3)
  x = rng.randn(B, T, In).astype(f32)
  st = np.ones((B, T), np.int32)
  st[:, t0] = 0
  dh = rng.randn(B, T, H).astype(f32)
  d = lambda a: torch.as_tensor(a, device=cuda)
  hs, dgs = [], []
  for pert in (0.0, 1.0):
    xp = x.copy()
    xp[:, :t0] += pert * rng.randn(B, t0, In).astype(f32)
    h, _, ctx = cell.forward_seq(d(xp.reshape(B * T, In)), d(st), B, T)
    hs.append(h.reshape(B, T, H)[:, t0:].cpu().numpy())
  _, _, ctx = cell.forward_seq(d(x.reshape(B * T, In)), d(st), B, T)
  for pert in (0.0, 1.0):
    dhp = dh.copy()
    dhp[:, t0:] += pert * rng.randn(B, T - t0, H).astype(f32)
    dgs.append(_bwd(cuda, cell, ctx, d(dhp.reshape(B * T, H)), B, T, H)[:, :t0].cpu().numpy())
  assert np.array_equal(hs[0], hs[1])
  assert np.array_equal(dgs[0], dgs[1])
  assert np.abs(dgs[0]).max() > 0


@pytest.mark.parametrize('H', [150, 255])
def test_many_clusters_repeat_bit_for_bit(cuda, H):
  """B = 4099 launches 257 clusters of 4 CTAs (H = 150) or 513 of 8 (H = 255), run in waves: two
  launches give the same h, gates, c and dG bit for bit."""
  rng = np.random.RandomState(H)
  B, T, In = 4099, 5, 11
  net, cell = _layer(cuda, In, H, 8)
  d = lambda a: torch.as_tensor(a, device=cuda)
  x = d(rng.randn(B * T, In).astype(f32))
  st = d(_steps(rng, B, T, 'random'))
  dh = d(rng.randn(B * T, H).astype(f32))
  runs = []
  for _ in range(2):
    h, _, ctx = cell.forward_seq(x, st, B, T)
    runs.append((h, ctx[1], ctx[2], _bwd(cuda, cell, ctx, dh, B, T, H)))
  for a, b in zip(*runs):
    assert torch.equal(a, b)


def test_collect_step_from_given_state(cuda):
  """The collect shape: one step (T = 1) from a given (h0, c0) over B = 4099 rows at H = 150
  (cs 4, ragged and padded).  h, hT and cT match float64; a row whose step is FIRST gives the same
  bits as a run with no initial state."""
  rng = np.random.RandomState(12)
  B, T, In, H = 4099, 1, 11, 150
  net, cell = _layer(cuda, In, H, 12)
  with torch.no_grad():
    cell.recurrent_kernel.mul_(1.5)
    cell.bias.uniform_(-0.5, 0.5)
  x = rng.randn(B, In).astype(f32)
  st = _steps(rng, B, T, 'random')
  h0, c0 = rng.randn(B, H).astype(f32) * 0.5, rng.randn(B, H).astype(f32) * 0.5
  d = lambda a: torch.as_tensor(a, device=cuda)
  h, (hT, cT), _ = cell.forward_seq(d(x), d(st), B, T, (d(h0), d(c0)))
  hz, (hTz, cTz), _ = cell.forward_seq(d(x), d(st), B, T)
  W, U, b = (t.detach().cpu().numpy().astype(np.float64) for t in
             (cell.kernel, cell.recurrent_kernel, cell.bias))
  wh, (whT, wcT), _ = olstm.lstm_forward(x.astype(np.float64)[:, None], W, U, b, st,
                                         h0.astype(np.float64), c0.astype(np.float64))
  g = lambda t: t.cpu().numpy()
  rel = dict(h=_rel(g(h), wh[:, 0]), hT=_rel(g(hT), whT), cT=_rel(g(cT), wcT))
  record_parity('lstm_seq_fwd_collect_step', **{k + '_rel': v for k, v in rel.items()})
  for k, v in rel.items():
    assert v <= 2e-5, (k, v)
  first = st[:, 0] == 0
  assert 0 < first.sum() < B
  for a, z in ((h, hz), (hT, hTz), (cT, cTz)):
    assert np.array_equal(g(a)[first], g(z)[first])
    assert not np.array_equal(g(a)[~first], g(z)[~first])


def test_saturated_gates(cuda):
  """Gate pre-activations of scale 30 at H = 255 (cs 8, ragged and padded): most |z| are far past
  20, where the sigmoids and tanh saturate.  Every output and gate gradient is finite and matches
  float64."""
  rng = np.random.RandomState(13)
  B, T, H = 17, 33, 255
  xw = (30 * rng.randn(B, T, 4 * H)).astype(f32)
  assert (np.abs(xw) > 20).mean() > 0.4
  U = (1.5 * rng.randn(H, 4 * H) / np.sqrt(H)).astype(f32)
  st = _steps(rng, B, T, 'random')
  dh = rng.randn(B, T, H).astype(f32)
  d = lambda a: torch.as_tensor(a, device=cuda)
  xw_d, U_d, st_d, dh_d = d(xw), d(U), d(st), d(dh)
  e = lambda *s: torch.empty(s, device=cuda)
  h, c, h_used = e(B, T, H), e(B, T, H), e(B, T, H)
  gates, dG, hT, cT = e(B, T, 4 * H), e(B, T, 4 * H), e(B, H), e(B, H)
  _lib.call('b200rl_lstm_seq_fwd', _lib.ptr(xw_d), _lib.ptr(U_d), _lib.ptr(st_d), None, None, B,
            T, H, _lib.ptr(h), _lib.ptr(gates), _lib.ptr(c), _lib.ptr(h_used), _lib.ptr(hT),
            _lib.ptr(cT), _lib.stream())
  _lib.call('b200rl_lstm_seq_bwd', _lib.ptr(dh_d), _lib.ptr(gates), _lib.ptr(c), None,
            _lib.ptr(U_d), _lib.ptr(st_d), B, T, H, _lib.ptr(dG), _lib.stream())
  # x = xw with W = I and b = 0 feeds the pre-activations to the float64 recurrence unchanged
  wh, (whT, wcT), cache = olstm.lstm_forward(xw.astype(np.float64), np.eye(4 * H),
                                             U.astype(np.float64), np.zeros(4 * H), st)
  wdG = olstm.lstm_backward(cache, dh.astype(np.float64))[4]
  g = lambda t: t.cpu().numpy()
  for t in (h, gates, c, hT, cT, dG):
    assert np.isfinite(g(t)).all()
  fwd = dict(h=_rel(g(h), wh), hT=_rel(g(hT), whT), cT=_rel(g(cT), wcT),
             gates=_rel(g(gates), cache['gates']), c=_rel(g(c), cache['c']),
             h_used=_rel(g(h_used), cache['h_used']))
  bwd = dict(dG=_rel(g(dG), wdG))
  record_parity('lstm_seq_fwd_saturated', **{k + '_rel': v for k, v in fwd.items()})
  record_parity('lstm_seq_bwd_saturated', **{k + '_rel': v for k, v in bwd.items()})
  for k, v in fwd.items():
    assert v <= 2e-5, (k, v)
  assert bwd['dG'] <= 1e-4, bwd


def test_batch_past_the_grid_limit_raises_before_launch(cuda):
  """B = 65535 * 16 + 1 needs a 65536th tile along gridDim.y: b200rl_lstm_seq_fwd / _bwd raise
  ValueError without launching, and so does the layer's forward."""
  B, T, H, In = 65535 * 16 + 1, 1, 1, 3
  net, cell = _layer(cuda, In, H, 0)
  z = lambda *s: torch.zeros(s, device=cuda)
  xw, gates = z(B, 4 * H), z(B, 4 * H)
  h, c, h_used, hT, cT = z(B, H), z(B, H), z(B, H), z(B, H), z(B, H)
  st = torch.zeros((B, T), dtype=torch.int32, device=cuda)
  limit = r'B must be <= %d for %d units' % (65535 * 16, H)
  n0 = _lib.launch_count()
  with pytest.raises(ValueError, match=limit):
    _lib.call('b200rl_lstm_seq_fwd', _lib.ptr(xw), _lib.ptr(cell.recurrent_kernel), _lib.ptr(st),
              None, None, B, T, H, _lib.ptr(h), _lib.ptr(gates), _lib.ptr(c), _lib.ptr(h_used),
              _lib.ptr(hT), _lib.ptr(cT), _lib.stream())
  with pytest.raises(ValueError, match=limit):
    _lib.call('b200rl_lstm_seq_bwd', _lib.ptr(h), _lib.ptr(gates), _lib.ptr(c), None,
              _lib.ptr(cell.recurrent_kernel), _lib.ptr(st), B, T, H, _lib.ptr(xw),
              _lib.stream())
  assert _lib.launch_count() == n0
  with pytest.raises(ValueError, match=limit):
    cell.forward_seq(z(B * T, In), st, B, T)
  torch.cuda.synchronize()


def _dense64(l):
  return (l.kernel.detach().cpu().numpy().astype(np.float64),
          l.bias.detach().cpu().numpy().astype(np.float64))


def test_stacked_network_matches_float64(cuda):
  """fc (16,) -> LSTM (150, 89) -> fc (8,) over [19, 40] with random resets.  The first LSTM runs
  cs 4 with a ragged, padded last slice; the second the forward ring of 2 and the 8-row backward.
  The output, every gradient in flat_grads and dLoss/d(first LSTM input) match oracle/lstm.py in
  float64 (dense layers in float64 beside it).  The input-gradient-only backward, which DDPG and
  SAC take for dQ/da, returns the same dx bit for bit and leaves flat_grads untouched."""
  rng = np.random.RandomState(14)
  B, T, D = 19, 40, 6
  net = len_.LSTMEncodingNetwork(tensor_spec.TensorSpec((D,), torch.float32),
                                 input_fc_layer_params=(16,), lstm_size=(150, 89),
                                 output_fc_layer_params=(8,), device=cuda).set_seed(14)
  net.create_variables()
  assert _plan(B, 150)[0] == 4 and _plan(B, 89)[3:] == (2, 4) and _plan(B, 89)[2] == 8
  obs = rng.randn(B, T, D).astype(f32)
  st = _steps(rng, B, T, 'random')
  dy = rng.randn(B * T, 8).astype(f32)
  d = lambda a: torch.as_tensor(a, device=cuda)
  out, tape = net.forward_train(d(obs), d(st))
  grads = net.backward(tape, d(dy)).clone()
  got = [v.cpu().numpy() for v in net._grad_views]
  _, ctxs, post_tape = tape
  dx = net._backward_recurrent(ctxs, post_tape, d(dy), need_dx=True, need_param_grads=False)
  assert torch.equal(net.flat_grads, grads)
  dx_with_grads = net._backward_recurrent(ctxs, post_tape, d(dy), need_dx=True)
  assert torch.equal(dx, dx_with_grads)

  (w1, b1), (w2, b2) = _dense64(net._pre[0]), _dense64(net._post[0])
  cells = [[t.detach().cpu().numpy().astype(np.float64)
            for t in (c.kernel, c.recurrent_kernel, c.bias)] for c in net._cells]
  y1 = np.maximum(obs.reshape(B * T, D).astype(np.float64) @ w1 + b1, 0)
  hs, _, caches = olstm.stacked_forward(y1.reshape(B, T, 16), cells, st)
  hs = hs.reshape(B * T, -1)
  y2 = np.maximum(hs @ w2 + b2, 0)
  dz2 = dy * (y2 > 0)
  wdx, cgrads = olstm.stacked_backward(caches, (dz2 @ w2.T).reshape(B, T, -1))
  wdx = wdx.reshape(B * T, 16)
  dz1 = wdx * (y1 > 0)
  want = [obs.reshape(B * T, D).T @ dz1, dz1.sum(0)] + [g for cg in cgrads for g in cg] + [
      hs.T @ dz2, dz2.sum(0)]
  assert len(got) == len(want)
  rel = dict(out=_rel(out.cpu().numpy(), y2), dx=_rel(dx.cpu().numpy(), wdx),
             grads=max(_rel(a, b) for a, b in zip(got, want)))
  record_parity('lstm_stacked_network', **{k + '_rel': v for k, v in rel.items()})
  for k, v in rel.items():
    assert v <= 1e-4, (k, v)


def test_value_rnn_network_structure(cuda):
  """value_rnn_network_test.py:37-82: conv + fc + LSTM(7) + fc + Dense(1) -> 11 variables."""
  spec = tensor_spec.TensorSpec((8, 8, 3), torch.float32)
  net = vrn.ValueRnnNetwork(spec, conv_layer_params=((4, 2, 2),), input_fc_layer_params=(5,),
                            lstm_size=(7,), output_fc_layer_params=(5,), device=cuda)
  net.create_variables()
  shapes = [tuple(v.shape) for v in net.variables]
  assert len(shapes) == 11
  assert shapes[4:7] == [(5, 28), (7, 28), (28,)]
  assert [tuple(s.shape) for s in net.state_spec] == [(7,), (7,)]
  assert [s.name for s in net.state_spec] == ['network_state_0', 'network_state_1']
  obs = torch.randn(3, 8, 8, 3, device=cuda)
  v, (h, c) = net(obs, torch.zeros(3, dtype=torch.int32, device=cuda))
  assert tuple(v.shape) == (3,) and tuple(h.shape) == (3, 7) and tuple(c.shape) == (3, 7)
  v2, _ = net(obs.reshape(3, 1, 8, 8, 3), torch.zeros(3, 1, dtype=torch.int32, device=cuda))
  assert tuple(v2.shape) == (3, 1)
  assert torch.equal(v2[:, 0], v)


def test_stacked_state_nest_and_forget_bias(cuda):
  spec = tensor_spec.TensorSpec((4,), torch.float32)
  aspec = tensor_spec.BoundedTensorSpec((2,), torch.float32, -1.0, 1.0)
  net = adrn.ActorDistributionRnnNetwork(spec, aspec, lstm_size=(7, 5), device=cuda)
  net.create_variables()
  names = [s.name for pair in net.state_spec for s in pair]
  assert names == ['network_state_%d' % i for i in range(4)]
  st = net.get_initial_state(3)
  assert [tuple(t.shape) for pair in st for t in pair] == [(3, 7), (3, 7), (3, 5), (3, 5)]
  cell = net.layers[2]
  b = cell.bias.cpu().numpy()
  assert np.all(b[7:14] == 1) and np.all(b[:7] == 0) and np.all(b[14:] == 0)
  u = cell.recurrent_kernel.cpu().numpy().astype(np.float64)
  np.testing.assert_allclose(u @ u.T, np.eye(7), atol=1e-5)
  np.testing.assert_allclose(net._std.bias.cpu().numpy(), np.log(np.expm1(0.35)), rtol=1e-6)
  with pytest.raises(NotImplementedError):
    adrn.ActorDistributionRnnNetwork(spec, aspec, lstm_size=(7,), rnn_construction_fn=len)
  with pytest.raises(NotImplementedError):
    adrn.ActorDistributionRnnNetwork(spec, aspec, lstm_size=(7,), input_dropout_layer_params=(0.1,))
  with pytest.raises(NotImplementedError):
    len_.LSTMEncodingNetwork(spec, lstm_size=(7,), preprocessing_combiner=object())


@pytest.mark.parametrize('lstm_size', [(20,), (7, 5), (150, 89)])
def test_sequence_call_matches_chained_steps(cuda, lstm_size):
  """The sequence call runs each GEMM over B*T rows, a step over B rows.  With the FFMA GEMMs
  (mode 0) a row's result does not depend on the row count, so the two agree bit for bit.  With
  the default GEMMs the B*T rows may take the 3xTF32 tensor cores and round differently: within
  1e-6 relative, 2e-6 where the 150-unit layer feeds K = 150 reductions (measured 1.1e-6)."""
  rng = np.random.RandomState(2)
  B, T, D = 4, 12, 5
  spec = tensor_spec.TensorSpec((D,), torch.float32)
  aspec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 3)
  net = adrn.ActorDistributionRnnNetwork(spec, aspec, input_fc_layer_params=(16,),
                                         lstm_size=lstm_size, output_fc_layer_params=(8,),
                                         device=cuda).set_seed(4)
  obs = torch.as_tensor(rng.randn(B, T, D).astype(f32), device=cuda)
  st = np.ones((B, T), np.int32)
  st[:, 0] = 0
  st[1, 5] = 0
  st = torch.as_tensor(st, device=cuda)

  def run():
    full, fstate = net(obs, st, net.get_initial_state(B))
    state = net.get_initial_state(B)
    outs = []
    for t in range(T):
      o, state = net(obs[:, t], st[:, t], state)
      outs.append(o)
    leaves = torch.utils._pytree.tree_leaves
    return full, torch.stack(outs, 1), leaves(fstate), leaves(state)

  full, step, fstate, state = run()
  rel = (step - full).abs().max().item() / full.abs().max().item()
  record_parity('lstm_network_chained', rel=rel)
  bar = 2e-6 if max(lstm_size) > 20 else 1e-6
  assert rel <= bar
  for a, b in zip(fstate, state):
    assert (a - b).abs().max().item() <= bar * max(1.0, b.abs().max().item())
  _lib.call('b200rl_set_gemm_mode', 0)
  try:
    full, step, fstate, state = run()
  finally:
    _lib.call('b200rl_set_gemm_mode', int(os.environ.get('B200RL_GEMM_MODE', '1')))
  assert torch.equal(step, full)
  for a, b in zip(fstate, state):
    assert torch.equal(a, b)
