"""LSTM sequence kernels (csrc/lstm.cu) and the recurrent networks against float64.

Kernels: the forward (outputs, gates, c, consumed h, final state) within 2e-5 relative of
oracle/lstm.py in float64, and the backward (dG) plus the layer's dW, dU, db and dx within 1e-4,
over H covering every cluster size the launcher picks, T up to 1001, B across the tile boundary and
four reset patterns.  Networks: the reference's structure tests and [B, T] == T chained [B, 1]
calls."""
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
  import ctypes
  cs, rows = ctypes.c_int(), ctypes.c_int()
  _lib.call('b200rl_lstm_plan', B, H, ctypes.byref(cs), ctypes.byref(rows), None, None, None,
            None, None)
  return cs.value, rows.value


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


@pytest.mark.parametrize('B,T,H', CASES)
@pytest.mark.parametrize('pattern', ['none', 'first', 'random', 'every'])
def test_lstm_seq_kernels_match_float64(cuda, B, T, H, pattern):
  if T == 1001 and pattern in ('none', 'every'):
    pytest.skip('long sequences run the first-step and random reset patterns')
  fwd, bwd = _run(cuda, B, T, 11, H, pattern, seed=B * 1000 + H + T)
  record_parity('lstm_seq_fwd', **{k + '_rel': v for k, v in fwd.items()})
  record_parity('lstm_seq_bwd', **{k + '_rel': v for k, v in bwd.items()})
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


@pytest.mark.parametrize('lstm_size', [(20,), (7, 5)])
def test_sequence_call_matches_chained_steps(cuda, lstm_size):
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
  full, fstate = net(obs, st, net.get_initial_state(B))
  state = net.get_initial_state(B)
  outs = []
  for t in range(T):
    o, state = net(obs[:, t], st[:, t], state)
    outs.append(o)
  step = torch.stack(outs, 1)
  rel = (step - full).abs().max().item() / full.abs().max().item()
  record_parity('lstm_network_chained', rel=rel)
  assert rel <= 1e-6
  for a, b in zip(torch.utils._pytree.tree_leaves(fstate), torch.utils._pytree.tree_leaves(state)):
    assert (a - b).abs().max().item() <= 1e-6 * max(1.0, b.abs().max().item())
