"""fp32 dense / conv forward+backward kernels vs the numpy oracle (oracle/nn.py)."""
import numpy as np
import pytest
import torch

from agents_b200.networks import layers as L
from agents_b200.networks import q_network
from agents_b200.networks import sequential
from agents_b200.specs import tensor_spec
from oracle import nn as onn
from conftest import record_parity

pytestmark = pytest.mark.gpu
f32 = np.float32


def _close(got, want, rtol=2e-5, atol=None, tag=None):
  """Forward outputs: 2e-5 elementwise.  Gradients (`tag` given) are sums of up to 70 001 products of
  both signs: numpy sums them pairwise, the kernels in K-tile order with split-K / col2im atomics, and
  3xTF32 drops the lo*lo term (2^-22 per product), so single ELEMENTS of a cancelling sum differ by
  up to ~1e-4 of their own value while the error relative to the largest element stays near 1e-6;
  that figure is recorded per tag (gpurun_out/parity_measured.json -> profiles/) and the loss-level
  1e-5 bound of the north star is asserted in tests/test_baseline_parity_gpu.py."""
  want = np.asarray(want)
  if atol is None:
    atol = 2e-6 * max(1.0, float(np.abs(want).max()))
  got = got.cpu().numpy()
  if tag is not None:
    record_parity('nn_layers_err_rel_to_max', **{
        tag: float(np.abs(got - want).max()) / max(float(np.abs(want).max()), 1e-30)})
  np.testing.assert_allclose(got, want, rtol=rtol, atol=atol)


def _net_and_oracle(cuda, layers, input_shape, in_dtype=torch.float32):
  net = sequential.Sequential(layers, input_spec=tensor_spec.TensorSpec(input_shape, in_dtype),
                              device=cuda).set_seed(3)
  net.create_variables()
  olayers = []
  for l in net.layers:
    if isinstance(l, L.CastScale):
      olayers.append(dict(kind='cast_scale', divisor=l.divisor))
    elif isinstance(l, L.Conv2D):
      olayers.append(dict(kind='conv', w=l.kernel.cpu().numpy().copy(), b=l.bias.cpu().numpy().copy(),
                          stride=l.stride, act=l.activation))
    elif isinstance(l, L.Flatten):
      olayers.append(dict(kind='flatten'))
    elif isinstance(l, L.Dense):
      olayers.append(dict(kind='dense', w=l.kernel.cpu().numpy().copy(),
                          b=None if l.bias is None else l.bias.cpu().numpy().copy(), act=l.activation))
  return net, onn.Sequential(olayers)


@pytest.mark.parametrize('M,K,N,act', [
    (1, 4, 2, None), (64, 4, 100, 'relu'), (256, 100, 2, None), (256, 3136, 512, 'relu'),
    (256, 512, 6, None), (4096, 17, 200, 'tanh'), (1000, 200, 100, 'tanh'), (33, 65, 129, 'relu'),
    (5000, 23, 256, 'relu'), (37, 32, 20, None), (300, 8, 64, 'relu'), (70001, 17, 200, 'tanh')])
def test_dense_fwd_bwd(cuda, M, K, N, act):
  rng = np.random.RandomState(M + K + N)
  net, orc = _net_and_oracle(cuda, [L.Dense(N, activation=act)], (K,))
  x = (rng.randn(M, K) * 0.5).astype(f32)
  y, tape = net.forward_train(torch.as_tensor(x, device=cuda))
  wy, wtape = orc.forward(x, keep=True)
  _close(y, wy)
  dy = rng.randn(M, N).astype(f32)
  net.backward(tape, torch.as_tensor(dy, device=cuda))
  wg = orc.backward(wtape, dy)
  lay = net.layers[0]
  _close(lay.d_kernel, wg[0], rtol=1e-4, tag='dense_dW')
  _close(lay.d_bias, wg[1], rtol=1e-4, tag='dense_db')
  dx = lay.backward(torch.as_tensor(x, device=cuda), y, torch.as_tensor(dy, device=cuda), need_dx=True)
  wdz = onn.act_bwd(wy, dy, act)
  _close(dx, wdz @ orc.layers[0]['w'].T, rtol=1e-4, tag='dense_dX')


def test_dense_strided_batch_input(cuda):
  rng = np.random.RandomState(0)
  B, T, K, N = 37, 3, 17, 20
  net, orc = _net_and_oracle(cuda, [L.Dense(N, activation='tanh')], (K,))
  x = rng.randn(B, T, K).astype(f32)
  xt = torch.as_tensor(x, device=cuda)
  for t in range(T):
    y, tape = net.forward_train(xt[:, t])           # non-contiguous view, no copy
    _close(y, orc.forward(x[:, t]))
    dy = rng.randn(B, N).astype(f32)
    net.backward(tape, torch.as_tensor(dy, device=cuda))
    _, wtape = orc.forward(x[:, t], keep=True)
    _close(net.layers[0].d_kernel, orc.backward(wtape, dy)[0], rtol=1e-4, tag='dense_dW')


@pytest.mark.parametrize('N,H,W,C,F,ks,st,u8', [
    (2, 12, 12, 3, 8, 4, 2, True), (3, 84, 84, 4, 32, 8, 4, True), (3, 20, 20, 32, 64, 4, 2, False),
    (3, 9, 9, 64, 64, 3, 1, False), (1, 7, 9, 5, 3, 3, 2, False), (5, 10, 10, 1, 16, 3, 1, True)])
def test_conv_fwd_bwd(cuda, N, H, W, C, F, ks, st, u8):
  rng = np.random.RandomState(N * H + C)
  layers = ([L.CastScale(255.)] if u8 else []) + [L.Conv2D(F, ks, st, activation='relu')]
  net, orc = _net_and_oracle(cuda, layers, (H, W, C), torch.uint8 if u8 else torch.float32)
  conv = [l for l in net.layers if isinstance(l, L.Conv2D)][0]
  with torch.no_grad():
    conv.bias.copy_(torch.as_tensor(rng.randn(F).astype(f32) * 0.1))
  [l for l in orc.layers if l['kind'] == 'conv'][0]['b'] = conv.bias.cpu().numpy().copy()
  x = rng.randint(0, 256, size=(N, H, W, C)).astype(np.uint8) if u8 else rng.randn(N, H, W, C).astype(f32)
  y, tape = net.forward_train(torch.as_tensor(x, device=cuda))
  wy, wtape = orc.forward(x, keep=True)
  _close(y, wy)
  dy = rng.randn(*wy.shape).astype(f32)
  net.backward(tape, torch.as_tensor(dy, device=cuda))
  wg = orc.backward(wtape, dy)
  _close(conv.d_kernel, wg[0], rtol=1e-4, tag='conv_dW')
  _close(conv.d_bias, wg[1], rtol=1e-4, tag='conv_db')
  if not u8:
    dx = conv.backward(torch.as_tensor(x, device=cuda), y, torch.as_tensor(dy, device=cuda), need_dx=True)
    wdz = onn.act_bwd(wy, dy, 'relu')
    wdx, _, _ = onn.conv2d_bwd(x, orc.layers[0]['w'], wdz, st)
    _close(dx, wdx, rtol=1e-4, tag='conv_dX')


def test_conv_strided_batch_u8(cuda):
  """obs[:, t] of a [B,T,H,W,C] uint8 batch is consumed in place (x_batch_stride)."""
  rng = np.random.RandomState(1)
  B, T = 4, 2
  net, orc = _net_and_oracle(cuda, [L.CastScale(255.), L.Conv2D(8, 4, 2, activation='relu')],
                             (12, 12, 3), torch.uint8)
  x = rng.randint(0, 256, size=(B, T, 12, 12, 3)).astype(np.uint8)
  xt = torch.as_tensor(x, device=cuda)
  for t in range(T):
    y, _ = net(xt[:, t])
    _close(y, orc.forward(x[:, t]))


def test_mnih_q_network_forward_backward(cuda):
  """The Atari network of examples/dqn/mnih15/dqn_train_eval_atari.py:104-110 at batch 8."""
  rng = np.random.RandomState(5)
  obs_spec = tensor_spec.TensorSpec((84, 84, 4), torch.uint8)
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 5)
  net = q_network.QNetwork(obs_spec, act_spec, preprocessing_layers=L.CastScale(255.),
                           conv_layer_params=((32, 8, 4), (64, 4, 2), (64, 3, 1)),
                           fc_layer_params=(512,), device=cuda).set_seed(11)
  net.create_variables()
  _, orc = None, None
  olayers = []
  for l in net.layers:
    if isinstance(l, L.CastScale): olayers.append(dict(kind='cast_scale', divisor=255.0))
    elif isinstance(l, L.Conv2D): olayers.append(dict(kind='conv', w=l.kernel.cpu().numpy(), b=l.bias.cpu().numpy(), stride=l.stride, act='relu'))
    elif isinstance(l, L.Flatten): olayers.append(dict(kind='flatten'))
    else: olayers.append(dict(kind='dense', w=l.kernel.cpu().numpy(), b=l.bias.cpu().numpy(), act=l.activation))
  orc = onn.Sequential(olayers)
  assert net.flat_params.numel() >= 1686180 - 6 * 512  # ~1.69 M parameters
  x = rng.randint(0, 256, size=(8, 84, 84, 4)).astype(np.uint8)
  q, tape = net.forward_train(torch.as_tensor(x, device=cuda))
  wq, wtape = orc.forward(x, keep=True)
  _close(q, wq)
  dq = rng.randn(8, 6).astype(f32)
  net.backward(tape, torch.as_tensor(dq, device=cuda))
  wg = orc.backward(wtape, dq)
  for g, w in zip(net._grad_views, wg):
    _close(g, w, rtol=2e-4, tag='mnih_net_grads_b8')   # 4 layers deep: errors of the dX chain compound
