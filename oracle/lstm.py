"""numpy restatement of the LSTM sequence layer (TEST INFRASTRUCTURE).

keras LSTMCell (implementation=2): z = x W + b + h_{t-1} U with gate columns i, f, g, o;
i, f, o = sigmoid, g = tanh; c_t = f c_{t-1} + i g; h_t = o tanh(c_t).  tf_agents' DynamicUnroll
(keras_layers/dynamic_unroll_layer.py) resets the state to zero at every step whose step_type is
FIRST.  Stacked cells (StackedRNNCells) run layer by layer over the whole sequence: layer l at
step t reads layer l-1 at step t and layer l at step t-1 only.
Every function keeps the dtype of its inputs, so the same code gives the float32 oracle and the
float64 reference the kernels are checked against.
"""
import numpy as np

from oracle import nn

STEP_FIRST = 0


def sigmoid(z):
  return 1 / (1 + np.exp(-z))


def lstm_forward(x, W, U, b, step_type, h0=None, c0=None):
  """x [B, T, In] -> (h [B, T, H], (h_T, c_T), cache).  h0 / c0 [B, H] (None: zeros)."""
  B, T, _ = x.shape
  H = U.shape[0]
  dt = np.result_type(x, W)
  h = np.zeros((B, H), dt) if h0 is None else np.asarray(h0, dt)
  c = np.zeros((B, H), dt) if c0 is None else np.asarray(c0, dt)
  xw = x @ W + b
  hs = np.zeros((B, T, H), dt)
  gates = np.zeros((B, T, 4 * H), dt)
  cs = np.zeros((B, T, H), dt)
  h_used = np.zeros((B, T, H), dt)
  c_prev = np.zeros((B, T, H), dt)
  for t in range(T):
    keep = (step_type[:, t] != STEP_FIRST)[:, None].astype(dt)
    h, c = h * keep, c * keep
    z = xw[:, t] + h @ U
    i, f, g, o = sigmoid(z[:, :H]), sigmoid(z[:, H:2 * H]), np.tanh(z[:, 2 * H:3 * H]), sigmoid(z[:, 3 * H:])
    h_used[:, t], c_prev[:, t] = h, c
    c = f * c + i * g
    h = o * np.tanh(c)
    hs[:, t], cs[:, t] = h, c
    gates[:, t] = np.concatenate([i, f, g, o], 1)
  cache = dict(x=x, W=W, U=U, step_type=step_type, gates=gates, c=cs, c_prev=c_prev,
               h_used=h_used)
  return hs, (h, c), cache


def lstm_backward(cache, dh):
  """BPTT from dh [B, T, H] -> (dx, dW, dU, db, dG).  No gradient crosses a reset step, and none
  reaches the initial state."""
  gates, cs, c_prev, st = cache['gates'], cache['c'], cache['c_prev'], cache['step_type']
  B, T, H = dh.shape
  U = cache['U']
  dG = np.zeros_like(gates)
  dh_rec = np.zeros((B, H), dh.dtype)
  dc_rec = np.zeros((B, H), dh.dtype)
  for t in range(T - 1, -1, -1):
    i, f, g, o = (gates[:, t, k * H:(k + 1) * H] for k in range(4))
    tc = np.tanh(cs[:, t])
    dht = dh[:, t] + dh_rec
    dct = dc_rec + dht * o * (1 - tc * tc)
    dz = np.concatenate([dct * g * i * (1 - i), dct * c_prev[:, t] * f * (1 - f),
                         dct * i * (1 - g * g), dht * tc * o * (1 - o)], 1)
    dG[:, t] = dz
    keep = (st[:, t] != STEP_FIRST)[:, None].astype(dh.dtype)
    dh_rec = (dz @ U.T) * keep
    dc_rec = dct * f * keep
  x = cache['x']
  In = x.shape[-1]
  g2 = dG.reshape(B * T, 4 * H)
  dx = (g2 @ cache['W'].T).reshape(B, T, In)
  dW = x.reshape(B * T, In).T @ g2
  dU = cache['h_used'].reshape(B * T, H).T @ g2
  db = g2.sum(0)
  return dx, dW, dU, db, dG


def stacked_forward(x, cells, step_type, state=None):
  """cells: [(W, U, b)] per layer; state: [(h0, c0)] per layer or None.  Returns
  (h_top [B, T, H_last], [(h_T, c_T)] per layer, caches)."""
  caches, finals = [], []
  for l, (W, U, b) in enumerate(cells):
    h0, c0 = (None, None) if state is None else state[l]
    x, fin, cache = lstm_forward(x, W, U, b, step_type, h0, c0)
    caches.append(cache)
    finals.append(fin)
  return x, finals, caches


def stacked_backward(caches, dh):
  """Returns (dx, [(dW, dU, db)] per layer)."""
  grads = [None] * len(caches)
  for l in range(len(caches) - 1, -1, -1):
    dh, dW, dU, db, _ = lstm_backward(caches[l], dh)
    grads[l] = (dW, dU, db)
  return dh, grads


def _dense_stack_fwd(layers, x):
  tape = []
  for l in layers:
    y = nn.dense_fwd(x, l['w'], l['b'], l.get('act'))
    tape.append((x, y))
    x = y
  return x, tape


def _dense_stack_bwd(layers, tape, dy):
  """Returns (dx, grads aligned with the layers' [w, b] params)."""
  grads = []
  for l, (x, y) in zip(reversed(layers), reversed(tape)):
    dx, dw, db = nn.dense_bwd(x, l['w'], nn.act_bwd(y, dy, l.get('act')))
    grads = [dw, db] + grads
    dy = dx
  return dy, grads


class RnnNet(object):
  """Dense stack -> stacked LSTM -> Dense stack over [B, T] sequences, with the interface of
  oracle.nn.Sequential (forward(x [B*T, D], keep) / backward(tape, dy) / params()), so PPOOracle
  trains it unchanged.  pre / post: lists of {'w', 'b', 'act'} dense layers; cells: [W, U, b]
  per LSTM layer.  `step_type` [B, T] must be set before each forward: the rows of x are the B*T
  steps in batch-major order, and every sequence starts from the zero state."""

  def __init__(self, pre, cells, post):
    self.pre, self.cells, self.post = pre, [list(c) for c in cells], post
    self.step_type = None

  def params(self):
    out = [p for l in self.pre for p in (l['w'], l['b'])]
    out += [p for c in self.cells for p in c]
    return out + [p for l in self.post for p in (l['w'], l['b'])]

  def forward(self, x, keep=False):
    B, T = self.step_type.shape
    y, ptape = _dense_stack_fwd(self.pre, x)
    hs, _, caches = stacked_forward(y.reshape(B, T, -1), self.cells, self.step_type)
    out, otape = _dense_stack_fwd(self.post, hs.reshape(B * T, -1))
    return (out, (ptape, caches, otape)) if keep else out

  def backward(self, tape, dy):
    ptape, caches, otape = tape
    B, T = self.step_type.shape
    dh, gpost = _dense_stack_bwd(self.post, otape, dy)
    dx, cgrads = stacked_backward(caches, dh.reshape(B, T, -1))
    _, gpre = _dense_stack_bwd(self.pre, ptape, dx.reshape(B * T, -1))
    return gpre + [g for cg in cgrads for g in cg] + gpost
