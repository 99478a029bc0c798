"""oracle/lstm.py against float64 torch autograd of a hand-written LSTM cell loop: forward,
final state and BPTT with resets at t = 0, mid-row and on every step, stacked (7, 5) cells, and a
given or zero initial state."""
import numpy as np
import pytest
import torch

from oracle import lstm as olstm


def _torch_loop(x, cells, st, state):
  B, T, _ = x.shape
  outs = x
  finals = []
  for l, (W, U, b) in enumerate(cells):
    H = U.shape[0]
    h, c = (torch.zeros(B, H, dtype=torch.float64), torch.zeros(B, H, dtype=torch.float64)) \
        if state is None else state[l]
    hs = []
    for t in range(T):
      keep = torch.as_tensor(st[:, t] != 0, dtype=torch.float64)[:, None]
      h, c = h * keep, c * keep
      z = outs[:, t] @ W + b + h @ U
      i, f, g, o = torch.sigmoid(z[:, :H]), torch.sigmoid(z[:, H:2 * H]), torch.tanh(
          z[:, 2 * H:3 * H]), torch.sigmoid(z[:, 3 * H:])
      c = f * c + i * g
      h = o * torch.tanh(c)
      hs.append(h)
    outs = torch.stack(hs, 1)
    finals.append((h, c))
  return outs, finals


@pytest.mark.parametrize('sizes', [(6,), (7, 5)])
@pytest.mark.parametrize('pattern', ['first', 'mid', 'every'])
@pytest.mark.parametrize('given_state', [False, True])
def test_oracle_matches_autograd(sizes, pattern, given_state):
  rng = np.random.RandomState(len(sizes) * 10 + len(pattern))
  B, T, In = 3, 9, 4
  st = np.ones((B, T), np.int32)
  if pattern == 'first':
    st[:, 0] = 0
  elif pattern == 'mid':
    st[0, 4] = 0
    st[2, 1] = 0
  else:
    st[:] = 0
  cells, dims = [], In
  for H in sizes:
    cells.append([rng.randn(dims, 4 * H) * 0.5, rng.randn(H, 4 * H) * 0.5, rng.randn(4 * H) * 0.3])
    dims = H
  x = rng.randn(B, T, In)
  state = [(rng.randn(B, H) * 0.5, rng.randn(B, H) * 0.5) for H in sizes] if given_state else None
  dh = rng.randn(B, T, sizes[-1])
  out, finals, caches = olstm.stacked_forward(x, cells, st, state)
  dx, grads = olstm.stacked_backward(caches, dh)

  tx = torch.tensor(x, requires_grad=True)
  tcells = [[torch.tensor(p, requires_grad=True) for p in c] for c in cells]
  tstate = None if state is None else [tuple(torch.tensor(s) for s in p) for p in state]
  tout, tfinals = _torch_loop(tx, tcells, st, tstate)
  (tout * torch.tensor(dh)).sum().backward()
  np.testing.assert_allclose(out, tout.detach().numpy(), rtol=1e-12, atol=1e-12)
  for (h, c), (th, tc) in zip(finals, tfinals):
    np.testing.assert_allclose(h, th.detach().numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(c, tc.detach().numpy(), rtol=1e-12, atol=1e-12)
  np.testing.assert_allclose(dx, tx.grad.numpy(), rtol=1e-10, atol=1e-12)
  for g, tc in zip(grads, tcells):
    for a, b in zip(g, tc):
      np.testing.assert_allclose(a, b.grad.numpy(), rtol=1e-10, atol=1e-12)
