"""numpy restatement of BehavioralCloningAgent's losses and train step (TEST INFRASTRUCTURE).

Follows agents/behavioral_cloning/behavioral_cloning_agent.py: _discrete_loss
(tf.nn.sparse_softmax_cross_entropy_with_logits(labels=action - minimum, logits)),
_continuous_loss_fn (tf.losses.mse(action, prediction), the mean over the action axis, with the
prediction an ActorNetwork's scale_to_spec output or a Normal's reparameterised sample
loc + scale z), common.aggregate_losses (tf.math.multiply_no_nan(per_example, weights), the sum over
the N rows / N, plus the L2 regularisation losses) and tf_agent._apply_loss (clip_gradient_norms
per variable, then the optimiser).  The losses are computed in float64 and returned in float32;
the layers are oracle/nn.py's float32 stacks.  The Normal draws z are supplied by the caller.
"""
import numpy as np

from oracle import nn
from oracle import optim
from oracle.ppo import softplus

f32 = np.float32
LOGITS, DETERMINISTIC, NORMAL = 'logits', 'deterministic', 'normal'


def row_weights(weights, outer):
  """[N] float64 row weights of a scalar, [B] (broadcast over T) or [B, T] weight; None -> 1."""
  n = int(np.prod(outer))
  if weights is None:
    return np.ones(n)
  w = np.asarray(weights, np.float64)
  if w.size == 1:
    return np.full(n, float(w.reshape(())))
  if w.shape == tuple(outer):
    return w.reshape(n)
  return np.repeat(w, n // w.shape[0])          # [B] over [B, T]


def multiply_no_nan(x, w):
  """tf.math.multiply_no_nan: 0 where w == 0, even when x is inf or NaN."""
  with np.errstate(invalid='ignore'):
    return np.where(w == 0, 0.0, x * w)


def discrete_loss(logits, labels, weights=None):
  """logits [N, A], labels [N] (action - minimum); weights: row weights [N] or None.
  Returns (loss, per_example [N], dloss/dlogits [N, A]).  A label outside [0, A) gives a NaN
  per-example loss (its gradient row uses the clamped label)."""
  z = np.asarray(logits, np.float64)
  n, a = z.shape
  w = np.ones(n) if weights is None else np.asarray(weights, np.float64)
  labels = np.asarray(labels, np.int64)
  bad = (labels < 0) | (labels >= a)
  lab = np.clip(labels, 0, a - 1)
  with np.errstate(invalid='ignore', over='ignore'):
    m = z.max(axis=1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(z - m).sum(axis=1))
    pe = np.where(bad, np.nan, lse - z[np.arange(n), lab])
    p = np.exp(z - lse[:, None])
    onehot = np.zeros_like(z)
    onehot[np.arange(n), lab] = 1.0
    g = (w / n)[:, None] * (p - onehot)
  g[w == 0] = 0.0
  loss = multiply_no_nan(pe, w).sum() / n
  return f32(loss), pe.astype(f32), g.astype(f32)


def continuous_loss(pred, target, weights=None, amin=None, amax=None, scale=None, z=None):
  """pred [N, A]: an ActorNetwork's tanh output y (with amin/amax: a = scale_to_spec(y)), or the
  loc of a Normal (with scale and the draws z: a = loc + scale z).  Returns (loss, per_example,
  dloss/dpred, dloss/dscale or None)."""
  y = np.asarray(pred, np.float64)
  t = np.asarray(target, np.float64)
  n, a_dim = y.shape
  w = np.ones(n) if weights is None else np.asarray(weights, np.float64)
  with np.errstate(invalid='ignore', over='ignore'):
    if scale is None:
      lo, hi = np.asarray(amin, np.float64), np.asarray(amax, np.float64)
      act = 0.5 * (hi + lo) + 0.5 * (hi - lo) * y
      dmul = 0.5 * (hi - lo)
    else:
      zz = np.asarray(z, np.float64)
      act = y + np.asarray(scale, np.float64) * zz
      dmul = 1.0
    d = act - t
    pe = (d * d).mean(axis=1)
    gd = (2.0 * w / (n * a_dim))[:, None] * d
  gd[w == 0] = 0.0
  loss = multiply_no_nan(pe, w).sum() / n
  dscale = None if scale is None else (gd * zz).astype(f32)
  return f32(loss), pe.astype(f32), (dmul * gd).astype(f32), dscale


class BcOracle(object):
  """net: oracle.nn.Sequential of the cloning network's layer stack (ending at the logits, the
  tanh output of an ActorNetwork, or the Normal head's mean layer).  For NORMAL, std_bias [A] is
  the head's softplus bias and loc = tanh-squash of the mean layer to [amin, amax].
  l2: [(coef, param index in params())] kernel regularisers."""

  def __init__(self, net, kind, amin=None, amax=None, std_bias=None, minimum=0, optimizer=None,
               gradient_clipping=None, l2=()):
    self.net, self.kind, self.minimum = net, kind, int(minimum)
    self.amin = None if amin is None else np.asarray(amin, f32)
    self.amax = None if amax is None else np.asarray(amax, f32)
    self.std_bias = None if std_bias is None else np.asarray(std_bias, f32).copy()
    self.opt = optimizer or optim.AdamTF()
    self.clip, self.l2 = gradient_clipping, list(l2)

  def params(self):
    return self.net.params() + ([self.std_bias] if self.kind == NORMAL else [])

  def loss_and_grads(self, obs, action, weights=None, z=None, outer=None):
    """obs [N, ...], action [N] (discrete) or [N, A]; weights as row_weights(weights, outer).
    Returns (total loss, per_example [N], gradients aligned with params())."""
    obs = np.asarray(obs)
    n = obs.shape[0]
    w = row_weights(weights, outer or (n,))
    out, tape = self.net.forward(obs, keep=True)
    if self.kind == LOGITS:
      loss, pe, g = discrete_loss(out, np.asarray(action).reshape(n) - self.minimum, w)
      grads = self.net.backward(tape, g)
    elif self.kind == DETERMINISTIC:
      loss, pe, g, _ = continuous_loss(out, action, w, self.amin, self.amax)
      grads = self.net.backward(tape, g)
    else:
      mag, mid = f32(0.5) * (self.amax - self.amin), f32(0.5) * (self.amax + self.amin)
      th = np.tanh(out).astype(f32)
      loc = (mid + mag * th).astype(f32)
      scale = np.broadcast_to(softplus(self.std_bias), loc.shape)
      loss, pe, dloc, dscale = continuous_loss(loc, action, w, scale=scale, z=z)
      dm = (dloc * mag * (f32(1) - th * th)).astype(f32)
      sig = (1.0 / (1.0 + np.exp(-self.std_bias.astype(np.float64))))
      grads = self.net.backward(tape, dm) + [(dscale.astype(np.float64) * sig).sum(0).astype(f32)]
    params = self.params()
    for coef, i in self.l2:
      loss = f32(loss + f32(coef) * np.sum(params[i].astype(np.float64) ** 2))
      grads[i] = (grads[i] + f32(2 * coef) * params[i]).astype(f32)
    return f32(loss), pe, grads

  def train(self, obs, action, weights=None, z=None, outer=None):
    loss, pe, grads = self.loss_and_grads(obs, action, weights, z, outer)
    if self.clip is not None:
      grads = [optim.clip_by_norm(g, self.clip) for g in grads]
    self.opt.apply(self.params(), grads)
    return loss, pe
