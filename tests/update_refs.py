"""float64 restatements of the update half of a train step, and the metrics the update tests
compare the kernels with.

Host-only: nothing here needs a CUDA device.  test_update_kernels_gpu.py and
test_agent_updates_gpu.py step these functions from the state the device held before each
launch; test_update_metric_host.py shows that, at the bounds below, the metrics reject the
mistakes an optimizer test must catch.

Every step function takes the pre-step state (parameters, slots, step counter, gradient scale)
and returns the post-step state.  Hyperparameters are rounded to fp32 first, because the kernels
receive `float`: 1 − fp32(0.999) is already 1.3e-5 away from 0.001.

Restated: TF ApplyAdam (tf.compat.v1.train.AdamOptimizer and tf.keras.optimizers.Adam use the
same rule; only the default ε differs), ApplyRMSProp / ApplyCenteredRMSProp (ms starts at 1 in
tf.compat.v1.train.RMSPropOptimizer and at 0 in tf.keras.optimizers.RMSprop), tf.clip_by_norm,
tf.clip_by_global_norm, utils/common.py soft_variables_update :250-346 and Periodically :450-507.

Gradients in the tests span 1e-6 .. 1e2 in magnitude, plus exact zeros.  They stay above ~1e-18:
below that g² (Adam's v, RMSProp's ms) falls into the fp32 subnormal range or to zero, and the
fp32 slots no longer carry the gradient that the float64 reference does.
"""
import math

import numpy as np

from grad_refs import grad_errors  # noqa: F401  (the slot metric; re-exported for the tests)

U32 = 2.0 ** -24          # fp32 unit roundoff

# Bounds, each at least 4x the largest error measured on an H100 80GB HBM3 at a 400 W power limit
# (record_parity keeps the measured values).
TOL_UPDATE = 4e-6         # update metric, well-conditioned part (see update_error); measured 9.0e-7
COND_ULPS = 8.0           # ulps allowed in the operations `cond` amplifies (powf, 1 − β^t, ms − mg²)
TOL_SLOT = 1e-6           # grad_errors (relative L2 and max) of m, v, ms, mg; measured 2.0e-7
TOL_NORM = 5e-7           # a global squared-sum norm against float64; measured 7.3e-8
TOL_CLIP = 1.5e-6         # clipped gradients and clip scales; measured 3.5e-7 (1.6 M-float segment)
TOL_POLYAK = 2.5e-7       # Polyak blend: max error over max(|target|, |source|); measured 5.3e-8


def h32(x):
  """A hyperparameter as the kernel receives it: rounded to fp32, returned as a python float."""
  return float(np.float32(x))


def f64(a):
  """float64 numpy copy of a numpy array, python number or (CUDA) torch tensor."""
  if hasattr(a, 'detach'):
    a = a.detach().cpu().numpy()
  return np.array(a, dtype=np.float64)


def gradients(rng, n, zeros=0.05):
  """fp32 gradients with log-uniform magnitudes in [1e-6, 1e2], random signs, and a fraction
  `zeros` of exact zeros."""
  g = 10.0 ** rng.uniform(-6.0, 2.0, n) * np.where(rng.rand(n) < 0.5, -1.0, 1.0)
  g[rng.rand(n) < zeros] = 0.0
  return g.astype(np.float32)


def _scaled(g, scale):
  return f64(g) * (1.0 if scale is None else h32(scale))


# ---- optimizers -----------------------------------------------------------------------------------
def adam(p, g, m, v, step, lr, beta1, beta2, eps, scale=None):
  """One ApplyAdam step from the pre-step state; `step` is the counter before the step and
  `scale` the global-norm clip scale that multiplies g (None: 1).

    t = step + 1,  lr_t = lr·sqrt(1 − β2^t) / (1 − β1^t)
    m += (g − m)(1 − β1),  v += (g² − v)(1 − β2),  p −= m·lr_t / (sqrt(v) + ε)

  Returns dict(p, m, v, step, u, cond), with p_new = p − u.  `cond` ≥ 1 is the conditioning of
  lr_t: 1 − β^t cancels at small t, so a relative error δ in the fp32 powf becomes
  δ·β^t / (1 − β^t) in 1 − β^t (half that under the square root)."""
  lr, b1, b2, eps = h32(lr), h32(beta1), h32(beta2), h32(eps)
  g = _scaled(g, scale)
  m, v = f64(m), f64(v)
  t = int(step) + 1
  b1p, b2p = b1 ** t, b2 ** t
  lr_t = lr * math.sqrt(1.0 - b2p) / (1.0 - b1p)
  m = m + (g - m) * (1.0 - b1)
  v = v + (g * g - v) * (1.0 - b2)
  u = m * lr_t / (np.sqrt(v) + eps)
  cond = 1.0 + 0.5 * b2p / (1.0 - b2p) + b1p / (1.0 - b1p)
  return dict(p=f64(p) - u, m=m, v=v, step=t, u=u, cond=cond)


def rmsprop(p, g, ms, mg, mom, lr, decay, momentum, eps, centered, scale=None):
  """One ApplyRMSProp (centered: ApplyCenteredRMSProp) step from the pre-step state:

    ms += (g² − ms)(1 − ρ);  centered: mg += (g − mg)(1 − ρ), d = ms − mg² + ε; else d = ms + ε
    mom = μ·mom + lr·g / sqrt(d),  p −= mom

  `mg` is ignored unless centered.  Returns dict(p, ms, mg, mom, u, cond), with u = mom the
  update.  `cond` is per element: κ = (ms + mg²) / (ms − mg² + ε) for the centered form, whose
  denominator cancels after many steps of near-constant gradients; 1 for the plain form."""
  lr, rho, mu, eps = h32(lr), h32(decay), h32(momentum), h32(eps)
  g = _scaled(g, scale)
  ms = f64(ms)
  ms = ms + (g * g - ms) * (1.0 - rho)
  if centered:
    mg = f64(mg)
    mg = mg + (g - mg) * (1.0 - rho)
    d = ms - mg * mg + eps
    cond = (ms + mg * mg) / d
  else:
    mg = None
    d = ms + eps
    cond = np.ones_like(ms)
  mom = f64(mom) * mu + lr * g / np.sqrt(d)
  return dict(p=f64(p) - mom, ms=ms, mg=mg, mom=mom, u=mom, cond=np.maximum(cond, 1.0))


# ---- clipping -------------------------------------------------------------------------------------
def clip_by_norm_segments(g, offsets, clip):
  """tf.clip_by_norm on each segment [offsets[i], offsets[i+1]) of the flat gradient:
  g·clip / max(‖g‖, clip).  Returns (clipped gradient, per-segment norms)."""
  g = f64(g).copy()
  clip = h32(clip)
  norms = []
  for b, e in zip(offsets[:-1], offsets[1:]):
    nrm = float(np.sqrt((g[b:e] ** 2).sum()))
    norms.append(nrm)
    if e > b:
      g[b:e] *= clip / max(nrm, clip)
  return g, np.array(norms)


def global_norm_scale(g, clip):
  """(scale, norm) of tf.clip_by_global_norm over the flat gradient: scale = clip / max(‖g‖,
  clip).  clip ≤ 0 means no clipping (scale 1), as b200rl_global_norm_scale documents."""
  nrm = float(np.sqrt((f64(g) ** 2).sum()))
  clip = h32(clip)
  return (clip / max(nrm, clip) if clip > 0 else 1.0), nrm


# ---- target networks ------------------------------------------------------------------------------
class Periodically(object):
  """utils/common.py:484-497: period None never fires; period 1 always fires and keeps no
  counter; otherwise the counter advances on every call (assign_add before tf.cond) and the body
  runs when the new count is a multiple of the period."""

  def __init__(self, period):
    self.period, self.counter = period, 0

  def __call__(self):
    if self.period is None:
      return False
    if self.period == 1:
      return True
    self.counter += 1
    return self.counter % self.period == 0


def polyak(target, source, tau):
  """soft_variables_update: (1 − τ)·target + τ·source; τ = 1 copies, τ = 0 is a no-op."""
  t, s = f64(target), f64(source)
  if tau == 0:
    return t
  if tau == 1:
    return s
  tau = h32(tau)
  return (1.0 - tau) * t + tau * s


def polyak_step(gate, target, source, tau):
  """One Periodically-gated soft update: (new target, fired)."""
  fired = gate()
  return (polyak(target, source, tau) if fired else f64(target)), fired


# ---- metrics --------------------------------------------------------------------------------------
def _allowance(cond):
  """The update bound, relative to max|u|, at conditioning `cond` (scalar or per element)."""
  return TOL_UPDATE + COND_ULPS * U32 * (np.asarray(cond, dtype=np.float64) - 1.0)


def _half_ulp(x):
  return 0.5 * np.spacing(np.abs(np.asarray(x, dtype=np.float32))).astype(np.float64)


def update_error(p_new, p, u, cond=1.0):
  """(raw, ratio) error of an updated fp32 parameter tensor against p − u_ref.

  p_new = fp32(p − u) always loses up to half an ulp of p_new, which does not depend on u; that
  much is forgiven per element.  raw = max_i max(|p_new − (p − u)| − ½ulp(p_new), 0) / max|u|.
  ratio divides each element's error by its bound TOL_UPDATE + COND_ULPS·U32·(cond_i − 1), so
  ratio ≤ 1 passes.  A tensor whose reference update is exactly 0 must not move at all."""
  pn = f64(p_new)
  if not np.isfinite(pn).all():
    return math.inf, math.inf
  ex = np.maximum(np.abs(pn - (f64(p) - u)) - _half_ulp(pn), 0.0)
  um = float(np.abs(u).max()) if u.size else 0.0
  if um == 0.0:
    bad = float(ex.max()) if ex.size else 0.0
    return (0.0, 0.0) if bad == 0.0 else (math.inf, math.inf)
  rel = ex / um
  return float(rel.max()), float((rel / _allowance(cond)).max())


def cond_error(got, ref, cond=1.0):
  """(raw, ratio) of a stored update (RMSProp's mom): max|got − ref| / max|ref|, and the same
  per element over its bound TOL_UPDATE + COND_ULPS·U32·(cond_i − 1)."""
  g = f64(got)
  if not np.isfinite(g).all():
    return math.inf, math.inf
  d = np.abs(g - ref)
  rm = float(np.abs(ref).max()) if ref.size else 0.0
  if rm == 0.0:
    return (0.0, 0.0) if float(d.max()) == 0.0 else (math.inf, math.inf)
  rel = d / rm
  return float(rel.max()), float((rel / _allowance(cond)).max())


def rel_error(got, ref):
  """|got − ref| / |ref| of a scalar (a norm or a clip scale)."""
  got, ref = float(got), float(ref)
  if not math.isfinite(got):
    return math.inf
  return abs(got - ref) / abs(ref) if ref != 0 else (0.0 if got == 0 else math.inf)


def polyak_error(got, target, source, ref):
  """max|got − ref| / max(max|target|, max|source|) of a blended target."""
  g = f64(got)
  if not np.isfinite(g).all():
    return math.inf
  scale = max(float(np.abs(f64(target)).max()), float(np.abs(f64(source)).max()), 1e-30)
  return float(np.abs(g - ref).max()) / scale


def slot_errors(got, ref):
  """The slot metric: grad_errors' (relative L2, max error over max|ref|)."""
  return grad_errors(got, ref)
