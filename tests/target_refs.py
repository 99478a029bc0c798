"""float64 references for the training targets, and the metrics the target tests compare the
kernels with.

Host-only: nothing here needs a CUDA device (Out allocates on the device it is given).
test_target_kernels_gpu.py and test_agent_targets_gpu.py compare the kernels of csrc/scans.cu
and csrc/ppo.cu with these functions; test_target_metric_host.py shows that, at the bounds
below, the metrics accept the kernels' own fp32 association orders and reject the mistakes a
target test must catch.

Restated: utils/value_ops.py discounted_return :21-99 and generalized_advantage_estimation
:102-164, trajectories/trajectory.py n-step reduction :815-832, agents/ppo/ppo_agent.py discounts
:632-660 and ppo_utils.make_trajectory_mask :35-59, update_adaptive_kl_beta :1632-1675,
utils/tensor_normalizer.py parallel_variance_calculation :397-445 and normalize :134-205.

Scans.  Both are the reverse linear recurrence y_t = a_t·y_{t+1} + b_t, y_T = init.  The float64
reference also returns the condition sum S_t = Σ_{k≥t} |Π_{t≤j<k} a_j|·|b_k| + |Π_{j≥t} a_j|·|init|:
a rounding of relative size u in any term moves y_t by at most u·S_t, whatever the association
order.  For GAE, |b_k| is |r_k| + |d_k·V_{k+1}| + |V_k|, so the rounding of δ is covered.  The
scan metric is |got − ref| / (u·S_t) per element, u = 2⁻²⁴.  It is not O(1): every rounding
along the chain adds up to u·S_t, and a far term crosses one carry per 32-step tile (the
batch-major order) or one step per element (the serial order).  Both orders reach about 20·u·S_t
on rows of a few hundred steps at γ = 0.99; TOL_SCAN is set from that.
"""
import math

import numpy as np

U32 = 2.0 ** -24          # fp32 unit roundoff
f32 = np.float32
STEP_FIRST, STEP_MID, STEP_LAST = 0, 1, 2

# Bounds, each at least 4x the largest error measured on an H100 80GB HBM3 at a 700 W power limit
# (record_parity keeps the measured values); all are in units of u.
TOL_SCAN = 128.0          # scans and n-step rewards: |got − ref| / (u·S_t)
TOL_NSTEP_DISC = 2.0      # n-step discount, relative error / (u·(T + 1)) (one rounding per factor)
TOL_NORMALIZE = 16.0      # normalize: |got − ref| / (u·(|x| + |μ|)·inv)
TOL_MEAN = 128.0          # column mean: |got − ref| / (u·mean|x|)
TOL_M2 = 32.0             # centred second moment: see m2_error
TOL_COUNT = 4.0           # running count: relative error / u


def h32(x):
  """A scalar as the kernel receives it: rounded to fp32, returned as a python float."""
  return float(np.float32(x))


def f64(a):
  """float64 numpy copy of a numpy array, python number or (CUDA) torch tensor."""
  if hasattr(a, 'detach'):
    a = a.detach().cpu().numpy()
  return np.array(a, dtype=np.float64)


def bits(a):
  """The bit patterns of an fp32 array (distinguishes ±0 and NaN payloads)."""
  if hasattr(a, 'detach'):
    a = a.detach().cpu().numpy()
  return np.ascontiguousarray(a, dtype=f32).view(np.int32)


# ---- scans ---------------------------------------------------------------------------------------
def recurrence(a, b, init, bmag=None):
  """y_t = a_t·y_{t+1} + b_t over the last axis of batch-major [B, T] arrays, y_T = init [B].
  Returns (y, S) in float64; `bmag` (default |b|) is the magnitude each b_k is rounded at."""
  a, b = f64(a), f64(b)
  B, T = a.shape
  bmag = np.abs(b) if bmag is None else f64(bmag)
  y = np.empty((B, T))
  S = np.empty((B, T))
  acc = f64(init).reshape(B) if init is not None else np.zeros(B)
  cnd = np.abs(acc)
  for t in range(T - 1, -1, -1):
    acc = a[:, t] * acc + b[:, t]
    cnd = np.abs(a[:, t]) * cnd + bmag[:, t]
    y[:, t] = acc
    S[:, t] = cnd
  return y, S


def discounted_return(r, d, final=None):
  """Batch-major discounted return: (y, S)."""
  return recurrence(d, r, final)


def gae_terms(v, final, d, r, lam):
  """(a, b, |b|) of GAE in float64: a = d·λ, b = δ = r + d·V' − V with V' = V_{t+1}, and
  final at t = T-1."""
  v, d, r = f64(v), f64(d), f64(r)
  nv = np.concatenate([v[:, 1:], f64(final).reshape(-1, 1)], axis=1)
  return d * h32(lam), r + d * nv - v, np.abs(r) + np.abs(d * nv) + np.abs(v)


def gae(v, final, d, r, lam):
  """Batch-major GAE (init 0): (y, S)."""
  a, b, bmag = gae_terms(v, final, d, r, lam)
  return recurrence(a, b, None, bmag)


def scan_error(got, ref, S):
  """max over elements of |got − ref| / (u·S_t); inf on a non-finite output."""
  g = f64(got)
  if not np.isfinite(g).all():
    return math.inf
  if g.size == 0:
    return 0.0
  return float((np.abs(g - ref) / (U32 * np.maximum(S, 1e-300))).max())


# ---- the kernels' own fp32 association orders (numpy fp32 ops are IEEE round-to-nearest, like
# __fmul_rn / __fadd_rn, so these are exact restatements) ------------------------------------------
def scan_kernel_order(a, b, init, carry_lane=0, ntiles=None):
  """scan_batch_major's order: 32-step tiles walked from the end; in a tile the affine maps
  (a, b) are suffix-composed with shfl_down offsets 1, 2, 4, 8, 16 (lanes with lane + o ≥ 32
  keep their map; lanes past T hold the identity (1, 0)); y = A·carry + B; the next carry is
  lane `carry_lane`'s y.  `carry_lane` and `ntiles` exist for the host test's mutants."""
  a = np.ascontiguousarray(a, dtype=f32)
  b = np.ascontiguousarray(b, dtype=f32)
  B, T = a.shape
  carry = np.zeros(B, f32) if init is None else np.asarray(init, f32).reshape(B).copy()
  y = np.full((B, T), np.nan, f32)
  for tile in range((T + 31) // 32 - 1 if ntiles is None else ntiles - 1, -1, -1):
    lo = tile * 32
    n = min(T - lo, 32)
    ma, mb = np.ones((B, 32), f32), np.zeros((B, 32), f32)
    ma[:, :n], mb[:, :n] = a[:, lo:lo + n], b[:, lo:lo + n]
    for o in (1, 2, 4, 8, 16):
      a2, b2 = ma[:, o:].copy(), mb[:, o:].copy()
      mb[:, :32 - o] = ma[:, :32 - o] * b2 + mb[:, :32 - o]
      ma[:, :32 - o] = ma[:, :32 - o] * a2
    yt = ma * carry[:, None] + mb
    y[:, lo:lo + n] = yt[:, :n]
    carry = yt[:, carry_lane]
  return y


def gae_terms_fp32(v, final, d, r, lam):
  """(a, δ) as scan_batch_major<1> forms them: a = fp32(d·λ), δ = fp32(fp32(r + fp32(d·V')) − V)."""
  v, d, r = (np.ascontiguousarray(x, dtype=f32) for x in (v, d, r))
  nv = np.concatenate([v[:, 1:], np.asarray(final, f32).reshape(-1, 1)], axis=1)
  return d * f32(lam), (r + d * nv) - v


def discounted_return_kernel_order(r, d, final=None):
  return scan_kernel_order(d, r, final)


def gae_kernel_order(v, final, d, r, lam):
  a, delta = gae_terms_fp32(v, final, d, r, lam)
  return scan_kernel_order(a, delta, None)


# ---- n-step reduction ----------------------------------------------------------------------------
def nstep_reduce(reward, discount, gamma):
  """trajectory.py:815-832 on [B, T] rows, n = T − 1: reward = Σ_{t<n} r_t·Π_{j<t} γ·d_j, discount
  = γ^(T−2)·Π_{j<n} d_j.  γ reaches the reward kernel as fp32 and γ^(T−2) is formed in double.
  Returns (reward, S, discount) in float64."""
  r, d = f64(reward), f64(discount)
  n = r.shape[1] - 1
  y, S = recurrence(h32(gamma) * d[:, :n], r[:, :n], None)
  return y[:, 0], S[:, 0], float(gamma) ** (n - 1) * np.prod(d[:, :n], axis=1)


def rel_error_u(got, ref):
  """max |got − ref| / (u·|ref|) (0 where both are 0, inf where only ref is)."""
  g, r = f64(got), f64(ref)
  if not np.isfinite(g).all():
    return math.inf
  d = np.abs(g - r)
  with np.errstate(divide='ignore', invalid='ignore'):
    q = np.where(d == 0, 0.0, d / (U32 * np.abs(r)))
  return float(q.max()) if q.size else 0.0


# ---- PPO / REINFORCE masks and weights: exact fp32 restatements ----------------------------------
def ppo_discounts(discount, next_step_type, gamma):
  """fp32(fp32(discount·γ)·mask), mask = 0 where next_step_type is LAST (ppo_agent.py:632-660)."""
  d = np.asarray(discount, f32)
  mask = np.where(np.asarray(next_step_type) == STEP_LAST, f32(0), f32(1)).astype(f32)
  return (d * f32(gamma)) * mask


def ppo_weights(step_type, ret, adv, weights=None):
  """[weights ·] (step_type != LAST) & !(ret == 0 & adv == 0) (ppo_utils.py:35-59): the weight
  itself where valid (1 when absent), +0 elsewhere."""
  ret, adv = np.asarray(ret, f32), np.asarray(adv, f32)
  valid = (np.asarray(step_type) != STEP_LAST) & ~((ret == 0) & (adv == 0))
  w = np.ones(ret.shape, f32) if weights is None else np.asarray(weights, f32)
  return np.where(valid, w, f32(0)).astype(f32)


def kl_beta_update(mean_kl, beta, target, tol):
  """update_adaptive_kl_beta in fp32: ×1.5 when mean_kl > target·(1 + tol), ÷1.5 (as ×fp32(1/1.5))
  when mean_kl < target·(1 − tol), clipped to [10e-16, 10e16]."""
  m, b, t, tl = f32(mean_kl), f32(beta), f32(target), f32(tol)
  lo, hi = f32(t * f32(f32(1) - tl)), f32(t * f32(f32(1) + tl))
  f = f32(1)
  if m < lo:
    f = f32(f32(1) / f32(1.5))
  elif m > hi:
    f = f32(1.5)
  return f32(min(max(f32(b * f), f32(10e-16)), f32(10e16)))


# ---- moments, the streaming normaliser and normalize ---------------------------------------------
def column_moments(x):
  """Two-pass float64 moments of [rows, cols]: (mean, m2 = Σ(x − mean)², mean|x|)."""
  x = f64(x)
  mu = x.mean(axis=0)
  return mu, ((x - mu) ** 2).sum(axis=0), np.abs(x).mean(axis=0)


def mean_error(got, ref, absmean):
  """max over columns of |got − ref| / (u·mean|x|)."""
  g = f64(got)
  if not np.isfinite(g).all():
    return math.inf
  return float((np.abs(g - ref) / (U32 * np.maximum(absmean, 1e-300))).max())


def m2_error(got, ref, slack):
  """max over columns of |got − ref| / (u·ref + slack): in units of u where the mean is well
  conditioned.

  m2 is conditioned on the mean: a centre off by e moves Σ(x − c)² by rows·e², and Chan's merge
  term n_a·n_b/n_ab·Δ² by n_eff·(2|Δ|e + e²).  `slack` is that shift with e at the mean bound
  (TOL_MEAN·u·mean|x|); it is negligible unless |mean| ≫ std."""
  g = f64(got)
  if not np.isfinite(g).all():
    return math.inf
  return float((np.abs(g - ref) / (U32 * ref + slack + 1e-300)).max())


def moments_slack(rows, absmean):
  """rows·e² with e = TOL_MEAN·u·mean|x|: the m2 shift of a centre at the mean bound."""
  return rows * (TOL_MEAN * U32 * f64(absmean)) ** 2


class ChanMerge(object):
  """StreamingTensorNormalizer's running state in float64 (count starts at 1e-10), with the
  running mean|x| and the m2 slack of m2_error."""

  def __init__(self, cols):
    self.count = np.full(cols, 1e-10)
    self.avg = np.zeros(cols)
    self.m2 = np.zeros(cols)
    self.abs_sum = np.zeros(cols)
    self.slack = np.zeros(cols)

  @property
  def absmean(self):
    return self.abs_sum / np.maximum(self.count, 1.0)

  def update(self, x):
    x = f64(x)
    n_a = float(x.shape[0])
    avg_a, m2_a, abs_a = column_moments(x)
    e_b = TOL_MEAN * U32 * self.absmean
    e_a = TOL_MEAN * U32 * abs_a
    n_b = self.count
    n_ab = n_a + n_b
    delta = self.avg - avg_a
    n_eff = n_a * n_b / n_ab
    self.slack += n_a * e_a ** 2 + n_eff * (2 * np.abs(delta) * (e_a + e_b) + (e_a + e_b) ** 2)
    self.avg = avg_a + delta * n_b / n_ab
    self.m2 = self.m2 + m2_a + delta * delta * n_eff
    self.count = n_ab
    self.abs_sum += np.abs(x).sum(axis=0)


def normalize(x, mean, m2, count, eps, clip):
  """normalize_kernel in float64 on [rows, cols]: (x − μ)·inv, inv = 1/sqrt(var + eps), var =
  m2/count (m2 itself when count is None), clipped to ±clip when clip > 0.  `mean` None is the
  uncentred form.  Returns (y, M) with M = (|x| + |μ|)·inv, the scale of normalize_error: the
  kernel forms x·inv − μ·inv, whose roundings (and the rsqrtf / division / +eps ones on inv) are
  relative to |x|·inv and |μ|·inv."""
  x = f64(x)
  cols = x.shape[-1]
  mu = np.zeros(cols) if mean is None else f64(mean).reshape(cols)
  var = f64(m2).reshape(cols) if count is None else f64(m2).reshape(cols) / f64(count).reshape(cols)
  inv = 1.0 / np.sqrt(var + h32(eps))
  y = (x - mu) * inv
  if clip > 0:
    c = h32(clip)
    y = np.clip(y, -c, c)
  return y, (np.abs(x) + np.abs(mu)) * inv


def normalize_error(got, ref, M):
  """max over elements of |got − ref| / (u·M)."""
  g = f64(got)
  if not np.isfinite(g).all():
    return math.inf
  return float((np.abs(g - ref) / (U32 * np.maximum(M, 1e-300))).max())


# ---- outputs with canaries -----------------------------------------------------------------------
TAIL = 64


def _canary(n, offset=0.0):
  import torch
  return torch.arange(n, dtype=torch.float32) * 0.25 - 9.75 + offset


class Out(object):
  """A NaN-filled [rows, ld] float32 device output with canary columns [cols, ld) and a canary
  tail; check_canaries asserts the kernel wrote neither."""

  def __init__(self, cuda, rows, cols, ld=None):
    import torch
    ld = cols if ld is None else ld
    self.rows, self.cols, self.ld = rows, cols, ld
    self.buf = torch.full((rows * ld + TAIL,), float('nan'), device=cuda)
    want = self.buf.clone()
    want[rows * ld:] = _canary(TAIL).to(cuda)
    if ld > cols:
      want[:rows * ld].view(rows, ld)[:, cols:] = _canary(ld - cols, 100.0).to(cuda)
    self.buf.copy_(want)
    self.want = want

  def ptr(self):
    return self.buf.data_ptr()

  def value(self):
    return self.buf[:self.rows * self.ld].view(self.rows, self.ld)[:, :self.cols]

  def numpy(self):
    return self.value().cpu().numpy()

  def check_canaries(self, what):
    import torch
    n = self.rows * self.ld
    assert torch.equal(self.buf[n:], self.want[n:]), f'{what}: canary tail overwritten'
    if self.ld > self.cols:
      got = self.buf[:n].view(self.rows, self.ld)[:, self.cols:]
      want = self.want[:n].view(self.rows, self.ld)[:, self.cols:]
      assert torch.equal(got, want), f'{what}: canary columns past the output overwritten'
