"""float64 references for the policy / value loss kernels, and the metrics their tests use.

Host-only: nothing here needs a CUDA device.  test_loss_kernels_gpu.py compares the kernels of
csrc/ppo.cu (ppo_loss, ppo_kl and their categorical twins, categorical_logp), csrc/reinforce.cu
(reinforce_loss) and csrc/cql.cu (cql_loss) with these functions; test_loss_metric_host.py shows
that, at the bounds below, the metrics accept the kernels' own fp32 association orders and reject
the mistakes a loss test must catch.

Restated: agents/ppo/ppo_agent.py policy_gradient_loss :1329-1512, value_estimation_loss
:1203-1327, entropy_regularization_loss :1159-1201, kl_penalty_loss :1514-1630;
agents/reinforce/reinforce_agent.py :48-80, :327-567; agents/cql/cql_sac_agent.py _cql_loss
:534-679.  The branch rules are the kernels' own: the `obj <= obj_c` choice, a zero derivative
outside the ratio clip and outside the logp clip, the value clip taken only when err_c > err, the
clip fraction as the unweighted count of |ratio - 1| > eps over N.

Metrics.  Every reference also returns a condition magnitude per output: the sum of the absolute
values of the terms that form it, each scaled by its own relative condition (a rounding of
relative size u anywhere in the kernel's computation moves the output by at most about u times
that magnitude, whatever the association order).  A sum over rows is measured in units of
u·Σ|term_i|/denom, a per-row output in units of u·(its own magnitude): there is no batch-wide
floor, so a wrong small element cannot hide behind a large one.

Probabilities below the fp32 normal range carry an absolute error up to 2^-126 (the kernels' expf
underflows there), so p's magnitude includes that floor (TINY_P); the products it enters are capped
at |log p| <= 1e3, since a p that underflows completely is exactly 0 in the kernel.
"""
import math

import numpy as np

U32 = 2.0 ** -24                    # fp32 unit roundoff
f32 = np.float32
LOG2PI = math.log(2 * math.pi)
EPS_F32 = 1.1920928955078125e-07   # np.finfo(np.float32).eps, REINFORCE's D = sigma + eps
MASKED = -3.4028235e38              # CategoricalProjectionNetwork's logit for a masked action
STEP_LAST = 2
TINY_P = 2.0 ** -126 / U32          # absolute error of an fp32 probability below the normal range

# Bounds, in units of u, from the kernels' operation counts (the measured values are kept by
# record_parity; each is far below its bound).
#
# TOL_SUM, a loss over rows: one thread's serial sum over at most 8 grid-stride passes (524 288 rows
# / 67 584 threads), the 5-level warp tree, the 3-level tree over 8 warps, the 9-level tree over
# 512 partials, the division by denom and a coefficient: 27 roundings of partial sums bounded by
# Σ|term|, plus the per-row roundings the magnitudes carry (at most 4 per term), about 31 at worst;
# doubled.  REINFORCE's loss stage has the same depth.
TOL_SUM = 64.0
# TOL_ELEM, a per-row output (gradient element, log-prob, per-row KL): the longest chain is a
# row's serial sum over its action dimensions or strided columns (17 for the Normal head's A = 17;
# ceil(300/32) + 5 shuffle levels = 15 for a G = 32 row) plus at most 10 roundings after it
# (ratio, the products of the gradient); doubled.
TOL_ELEM = 64.0
# TOL_DV_NORM, REINFORCE's stage-5 dV: the products over g, g_bar, S and sigma (each a full
# reduction) add TOL_SUM's depth to the row's chain.
TOL_DV_NORM = 128.0


def h32(x):
  """A scalar as the kernel receives it: rounded to fp32, returned as a python float."""
  return float(np.float32(x))


def f64(a):
  """float64 numpy copy of a numpy array, python number or (CUDA) torch tensor."""
  if hasattr(a, 'detach'):
    a = a.detach().cpu().numpy()
  return np.array(a, dtype=np.float64)


def bits(a):
  if hasattr(a, 'detach'):
    a = a.detach().cpu().numpy()
  return np.ascontiguousarray(a, dtype=f32).view(np.int32)


# ---- metrics -------------------------------------------------------------------------------------
def elem_error(got, ref, cond):
  """max over elements of |got − ref| / (u·cond); inf on a non-finite output.  An element the
  reference says is exactly 0 with 0 magnitude must be exactly 0."""
  g = f64(got)
  if not np.isfinite(g).all():
    return math.inf
  if g.size == 0:
    return 0.0
  d = np.abs(g - f64(ref))
  c = U32 * f64(cond)
  with np.errstate(divide='ignore', invalid='ignore'):
    q = np.where(d == 0, 0.0, d / c)
  return float(q.max())


def sum_error(got, ref, cond):
  """A scalar loss: |got − ref| / (u·cond), cond = Σ|term_i| / denom as the reference gives it."""
  return elem_error(np.asarray([got]), np.asarray([ref]), np.asarray([cond]))


# ---- Normal head ---------------------------------------------------------------------------------
def normal_terms(loc, scale, action):
  """Per-row log-prob and entropy of the diagonal Normal with their magnitudes, and the per-element
  pieces the gradients use."""
  loc, scale, action = f64(loc), f64(scale), f64(action)
  d = action - loc
  inv = 1.0 / scale
  z = d * inv
  lsg = np.log(scale)
  c = 0.5 * LOG2PI
  logp = (-0.5 * z * z - lsg - c).sum(axis=1)
  # z = d / s carries two roundings, z² three: 3·z²/2 covers them
  cl = (1.5 * z * z + np.abs(lsg) + c).sum(axis=1)
  ent = (0.5 + c + lsg).sum(axis=1)
  ce = (0.5 + c + np.abs(lsg)).sum(axis=1)
  return dict(d=d, inv=inv, logp=logp, cl=cl, ent=ent, ce=ce)


def normal_kl(old_loc, old_scale, loc, scale):
  """Per-element KL(Normal(old) || Normal(new)) in TFP's closed form, with its magnitude.  The
  closed form cancels (expm1(2d)/2 − d ≈ d²), so the magnitude keeps every piece."""
  mo, so, mu, s = f64(old_loc), f64(old_scale), f64(loc), f64(scale)
  lso, ls = np.log(so), np.log(s)
  d = lso - ls
  z = mo / s - mu / s
  kl = 0.5 * z * z + 0.5 * np.expm1(2 * d) - d
  ck = (np.abs(z) * (np.abs(mo) + np.abs(mu)) / s * 2 + 0.5 * z * z + 0.5 * np.abs(np.expm1(2 * d)) +
        (np.exp(2 * d) + 1) * (np.abs(lso) + np.abs(ls)) + np.abs(d))
  return kl, ck


# ---- PPO: the surrogate / value / entropy terms shared by both heads -----------------------------
def _ppo_rows(logp, cl, ent, ce, old_logp, adv, ret, v, v_old, w, clip_eps, value_clip, logp_clip):
  old, A, R, V, W = f64(old_logp), f64(adv), f64(ret), f64(v), f64(w)
  eps, vcl, L = h32(clip_eps), h32(value_clip), h32(logp_clip)
  lp, dlp, clp = logp.copy(), np.ones_like(logp), cl.copy()
  if L > 0:
    out = (logp < -L) | (logp > L)
    lp = np.clip(logp, -L, L)
    dlp = np.where(out, 0.0, 1.0)
    clp = np.where(out, 0.0, cl)
  x = lp - old
  ratio = np.exp(x)
  cr = ratio * (clp + np.abs(old) + np.abs(x) + 2)          # exp's argument and exp itself
  lo, hi = 1.0 - eps, 1.0 + eps
  outside = (ratio < lo) | (ratio > hi)
  if eps > 0:
    rc = np.clip(ratio, lo, hi)
    obj, obj_c = ratio * A, rc * A
    pg = -np.minimum(obj, obj_c)
    dobj = np.where(obj <= obj_c, A, np.where(outside, 0.0, A))
    clipped = (np.abs(ratio - 1.0) > eps).astype(np.float64)
    cpg = np.abs(A) * (cr + hi)
  else:
    pg, dobj, clipped = -ratio * A, A.copy(), np.zeros_like(ratio)
    cpg = np.abs(A) * cr
  e = R - V
  err, derr = e * e, -2 * e
  cv = np.abs(R) + np.abs(V)
  if vcl > 0:
    vo = f64(v_old)
    dvv = V - vo
    vc = vo + np.clip(dvv, -vcl, vcl)
    ec = R - vc
    take = ec * ec > err
    err = np.where(take, ec * ec, err)
    dout = (dvv < -vcl) | (dvv > vcl)
    derr = np.where(take, np.where(dout, 0.0, -2 * ec), derr)
    cv = cv + np.abs(vo) + np.abs(vc)
  cve = 2 * np.sqrt(err) * cv + err
  return dict(ratio=ratio, cr=cr, dlp=dlp, dobj=dobj, pg=pg, cpg=cpg, err=err, derr=derr, cv=cv,
              cve=cve, clipped=clipped, outside=outside, x=x, lp=lp, w=W)


def _ppo_losses(r, ent, ce, N, T, global_batch, vf_coef, ent_coef, kl_terms):
  w = r['w']
  den = float(np.float32(T) * np.float32(global_batch))
  vf, ec = h32(vf_coef), h32(ent_coef)
  sums = np.array([(r['pg'] * w).sum(), (r['err'] * w).sum(), (-ent * w).sum(), r['clipped'].sum()])
  conds = np.array([(r['cpg'] * np.abs(w)).sum(), (r['cve'] * np.abs(w)).sum(), (ce * np.abs(w)).sum(), 0])
  kl = 0.0 if kl_terms is None else h32(kl_terms[0]) + h32(kl_terms[1])
  ckl = 0.0 if kl_terms is None else abs(h32(kl_terms[0])) + abs(h32(kl_terms[1]))
  pg, ve, en = sums[0] / den, vf * sums[1] / den, ec * sums[2] / den
  losses = np.array([pg, ve, en, sums[3] / N, pg + ve + en + kl, kl])
  c = np.array([conds[0] / den, abs(vf) * conds[1] / den, abs(ec) * conds[2] / den, 0.0])
  lconds = np.array([c[0], c[1], c[2], 0.0, c[0] + c[1] + c[2] + ckl, ckl])
  return den, sums, conds, losses, lconds


def ppo_loss(loc, scale, action, old_logp, adv, ret, v, v_old, w, T, global_batch, clip_eps,
             value_clip, vf_coef, ent_coef, logp_clip, kl=None):
  """b200rl_ppo_loss in float64.  kl: None or dict(old_loc, old_scale, terms[3], grad_scale).
  Returns a dict: sums[4] (the four partial sums), losses[6], dloc, dscale, dv, each with its
  magnitude (c_*), and the per-row internals (ratio, dobj, ...)."""
  nt = normal_terms(loc, scale, action)
  N = nt['logp'].shape[0]
  r = _ppo_rows(nt['logp'], nt['cl'], nt['ent'], nt['ce'], old_logp, adv, ret, v, v_old, w,
                clip_eps, value_clip, logp_clip)
  den, sums, conds, losses, lconds = _ppo_losses(r, nt['ent'], nt['ce'], N, T, global_batch, vf_coef,
                                                  ent_coef, None if kl is None else kl['terms'])
  w = r['w']
  ec, vf = h32(ent_coef), h32(vf_coef)
  g_logp = -r['dobj'] * r['ratio'] * r['dlp'] * w / den
  cg = np.abs(r['dobj'] * w / den) * r['dlp'] * (r['cr'] + r['ratio'])
  g_ent = -ec * w / den
  d, inv = nt['d'], nt['inv']
  dloc = g_logp[:, None] * d * inv * inv
  dscale = g_logp[:, None] * (d * d * inv ** 3 - inv) + g_ent[:, None] * inv
  c_dloc = cg[:, None] * np.abs(d) * inv * inv * 2
  c_dscale = cg[:, None] * (d * d * inv ** 3 + inv) * 2 + np.abs(g_ent)[:, None] * inv * 2
  if kl is not None:
    g_kl = h32(kl['terms'][2]) * h32(kl['grad_scale']) * w
    mu, so = f64(loc), f64(kl['old_scale'])
    dm = f64(kl['old_loc']) - mu
    dloc += g_kl[:, None] * (-dm * inv * inv)
    dscale += g_kl[:, None] * (inv - (dm * dm + so * so) * inv ** 3)
    c_dloc += np.abs(g_kl)[:, None] * np.abs(dm) * inv * inv * 3
    c_dscale += np.abs(g_kl)[:, None] * (inv + (dm * dm + so * so) * inv ** 3) * 3
  dv = vf * r['derr'] * w / den
  c_dv = abs(vf) * np.abs(w) / den * 2 * r['cv'] * 2
  return dict(sums=sums, c_sums=conds, losses=losses, c_losses=lconds, dloc=dloc, c_dloc=c_dloc,
              dscale=dscale, c_dscale=c_dscale, dv=dv, c_dv=c_dv, denom=den, g_logp=g_logp,
              logp=nt['logp'], **{k: r[k] for k in ('ratio', 'dobj', 'dlp', 'clipped', 'x', 'lp')})


def ppo_kl(loc, scale, old_loc, old_scale, w, out_scale):
  """b200rl_ppo_kl: per-row weighted KL(old || new) and out_scale·Σ, with magnitudes."""
  kl, ck = normal_kl(old_loc, old_scale, loc, scale)
  W = np.ones(kl.shape[0]) if w is None else f64(w)
  row = kl.sum(axis=1) * W
  crow = ck.sum(axis=1) * np.abs(W)
  s = h32(out_scale)
  return dict(kl=row, c_kl=crow, total=row.sum() * s, c_total=crow.sum() * abs(s))


# ---- Categorical head ----------------------------------------------------------------------------
def softmax_terms(z):
  """Max-subtracted log-softmax of [N, A] logits (MASKED entries allowed) with magnitudes:
  lp = log p, p, ent, and their conditions (cls: log s; clp: log p_j; cp: p_j, absolute)."""
  z = f64(z)
  m = z.max(axis=1, keepdims=True)
  d = z - m
  e = np.exp(d)
  s = e.sum(axis=1, keepdims=True)
  ls = np.log(s)
  p = e / s
  pd = p * np.abs(d)                                   # 0 where p underflows (d finite)
  spd = pd.sum(axis=1, keepdims=True)
  t = (e * d).sum(axis=1, keepdims=True)
  ent = ls - t / s
  cls = spd + 1 + np.abs(ls)
  lp = d - ls
  clp = np.abs(d) + cls
  cp = p * (clp + 1) + TINY_P
  cent = cls + (pd * (np.abs(d) + 2)).sum(axis=1, keepdims=True) + spd * (spd + 1) + np.abs(ent)
  return dict(d=d, p=p, lp=lp, ent=ent[:, 0], cls=cls[:, 0], clp=clp, cp=cp, cent=cent[:, 0])


def categorical_logp(z, action):
  st = softmax_terms(z)
  n = np.arange(st['p'].shape[0])
  a = np.asarray(action)
  return st['lp'][n, a], st['clp'][n, a]


def categorical_kl(old_logits, logits, w=None):
  """Per-row KL(Categorical(old) || Categorical(new)) = Σ_j q_j (log q_j − log p_j) over q_j > 0,
  weighted, with its magnitude."""
  so, sn = softmax_terms(old_logits), softmax_terms(logits)
  q = so['p']
  diff = np.where(q > 0, so['lp'] - sn['lp'], 0.0)
  kl = (q * diff).sum(axis=1)
  capped = np.minimum(np.abs(diff), 1e3)
  ck = (so['cp'] * capped + q * (so['clp'] + sn['clp'])).sum(axis=1)
  W = np.ones(kl.shape[0]) if w is None else f64(w)
  return kl * W, ck * np.abs(W)


def ppo_kl_categorical(logits, old_logits, w, out_scale):
  kl, ck = categorical_kl(old_logits, logits, w)
  s = h32(out_scale)
  return dict(kl=kl, c_kl=ck, total=kl.sum() * s, c_total=ck.sum() * abs(s))


def ppo_loss_categorical(logits, action, old_logp, adv, ret, v, v_old, w, T, global_batch, clip_eps,
                         value_clip, vf_coef, ent_coef, logp_clip, kl=None):
  """b200rl_ppo_loss_categorical in float64 (kl: None or dict(old_logits, terms, grad_scale)):
  dL/dz_j = g_logp (1[j=a] − p_j) + g_ent (−p_j (log p_j + H)) + g_kl (p_j − q_j)."""
  st = softmax_terms(logits)
  N, A = st['p'].shape
  n = np.arange(N)
  act = np.asarray(action)
  logp, cl = st['lp'][n, act], st['clp'][n, act]
  r = _ppo_rows(logp, cl, st['ent'], st['cent'], old_logp, adv, ret, v, v_old, w, clip_eps,
                value_clip, logp_clip)
  den, sums, conds, losses, lconds = _ppo_losses(r, st['ent'], st['cent'], N, T, global_batch,
                                                  vf_coef, ent_coef, None if kl is None else kl['terms'])
  w = r['w']
  ec, vf = h32(ent_coef), h32(vf_coef)
  g_logp = -r['dobj'] * r['ratio'] * r['dlp'] * w / den
  cg = np.abs(r['dobj'] * w / den) * r['dlp'] * (r['cr'] + r['ratio'])
  g_ent = -ec * w / den
  onehot = np.zeros((N, A))
  onehot[n, act] = 1.0
  p, lp, ent = st['p'], st['lp'], st['ent'][:, None]
  lpe = np.where(p > 0, lp + ent, 0.0)
  dz = g_logp[:, None] * (onehot - p) + g_ent[:, None] * (-p * lpe)
  c_lpe = np.minimum(np.abs(lp + ent), 1e3)
  c_dz = (cg[:, None] * (onehot + p) + np.abs(g_logp)[:, None] * st['cp'] +
          np.abs(g_ent)[:, None] * (st['cp'] * c_lpe + p * (st['clp'] + st['cent'][:, None] + c_lpe)))
  if kl is not None:
    so = softmax_terms(kl['old_logits'])
    g_kl = h32(kl['terms'][2]) * h32(kl['grad_scale']) * w
    dz += g_kl[:, None] * (p - so['p'])
    c_dz += np.abs(g_kl)[:, None] * (st['cp'] + so['cp'] + p + so['p'])
  dv = vf * r['derr'] * w / den
  c_dv = abs(vf) * np.abs(w) / den * 2 * r['cv'] * 2
  return dict(sums=sums, c_sums=conds, losses=losses, c_losses=lconds, dlogits=dz, c_dlogits=c_dz,
              dv=dv, c_dv=c_dv, denom=den, logp=logp, c_logp=cl, g_logp=g_logp,
              **{k: r[k] for k in ('ratio', 'dobj', 'dlp', 'clipped', 'x', 'lp')})


# ---- REINFORCE -----------------------------------------------------------------------------------
def reinforce_loss(params, action, ret, value, step_type, next_step_type, weights, use_advantage,
                   normalize, entropy_coef, value_coef, discrete):
  """b200rl_reinforce_loss in float64, all five stages.  params: (loc, scale) or logits [N, A];
  ret / value / step types / weights [B, T].  Returns the per-trajectory last index, the valid
  mask, num_episodes, mean / sigma / D, losses[6], the parameter gradients and dV, with
  magnitudes.  sigma is the population σ over all B·T advantages; when it is 0 the σ-derivative
  term of dV is 0 (the kernel's sc[6] = 0 rule)."""
  ret = f64(ret)
  B, T = ret.shape
  N = B * T
  nst, st_ = np.asarray(next_step_type).reshape(B, T), np.asarray(step_type).reshape(B, T)
  is_last = nst == STEP_LAST
  tt = np.arange(T)
  last = np.where(is_last.any(axis=1), np.where(is_last, tt, -1).max(axis=1), -1)
  episodes = float(is_last.sum())
  valid = (tt[None, :] <= last[:, None]).astype(np.float64)
  W = valid if weights is None else f64(weights) * valid
  c = np.where(st_ == STEP_LAST, 0.0, W)
  V = None if value is None else f64(value)
  use_adv = bool(use_advantage) and V is not None
  adv = ret - V if use_adv else ret.copy()
  cadv = np.abs(ret) + (np.abs(V) if use_adv else 0.0)       # magnitude of adv's own rounding
  mean = adv.mean()
  adv_c = adv - mean
  sigma = math.sqrt((adv_c ** 2).mean())
  D = sigma + EPS_F32
  m1 = np.abs(adv).mean()
  cac = cadv + abs(mean) + m1 + np.abs(adv_c)                # adv − mean, the mean's own error
  # sigma's relative magnitude: Σ|adv_c|·cac / (N σ²) (the moments' roundings), plus a few roundings
  rsig = (np.abs(adv_c) * cac).sum() / (N * sigma * sigma) + 4 if sigma > 0 else 0.0
  if normalize:
    adv_n = adv_c / D
    can = cac / D + np.abs(adv_n) * (rsig + 1)
  else:
    adv_n, can = adv, cadv + np.abs(adv)
  inv_ep = 1.0 / episodes if episodes > 0 else 0.0
  if discrete:
    sm = softmax_terms(np.asarray(params).reshape(N, -1))
    n = np.arange(N)
    a = np.asarray(action).reshape(N)
    logp, cl = sm['lp'][n, a].reshape(B, T), sm['clp'][n, a].reshape(B, T)
    ent, ce = sm['ent'].reshape(B, T), sm['cent'].reshape(B, T)
  else:
    nt = normal_terms(params[0], params[1], action)
    logp, cl = nt['logp'].reshape(B, T), nt['cl'].reshape(B, T)
    ent, ce = nt['ent'].reshape(B, T), nt['ce'].reshape(B, T)
  ec, vc_ = h32(entropy_coef or 0.0), h32(value_coef)
  s_pg = (-logp * c * adv_n).sum()
  c_pg = (np.abs(c) * (cl * np.abs(adv_n) + np.abs(logp) * can)).sum()
  s_ent = (-ent * W).sum()
  c_ent = (ce * np.abs(W)).sum()
  pg, c_pgl = s_pg * inv_ep, c_pg * inv_ep
  en = ec * s_ent / N if ec != 0 else 0.0
  c_en = abs(ec) * c_ent / N
  if V is not None:
    e = ret - V
    s_v = (e * e * W).sum()
    c_v = (np.abs(W) * (2 * np.abs(e) * (np.abs(ret) + np.abs(V)) + e * e)).sum()
    ve, c_ve = s_v * vc_ * inv_ep, c_v * abs(vc_) * inv_ep
  else:
    ve = c_ve = 0.0
  losses = np.array([pg, 0.0, en, ve, 0.0, pg + en + ve])
  c_losses = np.array([c_pgl, 0.0, c_en, c_ve, 0.0, c_pgl + c_en + c_ve])
  # parameter gradients
  g_lp = (-c * adv_n * inv_ep).reshape(N)
  cg = (np.abs(c) * can * inv_ep).reshape(N)
  g_ent = (-ec * W / N).reshape(N)
  if discrete:
    p, lp = sm['p'], sm['lp']
    onehot = np.zeros_like(p)
    onehot[n, a] = 1.0
    lpe = np.where(p > 0, lp + sm['ent'][:, None], 0.0)
    c_lpe = np.minimum(np.abs(lp + sm['ent'][:, None]), 1e3)
    grads = [g_lp[:, None] * (onehot - p) + g_ent[:, None] * (-p * lpe)]
    conds = [cg[:, None] * (onehot + p) + np.abs(g_lp)[:, None] * sm['cp'] +
             np.abs(g_ent)[:, None] * (sm['cp'] * c_lpe + p * (sm['clp'] + sm['cent'][:, None] + c_lpe))]
  else:
    d, inv = nt['d'], nt['inv']
    grads = [g_lp[:, None] * d * inv * inv,
             g_lp[:, None] * (d * d * inv ** 3 - inv) + g_ent[:, None] * inv]
    conds = [cg[:, None] * np.abs(d) * inv * inv * 2,
             cg[:, None] * (d * d * inv ** 3 + inv) * 2 + np.abs(g_ent)[:, None] * inv * 2]
  out = dict(last=last, valid=valid, episodes=episodes, mean=mean, sigma=sigma, D=D,
             losses=losses, c_losses=c_losses, grads=grads, c_grads=conds, dv=None, c_dv=None,
             logp=logp, adv_n=adv_n)
  if V is None:
    return out
  dv = vc_ * 2 * (V - ret) * W * inv_ep
  c_dv = abs(vc_) * 2 * (np.abs(V) + np.abs(ret)) * np.abs(W) * inv_ep * 2
  if use_adv:
    g = -logp * c * inv_ep                                   # d(pg) / d(adv_n)
    cgv = cl * np.abs(c) * inv_ep + np.abs(g)
    if normalize:
      g_bar = g.mean()
      S = (g * adv_c).sum()
      k6 = S / (N * sigma * D * D) if sigma > 0 else 0.0
      dv = dv - ((g - g_bar) / D - adv_c * k6)
      c_gbar = (cgv.sum() + np.abs(g).sum()) / N
      c_S = (cgv * np.abs(adv_c) + np.abs(g) * cac).sum()
      c_k6 = (c_S + abs(S) * 3 * (rsig + 1)) / (N * sigma * D * D) if sigma > 0 else 0.0
      c_dv = c_dv + (cgv + c_gbar + np.abs(g - g_bar) * (rsig + 1)) / D + cac * abs(k6) + np.abs(adv_c) * c_k6
      out.update(g=g, g_bar=g_bar, S=S, k6=k6)
    else:
      dv = dv - g                                            # adv = R − V
      c_dv = c_dv + cgv
  out.update(dv=dv, c_dv=c_dv)
  return out


# ---- CQL -----------------------------------------------------------------------------------------
def cql_loss(q1, q2, logp, B, N, uniform_logp, temperature, alpha, clip, tau, bc_debug, critic_loss,
             dq_init, log_alpha=None):
  """b200rl_cql_loss in float64 (the float64 autograd of test_cql_sac_gpu.py, restated
  analytically): per state b and critic i, lse_i = logsumexp_j(τ·Q_ij − log density_j)/τ over the
  2N candidates; cql = Σ_b [(lse_1 − q1_b) + (lse_2 − q2_b)] / (2B); dQ_candidate = α/(2B)·softmax,
  the data rows get dq_init − α/(2B) (−α/(2B) with bc_debug).  With log_alpha, α =
  exp(clip(log_alpha)) and dlog_alpha = −α (cql − τ_cql) inside [lo, hi] (bounds included)."""
  temp = h32(temperature)
  lp = f64(logp).reshape(B, N)
  ul = h32(uniform_logp)
  if log_alpha is not None:
    la = h32(log_alpha)
    a = math.exp(min(max(la, h32(clip[0])), h32(clip[1])))
  else:
    a = h32(alpha)
  g = a / (2.0 * B)
  out = {}
  terms, cterms = np.zeros(B), np.zeros(B)
  for i, q in enumerate((q1, q2)):
    q = f64(q)
    qp = q[B:B + B * N].reshape(B, N)
    qu = q[B + B * N:].reshape(B, N)
    x = np.concatenate([qp * temp - lp, qu * temp - ul], axis=1)
    cx = np.concatenate([2 * np.abs(qp * temp) + np.abs(lp), 2 * np.abs(qu * temp) + abs(ul)], axis=1) + np.abs(x)
    m = x.max(axis=1, keepdims=True)
    e = np.exp(x - m)
    s = e.sum(axis=1, keepdims=True)
    sm = e / s
    rel = cx + np.abs(x - m) + 1
    srel = (sm * rel).sum(axis=1, keepdims=True)
    lse = (m + np.log(s)) / temp
    clse = (srel + np.abs(m) + np.abs(np.log(s)) + np.abs(m + np.log(s))) / temp
    terms += lse[:, 0] - q[:B]
    cterms += clse[:, 0] + np.abs(q[:B]) + np.abs(lse[:, 0] - q[:B])
    dq = np.full(q.shape, np.nan)
    dq[B:B + B * N] = (g * sm[:, :N]).reshape(-1)
    dq[B + B * N:] = (g * sm[:, N:]).reshape(-1)
    cdq = np.full(q.shape, np.nan)
    cgs = g * (sm * (rel + srel + 2) + TINY_P)
    cdq[B:B + B * N] = cgs[:, :N].reshape(-1)
    cdq[B + B * N:] = cgs[:, N:].reshape(-1)
    init = f64(dq_init[i])
    dq[:B] = -g if bc_debug else init - g
    cdq[:B] = g * 2 + (0.0 if bc_debug else np.abs(init) + np.abs(init - g))
    out[f'dq{i + 1}'], out[f'c_dq{i + 1}'] = dq, cdq
  cql = terms.sum() / (2 * B)
  ccql = cterms.sum() / (2 * B)
  cl = h32(critic_loss)
  o2 = cql * a if bc_debug else cl + cql * a
  c2 = (ccql * a + abs(cql * a) * 3) + (0.0 if bc_debug else abs(cl) + abs(o2))
  closs, cclo, dla = 0.0, 0.0, None
  if log_alpha is not None:
    closs = -a * (cql - h32(tau))
    cclo = a * (ccql + abs(cql) + abs(h32(tau))) + 3 * abs(closs)
    dla = closs if h32(clip[0]) <= la <= h32(clip[1]) else 0.0
  out.update(out=np.array([cql, a, o2, closs]), c_out=np.array([ccql, 2 * a, c2, cclo]), dla=dla)
  return out


# ---- the kernels' fp32 association order (host emulation) -----------------------------------------
def warp_tree(v):
  """warp_sum over the last axis (32 lanes): the xor butterfly, offsets 16 .. 1, in fp32."""
  v = np.asarray(v, f32)
  lane = np.arange(32)
  for o in (16, 8, 4, 2, 1):
    v = (v + v[..., lane ^ o]).astype(f32)
  return v[..., 0]


def block_tree(v):
  """block_sum over the last axis (blockDim threads, a multiple of 32): each warp's butterfly, then
  warp 0's butterfly over the per-warp totals (zeros past the warp count)."""
  v = np.asarray(v, f32)
  nw = v.shape[-1] // 32
  per = warp_tree(v.reshape(v.shape[:-1] + (nw, 32)))
  pad = np.zeros(v.shape[:-1] + (32,), f32)
  pad[..., :nw] = per
  return warp_tree(pad)


def grid_sums(terms, nb, G=1, threads=256, passes=None):
  """The per-block partials of a grid-stride kernel whose row n is summed by lane 0 of its group
  of G lanes: each thread's serial sum over its passes, then block_tree.  `passes` (default all)
  exists for the host test's mutants."""
  terms = np.asarray(terms, f32)
  rows_per_pass = nb * threads // G
  P = -(-terms.shape[0] // rows_per_pass) if terms.shape[0] else 0
  if passes is not None:
    P = min(P, passes)
  pad = np.zeros(P * rows_per_pass, f32)
  n = min(terms.shape[0], P * rows_per_pass)
  pad[:n] = terms[:n]
  acc = np.zeros(rows_per_pass, f32)
  for p in pad.reshape(P, rows_per_pass):
    acc = (acc + p).astype(f32)
  th = np.zeros(nb * threads, f32)
  th[::G] = acc
  return block_tree(th.reshape(nb, threads))


def final_sum(partials, threads=512, nblocks=None):
  """The single-CTA final kernel: thread i takes partial i (i < nblocks), then block_tree."""
  p = np.asarray(partials, f32)
  nb = p.shape[0] if nblocks is None else nblocks
  th = np.zeros(threads, f32)
  th[:nb] = p[:nb]
  return block_tree(th)


# fp32 restatements of the loss kernels in their own association order (numpy fp32 ops round to
# nearest like the kernels; expf / logf and nvcc's FMA contraction differ in the last bit, so these
# are association-order emulations, not bit-exact twins).  `mutant` names one deliberate mistake
# for test_loss_metric_host.py; None is the kernel.
def _f(x):
  return np.asarray(x, f32)


def exp32(x):
  """expf correctly rounded (numpy's fp32 exp is not, and misses exact ties like 1.25)."""
  return np.exp(np.asarray(x, np.float64)).astype(f32)


def group_stats(z, G, drop_last_col=False):
  """row_softmax_stats<G> on [N, A] fp32 logits: lane l reads columns l, l+G, ... serially, then a
  G-lane xor tree.  Returns (m, s, t) as [N] fp32."""
  z = _f(z)
  N, A = z.shape
  if drop_last_col:
    z = z[:, :A - 1]
    A -= 1
  P = -(-A // G)
  pad = np.full((N, P * G), -np.inf, f32)
  pad[:, :A] = z
  cols = pad.reshape(N, P, G)
  m = pad.max(axis=1)
  with np.errstate(invalid='ignore', over='ignore'):
    s, t = np.zeros((N, G), f32), np.zeros((N, G), f32)
    for k in range(P):
      d = (cols[:, k, :] - m[:, None]).astype(f32)
      e = np.exp(d).astype(f32)
      s = (s + e).astype(f32)
      t = (t + np.where(e > 0, (e * d).astype(f32), f32(0))).astype(f32)
  lane = np.arange(G)
  o = G // 2
  while o > 0:
    s = (s + s[:, lane ^ o]).astype(f32)
    t = (t + t[:, lane ^ o]).astype(f32)
    o //= 2
  return m, s[:, 0], t[:, 0]


def _surrogate_fp32(logp, old, adv, ret, v, vo, w, eps, vcl, L, mutant):
  """The per-row surrogate / value terms of ppo_loss_kernel and ppo_loss_cat_kernel in fp32."""
  eps, vcl, L = f32(eps), f32(vcl), f32(L)
  lp, dlp = logp, np.ones_like(logp)
  if L > 0:
    lp = np.minimum(np.maximum(logp, -L), L)
    if mutant != 'logp_clip_derivative_kept':
      dlp = np.where((logp < -L) | (logp > L), f32(0), f32(1)).astype(f32)
  ratio = exp32((lp - old).astype(f32))
  lo, hi = f32(f32(1) - eps), f32(f32(1) + eps)
  rc = np.minimum(np.maximum(ratio, lo), hi)
  obj, obj_c = (ratio * adv).astype(f32), (rc * adv).astype(f32)
  pg = -np.minimum(obj, obj_c)
  outside = (ratio < lo) | (ratio > hi)
  dobj = np.where(obj <= obj_c, adv, np.where(outside, f32(0), adv)).astype(f32)
  if mutant == 'unclipped_gradient_outside_clip':
    dobj = adv
  r1 = np.abs((ratio - f32(1)).astype(f32))
  clipped = ((r1 >= eps) if mutant == 'clip_count_ge' else (r1 > eps)).astype(f32)
  e = (ret - v).astype(f32)
  err, derr = (e * e).astype(f32), (f32(-2) * e).astype(f32)
  if vcl > 0:
    dvv = (v - vo).astype(f32)
    vc = (vo + np.minimum(np.maximum(dvv, -vcl), vcl)).astype(f32)
    ec = (ret - vc).astype(f32)
    errc = (ec * ec).astype(f32)
    take = (errc < err) if mutant == 'value_clip_min' else (errc > err)
    dout = (dvv < -vcl) | (dvv > vcl)
    derr = np.where(take, np.where(dout, f32(0), (f32(-2) * ec).astype(f32)), derr).astype(f32)
    err = np.where(take, errc, err).astype(f32)
  return ratio, dobj, dlp, pg, err, derr, clipped


def _ppo_final_fp32(parts, nb, T, gb, N, vf, ec, kl_terms, mutant):
  if mutant == 'last_partial_block_dropped':
    nb -= 1
  v = [final_sum(parts[:, j], 512, nb) for j in range(4)]
  den = f32(N) if mutant == 'denom_N' else f32(f32(T) * f32(gb))
  pg, ve, en = f32(v[0] / den), f32(f32(vf) * v[1] / den), f32(f32(ec) * v[2] / den)
  kl = f32(0) if kl_terms is None else f32(f32(kl_terms[0]) + f32(kl_terms[1]))
  return np.array([pg, ve, en, f32(v[3] / f32(N)), f32(f32(f32(pg + ve) + en) + kl), kl], f32)


def ppo_loss_fp32(loc, scale, action, old_logp, adv, ret, v, v_old, w, T, global_batch, clip_eps,
                  value_clip, vf_coef, ent_coef, logp_clip, kl=None, mutant=None):
  """ppo_loss_kernel + ppo_loss_final_kernel in fp32: one thread per row, kRedBlocks = 264."""
  loc, scale, action = _f(loc), _f(scale), _f(action)
  N, A = loc.shape
  c = f32(0.5) * f32(LOG2PI)
  logp, ent = np.zeros(N, f32), np.zeros(N, f32)
  for k in range(A):
    z = ((action[:, k] - loc[:, k]).astype(f32) / scale[:, k]).astype(f32)
    lsg = np.log(scale[:, k]).astype(f32)
    logp = (logp + (((f32(-0.5) * z).astype(f32) * z).astype(f32) - lsg - c).astype(f32)).astype(f32)
    ent = (ent + ((f32(0.5) + c) + lsg).astype(f32)).astype(f32)
  w = _f(w)
  ratio, dobj, dlp, pg, err, derr, clipped = _surrogate_fp32(
      logp, _f(old_logp), _f(adv), _f(ret), _f(v), _f(v_old), w, clip_eps, value_clip, logp_clip, mutant)
  terms = np.stack([(pg * w).astype(f32), (err * w).astype(f32), (-ent * w).astype(f32), clipped], 1)
  nb = min(-(-N // 256), 264)
  passes = 1 if mutant == 'second_pass_dropped' else None
  parts = np.stack([grid_sums(terms[:, j], nb, 1, 256, passes) for j in range(4)], 1)
  losses = _ppo_final_fp32(parts, nb, T, global_batch, N, vf_coef, ent_coef,
                           None if kl is None else kl['terms'], mutant)
  den = f32(N) if mutant == 'denom_N' else f32(f32(T) * f32(global_batch))
  g_logp = ((((-dobj * ratio).astype(f32) * dlp).astype(f32) * w).astype(f32) / den).astype(f32)
  g_ent = ((f32(-ent_coef) * w).astype(f32) / den).astype(f32)
  d = (action - loc).astype(f32)
  inv = (f32(1) / scale).astype(f32)
  gi = g_logp[:, None]
  dloc = (((gi * d).astype(f32) * inv).astype(f32) * inv).astype(f32)
  ddi = (((d * d).astype(f32) * inv).astype(f32) * inv).astype(f32)
  dscale = ((gi * ((ddi * inv).astype(f32) - inv).astype(f32)).astype(f32) + (g_ent[:, None] * inv).astype(f32)).astype(f32)
  if kl is not None:
    g_kl = ((f32(kl['terms'][2]) * f32(kl['grad_scale'])).astype(f32) * w).astype(f32)[:, None]
    mo, so = _f(kl['old_loc']), _f(kl['old_scale'])
    dm = (mo - loc).astype(f32)
    dloc = (dloc + (g_kl * (((-dm) * inv).astype(f32) * inv).astype(f32)).astype(f32)).astype(f32)
    q = ((dm * dm).astype(f32) if mutant == 'kl_scale_grad_without_so2'
         else ((dm * dm).astype(f32) + (so * so).astype(f32)).astype(f32))
    q = (((q * inv).astype(f32) * inv).astype(f32) * inv).astype(f32)
    dscale = (dscale + (g_kl * (inv - q).astype(f32)).astype(f32)).astype(f32)
  dv = (((f32(vf_coef) * derr).astype(f32) * w).astype(f32) / den).astype(f32)
  return dict(losses=losses, dloc=dloc, dscale=dscale, dv=dv, nb=nb)


def ppo_loss_categorical_fp32(logits, action, old_logp, adv, ret, v, v_old, w, T, global_batch,
                              clip_eps, value_clip, vf_coef, ent_coef, logp_clip, kl=None,
                              mutant=None):
  """ppo_loss_cat_kernel<G> + ppo_loss_final_kernel in fp32, G from A, kCatRedBlocks = 512."""
  z = _f(logits)
  N, A = z.shape
  G = cat_group(A)
  m, s, t = group_stats(z, G, mutant == 'last_strided_column_dropped')
  ls = np.log(s).astype(f32)
  ent = (ls - (t / s).astype(f32)).astype(f32)
  n = np.arange(N)
  act = np.asarray(action)
  logp = ((z[n, act] - m).astype(f32) - ls).astype(f32)
  w = _f(w)
  ratio, dobj, dlp, pg, err, derr, clipped = _surrogate_fp32(
      logp, _f(old_logp), _f(adv), _f(ret), _f(v), _f(v_old), w, clip_eps, value_clip, logp_clip, mutant)
  terms = np.stack([(pg * w).astype(f32), (err * w).astype(f32), (-ent * w).astype(f32), clipped], 1)
  nb = min(-(-N * G // 256), 512)
  passes = 1 if mutant == 'second_pass_dropped' else None
  parts = np.stack([grid_sums(terms[:, j], nb, G, 256, passes) for j in range(4)], 1)
  losses = _ppo_final_fp32(parts, nb, T, global_batch, N, vf_coef, ent_coef,
                           None if kl is None else kl['terms'], mutant)
  den = f32(N) if mutant == 'denom_N' else f32(f32(T) * f32(global_batch))
  g_logp = ((((-dobj * ratio).astype(f32) * dlp).astype(f32) * w).astype(f32) / den).astype(f32)
  g_ent = ((f32(-ent_coef) * w).astype(f32) / den).astype(f32)
  lpj = ((z - m[:, None]).astype(f32) - ls[:, None]).astype(f32)
  p = np.exp(lpj).astype(f32)
  onehot = np.zeros((N, A), f32)
  onehot[n, act] = 1
  with np.errstate(invalid='ignore', over='ignore'):      # the dropped-column mutant's NaN rows
    pe = (-p * (lpj if mutant == 'entropy_grad_without_ent' else (lpj + ent[:, None]).astype(f32))).astype(f32)
    dz = ((g_logp[:, None] * (onehot - p).astype(f32)).astype(f32) + (g_ent[:, None] * pe).astype(f32)).astype(f32)
  if kl is not None:
    mo, so_, _ = group_stats(kl['old_logits'], G)
    q = np.exp(((_f(kl['old_logits']) - mo[:, None]).astype(f32) - np.log(so_).astype(f32)[:, None]).astype(f32)).astype(f32)
    g_kl = ((f32(kl['terms'][2]) * f32(kl['grad_scale'])).astype(f32) * w).astype(f32)[:, None]
    dz = (dz + (g_kl * (p - q).astype(f32)).astype(f32)).astype(f32)
  dv = (((f32(vf_coef) * derr).astype(f32) * w).astype(f32) / den).astype(f32)
  return dict(losses=losses, dlogits=dz, dv=dv, logp=logp, nb=nb, G=G)


def cat_group(A):
  """Lanes per logits row (cat_group in ppo.cu, rf_group in reinforce.cu, cql_group of 2N)."""
  return 1 if A <= 8 else (8 if A <= 64 else 32)


def _mom_merge(an, am, a2, bn, bm, b2):
  """mom_merge in fp32 on arrays (b.n == 0 keeps a)."""
  n = (an + bn).astype(f32)
  with np.errstate(invalid='ignore', divide='ignore'):
    d = (bm - am).astype(f32)
    f = (bn / n).astype(f32)
    mean = (am + (d * f).astype(f32)).astype(f32)
    m2 = ((a2 + b2).astype(f32) + ((((d * d).astype(f32) * an).astype(f32)) * f).astype(f32)).astype(f32)
  keep = bn == 0
  return (np.where(keep, an, n).astype(f32), np.where(keep, am, mean).astype(f32),
          np.where(keep, a2, m2).astype(f32))


def _mom_tree(n, m, s):
  """warp_mom on [..., 32] lanes: lanes [0, o) merge lanes [o, 2o), o = 16 .. 1; lane 0's result."""
  n, m, s = n.copy(), m.copy(), s.copy()
  for o in (16, 8, 4, 2, 1):
    n[..., :o], m[..., :o], s[..., :o] = _mom_merge(n[..., :o], m[..., :o], s[..., :o],
                                                     n[..., o:2 * o], m[..., o:2 * o], s[..., o:2 * o])
  return n[..., 0], m[..., 0], s[..., 0]


def reinforce_moments_fp32(adv, mutant=None):
  """rf_stats_kernel + rf_stats_final_kernel's moments in fp32: Welford per lane over t = l, l+32,
  ..., the warp tree per trajectory, each warp's trajectories merged in order, thread 0 merging the
  8 warps, the final warp merging the block partials.  Returns (mean, sigma, D) as fp32."""
  adv = _f(adv)
  B, T = adv.shape
  P = -(-T // 32)
  n = np.zeros((B, 32), f32)
  m, s = np.zeros((B, 32), f32), np.zeros((B, 32), f32)
  for p in range(P):
    x = np.zeros((B, 32), f32)
    k = np.zeros((B, 32), f32)
    hi = min(T, (p + 1) * 32) - p * 32
    x[:, :hi] = adv[:, p * 32:p * 32 + hi]
    k[:, :hi] = 1
    n, m, s = _mom_merge(n, m, s, k, x, np.zeros_like(x))
  tn, tm, ts = _mom_tree(n, m, s)                       # per trajectory
  nb1 = min(-(-B // 8), 264)
  warps = nb1 * 8
  Pw = -(-B // warps)
  wn, wm, ws = (np.zeros(warps, f32) for _ in range(3))
  for p in range(Pw):
    lo, hi = p * warps, min(B, (p + 1) * warps)
    bn, bm, bs = (np.zeros(warps, f32) for _ in range(3))
    bn[:hi - lo], bm[:hi - lo], bs[:hi - lo] = tn[lo:hi], tm[lo:hi], ts[lo:hi]
    wn, wm, ws = _mom_merge(wn, wm, ws, bn, bm, bs)
  wn, wm, ws = (x.reshape(nb1, 8) for x in (wn, wm, ws))
  rn, rm, rs = wn[:, 0], wm[:, 0], ws[:, 0]
  for i in range(1, 8):
    rn, rm, rs = _mom_merge(rn, rm, rs, wn[:, i], wm[:, i], ws[:, i])
  Pl = -(-nb1 // 32)
  ln_, lm, ls_ = (np.zeros(32, f32) for _ in range(3))
  for p in range(Pl):
    lo, hi = p * 32, min(nb1, (p + 1) * 32)
    bn, bm, bs = (np.zeros(32, f32) for _ in range(3))
    bn[:hi - lo], bm[:hi - lo], bs[:hi - lo] = rn[lo:hi], rm[lo:hi], rs[lo:hi]
    ln_, lm, ls_ = _mom_merge(ln_, lm, ls_, bn, bm, bs)
  n, mean, m2 = _mom_tree(ln_, lm, ls_)
  div = f32(n - 1) if mutant == 'bessel_sigma' else n
  sigma = f32(np.sqrt(f32(m2 / div)))
  return f32(mean), sigma, f32(sigma + f32(EPS_F32))


def reinforce_loss_fp32(params, action, ret, value, step_type, next_step_type, weights,
                        use_advantage, normalize, entropy_coef, value_coef, discrete, mutant=None):
  """The five stages of b200rl_reinforce_loss in fp32 (G from A for the categorical head,
  kRfLossBlocks = 512)."""
  ret = _f(ret)
  B, T = ret.shape
  N = B * T
  nst, st_ = np.asarray(next_step_type).reshape(B, T), np.asarray(step_type).reshape(B, T)
  is_last = nst == STEP_LAST
  tt = np.arange(T)
  last = np.where(is_last.any(axis=1), np.where(is_last, tt, -1).max(axis=1), -1)
  episodes = f32(is_last.sum())
  valid = (tt[None, :] <= last[:, None]).astype(f32)
  W = valid if weights is None else (_f(weights) * valid).astype(f32)
  c = np.where(st_ == STEP_LAST, f32(0), W).astype(f32).reshape(N)
  W = W.reshape(N)
  V = None if value is None else _f(value)
  use_adv = bool(use_advantage) and V is not None
  adv = (ret - V).astype(f32) if use_adv else ret
  mean, sigma, D = reinforce_moments_fp32(adv, mutant)
  adv = adv.reshape(N)
  adv_c = (adv - mean).astype(f32)
  adv_n = (adv_c / D).astype(f32) if normalize else adv
  inv_ep = f32(f32(1) / episodes) if episodes > 0 else f32(0)
  inv_n = f32(f32(1) / f32(N))
  ec, vc_ = f32(entropy_coef or 0.0), f32(value_coef)
  if discrete:
    z = _f(params).reshape(N, -1)
    A = z.shape[1]
    G = cat_group(A)
    m, s, t = group_stats(z, G)
    ls = np.log(s).astype(f32)
    ent = (ls - (t / s).astype(f32)).astype(f32)
    n = np.arange(N)
    a = np.asarray(action).reshape(N)
    logp = ((z[n, a] - m).astype(f32) - ls).astype(f32)
  else:
    G = 1
    loc, scale, act = _f(params[0]), _f(params[1]), _f(action)
    A = loc.shape[1]
    cc = f32(0.5) * f32(LOG2PI)
    logp, ent = np.zeros(N, f32), np.zeros(N, f32)
    for k in range(A):
      zz = ((act[:, k] - loc[:, k]).astype(f32) / scale[:, k]).astype(f32)
      lsg = np.log(scale[:, k]).astype(f32)
      logp = (logp + (((f32(-0.5) * zz).astype(f32) * zz).astype(f32) - lsg - cc).astype(f32)).astype(f32)
      ent = (ent + ((f32(0.5) + cc) + lsg).astype(f32)).astype(f32)
  s_pg = (-((logp * c).astype(f32) * adv_n)).astype(f32)
  s_ent = (-(ent * W)).astype(f32)
  zero = np.zeros(N, f32)
  s_v, s_g, s_gd = zero, zero, zero
  g = None
  if V is not None:
    e = (ret.reshape(N) - V.reshape(N)).astype(f32)
    s_v = ((e * e).astype(f32) * W).astype(f32)
    dv = ((((vc_ * f32(2)) * (-e)).astype(f32) * W).astype(f32) * inv_ep).astype(f32)
    if use_adv:
      g = ((-logp * c).astype(f32) * inv_ep).astype(f32)
      if normalize:
        s_g, s_gd = g, (g * adv_c).astype(f32)
      else:
        dv = (dv - g).astype(f32)
  nb3 = min(-(-N * G // 256), 512)
  parts = [grid_sums(x, nb3, G, 256) for x in (s_pg, s_ent, s_v, s_g, s_gd)]
  v = [final_sum(p, 512) for p in parts]
  pg = f32(v[0] * inv_ep)
  en = f32(ec * f32(v[1] / f32(N))) if ec != 0 else f32(0)
  ve = f32(f32(v[2] * vc_) * inv_ep) if V is not None else f32(0)
  losses = np.array([pg, 0, en, ve, 0, f32(f32(pg + en) + ve)], f32)
  g_lp = ((-c * adv_n).astype(f32) * inv_ep).astype(f32)
  g_ent = ((-ec * W).astype(f32) * inv_n).astype(f32)
  if discrete:
    lpj = ((z - m[:, None]).astype(f32) - ls[:, None]).astype(f32)
    p = np.exp(lpj).astype(f32)
    onehot = np.zeros_like(p)
    onehot[n, a] = 1
    grads = [((g_lp[:, None] * (onehot - p).astype(f32)).astype(f32) +
              (g_ent[:, None] * (-p * (lpj + ent[:, None]).astype(f32)).astype(f32)).astype(f32)).astype(f32)]
  else:
    d = (act - loc).astype(f32)
    inv = (f32(1) / scale).astype(f32)
    gi = g_lp[:, None]
    ddi = (((d * d).astype(f32) * inv).astype(f32) * inv).astype(f32)
    grads = [(((gi * d).astype(f32) * inv).astype(f32) * inv).astype(f32),
             ((gi * ((ddi * inv).astype(f32) - inv).astype(f32)).astype(f32) + (g_ent[:, None] * inv).astype(f32)).astype(f32)]
  out = dict(losses=losses, grads=grads, dv=None, episodes=episodes)
  if V is None:
    return out
  if use_adv and normalize and mutant != 'stage5_dv_omitted':
    g_bar = f32(v[3] / f32(N))
    k6 = f32(v[4] / f32(f32(f32(f32(N) * sigma) * D) * D)) if sigma > 0 else f32(0)
    dv = (dv - ((((g - g_bar).astype(f32) / D).astype(f32)) - (adv_c * k6).astype(f32)).astype(f32)).astype(f32)
  out['dv'] = dv.reshape(B, T)
  return out


def cql_loss_fp32(q1, q2, logp, B, N, uniform_logp, temperature, alpha, tau, bc_debug, critic_loss,
                  dq_init):
  """cql_loss_rows_kernel<G> + cql_loss_final_kernel in fp32 (fixed alpha), G from 2N,
  kCqlRedBlocks = 256."""
  temp, ul, a = f32(temperature), f32(uniform_logp), f32(alpha)
  g = f32(a / f32(f32(2) * f32(B)))
  M = 2 * N
  G = cat_group(M)
  lp = _f(logp).reshape(B, N)
  term = np.zeros(B, f32)
  out = {}
  for i, q in enumerate((q1, q2)):
    q = _f(q)
    x = np.concatenate([((q[B:B + B * N].reshape(B, N) * temp).astype(f32) - lp).astype(f32),
                        ((q[B + B * N:].reshape(B, N) * temp).astype(f32) - ul).astype(f32)], axis=1)
    P = -(-M // G)
    pad = np.full((B, P * G), -np.inf, f32)
    pad[:, :M] = x
    m = x.max(axis=1)
    s = np.zeros((B, G), f32)
    for k in range(P):
      s = (s + np.exp((pad.reshape(B, P, G)[:, k, :] - m[:, None]).astype(f32)).astype(f32)).astype(f32)
    lane = np.arange(G)
    o = G // 2
    while o > 0:
      s = (s + s[:, lane ^ o]).astype(f32)
      o //= 2
    s = s[:, 0]
    term = (term + (((m + np.log(s).astype(f32)).astype(f32) / temp).astype(f32) - q[:B]).astype(f32)).astype(f32)
    gs = (g / s).astype(f32)
    e = np.exp((x - m[:, None]).astype(f32)).astype(f32)
    dq = np.full(q.shape, np.nan, f32)
    dq[B:B + B * N] = (gs[:, None] * e[:, :N]).reshape(-1)
    dq[B + B * N:] = (gs[:, None] * e[:, N:]).reshape(-1)
    dq[:B] = -g if bc_debug else (_f(dq_init[i]) - g).astype(f32)
    out[f'dq{i + 1}'] = dq
  nb = min(-(-B * G // 256), 256)
  s = final_sum(grid_sums(term, nb, G, 256), 256)
  cql = f32(s / f32(f32(2) * f32(B)))
  o2 = f32(cql * a) if bc_debug else f32(f32(critic_loss) + f32(cql * a))
  out['out'] = np.array([cql, a, o2, 0], f32)
  return out


# ---- inputs with their branch margins --------------------------------------------------------------
MARGIN = 1e-4    # relative distance every branch input keeps from its threshold


def _margins_ok(ratio, logp, dvv, err, errc, eps, vcl, L):
  ok = np.ones(ratio.shape, bool)
  if eps > 0:
    for t in (1 - eps, 1 + eps):
      ok &= np.abs(ratio - t) >= MARGIN * t
  if L > 0:
    ok &= np.abs(np.abs(logp) - L) >= MARGIN * L
  if vcl > 0:
    ok &= np.abs(np.abs(dvv) - vcl) >= MARGIN * vcl
    ok &= (np.abs(dvv) < vcl) | (np.abs(errc - err) >= MARGIN * np.maximum(err, errc))
  return ok


def branch_margins(logp, old_logp, v, v_old, ret, clip_eps, value_clip, logp_clip):
  """The rows whose float64 ratio, logp and value-clip inputs keep MARGIN from every threshold (no
  row may take another branch in fp32 than in float64)."""
  eps, vcl, L = h32(clip_eps), h32(value_clip), h32(logp_clip)
  lp = np.clip(logp, -L, L) if L > 0 else logp
  ratio = np.exp(lp - f64(old_logp))
  V, vo, R = f64(v), f64(v_old), f64(ret)
  dvv = V - vo
  vc = vo + np.clip(dvv, -vcl, vcl)
  return _margins_ok(ratio, logp, dvv, (R - V) ** 2, (R - vc) ** 2, eps, vcl, L)


def ppo_rows(rng, logp, clip_eps, value_clip, logp_clip, ratio_lo=0.55, ratio_hi=1.6):
  """old_logp / adv / ret / v / v_old / w [N] for rows of log-prob `logp` (float64): ratios spread
  over [ratio_lo, ratio_hi] (both sides of the clip), advantages of both signs across 1e-2 .. 1e2
  with exact zeros, value errors on both sides of the value clip, weights 0, 1 and non-binary.
  Rows are redrawn until every one keeps MARGIN from every branch threshold."""
  N = logp.shape[0]
  L = h32(logp_clip)
  lp = np.clip(logp, -L, L) if L > 0 else logp
  adv = rng.randn(N) * 10.0 ** rng.uniform(-2, 2, N)
  adv[rng.rand(N) < 0.05] = 0
  w = np.where(rng.rand(N) < 0.5, 1.0, rng.uniform(0, 2, N))
  w[rng.rand(N) < 0.05] = 0
  old = np.empty(N, f32)
  v, vo, ret = np.empty(N, f32), np.empty(N, f32), np.empty(N, f32)
  todo = np.ones(N, bool)
  for _ in range(30):
    k = int(todo.sum())
    if k == 0:
      break
    old[todo] = (lp[todo] - np.log(rng.uniform(ratio_lo, ratio_hi, k))).astype(f32)
    v[todo] = rng.randn(k).astype(f32)
    vo[todo] = (v[todo] + rng.randn(k) * 0.4).astype(f32)
    ret[todo] = (v[todo] + rng.randn(k)).astype(f32)
    todo = ~branch_margins(logp, old, v, vo, ret, clip_eps, value_clip, logp_clip)
  assert not todo.any()
  return dict(old_logp=old, adv=adv.astype(f32), ret=ret, v=v, v_old=vo, w=w.astype(f32))


def logp_clip_for(logp, q):
  """A logp clip near the q-quantile of |logp| that keeps MARGIN from every row's |logp|."""
  L = h32(np.quantile(np.abs(logp), q)) + 0.01
  while (np.abs(np.abs(logp) - L) < 2 * MARGIN * L).any():
    L = h32(L * 1.0007)
  return L


def normal_params(rng, N, A):
  """loc, scale (1e-3 .. 1e2) and actions within a few scales of loc, [N, A] fp32."""
  loc = (rng.randn(N, A) * 2).astype(f32)
  scale = (10.0 ** rng.uniform(-3, 2, (N, A))).astype(f32)
  action = (loc + scale * rng.randn(N, A) * 1.5).astype(f32)
  return loc, scale, action


def logits_rows(rng, N, A):
  """[N, A] logits and actions with the numeric edges mixed in by row: masked columns at
  MASKED (never the action's), one dominant logit (the others' p underflow to 0), all-equal
  logits, a common offset of ±1e4, and actions at 0 and A − 1."""
  z = rng.randn(N, A) * 2
  act = rng.randint(0, A, N)
  kind = np.arange(N) % 8
  act[kind == 1] = 0
  act[kind == 2] = A - 1
  if A > 1:
    dom = kind == 3
    z[dom] = rng.randn(int(dom.sum()), A)
    z[dom, rng.randint(0, A, int(dom.sum())) if A else 0] += 120.0
  z[kind == 4] = 0.7
  z[kind == 5] += 1e4
  z[kind == 6] -= 1e4
  if A > 2:
    msk = (kind == 7)[:, None] & (rng.rand(N, A) < 0.4)
    msk[np.arange(N), act] = False
    z[msk] = MASKED
  return z.astype(f32), act.astype(np.int32)


def old_logits_like(rng, z):
  """Behaviour-policy logits near z with the same masked columns."""
  zo = (z + rng.randn(*z.shape) * 0.3).astype(f32)
  zo[z == f32(MASKED)] = f32(MASKED)
  return zo


def reinforce_steps(rng, B, T, p_last=0.15):
  """step_type / next_step_type [B, T] (FIRST follows LAST): episodes ending at t = 0 on rows
  b % 6 == 1 and at t = T − 1 on rows b % 6 == 2; rows b % 6 == 5 have no LAST at all."""
  s = np.where(rng.rand(B, T + 1) < p_last, STEP_LAST, 1).astype(np.int32)
  s[:, 0] = 0
  s[:, 1:][s[:, :-1] == STEP_LAST] = 0
  b = np.arange(B)
  s[b % 6 == 1, 1] = STEP_LAST
  s[b % 6 == 2, T] = STEP_LAST
  s[b % 6 == 5, 1:] = 1
  return s[:, :T].copy(), s[:, 1:].copy()
