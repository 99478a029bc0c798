"""float64 torch restatements of everything between an agent's loss and its optimizer, and the
gradient metric the gradient tests compare against them.

Host-only: nothing here needs a CUDA device.  The GPU tests (test_grad_kernels_gpu.py,
test_agent_grads_gpu.py) differentiate these functions with autograd and compare the result with
what the kernels and agents hand to the optimizer; test_grad_metric_host.py shows that the metric
rejects the gradient errors Adam would hide (a constant factor, a missing `half`, α = 1, a missing
l2 term, 1/B instead of 1/global_batch).

Sources restated: agents/sac/sac_agent.py (critic_loss :559-643, actor_loss :645-694, alpha_loss
:696-739), distributions/utils.py SquashToSpecNormal + tanh_bijector_stable.py:68-82 (tanh-Normal
log-prob), networks/normal_projection_network.py (tanh-squashed mean, softplus std bias),
agents/ppo/ppo_agent.py (policy_gradient_loss :1329-1512, value_estimation_loss :1203-1327,
entropy_regularization_loss :1159-1201, kl_cutoff_loss / adaptive_kl_loss :1514-1558,
l2_regularization_loss :1088-1157), agents/dqn/dqn_agent.py (_loss :462-579), utils/common.py
aggregate_losses :1400-1476.
"""
import math

import numpy as np
import torch

F64 = torch.float64
LOG2PI = math.log(2.0 * math.pi)
LOG2 = math.log(2.0)
# No gradient bound in the tests may exceed this: a 1 % error in any gradient must still fail.
MAX_BOUND = 1e-3
FLOOR = 1e-9


def t64(a):
  """float64 CPU tensor of a numpy array, python number or (CUDA) tensor; detached copy."""
  if isinstance(a, torch.Tensor):
    return a.detach().to('cpu', F64).clone()
  return torch.as_tensor(np.asarray(a, dtype=np.float64))


# ---- the gradient metric --------------------------------------------------------------------------
def grad_errors(got, ref):
  """(‖g − g_ref‖ / ‖g_ref‖, max|g − g_ref| / max|g_ref|) of one gradient tensor."""
  g, r = t64(got).reshape(-1), t64(ref).reshape(-1)
  if g.shape != r.shape:
    raise ValueError(f'gradient shapes differ: {tuple(g.shape)} vs {tuple(r.shape)}')
  d = g - r
  rn, rm = float(r.norm()), float(r.abs().max()) if r.numel() else 0.0
  dn, dm = float(d.norm()), float(d.abs().max()) if d.numel() else 0.0
  if not (math.isfinite(dn) and math.isfinite(dm)):
    return math.inf, math.inf
  return (dn / rn if rn > 0 else (0.0 if dn <= FLOOR else math.inf),
          dm / rm if rm > 0 else (0.0 if dm <= FLOOR else math.inf))


def grad_close(got, ref, rel_l2, rel_max):
  """‖g − g_ref‖ ≤ rel_l2·‖g_ref‖ + 1e-9 and max|g − g_ref| ≤ rel_max·max|g_ref| + 1e-9."""
  g, r = t64(got).reshape(-1), t64(ref).reshape(-1)
  if g.shape != r.shape or not bool(torch.isfinite(g).all()):
    return False
  d = g - r
  return (float(d.norm()) <= rel_l2 * float(r.norm()) + FLOOR and
          float(d.abs().max()) <= rel_max * float(r.abs().max()) + FLOOR)


def assert_grad_close(name, got, ref, rel_l2, rel_max):
  assert rel_l2 <= MAX_BOUND and rel_max <= MAX_BOUND, f'{name}: bound above {MAX_BOUND}'
  if not grad_close(got, ref, rel_l2, rel_max):
    e = grad_errors(got, ref)
    raise AssertionError(f'{name}: relative L2 error {e[0]:.3g} (bound {rel_l2:.3g}), '
                         f'max error / max|ref| {e[1]:.3g} (bound {rel_max:.3g})')


# ---- networks -------------------------------------------------------------------------------------
def activate(x, act):
  if act == 'relu':
    return torch.relu(x)
  if act == 'tanh':
    return torch.tanh(x)
  if act is None:
    return x
  raise ValueError(f'activation {act!r}')


def mlp(layers, x):
  """layers: [(kernel [in, out], bias [out], activation)] -> x @ W + b, activated, per layer."""
  for w, b, act in layers:
    x = activate(x @ w + b, act)
  return x


def tf_min(x, y):
  """tf.minimum with TF's gradient routing: all of it to x where x <= y (torch.minimum would
  split it between x and y on ties)."""
  return torch.where(x <= y, x, y)


def tf_max(x, y):
  """tf.maximum: the gradient goes to x where x >= y."""
  return torch.where(x >= y, x, y)


def softplus(x):
  """Exact softplus (no threshold branch)."""
  return torch.logaddexp(x, torch.zeros_like(x))


def aggregate(per_example, weights, global_batch):
  """common.aggregate_losses: weight (multiply_no_nan), sum, divide by the global batch."""
  if weights is not None:
    per_example = torch.where(weights == 0, torch.zeros_like(per_example), per_example * weights)
  return per_example.sum() / global_batch


# ---- SAC ------------------------------------------------------------------------------------------
def sac_sample(head, eps, amin, amax):
  """head [N, 2A] = (loc | log_std) -> (action, u, log_prob) of the tanh-squashed Normal with the
  noise `eps` held fixed: u = loc + exp(log_std)·eps, a = shift + half·tanh(u)."""
  A = head.shape[1] // 2
  loc, log_std = head[:, :A], head[:, A:]
  u = loc + torch.exp(log_std) * eps
  half, shift = (amax - amin) / 2, (amax + amin) / 2
  action = shift + half * torch.tanh(u)
  logp = (-0.5 * eps * eps - log_std - 0.5 * LOG2PI - torch.log(half)
          - 2.0 * (LOG2 - u - softplus(-2.0 * u))).sum(dim=1)
  return action, u, logp


def sac_critic_loss(q1, q2, tq1, tq2, next_logp, reward, discount, log_alpha, gamma,
                    reward_scale, loss_weight, global_batch, weights=None):
  """Returns (loss, td_targets); the targets are constants of the critic gradient."""
  alpha = torch.exp(torch.as_tensor(log_alpha, dtype=F64)).detach()
  target_q = tf_min(tq1, tq2) - alpha * next_logp
  y = (reward_scale * reward + gamma * discount * target_q).detach()
  per = (y - q1) ** 2 + (y - q2) ** 2
  return loss_weight * aggregate(per, weights, global_batch), y


def sac_actor_loss(q1, q2, logp, log_alpha, loss_weight, global_batch, weights=None):
  alpha = torch.exp(torch.as_tensor(log_alpha, dtype=F64)).detach()
  return loss_weight * aggregate(alpha * logp - tf_min(q1, q2), weights, global_batch)


def sac_alpha_loss(logp, log_alpha, target_entropy, use_log_alpha, loss_weight, global_batch,
                   weights=None):
  """log_alpha: a float64 tensor (differentiated); log_pi is a constant of this loss."""
  diff = (-logp - target_entropy).detach()
  coef = log_alpha if use_log_alpha else torch.exp(log_alpha)
  return loss_weight * aggregate(coef * diff, weights, global_batch)


# ---- Normal projection head and PPO -------------------------------------------------------------
def normal_projection(m_raw, std_bias, amin, amax):
  """loc = shift + half·tanh(m_raw), scale = softplus(std_bias) broadcast over the batch."""
  loc = (amax + amin) / 2 + (amax - amin) / 2 * torch.tanh(m_raw)
  return loc, softplus(std_bias).expand_as(m_raw)


def normal_log_prob(loc, scale, action):
  z = (action - loc) / scale
  return (-0.5 * z * z - torch.log(scale) - 0.5 * LOG2PI).sum(dim=-1)


def normal_entropy(scale):
  return (0.5 + 0.5 * LOG2PI + torch.log(scale)).sum(dim=-1)


def normal_kl(loc_a, scale_a, loc_b, scale_b):
  """Σ_k KL(N(loc_a, scale_a) ‖ N(loc_b, scale_b))."""
  return (torch.log(scale_b / scale_a) + (scale_a ** 2 + (loc_a - loc_b) ** 2) / (2 * scale_b ** 2)
          - 0.5).sum(dim=-1)


def categorical_log_prob(logits, action):
  return torch.log_softmax(logits, dim=-1).gather(1, action.long().reshape(-1, 1))[:, 0]


def categorical_entropy(logits):
  ls = torch.log_softmax(logits, dim=-1)
  return -(ls.exp() * ls).sum(dim=-1)


def categorical_kl(logits_a, logits_b):
  la, lb = torch.log_softmax(logits_a, dim=-1), torch.log_softmax(logits_b, dim=-1)
  return (la.exp() * (la - lb)).sum(dim=-1)


def ppo_loss(logp, entropy, old_logp, adv, ret, v, v_old, w, denom, clip_eps, value_clip,
             vf_coef, ent_coef):
  """policy-gradient + value + entropy terms of PPOAgent.get_loss, each Σ_n(·)·w_n / denom with
  denom = T·global_batch (the mean over time, then the sum over the batch / global batch)."""
  ratio = torch.exp(logp - old_logp)
  obj = ratio * adv
  if clip_eps > 0:
    obj = tf_min(obj, torch.clamp(ratio, 1 - clip_eps, 1 + clip_eps) * adv)
  err = (ret - v) ** 2
  if value_clip > 0:
    vc = v_old + torch.clamp(v - v_old, -value_clip, value_clip)
    err = tf_max(err, (ret - vc) ** 2)
  return ((-obj * w).sum() + vf_coef * (err * w).sum() + ent_coef * (-entropy * w).sum()) / denom


def kl_penalty(kl, w, n_global, kl_cutoff_factor, adaptive_kl_target, kl_cutoff_coef, beta):
  """kl_cutoff_loss + adaptive_kl_loss of mean_kl = Σ w·KL(old ‖ new) / N_global."""
  mean_kl = (kl * w).sum() / n_global
  out = beta * mean_kl
  if kl_cutoff_factor > 0:
    over = torch.clamp(mean_kl - kl_cutoff_factor * adaptive_kl_target, min=0.0)
    out = out + kl_cutoff_coef * over * over
  return out


def l2_loss(kernels, coef):
  """coef · Σ kernel² over the given kernels (biases are not regularised)."""
  return coef * sum((k * k).sum() for k in kernels)


# ---- DQN ------------------------------------------------------------------------------------------
def huber(err):
  a = err.abs()
  q = torch.clamp(a, max=1.0)
  return 0.5 * q * q + (a - q)


def n_step_targets(reward, discount, next_q, gamma, reward_scale):
  """reward / discount [B, T], next_q [B] (the bootstrap value at step T-1): n = T-1 step target
  reward_scale·Σ_k γ^k Π_{j<k} d_j r_k + γ^n Π_{j<n} d_j · next_q."""
  n = reward.shape[1] - 1
  R = torch.zeros_like(next_q)
  for k in range(n - 1, -1, -1):
    R = R * (gamma * discount[:, k]) + reward[:, k]
  D = gamma ** n * torch.prod(discount[:, :n], dim=1)
  return reward_scale * R + D * next_q


def clip_by_norm(g, clip):
  """tf.clip_by_norm: g · clip / max(‖g‖, clip)."""
  return g * (clip / torch.clamp(g.norm(), min=clip))
