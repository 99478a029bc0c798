"""CEMPolicy (tf_agents/policies/qtopt_cem_policy.py): the action that a cross-entropy-method
search finds best under a critic Q(s, a), for one rank-1 bounded float action.

Per state the search starts from N(init_mean, init_var) and, num_iterations times: floors the
variance at minimal_var, draws num_samples (N) actions and clips them to the spec, scores all B*N
(state, action) pairs with the critic, keeps the top num_elites (M) (tf.nn.top_k: ties to the
lower index) and refits mean and var to them (tf.nn.moments).  The action is the best sample of
the LAST iteration, as in the reference (not the best over all iterations); it is deterministic
given the draws.

Device work per search (csrc/qtopt.cu): one b200rl_cem_sample launch, which also tiles the
observation (or, with an observation branch, h_obs computed on the B rows only) into the critic's
[B*N, W] joint-stack input, then num_iterations x (critic joint-stack forward over the B*N rows +
one b200rl_cem_refit launch, which selects, refits and draws the next samples straight into the
input, or writes the best action and score on the last iteration).  The Philox call counter is a
device tensor, so a captured search draws fresh samples on every replay.

Not supported (raise): actor_policy, emit_log_probability, preprocess_state_action=False, the
one-hot / hybrid samplers' weights, RNN critics, and info specs (the target_q info of
in_graph_bellman_update=False).

Extension (keyword-only): `search(observation, z=...)` supplies the N(0, 1) draws z
[num_iterations, B, N, A], so parity tests are independent of the RNG stream.
"""
import numpy as np
import torch

from agents_b200 import _lib
from agents_b200.policies import tf_policy
from agents_b200.trajectories import policy_step
from agents_b200.utils import nest

_CEM_SEED_TAG = 0x43454D5F504F4C49


class CEMPolicy(tf_policy.TFPolicy):
  """Cross-entropy-method action search over a critic."""

  def __init__(self, time_step_spec, action_spec, q_network, sampler, init_mean, init_var,
               actor_policy=None, minimal_var=0.0001, info_spec=(), num_samples=32, num_elites=4,
               num_iterations=32, emit_log_probability=False, preprocess_state_action=True,
               training=False, weights=None, name=None, seed=0):
    if actor_policy is not None:
      raise NotImplementedError('CEMPolicy does not support actor_policy.')
    if emit_log_probability:
      raise NotImplementedError('CEMPolicy does not support emit_log_probability.')
    if not preprocess_state_action:
      raise NotImplementedError('CEMPolicy always tiles the state (preprocess_state_action).')
    if weights is not None:
      raise NotImplementedError('CEM weights belong to the one-hot sampler, which is not '
                                'supported.')
    if info_spec:
      raise NotImplementedError('CEMPolicy emits no policy info (in_graph_bellman_update=False '
                                'is not supported).')
    if getattr(q_network, 'state_spec', ()):
      raise NotImplementedError('CEMPolicy supports stateless (non-RNN) critics only.')
    flat = nest.flatten(action_spec)
    if len(flat) != 1 or not flat[0].dtype.is_floating_point or len(flat[0].shape) != 1:
      raise ValueError('CEMPolicy supports one rank-1 bounded float action.')
    if init_mean is None or init_var is None:
      raise ValueError('init_mean and init_var are required.')
    if not 1 <= int(num_elites) <= int(num_samples):
      raise ValueError('num_elites must be in [1, num_samples].')
    if int(num_iterations) < 1:
      raise ValueError('num_iterations must be >= 1.')
    super().__init__(time_step_spec, action_spec, info_spec=(), name=name)
    q_network.create_variables()
    self._q_network = q_network
    self._sampler = sampler
    A = int(flat[0].shape[0])
    self._num_actions = A
    device = q_network.device
    self._init_mean = torch.as_tensor(
        np.broadcast_to(np.asarray(init_mean, np.float32), (A,)).copy(), device=device)
    self._init_var = torch.as_tensor(
        np.broadcast_to(np.asarray(init_var, np.float32), (A,)).copy(), device=device)
    self._amin, self._amax = sampler.bounds(device)
    self._minimal_var = float(minimal_var)
    self._num_samples, self._num_elites = int(num_samples), int(num_elites)
    self._num_iterations = int(num_iterations)
    self._training = training
    self._seed = (int(seed) ^ _CEM_SEED_TAG) & 0xFFFFFFFFFFFFFFFF
    self._cem_rng = torch.zeros(2, dtype=torch.int64, device=device)

  @property
  def q_network(self):
    return self._q_network

  def variables(self):
    return self._q_network.variables

  def search(self, observation, z=None):
    """(best_action [B, A], best_score [B]) of a CEM search at observation [B, D]."""
    net, A = self._q_network, self._num_actions
    N, M, I = self._num_samples, self._num_elites, self._num_iterations
    obs = nest.flatten(observation)[0].float()
    if obs.stride(-1) != 1:
      obs = obs.contiguous()
    B, dev = obs.shape[0], obs.device
    if net.has_observation_branch:
      src, _ = net.observation_features(obs)
    else:
      src = obs
    C = src.shape[1]
    if z is not None:
      z = z.float().contiguous()
      if tuple(z.shape) != (I, B, N, A):
        raise ValueError('z must be [num_iterations, B, num_samples, A] = {}, got {}'.format(
            (I, B, N, A), tuple(z.shape)))
    zi = lambda i: None if z is None else z[i].data_ptr()
    rng, st = _lib.ptr(self._cem_rng), _lib.stream()
    lo, hi = _lib.ptr(self._amin), _lib.ptr(self._amax)
    x = torch.empty((B * N, C + A), dtype=torch.float32, device=dev)
    mean = torch.empty((B, A), dtype=torch.float32, device=dev)
    var = torch.empty_like(mean)
    best_action = torch.empty_like(mean)
    best_score = torch.empty(B, dtype=torch.float32, device=dev)
    _lib.call('b200rl_cem_sample', _lib.dptr(src), src.stride(0), B, N, C, A,
              _lib.ptr(self._init_mean), 0, _lib.ptr(self._init_var), 0, self._minimal_var, lo,
              hi, zi(0), self._seed, rng, _lib.ptr(x), C + A, st)
    for i in range(I):
      q, _ = net.forward_stack(x)
      last = i == I - 1
      _lib.call('b200rl_cem_refit', _lib.ptr(q), None, _lib.ptr(x), C + A, C, B, N, M, A,
                self._minimal_var, lo, hi, int(last), None if last else zi(i + 1), self._seed,
                rng, _lib.ptr(mean), _lib.ptr(var), _lib.ptr(best_action), _lib.ptr(best_score),
                st)
    return best_action, best_score

  def _action(self, time_step, policy_state, seed):
    best_action, _ = self.search(time_step.observation)
    return policy_step.PolicyStep(best_action, policy_state, ())

  def distribution(self, time_step, policy_state=()):
    raise NotImplementedError('CEMPolicy emits its action directly (a Deterministic '
                              'distribution in the reference); use action().')
