"""PPO agent on libb200rl.

Drop-in for `tf_agents.agents.ppo.ppo_agent.PPOAgent` restricted to what PPOClipAgent uses
(reference agents/ppo/ppo_agent.py:114-1076, ppo_clip_agent.py:70-233): clipped-ratio
surrogate, value loss (optionally clipped), entropy bonus, L2 regularisation, GAE / TD-lambda
returns, advantage normalisation, observation / reward normalisers, `num_epochs` full-batch
updates per `train` call with global-norm clipping and ONE optimiser over actor + value
parameters, and the KL penalty of the original formulation (ppo_agent.py:1514-1690): squared
KL-cutoff loss + adaptive-beta loss inside every epoch, beta updated once after the epochs.
PPOClipAgent sets both to zero (ppo_clip_agent.py:226-232) and skips that work entirely.
The policy is a diagonal Normal for a continuous action spec and a Categorical over logits for a
discrete one (ppo_agent.py:48, actor_distribution_network.py:157-158); `_train` is shared and only
the behaviour log-probs, the loss launch, the KL and the actor backward follow the distribution.

Device work of `train(experience[B, T])` (csrc/ppo.cu, scans.cu, nn.cu, optim.cu):
  value net on B*T observations -> gamma*d*episode_mask -> returns scan -> GAE scan (warp-shuffle
  affine scans over T-1 steps) -> trajectory mask/weights -> behaviour log-probs -> advantage
  moments + normalisation, then per epoch: actor + value forward, fused surrogate/value/entropy
  loss with gradients, backward, global-norm scale, fused Adam on the joint flat buffer.
A recurrent actor or value net (ActorDistributionRnnNetwork, ValueRnnNetwork) runs over the whole
[B, T] sequence from the zero state with the step-type resets in the three network passes: the
value pass of preprocessing, each epoch's forward and backward, and the post-epoch KL pass
(ppo_agent.py:525-530, 981-986).  The loss kernels, GAE and the optimiser step are unchanged over
the N = B*T rows.
"""
import collections
import ctypes

import torch

from agents_b200 import _lib
from agents_b200.agents import tf_agent
from agents_b200.agents.ppo import ppo_policy
from agents_b200.networks import network as network_lib
from agents_b200.policies import actor_policy
from agents_b200.specs import tensor_spec
from agents_b200.trajectories import trajectory
from agents_b200.utils import nest
from agents_b200.utils import tensor_normalizer
from agents_b200.utils import workspace

PPOLossInfo = collections.namedtuple('PPOLossInfo', (
    'policy_gradient_loss', 'value_estimation_loss', 'l2_regularization_loss',
    'entropy_regularization_loss', 'kl_penalty_loss', 'clip_fraction'))


class PPOAgent(tf_agent.TFAgent):
  """A PPO agent (Schulman et al. 2017), clipped-surrogate form."""

  def __init__(self, time_step_spec, action_spec, optimizer=None, actor_net=None,
               value_net=None, greedy_eval=True, importance_ratio_clipping=0.0,
               lambda_value=0.95, discount_factor=0.99, entropy_regularization=0.0,
               policy_l2_reg=0.0, value_function_l2_reg=0.0, shared_vars_l2_reg=0.0,
               value_pred_loss_coef=0.5, num_epochs=25, use_gae=False,
               use_td_lambda_return=False, normalize_rewards=True, reward_norm_clipping=10.0,
               normalize_observations=True, log_prob_clipping=0.0, kl_cutoff_factor=2.0,
               kl_cutoff_coef=1000.0, initial_adaptive_kl_beta=1.0, adaptive_kl_target=0.01,
               adaptive_kl_tolerance=0.3, gradient_clipping=None, value_clipping=None,
               check_numerics=False, compute_value_and_advantage_in_train=True,
               update_normalizers_in_train=True, aggregate_losses_across_replicas=True,
               debug_summaries=False, summarize_grads_and_vars=False, train_step_counter=None,
               name=None, seed=0):
    if actor_net is None or value_net is None:
      raise ValueError('actor_net and value_net must be given.')
    actor_policy.reject_tanh_normal(actor_net, 'PPOAgent')
    if not use_gae:
      raise NotImplementedError('Only use_gae=True is supported (PPO examples use GAE).')
    if shared_vars_l2_reg:
      raise NotImplementedError('shared_vars_l2_reg needs shared actor/value variables.')
    self._optimizer = optimizer
    self._actor_net, self._value_net = actor_net, value_net
    actor_net.create_variables(time_step_spec.observation)
    value_net.create_variables(time_step_spec.observation)
    self._flat_params, self._flat_grads = network_lib.allocate_jointly([actor_net, value_net])
    device = actor_net.device
    self._importance_ratio_clipping = importance_ratio_clipping
    self._lambda, self._discount_factor = lambda_value, discount_factor
    self._entropy_regularization = entropy_regularization
    self._policy_l2_reg, self._value_function_l2_reg = policy_l2_reg, value_function_l2_reg
    self._value_pred_loss_coef = value_pred_loss_coef
    # KL penalty configuration (ppo_agent.py:319-345); beta is a device-resident variable
    self._kl_cutoff_factor = float(kl_cutoff_factor)
    self._kl_cutoff_coef = float(kl_cutoff_coef)
    self._initial_adaptive_kl_beta = float(initial_adaptive_kl_beta)
    self._adaptive_kl_target = float(adaptive_kl_target)
    self._adaptive_kl_tolerance = float(adaptive_kl_tolerance)
    self._adaptive_kl_beta = None
    if initial_adaptive_kl_beta > 0.0:
      self._adaptive_kl_beta = torch.full((1,), float(initial_adaptive_kl_beta),
                                          dtype=torch.float32, device=device)
    self._kl_mean = torch.zeros(1, dtype=torch.float32, device=device)
    self._kl_terms = torch.zeros(3, dtype=torch.float32, device=device)
    self._num_epochs = num_epochs
    self._use_td_lambda_return = use_td_lambda_return
    self._reward_norm_clipping = reward_norm_clipping
    self._log_prob_clipping = log_prob_clipping
    self._gradient_clipping = gradient_clipping or 0.0
    self._value_clipping = value_clipping or 0.0
    self.update_normalizers_in_train = update_normalizers_in_train
    self._compute_value_and_advantage_in_train = compute_value_and_advantage_in_train
    self._reward_normalizer = None
    if normalize_rewards:
      self._reward_normalizer = tensor_normalizer.StreamingTensorNormalizer(
          time_step_spec.reward, scope='normalize_reward', device=device)
    self._observation_normalizer = None
    if normalize_observations:
      self._observation_normalizer = tensor_normalizer.StreamingTensorNormalizer(
          time_step_spec.observation, scope='normalize_observations', device=device)
    policy = ppo_policy.PPOPolicy(time_step_spec, action_spec, actor_net, value_net,
                                  self._observation_normalizer, clip=False, collect=False)
    collect_policy = ppo_policy.PPOPolicy(
        time_step_spec, action_spec, actor_net, value_net, self._observation_normalizer,
        clip=False, collect=True,
        compute_value_and_advantage_in_train=compute_value_and_advantage_in_train, seed=seed)
    # training_data_spec = collect_data_spec + {'return', 'advantage'} when the advantages are
    # computed by preprocess_sequence in the data pipeline (ppo_agent.py:394-409)
    training_data_spec = None
    if not compute_value_and_advantage_in_train:
      info = dict(collect_policy.info_spec)
      info['return'] = tensor_spec.TensorSpec((), torch.float32, 'return')
      info['advantage'] = tensor_spec.TensorSpec((), torch.float32, 'advantage')
      training_data_spec = collect_policy.trajectory_spec._replace(policy_info=info)
    super(PPOAgent, self).__init__(
        time_step_spec, action_spec, policy, collect_policy, train_sequence_length=None,
        training_data_spec=training_data_spec, debug_summaries=debug_summaries, summarize_grads_and_vars=summarize_grads_and_vars,
        train_step_counter=train_step_counter, device=device)
    self._nan_flag = torch.zeros(1, dtype=torch.int32, device=device)
    self._scale_dev = torch.ones(1, dtype=torch.float32, device=device)
    self._norm_dev = torch.zeros(1, dtype=torch.float32, device=device)
    self.replicas = 1
    self._grad_sync = None       # callable(flat_grads) for data-parallel runs (train.Learner)
    self._stat_sync = None       # callable(tensor) SUM-all-reduce of small statistics
    self._replica_rank = 0       # this process's index among `replicas` (set by train.Learner)

  @property
  def actor_net(self):
    return self._actor_net

  @property
  def value_net(self):
    return self._value_net

  def _initialize(self):
    pass

  # ---- preprocessing (ppo_agent.py:617-807) ---------------------------------------------------
  def _flat_obs(self, experience):
    obs = nest.flatten(experience.observation)[0]
    B, T = obs.shape[0], obs.shape[1]
    return obs.reshape((B * T,) + tuple(obs.shape[2:])).contiguous(), B, T

  def _preprocess(self, experience):
    """Returns (value_preds, returns, advantages), each [B, T] with a zero last column."""
    obs, B, T = self._flat_obs(experience)
    if T <= 1:
      raise ValueError('Experience used for advantage calculation must have >1 num_steps.')
    dev = obs.device
    if self._compute_value_and_advantage_in_train:
      vp, _ = self._collect_policy.apply_value_network(obs, *self._seq(self._value_net, experience))
      vp = vp.reshape(B, T).contiguous()
    else:                                                         # :775-776
      vp = experience.policy_info['value_prediction'].float().reshape(B, T).contiguous()
    reward = experience.reward.float().contiguous()
    if self._reward_normalizer is not None:                       # :651-654
      reward = self._reward_normalizer.normalize(reward, center_mean=False,
                                                 clip_value=self._reward_norm_clipping)
    disc = torch.empty((B, T), dtype=torch.float32, device=dev)
    _lib.call('b200rl_ppo_discounts', _lib.ptr(experience.discount.float().contiguous()),
              _lib.ptr(experience.next_step_type.to(torch.int32).contiguous()),
              float(self._discount_factor), B * T, _lib.ptr(disc), _lib.stream())
    returns = torch.zeros((B, T), dtype=torch.float32, device=dev)
    adv = torch.zeros((B, T), dtype=torch.float32, device=dev)
    # returns bootstrap from V[:, T-1] (:662-668); GAE from V[:, T-2] (sic, :464-470)
    _lib.call('b200rl_discounted_return_ld', _lib.ptr(reward), _lib.ptr(disc),
              vp.data_ptr() + 4 * (T - 1), _lib.ptr(returns), B, T - 1, T, T, T, _lib.stream())
    _lib.call('b200rl_gae_ld', _lib.ptr(vp), vp.data_ptr() + 4 * (T - 2), _lib.ptr(disc),
              _lib.ptr(reward), float(self._lambda), _lib.ptr(adv), B, T - 1, T, T, T,
              _lib.stream())
    if self._use_td_lambda_return:                                # :708-717
      returns[:, :-1] = adv[:, :-1] + vp[:, :-1]
    return vp, returns, adv

  def preprocess_sequence(self, experience):
    """`_preprocess_sequence` (ppo_agent.py:809-832): a no-op when the advantages are computed
    inside train(); otherwise returns `experience` with `value_prediction`, `return` and
    `advantage` (zero for the last step) in its policy_info, for use as
    `replay_buffer.as_dataset(sequence_preprocess_fn=agent.preprocess_sequence)`."""
    if self._compute_value_and_advantage_in_train:
      return experience
    squeeze = experience.discount.dim() == 1                      # [T, ...] -> [1, T, ...]
    if squeeze:
      experience = nest.map_structure(lambda t: t.unsqueeze(0), experience)
    vp, returns, adv = self._preprocess(experience)
    info = {'dist_params': experience.policy_info['dist_params'], 'value_prediction': vp,
            'return': returns, 'advantage': adv}
    out = experience._replace(policy_info=info)
    if squeeze:
      out = nest.map_structure(lambda t: t.squeeze(0), out)
    return out

  @property
  def recurrent(self):
    return bool(self._actor_net.state_spec or self._value_net.state_spec)

  @staticmethod
  def _seq(net, experience):
    """Extra arguments of a network pass over the flattened [B, T] rows: the step types for a
    recurrent net (its sequences start from the zero state), none for a feed-forward one."""
    return (experience.step_type,) if net.state_spec else ()

  # ---- train (ppo_agent.py:834-1076) ------------------------------------------------------------
  def _train(self, experience, weights=None):
    if self._optimizer is None:
      raise ValueError('Optimizer is undefined.')
    if self.recurrent and self.replicas > 1:
      raise NotImplementedError('PPOAgent with a recurrent network trains on one replica.')
    if not isinstance(experience, trajectory.Trajectory):
      raise TypeError('Input type not supported: {}'.format(type(experience)))
    tf_agent.validate_trajectory(experience, self.training_data_spec, None)
    obs, B, T = self._flat_obs(experience)
    N = B * T
    dev = obs.device
    A = self._actor_net.num_actions
    ws, nb = workspace.get(dev)
    st = _lib.stream()
    if self._compute_value_and_advantage_in_train:
      vp, returns, adv = self._preprocess(experience)
    else:                                                         # :843-846, :890-891, :908
      info = experience.policy_info
      vp, returns, adv = (info[k].float().reshape(B, T).contiguous()
                          for k in ('value_prediction', 'return', 'advantage'))
    w = torch.empty(N, dtype=torch.float32, device=dev)
    if weights is not None:
      weights = torch.as_tensor(weights, dtype=torch.float32, device=dev).expand(B, T).contiguous()
    _lib.call('b200rl_ppo_weights', _lib.ptr(experience.step_type.to(torch.int32).contiguous()),
              _lib.ptr(returns), _lib.ptr(adv), _lib.ptr(weights), N, _lib.ptr(w), st)
    discrete = self._actor_net.discrete
    old = experience.policy_info['dist_params']
    old_logp = torch.empty(N, dtype=torch.float32, device=dev)
    if discrete:                                                  # integer actions read as int32
      action = experience.action.reshape(N).to(torch.int32).contiguous()
      old_params = old['logits'].float().reshape(N, A).contiguous()
      _lib.call('b200rl_categorical_logp', _lib.ptr(old_params), A, _lib.ptr(action), N, A,
                _lib.ptr(old_logp), _lib.ptr(self._nan_flag), st)
    else:
      action = experience.action.float().reshape(N, A).contiguous()
      old_loc = old['loc'].float().reshape(N, A).contiguous()
      old_scale = old['scale'].float().reshape(N, A).contiguous()
      old_params = (old_loc, old_scale)
      _lib.call('b200rl_normal_logp', _lib.ptr(old_loc), _lib.ptr(old_scale), A, _lib.ptr(action),
                N, A, _lib.ptr(old_logp), st)
    # _normalize_advantages over axes (0, 1), unmasked (:893-895, :100-110); sharded runs merge
    # the per-rank moments with one collective (tensor_normalizer.batch_moments)
    mean = torch.empty(1, dtype=torch.float32, device=dev)
    var = torch.empty(1, dtype=torch.float32, device=dev)
    n_glob = float(N * self.replicas)
    tensor_normalizer.batch_moments(adv.reshape(N, 1), 1, mean, var, self._stat_sync,
                                    self.replicas, self._replica_rank)
    var.mul_(1.0 / n_glob)                                         # m2 -> population variance
    adv_n = torch.empty(N, dtype=torch.float32, device=dev)
    _lib.call('b200rl_normalize', _lib.ptr(adv), _lib.ptr(adv_n), N, 1, _lib.ptr(mean),
              _lib.ptr(var), None, 1e-8, 0.0, st)
    obs_n = obs
    if self._observation_normalizer is not None:
      obs_n = self._observation_normalizer.normalize(obs)
    losses = torch.empty(6, dtype=torch.float32, device=dev)
    use_kl = not (self._initial_adaptive_kl_beta == 0 and self._kl_cutoff_factor == 0)  # :586
    kl_arg = None
    if use_kl:
      # mean_kl is the mean over the GLOBAL batch (per-rank partial sums are SUM-reduced) and the
      # KL gradient carries 1/N_global, so R replicas reproduce the one-device update on the
      # concatenated batch (the reference's per-replica reduce_mean would weigh the penalty R x).
      if discrete:
        kl_arg = _lib.PpoKlLogits(_lib.ptr(old_params), A, _lib.ptr(self._kl_terms), 1.0 / n_glob)
      else:
        kl_arg = _lib.PpoKl(_lib.ptr(old_loc), _lib.ptr(old_scale), A, _lib.ptr(self._kl_terms),
                            1.0 / n_glob)
    l2 = torch.zeros(1, dtype=torch.float32, device=dev)
    if discrete:
      dlogits = torch.empty((N, A), dtype=torch.float32, device=dev)
    else:
      dloc = torch.empty((N, A), dtype=torch.float32, device=dev)
      dscale = torch.empty((N, A), dtype=torch.float32, device=dev)
    dv = torch.empty((N, 1), dtype=torch.float32, device=dev)
    gb = float(B * self.replicas)
    scalars = (float(self._importance_ratio_clipping), float(self._value_clipping),
               float(self._value_pred_loss_coef), float(self._entropy_regularization),
               float(self._log_prob_clipping))
    aseq = self._seq(self._actor_net, experience)
    vseq = self._seq(self._value_net, experience)
    for _ in range(self._num_epochs):                             # :925-967
      params, actx = self._actor_net.forward_train(obs_n, *aseq)
      v, vtape = self._value_net.forward_train(obs_n, *vseq)
      if use_kl:
        self._mean_kl(params, old_params, w, N, A, n_glob)
        self._kl_penalty_terms()
      if discrete:
        _lib.call('b200rl_ppo_loss_categorical', _lib.ptr(params), A, _lib.ptr(action),
                  _lib.ptr(old_logp), _lib.ptr(adv_n), _lib.ptr(returns), _lib.ptr(v),
                  _lib.ptr(vp), _lib.ptr(w), N, A, T, gb, *scalars, _lib.ptr(losses),
                  _lib.ptr(dlogits), A, _lib.ptr(dv), _lib.ptr(self._nan_flag),
                  ctypes.byref(kl_arg) if use_kl else None, _lib.ptr(ws), nb, st)
        self._actor_net.backward(actx, dlogits)
      else:
        loc, scale = params
        _lib.call('b200rl_ppo_loss', _lib.ptr(loc), _lib.ptr(scale), A, _lib.ptr(action),
                  _lib.ptr(old_logp), _lib.ptr(adv_n), _lib.ptr(returns), _lib.ptr(v),
                  _lib.ptr(vp), _lib.ptr(w), N, A, T, gb, *scalars, _lib.ptr(losses),
                  _lib.ptr(dloc), _lib.ptr(dscale), A, _lib.ptr(dv), _lib.ptr(self._nan_flag),
                  ctypes.byref(kl_arg) if use_kl else None, _lib.ptr(ws), nb, st)
        self._actor_net.backward(actx, (dloc, dscale))
      self._value_net.backward(vtape, dv)
      l2.zero_()
      self._l2_regularization(l2)
      if self._grad_sync is not None:
        self._grad_sync(self._flat_grads)
      scale_dev = None
      if self._gradient_clipping > 0:                             # tf.clip_by_global_norm :948-949
        _lib.call('b200rl_global_norm_scale', _lib.ptr(self._flat_grads), self._flat_grads.numel(),
                  float(self._gradient_clipping), _lib.ptr(self._scale_dev),
                  _lib.ptr(self._norm_dev), _lib.ptr(ws), nb, st)
        scale_dev = self._scale_dev
      self._optimizer.apply_flat(self._flat_params, self._flat_grads, scale_dev)
      self._bump_train_step(1)
    if self._initial_adaptive_kl_beta > 0:                        # :978-989
      params = self._actor_net.distribution_params(obs_n, *aseq)
      if aseq:
        params = params[0]                                        # (params, final state)
      self._mean_kl(params, old_params, w, N, A, n_glob)
      self._update_beta()
    if self.update_normalizers_in_train:                          # :991-993
      self.update_observation_normalizer(obs)
      self.update_reward_normalizer(experience.reward)
    zero = torch.zeros((), dtype=torch.float32, device=dev)
    extra = PPOLossInfo(policy_gradient_loss=losses[0], value_estimation_loss=losses[1],
                        l2_regularization_loss=l2.reshape(()),
                        entropy_regularization_loss=losses[2],
                        kl_penalty_loss=losses[5] if use_kl else zero, clip_fraction=losses[3])
    return tf_agent.LossInfo(losses[4] + l2.reshape(()), extra)

  # ---- KL penalty (ppo_agent.py:1514-1690) ------------------------------------------------------
  def _mean_kl(self, params, old_params, w, N, A, n_glob, out_kl=None):
    """self._kl_mean <- sum_n w_n KL(old_n || new_n) / N_global (all-reduced when sharded).
    params / old_params: [N, A] logits (Categorical) or (loc, scale) pairs (Normal)."""
    if self._actor_net.discrete:
      ws, nb = workspace.get(params.device)
      _lib.call('b200rl_ppo_kl_categorical', _lib.ptr(params), A, _lib.ptr(old_params), A,
                _lib.ptr(w), N, A, 1.0 / n_glob, _lib.ptr(out_kl), _lib.ptr(self._kl_mean),
                _lib.ptr(ws), nb, _lib.stream())
    else:
      (loc, scale), (old_loc, old_scale) = params, old_params
      ws, nb = workspace.get(loc.device)
      _lib.call('b200rl_ppo_kl', _lib.ptr(loc), _lib.ptr(scale), A, _lib.ptr(old_loc),
                _lib.ptr(old_scale), A, _lib.ptr(w), N, A, 1.0 / n_glob, _lib.ptr(out_kl),
                _lib.ptr(self._kl_mean), _lib.ptr(ws), nb, _lib.stream())
    if self._stat_sync is not None:
      self._stat_sync(self._kl_mean)

  def _kl_penalty_terms(self):
    _lib.call('b200rl_ppo_kl_terms', _lib.ptr(self._kl_mean), _lib.ptr(self._adaptive_kl_beta),
              self._kl_cutoff_factor, self._adaptive_kl_target, self._kl_cutoff_coef,
              _lib.ptr(self._kl_terms), _lib.stream())

  def _update_beta(self):
    _lib.call('b200rl_ppo_kl_beta_update', _lib.ptr(self._kl_mean),
              _lib.ptr(self._adaptive_kl_beta), self._adaptive_kl_target,
              self._adaptive_kl_tolerance, _lib.stream())

  def _set_mean_kl(self, kl_divergence):
    kl = torch.as_tensor(kl_divergence, dtype=torch.float32, device=self._kl_mean.device)
    kl = kl.reshape(-1).contiguous()
    ws, nb = workspace.get(kl.device)
    _lib.call('b200rl_colsum', _lib.ptr(kl), None, 0, kl.numel(), 1, 1.0 / kl.numel(),
              _lib.ptr(self._kl_mean), _lib.ptr(ws), nb, _lib.stream())

  def kl_cutoff_loss(self, kl_divergence, debug_summaries=False):
    """coef * max(mean(kl) - factor * target, 0)^2 (ppo_agent.py:1514-1539)."""
    self._set_mean_kl(kl_divergence)
    self._kl_penalty_terms()
    return self._kl_terms[0].clone()

  def adaptive_kl_loss(self, kl_divergence, debug_summaries=False):
    """beta * mean(kl) (ppo_agent.py:1541-1558)."""
    self._set_mean_kl(kl_divergence)
    self._kl_penalty_terms()
    return self._kl_terms[1].clone()

  def update_adaptive_kl_beta(self, kl_divergence):
    """beta <- clip(beta * {1/1.5, 1, 1.5}) depending on mean(kl) vs target*(1 -/+ tolerance)
    (ppo_agent.py:1632-1675); returns beta."""
    if self._adaptive_kl_beta is None:
      return None
    self._set_mean_kl(kl_divergence)
    self._update_beta()
    return self._adaptive_kl_beta[0].clone()

  def kl_penalty_loss(self, time_steps, action_distribution_parameters,
                      current_policy_distribution, weights, debug_summaries=False):
    """kl_cutoff_loss + adaptive_kl_loss of weights * KL(old || current) (:1586-1630).
    `current_policy_distribution` is a (loc, scale) pair of [N, A] tensors, or the [N, A] logits
    for a discrete action (then `action_distribution_parameters` holds 'logits')."""
    flat = lambda t: t.float().reshape(-1, t.shape[-1]).contiguous()
    if self._actor_net.discrete:
      params = flat(current_policy_distribution)
      old_params = flat(action_distribution_parameters['logits'])
      dev, (N, A) = params.device, params.shape
    else:
      params = tuple(flat(t) for t in current_policy_distribution)
      old_params = (flat(action_distribution_parameters['loc']),
                    flat(action_distribution_parameters['scale']))
      dev, (N, A) = params[0].device, params[0].shape
    w = torch.as_tensor(weights, dtype=torch.float32, device=dev).reshape(-1).contiguous()
    kl = torch.empty(N, dtype=torch.float32, device=dev)
    self._mean_kl(params, old_params, w, N, A, float(N * self.replicas), out_kl=kl)
    # through the public methods, like the reference (its test mocks them)
    return self.kl_cutoff_loss(kl, debug_summaries) + self.adaptive_kl_loss(kl, debug_summaries)

  def _l2_regularization(self, l2_accum):
    """l2_regularization_loss (:1088-1157): coef * sum(kernel^2) over kernels (not biases);
    adds the loss into `l2_accum` and its gradient into the flat gradient buffer."""
    for net, coef in ((self._actor_net, self._policy_l2_reg),
                      (self._value_net, self._value_function_l2_reg)):
      if not coef:
        continue
      for l in net.layers:
        if getattr(l, 'kernel', None) is None:
          continue
        # every variable named '*kernel*' (:1097-1103): an LSTM's recurrent_kernel too
        pairs = [(l.kernel, l.d_kernel)]
        if getattr(l, 'recurrent_kernel', None) is not None:
          pairs.append((l.recurrent_kernel, l.d_recurrent_kernel))
        for k, dk in pairs:
          _lib.call('b200rl_l2_sum', _lib.ptr(k), k.numel(), float(coef) / self.replicas,
                    _lib.ptr(l2_accum), _lib.stream())
          _lib.call('b200rl_add_scaled', _lib.ptr(dk), _lib.ptr(k), k.numel(),
                    2.0 * float(coef) / self.replicas, _lib.stream())

  def update_observation_normalizer(self, batched_observations):
    if self._observation_normalizer is not None:
      self._observation_normalizer.update(batched_observations, stat_sync=self._stat_sync,
                                          replicas=self.replicas, rank=self._replica_rank)

  def update_reward_normalizer(self, batched_rewards):
    if self._reward_normalizer is not None:
      self._reward_normalizer.update(batched_rewards, stat_sync=self._stat_sync,
                                     replicas=self.replicas, rank=self._replica_rank)

  def check_numerics(self):
    if int(self._nan_flag.item()) != 0:
      raise FloatingPointError('Loss is inf or nan')
