"""Learner (tf_agents/train/learner.py:42-378): pulls experience from a dataset and runs
`agent.train` `iterations` times per `run` call, under a distribution strategy.

Reference behaviour kept: `run(iterations, iterator)` -> LossInfo of the last step reduced with
SUM over replicas (:322-336); triggers are called after every `run` (:301-303); the agent
(parameters + optimiser slots + train_step) is checkpointed every `checkpoint_interval` train
steps and the latest checkpoint is restored on construction (:231-243); per-replica losses are
divided by the global batch inside the agent (utils/common.py:1465-1467).

What is different: there is no tf.function/while_loop — each step only enqueues launches on
the CUDA stream; with `strategy.num_replicas_in_sync > 1` the learner installs ONE flat-buffer
SUM all-reduce per optimiser step into the agent (`agent._grad_sync`) and broadcasts rank 0's
parameters at start so replicas are mirrored.
"""
import os

import torch

from agents_b200.agents import tf_agent
from agents_b200.train.utils import strategy_utils
from agents_b200.utils import nest

TRAIN_DIR = 'train'
POLICY_SAVED_MODEL_DIR = 'policies'


def _agent_state_tensors(agent):
  """Flat parameter / slot tensors that define the agent's state (for mirroring + checkpoints)."""
  out = {}
  for name in ('_q_network', '_target_q_network', '_actor_net', '_value_net', '_actor_network',
               '_value_network', '_critic_network_1', '_critic_network_2', '_target_critic_network_1',
               '_target_critic_network_2', '_target_actor_network', '_critic_network',
               '_target_critic_network', '_target_q_network_delayed',
               '_target_q_network_delayed_2', '_cloning_network'):
    net = getattr(agent, name, None)
    if net is not None and hasattr(net, 'flat_params'):
      out[name] = net.flat_params
  # OUNoisePolicy's process value and Philox counter (agent-tracked variables in the reference),
  # so a restored run draws the exploration noise it would have drawn
  collect = getattr(agent, '_collect_policy', None)
  for name in ('_ou_state', '_ou_rng'):
    t = getattr(collect, name, None)
    if isinstance(t, torch.Tensor):
      out['_collect_policy/' + name] = t
  # QT-Opt: the Philox counters of the float epsilon-greedy draw and of CEMPolicy's search (the
  # train step searches with the same policy), so a restored run draws what it would have drawn
  t = getattr(collect, '_uniform_rng', None)
  if isinstance(t, torch.Tensor):
    out['_collect_policy/_uniform_rng'] = t
  t = getattr(getattr(agent, '_policy', None), '_cem_rng', None)
  if isinstance(t, torch.Tensor):
    out['_policy/_cem_rng'] = t
  # SAC temperature; CQL-SAC's weight (a device scalar, or log_cql_alpha with Lagrange); TD3's
  # target-smoothing and behavioral cloning's Normal-sample Philox counters (a restored run draws
  # the noise it would have drawn)
  for name in ('_log_alpha', '_cql_alpha', '_log_cql_alpha', '_target_noise_rng', '_sample_rng'):
    t = getattr(agent, name, None)
    if isinstance(t, torch.Tensor):
      out[name] = t
  # PPO: streaming normalisers (tf.Module variables of the agent in the reference, so they are
  # checkpointed and mirrored with it) and the adaptive KL coefficient (ppo_agent.py:341-343)
  for name in ('_observation_normalizer', '_reward_normalizer'):
    norm = getattr(agent, name, None)
    if norm is not None and hasattr(norm, 'variables'):
      for i, v in enumerate(norm.variables):
        out[f'{name}/{i}'] = v
  beta = getattr(agent, '_adaptive_kl_beta', None)
  if isinstance(beta, torch.Tensor):
    out['_adaptive_kl_beta'] = beta
  upd = getattr(agent, '_update_target', None)       # Periodically counter (a tf.Variable there)
  if isinstance(getattr(upd, '_counter', None), torch.Tensor):
    out['_update_target/counter'] = upd._counter
  for name in ('_target_updater_delayed', '_target_updater_delayed_2'):   # QT-Opt's delayed chain
    upd = getattr(agent, name, None)
    if isinstance(getattr(upd, '_counter', None), torch.Tensor):
      out[name + '/counter'] = upd._counter
  # optimiser slots are created lazily on the first apply; materialise them for the parameter
  # buffers each agent steps, so that a freshly built agent can be restored into
  pairs = (('_optimizer', '_flat_params'), ('_critic_optimizer', '_critic_params'),
           ('_alpha_optimizer', '_log_alpha'), ('_cql_alpha_optimizer', '_log_cql_alpha'))
  nets = (('_optimizer', '_q_network'), ('_actor_optimizer', '_actor_network'),
          ('_optimizer', '_cloning_network'))
  for oname, pname in pairs:
    opt, p = getattr(agent, oname, None), getattr(agent, pname, None)
    if hasattr(opt, '_get_slots') and isinstance(p, torch.Tensor):
      opt._get_slots(p)
  for oname, nname in nets:
    opt, net = getattr(agent, oname, None), getattr(agent, nname, None)
    if hasattr(opt, '_get_slots') and net is not None and hasattr(net, 'flat_params') and \
        not isinstance(getattr(agent, '_flat_params', None), torch.Tensor):
      opt._get_slots(net.flat_params)
  for oname in ('_optimizer', '_actor_optimizer', '_critic_optimizer', '_alpha_optimizer',
                '_cql_alpha_optimizer'):
    opt = getattr(agent, oname, None)
    if opt is not None and hasattr(opt, '_slots'):
      for i, slots in enumerate(opt._slots.values()):
        for k, v in slots.items():
          out[f'{oname}/{i}/{k}'] = v
  return out


class Learner(object):
  """Manages all the learning details needed when training an agent."""

  def __init__(self, root_dir, train_step, agent, experience_dataset_fn=None,
               after_train_strategy_step_fn=None, triggers=None, checkpoint_interval=100000,
               summary_interval=1000, max_checkpoints_to_keep=3,
               use_kwargs_in_agent_train=False, strategy=None, run_optimizer_variable_init=True,
               use_reverb_v2=False, direct_sampling=False, experience_dataset_options=None,
               strategy_run_options=None, summary_root_dir=None):
    if checkpoint_interval < 0:
      raise ValueError('checkpoint_interval must be >= 0.')
    self._train_dir = os.path.join(root_dir, TRAIN_DIR)
    self.train_step = train_step
    self._agent = agent
    self.use_kwargs_in_agent_train = use_kwargs_in_agent_train
    self.strategy = strategy or strategy_utils.get_strategy()
    self._after_train_strategy_step_fn = after_train_strategy_step_fn
    self.triggers = triggers or []
    self._checkpoint_interval = checkpoint_interval
    self._max_checkpoints_to_keep = max_checkpoints_to_keep
    self.direct_sampling = direct_sampling
    self._experience_iterator = None
    if experience_dataset_fn is not None:
      self._experience_iterator = iter(experience_dataset_fn())
    n = self.strategy.num_replicas_in_sync
    if n > 1:
      agent.replicas = n
      agent._grad_sync = self.strategy.all_reduce_sum
      if hasattr(agent, '_stat_sync'):
        agent._stat_sync = self.strategy.all_reduce_sum
        agent._replica_rank = self.strategy.rank
      for t in _agent_state_tensors(agent).values():   # mirror rank 0 (MirroredStrategy semantics)
        self.strategy.broadcast(t, src=0)
    self._last_checkpoint_step = None
    self._restore_latest()

  @property
  def train_step_numpy(self):
    """The current train_step as a numpy scalar (learner.py:256-263)."""
    import numpy as np
    return np.int64(self._agent._train_step_host)

  # ---- checkpoints (learner.py:231-263) ----------------------------------------------------------
  def _ckpt_dir(self):
    return os.path.join(self._train_dir, 'checkpoints')

  def _restore_latest(self):
    d = self._ckpt_dir()
    if not os.path.isdir(d):
      return
    files = sorted(f for f in os.listdir(d) if f.startswith('ckpt-') and f.endswith('.pt'))
    if not files:
      return
    state = torch.load(os.path.join(d, files[-1]), map_location='cpu')
    cur = _agent_state_tensors(self._agent)
    for k, v in state['tensors'].items():
      if k in cur:
        cur[k].copy_(v.to(cur[k].device))
    step = int(state['train_step'])
    self._agent.train_step_counter.fill_(step)
    self._agent._train_step_host = step
    if self.train_step is not self._agent.train_step_counter:
      self.train_step.fill_(step)
    self._last_checkpoint_step = step

  def _maybe_checkpoint(self):
    if not self._checkpoint_interval or self.strategy.rank != 0:
      return
    step = self._agent._train_step_host
    last = self._last_checkpoint_step or 0
    if step // self._checkpoint_interval == last // self._checkpoint_interval and last:
      return
    if step < self._checkpoint_interval and self._last_checkpoint_step is not None:
      return
    if step // self._checkpoint_interval == 0:
      return
    d = self._ckpt_dir()
    os.makedirs(d, exist_ok=True)
    tensors = {k: v.detach().cpu() for k, v in _agent_state_tensors(self._agent).items()}
    torch.save({'tensors': tensors, 'train_step': step}, os.path.join(d, f'ckpt-{step:012d}.pt'))
    self._last_checkpoint_step = step
    files = sorted(f for f in os.listdir(d) if f.startswith('ckpt-') and f.endswith('.pt'))
    for f in files[:-self._max_checkpoints_to_keep]:
      os.remove(os.path.join(d, f))

  # ---- run (learner.py:265-378) ------------------------------------------------------------------
  def run(self, iterations=1, iterator=None, parallel_iterations=10):
    """Runs `iterations` train steps; returns the SUM-reduced LossInfo of the last one."""
    assert iterations >= 1, 'Iterations must be greater or equal to 1, was %d' % iterations
    iterator = iterator or self._experience_iterator
    if iterator is None:
      raise ValueError('No experience iterator: pass `iterator` or `experience_dataset_fn`.')
    loss_info = None
    for _ in range(iterations):
      loss_info = self.single_train_step(iterator)
    loss_info = self._reduce(loss_info)
    for trigger in self.triggers:
      trigger(self._agent._train_step_host)
    self._maybe_checkpoint()
    return loss_info

  def single_train_step(self, iterator):
    sample = next(iterator)
    if isinstance(sample, tuple) and len(sample) == 2 and not hasattr(sample, '_fields'):
      experience, sample_info = sample
    else:
      experience, sample_info = sample, None
    if self.use_kwargs_in_agent_train:
      loss_info = self._agent.train(**experience)
    else:
      loss_info = self._agent.train(experience)
    if self._after_train_strategy_step_fn:
      self._after_train_strategy_step_fn((experience, sample_info), loss_info)
    return loss_info

  def _reduce(self, loss_info):
    """strategy.reduce(SUM) over every leaf of LossInfo (learner.py:322-336)."""
    if self.strategy.num_replicas_in_sync == 1:
      return loss_info
    flat = nest.flatten(loss_info)
    reduced = [self.strategy.all_reduce_sum(t.clone()) if isinstance(t, torch.Tensor) else t
               for t in flat]
    return nest.pack_sequence_as(loss_info, reduced)

  def loss(self, experience_and_sample_info=None, reduce_op='sum'):
    """agent.loss on one sample, SUM-reduced (learner.py:380-470)."""
    if experience_and_sample_info is None:
      experience_and_sample_info = next(self._experience_iterator)
    experience = experience_and_sample_info[0] if isinstance(
        experience_and_sample_info, tuple) and not hasattr(
            experience_and_sample_info, '_fields') else experience_and_sample_info
    return self._reduce(self._agent.loss(experience))
