"""Measurements of BASELINE.json configs 1, 3, 4, 5 and the data-parallel parity check, as
functions `bench.py` calls after its own (config 2) measurement so that every driver record
(BENCH / SCALE json) carries them.  Each returns a small dict; `strategy` is the process-group
strategy of the run (train/utils/strategy_utils.py), so under torchrun the PPO / SAC updates are
sharded over the ranks (strong scaling) and the gather sweep shards the ring by segment.

  ppo_update     config 3  PPOClipAgent.train on 4096 envs x T=128, 25 epochs, (200,100) tanh
  sac_step       config 4  get_next(1024/N, 2) + SacAgent.train, nets (256,256)
  cartpole_iter  config 1  collect 1 step + sample 64x2 + DqnAgent.train, Dense(100) net
  gather_sweep   config 5  b200rl_rb_sample GB/s over ring capacity x batch
  dp_parity      N replicas on shards of a batch vs ONE replica on the whole batch
"""
import ctypes
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)

from agents_b200 import _lib, optimizers  # noqa: E402
from agents_b200.specs import tensor_spec  # noqa: E402
from agents_b200.trajectories import time_step as ts  # noqa: E402
from agents_b200.trajectories import trajectory  # noqa: E402
from agents_b200.utils import common, nest  # noqa: E402

ROW_ATARI = 28244


def _max_over_ranks(ms, dev, world):
  if world > 1:
    t = torch.tensor([ms], device=dev, dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms = float(t.item())
  return ms


def _agree(ok, dev, world):
  if world > 1:
    flag = torch.tensor([int(ok)], device=dev, dtype=torch.int32)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    ok = bool(flag.item())
  return ok


def _captured(step, eager_step, dev, world, rank):
  """common.function(step) with the rank-agreement dance of bench.py; returns (fn, used_graph)."""
  fn = common.function(step, warmup=1)
  fn()
  ok = True
  try:
    fn()
  except Exception as e:  # pylint: disable=broad-except
    sys.stderr.write(f'[rank {rank}] graph capture failed ({type(e).__name__}: {e}); eager\n')
    ok = False
    torch.cuda.synchronize()
    eager_step()
  ok = _agree(ok, dev, world)
  return (fn if ok else eager_step), ok


def _time(fn, n, dev, world):
  torch.cuda.synchronize()
  if world > 1:
    dist.barrier()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  out = None
  for _ in range(n):
    out = fn()
  e1.record()
  torch.cuda.synchronize()
  return _max_over_ranks(e0.elapsed_time(e1) / n, dev, world), out


# ---- config 3 ------------------------------------------------------------------------------------
def _ppo_agent(dev, D, A, epochs, normalize, seed_a=1, seed_v=2, hidden=(200, 100), **kw):
  from agents_b200.agents.ppo import ppo_clip_agent
  from agents_b200.networks import actor_distribution_network, value_network
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, -1.0, 1.0, 'action')
  actor = actor_distribution_network.ActorDistributionNetwork(
      obs_spec, act_spec, fc_layer_params=hidden, activation_fn='tanh', device=dev).set_seed(seed_a)
  value = value_network.ValueNetwork(obs_spec, fc_layer_params=hidden, activation_fn='tanh',
                                     device=dev).set_seed(seed_v)
  agent = ppo_clip_agent.PPOClipAgent(
      ts.time_step_spec(obs_spec), act_spec, optimizer=optimizers.Adam(3e-4), actor_net=actor,
      value_net=value, importance_ratio_clipping=0.2, use_gae=True, lambda_value=0.95,
      discount_factor=0.99, num_epochs=epochs, normalize_observations=normalize,
      normalize_rewards=normalize, **kw)
  agent.initialize()
  return agent


def _ppo_experience(dev, B, T, D, A, seed):
  g = torch.Generator(device=dev).manual_seed(seed)
  r = lambda *s: torch.rand(*s, device=dev, generator=g)
  return trajectory.Trajectory(
      torch.ones(B, T, dtype=torch.int32, device=dev), torch.randn(B, T, D, device=dev, generator=g),
      r(B, T, A) * 2 - 1,
      {'dist_params': {'loc': (r(B, T, A) - .5) * .2, 'scale': torch.full((B, T, A), .7, device=dev)}},
      torch.ones(B, T, dtype=torch.int32, device=dev), r(B, T), torch.ones(B, T, device=dev))


def ppo_update(strategy, dev, peaks, reps=3):
  """Strong scaling: 4096 trajectories sharded over the ranks; one all-reduce of the 62 k-parameter
  gradient per epoch, the advantage moments and the normaliser statistics merged per train()."""
  from agents_b200.train import learner as learner_lib
  world, rank = strategy.num_replicas_in_sync, strategy.rank
  B_total, T, D, A, epochs = 4096, 128, 17, 6, 25
  lo, hi = strategy.shard_range(B_total)
  B = hi - lo
  agent = _ppo_agent(dev, D, A, epochs, normalize=True)
  learner_lib.Learner('/tmp/b200rl_ppo_bench', agent.train_step_counter, agent, strategy=strategy,
                      checkpoint_interval=0)
  exp = _ppo_experience(dev, B, T, D, A, 100 + rank)
  fn, graph = _captured(lambda: agent.train(exp), lambda: agent.train(exp), dev, world, rank)
  fn()
  ms, info = _time(fn, reps, dev, world)
  n_params = int(agent._flat_params.numel())
  # fp32-equivalent GEMM work: fwd + bwd(2x) of both MLPs over all samples and epochs
  macs = (D * 200 + 200 * 100 + 100 * A) + (D * 200 + 200 * 100 + 100)
  flops = 3 * 2.0 * macs * B_total * T * epochs
  # HBM floor of one epoch: activations of both nets written in the forward and read in the
  # backward (x, 200, 100 wide; fp32) + the loss kernel's per-sample streams
  act_bytes = 2 * (200 + 100) * 4 * 2 + (D + 6 * A + 8) * 4
  hbm = act_bytes * B_total * T * epochs
  tf = flops / (ms * 1e-3) / 1e12
  gbs = hbm / (ms * 1e-3) / 1e9
  return dict(train_ms=ms, ms_per_epoch=ms / epochs, n_gpus=world, envs_total=B_total,
              envs_per_gpu=B, T=T, epochs=epochs, scaling='strong', cuda_graph=graph,
              normalizers=True, params=n_params, samples_per_s=B_total * T * epochs / (ms * 1e-3),
              loss=float(info.loss.item()),
              roofline=dict(bound='tensor', achieved=tf, peak=peaks['tensor'], unit='TFLOP/s',
                            frac=tf / peaks['tensor'], algorithmic_flops=flops,
                            hbm_achieved_gbs=gbs, hbm_frac=gbs / peaks['hbm'],
                            algorithmic_bytes=hbm))


# ---- config 4 ------------------------------------------------------------------------------------
def sac_step(strategy, dev, peaks, steps=200):
  from agents_b200.agents.sac import sac_agent
  from agents_b200.networks import critic_network
  from agents_b200.networks import tanh_normal_projection_network as tnp
  from agents_b200.replay_buffers import tf_uniform_replay_buffer as rb_mod
  from agents_b200.train import learner as learner_lib
  world, rank = strategy.num_replicas_in_sync, strategy.rank
  D, A, B_global, B_env, L = 17, 6, 1024, 256, 4096
  B = B_global // world
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, -1.0, 1.0, 'action')
  actor = tnp.TanhNormalActorNetwork(obs_spec, act_spec, fc_layer_params=(256, 256), device=dev).set_seed(1)
  critic = critic_network.CriticNetwork((obs_spec, act_spec), joint_fc_layer_params=(256, 256),
                                        device=dev).set_seed(2)
  agent = sac_agent.SacAgent(ts.time_step_spec(obs_spec), act_spec, critic_network=critic,
                             actor_network=actor, actor_optimizer=optimizers.Adam(3e-4),
                             critic_optimizer=optimizers.Adam(3e-4),
                             alpha_optimizer=optimizers.Adam(3e-4), target_update_tau=0.005,
                             target_update_period=1, gamma=0.99, reward_scale_factor=0.1)
  agent.initialize()
  learner_lib.Learner('/tmp/b200rl_sac_bench', agent.train_step_counter, agent, strategy=strategy,
                      checkpoint_interval=0)
  rb = rb_mod.TFUniformReplayBuffer(agent.collect_data_spec, batch_size=B_env, max_length=L,
                                    device=dev, seed=0x5eed0000 + rank)
  g = torch.Generator(device=dev).manual_seed(100 + rank)
  for _ in range(64):
    rb.add_batch(trajectory.Trajectory(
        torch.ones(B_env, dtype=torch.int32, device=dev), torch.randn(B_env, D, device=dev, generator=g),
        torch.rand(B_env, A, device=dev, generator=g) * 2 - 1, (),
        torch.ones(B_env, dtype=torch.int32, device=dev), torch.rand(B_env, device=dev, generator=g),
        torch.ones(B_env, device=dev)))

  def step():
    exp, _ = rb.get_next(sample_batch_size=B, num_steps=2)
    return agent.train(exp).loss

  fn, graph = _captured(step, step, dev, world, rank)
  for _ in range(10):
    fn()
  ms, loss = _time(fn, steps, dev, world)
  flops = 2.5e9                                   # SURVEY §8d: ~2.5 GFLOP per 1024-batch step
  tf = flops / (ms * 1e-3) / 1e12
  return dict(ms_per_step=ms, steps_per_s=1000.0 / ms, n_gpus=world, global_batch=B_global,
              per_gpu_batch=B, scaling='strong', cuda_graph=graph, loss=float(loss.item()),
              roofline=dict(bound='latency (launch-bound; tensor figure for context)', achieved=tf,
                            peak=peaks['tensor'], unit='TFLOP/s', frac=tf / peaks['tensor'],
                            algorithmic_flops=flops))


# ---- config 1 ------------------------------------------------------------------------------------
def cartpole_iter(dev, iters=2000):
  from agents_b200.agents.dqn import dqn_agent
  from agents_b200.drivers import dynamic_step_driver
  from agents_b200.environments import random_tf_environment
  from agents_b200.networks import layers as L
  from agents_b200.networks import sequential
  from agents_b200.replay_buffers import tf_uniform_replay_buffer as rb_mod
  env = random_tf_environment.CartPoleTFEnvironment(batch_size=1, seed=0, device=dev,
                                                    action_dtype=torch.int32)
  tss, act_spec = env.time_step_spec(), env.action_spec()
  net = sequential.Sequential([L.Dense(100, activation='relu'), L.Dense(2)], input_spec=tss.observation,
                              device=dev).set_seed(0)
  agent = dqn_agent.DqnAgent(tss, act_spec, q_network=net, optimizer=optimizers.AdamOptimizer(1e-3),
                             gamma=0.99, epsilon_greedy=0.1, target_update_tau=0.05,
                             target_update_period=5,
                             td_errors_loss_fn=common.element_wise_squared_loss)
  agent.initialize()
  rb = rb_mod.TFUniformReplayBuffer(agent.collect_data_spec, batch_size=1, max_length=10000, device=dev)
  driver = dynamic_step_driver.DynamicStepDriver(env, agent.collect_policy, observers=[rb.add_batch],
                                                 num_steps=1)
  state = {'ts': None, 'ps': None}
  for _ in range(200):
    state['ts'], state['ps'] = driver.run(state['ts'], state['ps'], maximum_iterations=1)

  def iteration():
    state['ts'], state['ps'] = driver.run(state['ts'], state['ps'], maximum_iterations=1)
    exp, _ = rb.get_next(sample_batch_size=64, num_steps=2)
    return agent.train(exp).loss

  out = dict(config='DQN CartPole: collect 1 + sample 64x2 + train, Dense(100) net, buffer 10k')
  for _ in range(20):
    iteration()
  ms, loss = _time(iteration, 200, dev, 1)
  out.update(eager_iters_per_s=1000.0 / ms, loss=float(loss.item()))
  try:
    fn = common.function(iteration, warmup=1)
    for _ in range(5):
      fn()
    ms, loss = _time(fn, iters, dev, 1)
    out.update(graph_iters_per_s=1000.0 / ms, us_per_iter=ms * 1e3, loss_graph=float(loss.item()))
  except Exception as e:  # pylint: disable=broad-except
    out['graph_error'] = f'{type(e).__name__}: {e}'
  return out


# ---- config 5 ------------------------------------------------------------------------------------
def gather_sweep(dev, world, rank, peaks, caps_m=(1, 2), batches=(64, 256, 1024, 4096), T=2,
                 nl=20, reps=5):
  """b200rl_rb_sample on Atari-shape rows.  `caps_m` are GLOBAL capacities in Mi slots; each rank
  owns capacity/world of it (shard by segment, no exchange) and samples batch/world windows, so
  the cell's GB/s is the sum over ranks.  Cells whose per-rank shard does not fit in free HBM are
  reported as infeasible."""
  from agents_b200.replay_buffers import tf_uniform_replay_buffer as rb_mod
  spec = trajectory.Trajectory(
      tensor_spec.TensorSpec([], torch.int32, 'step_type'),
      tensor_spec.TensorSpec((84, 84, 4), torch.uint8, 'observation'),
      tensor_spec.TensorSpec([], torch.int32, 'action'), (),
      tensor_spec.TensorSpec([], torch.int32, 'next_step_type'),
      tensor_spec.TensorSpec([], torch.float32, 'reward'),
      tensor_spec.TensorSpec([], torch.float32, 'discount'))
  flat = nest.flatten(spec)
  cells = []
  for cap_m in caps_m:
    cap = cap_m << 20
    per_rank = cap // world
    need = per_rank * (ROW_ATARI + 8)
    free, _ = torch.cuda.mem_get_info(dev)
    feasible = _agree(need + (8 << 30) < free, dev, world)
    if not feasible:
      for B in batches:
        cells.append(dict(capacity_m=cap_m, B=B, infeasible=f'{need / 2**30:.0f} GiB per GPU'))
      continue
    L = 4096
    rb = rb_mod.TFUniformReplayBuffer(spec, batch_size=per_rank // L, max_length=L, device=dev,
                                      seed=1 + rank)
    rb._last_id.fill_(3 * L)
    rb._last_id_host = 3 * L
    for B in batches:
      Bl = max(1, B // world)
      bufs = []
      for _ in range(4):
        outs = [torch.empty((Bl, T) + s.shape, dtype=s.dtype, device=dev) for s in flat]
        bufs.append((outs, _lib.ptr_array(outs), torch.empty((Bl, T), dtype=torch.int64, device=dev),
                     torch.empty(Bl, dtype=torch.float32, device=dev)))

      def launch(i):
        outs, ptrs, ids, prob = bufs[i % 4]
        _lib.call('b200rl_rb_sample', ctypes.byref(rb._ring), Bl, T, None, None, rb._seed,
                  _lib.ptr(rb._ctrl[0:1]), ptrs, _lib.ptr(ids), None, _lib.ptr(prob),
                  _lib.ptr(rb._ctrl[1:2]), _lib.stream())

      for i in range(3):
        launch(i)
      torch.cuda.synchronize()
      g = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g):
        for i in range(nl):
          launch(i)
      g.replay()
      ms, _ = _time(g.replay, reps, dev, world)
      us = ms * 1e3 / nl
      nbytes = (2 * Bl * T * ROW_ATARI + 8 * Bl * T) * world
      gbs = nbytes / (us * 1e-6) / 1e9
      cells.append(dict(capacity_m=cap_m, B=B, us=round(us, 2), gbs=round(gbs, 1),
                        frac=round(gbs / (peaks['hbm'] * world), 4)))
      del bufs, g
    del rb
    torch.cuda.empty_cache()
  return dict(row_bytes=ROW_ATARI, T=T, n_gpus=world, peak_gbs_per_gpu=peaks['hbm'],
              kernel='row_copy_tma<MODE_SAMPLE>', cells=cells)


# ---- data-parallel parity --------------------------------------------------------------------------
def dp_parity(strategy, dev):
  """Every rank trains (a) its shard of a global batch as one of N replicas (losses / global batch,
  SUM all-reduce of the gradient, merged statistics) and (b) the WHOLE batch alone with a second,
  identically initialised agent.  Reports max |theta_a - theta_b| / max |theta_b| after a few
  steps -- the reference's equal-across-strategies contract (train/learner_test.py:442-540)."""
  from agents_b200.agents.dqn import dqn_agent
  from agents_b200.networks import layers as Ly
  from agents_b200.networks import q_network
  from agents_b200.train import learner as learner_lib
  from agents_b200.train.utils import strategy_utils
  world, rank = strategy.num_replicas_in_sync, strategy.rank
  out = {}

  def rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-20))

  # DQN: conv net on uint8 frames, per-replica batch 32
  obs_spec = tensor_spec.TensorSpec((20, 20, 4), torch.uint8, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 3, 'action')

  def make_dqn():
    net = q_network.QNetwork(obs_spec, act_spec, preprocessing_layers=Ly.CastScale(255.),
                             conv_layer_params=((16, 4, 2),), fc_layer_params=(64,),
                             device=dev).set_seed(3)
    a = dqn_agent.DqnAgent(ts.time_step_spec(obs_spec), act_spec, q_network=net,
                           optimizer=optimizers.AdamOptimizer(1e-3), gamma=0.99)
    a.initialize()
    return a, net
  dp, dp_net = make_dqn()
  ref, ref_net = make_dqn()
  learner_lib.Learner('/tmp/b200rl_dp_parity_dqn', dp.train_step_counter, dp, strategy=strategy,
                      checkpoint_interval=0)
  g = torch.Generator(device=dev).manual_seed(7)            # same stream on every rank
  per = 32
  G = per * world
  losses = []
  for _ in range(3):
    exp = trajectory.Trajectory(
        torch.ones(G, 2, dtype=torch.int32, device=dev),
        torch.randint(0, 256, (G, 2, 20, 20, 4), dtype=torch.uint8, device=dev, generator=g),
        torch.randint(0, 4, (G, 2), dtype=torch.int32, device=dev, generator=g), (),
        torch.ones(G, 2, dtype=torch.int32, device=dev), torch.rand(G, 2, device=dev, generator=g),
        torch.ones(G, 2, device=dev))
    shard = nest.map_structure(lambda t: t[rank * per:(rank + 1) * per].contiguous(), exp)
    l_dp = dp.train(shard).loss.clone()
    strategy.all_reduce_sum(l_dp)                          # LossInfo is SUM-reduced (learner.py:322-336)
    l_ref = ref.train(exp).loss
    losses.append(abs(float(l_dp) - float(l_ref)) / max(abs(float(l_ref)), 1e-12))
  out['dqn_param_rel'] = rel(dp_net.flat_params, ref_net.flat_params)
  out['dqn_loss_rel'] = max(losses)

  # PPO with both normalisers on: per-replica 16 trajectories x T=16, 2 epochs, 2 train calls
  D, A, T, per = 17, 6, 16, 16
  dp = _ppo_agent(dev, D, A, 2, normalize=True, hidden=(64, 32))
  ref = _ppo_agent(dev, D, A, 2, normalize=True, hidden=(64, 32))
  learner_lib.Learner('/tmp/b200rl_dp_parity_ppo', dp.train_step_counter, dp, strategy=strategy,
                      checkpoint_interval=0)
  losses = []
  for it in range(2):
    exp = _ppo_experience(dev, per * world, T, D, A, 50 + it)
    shard = nest.map_structure(lambda t: t[rank * per:(rank + 1) * per].contiguous(), exp)
    l_dp = dp.train(shard).loss.clone()
    strategy.all_reduce_sum(l_dp)
    l_ref = ref.train(exp).loss
    losses.append(abs(float(l_dp) - float(l_ref)) / max(abs(float(l_ref)), 1e-12))
  out['ppo_param_rel'] = rel(dp._flat_params, ref._flat_params)
  out['ppo_loss_rel'] = max(losses)
  out['ppo_obs_norm_rel'] = rel(dp._observation_normalizer.variables[2],
                                ref._observation_normalizer.variables[2])
  out['replicas'] = world
  # worst case over ranks
  if world > 1:
    keys = sorted(k for k in out if k.endswith('_rel'))
    t = torch.tensor([out[k] for k in keys], device=dev, dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    for k, v in zip(keys, t.tolist()):
      out[k] = v
  return out


if __name__ == '__main__':
  # python profiles/configs.py [ppo|sac|cartpole|gather|parity]   (torchrun for N > 1)
  from agents_b200.train.utils import strategy_utils
  which = sys.argv[1] if len(sys.argv) > 1 else 'ppo'
  world = int(os.environ.get('WORLD_SIZE', '1'))
  local = int(os.environ.get('LOCAL_RANK', '0'))
  torch.cuda.set_device(local)
  dev = torch.device('cuda', local)
  if world > 1:
    strategy_utils.configure_nccl_env()
    dist.init_process_group('nccl', device_id=dev)
  strategy = strategy_utils.get_strategy()
  pk = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json'))) if os.path.exists(
      os.path.join(ROOT, 'MEASURED_PEAKS.json')) else dict(hbm_gbs=3350.0, bf16_tflops_sustained=989.0)   # H100 SXM data sheet
  peaks = dict(hbm=pk['hbm_gbs'], tensor=pk.get('bf16_tflops_sustained', pk.get('bf16_tflops', 989.0)))
  res = dict(ppo=lambda: ppo_update(strategy, dev, peaks), sac=lambda: sac_step(strategy, dev, peaks),
             cartpole=lambda: cartpole_iter(dev),
             gather=lambda: gather_sweep(dev, world, strategy.rank, peaks),
             parity=lambda: dp_parity(strategy, dev))[which]()
  if strategy.rank == 0:
    print(json.dumps({which: res}), flush=True)
  if world > 1:
    dist.barrier()
    torch.cuda.synchronize()
    sys.stdout.flush()
    os._exit(0)
