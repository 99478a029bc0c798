"""REINFORCE benchmark (one JSON line each, with the GPU name and power limit read in the same run).

  cartpole  one iteration of the CartPole recipe: DynamicEpisodeDriver collect of 8 episodes on 8
            device envs (at most 600 driver iterations) + gather_all + ReinforceAgent.train +
            clear, eager (the driver reads its episode counter on the host), value baseline,
            (64,) nets.  ms per iteration from CUDA events, averaged over 20 iterations.
  mujoco    ReinforceAgent.train captured with common.function at a MuJoCo shape: 17-d
            observations, 6-d Normal actions, (200, 100) tanh actor and value nets,
            B = 32 x T = 1024 = 32768 rows, normalised advantages with a baseline.
  kernel    b200rl_reinforce_loss alone at N = 32768 rows (baseline, normalisation, entropy), for
            Categorical A = 2 and Normal A = 6: CUDA events over 2000 launches, algorithmic bytes
            per row (Normal 20A + 24, Categorical 8A + 28: parameters, actions, returns, V,
            step types and weights in; parameter gradients and dV out) and the share of the
            3.35 TB/s H100 SXM data-sheet HBM bandwidth those bytes imply.
Usage: python profiles/reinforce_bench.py [cartpole|mujoco|kernel ...]
"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from agents_b200 import _lib, optimizers  # noqa: E402
from agents_b200.agents.reinforce import reinforce_agent  # noqa: E402
from agents_b200.drivers import dynamic_episode_driver  # noqa: E402
from agents_b200.environments import random_tf_environment  # noqa: E402
from agents_b200.networks import actor_distribution_network, value_network  # noqa: E402
from agents_b200.replay_buffers import tf_uniform_replay_buffer as rb_mod  # noqa: E402
from agents_b200.specs import tensor_spec  # noqa: E402
from agents_b200.trajectories import time_step as ts  # noqa: E402
from agents_b200.trajectories import trajectory  # noqa: E402
from agents_b200.utils import common  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def gpu_identity():
  name = torch.cuda.get_device_name(0)
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = ''
  return name, out or 'not measured'


def _events():
  return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def bench_cartpole(dev):
  B, NE, TMAX, iters = 8, 8, 600, 20
  env = random_tf_environment.CartPoleTFEnvironment(batch_size=B, seed=0, device=dev)
  tss, act_spec = env.time_step_spec(), env.action_spec()
  actor = actor_distribution_network.ActorDistributionNetwork(tss.observation, act_spec,
                                                              fc_layer_params=(64,), device=dev).set_seed(0)
  value = value_network.ValueNetwork(tss.observation, fc_layer_params=(64,), device=dev).set_seed(1)
  agent = reinforce_agent.ReinforceAgent(tss, act_spec, actor, optimizers.Adam(3e-3), value_network=value,
                                         gamma=0.99)
  agent.initialize()
  rb = rb_mod.TFUniformReplayBuffer(agent.collect_data_spec, batch_size=B, max_length=TMAX, device=dev)
  driver = dynamic_episode_driver.DynamicEpisodeDriver(env, agent.collect_policy,
                                                       observers=[rb.add_batch], num_episodes=NE)

  def iteration():
    driver.run(maximum_iterations=TMAX)
    exp = rb.gather_all()
    agent.train(exp)
    rb.clear()
    return exp.action.shape[1]

  for _ in range(3):
    iteration()
  torch.cuda.synchronize()
  e0, e1 = _events()
  steps = 0
  e0.record()
  for _ in range(iters):
    steps += iteration()
  e1.record()
  torch.cuda.synchronize()
  agent.check_numerics()
  ms = e0.elapsed_time(e1) / iters
  return dict(config='cartpole', envs=B, episodes_per_iteration=NE, iteration_ms=ms,
              mean_driver_steps=steps / iters, cuda_graph=False)


def bench_mujoco(dev):
  B, T, D, A = 32, 1024, 17, 6
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, -1, 1, 'action')
  actor = actor_distribution_network.ActorDistributionNetwork(
      obs_spec, act_spec, fc_layer_params=(200, 100), activation_fn='tanh', device=dev).set_seed(1)
  value = value_network.ValueNetwork(obs_spec, fc_layer_params=(200, 100), activation_fn='tanh',
                                     device=dev).set_seed(2)
  agent = reinforce_agent.ReinforceAgent(ts.time_step_spec(obs_spec), act_spec, actor,
                                         optimizers.Adam(1e-4), value_network=value, gamma=0.99,
                                         entropy_regularization=0.01)
  agent.initialize()
  g = torch.Generator(device=dev).manual_seed(100)
  nst = torch.ones(B, T, dtype=torch.int32, device=dev)
  nst[:, 199::200] = 2                     # episodes of 200 steps, partial ones at the row ends
  st = torch.ones_like(nst)
  st[:, 0] = 0
  st[:, 1:][nst[:, :-1] == 2] = 2
  exp = trajectory.Trajectory(st, torch.randn(B, T, D, device=dev, generator=g),
                              torch.rand(B, T, A, device=dev, generator=g) * 2 - 1, (), nst,
                              torch.rand(B, T, device=dev, generator=g),
                              (nst != 2).float())
  fn = common.function(agent.train, warmup=1)
  fn(exp)
  fn(exp)
  fn(exp)
  torch.cuda.synchronize()
  reps = 20
  e0, e1 = _events()
  e0.record()
  for _ in range(reps):
    info = fn(exp)
  e1.record()
  torch.cuda.synchronize()
  agent.check_numerics()
  return dict(config='mujoco', rows=B * T, obs_dim=D, action_dim=A, hidden=[200, 100],
              train_ms=e0.elapsed_time(e1) / reps, cuda_graph=True, loss=float(info.loss.item()))


def kernel_bytes(N, A, discrete):
  return N * ((8 * A + 28) if discrete else (20 * A + 24))


def bench_kernel(dev, discrete, A, N=32768, T=1024, iters=2000):
  B = N // T
  g = torch.Generator(device=dev).manual_seed(3)
  if discrete:
    p0, p1 = torch.randn(N, A, device=dev, generator=g), None
    act = torch.randint(0, A, (N,), device=dev, dtype=torch.int32, generator=g)
    d0, d1 = torch.empty(N, A, device=dev), None
  else:
    p0 = torch.randn(N, A, device=dev, generator=g)
    p1 = torch.rand(N, A, device=dev, generator=g) + 0.5
    act = torch.randn(N, A, device=dev, generator=g)
    d0, d1 = torch.empty(N, A, device=dev), torch.empty(N, A, device=dev)
  ret, V, w = (torch.randn(N, device=dev, generator=g) for _ in range(3))
  nst = torch.ones(B, T, dtype=torch.int32, device=dev)
  nst[:, 199::200] = 2
  st = torch.ones_like(nst)
  st[:, 1:][nst[:, :-1] == 2] = 2
  losses, dv = torch.empty(6, device=dev), torch.empty(N, device=dev)
  flag = torch.zeros(1, dtype=torch.int32, device=dev)
  ws = torch.empty(4 * (4096 + B + N), dtype=torch.uint8, device=dev)

  def launch():
    _lib.call('b200rl_reinforce_loss', _lib.ptr(p0), _lib.ptr(p1), A, _lib.ptr(act), A, _lib.ptr(ret),
              _lib.ptr(V), _lib.ptr(st), _lib.ptr(nst), _lib.ptr(w), B, T, 1, 1, 0.01, 0.2,
              _lib.ptr(losses), _lib.ptr(d0), _lib.ptr(d1), A, _lib.ptr(dv), None, _lib.ptr(flag),
              _lib.ptr(ws), ws.numel(), _lib.stream())

  for _ in range(50):
    launch()
  e0, e1 = _events()
  e0.record()
  for _ in range(iters):
    launch()
  e1.record()
  torch.cuda.synchronize()
  us = e0.elapsed_time(e1) / iters * 1e3
  nbytes = kernel_bytes(N, A, discrete)
  return dict(config='kernel', head='categorical' if discrete else 'normal', rows=N, num_actions=A,
              launches=iters, loss_kernel_us=us, loss_kernel_bytes=nbytes,
              loss_kernel_hbm_share=nbytes / (us * 1e-6) / HBM_BYTES_PER_S)


def main():
  if not torch.cuda.is_available():
    raise SystemExit('reinforce_bench needs a CUDA device (no CPU fallback).')
  dev = torch.device('cuda', 0)
  gpu, power = gpu_identity()
  for name in (sys.argv[1:] or ['cartpole', 'mujoco', 'kernel']):
    if name == 'kernel':
      results = [bench_kernel(dev, True, 2), bench_kernel(dev, False, 6)]
    elif name == 'cartpole':
      results = [bench_cartpole(dev)]
    else:
      results = [bench_mujoco(dev)]
    for r in results:
      print(json.dumps(dict(bench='reinforce', gpu=gpu, power_limit=power, **r)), flush=True)


if __name__ == '__main__':
  main()
