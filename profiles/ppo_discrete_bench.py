"""Discrete-action PPO benchmark: PPOClipAgent with a Categorical actor on synthetic experience.

Configs (one JSON line each):
  a  4096 envs x T=128, 17-d f32 observations, A=18, (200, 100) tanh nets, 25 epochs, Adam:
     the config-3 (continuous PPO) networks with a categorical head.
  b  Atari shape: 8 envs x T=128, 84x84x4 uint8 observations, CastScale(255) + Mnih'15 conv torso
     ((32,8,4), (64,4,2), (64,3,1)) + Dense(512) on actor and value, A=6, 4 epochs,
     normalize_observations=False.
Each line has the GPU name and power limit read in the same run, train() ms from CUDA events
after warm-up (the step captured with common.function, as profiles/ppo_bench.py does), and the
categorical loss kernel alone (b200rl_ppo_loss_categorical, CUDA events over many launches) with
its algorithmic bytes computed from the shapes and the share of the 3.35 TB/s H100 SXM data-sheet
HBM bandwidth those bytes imply.  Usage: python profiles/ppo_discrete_bench.py [a|b ...]
"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from agents_b200 import _lib, optimizers  # noqa: E402
from agents_b200.agents.ppo import ppo_clip_agent  # noqa: E402
from agents_b200.networks import actor_distribution_network, layers as L, value_network  # noqa: E402
from agents_b200.specs import tensor_spec  # noqa: E402
from agents_b200.trajectories import time_step as ts  # noqa: E402
from agents_b200.trajectories import trajectory  # noqa: E402
from agents_b200.utils import common, workspace  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet
CONFIGS = {
    'a': dict(B=4096, T=128, obs=(17,), u8=False, A=18, hidden=(200, 100), act='tanh', conv=None,
              epochs=25, normalize_observations=True),
    'b': dict(B=8, T=128, obs=(84, 84, 4), u8=True, A=6, hidden=(512,), act='relu',
              conv=((32, 8, 4), (64, 4, 2), (64, 3, 1)), epochs=4, normalize_observations=False),
}


def gpu_identity():
  name = torch.cuda.get_device_name(0)
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = ''
  return name, out or 'not measured'


def loss_kernel_bytes(N, A):
  """HBM bytes one b200rl_ppo_loss_categorical launch needs at least (clip only, no KL / value
  clip): logits + int32 action + old_logp/adv/ret/v/w in, dlogits + dv out, per row."""
  return N * (4 * A + 4 + 5 * 4 + 4 * A + 4)


def time_loss_kernel(dev, N, A, T, iters=200):
  g = torch.Generator(device=dev).manual_seed(3)
  z = torch.randn(N, A, device=dev, generator=g)
  act = torch.randint(0, A, (N,), device=dev, dtype=torch.int32, generator=g)
  vec = [torch.randn(N, device=dev, generator=g) for _ in range(5)]
  w = torch.ones(N, device=dev)
  losses = torch.empty(6, device=dev)
  dz = torch.empty(N, A, device=dev)
  dv = torch.empty(N, device=dev)
  flag = torch.zeros(1, dtype=torch.int32, device=dev)
  ws, nb = workspace.get(dev)

  def launch():
    _lib.call('b200rl_ppo_loss_categorical', _lib.ptr(z), A, _lib.ptr(act), _lib.ptr(vec[0]),
              _lib.ptr(vec[1]), _lib.ptr(vec[2]), _lib.ptr(vec[3]), None, _lib.ptr(w), N, A, T,
              float(N // T), 0.2, 0.0, 0.5, 0.01, 0.0, _lib.ptr(losses), _lib.ptr(dz), A,
              _lib.ptr(dv), _lib.ptr(flag), None, _lib.ptr(ws), nb, _lib.stream())

  for _ in range(20):
    launch()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(iters):
    launch()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / iters      # ms per launch (the loss kernel + its 1-CTA final)


def run(name):
  c = CONFIGS[name]
  dev = torch.device('cuda', 0)
  B, T, A = c['B'], c['T'], c['A']
  obs_spec = tensor_spec.TensorSpec(c['obs'], torch.uint8 if c['u8'] else torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, A - 1, 'action')
  extra = {}
  if c['conv']:
    extra = dict(conv_layer_params=c['conv'])
  actor = actor_distribution_network.ActorDistributionNetwork(
      obs_spec, act_spec, fc_layer_params=c['hidden'], activation_fn=c['act'], device=dev,
      preprocessing_layers=L.CastScale(255.) if c['conv'] else None, **extra).set_seed(1)
  value = value_network.ValueNetwork(
      obs_spec, fc_layer_params=c['hidden'], activation_fn=c['act'], device=dev,
      preprocessing_layers=L.CastScale(255.) if c['conv'] else None, **extra).set_seed(2)
  agent = ppo_clip_agent.PPOClipAgent(
      ts.time_step_spec(obs_spec), act_spec, optimizer=optimizers.Adam(3e-4), actor_net=actor,
      value_net=value, importance_ratio_clipping=0.2, use_gae=True, lambda_value=0.95,
      discount_factor=0.99, num_epochs=c['epochs'], entropy_regularization=0.01,
      normalize_observations=c['normalize_observations'], normalize_rewards=False)
  agent.initialize()
  g = torch.Generator(device=dev).manual_seed(100)
  if c['u8']:
    obs = torch.randint(0, 256, (B, T) + c['obs'], dtype=torch.uint8, device=dev, generator=g)
  else:
    obs = torch.randn((B, T) + c['obs'], device=dev, generator=g)
  exp = trajectory.Trajectory(
      torch.ones(B, T, dtype=torch.int32, device=dev), obs,
      torch.randint(0, A, (B, T), dtype=torch.int32, device=dev, generator=g),
      {'dist_params': {'logits': torch.randn(B, T, A, device=dev, generator=g) * 0.5}},
      torch.ones(B, T, dtype=torch.int32, device=dev), torch.rand(B, T, device=dev, generator=g),
      torch.ones(B, T, device=dev))
  fn = common.function(agent.train, warmup=1)
  fn(exp)                                  # eager warm-up
  fn(exp)                                  # capture + first replay
  fn(exp)
  torch.cuda.synchronize()
  reps = 5
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(reps):
    info = fn(exp)
  e1.record()
  torch.cuda.synchronize()
  train_ms = e0.elapsed_time(e1) / reps
  agent.check_numerics()
  N = B * T
  k_ms = time_loss_kernel(dev, N, A, T)
  nbytes = loss_kernel_bytes(N, A)
  gpu, power = gpu_identity()
  return dict(bench='ppo_discrete', config=name, gpu=gpu, power_limit=power, envs=B, T=T,
              obs_shape=list(c['obs']), num_actions=A, epochs=c['epochs'], train_ms=train_ms,
              ms_per_epoch=train_ms / c['epochs'], cuda_graph=True, loss=float(info.loss.item()),
              loss_kernel_us=k_ms * 1e3, loss_kernel_bytes=nbytes,
              loss_kernel_hbm_share=nbytes / (k_ms * 1e-3) / HBM_BYTES_PER_S)


def main():
  if not torch.cuda.is_available():
    raise SystemExit('ppo_discrete_bench needs a CUDA device (no CPU fallback).')
  for name in (sys.argv[1:] or sorted(CONFIGS)):
    print(json.dumps(run(name)), flush=True)


if __name__ == '__main__':
  main()
