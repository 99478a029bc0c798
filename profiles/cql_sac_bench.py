"""CQL-SAC step time next to the SAC step, one GPU, one process (SURVEY §8d config 4 nets: obs 17,
act 6, (256, 256) relu critics and actor, tau 0.005, reward_scale 0.1, Adam 3e-4).

One step = get_next(256, 2) from a 1 M-slot ring + agent.train, captured in one CUDA graph.
CqlSacAgent runs with num_cql_samples = 10 (the reference's default), so each critic sees
256 * (2*10 + 1) = 5376 joint rows in the critic step instead of 256.  The two agents are timed in
alternating blocks; the JSON line gives every block's ms/step, the critic-step GEMM FLOPs per step
computed from the shapes, and the b200rl_cql_loss time from CUDA events over many launches.  The
card's name and power limit are printed with the numbers.
Launch: python profiles/cql_sac_bench.py [--blocks 3] [--steps 300]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from agents_b200 import _lib  # noqa: E402
from agents_b200 import optimizers  # noqa: E402
from agents_b200.agents.cql import cql_sac_agent  # noqa: E402
from agents_b200.agents.sac import sac_agent  # noqa: E402
from agents_b200.networks import critic_network  # noqa: E402
from agents_b200.networks import tanh_normal_projection_network as tnp  # noqa: E402
from agents_b200.replay_buffers import tf_uniform_replay_buffer as rb_mod  # noqa: E402
from agents_b200.specs import tensor_spec  # noqa: E402
from agents_b200.trajectories import time_step as ts  # noqa: E402
from agents_b200.trajectories import trajectory  # noqa: E402
from agents_b200.utils import common  # noqa: E402

D, A, B, N, HIDDEN = 17, 6, 256, 10, (256, 256)
B_ENV, L = 256, 4096                   # 1 M slots


def critic_step_gemm_flops(rows):
  """Both critics' forward + backward GEMMs in the critic step over `rows` joint rows: forward
  2·rows·in·out per layer, weight gradients the same again, input gradients for every layer but
  the first (the joint input needs none)."""
  dims = [D + A] + list(HIDDEN) + [1]
  layers = list(zip(dims[:-1], dims[1:]))
  fwd = sum(2 * rows * i * o for i, o in layers)
  dx = sum(2 * rows * i * o for i, o in layers[1:])
  return 2 * (fwd + fwd + dx)


def _card():
  name = torch.cuda.get_device_name()
  try:
    power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader',
                            '-i', str(torch.cuda.current_device())], capture_output=True,
                           text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    power = 'unknown'
  return name, power


def _agent(cls, dev, **kw):
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, -1.0, 1.0, 'action')
  actor = tnp.TanhNormalActorNetwork(obs_spec, act_spec, fc_layer_params=HIDDEN, device=dev).set_seed(1)
  critic = critic_network.CriticNetwork((obs_spec, act_spec), joint_fc_layer_params=HIDDEN,
                                        device=dev).set_seed(2)
  agent = cls(ts.time_step_spec(obs_spec), act_spec, critic_network=critic, actor_network=actor,
              actor_optimizer=optimizers.Adam(3e-4), critic_optimizer=optimizers.Adam(3e-4),
              alpha_optimizer=optimizers.Adam(3e-4), target_update_tau=0.005,
              target_update_period=1, gamma=0.99, reward_scale_factor=0.1, **kw)
  agent.initialize()
  return agent


def _captured_step(agent, rb):
  def step():
    exp, _ = rb.get_next(sample_batch_size=B, num_steps=2)
    return agent.train(exp).loss
  fn = common.function(step, warmup=1)
  for _ in range(12):
    fn()
  torch.cuda.synchronize()
  return fn


def _time(fn, n):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(n):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / n


def cql_loss_kernel_ms(dev, launches=2000):
  rows = B + 2 * B * N
  g = torch.Generator(device=dev).manual_seed(7)
  q1, q2 = (torch.randn(rows, device=dev, generator=g) for _ in range(2))
  logp = torch.randn(B * N, device=dev, generator=g)
  alpha, closs = torch.tensor(1.0, device=dev), torch.zeros(1, device=dev)
  dq1, dq2 = torch.zeros(rows, device=dev), torch.zeros(rows, device=dev)
  out, ws = torch.empty(4, device=dev), torch.empty(256, device=dev)
  st = _lib.stream()

  def launch():
    _lib.call('b200rl_cql_loss', _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(logp), B, N, -6 * 0.6931472,
              1.0, _lib.ptr(alpha), None, float('-inf'), float('inf'), 10.0, 0, _lib.ptr(closs),
              _lib.ptr(dq1), _lib.ptr(dq2), _lib.ptr(out), None, None, _lib.ptr(ws), 4 * 256, st)
  for _ in range(20):
    launch()
  torch.cuda.synchronize()
  return _time(launch, launches)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--blocks', type=int, default=3)
  ap.add_argument('--steps', type=int, default=300)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('cql_sac_bench needs a CUDA device.')
  dev = torch.device('cuda', 0)
  sac = _agent(sac_agent.SacAgent, dev)
  cql = _agent(cql_sac_agent.CqlSacAgent, dev, cql_alpha=5.0, num_cql_samples=N,
               include_critic_entropy_term=False, use_lagrange_cql_alpha=False)
  rb = rb_mod.TFUniformReplayBuffer(sac.collect_data_spec, batch_size=B_ENV, max_length=L, device=dev,
                                    seed=0x5eed)
  g = torch.Generator(device=dev).manual_seed(100)
  for _ in range(64):                      # a fixed synthetic dataset; the learner only samples
    rb.add_batch(trajectory.Trajectory(
        torch.ones(B_ENV, dtype=torch.int32, device=dev), torch.randn(B_ENV, D, device=dev, generator=g),
        torch.rand(B_ENV, A, device=dev, generator=g) * 2 - 1, (),
        torch.ones(B_ENV, dtype=torch.int32, device=dev), torch.rand(B_ENV, device=dev, generator=g),
        torch.ones(B_ENV, device=dev)))
  fns = dict(sac=_captured_step(sac, rb), cql=_captured_step(cql, rb))
  ms = dict(sac=[], cql=[])
  for _ in range(args.blocks):
    for name in ('sac', 'cql'):
      ms[name].append(_time(fns[name], args.steps))
  k_ms = cql_loss_kernel_ms(dev)
  name, power = _card()
  med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
  print(json.dumps(dict(
      bench='cql_sac_step', gpu=name, power_limit=power, batch=B, num_cql_samples=N,
      nets=list(HIDDEN), cuda_graph=True, ms_per_step_sac=ms['sac'], ms_per_step_cql=ms['cql'],
      median_ms_sac=med['sac'], median_ms_cql=med['cql'], cql_over_sac=med['cql'] / med['sac'],
      critic_step_gemm_gflop_sac=critic_step_gemm_flops(B) / 1e9,
      critic_step_gemm_gflop_cql=critic_step_gemm_flops(B * (2 * N + 1)) / 1e9,
      cql_loss_kernel_us=1000 * k_ms)), flush=True)


if __name__ == '__main__':
  main()
