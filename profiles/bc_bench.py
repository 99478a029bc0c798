"""Behavioral cloning (BehavioralCloningAgent) step and loss-kernel times, one GPU, one process.

* Discrete BC on the Atari conv QNetwork of the DQN benchmark (84x84x4 uint8, Mnih'15 net, A = 6,
  centered RMSProp) next to DqnAgent.train on the same network and batch, at B = 32 and 256.  One
  step = agent.train on a fixed batch, captured in one CUDA graph; the two are timed in
  alternating blocks.  A BC step runs one forward, a DQN step also the target network's.
* Continuous BC on the (400, 300) actor, obs 17, act 6, at B = 256: the deterministic ActorNetwork
  and the Normal ActorDistributionNetwork, captured.
* Each loss kernel alone, from CUDA events over many launches: b200rl_bc_discrete_loss at
  N in {4096, 131072, 1048576} and A in {6, 18, 100, 1000}, b200rl_bc_continuous_loss (both modes,
  A = 6) at the same N.  Bytes moved come from the shapes (each input read once, each output
  written once); the rate is shown against the H100 SXM's 3.35 TB/s.
The card's name and power limit are read in the same run and printed with the numbers.
Launch: python profiles/bc_bench.py [--blocks 3] [--steps 200]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from agents_b200 import _lib  # noqa: E402
from agents_b200 import optimizers  # noqa: E402
from agents_b200.agents.behavioral_cloning import behavioral_cloning_agent as bca  # noqa: E402
from agents_b200.agents.dqn import dqn_agent  # noqa: E402
from agents_b200.networks import actor_distribution_network as adn  # noqa: E402
from agents_b200.networks import actor_network  # noqa: E402
from agents_b200.networks import layers as Ly  # noqa: E402
from agents_b200.networks import q_network  # noqa: E402
from agents_b200.specs import tensor_spec  # noqa: E402
from agents_b200.trajectories import time_step as ts  # noqa: E402
from agents_b200.trajectories import trajectory  # noqa: E402
from profiles import c51_bench  # noqa: E402
from profiles import td3_bench  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def _atari(dev):
  obs_spec = tensor_spec.TensorSpec((84, 84, 4), torch.uint8, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, c51_bench.A - 1, 'action')
  opt = lambda: optimizers.RMSPropOptimizer(2.5e-4, decay=0.95, momentum=0.0, epsilon=1e-5,
                                            centered=True)
  net = lambda: q_network.QNetwork(obs_spec, act_spec, preprocessing_layers=Ly.CastScale(255.),
                                   conv_layer_params=c51_bench.CONV, fc_layer_params=c51_bench.FC,
                                   device=dev).set_seed(0)
  dqn = dqn_agent.DqnAgent(ts.time_step_spec(obs_spec), act_spec, q_network=net(),
                           optimizer=opt(), epsilon_greedy=0.01, target_update_period=2500,
                           gamma=0.99)
  dqn.initialize()
  bc = bca.BehavioralCloningAgent(ts.time_step_spec(obs_spec), act_spec, net(), opt())
  return dqn, bc


def _traj(dev, outer, obs_shape, obs_dtype, action):
  g = torch.Generator(device=dev).manual_seed(3)
  if obs_dtype == torch.uint8:
    obs = torch.randint(0, 256, outer + obs_shape, dtype=torch.uint8, device=dev, generator=g)
  else:
    obs = torch.randn(outer + obs_shape, device=dev, generator=g)
  one = torch.ones(outer, dtype=torch.int32, device=dev)
  rew = torch.rand(outer, device=dev, generator=g)
  return trajectory.Trajectory(one, obs, action, (), one, rew, torch.ones(outer, device=dev))


def atari_steps(dev, blocks, steps):
  out = []
  for B in (32, 256):
    dqn, bc = _atari(dev)
    act2 = torch.randint(0, c51_bench.A, (B, 2), dtype=torch.int32, device=dev)
    fns = dict(
        bc=td3_bench._captured_step(bc, _traj(dev, (B,), (84, 84, 4), torch.uint8, act2[:, 0].contiguous())),
        dqn=td3_bench._captured_step(dqn, _traj(dev, (B, 2), (84, 84, 4), torch.uint8, act2)))
    ms = dict(bc=[], dqn=[])
    for _ in range(blocks):
      for k in ('bc', 'dqn'):
        ms[k].append(td3_bench._time(fns[k], steps))
    med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
    out.append(dict(batch=B, ms_per_step_bc=ms['bc'], ms_per_step_dqn=ms['dqn'],
                    median_ms_bc=med['bc'], median_ms_dqn=med['dqn'],
                    bc_over_dqn=med['bc'] / med['dqn']))
  return out


def continuous_steps(dev, blocks, steps, B=256, D=17, A=6):
  obs_spec = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((A,), torch.float32, -1.0, 1.0, 'action')
  nets = dict(
      deterministic=actor_network.ActorNetwork(obs_spec, act_spec, fc_layer_params=(400, 300),
                                               device=dev).set_seed(1),
      normal=adn.ActorDistributionNetwork(obs_spec, act_spec, fc_layer_params=(400, 300),
                                          device=dev).set_seed(1))
  act = torch.rand(B, A, device=dev) * 2 - 1
  fns = {k: td3_bench._captured_step(
      bca.BehavioralCloningAgent(ts.time_step_spec(obs_spec), act_spec, n, optimizers.Adam(1e-3)),
      _traj(dev, (B,), (D,), torch.float32, act)) for k, n in nets.items()}
  ms = {k: [] for k in fns}
  for _ in range(blocks):
    for k in fns:
      ms[k].append(td3_bench._time(fns[k], steps))
  return dict(batch=B, ms_per_step=ms, median_ms={k: sorted(v)[len(v) // 2] for k, v in ms.items()})


def _launches(nbytes):
  return int(max(20, min(2000, 2e10 // nbytes)))


def _rate(name, fn, nbytes):
  for _ in range(10):
    fn()
  torch.cuda.synchronize()
  us = 1000 * td3_bench._time(fn, _launches(nbytes))
  return dict(kernel=name, us=us, bytes=nbytes, tb_per_s=nbytes / us / 1e6,
              hbm_share=nbytes / us / 1e6 / (HBM_BYTES_PER_S / 1e12))


def kernel_rates(dev):
  out = []
  ws = torch.empty(512, device=dev)
  loss, flag, st = torch.empty(1, device=dev), torch.zeros(1, dtype=torch.int32, device=dev), _lib.stream()
  for N in (4096, 131072, 1048576):
    pe = torch.empty(N, device=dev)
    for A in (6, 18, 100, 1000):
      z = torch.randn(N, A, device=dev)
      g = torch.empty(N, A, device=dev)
      a = torch.randint(0, A, (N,), dtype=torch.int32, device=dev)
      fn = (lambda z=z, g=g, a=a, N=N, A=A: _lib.call(
          'b200rl_bc_discrete_loss', _lib.ptr(z), A, _lib.ptr(a), 1, 0, None, 1, N, A,
          _lib.ptr(loss), _lib.ptr(pe), _lib.ptr(g), A, _lib.ptr(flag), _lib.ptr(ws), 2048, st))
      out.append(dict(N=N, A=A, **_rate('bc_discrete_loss', fn, 4 * (2 * N * A + 2 * N))))
      del z, g
    A = 6
    y, s, t = (torch.rand(N, A, device=dev) for _ in range(3))
    dp, ds = torch.empty(N, A, device=dev), torch.empty(N, A, device=dev)
    lo, hi = -torch.ones(A, device=dev), torch.ones(A, device=dev)
    rng = torch.zeros(2, dtype=torch.int64, device=dev)
    det = lambda: _lib.call('b200rl_bc_continuous_loss', _lib.ptr(y), None, A, _lib.ptr(t), A,
                            _lib.ptr(lo), _lib.ptr(hi), None, 3, None, 0, None, 1, N, A,
                            _lib.ptr(loss), _lib.ptr(pe), _lib.ptr(dp), None, A, _lib.ptr(flag),
                            _lib.ptr(ws), 2048, st)
    nrm = lambda: _lib.call('b200rl_bc_continuous_loss', _lib.ptr(y), _lib.ptr(s), A, _lib.ptr(t),
                            A, None, None, None, 3, _lib.ptr(rng), 1, None, 1, N, A,
                            _lib.ptr(loss), _lib.ptr(pe), _lib.ptr(dp), _lib.ptr(ds), A,
                            _lib.ptr(flag), _lib.ptr(ws), 2048, st)
    out.append(dict(N=N, A=A, **_rate('bc_continuous_loss_deterministic', det, 4 * (3 * N * A + N))))
    out.append(dict(N=N, A=A, **_rate('bc_continuous_loss_normal', nrm, 4 * (5 * N * A + N))))
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--blocks', type=int, default=3)
  ap.add_argument('--steps', type=int, default=200)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bc_bench needs a CUDA device.')
  dev = torch.device('cuda', 0)
  name, power = c51_bench._card()
  print(json.dumps(dict(bench='bc_atari_step', gpu=name, power_limit=power, cuda_graph=True,
                        results=atari_steps(dev, args.blocks, args.steps))), flush=True)
  print(json.dumps(dict(bench='bc_continuous_step', gpu=name, power_limit=power, cuda_graph=True,
                        actor=[400, 300], **continuous_steps(dev, args.blocks, args.steps))),
        flush=True)
  print(json.dumps(dict(bench='bc_loss_kernels', gpu=name, power_limit=power,
                        hbm_peak_tb_per_s=HBM_BYTES_PER_S / 1e12, results=kernel_rates(dev))),
        flush=True)


if __name__ == '__main__':
  main()
