"""Recurrent DDPG train() time and the two sequence-loss kernels' times, one GPU, one process.

* DdpgAgent.train on ActorRnnNetwork + CriticRnnNetwork at the shape of the reference's
  ddpg/examples/v2/train_eval_rnn.py: cartpole-balance position observations (3), A = 1, actor
  input_fc (400, 300) -> LSTM (40,) -> output_fc (100,), critic observation_fc (400,), no action
  branch, joint_fc (300,), LSTM (40,), output_fc (100,), B = 64 sequences of T = 11 steps
  (train_sequence_length 10 + 1) -- next to feed-forward DdpgAgent.train on ActorNetwork (400, 300)
  and CriticNetwork (observation (400,), joint (300,)) at the same B (T = 2).  Both run as captured
  graphs (common.function), timed with CUDA events in alternating blocks after warm-up.
* b200rl_ddpg_seq_critic_loss and b200rl_ddpg_seq_actor_loss alone at (B 64, T-1 10) and
  (B 4096, T-1 80), A = 1: 100 launches captured in one CUDA graph, CUDA events over the
  replays, so the figure is device time and not the Python enqueue; achieved bytes/s from the
  bytes each launch needs.
The card's name and power limit are read in the same run and printed with the numbers.
Launch: python profiles/ddpg_rnn_bench.py [--blocks 5] [--steps 200] [--reps 20000]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from agents_b200 import _lib  # noqa: E402
from agents_b200 import optimizers  # noqa: E402
from agents_b200.agents.ddpg import ddpg_agent  # noqa: E402
from agents_b200.networks import actor_network  # noqa: E402
from agents_b200.networks import actor_rnn_network  # noqa: E402
from agents_b200.networks import critic_network  # noqa: E402
from agents_b200.networks import critic_rnn_network  # noqa: E402
from agents_b200.specs import tensor_spec  # noqa: E402
from agents_b200.trajectories import time_step as ts  # noqa: E402
from agents_b200.trajectories import trajectory  # noqa: E402
from agents_b200.utils import common  # noqa: E402

B, D, A = 64, 3, 1


def _card():
  return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                        capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]


def _agent(dev, rnn):
  obs = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act = tensor_spec.BoundedTensorSpec((A,), torch.float32, -1.0, 1.0, 'action')
  if rnn:
    actor = actor_rnn_network.ActorRnnNetwork(obs, act, input_fc_layer_params=(400, 300),
                                              lstm_size=(40,), output_fc_layer_params=(100,),
                                              device=dev).set_seed(1)
    critic = critic_rnn_network.CriticRnnNetwork(
        (obs, act), observation_fc_layer_params=(400,), action_fc_layer_params=None,
        joint_fc_layer_params=(300,), lstm_size=(40,), output_fc_layer_params=(100,),
        device=dev).set_seed(2)
  else:
    actor = actor_network.ActorNetwork(obs, act, fc_layer_params=(400, 300),
                                       device=dev).set_seed(1)
    critic = critic_network.CriticNetwork((obs, act), observation_fc_layer_params=(400,),
                                          joint_fc_layer_params=(300,), device=dev).set_seed(2)
  agent = ddpg_agent.DdpgAgent(ts.time_step_spec(obs), act, actor_network=actor,
                               critic_network=critic, actor_optimizer=optimizers.Adam(1e-4),
                               critic_optimizer=optimizers.Adam(1e-3), target_update_tau=0.05,
                               target_update_period=5, gamma=0.995)
  agent.initialize()
  return agent


def _experience(dev, T):
  g = torch.Generator(device='cpu').manual_seed(0)
  st = torch.ones((B, T), dtype=torch.int32)
  st[:, 0] = 0
  d = lambda t: t.to(dev)   # noqa: E731
  return trajectory.Trajectory(
      d(st), d(torch.randn((B, T, D), generator=g)), d(torch.rand((B, T, A), generator=g) * 2 - 1),
      (), d(torch.ones((B, T), dtype=torch.int32)), d(torch.rand((B, T), generator=g)),
      d(torch.ones(B, T)))


def _time(fn, n):
  s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  s.record()
  for _ in range(n):
    fn()
  e.record()
  e.synchronize()
  return s.elapsed_time(e) / n


def _graph_time(call, reps):
  call()
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    for _ in range(100):
      call()
  g.replay()
  torch.cuda.synchronize()
  return _time(g.replay, max(1, reps // 100)) / 100


def _kernel_grid(dev, reps):
  rows = []
  amin, amax = -torch.ones(A, device=dev), torch.ones(A, device=dev)
  for b, tm in ((64, 10), (4096, 80)):
    n, T = b * tm, tm + 1
    q, tq, dq = torch.randn(n, device=dev), torch.randn(n, device=dev), torch.empty(n, device=dev)
    rew, disc = torch.randn(b, T, device=dev), torch.ones(b, T, device=dev)
    dqda, dy = torch.randn(n, A, device=dev), torch.empty(n, A, device=dev)
    loss = torch.empty(1, device=dev)
    partials = torch.empty(_lib.DDPG_SEQ_MAX_BLOCKS, device=dev)
    ticket = torch.zeros(1, dtype=torch.int32, device=dev)
    critic = lambda: _lib.call(   # noqa: E731
        'b200rl_ddpg_seq_critic_loss', _lib.ptr(q), _lib.ptr(tq), _lib.ptr(rew), _lib.ptr(disc),
        T, 1, None, 0, b, T, 0.995, 1.0, _lib.LOSS_HUBER, _lib.ptr(loss), _lib.ptr(dq), None,
        _lib.ptr(partials), _lib.ptr(ticket), _lib.stream())
    actor = lambda: _lib.call(   # noqa: E731
        'b200rl_ddpg_seq_actor_loss', _lib.ptr(dqda), A, None, 0, b, T, A, 0, 0.0, _lib.ptr(amin),
        _lib.ptr(amax), _lib.ptr(loss), _lib.ptr(dy), None, _lib.ptr(partials), _lib.ptr(ticket),
        _lib.stream())
    # bytes each launch needs: critic reads q, tq and the [B, T-1] reward / discount, writes dq;
    # actor reads dqda and writes dy
    for name, call, nbytes in (('seq_critic_loss', critic, 4 * (2 * n + 2 * n + n)),
                               ('seq_actor_loss', actor, 4 * (2 * n * A))):
      ms = _graph_time(call, reps)
      rows.append(dict(kernel=name, B=b, T_minus_1=tm, A=A, us=round(1e3 * ms, 3),
                       GB_per_s=round(nbytes / (ms * 1e-3) / 1e9, 1)))
  return rows


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--blocks', type=int, default=5)
  p.add_argument('--steps', type=int, default=200)
  p.add_argument('--reps', type=int, default=20000)
  a = p.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('ddpg_rnn_bench needs a CUDA device.')
  dev = torch.device('cuda:0')
  runs = {}
  for name, rnn, T in (('rnn_T11', True, 11), ('ff_T2', False, 2)):
    agent, exp = _agent(dev, rnn), _experience(dev, T)
    agent.train(exp)                                # eager warm-up: module load, workspace sizing
    fn = common.function(agent.train)
    for _ in range(3):
      fn(exp)
    torch.cuda.synchronize()
    runs[name] = (fn, exp)
  times = {k: [] for k in runs}
  for _ in range(a.blocks):
    for k, (fn, exp) in runs.items():
      times[k].append(_time(lambda: fn(exp), a.steps))
  out = dict(card=_card(), B=B, obs=D, A=A,
             train_ms_per_step={k: dict(median=round(float(np.median(v)), 4),
                                        all=[round(x, 4) for x in v]) for k, v in times.items()},
             seq_loss_kernels=_kernel_grid(dev, a.reps))
  print(json.dumps(out, indent=1))


if __name__ == '__main__':
  main()
