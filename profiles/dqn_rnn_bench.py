"""Recurrent DQN train() time and b200rl_dqn_seq_td_loss time, one GPU, one process.

* DqnAgent.train on a QRnnNetwork at the shape of the reference's `dqn_rnn` example: CartPole
  observations (4), A = 2, input_fc (50,), LSTM (20,), output_fc (20,), B = 64 sequences of
  T = 11 steps (train_sequence_length 10 + 1) -- next to feed-forward DqnAgent.train on a
  QNetwork with fc (50, 20) at the same B (T = 2).  Both run as captured graphs
  (common.function), timed with CUDA events in alternating blocks after warm-up.
* b200rl_dqn_seq_td_loss alone for B in {64, 256, 4096} and T-1 in {10, 80} (A = 2): 100
  launches captured in one CUDA graph, CUDA events over the replays, so the figure is device time
  and not the Python enqueue.
The card's name and power limit are read in the same run and printed with the numbers.
Launch: python profiles/dqn_rnn_bench.py [--blocks 5] [--steps 200] [--reps 20000]
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
from agents_b200.agents.dqn import dqn_agent  # noqa: E402
from agents_b200.networks import q_network  # noqa: E402
from agents_b200.networks import q_rnn_network  # noqa: E402
from agents_b200.specs import tensor_spec  # noqa: E402
from agents_b200.trajectories import time_step as ts  # noqa: E402
from agents_b200.trajectories import trajectory  # noqa: E402
from agents_b200.utils import common  # noqa: E402

B, D, A = 64, 4, 2


def _card():
  return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                        capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]


def _agent(dev, rnn):
  obs = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act = tensor_spec.BoundedTensorSpec((), torch.int32, 0, A - 1, 'action')
  if rnn:
    net = q_rnn_network.QRnnNetwork(obs, act, input_fc_layer_params=(50,), lstm_size=(20,),
                                    output_fc_layer_params=(20,), device=dev).set_seed(1)
  else:
    net = q_network.QNetwork(obs, act, fc_layer_params=(50, 20), device=dev).set_seed(1)
  agent = dqn_agent.DqnAgent(ts.time_step_spec(obs), act, q_network=net,
                             optimizer=optimizers.AdamOptimizer(1e-3), gamma=0.99,
                             target_update_period=5)
  agent.initialize()
  return agent


def _experience(dev, T):
  g = torch.Generator(device='cpu').manual_seed(0)
  st = torch.ones((B, T), dtype=torch.int32)
  st[:, 0] = 0
  d = lambda t: t.to(dev)
  return trajectory.Trajectory(
      d(st), d(torch.randn((B, T, D), generator=g)), d(torch.randint(0, A, (B, T), generator=g,
                                                                    dtype=torch.int32)),
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


def _kernel_grid(dev, reps):
  rows = []
  for b in (64, 256, 4096):
    for tm in (10, 80):
      n, T = b * tm, tm + 1
      q, nt = (torch.randn(n, A, device=dev) for _ in range(2))
      act = torch.randint(0, A, (b, T), dtype=torch.int32, device=dev)
      st = torch.ones((b, T), dtype=torch.int32, device=dev)
      rew, disc = torch.randn(b, T, device=dev), torch.ones(b, T, device=dev)
      loss, td_loss = torch.empty(1, device=dev), torch.empty(b, device=dev)
      td_error, dq = torch.empty(n, device=dev), torch.empty_like(q)
      partials = torch.empty(_lib.DQN_SEQ_MAX_BLOCKS, device=dev)
      ticket = torch.zeros(1, dtype=torch.int32, device=dev)
      call = lambda: _lib.call(
          'b200rl_dqn_seq_td_loss', _lib.ptr(q), _lib.ptr(nt), _lib.ptr(nt), None, _lib.ptr(act),
          T, 1, _lib.ptr(st), T, 1, _lib.ptr(rew), _lib.ptr(disc), None, 0, b, A, T, 0.99, 1.0,
          _lib.LOSS_HUBER, float(b), _lib.ptr(loss), _lib.ptr(td_loss), _lib.ptr(td_error),
          _lib.ptr(dq), None, _lib.ptr(partials), _lib.ptr(ticket), _lib.stream())
      call()
      torch.cuda.synchronize()
      g = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g):
        for _ in range(100):
          call()
      g.replay()
      torch.cuda.synchronize()
      ms = _time(g.replay, max(1, reps // 100)) / 100
      # bytes the launch needs: two [n, A] tables read, dq written, td_error written, the
      # action / step / reward / discount columns read, td_loss written
      nbytes = 4 * (3 * n * A + n + 4 * b * T + b)
      rows.append(dict(B=b, T_minus_1=tm, A=A, us=round(1e3 * ms, 3),
                       GB_per_s=round(nbytes / (ms * 1e-3) / 1e9, 1)))
  return rows


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--blocks', type=int, default=5)
  p.add_argument('--steps', type=int, default=200)
  p.add_argument('--reps', type=int, default=20000)
  a = p.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('dqn_rnn_bench needs a CUDA device.')
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
             seq_td_loss_kernel=_kernel_grid(dev, a.reps))
  print(json.dumps(out, indent=1))


if __name__ == '__main__':
  main()
