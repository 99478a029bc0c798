"""Recurrent PPO train() time and LSTM sequence-kernel times, one GPU, one process.

* PPOClipAgent.train at the shape of the reference's `use_rnns` PPO example: obs 17, act 6,
  actor input_fc (200, 100) + LSTM 20 + output_fc (200, 100), value input_fc (200, 100) + LSTM 40 +
  output_fc (75, 40), B = 30, T = 1001, num_epochs 25 -- next to feed-forward PPO on the same fc
  layers.  The two are timed in alternating blocks after a warm-up call, eager (no graph), with
  CUDA events around each train() call.
* b200rl_lstm_seq_fwd / b200rl_lstm_seq_bwd alone over a (B, T, H) grid spanning cluster sizes
  1, 2, 4 and 8; time per step = kernel time / T.
The card's name and power limit are read in the same run and printed with the numbers.
Launch: python profiles/ppo_rnn_bench.py [--blocks 3] [--epochs 25]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from agents_b200 import _lib  # noqa: E402
from agents_b200 import optimizers  # noqa: E402
from agents_b200.agents.ppo import ppo_clip_agent  # noqa: E402
from agents_b200.networks import actor_distribution_network as adn  # noqa: E402
from agents_b200.networks import actor_distribution_rnn_network as adrn  # noqa: E402
from agents_b200.networks import value_network  # noqa: E402
from agents_b200.networks import value_rnn_network as vrn  # noqa: E402
from agents_b200.specs import tensor_spec  # noqa: E402
from agents_b200.trajectories import time_step as ts  # noqa: E402
from agents_b200.trajectories import trajectory  # noqa: E402


def _card():
  out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
  return out


def _agent(dev, rnn, epochs):
  D, A = 17, 6
  obs = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act = tensor_spec.BoundedTensorSpec((A,), torch.float32, -1.0, 1.0, 'action')
  if rnn:
    actor = adrn.ActorDistributionRnnNetwork(obs, act, input_fc_layer_params=(200, 100),
                                             lstm_size=(20,), output_fc_layer_params=(200, 100),
                                             activation_fn='tanh', device=dev).set_seed(1)
    value = vrn.ValueRnnNetwork(obs, input_fc_layer_params=(200, 100), lstm_size=(40,),
                                output_fc_layer_params=(75, 40), activation_fn='tanh',
                                device=dev).set_seed(2)
  else:
    actor = adn.ActorDistributionNetwork(obs, act, fc_layer_params=(200, 100), activation_fn='tanh',
                                         device=dev).set_seed(1)
    value = value_network.ValueNetwork(obs, fc_layer_params=(200, 100), activation_fn='tanh',
                                       device=dev).set_seed(2)
  agent = ppo_clip_agent.PPOClipAgent(ts.time_step_spec(obs), act, optimizer=optimizers.Adam(3e-4),
                                      actor_net=actor, value_net=value, num_epochs=epochs,
                                      importance_ratio_clipping=0.2, use_gae=True)
  agent.initialize()
  return agent


def _experience(dev, B=30, T=1001, D=17, A=6):
  g = torch.Generator(device='cpu').manual_seed(0)
  st = torch.ones((B, T), dtype=torch.int32)
  st[:, 0] = 0
  nst = torch.ones((B, T), dtype=torch.int32)
  d = lambda t: t.to(dev)
  return trajectory.Trajectory(
      d(st), d(torch.randn((B, T, D), generator=g)), d(torch.rand((B, T, A), generator=g) * 2 - 1),
      {'dist_params': {'loc': d(torch.zeros(B, T, A)), 'scale': d(torch.full((B, T, A), 0.5))}},
      d(nst), d(torch.rand((B, T), generator=g)), d(torch.ones(B, T)))


def _time(fn, n=1):
  s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  s.record()
  for _ in range(n):
    fn()
  e.record()
  e.synchronize()
  return s.elapsed_time(e) / n


def _kernel_grid(dev, reps):
  rows = []
  for B, T, H in ((30, 1001, 20), (30, 1001, 40), (30, 1001, 64), (30, 1001, 128),
                  (30, 1001, 160), (30, 1001, 256), (256, 1001, 40)):
    cs, btf, btb = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    smf, smb = ctypes.c_int64(), ctypes.c_int64()
    _lib.call('b200rl_lstm_plan', B, H, ctypes.byref(cs), ctypes.byref(btf), ctypes.byref(btb),
              None, None, ctypes.byref(smf), ctypes.byref(smb))
    xw = torch.randn(B * T, 4 * H, device=dev) * 0.3
    U = torch.randn(H, 4 * H, device=dev) * (1.0 / np.sqrt(H))
    st = torch.ones(B, T, dtype=torch.int32, device=dev)
    h, c, hu = (torch.empty(B * T, H, device=dev) for _ in range(3))
    gates = torch.empty(B * T, 4 * H, device=dev)
    dh = torch.randn(B * T, H, device=dev)
    dG = torch.empty_like(gates)
    fwd = lambda: _lib.call('b200rl_lstm_seq_fwd', _lib.ptr(xw), _lib.ptr(U), _lib.ptr(st), None,
                            None, B, T, H, _lib.ptr(h), _lib.ptr(gates), _lib.ptr(c), _lib.ptr(hu),
                            None, None, _lib.stream())
    bwd = lambda: _lib.call('b200rl_lstm_seq_bwd', _lib.ptr(dh), _lib.ptr(gates), _lib.ptr(c), None,
                            _lib.ptr(U), _lib.ptr(st), B, T, H, _lib.ptr(dG), _lib.stream())
    fwd(); bwd()
    torch.cuda.synchronize()
    tf, tb = _time(fwd, reps), _time(bwd, reps)
    rows.append(dict(B=B, T=T, H=H, cluster=cs.value, rows_per_cluster_fwd=btf.value, rows_per_cluster_bwd=btb.value,
                     smem_fwd_kb=smf.value / 1024, smem_bwd_kb=smb.value / 1024,
                     fwd_ms=round(tf, 4), bwd_ms=round(tb, 4),
                     fwd_us_per_step=round(1e3 * tf / T, 3), bwd_us_per_step=round(1e3 * tb / T, 3)))
  return rows


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--blocks', type=int, default=3)
  p.add_argument('--epochs', type=int, default=25)
  p.add_argument('--reps', type=int, default=20)
  a = p.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('ppo_rnn_bench needs a CUDA device.')
  dev = torch.device('cuda:0')
  exp = _experience(dev)
  agents = {'rnn': _agent(dev, True, a.epochs), 'ff': _agent(dev, False, a.epochs)}
  for ag in agents.values():
    ag.train(exp)                                   # warm-up: module load, workspace sizing
  torch.cuda.synchronize()
  times = {k: [] for k in agents}
  for _ in range(a.blocks):
    for k, ag in agents.items():
      times[k].append(_time(lambda: ag.train(exp)))
  out = dict(card=_card(), B=30, T=1001, num_epochs=a.epochs,
             train_ms={k: dict(median=float(np.median(v)), all=[round(x, 2) for x in v])
                       for k, v in times.items()},
             kernels=_kernel_grid(dev, a.reps))
  print(json.dumps(out, indent=1))


if __name__ == '__main__':
  main()
