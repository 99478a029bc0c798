"""C51 (CategoricalDqnAgent, N = 51) step time next to the DqnAgent step at the bench.py config-2
shapes: 84x84x4 uint8 frames from a 1 M-slot ring, the Mnih'15 net, A = 6, centered RMSProp,
gamma 0.99.  One step = get_next(B, 2) + agent.train, captured in one CUDA graph; the two agents
are timed in alternating blocks at B = 32 (the C51 Atari example's batch) and B = 256 (the bench
batch).  Also times b200rl_c51_loss and b200rl_c51_q_values at B = 256 with CUDA events over 2000
launches, and with --kernels prints the per-kernel CUDA time of one eager step of each agent
(torch.profiler), to show where a difference goes.  The card's name and power limit are read in
the same run and printed with the numbers.
Launch: python profiles/c51_bench.py [--blocks 3] [--steps 200] [--kernels]
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
from agents_b200.agents.categorical_dqn import categorical_dqn_agent  # noqa: E402
from agents_b200.agents.dqn import dqn_agent  # noqa: E402
from agents_b200.networks import categorical_q_network  # noqa: E402
from agents_b200.networks import layers as Ly  # noqa: E402
from agents_b200.networks import q_network  # noqa: E402
from agents_b200.replay_buffers import tf_uniform_replay_buffer as rb_mod  # noqa: E402
from agents_b200.specs import tensor_spec  # noqa: E402
from agents_b200.trajectories import time_step as ts  # noqa: E402
from agents_b200.utils import common  # noqa: E402

A, N_ATOMS = 6, 51
B_ENV, L = 256, 4096                   # 1 M slots
CONV = ((32, 8, 4), (64, 4, 2), (64, 3, 1))
FC = (512,)


def _card():
  name = torch.cuda.get_device_name()
  try:
    power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader',
                            '-i', str(torch.cuda.current_device())], capture_output=True,
                           text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    power = 'unknown'
  return name, power


def _agents(dev):
  obs_spec = tensor_spec.TensorSpec((84, 84, 4), torch.uint8, 'observation')
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, A - 1, 'action')
  opt = lambda: optimizers.RMSPropOptimizer(2.5e-4, decay=0.95, momentum=0.0, epsilon=1e-5,
                                            centered=True)
  kw = dict(epsilon_greedy=0.01, n_step_update=1, target_update_tau=1.0,
            target_update_period=2500, gamma=0.99)
  qnet = q_network.QNetwork(obs_spec, act_spec, preprocessing_layers=Ly.CastScale(255.),
                            conv_layer_params=CONV, fc_layer_params=FC, device=dev).set_seed(0)
  dqn = dqn_agent.DqnAgent(ts.time_step_spec(obs_spec), act_spec, q_network=qnet,
                           optimizer=opt(), **kw)
  cnet = categorical_q_network.CategoricalQNetwork(
      obs_spec, act_spec, num_atoms=N_ATOMS, preprocessing_layers=Ly.CastScale(255.),
      conv_layer_params=CONV, fc_layer_params=FC, device=dev).set_seed(0)
  c51 = categorical_dqn_agent.CategoricalDqnAgent(ts.time_step_spec(obs_spec), act_spec, cnet,
                                                  opt(), **kw)
  dqn.initialize()
  c51.initialize()
  return dqn, c51


def _ring(spec, dev):
  rb = rb_mod.TFUniformReplayBuffer(spec, batch_size=B_ENV, max_length=L, device=dev, seed=0x5eed)
  g = torch.Generator(device=dev).manual_seed(1234)
  st_store, obs_store, act_store, nst_store, rew_store, disc_store = rb._data_table.variables()
  cap = B_ENV * L
  chunk = 1 << 15
  for i in range(0, cap, chunk):               # random frames written in place, as bench.py does
    obs_store[i:i + chunk].view(-1).view(torch.int64).random_(generator=g)
  st_store.copy_(torch.randint(0, 3, (cap,), device=dev, generator=g, dtype=torch.int32))
  nst_store.copy_(torch.randint(0, 3, (cap,), device=dev, generator=g, dtype=torch.int32))
  act_store.copy_(torch.randint(0, A, (cap,), device=dev, generator=g, dtype=torch.int32))
  rew_store.copy_(torch.rand(cap, device=dev, generator=g))
  disc_store.copy_((torch.rand(cap, device=dev, generator=g) > 0.1).float())
  last_id = 2 * L + 77
  pos = torch.arange(cap, device=dev, dtype=torch.int64) % L
  rb._id_table.variables()[0].copy_(torch.where(pos <= last_id % L, last_id - last_id % L + pos,
                                                last_id - last_id % L - L + pos))
  rb._last_id.fill_(last_id)
  rb._last_id_host = last_id
  return rb


def _captured_step(agent, rb, B):
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


def kernel_us(dev, B=256, launches=2000):
  """b200rl_c51_loss (n_step 1, with a mask) and b200rl_c51_q_values at [B, A*51]."""
  g = torch.Generator(device=dev).manual_seed(7)
  q = torch.randn(B, A * N_ATOMS, device=dev, generator=g)
  nq = torch.randn(B, A * N_ATOMS, device=dev, generator=g)
  mask = (torch.rand(B, A, device=dev, generator=g) > 0.2).int()
  act = torch.randint(0, A, (B,), device=dev, generator=g, dtype=torch.int32)
  rew, disc = torch.randn(B, 2, device=dev, generator=g), torch.ones(B, 2, device=dev)
  z = torch.linspace(-10.0, 10.0, N_ATOMS, device=dev)
  loss, dq, rows = torch.empty(1, device=dev), torch.empty_like(q), torch.empty(B, device=dev)
  qv = torch.empty(B, A, device=dev)
  flag = torch.zeros(1, dtype=torch.int32, device=dev)
  st = _lib.stream()

  def c51_loss():
    _lib.call('b200rl_c51_loss', _lib.ptr(q), _lib.ptr(nq), _lib.ptr(mask), _lib.ptr(act), 1,
              _lib.ptr(rew), _lib.ptr(disc), _lib.ptr(z), None, B, A, N_ATOMS, 2, 0.99, 1.0, float(B),
              _lib.ptr(loss), _lib.ptr(dq), _lib.ptr(flag), _lib.ptr(rows), 4 * B, st)

  def q_values():
    _lib.call('b200rl_c51_q_values', _lib.ptr(q), _lib.ptr(z), B, A, N_ATOMS, _lib.ptr(qv), st)

  out = {}
  for name, fn in (('c51_loss', c51_loss), ('c51_q_values', q_values)):
    for _ in range(20):
      fn()
    torch.cuda.synchronize()
    out[name] = 1000 * _time(fn, launches)
  return out


def kernel_breakdown(agent, rb, B, steps=10):
  """CUDA time per kernel name over `steps` eager train steps, in us per step."""
  from torch.profiler import ProfilerActivity, profile
  for _ in range(3):
    agent.train(rb.get_next(sample_batch_size=B, num_steps=2)[0])
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(steps):
      agent.train(rb.get_next(sample_batch_size=B, num_steps=2)[0])
    torch.cuda.synchronize()
  rows = [(e.key, e.device_time_total / steps) for e in prof.key_averages()
          if e.device_time_total > 0]
  return sorted(rows, key=lambda r: -r[1])[:25]


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--blocks', type=int, default=3)
  ap.add_argument('--steps', type=int, default=200)
  ap.add_argument('--kernels', action='store_true')
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('c51_bench needs a CUDA device.')
  dev = torch.device('cuda', 0)
  dqn, c51 = _agents(dev)
  rb = _ring(dqn.collect_data_spec, dev)
  name, power = _card()
  for B in (32, 256):
    fns = dict(dqn=_captured_step(dqn, rb, B), c51=_captured_step(c51, rb, B))
    ms = dict(dqn=[], c51=[])
    for _ in range(args.blocks):
      for k in ('dqn', 'c51'):
        ms[k].append(_time(fns[k], args.steps))
    med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
    print(json.dumps(dict(bench='c51_step', gpu=name, power_limit=power, batch=B, num_atoms=N_ATOMS,
                          cuda_graph=True, ms_per_step_dqn=ms['dqn'], ms_per_step_c51=ms['c51'],
                          median_ms_dqn=med['dqn'], median_ms_c51=med['c51'],
                          c51_over_dqn=med['c51'] / med['dqn'])), flush=True)
    del fns
  k = kernel_us(dev)
  print(json.dumps(dict(bench='c51_kernels', gpu=name, power_limit=power, batch=256, A=A,
                        num_atoms=N_ATOMS, launches=2000, c51_loss_us=k['c51_loss'],
                        c51_q_values_us=k['c51_q_values'])), flush=True)
  if args.kernels:
    for label, agent in (('dqn', dqn), ('c51', c51)):
      print(json.dumps(dict(bench='c51_step_kernels', agent=label, batch=256, gpu=name,
                            power_limit=power, us_per_step=kernel_breakdown(agent, rb, 256))),
            flush=True)


if __name__ == '__main__':
  main()
