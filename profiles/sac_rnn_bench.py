"""Recurrent SAC train() time and the three sequence-loss kernels' times, one GPU, one process.

* SacAgent.train on a tanh-Normal ActorDistributionRnnNetwork + CriticRnnNetwork critics at the
  shape of the reference's sac/examples/v2/train_eval_rnn.py: cartpole-balance position
  observations (3), A = 1, actor input_fc (400, 300) -> LSTM (40,) -> output_fc (100,) ->
  TanhNormalProjectionNetwork, critics with no observation / action branch, joint_fc (300,),
  LSTM (40,), output_fc (100,), B = 256 sequences of T = 21 steps (train_sequence_length 20 + 1)
  -- next to feed-forward SacAgent.train on TanhNormalActorNetwork (400, 300) and CriticNetwork
  (joint (300,)) at the same B (T = 2).  Both run as captured graphs (common.function), timed with
  CUDA events in alternating blocks after warm-up.
* b200rl_sac_seq_critic_loss, b200rl_sac_seq_actor_loss and b200rl_sac_seq_alpha_loss alone at
  (B 256, T-1 20) and (B 4096, T-1 80): 100 launches captured in one CUDA graph, CUDA events over
  the replays, so the figure is device time and not the Python enqueue; achieved bytes/s from the
  bytes each launch needs.
The card's name and power limit are read in the same run and printed with the numbers.
Launch: python profiles/sac_rnn_bench.py [--blocks 5] [--steps 100] [--reps 20000]
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
from agents_b200.agents.sac import sac_agent  # noqa: E402
from agents_b200.networks import actor_distribution_rnn_network  # noqa: E402
from agents_b200.networks import critic_network  # noqa: E402
from agents_b200.networks import critic_rnn_network  # noqa: E402
from agents_b200.networks import tanh_normal_projection_network as tnp  # noqa: E402
from agents_b200.specs import tensor_spec  # noqa: E402
from agents_b200.trajectories import time_step as ts  # noqa: E402
from agents_b200.trajectories import trajectory  # noqa: E402
from agents_b200.utils import common  # noqa: E402

B, D, A = 256, 3, 1


def _card():
  return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                        capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]


def _agent(dev, rnn):
  obs = tensor_spec.TensorSpec((D,), torch.float32, 'observation')
  act = tensor_spec.BoundedTensorSpec((A,), torch.float32, -1.0, 1.0, 'action')
  if rnn:
    actor = actor_distribution_rnn_network.ActorDistributionRnnNetwork(
        obs, act, input_fc_layer_params=(400, 300), lstm_size=(40,),
        output_fc_layer_params=(100,), continuous_projection_net=tnp.TanhNormalProjectionNetwork,
        device=dev).set_seed(1)
    critic = critic_rnn_network.CriticRnnNetwork(
        (obs, act), observation_fc_layer_params=None, action_fc_layer_params=None,
        joint_fc_layer_params=(300,), lstm_size=(40,), output_fc_layer_params=(100,),
        device=dev).set_seed(2)
  else:
    actor = tnp.TanhNormalActorNetwork(obs, act, fc_layer_params=(400, 300),
                                       device=dev).set_seed(1)
    critic = critic_network.CriticNetwork((obs, act), observation_fc_layer_params=None,
                                          joint_fc_layer_params=(300,), device=dev).set_seed(2)
  agent = sac_agent.SacAgent(ts.time_step_spec(obs), act, actor_network=actor,
                             critic_network=critic, actor_optimizer=optimizers.Adam(3e-4),
                             critic_optimizer=optimizers.Adam(3e-4),
                             alpha_optimizer=optimizers.Adam(3e-4), target_update_tau=0.05,
                             target_update_period=5, gamma=0.99, reward_scale_factor=0.1)
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
  for b, tm in ((256, 20), (4096, 80)):
    n, T = b * tm, tm + 1
    q1, q2, tq1, tq2, lp = (torch.randn(n, device=dev) for _ in range(5))
    g1, g2, g3 = (torch.empty(n, device=dev) for _ in range(3))
    rew, disc = torch.randn(b, T, device=dev), torch.ones(b, T, device=dev)
    la, dla = torch.zeros(4, device=dev), torch.zeros(4, device=dev)
    loss = torch.empty(1, device=dev)
    partials = torch.empty(_lib.SAC_SEQ_MAX_BLOCKS, device=dev)
    ticket = torch.zeros(1, dtype=torch.int32, device=dev)
    scratch = (None, _lib.ptr(partials), _lib.ptr(ticket))   # the stream is read at each call
    critic = lambda: _lib.call(   # noqa: E731
        'b200rl_sac_seq_critic_loss', _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(tq1), _lib.ptr(tq2),
        _lib.ptr(lp), _lib.ptr(rew), _lib.ptr(disc), T, 1, None, 0, _lib.ptr(la), b, T, 0.99, 0.1,
        0.5, _lib.ptr(loss), _lib.ptr(g1), _lib.ptr(g2), *scratch, _lib.stream())
    actor = lambda: _lib.call(   # noqa: E731
        'b200rl_sac_seq_actor_loss', _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(lp), None, 0,
        _lib.ptr(la), b, T, 1.0, _lib.ptr(loss), _lib.ptr(g1), _lib.ptr(g2), _lib.ptr(g3),
        *scratch, _lib.stream())
    alpha = lambda: _lib.call(   # noqa: E731
        'b200rl_sac_seq_alpha_loss', _lib.ptr(lp), None, 0, _lib.ptr(la), b, T, -0.5, 1, 1.0,
        _lib.ptr(loss), _lib.ptr(dla), *scratch, _lib.stream())
    # bytes each launch needs: critic reads q1, q2, tq1, tq2, next_logp and the [B, T-1] reward /
    # discount, writes dq1, dq2; actor reads q1, q2, logp, writes dlogp, dq1, dq2; alpha reads logp
    for name, call, nbytes in (('seq_critic_loss', critic, 4 * 9 * n),
                               ('seq_actor_loss', actor, 4 * 6 * n),
                               ('seq_alpha_loss', alpha, 4 * n)):
      ms = _graph_time(call, reps)
      rows.append(dict(kernel=name, B=b, T_minus_1=tm, us=round(1e3 * ms, 3),
                       GB_per_s=round(nbytes / (ms * 1e-3) / 1e9, 1)))
  return rows


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--blocks', type=int, default=5)
  p.add_argument('--steps', type=int, default=100)
  p.add_argument('--reps', type=int, default=20000)
  a = p.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('sac_rnn_bench needs a CUDA device.')
  dev = torch.device('cuda:0')
  runs = {}
  for name, rnn, T in (('rnn_T21', True, 21), ('ff_T2', False, 2)):
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
