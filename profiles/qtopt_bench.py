"""QT-Opt step and CEM action time next to the TD3 step, one GPU, one process, on the TD3 example
critic (obs 17, act 6; observation branch (400,), joint (300,); Adam 1e-3, tau 0.005).  TD3 runs
the same critic with an actor (400, 300) and actor_update_period 2.

At B = 64 and 256 states and N = 32 and 64 samples (M = 4 elites, 3 iterations), each captured in
one CUDA graph: a `CEMPolicy.action` on B states, and a full QtOptAgent.train step on a fixed
[B, 2] batch (enable_td3 on), timed in alternating blocks with the TD3 step at the same B.  To see
where a search spends its time, the pieces of one iteration are also timed alone from CUDA events
over many launches: the target critic's joint-stack forward over the B*N rows and one
b200rl_cem_refit.  The card's name and power limit are printed with the numbers.
Launch: python profiles/qtopt_bench.py [--blocks 3] [--steps 300]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from agents_b200 import _lib  # noqa: E402
from agents_b200 import optimizers  # noqa: E402
from agents_b200.agents.qtopt import qtopt_agent  # noqa: E402
from agents_b200.networks import critic_network  # noqa: E402
from agents_b200.policies.samplers import qtopt_cem_actions_sampler_continuous as samplers  # noqa: E402
from agents_b200.trajectories import time_step as ts  # noqa: E402
from agents_b200.utils import common  # noqa: E402
from profiles import td3_bench  # noqa: E402

D, A = td3_bench.D, td3_bench.A
M, ITERS = 4, 3


def _qtopt(dev, N):
  obs_spec, act_spec = td3_bench._specs()
  critic = critic_network.CriticNetwork((obs_spec, act_spec), observation_fc_layer_params=(400,),
                                        joint_fc_layer_params=(300,), device=dev).set_seed(2)
  agent = qtopt_agent.QtOptAgent(
      ts.time_step_spec(obs_spec), act_spec, critic, optimizers.Adam(1e-3),
      samplers.GaussianActionsSampler(act_spec), init_mean_cem=np.zeros(A),
      init_var_cem=np.full(A, 0.25), num_samples_cem=N, num_elites_cem=M, num_iter_cem=ITERS,
      target_update_tau=0.005, gamma=0.99)
  agent.initialize()
  return agent


def _captured(fn):
  g = common.function(fn, warmup=1)
  for _ in range(12):
    g()
  torch.cuda.synchronize()
  return g


def pieces_us(agent, obs, launches=1000):
  """One search iteration's parts alone: the joint-stack forward over B*N rows, one cem_refit."""
  pol = agent.policy
  net, N, B = pol.q_network, pol._num_samples, obs.shape[0]
  h, _ = net.observation_features(obs)
  x = torch.randn(B * N, h.shape[1] + A, device=obs.device)
  q, _ = net.forward_stack(x)
  mean, var = torch.empty(B, A, device=obs.device), torch.empty(B, A, device=obs.device)
  rng = torch.zeros(2, dtype=torch.int64, device=obs.device)
  H = h.shape[1]
  calls = {
      'forward_BN_rows': lambda: net.forward_stack(x),
      'cem_refit': lambda: _lib.call(
          'b200rl_cem_refit', _lib.ptr(q), None, _lib.ptr(x), H + A, H, B, N, M, A, 1e-4,
          _lib.ptr(pol._amin), _lib.ptr(pol._amax), 0, None, 1, _lib.ptr(rng), _lib.ptr(mean),
          _lib.ptr(var), None, None, _lib.stream()),
  }
  out = {}
  for name, fn in calls.items():
    for _ in range(20):
      fn()
    torch.cuda.synchronize()
    out[name] = 1000 * td3_bench._time(fn, launches)
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--blocks', type=int, default=3)
  ap.add_argument('--steps', type=int, default=300)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('qtopt_bench needs a CUDA device.')
  dev = torch.device('cuda', 0)
  name, power = td3_bench._card()
  for B in (64, 256):
    traj = td3_bench._batch(dev, B)
    td3 = td3_bench._captured_step(td3_bench._td3(dev), traj)
    obs = torch.randn(B, D, device=dev, generator=torch.Generator(device=dev).manual_seed(B))
    step = ts.restart(obs, batch_size=B)
    for N in (32, 64):
      agent = _qtopt(dev, N)
      fns = dict(action=_captured(lambda: agent.policy.action(step).action),
                 train=_captured(lambda: agent.train(traj).loss), td3=td3)
      ms = {k: [] for k in fns}
      for _ in range(args.blocks):
        for k, fn in fns.items():
          ms[k].append(td3_bench._time(fn, args.steps))
      med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
      print(json.dumps(dict(
          bench='qtopt', gpu=name, power_limit=power, batch=B, num_samples=N, num_elites=M,
          num_iter=ITERS, cuda_graph=True, critic=dict(obs=[400], joint=[300]),
          ms_per_call=ms, median_ms_cem_action=med['action'],
          median_ms_qtopt_train=med['train'], median_ms_td3_train=med['td3'],
          search_piece_us=pieces_us(agent, obs))), flush=True)


if __name__ == '__main__':
  main()
