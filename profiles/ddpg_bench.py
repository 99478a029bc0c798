"""DDPG step time next to the TD3 step, one GPU, one process, at the reference DDPG example shapes
(obs 17, act 6; actor (400, 300); critic observation branch (400,), joint (300,); Adam 1e-3,
tau 0.005).  TD3 runs the same networks with actor_update_period 2.

One step = agent.train on a fixed [B, 2] batch, captured in one CUDA graph, at B = 64 and 256.
The two agents are timed in alternating blocks; the JSON line gives every block's ms/step, and
the time of each new DDPG kernel from CUDA events over many launches (b200rl_ou_noise at N = 1
and N = 4096 rows).  The card's name and power limit are printed with the numbers.
Launch: python profiles/ddpg_bench.py [--blocks 3] [--steps 300]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from agents_b200 import _lib  # noqa: E402
from agents_b200 import optimizers  # noqa: E402
from agents_b200.agents.ddpg import ddpg_agent  # noqa: E402
from agents_b200.agents.td3 import td3_agent  # noqa: E402
from agents_b200.networks import actor_network  # noqa: E402
from agents_b200.networks import critic_network  # noqa: E402
from agents_b200.trajectories import time_step as ts  # noqa: E402
from profiles import td3_bench  # noqa: E402

D, A = td3_bench.D, td3_bench.A


def _nets(dev):
  obs_spec, act_spec = td3_bench._specs()
  actor = actor_network.ActorNetwork(obs_spec, act_spec, fc_layer_params=(400, 300),
                                     device=dev).set_seed(1)
  critic = critic_network.CriticNetwork((obs_spec, act_spec), observation_fc_layer_params=(400,),
                                        joint_fc_layer_params=(300,), device=dev).set_seed(2)
  return ts.time_step_spec(obs_spec), act_spec, actor, critic


def _ddpg(dev):
  step_spec, act_spec, actor, critic = _nets(dev)
  agent = ddpg_agent.DdpgAgent(step_spec, act_spec, actor_network=actor, critic_network=critic,
                               actor_optimizer=optimizers.Adam(1e-3),
                               critic_optimizer=optimizers.Adam(1e-3), target_update_tau=0.005,
                               gamma=0.99)
  agent.initialize()
  return agent


def _td3(dev):
  step_spec, act_spec, actor, critic = _nets(dev)
  agent = td3_agent.Td3Agent(step_spec, act_spec, actor_network=actor, critic_network=critic,
                             actor_optimizer=optimizers.Adam(1e-3),
                             critic_optimizer=optimizers.Adam(1e-3), target_update_tau=0.005,
                             actor_update_period=2, gamma=0.99)
  agent.initialize()
  return agent


def kernel_us(dev, B, launches=2000):
  """Each ddpg.cu kernel; the actor loss reads dQ/da at the 406-float row stride of the
  critic's input gradient, as in the agent."""
  g = torch.Generator(device=dev).manual_seed(7)
  r = lambda *s: torch.randn(*s, device=dev, generator=g)
  q, tq, rew, disc = (r(B) for _ in range(4))
  H = 400                                  # the input gradient is w.r.t. [h_obs (400) | a]
  dx = r(B, H + A)
  lo, hi = -torch.ones(A, device=dev), torch.ones(A, device=dev)
  loss, dq, dy = torch.empty(1, device=dev), r(B), r(B, A)
  st = _lib.stream()
  calls = {
      'ddpg_critic_loss': lambda: _lib.call(
          'b200rl_ddpg_critic_loss', _lib.ptr(q), _lib.ptr(tq), _lib.ptr(rew), _lib.ptr(disc),
          None, B, 0.99, 1.0, _lib.LOSS_HUBER, _lib.ptr(loss), _lib.ptr(dq), None, None, st),
      'ddpg_actor_loss': lambda: _lib.call(
          'b200rl_ddpg_actor_loss', dx.data_ptr() + 4 * H, H + A, None, B, A, 1, 0.5, _lib.ptr(lo),
          _lib.ptr(hi), _lib.ptr(loss), _lib.ptr(dy), None, st),
  }
  return _time_calls(calls, launches)


def ou_us(dev, launches=2000):
  """b200rl_ou_noise with device draws and the clamp, at N = 1 and N = 4096 rows."""
  lo, hi = -torch.ones(A, device=dev), torch.ones(A, device=dev)
  state, rng = torch.zeros(A, device=dev), torch.zeros(2, dtype=torch.int64, device=dev)
  calls = {}
  for n in (1, 4096):
    loc, out = torch.zeros(n, A, device=dev), torch.empty(n, A, device=dev)
    calls[f'ou_noise_n{n}'] = (lambda loc=loc, out=out, n=n: _lib.call(
        'b200rl_ou_noise', _lib.ptr(loc), A, n, A, _lib.ptr(state), 0.15, 0.2, None, 3,
        _lib.ptr(rng), _lib.ptr(lo), _lib.ptr(hi), _lib.ptr(out), A, _lib.stream()))
  return _time_calls(calls, launches)


def _time_calls(calls, launches):
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
    raise SystemExit('ddpg_bench needs a CUDA device.')
  dev = torch.device('cuda', 0)
  name, power = td3_bench._card()
  for B in (64, 256):
    fns = dict(ddpg=td3_bench._captured_step(_ddpg(dev), td3_bench._batch(dev, B)),
               td3=td3_bench._captured_step(_td3(dev), td3_bench._batch(dev, B)))
    ms = dict(ddpg=[], td3=[])
    for _ in range(args.blocks):
      for k in ('ddpg', 'td3'):
        ms[k].append(td3_bench._time(fns[k], args.steps))
    med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
    print(json.dumps(dict(
        bench='ddpg_step', gpu=name, power_limit=power, batch=B, cuda_graph=True,
        nets=dict(actor=[400, 300], critic_obs=[400], critic_joint=[300]),
        ms_per_step_ddpg=ms['ddpg'], ms_per_step_td3=ms['td3'], median_ms_ddpg=med['ddpg'],
        median_ms_td3=med['td3'], ddpg_over_td3=med['ddpg'] / med['td3'],
        kernel_us=kernel_us(dev, B))), flush=True)
  print(json.dumps(dict(bench='ou_noise', gpu=name, power_limit=power, A=A,
                        kernel_us=ou_us(dev))), flush=True)


if __name__ == '__main__':
  main()
