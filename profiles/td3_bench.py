"""TD3 step time next to the SAC step, one GPU, one process, at the reference TD3 example shapes
(obs 17, act 6; actor (400, 300); critic observation branch (400,), joint (300,); Adam 1e-3,
tau 0.005, actor_update_period 2).  SAC runs its config-4 nets ((256, 256) actor and critics).

One step = agent.train on a fixed [B, 2] batch, captured in one CUDA graph, at B = 64 and 256.
The two agents are timed in alternating blocks; the JSON line gives every block's ms/step, and
the time of each new TD3 kernel from CUDA events over many launches.  The card's name and power
limit are printed with the numbers.
Launch: python profiles/td3_bench.py [--blocks 3] [--steps 300]
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
from agents_b200.agents.sac import sac_agent  # noqa: E402
from agents_b200.agents.td3 import td3_agent  # noqa: E402
from agents_b200.networks import actor_network  # noqa: E402
from agents_b200.networks import critic_network  # noqa: E402
from agents_b200.networks import tanh_normal_projection_network as tnp  # noqa: E402
from agents_b200.specs import tensor_spec  # noqa: E402
from agents_b200.trajectories import time_step as ts  # noqa: E402
from agents_b200.trajectories import trajectory  # noqa: E402
from agents_b200.utils import common  # noqa: E402

D, A = 17, 6


def _card():
  name = torch.cuda.get_device_name()
  try:
    power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader',
                            '-i', str(torch.cuda.current_device())], capture_output=True,
                           text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    power = 'unknown'
  return name, power


def _specs():
  return (tensor_spec.TensorSpec((D,), torch.float32, 'observation'),
          tensor_spec.BoundedTensorSpec((A,), torch.float32, -1.0, 1.0, 'action'))


def _td3(dev):
  obs_spec, act_spec = _specs()
  actor = actor_network.ActorNetwork(obs_spec, act_spec, fc_layer_params=(400, 300),
                                     device=dev).set_seed(1)
  critic = critic_network.CriticNetwork((obs_spec, act_spec), observation_fc_layer_params=(400,),
                                        joint_fc_layer_params=(300,), device=dev).set_seed(2)
  agent = td3_agent.Td3Agent(ts.time_step_spec(obs_spec), act_spec, actor_network=actor,
                             critic_network=critic, actor_optimizer=optimizers.Adam(1e-3),
                             critic_optimizer=optimizers.Adam(1e-3), target_update_tau=0.005,
                             actor_update_period=2, gamma=0.99)
  agent.initialize()
  return agent


def _sac(dev):
  obs_spec, act_spec = _specs()
  actor = tnp.TanhNormalActorNetwork(obs_spec, act_spec, fc_layer_params=(256, 256),
                                     device=dev).set_seed(1)
  critic = critic_network.CriticNetwork((obs_spec, act_spec), joint_fc_layer_params=(256, 256),
                                        device=dev).set_seed(2)
  agent = sac_agent.SacAgent(ts.time_step_spec(obs_spec), act_spec, critic_network=critic,
                             actor_network=actor, actor_optimizer=optimizers.Adam(3e-4),
                             critic_optimizer=optimizers.Adam(3e-4),
                             alpha_optimizer=optimizers.Adam(3e-4), target_update_tau=0.005,
                             gamma=0.99, reward_scale_factor=0.1)
  agent.initialize()
  return agent


def _batch(dev, B):
  g = torch.Generator(device=dev).manual_seed(100 + B)
  one = torch.ones(B, 2, dtype=torch.int32, device=dev)
  return trajectory.Trajectory(one, torch.randn(B, 2, D, device=dev, generator=g),
                               torch.rand(B, 2, A, device=dev, generator=g) * 2 - 1, (), one,
                               torch.rand(B, 2, device=dev, generator=g), torch.ones(B, 2, device=dev))


def _captured_step(agent, traj):
  fn = common.function(lambda: agent.train(traj).loss, warmup=1)
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


def kernel_us(dev, B, launches=2000):
  """Each td3.cu kernel and the gated Adam over the TD3 actor's parameter count."""
  g = torch.Generator(device=dev).manual_seed(7)
  r = lambda *s: torch.randn(*s, device=dev, generator=g)
  q1, q2, tq1, tq2, rew, disc = (r(B) for _ in range(6))
  joint, y = r(B, D + A), torch.tanh(r(B, A))
  H = 400                                  # critic 1's input gradient is w.r.t. [h_obs (400) | a]
  dx = r(B, H + A)
  lo, hi = -torch.ones(A, device=dev), torch.ones(A, device=dev)
  loss, dq1, dq2, dy = torch.empty(1, device=dev), r(B), r(B), r(B, A)
  rng = torch.zeros(2, dtype=torch.int64, device=dev)
  n = 17 * 400 + 400 + 400 * 300 + 300 + 300 * A + A
  p, gr, m, v = r(n), r(n), torch.zeros(n, device=dev), torch.zeros(n, device=dev)
  step = torch.zeros(2, dtype=torch.int64, device=dev)
  ctr_on = torch.zeros((), dtype=torch.int64, device=dev)      # 0 % 2 == 0: the update runs
  ctr_off = torch.ones((), dtype=torch.int64, device=dev)      # 1 % 2 != 0: the update is skipped
  st = _lib.stream()
  calls = {
      'td3_scale_to_spec_noise': lambda: _lib.call(
          'b200rl_td3_scale_to_spec', _lib.ptr(y), A, B, A, _lib.ptr(lo), _lib.ptr(hi), 0.2, 0.5,
          None, 3, _lib.ptr(rng), 0, joint.data_ptr() + 4 * D, D + A, st),
      'td3_critic_loss': lambda: _lib.call(
          'b200rl_td3_critic_loss', _lib.ptr(q1), _lib.ptr(q2), _lib.ptr(tq1), _lib.ptr(tq2),
          _lib.ptr(rew), _lib.ptr(disc), None, B, 0.99, 1.0, _lib.LOSS_HUBER, _lib.ptr(loss),
          _lib.ptr(dq1), _lib.ptr(dq2), None, None, st),
      'td3_actor_loss': lambda: _lib.call(
          'b200rl_td3_actor_loss', _lib.ptr(q1), None, B, _lib.ptr(loss), _lib.ptr(dq1), None, st),
      'td3_actor_bwd': lambda: _lib.call(
          'b200rl_td3_actor_bwd', dx.data_ptr() + 4 * H, H + A, _lib.ptr(lo), _lib.ptr(hi),
          B, A, _lib.ptr(dy), st),
      'adam_tf_gated_skip': lambda: _lib.call(
          'b200rl_adam_tf_gated', _lib.ptr(p), _lib.ptr(gr), _lib.ptr(m), _lib.ptr(v), n, 1e-9,
          0.9, 0.999, 1e-7, _lib.ptr(step), None, _lib.ptr(ctr_off), 2, st),
      'adam_tf_gated_apply': lambda: _lib.call(
          'b200rl_adam_tf_gated', _lib.ptr(p), _lib.ptr(gr), _lib.ptr(m), _lib.ptr(v), n, 1e-9,
          0.9, 0.999, 1e-7, _lib.ptr(step), None, _lib.ptr(ctr_on), 2, st),
  }
  out = {}
  for name, fn in calls.items():
    for _ in range(20):
      fn()
    torch.cuda.synchronize()
    out[name] = 1000 * _time(fn, launches)
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--blocks', type=int, default=3)
  ap.add_argument('--steps', type=int, default=300)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('td3_bench needs a CUDA device.')
  dev = torch.device('cuda', 0)
  name, power = _card()
  for B in (64, 256):
    fns = dict(td3=_captured_step(_td3(dev), _batch(dev, B)),
               sac=_captured_step(_sac(dev), _batch(dev, B)))
    ms = dict(td3=[], sac=[])
    for _ in range(args.blocks):
      for k in ('td3', 'sac'):
        ms[k].append(_time(fns[k], args.steps))
    med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
    print(json.dumps(dict(
        bench='td3_step', gpu=name, power_limit=power, batch=B, cuda_graph=True,
        td3_nets=dict(actor=[400, 300], critic_obs=[400], critic_joint=[300]),
        sac_nets=[256, 256], ms_per_step_td3=ms['td3'], ms_per_step_sac=ms['sac'],
        median_ms_td3=med['td3'], median_ms_sac=med['sac'], td3_over_sac=med['td3'] / med['sac'],
        kernel_us=kernel_us(dev, B))), flush=True)


if __name__ == '__main__':
  main()
