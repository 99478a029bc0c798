"""Replay gather bandwidth sweep (BASELINE.json configs[4]): rows of 28 244 B, batch 64..4096,
T=2, 1M-slot ring, through the copy kernel the library picks (TMA bulk copy: the 28 224-byte
observation leaf is 16-byte aligned).

Each point: 20 launches of b200rl_rb_sample captured in one CUDA graph (fresh Philox rows per
launch, outputs rotate over 4 buffers so no launch rewrites L2-resident lines of the previous
one), graph replayed 10x, timed with CUDA events.  Algorithmic bytes = 2*B*T*row + 8*B*T.
Prints one JSON line per point plus a contiguous device-copy ceiling.
"""
import ctypes
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from agents_b200 import _lib  # noqa: E402
from agents_b200.replay_buffers import tf_uniform_replay_buffer as rb_mod  # noqa: E402
from agents_b200.specs import tensor_spec  # noqa: E402
from agents_b200.trajectories import trajectory  # noqa: E402
from agents_b200.utils import nest  # noqa: E402

ROW = 28244


def main():
  import argparse
  ap = argparse.ArgumentParser()
  ap.add_argument('--batches', default='64,256,1024,4096')
  args = ap.parse_args()
  batches = [int(v) for v in args.batches.split(',')]
  dev = torch.device('cuda:0')
  peak = 6571.6
  p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'MEASURED_PEAKS.json')
  if os.path.exists(p):
    peak = json.load(open(p))['hbm_gbs']
  spec = trajectory.Trajectory(
      tensor_spec.TensorSpec([], torch.int32, 'step_type'),
      tensor_spec.TensorSpec((84, 84, 4), torch.uint8, 'observation'),
      tensor_spec.TensorSpec([], torch.int32, 'action'), (),
      tensor_spec.TensorSpec([], torch.int32, 'next_step_type'),
      tensor_spec.TensorSpec([], torch.float32, 'reward'),
      tensor_spec.TensorSpec([], torch.float32, 'discount'))
  B_env, L = 256, 4096
  rb = rb_mod.TFUniformReplayBuffer(spec, batch_size=B_env, max_length=L, device=dev, seed=1)
  rb._last_id.fill_(3 * L)
  rb._last_id_host = 3 * L
  flat = nest.flatten(spec)
  T = 2
  nl, reps, nbuf = 20, 10, 4
  # contiguous copy ceiling
  a = torch.empty(1 << 30, dtype=torch.uint8, device=dev)
  b = torch.empty_like(a)
  for _ in range(3):
    b.copy_(a)
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(10):
    b.copy_(a)
  e1.record()
  torch.cuda.synchronize()
  print(json.dumps(dict(kind='copy_ceiling', gbs=2 * a.numel() * 10 / (e0.elapsed_time(e1) * 1e-3) / 1e9,
                        peak=peak)), flush=True)
  del a, b
  for B in batches:
    bufs = []
    for _ in range(nbuf):
      outs = [torch.empty((B, T) + s.shape, dtype=s.dtype, device=dev) for s in flat]
      bufs.append((outs, _lib.ptr_array(outs), torch.empty((B, T), dtype=torch.int64, device=dev),
                   torch.empty(B, dtype=torch.float32, device=dev)))

    def launch(i):
      outs, ptrs, ids, prob = bufs[i % nbuf]
      _lib.call('b200rl_rb_sample', ctypes.byref(rb._ring), B, T, None, None, rb._seed,
                _lib.ptr(rb._ctrl[0:1]), ptrs, _lib.ptr(ids), None, _lib.ptr(prob),
                _lib.ptr(rb._ctrl[1:2]), _lib.stream())

    for i in range(3):
      launch(i)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      for i in range(nl):
        launch(i)
    g.replay()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
      g.replay()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / (nl * reps)
    nbytes = 2 * B * T * ROW + 8 * B * T
    gbs = nbytes / (us * 1e-6) / 1e9
    print(json.dumps(dict(kind='gather', B=B, T=T, us=us, gbs=gbs, frac=gbs / peak,
                          bytes=nbytes)), flush=True)
    del bufs


if __name__ == '__main__':
  main()
