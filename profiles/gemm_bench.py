"""Q-network GEMM micro-benchmark: Mnih'15 net at batch 256, forward (+tape) and backward, per
GEMM engine (0 = fp32 FFMA, 1 = wgmma 3xTF32, 2 = wgmma 1xTF32).  CUDA events, 20 reps.
Usage: python profiles/gemm_bench.py [--modes 0,1] [--reps 20] [--layer conv2]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from agents_b200 import _lib  # noqa: E402
from agents_b200.networks import layers as L  # noqa: E402
from agents_b200.networks import q_network  # noqa: E402
from agents_b200.specs import tensor_spec  # noqa: E402


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--modes', default='0,1')
  ap.add_argument('--reps', type=int, default=20)
  ap.add_argument('--batch', type=int, default=256)
  args = ap.parse_args()
  dev = torch.device('cuda:0')
  obs_spec = tensor_spec.TensorSpec((84, 84, 4), torch.uint8)
  act_spec = tensor_spec.BoundedTensorSpec((), torch.int32, 0, 5)
  net = q_network.QNetwork(obs_spec, act_spec, preprocessing_layers=L.CastScale(255.),
                           conv_layer_params=((32, 8, 4), (64, 4, 2), (64, 3, 1)), fc_layer_params=(512,),
                           device=dev).set_seed(0)
  net.create_variables()
  x = torch.randint(0, 256, (args.batch, 84, 84, 4), dtype=torch.uint8, device=dev)
  dq = torch.randn(args.batch, 6, device=dev)
  flops_fwd = 2 * 9.35e6 * args.batch
  for mode in [int(m) for m in args.modes.split(',')]:
    _lib.call('b200rl_set_gemm_mode', mode)
    for _ in range(3):
      q, tape = net.forward_train(x)
      net.backward(tape, dq)
    torch.cuda.synchronize()
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    e[0].record()
    for _ in range(args.reps):
      q, tape = net.forward_train(x)
    e[1].record()
    for _ in range(args.reps):
      net.backward(tape, dq)
    e[2].record()
    torch.cuda.synchronize()
    fwd = e[0].elapsed_time(e[1]) / args.reps
    bwd = e[1].elapsed_time(e[2]) / args.reps
    print(json.dumps(dict(mode=mode, fwd_ms=fwd, bwd_ms=bwd, fwd_tflops=flops_fwd / fwd / 1e9,
                          bwd_tflops=2 * flops_fwd / bwd / 1e9)), flush=True)


if __name__ == '__main__':
  main()
