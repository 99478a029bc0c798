import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)
HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
  sys.path.insert(0, HERE)          # sibling helper modules (py_env_mocks)


def pytest_configure(config):
  config.addinivalue_line('markers', 'gpu: test needs a CUDA device (an H100)')


@pytest.fixture(scope='session')
def cuda():
  import torch
  if not torch.cuda.is_available():
    pytest.skip('needs a CUDA device')
  return torch.device('cuda:0')


def record_parity(name, **kw):
  """Keeps the LARGEST measured error per (name, key) in gpurun_out/parity_measured.json (merged back
  by gpurun; copied to profiles/ per round) so that every loosened tolerance in the GPU tests can be
  quoted against what was actually measured.  Never fails a test."""
  import json
  path = os.path.join(ROOT, 'gpurun_out', 'parity_measured.json')
  try:
    os.makedirs(os.path.dirname(path), exist_ok=True)
    cur = json.load(open(path)) if os.path.exists(path) else {}
    slot = cur.setdefault(name, {})
    for k, v in kw.items():
      slot[k] = max(float(v), float(slot.get(k, 0.0)))
    json.dump(cur, open(path, 'w'), indent=1, sort_keys=True)
  except (OSError, ValueError):
    pass
