"""Frame-dedup storage semantics (TEST INFRASTRUCTURE ONLY; no product kernel yet — DESIGN.md §8
"next", item 5).

The reference stores Atari observations as 4-frame stacks `[84, 84, 4]` in
`TFUniformReplayBuffer` and offers frame de-duplication only in the host-side
`PyHashedReplayBuffer` (replay_buffers/py_hashed_replay_buffer.py:37-181: frames are hashed,
each unique frame is stored once and stacks are rebuilt on sampling).  The CUDA plan keeps the
ring of `oracle/replay.py` but stores ONE frame per slot and rebuilds the stack in the gather
kernel.  This module fixes the semantics that kernel must reproduce:

  * the producer follows the frame-stack rule of the reference's Atari wrappers
    (environments/atari_wrappers.py:82-126 `FrameStack4`: on reset the deque is filled with the
    first frame, afterwards the newest frame is appended): `stack_rule` below;
  * a slot stores `stack[..., -1]` (the newest frame);
  * channel c of the rebuilt stack for the step with id `i` is the stored frame of id
    `max(i - (K-1-c), first_id_of_the_episode)` in the same segment: `rebuild`;
  * ids whose look-back could reach overwritten slots are not sampleable: the valid range's lower
    bound moves up by K-1 (`valid_range_ids`).
`tests/test_oracle_frame_stack.py` checks that, under these rules, the rebuilt stacks are
bit-identical to what the plain ring returns for the same ids.
"""
import numpy as np

from oracle import replay as oreplay

FIRST = 0


def stack_rule(frames, step_types, K):
  """Stacks a producer following FrameStack-K emits for one environment.

  frames [n, H, W], step_types [n] -> stacks [n, H, W, K]."""
  n = frames.shape[0]
  out = np.zeros(frames.shape + (K,), frames.dtype)
  for t in range(n):
    if step_types[t] == FIRST or t == 0:
      out[t] = np.repeat(frames[t][..., None], K, axis=-1)
    else:
      out[t, ..., :-1] = out[t - 1, ..., 1:]
      out[t, ..., -1] = frames[t]
  return out


def valid_range_ids(last_id, max_length, num_steps, K):
  """Sampleable window starts: the plain range (tf_uniform_replay_buffer.py:610-635) with the
  lower bound raised by K-1 once the ring has wrapped (older frames are gone)."""
  lo, hi = oreplay.valid_range_ids(last_id, max_length, num_steps)
  if last_id + 1 > max_length:
    lo += K - 1
  return lo, hi


def rebuild(frame_storage, step_type_storage, id_table, segment, id_, K, max_length):
  """Stack [H, W, K] of the item with id `id_` in `segment` from single-frame slots."""
  base = segment * max_length
  ids = []
  cur = id_
  for _ in range(K):                       # newest -> oldest; stop walking at the episode's FIRST
    ids.append(cur)
    row = base + cur % max_length
    assert id_table[row] == cur, 'look-back reached an overwritten slot'
    if step_type_storage[row] != FIRST and cur > 0:
      cur -= 1
  ids = ids[::-1]                          # channel 0 = oldest
  return np.stack([frame_storage[base + i % max_length] for i in ids], axis=-1)
