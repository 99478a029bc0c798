"""agents_b200 — the TF-Agents collect -> store -> sample -> update hot path on H100.

A thin Python host (same class surface as tf_agents: TFUniformReplayBuffer,
DynamicStepDriver, DqnAgent/PPOClipAgent/SacAgent, train.Learner) over the C ABI of
libb200rl.so (include/b200rl.h): hand-written sm_90a CUDA.  PyTorch only owns device memory.
"""
__version__ = '0.1.0'
