"""CPU oracle: a numpy restatement of the reference's algorithms for the hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under agents_b200/ imports this package; only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may.  Every
function cites the reference file:line (relative to tf_agents/ in the reference repository) it restates.

Pinning status (SURVEY.md §8c): ring / window / probability semantics, n-step, returns, GAE,
Q indexing, Polyak, Periodically, DQN/PPO/SAC scalar losses are pinned against the reference's
own test goldens in tests/test_oracle_goldens.py.  TensorFlow is not installable here, so the
RNG stream (tf.random.uniform), random initialisers and optimiser post-step values are
"parity unpinned" in the reference itself; the oracle fixes them by definition (Philox4x32-10
as in oracle/philox.py; TF's documented Adam/RMSProp formulas).
"""
