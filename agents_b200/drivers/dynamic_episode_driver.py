"""DynamicEpisodeDriver (tf_agents/drivers/dynamic_episode_driver.py:58-259).

Steps the environment with the policy until `sum(counter) >= num_episodes`, calling every observer
with the Trajectory of each step; `counter` counts boundary steps (`traj.is_boundary()`, :174), so
an episode is counted on the transition that leaves its LAST step.  Without a `time_step`, `run`
resets the environment (:233-234), where DynamicStepDriver continues from `current_time_step()`.

The host-read schedule is DynamicStepDriver's: each iteration only enqueues device work, and as
an iteration adds at most `batch_size` episodes, `ceil(remaining / batch_size)` iterations are
enqueued before the counter is read again.  The sequence of iterations is exactly the
reference's.  Once `maximum_iterations` is reached no read is made, so a bounded collect step can
be captured in a CUDA graph.  The bandit-environment branch (:147-154, :171-172) is not built.
"""
import torch

from agents_b200.drivers import driver
from agents_b200.environments import tf_environment
from agents_b200.policies import tf_policy
from agents_b200.trajectories import time_step as ts
from agents_b200.trajectories import trajectory


class DynamicEpisodeDriver(driver.Driver):
  """A driver that takes N episodes in an environment using a policy."""

  def __init__(self, env, policy, observers=None, transition_observers=None, num_episodes=1):
    if not isinstance(env, tf_environment.TFEnvironment):
      raise ValueError('`env` must be an instance of tf_environment.TFEnvironment.')
    if not isinstance(policy, tf_policy.TFPolicy):
      raise ValueError('`policy` must be an instance of tf_policy.TFPolicy.')
    super(DynamicEpisodeDriver, self).__init__(env, policy, observers, transition_observers)
    self._num_episodes = num_episodes

  def _loop_body(self, counter, time_step, policy_state):
    """One iteration of the reference loop body (:122-176)."""
    action_step = self.policy.action(time_step, policy_state)
    next_time_step = self.env.step(action_step.action)
    policy_state = action_step.state
    traj = trajectory.from_transition(time_step, action_step, next_time_step)
    for observer in self._observers:
      observer(traj)
    for observer in self._transition_observers:
      observer((time_step, action_step, next_time_step))
    counter += (traj.step_type == ts.StepType.LAST).sum()   # += is_boundary (:174)
    return next_time_step, policy_state

  def run(self, time_step=None, policy_state=None, num_episodes=None, maximum_iterations=None):
    """Returns (time_step, policy_state) after the loop (:180-259)."""
    if time_step is None:
      time_step = self.env.reset()
    if policy_state is None:
      policy_state = self.policy.get_initial_state(self.env.batch_size)
    num_episodes = num_episodes or self._num_episodes
    batch = max(int(self.env.batch_size or 1), 1)
    counter = torch.zeros((), dtype=torch.int64, device=time_step.step_type.device)
    counted, done_iters = 0, 0
    while counted < num_episodes:
      k = -(-(num_episodes - counted) // batch)
      if maximum_iterations is not None:
        k = min(k, int(maximum_iterations) - done_iters)
      if k <= 0:
        break
      for _ in range(k):
        time_step, policy_state = self._loop_body(counter, time_step, policy_state)
      done_iters += k
      if maximum_iterations is not None and done_iters >= int(maximum_iterations):
        break
      counted = int(counter.item())       # the only host read; skipped under maximum_iterations
    return time_step, policy_state
