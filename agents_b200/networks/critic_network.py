"""CriticNetwork (tf_agents/agents/ddpg/critic_network.py:163-178 as used by the SAC example
examples/sac/haarnoja18/sac_train_eval.py:184-187): concat(observation, action) -> joint MLP ->
Dense(1), output squeezed to [B].  Kernels default to glorot_uniform like the reference call.

With `observation_fc_layer_params` (the TD3 / DDPG examples pass (400,)) the observation first
goes through its own Dense stack: concat(h_obs, action) -> joint MLP -> Dense(1).  The network
still takes the [N, D+A] joint input; the observation branch reads its first D columns.  All
parameterised layers stay in `_layers` in flat-buffer order (observation, joint, output), so
copies, joint allocation, target updates and checkpoints see one flat buffer as before.
"""
import torch

from agents_b200 import _lib
from agents_b200.networks import layers as L
from agents_b200.networks import network
from agents_b200.utils import nest


class _ObservationColumns(L.Layer):
  """Shape-only marker: the observation branch reads the first D columns of the joint input."""

  def __init__(self, obs_dim):
    self.obs_dim = obs_dim

  def build(self, input_shape):
    return (self.obs_dim,)


class _ConcatAction(L.Layer):
  """Shape-only marker: the joint stack takes concat(h_obs, action)."""

  def __init__(self, act_dim):
    self.act_dim = act_dim

  def build(self, input_shape):
    return (int(input_shape[0]) + self.act_dim,)


class CriticNetwork(network.Network):

  def __init__(self, input_tensor_spec, observation_fc_layer_params=None,
               action_fc_layer_params=None, joint_fc_layer_params=(256, 256),
               activation_fn='relu', kernel_initializer=None, last_kernel_initializer=None,
               name='CriticNetwork', device='cuda'):
    if action_fc_layer_params:
      raise NotImplementedError('action_fc_layer_params is not supported: the action enters the '
                                'joint stack directly.')
    obs_spec, act_spec = input_tensor_spec
    obs_spec, act_spec = nest.flatten(obs_spec)[0], nest.flatten(act_spec)[0]
    if len(obs_spec.shape) != 1 or len(act_spec.shape) != 1:
      raise ValueError('CriticNetwork expects rank-1 observation and action specs.')
    self._obs_dim, self._act_dim = int(obs_spec.shape[0]), int(act_spec.shape[0])
    from agents_b200.specs import tensor_spec
    joint = tensor_spec.TensorSpec((self._obs_dim + self._act_dim,), torch.float32)
    super().__init__(input_tensor_spec=joint, state_spec=(), name=name, device=device)
    self._pair_spec = input_tensor_spec
    layers = []
    self._n_obs_layers = len(observation_fc_layer_params or [])
    if self._n_obs_layers:
      layers.append(_ObservationColumns(self._obs_dim))
      for units in observation_fc_layer_params:
        layers.append(L.Dense(units, activation=activation_fn,
                              kernel_initializer=kernel_initializer))
      layers.append(_ConcatAction(self._act_dim))
    for units in (joint_fc_layer_params or []):
      layers.append(L.Dense(units, activation=activation_fn, kernel_initializer=kernel_initializer))
    layers.append(L.Dense(1, activation=None, kernel_initializer=last_kernel_initializer))
    self._layers = layers

  def create_variables(self, input_tensor_spec=None, **kwargs):
    return super().create_variables(None)

  @property
  def obs_dim(self):
    return self._obs_dim

  @property
  def act_dim(self):
    return self._act_dim

  @property
  def action_column(self):
    """First column of the action inside the input gradient that `backward(...,
    need_input_grad=True)` returns: obs_dim for the joint-only network, the width of the last
    observation layer with an observation branch (the gradient is then w.r.t. concat(h_obs,
    action))."""
    if not self._n_obs_layers:
      return self._obs_dim
    return self._layers[self._n_obs_layers].units

  def joint_input(self, observation, action, out=None):
    """concat(observation, action) as one [N, D+A] buffer (either may be a strided view), written
    into the first N rows of `out` when given."""
    n = observation.shape[0]
    if out is None:
      out = torch.empty((n, self._obs_dim + self._act_dim), dtype=torch.float32,
                        device=observation.device)
    observation, action = observation.float(), action.float()
    lda = observation.stride(0) if observation.dim() == 2 and observation.stride(1) == 1 else None
    ldb = action.stride(0) if action.dim() == 2 and action.stride(1) == 1 else None
    if lda is None:
      observation, lda = observation.contiguous(), self._obs_dim
    if ldb is None:
      action, ldb = action.contiguous(), self._act_dim
    _lib.call('b200rl_concat2', _lib.dptr(observation), lda, self._obs_dim, _lib.dptr(action), ldb,
              self._act_dim, n, _lib.ptr(out), _lib.stream())
    return out

  @property
  def has_observation_branch(self):
    return bool(self._n_obs_layers)

  def __call__(self, inputs, step_type=None, network_state=(), training=False):
    observation, action = inputs
    out, _ = self.forward_stack(*self.stack_input(observation, action))
    return out.squeeze(-1), network_state

  def forward_train_joint(self, x):
    """x is the [N, D+A] joint input; returns (q [N, 1], tape)."""
    return self._run(x, keep=True)

  def stack_input(self, observation, action, keep=False):
    """(x, obs_tape): x is the input of the joint stack, concat(observation, action) [N, D+A]
    for the joint-only network and concat(h_obs, action) [N, H+A] with an observation branch,
    whose tape (when keep) is obs_tape.  The action sits at columns [action_column,
    action_column + A) of x, so a caller may rewrite it there before `forward_stack`."""
    if not self._n_obs_layers:
      return self.joint_input(observation, action), None
    h, obs_tape = self.observation_features(observation, keep)
    action = action.float()
    if action.stride(1) != 1:
      action = action.contiguous()
    n, hd = h.shape
    x = torch.empty((n, hd + self._act_dim), dtype=torch.float32, device=h.device)
    _lib.call('b200rl_concat2', _lib.ptr(h), hd, hd, _lib.dptr(action), action.stride(0),
              self._act_dim, n, _lib.ptr(x), _lib.stream())
    return x, obs_tape

  def observation_features(self, observation, keep=False):
    """(h_obs [N, H], obs_tape) of the observation branch, the part of the joint-stack input that
    does not depend on the action.  Requires an observation branch."""
    self._require_built()
    obs_tape = []
    h = observation.float()
    for l in self._layers[1:1 + self._n_obs_layers]:
      y = l.forward(h)
      if keep:
        obs_tape.append((l, h, y))
      h = y
    return h, obs_tape

  def forward_stack(self, x, obs_tape=None, keep=False):
    """(q [N, 1], tape for `backward`) from the joint-stack input `stack_input` returned."""
    if not self._n_obs_layers:
      return super()._run(x, keep)
    joint_tape = []
    for l in self._layers[2 + self._n_obs_layers:]:
      y = l.forward(x)
      if keep:
        joint_tape.append((l, x, y))
      x = y
    return x, (obs_tape, joint_tape)

  def _run(self, x, keep):
    if not self._n_obs_layers:
      return super()._run(x, keep)
    if x.stride(1) != 1:
      x = x.contiguous()
    return self.forward_stack(*self.stack_input(x[:, :self._obs_dim], x[:, self._obs_dim:], keep),
                              keep=keep)

  def backward(self, tape, dy, need_input_grad=False, need_param_grads=True, grad_hook=None,
               zero_grads=True):
    """As Network.backward.  With an observation branch the input gradient is w.r.t.
    concat(h_obs, action), the action at `action_column`.  The joint stack's first Dense gets no
    producer activation, so h_obs's ReLU derivative is applied by the observation stack's own
    backward to the h_obs columns only, never to the action columns."""
    if not self._n_obs_layers:
      return super().backward(tape, dy, need_input_grad, need_param_grads, grad_hook, zero_grads)
    obs_tape, joint_tape = tape
    grads, dj = super().backward(joint_tape, dy, True, need_param_grads, grad_hook, zero_grads)
    if need_param_grads:
      super().backward(obs_tape, dj[:, :self.action_column], False, True, grad_hook,
                       zero_grads=False)
    return (grads, dj) if need_input_grad else grads
