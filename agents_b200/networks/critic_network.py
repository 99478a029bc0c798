"""CriticNetwork (tf_agents/agents/ddpg/critic_network.py:163-178 as used by the SAC example
examples/sac/haarnoja18/sac_train_eval.py:184-187): concat(observation, action) -> joint MLP ->
Dense(1), output squeezed to [B].  Kernels default to glorot_uniform like the reference call."""
import torch

from agents_b200 import _lib
from agents_b200.networks import layers as L
from agents_b200.networks import network
from agents_b200.utils import nest


class CriticNetwork(network.Network):

  def __init__(self, input_tensor_spec, joint_fc_layer_params=(256, 256), activation_fn='relu',
               kernel_initializer=None, last_kernel_initializer=None, name='CriticNetwork',
               device='cuda'):
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

  def __call__(self, inputs, step_type=None, network_state=(), training=False):
    observation, action = inputs
    out, _ = self._run(self.joint_input(observation, action), keep=False)
    return out.squeeze(-1), network_state

  def forward_train_joint(self, x):
    """x is the [N, D+A] joint input; returns (q [N, 1], tape)."""
    return self._run(x, keep=True)
