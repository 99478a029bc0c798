"""CriticRnnNetwork (tf_agents/agents/ddpg/critic_rnn_network.py): the recurrent critic of DDPG.

observation branch (optional Conv2D stack, observation_fc (200,)) and action branch (action_fc
(200,), or None: the action enters the concat directly) -> concat -> joint_fc (100,) -> LSTM layers
over [B, T] -> output_fc (200, 100) -> Dense(1).  The two branches and the joint stack use
activation_fn and `kernel_initializer` (default VarianceScaling(1/3, fan_in, uniform)); the output
stack always uses ReLU and the `mlp_layers` default VarianceScaling(2.0, fan_in, truncated
normal); the value layer `last_kernel_initializer` (default U(-0.003, 0.003)).

It is an LSTMEncodingNetwork whose encoder is the two-branch front: the LSTM layers and the output
stack run on its sequence machinery.  Every parameterised layer sits in `_layers` in the
reference's variable order (observation, action, joint, LSTM, output, value), so copies, joint
allocation, target updates and checkpoints see one flat buffer.  The state is the reference's nest
of `map_structure(create_spec, cell.state_size)`: [h, c] named network_state_0 / _1 for one LSTM
layer, a tuple of [h, c] per layer when stacked.

`backward(tape, dq)` gives the parameter gradients; `action_gradient(tape, dq)` gives only
dLoss/d(action) [B*T, A], through the output stack, the LSTM recurrence (BPTT) and the joint and
action stacks, and leaves flat_grads untouched (DDPG's dQ/da).
"""
import torch

from agents_b200 import _lib
from agents_b200.networks import actor_distribution_network
from agents_b200.networks import actor_network
from agents_b200.networks import layers as L
from agents_b200.networks import lstm_encoding_network
from agents_b200.networks import network
from agents_b200.networks import q_network
from agents_b200.specs import tensor_spec
from agents_b200.utils import nest


class _ActionInput(L.Layer):
  """Shape-only marker: the action branch starts here, from the [A] action; it records the width of
  the observation features it follows."""

  def __init__(self, act_dim):
    self.act_dim = act_dim

  def build(self, input_shape):
    if len(input_shape) != 1:
      raise ValueError('CriticRnnNetwork needs rank-1 observation features before the concat, got '
                       '{}; give observation_conv_layer_params / observation_fc_layer_params.'
                       .format(tuple(input_shape)))
    self.obs_width = int(input_shape[0])
    return (self.act_dim,)


class _Concat(L.Layer):
  """Shape-only marker: the joint stack takes concat(observation features, action features)."""

  def __init__(self, action_input):
    self._action_input = action_input

  def build(self, input_shape):
    return (self._action_input.obs_width + int(input_shape[0]),)


class CriticRnnNetwork(lstm_encoding_network.LSTMEncodingNetwork):
  """`__call__((observation, action), step_type, network_state)` -> (q [B] or [B, T], state)."""

  def __init__(self, input_tensor_spec, observation_conv_layer_params=None,
               observation_fc_layer_params=(200,), action_fc_layer_params=(200,),
               joint_fc_layer_params=(100,), lstm_size=None, output_fc_layer_params=(200, 100),
               activation_fn='relu', kernel_initializer=None, last_kernel_initializer=None,
               rnn_construction_fn=None, rnn_construction_kwargs=None, name='CriticRnnNetwork',
               device='cuda'):
    if lstm_size is None and rnn_construction_fn is None:
      raise ValueError('Need to provide either custom rnn_construction_fn or lstm_size.')
    if lstm_size and rnn_construction_fn:
      raise ValueError('Cannot provide both custom rnn_construction_fn and lstm_size.')
    observation_spec, action_spec = input_tensor_spec
    if len(nest.flatten(observation_spec)) > 1:
      raise ValueError('Only a single observation is supported by this network.')
    if len(nest.flatten(action_spec)) > 1:
      raise ValueError('Only a single action is supported by this network.')
    act = nest.flatten(action_spec)[0]
    if len(act.shape) != 1:
      raise ValueError('CriticRnnNetwork expects a rank-1 action spec.')
    super().__init__(input_tensor_spec, input_fc_layer_params=None, lstm_size=lstm_size,
                     output_fc_layer_params=None, rnn_construction_fn=rnn_construction_fn,
                     name=name, device=device)
    counter = iter(range(2 * len(lstm_size)))

    def cell(n):
      return [tensor_spec.TensorSpec((n,), torch.float32, 'network_state_%d' % next(counter))
              for _ in range(2)]
    specs = tuple(cell(n) for n in lstm_size)
    self._state_spec = specs[0] if len(specs) == 1 else specs
    self._act_dim = int(act.shape[0])
    kinit = kernel_initializer or actor_network._hidden_init
    self._obs_layers = actor_distribution_network.encoder_layers(
        None, observation_conv_layer_params, observation_fc_layer_params, activation_fn, kinit)
    self._act_layers = [L.Dense(n, activation=activation_fn, kernel_initializer=kinit)
                        for n in (action_fc_layer_params or ())]
    self._joint_layers = [L.Dense(n, activation=activation_fn, kernel_initializer=kinit)
                          for n in (joint_fc_layer_params or ())]
    self._post = [L.Dense(n, activation='relu', kernel_initializer=q_network._vs_init)
                  for n in (output_fc_layer_params or ())]
    self._post.append(L.Dense(1, activation=None, kernel_initializer=(
        last_kernel_initializer or actor_network._last_init)))
    self._set_layers(_ActionInput(self._act_dim))

  def _set_layers(self, action_input):
    self._action_input = action_input
    self._pre = (self._obs_layers + [action_input] + self._act_layers +
                 [_Concat(action_input)] + self._joint_layers)
    self._layers = self._pre + self._cells + self._post

  def copy(self, **kwargs):
    """The copy's branch, joint, cell and output lists hold the copied layers."""
    new = network.Network.copy(self, **kwargs)
    it = iter(new._layers)
    take = lambda k: [next(it) for _ in range(k)]   # noqa: E731
    new._obs_layers = take(len(self._obs_layers))
    action_input = next(it)
    new._act_layers = take(len(self._act_layers))
    concat = next(it)
    concat._action_input = action_input
    new._joint_layers = take(len(self._joint_layers))
    new._cells = take(len(self._cells))
    new._post = take(len(self._post))
    new._action_input = action_input
    new._pre = new._layers[:len(self._pre)]
    return new

  def create_variables(self, input_tensor_spec=None, **kwargs):
    return super().create_variables(None)

  @property
  def act_dim(self):
    return self._act_dim

  def _pack_state(self, finals):
    layers = [list(f) for f in finals]
    return layers[0] if len(layers) == 1 else tuple(layers)

  # ---- execution --------------------------------------------------------------------------
  def _encode(self, obs, action):
    """(joint-stack output [N, ...], (obs_tape, act_tape, joint_tape))."""
    obs_tape, act_tape, joint_tape = [], [], []
    h = self._run_stack(self._obs_layers, obs, obs_tape)
    a = self._run_stack(self._act_layers, action, act_tape)
    h, a = h.float(), a.float()
    n, hw, aw = h.shape[0], h.shape[1], a.shape[1]
    if h.stride(1) != 1 or h.stride(0) < hw:
      h = h.contiguous()
    if a.stride(1) != 1 or a.stride(0) < aw:     # e.g. a broadcast action
      a = a.contiguous()
    ldh, lda = h.stride(0), a.stride(0)
    x = torch.empty((n, hw + aw), dtype=torch.float32, device=h.device)
    _lib.call('b200rl_concat2', _lib.dptr(h), ldh, hw, _lib.dptr(a), lda, aw, n, _lib.ptr(x),
              _lib.stream())
    x = self._run_stack(self._joint_layers, x, joint_tape)
    return x, (obs_tape, act_tape, joint_tape, hw)

  def _forward(self, inputs, step_type, network_state):
    observation, action = inputs
    obs, st, B, T, has_time = self._sequence(observation, step_type)
    action = nest.flatten(action)[0]
    action = action.reshape(B * T, self._act_dim)
    x, pre = self._encode(obs, action)
    q, state, ctxs, post_tape = self._run_recurrent(x, st, B, T, network_state)
    return q.reshape(B * T), state, (pre, ctxs, post_tape), (B, T, has_time)

  def __call__(self, inputs, step_type=None, network_state=(), training=False):
    q, state, _, (B, T, has_time) = self._forward(inputs, step_type, network_state)
    return self._unflatten(q, B, T, has_time), state

  def forward_train(self, inputs, step_type=None):
    """[B, T] forward from the zero state that records the tape; returns (q [B*T], tape).
    `inputs` is (observation, action), each [B, T, ...] or the B*T rows with step_type [B, T]."""
    q, _, tape, _ = self._forward(inputs, step_type, ())
    return q, tape

  def backward(self, tape, dq):
    """Back-propagates dLoss/dq [B*T] through `tape`, OVERWRITING flat_grads."""
    (obs_tape, act_tape, joint_tape, hw), ctxs, post_tape = tape
    dx = self._backward_recurrent(ctxs, post_tape, dq.reshape(-1, 1), need_dx=True)
    if joint_tape:
      _, dx = network.Network.backward(self, joint_tape, dx, need_input_grad=True,
                                       zero_grads=False)
    if obs_tape:
      network.Network.backward(self, obs_tape, dx[:, :hw], zero_grads=False)
    if act_tape:
      network.Network.backward(self, act_tape, dx[:, hw:], zero_grads=False)
    return self._grads

  def action_gradient(self, tape, dq):
    """dLoss/d(action) [B*T, A] from dLoss/dq [B*T]: input gradients only, flat_grads is left
    as it is.  The result may be a column view of a wider buffer (row stride `.stride(0)`)."""
    (_, act_tape, joint_tape, hw), ctxs, post_tape = tape
    dx = self._backward_recurrent(ctxs, post_tape, dq.reshape(-1, 1), need_dx=True,
                                  need_param_grads=False)
    if joint_tape:
      _, dx = network.Network.backward(self, joint_tape, dx, need_input_grad=True,
                                       need_param_grads=False)
    da = dx[:, hw:]
    if act_tape:
      _, da = network.Network.backward(self, act_tape, da, need_input_grad=True,
                                       need_param_grads=False)
    return da
