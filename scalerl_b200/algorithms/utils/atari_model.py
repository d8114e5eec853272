"""CPU actor-side stand-ins used when ScaleRL's own AtariNet / gym env are not available.

``ActorNet`` evaluates the AtariNet architecture (conv 8s4 -> 4s2 -> 3s1 -> fc512 -> [h, clipped reward, one-hot
last action] -> [2-layer LSTM] -> policy/baseline heads; reference: scalerl/algorithms/utils/atari_model.py:30-59,
93-134) for the actor's one-step calls on the CPU and samples an action.  It follows the reference model's CALLING
CONVENTION -- ``actor_model(env_output, agent_state) -> (dict(policy_logits, baseline, action), agent_state)``,
``initial_hidden_state(batch_size)``, ``state_dict()`` / ``load_state_dict()`` with the reference's parameter names and
layouts -- so ImpalaTrainer treats it and the reference's own ``AtariNet`` identically (either can be passed as
``actor_model_fn``); its parameters live in shared memory and are overwritten by the learner's weight publish.
``SyntheticAtariEnv`` emits the TorchEnvWrapper record schema (scalerl/envs/torch_envwrapper.py:43-50,77-84)
with random frames; it exists so the actor/ring/learner plumbing can be exercised without gymnasium/ale_py.
``AtariNet`` is the trainable drop-in for the reference's ``AtariNet`` (atari_model.py:8-143): the same submodules, parameters
and calling convention, with the encoder (obs -> conv1..3 -> fc -> [h, clipped reward, one-hot last action]), the 2-layer LSTM core
(use_lstm=True, bf16) and their backward on the learner's sm_90a kernels under torch autograd.
"""
import ctypes as C
from collections import OrderedDict

import torch
import torch.nn.functional as F
from torch import nn
from torch.autograd.function import once_differentiable

from ... import _lib
from ...learner import param_shapes, reference_param_order


class ActorNet(torch.nn.Module):
    def __init__(self, obs_shape=(4, 84, 84), num_actions=6, use_lstm=False, seed=0):
        super().__init__()
        self.observation_shape = tuple(obs_shape)
        self.num_actions = int(num_actions)
        self.use_lstm = bool(use_lstm)
        self.core_size = 513 + self.num_actions
        self.names = reference_param_order(self.use_lstm)
        g = torch.Generator().manual_seed(seed)
        fan = 1
        shapes = param_shapes(num_actions, self.use_lstm)
        # All parameters are views of ONE flat fp32 buffer laid out like the learner's flat parameter buffer
        # (srl_param_layout_ex): the weight publish is then a single D2H copy into shared memory (impala_atari.py:348).
        from ... import _lib
        from ...learner import PARAM_NAMES, LSTM_PARAM_NAMES
        total, off, cnt = _lib.param_layout(self.num_actions, self.use_lstm)
        lay_names = PARAM_NAMES + (LSTM_PARAM_NAMES if self.use_lstm else ())
        self.flat_layout = {n: (off[i], cnt[i]) for i, n in enumerate(lay_names)}
        self.flat_params = torch.zeros(total)
        for n in self.names:
            shp = shapes[n]
            if n.startswith('rnn_layer.'):
                fan = self.core_size                       # nn.LSTM: U(+-1/sqrt(hidden_size)) for every tensor
            elif n.endswith('.weight'):
                fan = 1
                for d in shp[1:]:
                    fan *= d
            bound = 1.0 / fan ** 0.5
            o, c = self.flat_layout[n]
            view = self.flat_params[o:o + c].view(shp)
            view.copy_((torch.rand(shp, generator=g) * 2 - 1) * bound)
            self.register_parameter(n.replace('.', '_'), torch.nn.Parameter(view, requires_grad=False))

    def share_memory(self):
        """moves the ONE underlying storage to shared memory; every parameter stays a view of it"""
        self.flat_params.share_memory_()
        for n in self.names:
            o, c = self.flat_layout[n]
            self._p(n).data = self.flat_params[o:o + c].view(self._p(n).shape)
        return self

    def _p(self, n):
        return getattr(self, n.replace('.', '_'))

    # ---- the reference model's parameter interface (names of atari_model.py:30-59) -----------------------------------
    def state_dict(self, *args, **kwargs):
        return OrderedDict((n, self._p(n).detach()) for n in self.names)

    def load_state_dict(self, sd, strict=True):
        missing = [n for n in self.names if n not in sd]
        extra = [k for k in sd if k not in self.names]
        if strict and (missing or extra):
            raise RuntimeError(f'ActorNet.load_state_dict: missing keys {missing}, unexpected keys {extra}')
        with torch.no_grad():
            for n in self.names:
                if n in sd:
                    self._p(n).copy_(sd[n])

    def initial_hidden_state(self, batch_size: int):
        """atari_model.py:61-75: () without LSTM, else (h0, c0) zeros [2, batch, 513 + A]"""
        if not self.use_lstm:
            return tuple()
        return tuple(torch.zeros(2, batch_size, self.core_size) for _ in range(2))

    def _lstm_step(self, x, state):
        """one time step of the 2-layer nn.LSTM (gate order i, f, g, o); state = (h [2,B,H], c [2,B,H])"""
        h_in, c_in = state
        hs, cs = [], []
        for layer in (0, 1):
            gates = (F.linear(x, self._p(f'rnn_layer.weight_ih_l{layer}'), self._p(f'rnn_layer.bias_ih_l{layer}'))
                     + F.linear(h_in[layer], self._p(f'rnn_layer.weight_hh_l{layer}'), self._p(f'rnn_layer.bias_hh_l{layer}')))
            i, f, g, o = gates.chunk(4, dim=-1)
            c = torch.sigmoid(f) * c_in[layer] + torch.sigmoid(i) * torch.tanh(g)
            x = torch.sigmoid(o) * torch.tanh(c)
            hs.append(x)
            cs.append(c)
        return x, (torch.stack(hs), torch.stack(cs))

    @torch.no_grad()
    def forward(self, inputs, rnn_state=()):
        x = inputs['obs']
        T, B = x.shape[:2]
        x = x.reshape(T * B, *x.shape[2:]).float() / 255.0
        x = F.relu(F.conv2d(x, self._p('conv1.weight'), self._p('conv1.bias'), stride=4))
        x = F.relu(F.conv2d(x, self._p('conv2.weight'), self._p('conv2.bias'), stride=2))
        x = F.relu(F.conv2d(x, self._p('conv3.weight'), self._p('conv3.bias'), stride=1))
        x = F.relu(F.linear(x.reshape(T * B, -1), self._p('fc.weight'), self._p('fc.bias')))
        one_hot = F.one_hot(inputs['action'].reshape(T * B), self.num_actions).float()
        core = torch.cat([x, torch.clamp(inputs['reward'], -1, 1).reshape(T * B, 1), one_hot], dim=-1)
        if self.use_lstm:
            core = core.view(T, B, -1)
            notdone = (~inputs['done']).float()
            outs = []
            for t in range(T):
                nd = notdone[t].view(1, B, 1)
                rnn_state = tuple(nd * s for s in rnn_state)        # state reset at episode ends (atari_model.py:114-116)
                y, rnn_state = self._lstm_step(core[t], rnn_state)
                outs.append(y)
            core = torch.cat(outs, 0)
        else:
            rnn_state = tuple()
        logits = F.linear(core, self._p('policy.weight'), self._p('policy.bias'))
        baseline = F.linear(core, self._p('baseline.weight'), self._p('baseline.bias'))
        if self.training:
            action = torch.multinomial(F.softmax(logits, dim=1), num_samples=1)
        else:
            action = torch.argmax(logits, dim=1)
        return dict(policy_logits=logits.view(T, B, -1), baseline=baseline.view(T, B), action=action.view(T, B)), rnn_state


PRECISIONS = {'bf16': 0, 'fp32_split': 1}     # ImpalaHParams.precision -> srl_config_t.precision
MAX_ACTIONS = 31                             # one warp lane per action plus one for the baseline, as B200ImpalaLearner
MAX_FRAMES = 65536                           # T * B of one call (MAX_FRAMES in csrc/kernels.h)
LSTM_WEIGHTS = tuple(f'{w}_l{l}' for l in (0, 1) for w in ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh'))   # srl_lstm_create order


class _EncoderContexts:
    """The native encoder contexts of one AtariNet, one per device: the stream lanes, their events and the precision (no
    activations: those belong to each call).  Created on the first forward on a device, released with the module; a deep copy
    starts without any."""

    def __init__(self, precision: int):
        self.precision = precision
        self.handles = {}

    def get(self, device: torch.device) -> C.c_void_p:
        h = self.handles.get(device.index)
        if h is None:
            h = C.c_void_p()
            with torch.cuda.device(device):
                _lib.check(_lib.lib().srl_encoder_create(self.precision, C.byref(h)), 'srl_encoder_create')
            self.handles[device.index] = h
        return h

    def __deepcopy__(self, memo):
        return _EncoderContexts(self.precision)

    def __getstate__(self):
        return {'precision': self.precision}

    def __setstate__(self, state):
        self.precision, self.handles = state['precision'], {}

    def __del__(self):
        try:
            for h in self.handles.values():
                _lib.lib().srl_encoder_destroy(h)
        except Exception:      # interpreter shutdown: the library may already be gone
            pass
        self.handles = {}


def encoder_block_sizes(frames: int, precision: str = 'bf16'):
    """(bytes a forward keeps for its backward, bytes of one call's scratch) for ``frames`` frames"""
    if precision not in PRECISIONS:
        raise ValueError(f"precision must be one of {sorted(PRECISIONS)}, got {precision!r}")
    saved, scratch = C.c_int64(), C.c_int64()
    _lib.check(_lib.lib().srl_encoder_sizes(int(frames), PRECISIONS[precision], C.byref(saved), C.byref(scratch)), 'srl_encoder_sizes')
    return saved.value, scratch.value


def _ptrs8(tensors):
    return (C.c_void_p * 8)(*[t.data_ptr() for t in tensors])


def _encoder_forward(handle, precision, num_actions, obs, reward, action, weights):
    """-> (core [N, 513+A], the forward's saved block); obs / reward / action flat over N frames, on the weights' device"""
    n, dev = reward.numel(), reward.device
    saved_bytes, scratch_bytes = encoder_block_sizes(n, precision)
    saved = torch.empty(saved_bytes, dtype=torch.uint8, device=dev)
    scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=dev)
    core = torch.empty(n, 513 + num_actions, dtype=torch.float32, device=dev)
    _lib.check(_lib.lib().srl_encoder_forward(handle, obs.data_ptr(), reward.data_ptr(), action.data_ptr(), n, num_actions, _ptrs8(weights),
                                              saved.data_ptr(), scratch.data_ptr(), core.data_ptr(), torch.cuda.current_stream(dev).cuda_stream),
               'srl_encoder_forward')
    return core, saved


class _EncoderCore(torch.autograd.Function):
    """core = [relu(fc(conv3(conv2(conv1(obs / 255))))), clamp(reward, -1, 1), one_hot(action)] (atari_model.py:91-107), differentiable
    in the 8 conv / fc tensors.  The forward's activations and packed weights are one block saved on ``ctx``: every call keeps its own,
    and the gradient is taken at the weights the forward ran with."""

    @staticmethod
    def forward(ctx, handle, precision, num_actions, obs, reward, action, *weights):
        core, saved = _encoder_forward(handle, precision, num_actions, obs, reward, action, weights)
        ctx.save_for_backward(saved)
        ctx.call = (handle, precision, num_actions, reward.numel(), [w.shape for w in weights])
        return core

    @staticmethod
    @once_differentiable
    def backward(ctx, dcore):
        handle, precision, num_actions, n, shapes = ctx.call
        (saved,) = ctx.saved_tensors
        dev = saved.device
        dcore = dcore.contiguous()
        grads = [torch.empty(s, dtype=torch.float32, device=dev) for s in shapes]
        scratch = torch.empty(encoder_block_sizes(n, precision)[1], dtype=torch.uint8, device=dev)
        _lib.check(_lib.lib().srl_encoder_backward(handle, dcore.data_ptr(), n, num_actions, saved.data_ptr(), scratch.data_ptr(),
                                                   _ptrs8(grads), torch.cuda.current_stream(dev).cuda_stream), 'srl_encoder_backward')
        return (None,) * 6 + tuple(grads)


def lstm_block_sizes(T1: int, B: int, num_actions: int):
    """(bytes an LSTM core forward keeps for its backward, bytes of one call's scratch) for T1 x B rows"""
    saved, scratch = C.c_int64(), C.c_int64()
    _lib.check(_lib.lib().srl_lstm_core_sizes(int(T1), int(B), int(num_actions), C.byref(saved), C.byref(scratch)), 'srl_lstm_core_sizes')
    return saved.value, scratch.value


def _lstm_forward(num_actions, core, done, h0, c0, weights):
    """-> (out [T1,B,H], hT, cT [2,B,H], the forward's saved block); core f32 [T1,B,H], done u8 [T1,B], all contiguous on one device"""
    T1, B, H = core.shape
    dev = core.device
    saved_bytes, scratch_bytes = lstm_block_sizes(T1, B, num_actions)
    saved = torch.empty(saved_bytes, dtype=torch.uint8, device=dev)
    scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=dev)
    out = torch.empty(T1, B, H, dtype=torch.float32, device=dev)
    hT, cT = (torch.empty(2, B, H, dtype=torch.float32, device=dev) for _ in range(2))
    _lib.check(_lib.lib().srl_lstm_core_forward(core.data_ptr(), done.data_ptr(), h0.data_ptr(), c0.data_ptr(), num_actions, T1, B,
                                                _ptrs8(weights), saved.data_ptr(), scratch.data_ptr(), out.data_ptr(), hT.data_ptr(),
                                                cT.data_ptr(), torch.cuda.current_stream(dev).cuda_stream), 'srl_lstm_core_forward')
    return out, hT, cT, saved


def _ptr_or_none(t):
    return None if t is None else t.data_ptr()


class _LstmCore(torch.autograd.Function):
    """(out, hT, cT) of the 2-layer LSTM over T1 steps with the state reset where done (atari_model.py:109-120), differentiable in the
    core, the initial state (h0, c0) and the 8 nn.LSTM tensors.  As _EncoderCore, the forward's activations and packed weights are one
    block saved on ``ctx``.  Unused gradients of hT / cT reach the kernels as NULL (no materialised zeros)."""

    @staticmethod
    def forward(ctx, num_actions, core, done, h0, c0, *weights):
        out, hT, cT, saved = _lstm_forward(num_actions, core, done, h0, c0, weights)
        ctx.save_for_backward(saved)
        ctx.call = (num_actions, tuple(core.shape), [w.shape for w in weights])
        ctx.set_materialize_grads(False)
        return out, hT, cT

    @staticmethod
    @once_differentiable
    def backward(ctx, dout, dhT, dcT):
        num_actions, (T1, B, H), shapes = ctx.call
        (saved,) = ctx.saved_tensors
        dev = saved.device
        dout = torch.zeros(T1, B, H, device=dev) if dout is None else dout.contiguous()
        dhT = None if dhT is None else dhT.contiguous()
        dcT = None if dcT is None else dcT.contiguous()
        want_h0, want_c0 = ctx.needs_input_grad[3], ctx.needs_input_grad[4]
        dcore = torch.empty(T1, B, H, device=dev)
        dh0 = torch.empty(2, B, H, device=dev) if want_h0 else None
        dc0 = torch.empty(2, B, H, device=dev) if want_c0 else None
        grads = [torch.empty(s, dtype=torch.float32, device=dev) for s in shapes]
        scratch = torch.empty(lstm_block_sizes(T1, B, num_actions)[1], dtype=torch.uint8, device=dev)
        _lib.check(_lib.lib().srl_lstm_core_backward(dout.data_ptr(), _ptr_or_none(dhT), _ptr_or_none(dcT), num_actions, T1, B, saved.data_ptr(),
                                                     scratch.data_ptr(), _ptrs8(grads), dcore.data_ptr(), _ptr_or_none(dh0), _ptr_or_none(dc0),
                                                     torch.cuda.current_stream(dev).cuda_stream), 'srl_lstm_core_backward')
        return (None, dcore if ctx.needs_input_grad[1] else None, None, dh0, dc0) + tuple(grads)


class AtariNet(nn.Module):
    """Drop-in for the reference's ``AtariNet`` (scalerl/algorithms/utils/atari_model.py:8-143) that trains on the sm_90a encoder.

    Submodules, their names, creation order and initialisation are the reference's, so ``state_dict()`` and the initial weights under
    ``torch.manual_seed`` match it.  ``forward(inputs, rnn_state)`` takes and returns what the reference's does; the encoder up to the
    LSTM / head input runs as one autograd function on the learner's kernels, and so does the LSTM core with ``precision='bf16'``
    (``rnn_state`` = (h0, c0) float32 [2, B, 513 + A] on the module's device; it returns (hT, cT) as ``nn.LSTM`` does).  ``rnn_layer``
    stays an ``nn.LSTM``: its tensors are the kernels' weights.  The heads and the action sampling are torch.
    ``precision``: 'bf16' or 'fp32_split', as ``ImpalaHParams.precision``; 'fp32_split' steps the LSTM with ``nn.LSTM`` (the LSTM kernels
    have bf16 operands only).  ``validate_inputs``: raise on actions outside [0, A) as ``F.one_hot`` does (one host synchronisation per
    forward); otherwise they are clamped.  CUDA only: CPU actors use ``ActorNet``."""

    def __init__(self, observation_shape, num_actions, use_lstm=False, *, precision='bf16', validate_inputs=False):
        super().__init__()
        if tuple(observation_shape) != (4, 84, 84):
            raise ValueError(f'observation_shape must be (4, 84, 84), got {tuple(observation_shape)}')
        if not 1 <= int(num_actions) <= MAX_ACTIONS:
            raise ValueError(f'num_actions={num_actions} must be in [1, {MAX_ACTIONS}]')
        if precision not in PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(PRECISIONS)}, got {precision!r}")
        self.observation_shape = observation_shape
        self.num_actions = int(num_actions)
        self.precision = precision
        self.validate_inputs = validate_inputs
        self.conv1 = nn.Conv2d(4, 32, kernel_size=8, stride=4)
        self.conv2 = nn.Conv2d(32, 64, kernel_size=4, stride=2)
        self.conv3 = nn.Conv2d(64, 64, kernel_size=3, stride=1)
        self.fc = nn.Linear(3136, 512)
        core_size = 512 + 1 + self.num_actions
        self.use_lstm = use_lstm
        if use_lstm:
            self.rnn_layer = nn.LSTM(core_size, core_size, num_layers=2)
        self.policy = nn.Linear(core_size, self.num_actions)
        self.baseline = nn.Linear(core_size, 1)
        self._contexts = _EncoderContexts(PRECISIONS[precision])

    def initial_hidden_state(self, batch_size: int):
        """() without the LSTM, else (h0, c0): zeros [num_layers, batch_size, hidden_size] on the CPU (atari_model.py:61-75)"""
        if not self.use_lstm:
            return tuple()
        return tuple(torch.zeros(self.rnn_layer.num_layers, batch_size, self.rnn_layer.hidden_size) for _ in range(2))

    def _encoder_weights(self):
        return [self.conv1.weight, self.conv1.bias, self.conv2.weight, self.conv2.bias, self.conv3.weight, self.conv3.bias,
                self.fc.weight, self.fc.bias]

    def encode(self, obs, reward, action):
        """core f32 [T*B, 513+A] = [relu(fc(...conv1(obs / 255))), clamp(reward, -1, 1), one_hot(action)] for obs u8 [T,B,4,84,84],
        reward f32 [T,B] and action i64 [T,B] on the module's CUDA device; differentiable in the conv / fc parameters."""
        weights = self._encoder_weights()
        for name, t in (('obs', obs), ('reward', reward), ('action', action)):
            if not isinstance(t, torch.Tensor) or not t.is_cuda:
                raise ValueError(f"inputs['{name}'] must be a CUDA tensor: AtariNet has no CPU path (CPU actors use ActorNet)")
        dev = weights[0].device
        if not dev.type == 'cuda':
            raise ValueError('AtariNet has no CPU path: move the module to a CUDA device (.cuda() / .to(device))')
        if any(t.device != dev for t in (obs, reward, action)):
            raise ValueError(f'inputs must be on the parameters\' device {dev}')
        if any(w.dtype != torch.float32 for w in weights):
            raise ValueError('the conv / fc parameters must be float32')
        if obs.dtype != torch.uint8 or obs.dim() != 5 or tuple(obs.shape[2:]) != (4, 84, 84):
            raise ValueError(f"inputs['obs'] must be uint8 [T, B, 4, 84, 84], got {obs.dtype} {tuple(obs.shape)}")
        T, B = obs.shape[:2]
        if not 1 <= T * B <= MAX_FRAMES:
            raise ValueError(f'T*B = {T * B} frames: must be in [1, {MAX_FRAMES}]')
        if reward.dtype != torch.float32 or tuple(reward.shape) != (T, B):
            raise ValueError(f"inputs['reward'] must be float32 [{T}, {B}], got {reward.dtype} {tuple(reward.shape)}")
        if action.dtype != torch.int64 or tuple(action.shape) != (T, B):
            raise ValueError(f"inputs['action'] must be int64 [{T}, {B}], got {action.dtype} {tuple(action.shape)}")
        if reward.requires_grad:
            raise ValueError("inputs['reward'] requires grad, but the encoder gives the reward column no gradient")
        if self.validate_inputs and bool(((action < 0) | (action >= self.num_actions)).any()):
            raise RuntimeError(f'Class values must be smaller than num_classes ({self.num_actions}) and non-negative: '
                               f"inputs['action'] has min {int(action.min())}, max {int(action.max())}")
        obs, reward, action = obs.contiguous(), reward.contiguous(), action.contiguous()
        weights = [w.contiguous() for w in weights]
        handle, prec = self._contexts.get(dev), self.precision
        if torch.is_grad_enabled() and any(w.requires_grad for w in weights):
            return _EncoderCore.apply(handle, prec, self.num_actions, obs, reward, action, *weights)
        return _encoder_forward(handle, prec, self.num_actions, obs, reward, action, weights)[0]

    def _check_lstm_inputs(self, done, rnn_state, T, B):
        H = self.rnn_layer.hidden_size
        if not isinstance(done, torch.Tensor) or done.dtype != torch.bool or tuple(done.shape) != (T, B):
            raise ValueError(f"inputs['done'] must be bool [{T}, {B}], got "
                             f"{(done.dtype, tuple(done.shape)) if isinstance(done, torch.Tensor) else type(done).__name__}")
        if not isinstance(rnn_state, (tuple, list)) or len(rnn_state) != 2:
            raise ValueError('rnn_state must be the 2-tuple (h, c) of float32 [2, B, 513 + A] tensors (initial_hidden_state(B) on the '
                             'module\'s device)')
        dev = self.conv1.weight.device
        for name, s in zip(('h', 'c'), rnn_state):
            if not isinstance(s, torch.Tensor) or s.dtype != torch.float32 or tuple(s.shape) != (2, B, H):
                raise ValueError(f'rnn_state {name} must be float32 [2, {B}, {H}], got '
                                 f'{(s.dtype, tuple(s.shape)) if isinstance(s, torch.Tensor) else type(s).__name__}')
        for name, s in zip(('h', 'c'), rnn_state):
            if not s.is_cuda or s.device != dev:
                raise ValueError(f"rnn_state {name} must be a CUDA tensor on the module's device {dev}, got {s.device}")
        if not done.is_cuda or done.device != dev:
            raise ValueError(f"inputs['done'] must be a CUDA tensor on the module's device {dev}, got {done.device}")

    def _lstm_core(self, core, done, rnn_state):
        """(out f32 [T,B,H], (hT, cT) [2,B,H]) of rnn_layer over core f32 [T,B,H] from rnn_state = (h0, c0), the state zeroed where
        done [T,B] before a step (atari_model.py:109-120), on the sm_90a LSTM kernels; differentiable in core, h0, c0 and rnn_layer's
        tensors.  forward checks the inputs first (_check_lstm_inputs)."""
        weights = [getattr(self.rnn_layer, n).contiguous() for n in LSTM_WEIGHTS]
        if any(w.dtype != torch.float32 for w in weights):
            raise ValueError('the rnn_layer parameters must be float32')
        h0, c0 = (s.contiguous() for s in rnn_state)
        core, done = core.contiguous(), done.contiguous().view(torch.uint8)
        if torch.is_grad_enabled() and any(t.requires_grad for t in [core, h0, c0, *weights]):
            out, hT, cT = _LstmCore.apply(self.num_actions, core, done, h0, c0, *weights)
        else:
            out, hT, cT, _ = _lstm_forward(self.num_actions, core, done, h0, c0, weights)
        return out, (hT, cT)

    def forward(self, inputs, rnn_state=()):
        """(dict(policy_logits [T,B,A], baseline [T,B], action [T,B]), rnn_state), as atari_model.py:77-143"""
        T, B = inputs['obs'].shape[:2]
        lstm_kernels = self.use_lstm and self.precision == 'bf16'      # the LSTM kernels have bf16 operands only
        if lstm_kernels:
            self._check_lstm_inputs(inputs.get('done'), rnn_state, T, B)
        core = self.encode(inputs['obs'], inputs['reward'], inputs['action'])
        if lstm_kernels:
            core, rnn_state = self._lstm_core(core.view(T, B, -1), inputs['done'], rnn_state)
            core = core.flatten(0, 1)
        elif self.use_lstm:
            steps = core.view(T, B, -1).unbind()
            notdone = (~inputs['done']).float().unbind()
            outs = []
            for x, nd in zip(steps, notdone):          # the state is zeroed where an episode ended before the step
                rnn_state = tuple(nd.view(1, -1, 1) * s for s in rnn_state)
                y, rnn_state = self.rnn_layer(x.unsqueeze(0), rnn_state)
                outs.append(y)
            core = torch.cat(outs).flatten(0, 1)
        else:
            rnn_state = tuple()
        policy_logits = self.policy(core)
        baseline = self.baseline(core)
        if self.training:
            action = torch.multinomial(F.softmax(policy_logits, dim=1), num_samples=1)
        else:
            action = torch.argmax(policy_logits, dim=1)
        return (dict(policy_logits=policy_logits.view(T, B, self.num_actions), baseline=baseline.view(T, B), action=action.view(T, B)),
                rnn_state)


class SyntheticAtariEnv:
    """random 84x84x4 uint8 frames, reward in {-1,0,1}, episodes of ~200 steps; record schema of TorchEnvWrapper"""

    def __init__(self, obs_shape=(4, 84, 84), num_actions=6, seed=0, episode_len=200):
        self.obs_shape, self.num_actions, self.episode_len = obs_shape, num_actions, episode_len
        self.g = torch.Generator().manual_seed(seed + 12345 + torch.initial_seed() % 1000)
        self.episode_return = torch.zeros(1, 1)
        self.episode_step = torch.zeros(1, 1, dtype=torch.int32)

    def _frame(self):
        return torch.randint(0, 256, (1, 1, *self.obs_shape), dtype=torch.uint8, generator=self.g)

    def reset(self):
        self.episode_return.zero_()
        self.episode_step.zero_()
        return dict(obs=self._frame(), reward=torch.zeros(1, 1), done=torch.ones(1, 1, dtype=torch.bool),
                    episode_return=self.episode_return.clone(), episode_step=self.episode_step.clone(),
                    action=torch.zeros(1, 1, dtype=torch.int64))

    def step(self, action):
        r = float(torch.randint(-1, 2, (1,), generator=self.g))
        self.episode_step += 1
        self.episode_return += r
        done = bool(self.episode_step.item() >= self.episode_len)
        out = dict(obs=self._frame(), reward=torch.full((1, 1), r), done=torch.tensor([[done]]),
                   episode_return=self.episode_return.clone(), episode_step=self.episode_step.clone(),
                   action=action.view(1, 1).to(torch.int64))
        if done:
            self.episode_return.zero_()
            self.episode_step.zero_()
        return out
