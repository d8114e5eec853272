"""B200R2D2Learner -- the R2D2 learner step (Kapturowski et al. 2019, "Recurrent Experience Replay in Distributed Reinforcement
Learning") on the sm_90a encoder and LSTM core, with B200ApexLearner's interface.

R2D2 is Ape-X with a recurrent Q network trained on stored sequences.  ``R2D2QNet`` is that network in torch (CPU-runnable):
AtariNet(use_lstm=True)'s conv1..3, fc and 2-layer ``rnn_layer`` over the row ``[relu(fc(x)), clamp(r_{t-1}, -1, 1), one_hot(a_{t-1})]``
(width H = 513 + A, the state multiplied by 1 - done_t before step t), then ``q = Linear(H, A)`` or the dueling head ``value =
Linear(H, 1)``, ``advantage = Linear(H, A)``, Q = V + Adv - mean(Adv).  Its state_dict names are AtariNet's, ``rnn_layer.*`` and
AtariQNet's head names, so checkpoints move between it and the learner.

One ``learn`` call is one update on B stored sequences of L = burn_in + T + n_step rows (IMPALA's row schema, time-major): the burn-in
rows run from the stored state without gradient, the T trained rows get the value-rescaled n-step double-Q targets, and each sequence's
priority eta max|delta| + (1 - eta) mean|delta| + eps goes straight into a ``GpuPrioritizedSampler`` -- all in libscalerl_b200.so
(srl_r2d2_learner_*), captured as one CUDA graph per input-address set.  The caller stores the sequences and their initial states.
"""
from __future__ import annotations

import ctypes as C
import math
import random
from collections import OrderedDict
from dataclasses import dataclass
from typing import ClassVar, Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from .. import _lib
from .apex.learner import MAX_FRAMES, B200ApexLearner, check_net_args
from .base import BaseAgent

LSTM_NAMES = tuple(f'rnn_layer.{w}_l{l}' for l in (0, 1) for w in ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh'))


def r2d2_param_shapes(num_actions: int, dueling: bool = True) -> 'OrderedDict[str, tuple]':
    """the named shapes of R2D2QNet's parameters in state_dict order (srl_r2d2_param_layout order)"""
    A, H = int(num_actions), 513 + int(num_actions)
    enc = [('conv1.weight', (32, 4, 8, 8)), ('conv1.bias', (32,)), ('conv2.weight', (64, 32, 4, 4)), ('conv2.bias', (64,)),
           ('conv3.weight', (64, 64, 3, 3)), ('conv3.bias', (64,)), ('fc.weight', (512, 3136)), ('fc.bias', (512,))]
    lstm = [(n, (4 * H, H) if 'weight' in n else (4 * H,)) for n in LSTM_NAMES]
    head = [('value.weight', (1, H)), ('value.bias', (1,)), ('advantage.weight', (A, H)), ('advantage.bias', (A,))] if dueling else \
        [('q.weight', (A, H)), ('q.bias', (A,))]
    return OrderedDict(enc + lstm + head)


class R2D2QNet(nn.Module):
    """The recurrent Q network: AtariNet(use_lstm=True)'s encoder and LSTM core, then q = Linear(H, A) or (``dueling``) value =
    Linear(H, 1) and advantage = Linear(H, A) combined as Q = V + Adv - mean_a Adv.  ``forward(frame, last_action, reward, done,
    state)``: frame u8 [T, B, 4, 84, 84], last_action int64 [T, B], reward float32 [T, B], done bool [T, B], state (h, c) float32
    [2, B, H] -> (Q [T, B, A], (hT, cT)).  Initialised by torch's default layer init."""

    def __init__(self, num_actions: int, dueling: bool = True):
        super().__init__()
        check_net_args(num_actions, 0.0)
        self.num_actions, self.dueling = int(num_actions), bool(dueling)
        H = 513 + self.num_actions
        self.conv1 = nn.Conv2d(4, 32, kernel_size=8, stride=4)
        self.conv2 = nn.Conv2d(32, 64, kernel_size=4, stride=2)
        self.conv3 = nn.Conv2d(64, 64, kernel_size=3, stride=1)
        self.fc = nn.Linear(3136, 512)
        self.rnn_layer = nn.LSTM(H, H, num_layers=2)
        if self.dueling:
            self.value = nn.Linear(H, 1)
            self.advantage = nn.Linear(H, self.num_actions)
        else:
            self.q = nn.Linear(H, self.num_actions)

    def initial_state(self, batch_size: int):
        H = 513 + self.num_actions
        return tuple(torch.zeros(2, batch_size, H) for _ in range(2))

    def forward(self, frame, last_action, reward, done, state):
        T, B = frame.shape[:2]
        x = frame.reshape(T * B, 4, 84, 84).float() / 255.0
        x = F.relu(self.conv1(x))
        x = F.relu(self.conv2(x))
        x = F.relu(self.conv3(x))
        x = F.relu(self.fc(x.reshape(T * B, -1)))
        core = torch.cat([x, reward.reshape(T * B, 1).float().clamp(-1, 1),
                          F.one_hot(last_action.reshape(T * B).long(), self.num_actions).float()], dim=1).view(T, B, -1)
        notdone = (~done.bool()).float()
        outs = []
        for t in range(T):
            state = tuple(notdone[t].view(1, B, 1) * s for s in state)
            y, state = self.rnn_layer(core[t:t + 1], state)
            outs.append(y)
        out = torch.cat(outs)
        if self.dueling:
            v, adv = self.value(out), self.advantage(out)
            return v + adv - adv.mean(dim=-1, keepdim=True), state
        return self.q(out), state


def default_r2d2_state_dict(num_actions: int, dueling: bool = True, seed: int = 0) -> 'OrderedDict[str, torch.Tensor]':
    """R2D2QNet's initial weights under ``torch.manual_seed(seed)``, drawn without disturbing the global RNG"""
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        net = R2D2QNet(num_actions, dueling)
    return OrderedDict((k, v.detach().clone()) for k, v in net.state_dict().items())


@dataclass
class R2D2HParams:
    """The learner's settings, with the defaults of the R2D2 paper (Kapturowski et al. 2019, Table 2): 64 sequences of 40 burn-in and
    80 trained rows, 5-step double-Q targets at gamma 0.997 with value rescaling (eps 1e-3), priority exponent eta 0.9, Adam at lr
    1e-4 and eps 1e-3, the dueling head, a target copy every 2500 updates.  The distributional and noisy heads and the fp32_split
    operand mode are not supported on the recurrent network (validate() refuses them)."""
    batch_size: int = 64
    num_actions: int = 18
    burn_in: int = 40
    seq_len: int = 80                   # T, the trained rows per sequence
    n_step: int = 5
    gamma: float = 0.997                # per step
    learning_rate: float = 1e-4
    adam_beta1: float = 0.9
    adam_beta2: float = 0.999
    adam_eps: float = 1e-3
    max_grad_norm: Optional[float] = None
    priority_eta: float = 0.9
    priority_eps: float = 1e-6          # keeps every priority > 0, as the sampler's trees need
    value_rescaling: bool = True
    rescale_eps: float = 1e-3
    dueling: bool = True
    target_update_frequency: int = 2500
    soft_update_tau: float = 1.0
    precision: str = 'bf16'
    categorical_dqn: bool = False
    quantile_dqn: bool = False
    distributional_dueling: bool = False
    noisy_dqn: bool = False
    optimizer: ClassVar[str] = 'adam'            # read by learner.py's optimizer-state converters
    lr_schedule: ClassVar[str] = 'constant'

    @property
    def seq_rows(self) -> int:
        """L = burn_in + seq_len + n_step rows per stored sequence"""
        return self.burn_in + self.seq_len + self.n_step

    def validate(self) -> None:
        for name in ('categorical_dqn', 'quantile_dqn', 'distributional_dueling', 'noisy_dqn'):
            if getattr(self, name):
                raise ValueError(f'{name} is not supported by the R2D2 learner (the recurrent network has the plain and dueling heads only)')
        if self.precision != 'bf16':
            raise ValueError(f"precision must be 'bf16' (the LSTM core has bf16 operands only), got {self.precision!r}")
        check_net_args(self.num_actions, 0.0)
        for name, lo in (('batch_size', 1), ('burn_in', 0), ('seq_len', 1), ('n_step', 1), ('target_update_frequency', 1)):
            v = getattr(self, name)
            if isinstance(v, bool) or not isinstance(v, int) or v < lo:
                raise ValueError(f'{name} must be an int >= {lo}, got {v!r}')
        if self.seq_rows * self.batch_size > MAX_FRAMES:
            raise ValueError(f'(burn_in + seq_len + n_step) * batch_size = {self.seq_rows * self.batch_size} frames: must be <= {MAX_FRAMES}')
        if not (math.isfinite(self.gamma) and 0.0 <= self.gamma <= 1.0):
            raise ValueError(f'gamma must be in [0, 1], got {self.gamma}')
        if not (math.isfinite(self.learning_rate) and self.learning_rate > 0.0):
            raise ValueError(f'learning_rate must be finite and > 0, got {self.learning_rate}')
        if not (0.0 <= self.adam_beta1 < 1.0 and 0.0 <= self.adam_beta2 < 1.0):
            raise ValueError(f'Adam betas must be in [0, 1), got ({self.adam_beta1}, {self.adam_beta2})')
        if not (math.isfinite(self.adam_eps) and self.adam_eps >= 0.0):
            raise ValueError(f'adam_eps must be finite and >= 0, got {self.adam_eps}')
        if self.max_grad_norm is not None and not self.max_grad_norm > 0.0:
            raise ValueError(f'max_grad_norm must be None or > 0, got {self.max_grad_norm}')
        if not 0.0 <= self.priority_eta <= 1.0:
            raise ValueError(f'priority_eta must be in [0, 1], got {self.priority_eta}')
        if not (math.isfinite(self.priority_eps) and self.priority_eps >= 0.0):
            raise ValueError(f'priority_eps must be finite and >= 0, got {self.priority_eps}')
        if self.value_rescaling and not (math.isfinite(self.rescale_eps) and self.rescale_eps > 0.0):
            raise ValueError(f'rescale_eps must be finite and > 0, got {self.rescale_eps}')
        if not 0.0 <= self.soft_update_tau <= 1.0:
            raise ValueError(f'soft_update_tau must be in [0, 1], got {self.soft_update_tau}')

    def to_c(self) -> _lib.SrlR2d2Config:
        self.validate()
        c = _lib.SrlR2d2Config()
        c.B, c.A, c.burn_in, c.T, c.n_step = self.batch_size, self.num_actions, self.burn_in, self.seq_len, self.n_step
        c.gamma = self.gamma
        c.dueling, c.value_rescaling = int(self.dueling), int(self.value_rescaling)
        c.rescale_eps, c.priority_eta, c.priority_eps = self.rescale_eps, self.priority_eta, self.priority_eps
        c.max_grad_norm = math.inf if self.max_grad_norm is None else self.max_grad_norm
        c.learning_rate, c.adam_beta1, c.adam_beta2, c.adam_eps = self.learning_rate, self.adam_beta1, self.adam_beta2, self.adam_eps
        return c


class B200R2D2Learner(B200ApexLearner):
    """The R2D2 learner on one GPU.  ``learn(sequences, weights, idxs, sampler)`` runs one update: ``sequences`` is a mapping with
    frame u8 [L, B, 4, 84, 84], last_action int64 [L, B], reward float32 [L, B], done bool / uint8 [L, B] and state = (h0, c0) float32
    [2, B, H] (the stored recurrent state before row 0), all contiguous CUDA tensors; importance weights float32 [B] (None = 1) and
    the sampled indices int64 [B] of ``sampler`` (a GpuPrioritizedSampler over stored sequences).  Row t holds s_t, the action and
    reward that led to it, and done_t; the transition of row t is (s_t, last_action[t+1], reward[t+1], done[t+1]).  The parameter,
    optimizer-state, checkpoint, target-cadence and graph-capture surface is B200ApexLearner's (one graph per input-address set:
    first call eager, second captures, later calls replay), on R2D2QNet's names and torch.optim.Adam(R2D2QNet(...).parameters())'s
    state layout."""

    def __init__(self, hp: R2D2HParams, device=None, init_state_dict: Optional[Dict[str, torch.Tensor]] = None, seed: int = 0,
                 use_graph: bool = True):
        if not torch.cuda.is_available():
            raise RuntimeError('B200R2D2Learner needs a CUDA device: scalerl_b200 has no CPU fallback')
        BaseAgent.__init__(self, hp)
        cfg = hp.to_c()
        self.hp = hp
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self._L = _lib.lib()
        self.shapes = r2d2_param_shapes(hp.num_actions, hp.dueling)
        self.names = tuple(self.shapes)
        self.hidden = 513 + hp.num_actions
        with torch.cuda.device(self.device):
            total, self._off, self._cnt = _lib.r2d2_param_layout(hp.num_actions, hp.dueling)
            z = lambda: torch.zeros(total, dtype=torch.float32, device=self.device)
            self.flat_params, self.flat_grads, self.exp_avg, self.exp_avg_sq, self.flat_target = z(), z(), z(), z(), z()
            self.params = self._views(self.flat_params)
            self.grads = self._views(self.flat_grads)
            self.target_params = self._views(self.flat_target)
            self._cfg = cfg
            h = C.c_void_p()
            _lib.check(self._L.srl_r2d2_learner_create(C.addressof(cfg), self.flat_params.data_ptr(), self.flat_grads.data_ptr(),
                                                       self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(), self.flat_target.data_ptr(),
                                                       C.byref(h)), 'srl_r2d2_learner_create')
            self._h = h
            self._stats = torch.zeros(4, device=self.device)      # {loss, gradient norm, clip coefficient, pad}
        sd = default_r2d2_state_dict(hp.num_actions, hp.dueling, seed) if init_state_dict is None else init_state_dict
        self.load_state_dict(sd)
        self.load_state_dict(sd, target=True)
        self.use_graph = use_graph
        self._graphs = {}
        self._seen = set()
        self._opt_steps = 0
        self.learner_update_step = 0
        self.target_model_update_step = 0

    # ------------------------------------------------------------------ counters and target
    def set_step(self, step: int) -> None:
        """Adam's step count and the target cadence's counters for a resumed run (B200ApexLearner.set_step's semantics)"""
        _lib.check(self._L.srl_r2d2_learner_set_step(self._h, int(step), self._stream()), 'srl_r2d2_learner_set_step')
        self._opt_steps = int(step)
        self.learner_update_step = int(step)
        self.target_model_update_step = -(-int(step) // self.hp.target_update_frequency)

    def update_target(self, tau: float) -> None:
        """target <- tau * online + (1 - tau) * target on the current stream"""
        _lib.check(self._L.srl_r2d2_learner_update_target(self._h, float(tau), self._stream()), 'srl_r2d2_learner_update_target')

    # ------------------------------------------------------------------ acting
    def initial_state(self, n: int):
        """the zero recurrent state (h, c), float32 [2, n, H] each, on the learner's device"""
        return tuple(torch.zeros(2, n, self.hidden, device=self.device) for _ in range(2))

    @torch.no_grad()
    def q_values(self, frame, last_action, reward, done, state):
        """Q of the online network over T1 rows of N columns from ``state``: frame u8 [T1, N, 4, 84, 84], last_action int64, reward
        float32 and done bool [T1, N] -> (Q float32 [T1, N, A], the state after the last row); one acting step may drop the T1 axis
        (frame [N, 4, 84, 84], the columns [N] -> Q [N, A]).  Runs on its own encoder context and buffers."""
        step = torch.as_tensor(frame).dim() == 4
        fix = lambda t, dt: (torch.as_tensor(t).unsqueeze(0) if step else torch.as_tensor(t)).to(self.device, dt).contiguous()
        frame, last_action, reward = fix(frame, torch.uint8), fix(last_action, torch.int64), fix(reward, torch.float32)
        done = fix(done, torch.bool).view(torch.uint8)
        if frame.dim() != 5 or tuple(frame.shape[2:]) != (4, 84, 84):
            raise ValueError(f'frame must be uint8 [T1, N, 4, 84, 84], got {tuple(frame.shape)}')
        T1, N = frame.shape[:2]
        for name, t in (('last_action', last_action), ('reward', reward), ('done', done)):
            if tuple(t.shape) != (T1, N):
                raise ValueError(f'{name} must be [{T1}, {N}], got {tuple(t.shape)}')
        h0, c0 = (s.to(self.device, torch.float32).contiguous() for s in state)
        for s in (h0, c0):
            if tuple(s.shape) != (2, N, self.hidden):
                raise ValueError(f'state must be two float32 [2, {N}, {self.hidden}] tensors, got {tuple(s.shape)}')
        q = torch.empty(T1, N, self.hp.num_actions, device=self.device)
        hT, cT = torch.empty_like(h0), torch.empty_like(c0)
        _lib.check(self._L.srl_r2d2_learner_q_values(self._h, frame.data_ptr(), last_action.data_ptr(), reward.data_ptr(), done.data_ptr(),
                                                     T1, N, h0.data_ptr(), c0.data_ptr(), q.data_ptr(), hT.data_ptr(), cT.data_ptr(),
                                                     self._stream()), 'srl_r2d2_learner_q_values')
        return (q[0] if step else q), (hT, cT)

    def predict(self, frame, last_action, reward, done, state):
        """(greedy actions int64 (argmax_a Q, the first maximal index), the next state)"""
        q, state = self.q_values(frame, last_action, reward, done, state)
        return torch.argmax(q, dim=-1), state

    def get_action(self, frame, last_action, reward, done, state, eps: float):
        """epsilon-greedy at the caller's epsilon (B200ApexLearner.get_action's draw) -> (actions, the next state); the state always
        advances through the network"""
        actions, state = self.predict(frame, last_action, reward, done, state)
        if random.random() < eps:
            a = np.argmax(np.random.uniform(0, 1, tuple(actions.shape) + (self.hp.num_actions,)), axis=-1)
            actions = torch.from_numpy(a).to(self.device)
        return actions, state

    # ------------------------------------------------------------------ learning
    def _sequence_inputs(self, sequences, weights, idxs, sampler):
        try:
            frame, last_action, reward, done, state = (sequences[k] for k in ('frame', 'last_action', 'reward', 'done', 'state'))
        except (KeyError, TypeError):
            raise ValueError("sequences must be a mapping with 'frame', 'last_action', 'reward', 'done' and 'state' = (h0, c0)") from None
        L, B, H = self.hp.seq_rows, self.hp.batch_size, self.hidden
        self._check(frame, 'frame', (L, B, 4, 84, 84), (torch.uint8,))
        self._check(last_action, 'last_action', (L, B), (torch.int64,))
        self._check(reward, 'reward', (L, B), (torch.float32,))
        self._check(done, 'done', (L, B), (torch.bool, torch.uint8))
        if not isinstance(state, (tuple, list)) or len(state) != 2:
            raise ValueError('state must be the pair (h0, c0)')
        self._check(state[0], 'h0', (2, B, H), (torch.float32,))
        self._check(state[1], 'c0', (2, B, H), (torch.float32,))
        if weights is not None:
            self._check(weights, 'weights', (B,), (torch.float32,))
        if (idxs is None) != (sampler is None):
            raise ValueError('idxs and sampler go together: pass both or neither')
        if idxs is not None:
            self._check(idxs, 'idxs', (B,), (torch.int64,))
        return frame, last_action, reward, done.view(torch.uint8), state[0], state[1], weights, idxs, sampler

    def _enqueue_sequences(self, frame, last_action, reward, done, h0, c0, weights, idxs, sampler):
        _lib.check(self._L.srl_r2d2_learner_step(
            self._h, frame.data_ptr(), last_action.data_ptr(), reward.data_ptr(), done.data_ptr(), h0.data_ptr(), c0.data_ptr(),
            weights.data_ptr() if weights is not None else None, idxs.data_ptr() if idxs is not None else None,
            sampler._h if sampler is not None else None, self._stats.data_ptr(), self._stream()), 'srl_r2d2_learner_step')

    @torch.no_grad()
    def learn(self, sequences, weights: Optional[torch.Tensor] = None, idxs: Optional[torch.Tensor] = None, sampler=None,
              sync_stats: bool = True, use_graph: Optional[bool] = None) -> Dict[str, float]:
        """one update -> {'loss': float} ((1 / (B T)) sum_b w_b sum_t delta^2), or {} with nothing synchronised"""
        args = self._sequence_inputs(sequences, weights, idxs, sampler)
        key = tuple(a.data_ptr() if isinstance(a, torch.Tensor) else (a._h.value if a is not None else None) for a in args)
        self._run(key, lambda: self._enqueue_sequences(*args), use_graph)
        return self._finish_update(sync_stats)

    def learn_from(self, memory, beta: float = 0.4, sync_stats: bool = True, use_graph: Optional[bool] = None):
        raise ValueError('B200R2D2Learner has no sequence replay memory: sample stored sequences with a GpuPrioritizedSampler and call learn()')

    def debug_buffer(self, name: str) -> torch.Tensor:
        """copy of one of the step's device buffers (tests only; names: srl_r2d2_learner_debug_buffer), flat"""
        p, n = C.c_void_p(), C.c_int64()
        _lib.check(self._L.srl_r2d2_learner_debug_buffer(self._h, name.encode(), C.byref(p), C.byref(n)), 'debug_buffer')
        dt = {'priorities': torch.float64, 'step': torch.int32}.get(name, torch.float32)
        out = torch.empty(n.value, dtype=dt, device=self.device)
        _lib.check(self._L.srl_memcpy_d2d(out.data_ptr(), p.value, n.value * out.element_size(), self._stream()), 'memcpy_d2d')
        torch.cuda.current_stream(self.device).synchronize()
        return out

    def close(self):
        if getattr(self, '_h', None) is not None:
            self._L.srl_r2d2_learner_destroy(self._h)
            self._h = None
