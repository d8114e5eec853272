"""GpuPrioritizedReplayBuffer -- the reference's PrioritizedReplayBuffer (scalerl/data/replay_buffer.py:132-381) with its storage,
n-step folding, sampling and gather on the GPU (srl_replay_*, csrc/replay.cu).  Same constructor arguments and method names:
``save_to_memory``, ``sample``, ``update_priorities``, ``__len__``, ``size``.

Transitions live in a ring of ``memory_size`` slots on the device: state / next_state uint8 [M, 4, 84, 84], action int64 [M],
reward float32 [M], done uint8 [M] (56,461 bytes per transition: M = 100k needs 5.65 GB).  Ring slot i is leaf i of the memory's
sampler trees (``sampler``, a GpuPrioritizedSampler over them), and the E envs of one vector step enter at slots ptr .. ptr + E - 1
(mod M) in env order, as the reference's ``_add`` does.  With ``n_step > 1`` each env keeps a window of its last n raw steps, folded
as ``_get_n_step_info`` folds it (replay_buffer.py:230-273): state and action of the oldest step, reward r0 + r1 * g1 + r2 * g2 ...
in float32 with g_k = float32(gamma ** k) and every product and sum rounded on its own (numpy's float32 arithmetic, bit for bit),
stopping at the first done, whose step gives next_state and done.

Deviations from the reference:
  * fields keep their stored dtypes, with shape [B] rather than [B, 1]: the reference converts every field to float32
    (replay_buffer.py:66-68), the learner reads uint8 frames.  Rewards are stored as float32.
  * ``save_to_memory`` returns nothing; the reference returns the 1-step transition for OffPolicyTrainer's twin-buffer pattern.
  * the ring index is the tree index at every fill level.  The reference's deque index stops matching its tree index once the
    memory is full (replay_buffer.py:41-44 vs :319-323); oracle/replay_oracle.py documents the mapping.
Everything runs on the current stream and is stream-ordered; adds are host calls and may come between replays of a graph that samples.

GpuFrameReplayBuffer (srl_frame_replay_*, csrc/frame_replay.cu) keeps the same transitions, trees and outputs with each 84x84 frame
stored once, in a FIFO pool of ``frame_capacity`` frames that the ring's slots reference by handle.
"""
import ctypes as C
import math

import numpy as np
import torch

from .. import _lib
from .per_sampler import GpuPrioritizedSampler

OBS_SHAPE = (4, 84, 84)
MAX_ENVS = 65536                # num_envs limit of srl_replay_create (MAX_FRAMES in csrc/kernels.h)
MAX_N_STEP = 32                 # REPLAY_MAX_NSTEP in csrc/replay.cu


def _int_in(name, v, lo, hi):
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not lo <= int(v) <= hi:
        raise ValueError(f'{name} must be an int in [{lo}, {hi}], got {v!r}')
    return int(v)


class _GpuReplay:
    """what the two device memories share: the argument checks, the field checks of ``save_to_memory``, the beta handling, sampling,
    gathering and the trees.  ``_abi`` names the C-ABI family (srl_replay, srl_frame_replay) whose entry points take the same arguments."""
    _abi = None

    def __init__(self, memory_size: int, num_envs: int, alpha: float = 0.6, n_step: int = 1, gamma: float = 0.99, device=None):
        self.memory_size = _int_in('memory_size', memory_size, 2, 1 << 30)
        self.num_envs = _int_in('num_envs', num_envs, 1, min(MAX_ENVS, self.memory_size))
        self.n_step = _int_in('n_step', n_step, 1, MAX_N_STEP)
        self.gamma, self.alpha = float(gamma), float(alpha)
        if not math.isfinite(self.gamma):
            raise ValueError(f'gamma must be finite, got {gamma}')
        if not math.isfinite(self.alpha):
            raise ValueError(f'alpha must be finite, got {alpha}')
        self._check_extra()
        if not torch.cuda.is_available():
            raise RuntimeError(f'{type(self).__name__} needs a CUDA device (no CPU fallback)')
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self._L = _lib.lib()
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self._fn('create')(self.memory_size, self.num_envs, self.n_step, self.gamma, self.alpha, *self._create_extra(), C.byref(h)),
                       f'{self._abi}_create')
            self._h = h
            self.sampler = GpuPrioritizedSampler._view(C.c_void_p(self._fn('per')(h)), self.memory_size, self.alpha, self.device)
            self._beta = torch.zeros(1, dtype=torch.float64, device=self.device)     # read by the sample kernel when it runs
        self._beta_value = None

    def _check_extra(self):
        """checks of the subclass's own constructor arguments (before any device work)"""

    def _create_extra(self):
        """the subclass's own arguments of <abi>_create, after alpha"""
        return ()

    def _fn(self, name):
        return getattr(self._L, f'{self._abi}_{name}')

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def __len__(self):
        return int(self._fn('size')(self._h))

    def size(self):
        return len(self)

    # ------------------------------------------------------------------ adding
    def _field(self, x, name, shape, kinds, dtype):
        t = torch.as_tensor(x)
        if tuple(t.shape) != shape or not kinds(t.dtype):
            raise ValueError(f'{name}: expected shape {shape} ({dtype}), got {tuple(t.shape)} {t.dtype}')
        if t.is_cuda and t.device != self.device:
            raise ValueError(f'{name} is on {t.device}, the memory on {self.device}')
        return t, dtype

    def save_to_memory(self, state, action, reward, next_state, done, is_vectorised: bool = False, priorities_from=None) -> None:
        """one env step: states uint8 [E, 4, 84, 84], action integer [E], reward floating [E], done bool / uint8 [E] (vectorised), or
        one env's [4, 84, 84] and scalars (``num_envs == 1``).  CUDA tensors of the stored dtypes are read in place; numpy arrays and
        CPU tensors are copied on the current stream.  Once n_step steps are staged, every call adds E n-step transitions at maximum
        priority (replay_buffer.py:197-218, 319-323) or, with ``priorities_from`` (a B200ApexActor on this device with this memory's
        num_envs), at the priorities that actor computes for them: |Q(s)[a] - (R + gamma^n (1 - d) max_a Q(s'))| + its priority_eps
        (apex/worker.py:59-79, apex/memory.py:43-64).  A non-finite priority enters as the plain add's and is counted by the sampler's
        invalid-update counter."""
        if priorities_from is not None:
            from ..algorithms.apex.actor import B200ApexActor
            if not isinstance(priorities_from, B200ApexActor):
                raise ValueError(f'priorities_from must be a B200ApexActor, got {type(priorities_from).__name__}')
            if priorities_from.device != self.device:
                raise ValueError(f'priorities_from is on {priorities_from.device}, the memory on {self.device}')
            if priorities_from.num_envs != self.num_envs:
                raise ValueError(f'priorities_from has num_envs={priorities_from.num_envs}, the memory {self.num_envs}')
        E = self.num_envs
        if is_vectorised:
            lead = (E,)
        elif E != 1:
            raise ValueError(f'save_to_memory without is_vectorised needs num_envs == 1, the memory has {E}')
        else:
            lead = ()
        u8 = lambda d: d == torch.uint8
        s = self._field(state, 'state', lead + OBS_SHAPE, u8, torch.uint8)
        ns = self._field(next_state, 'next_state', lead + OBS_SHAPE, u8, torch.uint8)
        a = self._field(action, 'action', lead, lambda d: not d.is_floating_point and not d.is_complex and d != torch.bool, torch.int64)
        r = self._field(reward, 'reward', lead, lambda d: d.is_floating_point, torch.float32)
        d = self._field(done, 'done', lead, lambda d: d in (torch.bool, torch.uint8), torch.uint8)
        # every field is checked before the first copy: a bad step adds nothing
        s, a, r, ns, d = ((t.view(torch.uint8) if t.dtype == torch.bool else t).to(self.device, dt).contiguous() for t, dt in (s, a, r, ns, d))
        with torch.cuda.device(self.device):
            if priorities_from is None:
                _lib.check(self._fn('add')(self._h, s.data_ptr(), a.data_ptr(), r.data_ptr(), ns.data_ptr(), d.data_ptr(), self._stream()),
                           f'{self._abi}_add')
            else:
                _lib.check(self._fn('add_prioritized')(self._h, priorities_from._h, s.data_ptr(), a.data_ptr(), r.data_ptr(), ns.data_ptr(),
                                                       d.data_ptr(), priorities_from.priority_eps, self._stream()),
                           f'{self._abi}_add_prioritized')

    # ------------------------------------------------------------------ sampling
    def _set_beta(self, beta: float) -> None:
        """the device beta the sample kernel reads: one fill when it changes, so captured graphs replay with the new value"""
        beta = float(beta)
        if not math.isfinite(beta):
            raise ValueError(f'beta must be finite, got {beta}')
        if beta != self._beta_value:
            self._beta.fill_(beta)
            self._beta_value = beta

    def _sample_into(self, uniforms, state, action, reward, next_state, done, idxs, weights) -> None:
        """<abi>_sample into caller-owned device buffers (no checks beyond the library's; nothing synchronised)"""
        _lib.check(self._fn('sample')(self._h, uniforms.data_ptr(), uniforms.numel(), self._beta.data_ptr(), state.data_ptr(),
                                      action.data_ptr(), reward.data_ptr(), next_state.data_ptr(), done.data_ptr(), idxs.data_ptr(),
                                      weights.data_ptr(), self._stream()), f'{self._abi}_sample')

    def _outputs(self, n):
        z = lambda *shape, dtype: torch.empty(*shape, dtype=dtype, device=self.device)
        return (z(n, *OBS_SHAPE, dtype=torch.uint8), z(n, dtype=torch.int64), z(n, dtype=torch.float32), z(n, *OBS_SHAPE, dtype=torch.uint8),
                z(n, dtype=torch.uint8))

    def sample(self, batch_size: int, beta: float = 0.4, uniforms=None):
        """-> (state, action, reward, next_state, done, weights float32 [B], idxs int64 [B]), new device tensors in the stored dtypes
        (replay_buffer.py:325-344).  ``uniforms`` (float64 [B] in [0, 1)) replaces the draw of random.uniform for reproducibility."""
        batch_size = _int_in('batch_size', batch_size, 1, MAX_ENVS)
        if len(self) < 2:
            raise ValueError(f'sample needs at least 2 stored transitions, the memory has {len(self)}')
        if uniforms is None:
            uniforms = torch.rand(batch_size, dtype=torch.float64, device=self.device)
        u = torch.as_tensor(uniforms).to(self.device, torch.float64).contiguous()
        if tuple(u.shape) != (batch_size,):
            raise ValueError(f'uniforms: expected shape ({batch_size},), got {tuple(u.shape)}')
        out = self._outputs(batch_size)
        idxs = torch.empty(batch_size, dtype=torch.int64, device=self.device)
        weights = torch.empty(batch_size, dtype=torch.float32, device=self.device)
        self._set_beta(beta)
        self._sample_into(u, *out, idxs, weights)
        return (*out, weights, idxs)

    def gather(self, idxs):
        """(state, action, reward, next_state, done) of ring slots ``idxs`` (int64 [n]), new device tensors"""
        idxs = torch.as_tensor(idxs).to(self.device, torch.int64).contiguous().reshape(-1)
        out = self._outputs(idxs.numel())
        _lib.check(self._fn('gather')(self._h, idxs.data_ptr(), idxs.numel(), *(t.data_ptr() for t in out), self._stream()),
                   f'{self._abi}_gather')
        return out

    def update_priorities(self, idxs, priorities, validate: bool = True) -> None:
        """replay_buffer.py:346-351 on the memory's trees (GpuPrioritizedSampler.update_priorities)"""
        self.sampler.update_priorities(torch.as_tensor(idxs), torch.as_tensor(priorities), validate=validate)

    def close(self):
        if getattr(self, '_h', None) is not None:
            self.sampler.close()
            self._fn('destroy')(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class GpuPrioritizedReplayBuffer(_GpuReplay):
    """the reference's PrioritizedReplayBuffer on the device, each transition stored as two 4x84x84 u8 stacks (56,461 B).  It makes no
    assumption about how the stacks of a stream relate, so it is the memory for streams whose stacks share no frames."""
    _abi = 'srl_replay'


class GpuFrameReplayBuffer(_GpuReplay):
    """GpuPrioritizedReplayBuffer's transitions, trees, methods and outputs (the same bytes for the same adds) with each 84x84 frame
    stored once.  It only saves memory when the stacks of the stream share frames, as Atari frame stacks do: a continuing episode then
    adds one 7,056-byte frame per env step.

    ``frame_capacity``: 84x84 frames in the pool, at least ``8 * num_envs * (n_step + 1)`` (so the staging window's frames are never
    overwritten); default ``memory_size + memory_size // 8 + 8 * num_envs * (n_step + 4)``, which retires nothing while episodes average
    at least 32 steps.  When new frames overwrite one that a stored transition references, that transition retires first: its priority
    becomes 0 (never sampled, outside the weights' p_min), ``gather`` leaves its output rows as they were, and ``update_priorities``
    skips it without raising.  An add that writes its slot makes it live again; ``len`` counts it throughout."""
    _abi = 'srl_frame_replay'

    def __init__(self, memory_size: int, num_envs: int, alpha: float = 0.6, n_step: int = 1, gamma: float = 0.99, frame_capacity=None,
                 device=None):
        self._frame_capacity_arg = frame_capacity
        super().__init__(memory_size, num_envs, alpha=alpha, n_step=n_step, gamma=gamma, device=device)

    def _check_extra(self):
        E, n, M = self.num_envs, self.n_step, self.memory_size
        fc = self._frame_capacity_arg
        lo = 8 * E * (n + 1)
        self.frame_capacity = M + M // 8 + 8 * E * (n + 4) if fc is None else _int_in('frame_capacity', fc, lo, 1 << 32)

    def _create_extra(self):
        return (self.frame_capacity,)

    def frames_allocated(self) -> int:
        """frames written to the pool since creation.  Synchronises the device (the count is known there)."""
        with torch.cuda.device(self.device):
            return self._counter('frames_allocated')

    def retired(self) -> int:
        """transitions retired since creation (each time one retires).  Synchronises the device (the count is known there)."""
        with torch.cuda.device(self.device):
            return self._counter('retired')

    def _counter(self, name):
        v = int(self._fn(name)(self._h, self._stream()))
        if v < 0:
            raise RuntimeError(f'{self._abi}_{name}: reading the device counter failed')
        return v
