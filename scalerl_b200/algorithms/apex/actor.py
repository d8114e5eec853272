"""B200ApexActor -- the acting side of Ape-X on the GPU: per-env epsilon-greedy actions and the initial priorities of new transitions.

The reference's Ape-X ``Actor`` (scalerl/algorithms/apex/worker.py:14-79) acts with an epsilon of its own on a copy of the learner's
weights and computes each transition's priority before it enters the memory (``compute_prior``, worker.py:59-79;
``PrioritizedReplayBuffer.add(..., prior)``, apex/memory.py:43-64).  Here one actor object serves ``num_envs`` envs, each with its own
epsilon, from a parameter snapshot on the device (srl_apex_actor_*, csrc/apex_actor.cu):

  * ``act(obs)``: the encoder forward and one kernel that picks, per env, a uniform action with probability eps[e], else the first
    argmax of Q.  Its random numbers are Philox keyed by ``seed`` and a device draw counter, so a captured ``act`` draws anew on every
    replay, and ``set_epsilons`` costs one copy, not a recapture.
  * ``GpuPrioritizedReplayBuffer.save_to_memory(..., priorities_from=actor)``: the transitions the add completes enter the trees with
    |Q(s)[a] - (R + gamma^n (1 - d) max_a Q(s'))| + priority_eps, computed with the learner's target and priority arithmetic.
  * ``sync_from(learner)``: one device copy of the learner's online parameters into the snapshot.

``dueling_dqn=True`` gives the actor the dueling head of ``ApexHParams(dueling_dqn=True)``; it syncs from dueling learners only.
``categorical_dqn=True`` (with ``v_min``, ``v_max``, ``num_atoms``) gives it the categorical head of ``ApexHParams(categorical_dqn=True)``:
it acts on the expected Q and prioritises by the learner's KL divergence, and syncs from learners with the same atoms and support only.
``noisy_dqn=True`` gives it the noisy layers of ``ApexHParams(noisy_dqn=True)`` (with any head): every ``act`` draws new noise for the
snapshot before its forward (one draw for all envs, from ``seed`` and a device counter, so a captured ``act`` draws anew on every
replay) and keeps it; ``q_values`` and the prioritized add use the kept draw on the snapshot as it is.  Its default epsilons are 0.
``quantile_dqn=True`` (with ``num_quantiles``, ``quantile_kappa``) gives it the quantile head of ``ApexHParams(quantile_dqn=True)``: it
acts on the quantile means and prioritises by the learner's quantile Huber loss, and syncs from learners with the same setting only.
``distributional_dueling=True`` (with ``categorical_dqn`` or ``quantile_dqn``) gives it the dueling rows of
``ApexHParams(distributional_dueling=True)``: every call composes the snapshot's value and advantage layers into the head rows as the
learner does, so its rows, Q values, actions and priorities are the learner's bits.
"""
from __future__ import annotations

import ctypes as C
import math
from collections import OrderedDict
from functools import cached_property
from typing import Dict, Optional

import numpy as np
import torch

from ... import _lib
from .learner import MAX_FRAMES, QHead, check_net_args, default_q_state_dict, flat_views, load_views

PRECISIONS = {'bf16': 0, 'fp32_split': 1}


def apex_epsilons(num_envs: int, eps: float = 0.4, alpha: float = 7.0) -> np.ndarray:
    """the Ape-X exploration schedule eps_i = eps ** (1 + alpha * i / (N - 1)), i = 0 .. N - 1 (eps alone for N = 1), float64 [N]"""
    if isinstance(num_envs, bool) or not isinstance(num_envs, (int, np.integer)) or num_envs < 1:
        raise ValueError(f'num_envs must be an int >= 1, got {num_envs!r}')
    if num_envs == 1:
        return np.array([eps], dtype=np.float64)
    i = np.arange(num_envs, dtype=np.float64)
    return eps ** (1.0 + alpha * i / (num_envs - 1))


class B200ApexActor:
    """``num_envs`` Ape-X actors on one GPU, acting on a snapshot of a ``B200ApexLearner``'s Q network (``AtariQNet`` names and
    shapes).  ``epsilons``: [num_envs] values in [0, 1] (None: ``apex_epsilons(num_envs)``); ``precision``: the encoder operands, as
    the learner's; ``priority_eps`` (> 0) is added to every priority the actor computes; ``dueling_dqn``, ``categorical_dqn`` (with
    ``v_min``, ``v_max``, ``num_atoms``), ``noisy_dqn`` (with ``noisy_std``, the initial sigma0 of the default weights), ``quantile_dqn``
    (with ``num_quantiles``, ``quantile_kappa``), ``distributional_dueling``: the learner's head (noisy: epsilons None means 0 for every
    env).  Calls run on the current stream and share the actor's buffers: issue them from one
    stream."""
    # the head settings as the constructor stores them; the class values are its defaults
    dueling_dqn, categorical_dqn, v_min, v_max, num_atoms, noisy_dqn = False, False, 0.0, 200.0, 51, False
    quantile_dqn, num_quantiles, quantile_kappa = False, 200, 1.0
    distributional_dueling = False

    def __init__(self, num_envs: int, num_actions: int, epsilons=None, seed: int = 0, precision: str = 'bf16', priority_eps: float = 1e-6,
                 device=None, init_state_dict: Optional[Dict[str, torch.Tensor]] = None, dueling_dqn: bool = False,
                 categorical_dqn: bool = False, v_min: float = 0.0, v_max: float = 200.0, num_atoms: int = 51, noisy_dqn: bool = False,
                 noisy_std: float = 0.5, quantile_dqn: bool = False, num_quantiles: int = 200, quantile_kappa: float = 1.0,
                 distributional_dueling: bool = False):
        if isinstance(num_envs, bool) or not isinstance(num_envs, (int, np.integer)) or not 1 <= num_envs <= MAX_FRAMES:
            raise ValueError(f'num_envs must be an int in [1, {MAX_FRAMES}], got {num_envs!r}')
        check_net_args(num_actions, noisy_std)
        if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)) or not 0 <= seed < 2 ** 64:
            raise ValueError(f'seed must be an int in [0, 2**64), got {seed!r}')
        if precision not in PRECISIONS:
            raise ValueError(f"precision must be 'bf16' or 'fp32_split', got {precision!r}")
        self.head = head = QHead.of(dueling_dqn, categorical_dqn, num_atoms, v_min, v_max, noisy_dqn, quantile_dqn, num_quantiles,
                                    quantile_kappa, distributional_dueling)
        priority_eps = float(priority_eps)
        if not (math.isfinite(priority_eps) and priority_eps > 0.0):
            raise ValueError(f'priority_eps must be finite and > 0 (a zero leaf makes the sampler\'s IS weight infinite), got {priority_eps}')
        self.num_envs, self.num_actions, self.seed, self.precision = int(num_envs), int(num_actions), int(seed), precision
        self.priority_eps, self.dueling_dqn, self.categorical_dqn = priority_eps, dueling_dqn, categorical_dqn
        self.v_min, self.v_max, self.num_atoms = float(v_min), float(v_max), int(num_atoms)
        self.noisy_dqn = noisy_dqn
        self.quantile_dqn, self.num_quantiles, self.quantile_kappa = quantile_dqn, int(num_quantiles), float(quantile_kappa)
        self.distributional_dueling = distributional_dueling
        if epsilons is None:
            epsilons = np.zeros(self.num_envs) if noisy_dqn else apex_epsilons(self.num_envs)
        eps = self._epsilons(epsilons)
        if not torch.cuda.is_available():
            raise RuntimeError('B200ApexActor needs a CUDA device: scalerl_b200 has no CPU fallback')
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self._L = _lib.lib()
        self.shapes = head.shapes(self.num_actions)
        with torch.cuda.device(self.device):
            total, off, cnt = head.layout(self.num_actions)
            self.flat_params = torch.zeros(total, dtype=torch.float32, device=self.device)
            self.params = flat_views(self.flat_params, off, cnt, self.shapes)
            self.epsilons = eps.to(self.device)           # read by the act kernel when it runs
            self._h = _lib.apex_actor_create(self.num_actions, self.num_envs, PRECISIONS[precision], self.seed, self.flat_params.data_ptr(), head)
        sd = default_q_state_dict(self.num_actions, self.seed, head.dueling, head.num_atoms, head.noisy, noisy_std, head.num_quantiles,
                                  head.dist_dueling) if init_state_dict is None else init_state_dict
        self.load_state_dict(sd)
        self.weights_version = 0

    @cached_property
    def head(self) -> QHead:
        """the Q head of the settings above (the constructor stores the one it built)"""
        return QHead.of(self.dueling_dqn, self.categorical_dqn, self.num_atoms, self.v_min, self.v_max, self.noisy_dqn, self.quantile_dqn,
                        self.num_quantiles, self.quantile_kappa, self.distributional_dueling)

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def _epsilons(self, eps) -> torch.Tensor:
        e = torch.as_tensor(eps, dtype=torch.float32).detach().cpu().reshape(-1)
        if e.numel() != self.num_envs:
            raise ValueError(f'epsilons: expected {self.num_envs} values, got {e.numel()}')
        if not bool(((e >= 0) & (e <= 1)).all()):
            raise ValueError('epsilons must all lie in [0, 1]')
        return e

    # ------------------------------------------------------------------ parameters
    def state_dict(self) -> 'OrderedDict[str, torch.Tensor]':
        """AtariQNet-compatible state_dict of the snapshot"""
        return OrderedDict((n, p.detach().clone()) for n, p in self.params.items())

    def load_state_dict(self, sd: Dict[str, torch.Tensor]) -> None:
        load_views(self.params, sd)

    def sync_from(self, learner) -> None:
        """the learner's online parameters -> the snapshot: one device-to-device copy on the current stream (ordered after the
        learner's work on that stream); bumps ``weights_version``"""
        from .learner import B200ApexLearner
        if not isinstance(learner, B200ApexLearner):
            raise ValueError(f'sync_from needs a B200ApexLearner, got {type(learner).__name__}')
        if learner.hp.num_actions != self.num_actions:
            raise ValueError(f'the learner has num_actions={learner.hp.num_actions}, the actor {self.num_actions}')
        if learner.hp.head != self.head:
            raise ValueError(f'the learner has {learner.hp.head}, the actor {self.head}')
        if learner.device != self.device:
            raise ValueError(f'the learner is on {learner.device}, the actor on {self.device}')
        self.flat_params.copy_(learner.flat_params)
        self.weights_version += 1

    def set_epsilons(self, eps) -> None:
        """[num_envs] values in [0, 1]: one copy into the device vector the act kernel reads, so a captured act follows it"""
        e = self._epsilons(eps)
        self.epsilons.copy_(e)

    # ------------------------------------------------------------------ acting
    def _obs(self, obs, n=None) -> torch.Tensor:
        obs = torch.as_tensor(obs)
        if obs.dtype != torch.uint8 or obs.dim() != 4 or tuple(obs.shape[1:]) != (4, 84, 84) or obs.shape[0] < 1 or \
                (n is not None and obs.shape[0] != n):
            want = f'[{n}, 4, 84, 84]' if n is not None else '[N, 4, 84, 84]'
            raise ValueError(f'obs must be uint8 {want}, got {tuple(obs.shape)} {obs.dtype}')
        if obs.is_cuda and obs.device != self.device:
            raise ValueError(f'obs is on {obs.device}, the actor on {self.device}')
        return obs.to(self.device).contiguous()

    @torch.no_grad()
    def act(self, obs) -> torch.Tensor:
        """obs uint8 [num_envs, 4, 84, 84] (a host array or tensor is copied on the current stream) -> int64 [num_envs] on the device:
        per env, a uniform action with probability epsilons[e], else the first argmax of Q(obs[e]) (noisy: under a new noise draw)"""
        obs = self._obs(obs, self.num_envs)
        actions = torch.empty(self.num_envs, dtype=torch.int64, device=self.device)
        _lib.check(self._L.srl_apex_actor_act(self._h, obs.data_ptr(), self.epsilons.data_ptr(), actions.data_ptr(), self._stream()),
                   'srl_apex_actor_act')
        return actions

    @torch.no_grad()
    def q_values(self, obs) -> torch.Tensor:
        """Q(obs) with the snapshot: uint8 [N, 4, 84, 84] -> float32 [N, A] on the device"""
        obs = self._obs(obs)
        q = torch.empty(obs.shape[0], self.num_actions, device=self.device)
        _lib.check(self._L.srl_apex_actor_q_values(self._h, obs.data_ptr(), obs.shape[0], q.data_ptr(), self._stream()),
                   'srl_apex_actor_q_values')
        return q

    def debug_buffer(self, name: str) -> torch.Tensor:
        """copy of one of the actor's device buffers (tests only; names: srl_apex_actor_debug_buffer), flat"""
        p, n = C.c_void_p(), C.c_int64()
        _lib.check(self._L.srl_apex_actor_debug_buffer(self._h, name.encode(), C.byref(p), C.byref(n)), 'debug_buffer')
        out = torch.empty(n.value, dtype=torch.float32, device=self.device)
        _lib.check(self._L.srl_memcpy_d2d(out.data_ptr(), p.value, n.value * 4, self._stream()), 'memcpy_d2d')
        torch.cuda.current_stream(self.device).synchronize()
        return out

    def close(self):
        if getattr(self, '_h', None) is not None:
            self._L.srl_apex_actor_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
