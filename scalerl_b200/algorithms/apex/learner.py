"""B200ApexLearner -- the learner step of Ape-X DQN on the sm_90a encoder, behind the interface of ScaleRL's ``DQNAgent``.

One ``learn`` call is the reference's Ape-X learner update (scalerl/algorithms/apex/worker.py:134-161) with the double-DQN,
clipping and target-update statements of ``DQNAgent.learn`` (scalerl/algorithms/dqn/dqn_agent.py:136-190): the Q values of the
batch, the bootstrapped targets, the importance-weighted squared TD loss, the new priorities written straight into a
``GpuPrioritizedSampler``, ``clip_grad_norm_`` and a ``torch.optim.Adam`` step -- all in libscalerl_b200.so (srl_apex_learner_*),
captured as one CUDA graph.  ``learn_from`` samples and gathers its batch from a ``GpuPrioritizedReplayBuffer`` (device-resident
n-step storage) inside the same graph.  ``B200ApexActor`` (actor.py) acts and computes initial priorities on a copy of its weights.
``AtariQNet`` is the CPU torch Q network with the learner's parameter names and shapes (the actors' copy).

``ApexHParams(dueling_dqn=True)`` replaces the Q head ``q = Linear(512, A)`` by the dueling head of Wang et al. 2016 (eq. 9):
``V = value(h)``, ``Adv = advantage(h)``, ``Q = V + Adv - Adv.mean(1, keepdim=True)``.  Both streams read the encoder's shared 512-unit
fc output (the paper's Atari network gives each stream an fc layer of its own), so the encoder is the plain network's.

``ApexHParams(categorical_dqn=True)`` makes the head categorical (C51, Bellemare et al. 2017): ``q = Linear(512, A * num_atoms)``,
a softmax over each action's ``num_atoms`` logits on the support ``z_k = v_min + k dz``, Q = sum_k z_k p_k for acting and the greedy
target, and the cross-entropy against the projected target distribution as the loss.  Priorities are the KL divergence of the target
from the online distribution (Hessel et al. 2018).  The state-dict names stay the plain head's ten.

``ApexHParams(noisy_dqn=True)`` makes fc and every head layer a noisy layer (Fortunato et al. 2018, factorised Gaussian noise):
``y = (mu_w + sigma_w * eps_w) x + mu_b + sigma_b * eps_b`` with ``eps_w = f(eps_out) f(eps_in)^T``, ``eps_b = f(eps_out)`` and
``f(x) = sgn(x) sqrt|x|``.  Update k draws new noise for the online network (shared by Q(s) and the double-DQN choice at s') and an
independent draw for the target network, both from (seed, k); ``q_values``, ``predict`` and ``get_action`` use the mean weights mu.

``ApexHParams(quantile_dqn=True)`` makes the head the quantile head of QR-DQN (Dabney et al. 2018): ``q = Linear(512, A *
num_quantiles)``, row a N + i quantile i of action a at the midpoint tau_i = (2 i + 1) / (2 N), Q = the mean of an action's quantiles
for acting and the greedy target, and the quantile Huber loss (threshold ``quantile_kappa``) against the target quantiles
``r + gamma theta'(s')[a*]`` as the loss and the priority.  It needs no support; the state-dict names stay the plain head's ten.

``ApexHParams(distributional_dueling=True)``, with ``categorical_dqn`` or ``quantile_dqn``, gives that head the dueling architecture per
atom or quantile, as in Rainbow (Hessel et al. 2018): ``value = Linear(512, W)`` and ``advantage = Linear(512, A * W)`` (W = num_atoms
or num_quantiles) on the shared fc output, combined into the head rows ``v.view(-1, 1, W) + adv.view(-1, A, W) - adv.view(-1, A,
W).mean(1, keepdim=True)``, which the C51 or QR update then reads as before.  The state-dict names are the dueling head's.
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

from ... import _lib
from ...learner import from_torch_optimizer_state, to_torch_optimizer_state
from ..base import BaseAgent

MAX_FRAMES = 65536           # frames of one encoder call (MAX_FRAMES in csrc/kernels.h)
PLAIN_SUFFIXES = ('weight', 'bias')
NOISY_SUFFIXES = ('weight_mu', 'weight_sigma', 'bias_mu', 'bias_sigma')     # NoisyLinear's parameters, in registration order


def apex_param_shapes(num_actions: int, dueling: bool = False, num_atoms: int = 0, noisy: bool = False, num_quantiles: int = 0,
                      dist_dueling: bool = False):
    """the named shapes of the Q network's parameters in state_dict order = AtariQNet.parameters() order = the integer keys of the
    Adam state (srl_apex_param_layout_dist_dueling order): conv1..3, fc, then q or value and advantage; num_atoms > 0: the categorical
    head q = Linear(512, num_actions * num_atoms); num_quantiles > 0: the quantile head q = Linear(512, num_actions * num_quantiles);
    dist_dueling: that head as value = Linear(512, W) and advantage = Linear(512, num_actions * W), W = num_atoms or num_quantiles;
    noisy: fc and the head layers as NoisyLinear's weight_mu, weight_sigma, bias_mu, bias_sigma"""
    lin = NOISY_SUFFIXES if noisy else PLAIN_SUFFIXES
    width = num_atoms or num_quantiles or 1
    rows = num_actions * width
    if dist_dueling:
        head = [('value', (width, 512)), ('advantage', (rows, 512))]
    else:
        head = [('value', (1, 512)), ('advantage', (num_actions, 512))] if dueling else [('q', (rows, 512))]
    layers = [('conv1', (32, 4, 8, 8), PLAIN_SUFFIXES), ('conv2', (64, 32, 4, 4), PLAIN_SUFFIXES), ('conv3', (64, 64, 3, 3), PLAIN_SUFFIXES),
              ('fc', (512, 3136), lin)] + [(l, w, lin) for l, w in head]
    return OrderedDict((f'{l}.{s}', w if s.startswith('weight') else w[:1]) for l, w, suffixes in layers for s in suffixes)


def apex_param_names(dueling: bool = False, noisy: bool = False):
    return tuple(apex_param_shapes(1, dueling, 0, noisy))


APEX_PARAM_NAMES = apex_param_names()
APEX_DUELING_PARAM_NAMES = apex_param_names(dueling=True)
APEX_NOISY_PARAM_NAMES = apex_param_names(noisy=True)
APEX_NOISY_DUELING_PARAM_NAMES = apex_param_names(dueling=True, noisy=True)


def check_net_args(num_actions, noisy_std) -> None:
    """ValueError unless num_actions is an int in [1, 31] and noisy_std (the noisy layers' sigma0) a finite number >= 0"""
    if isinstance(num_actions, bool) or not isinstance(num_actions, (int, np.integer)) or not 1 <= num_actions <= 31:
        raise ValueError(f'num_actions must be an int in [1, 31], got {num_actions!r}')
    if isinstance(noisy_std, bool) or not isinstance(noisy_std, (int, float)) or not (math.isfinite(noisy_std) and noisy_std >= 0.0):
        raise ValueError(f'noisy_std must be finite and >= 0, got {noisy_std!r}')


def scale_noise(x: torch.Tensor) -> torch.Tensor:
    """f(x) = sgn(x) sqrt|x| of factorised Gaussian noise"""
    return x.sign().mul(x.abs().sqrt())


class NoisyLinear(nn.Module):
    """The factorised Gaussian noisy layer of Fortunato et al. 2018: in train mode ``y = (weight_mu + weight_sigma * weight_epsilon) x
    + bias_mu + bias_sigma * bias_epsilon`` with ``weight_epsilon = outer(eps_out, eps_in)`` and ``bias_epsilon = eps_out``, the f-scaled
    noise vectors (non-persistent buffers, redrawn by ``reset_noise()`` or set by ``set_noise``); in eval mode ``y = weight_mu x +
    bias_mu``.  Init (section 3.2): mu ~ U[-1/sqrt(p), 1/sqrt(p)], sigma = std_init / sqrt(p), p = in_features."""

    def __init__(self, in_features: int, out_features: int, std_init: float = 0.5):
        super().__init__()
        self.in_features, self.out_features, self.std_init = int(in_features), int(out_features), float(std_init)
        self.weight_mu = nn.Parameter(torch.empty(out_features, in_features))
        self.weight_sigma = nn.Parameter(torch.empty(out_features, in_features))
        self.bias_mu = nn.Parameter(torch.empty(out_features))
        self.bias_sigma = nn.Parameter(torch.empty(out_features))
        self.register_buffer('eps_in', torch.zeros(in_features), persistent=False)
        self.register_buffer('eps_out', torch.zeros(out_features), persistent=False)
        self.register_buffer('weight_epsilon', torch.zeros(out_features, in_features), persistent=False)
        self.register_buffer('bias_epsilon', torch.zeros(out_features), persistent=False)
        self.reset_parameters()
        self.reset_noise()

    def reset_parameters(self) -> None:
        r = 1.0 / math.sqrt(self.in_features)
        with torch.no_grad():
            self.weight_mu.uniform_(-r, r)
            self.weight_sigma.fill_(self.std_init / math.sqrt(self.in_features))
            self.bias_mu.uniform_(-r, r)
            self.bias_sigma.fill_(self.std_init / math.sqrt(self.in_features))

    @torch.no_grad()
    def set_noise(self, eps_in: torch.Tensor, eps_out: torch.Tensor) -> None:
        """the f-scaled noise vectors [in_features] and [out_features]"""
        self.eps_in.copy_(eps_in)
        self.eps_out.copy_(eps_out)
        self.weight_epsilon.copy_(torch.outer(self.eps_out, self.eps_in))
        self.bias_epsilon.copy_(self.eps_out)

    def reset_noise(self) -> None:
        """new noise from torch's generator of the layer's device (capturable on a CUDA device)"""
        dev = self.eps_in.device
        self.set_noise(scale_noise(torch.randn(self.in_features, device=dev)), scale_noise(torch.randn(self.out_features, device=dev)))

    def effective(self):
        """(weight, bias) of the current mode"""
        if not self.training:
            return self.weight_mu, self.bias_mu
        return self.weight_mu + self.weight_sigma * self.weight_epsilon, self.bias_mu + self.bias_sigma * self.bias_epsilon

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return F.linear(x, *self.effective())


def categorical_support(num_atoms: int, v_min: float, v_max: float) -> torch.Tensor:
    """z_k = v_min + k dz in fp32, dz = (v_max - v_min) / (num_atoms - 1) rounded once to fp32 (the bounds rounded to fp32 first, as
    the C ABI receives them)"""
    lo, hi = float(np.float32(v_min)), float(np.float32(v_max))
    dz = torch.tensor((hi - lo) / (num_atoms - 1), dtype=torch.float32)
    return torch.tensor(lo, dtype=torch.float32) + torch.arange(num_atoms, dtype=torch.float32) * dz


def quantile_taus(num_quantiles: int) -> torch.Tensor:
    """the quantile midpoints tau_i = (2 i + 1) / (2 N), i = 0 .. N - 1, each one fp32 division"""
    return (2 * torch.arange(num_quantiles, dtype=torch.float32) + 1) / torch.tensor(2 * num_quantiles, dtype=torch.float32)


class AtariQNet(nn.Module):
    """Nature DQN on 4 stacked 84x84 frames: AtariNet's conv1..3 and fc (scalerl/algorithms/utils/atari_model.py:30-47, 91-101)
    followed by ``q = nn.Linear(512, num_actions)``, or, with ``dueling``, by ``value = nn.Linear(512, 1)`` and ``advantage =
    nn.Linear(512, num_actions)`` combined as Q = V + Adv - mean_a Adv (Wang et al. 2016, eq. 9), or, with ``categorical``, by
    ``q = nn.Linear(512, num_actions * num_atoms)`` whose row a * num_atoms + k is atom k of action a (C51): ``dist(obs)`` gives the
    softmax per action, ``forward`` its expectation on the support (a non-persistent buffer: the state-dict names are the plain ten).
    Initialised by torch's default layer init, so ``torch.manual_seed(s)`` before construction fixes the weights.  With ``noisy``, fc
    and the head layers are ``NoisyLinear(..., noisy_std)`` (train mode: the noisy weights, eval mode: mu; ``reset_noise()`` redraws
    every layer's noise).  With ``quantile``, ``q = nn.Linear(512, num_actions * num_quantiles)`` whose row a * num_quantiles + i is
    quantile i of action a (QR-DQN): ``quantiles(obs)`` gives them, ``forward`` their mean (the midpoints ``taus`` are a non-persistent
    buffer).  With ``distributional_dueling`` (and ``categorical`` or ``quantile``) the head rows are Rainbow's dueling ones per atom or
    quantile: ``value = nn.Linear(512, W)`` and ``advantage = nn.Linear(512, num_actions * W)`` combined as ``v.view(-1, 1, W) +
    adv.view(-1, A, W) - adv.view(-1, A, W).mean(1, keepdim=True)``, W = num_atoms or num_quantiles."""

    def __init__(self, num_actions: int, observation_shape=(4, 84, 84), dueling: bool = False, categorical: bool = False,
                 num_atoms: int = 51, v_min: float = 0.0, v_max: float = 200.0, noisy: bool = False, noisy_std: float = 0.5,
                 quantile: bool = False, num_quantiles: int = 200, distributional_dueling: bool = False):
        super().__init__()
        if dueling and categorical:
            raise ValueError('the categorical head with the dueling head is not supported')
        if quantile and (dueling or categorical):
            raise ValueError('the quantile head with the dueling or the categorical head is not supported')
        if distributional_dueling and not (categorical or quantile):
            raise ValueError('distributional_dueling needs the categorical or the quantile head')
        self.observation_shape = tuple(observation_shape)
        self.num_actions = int(num_actions)
        self.dueling = bool(dueling)
        self.categorical = bool(categorical)
        self.noisy = bool(noisy)
        self.num_atoms = int(num_atoms) if self.categorical else 0
        self.quantile = bool(quantile)
        self.num_quantiles = int(num_quantiles) if self.quantile else 0
        self.distributional_dueling = bool(distributional_dueling)
        width = self.num_atoms or self.num_quantiles
        linear = (lambda i, o: NoisyLinear(i, o, noisy_std)) if self.noisy else nn.Linear
        self.conv1 = nn.Conv2d(self.observation_shape[0], 32, kernel_size=8, stride=4)
        self.conv2 = nn.Conv2d(32, 64, kernel_size=4, stride=2)
        self.conv3 = nn.Conv2d(64, 64, kernel_size=3, stride=1)
        self.fc = linear(3136, 512)
        if self.dueling:
            self.value = linear(512, 1)
            self.advantage = linear(512, self.num_actions)
        elif self.distributional_dueling:
            self.value = linear(512, width)
            self.advantage = linear(512, self.num_actions * width)
        elif self.categorical or self.quantile:
            self.q = linear(512, self.num_actions * width)
        else:
            self.q = linear(512, self.num_actions)
        if self.categorical:
            self.register_buffer('support', categorical_support(self.num_atoms, v_min, v_max), persistent=False)
        if self.quantile:
            self.register_buffer('taus', quantile_taus(self.num_quantiles), persistent=False)

    def noisy_layers(self):
        """the NoisyLinear layers in state-dict order (none without noise)"""
        return [m for m in (self.fc, getattr(self, 'q', None), getattr(self, 'value', None), getattr(self, 'advantage', None))
                if isinstance(m, NoisyLinear)]

    def reset_noise(self) -> None:
        for m in self.noisy_layers():
            m.reset_noise()

    def _features(self, obs: torch.Tensor) -> torch.Tensor:
        x = obs.float() / 255.0
        x = F.relu(self.conv1(x))
        x = F.relu(self.conv2(x))
        x = F.relu(self.conv3(x))
        return F.relu(self.fc(x.reshape(x.shape[0], -1)))

    def _rows(self, obs: torch.Tensor) -> torch.Tensor:
        """a distributional head's rows [n, A, W] (logits or quantiles)"""
        x = self._features(obs)
        W = self.num_atoms or self.num_quantiles
        if self.distributional_dueling:
            v, adv = self.value(x).view(-1, 1, W), self.advantage(x).view(-1, self.num_actions, W)
            return v + adv - adv.mean(1, keepdim=True)
        return self.q(x).view(-1, self.num_actions, W)

    def dist(self, obs: torch.Tensor) -> torch.Tensor:
        """categorical head: obs u8 [N, 4, 84, 84] -> the atom probabilities p [N, A, num_atoms]"""
        if not self.categorical:
            raise ValueError('dist() needs the categorical head (AtariQNet(..., categorical=True))')
        return F.softmax(self._rows(obs), dim=2)

    def quantiles(self, obs: torch.Tensor) -> torch.Tensor:
        """quantile head: obs u8 [n, 4, 84, 84] -> the quantiles theta [n, A, num_quantiles]"""
        if not self.quantile:
            raise ValueError('quantiles() needs the quantile head (AtariQNet(..., quantile=True))')
        return self._rows(obs)

    def forward(self, obs: torch.Tensor) -> torch.Tensor:
        """obs u8 [N, 4, 84, 84] -> Q values [N, A]"""
        if self.categorical:
            return (self.dist(obs) * self.support).sum(2)
        if self.quantile:
            return self.quantiles(obs).mean(2)
        x = self._features(obs)
        if self.dueling:
            v, adv = self.value(x), self.advantage(x)
            return v + adv - adv.mean(dim=1, keepdim=True)
        return self.q(x)


@dataclass
class ApexHParams:
    """The learner's settings, with the names and defaults of ScaleRL's ``DQNArguments`` and the Ape-X ``Learner``
    (apex/worker.py:120-132): Adam at lr 1e-3 with torch's default betas / eps, no clipping, a hard target copy every 100 steps."""
    batch_size: int = 32
    num_actions: int = 6
    gamma: float = 0.99                  # pass gamma ** n for n-step transitions
    learning_rate: float = 1e-3
    max_grad_norm: Optional[float] = None
    double_dqn: bool = False
    dueling_dqn: bool = False            # the dueling head V + Adv - mean(Adv) on the shared fc output instead of q = Linear(512, A)
    noisy_dqn: bool = False              # fc and the head layers as factorised Gaussian noisy layers (Fortunato et al. 2018)
    noisy_std: float = 0.5               # their initial sigma0: sigma = noisy_std / sqrt(in_features)
    categorical_dqn: bool = False        # the categorical (C51) head q = Linear(512, A num_atoms) on the support [v_min, v_max]
    v_min: float = 0.0
    v_max: float = 200.0
    num_atoms: int = 51
    target_update_frequency: int = 100
    soft_update_tau: float = 1.0
    precision: str = 'bf16'              # encoder operands: 'bf16' | 'fp32_split' (fp32-accurate hi/lo bf16 pairs)
    priority_eps: float = 1e-6           # priority = |q - y| + priority_eps; 0 is the reference's value (which the tree asserts > 0)
    adam_beta1: float = 0.9
    adam_beta2: float = 0.999
    adam_eps: float = 1e-8
    quantile_dqn: bool = False           # the quantile (QR-DQN) head q = Linear(512, A num_quantiles) and the quantile Huber loss
    num_quantiles: int = 200             # N, the paper's Atari setting
    quantile_kappa: float = 1.0          # the Huber threshold kappa > 0 (1: QR-DQN-1)
    distributional_dueling: bool = False  # Rainbow's dueling head per atom / quantile (with categorical_dqn or quantile_dqn)
    optimizer: ClassVar[str] = 'adam'            # read by learner.py's optimizer-state converters
    lr_schedule: ClassVar[str] = 'constant'

    def validate(self) -> None:
        if not (isinstance(self.batch_size, int) and 1 <= self.batch_size <= MAX_FRAMES):
            raise ValueError(f'batch_size must be an int in [1, {MAX_FRAMES}], got {self.batch_size!r}')
        check_net_args(self.num_actions, self.noisy_std)
        self.head                            # ValueError on a bad head setting
        if not (math.isfinite(self.gamma) and self.gamma >= 0.0):
            raise ValueError(f'gamma must be finite and >= 0, got {self.gamma}')
        if not (math.isfinite(self.learning_rate) and self.learning_rate > 0.0):
            raise ValueError(f'learning_rate must be finite and > 0, got {self.learning_rate}')
        if self.max_grad_norm is not None and not self.max_grad_norm > 0.0:
            raise ValueError(f'max_grad_norm must be None or > 0, got {self.max_grad_norm}')
        if not (isinstance(self.target_update_frequency, int) and self.target_update_frequency >= 1):
            raise ValueError(f'target_update_frequency must be an int >= 1, got {self.target_update_frequency!r}')
        if not 0.0 <= self.soft_update_tau <= 1.0:
            raise ValueError(f'soft_update_tau must be in [0, 1], got {self.soft_update_tau}')
        if self.precision not in ('bf16', 'fp32_split'):
            raise ValueError(f"precision must be 'bf16' or 'fp32_split', got {self.precision!r}")
        if not (math.isfinite(self.priority_eps) and self.priority_eps >= 0.0):
            raise ValueError(f'priority_eps must be finite and >= 0, got {self.priority_eps}')
        if not (0.0 <= self.adam_beta1 < 1.0 and 0.0 <= self.adam_beta2 < 1.0):
            raise ValueError(f'Adam betas must be in [0, 1), got ({self.adam_beta1}, {self.adam_beta2})')
        if not (math.isfinite(self.adam_eps) and self.adam_eps >= 0.0):
            raise ValueError(f'adam_eps must be finite and >= 0, got {self.adam_eps}')

    @property
    def head(self) -> 'QHead':
        """the Q head these settings describe (ValueError on a bad one)"""
        return QHead.of(self.dueling_dqn, self.categorical_dqn, self.num_atoms, self.v_min, self.v_max, self.noisy_dqn, self.quantile_dqn,
                        self.num_quantiles, self.quantile_kappa, self.distributional_dueling)

    def to_c(self) -> _lib.SrlApexConfig:
        self.validate()
        c = _lib.SrlApexConfig()
        c.B, c.A = self.batch_size, self.num_actions
        c.precision = 0 if self.precision == 'bf16' else 1
        c.double_dqn = 1 if self.double_dqn else 0
        c.gamma = self.gamma
        c.max_grad_norm = math.inf if self.max_grad_norm is None else self.max_grad_norm
        c.learning_rate, c.adam_beta1, c.adam_beta2, c.adam_eps = self.learning_rate, self.adam_beta1, self.adam_beta2, self.adam_eps
        c.priority_eps = self.priority_eps
        c.dueling = 1 if self.dueling_dqn else 0
        c.num_atoms = self.atoms()
        c.v_min, c.v_max = self.v_min, self.v_max
        c.noisy = 1 if self.noisy_dqn else 0
        c.num_quantiles = self.quantiles()
        c.kappa = self.quantile_kappa
        c.dist_dueling = 1 if self.distributional_dueling else 0
        return c

    def atoms(self) -> int:
        """the categorical head's atom count, 0 for a scalar head"""
        return self.num_atoms if self.categorical_dqn else 0

    def quantiles(self) -> int:
        """the quantile head's quantile count, 0 for the other heads"""
        return self.num_quantiles if self.quantile_dqn else 0


@dataclass(frozen=True)
class QHead:
    """The Q head of the learner and its actors: q = Linear(512, A), the dueling head (``dueling``), the categorical head on
    ``num_atoms`` > 0 atoms of the support [v_min, v_max], or the quantile head on ``num_quantiles`` > 0 quantiles with the Huber
    threshold ``kappa``; ``noisy``: fc and the head layers are noisy layers; ``dist_dueling``: the categorical or quantile head as
    Rainbow's dueling rows.  A head keeps no setting of another kind, so equal heads compare equal."""
    dueling: bool = False
    num_atoms: int = 0
    v_min: float = 0.0
    v_max: float = 0.0
    noisy: bool = False
    num_quantiles: int = 0
    kappa: float = 0.0
    dist_dueling: bool = False

    @classmethod
    def of(cls, dueling_dqn, categorical_dqn, num_atoms, v_min, v_max, noisy_dqn=False, quantile_dqn=False, num_quantiles=200,
           quantile_kappa=1.0, distributional_dueling=False) -> 'QHead':
        """the head of ApexHParams' / B200ApexActor's settings, checked (the support and the quantile setting, as the kernels read
        them in fp32, even when their head is off)"""
        if not isinstance(dueling_dqn, bool):
            raise ValueError(f'dueling_dqn must be a bool, got {dueling_dqn!r}')
        if not isinstance(categorical_dqn, bool):
            raise ValueError(f'categorical_dqn must be a bool, got {categorical_dqn!r}')
        if isinstance(num_atoms, bool) or not isinstance(num_atoms, (int, np.integer)) or not 2 <= num_atoms <= 64:
            raise ValueError(f'num_atoms must be an int in [2, 64], got {num_atoms!r}')
        with np.errstate(over='ignore'):
            lo, hi = np.float32(v_min), np.float32(v_max)
        if not (np.isfinite(lo) and np.isfinite(hi) and lo < hi and np.isfinite(np.float32((float(hi) - float(lo)) / (num_atoms - 1)))):
            raise ValueError(f'v_min and v_max must be finite fp32 values with v_min < v_max, got ({v_min}, {v_max})')
        if not isinstance(noisy_dqn, bool):
            raise ValueError(f'noisy_dqn must be a bool, got {noisy_dqn!r}')
        if categorical_dqn and dueling_dqn:
            raise ValueError('categorical_dqn with dueling_dqn is not supported: choose one head')
        if not isinstance(quantile_dqn, bool):
            raise ValueError(f'quantile_dqn must be a bool, got {quantile_dqn!r}')
        if isinstance(num_quantiles, bool) or not isinstance(num_quantiles, (int, np.integer)) or not 2 <= num_quantiles <= 256:
            raise ValueError(f'num_quantiles must be an int in [2, 256], got {num_quantiles!r}')
        with np.errstate(over='ignore'):
            ok = not isinstance(quantile_kappa, bool) and isinstance(quantile_kappa, (int, float, np.floating)) and \
                np.isfinite(np.float32(quantile_kappa)) and np.float32(quantile_kappa) > 0
        if not ok:
            raise ValueError(f'quantile_kappa must be a finite fp32 value > 0, got {quantile_kappa!r}')
        if quantile_dqn and dueling_dqn:
            raise ValueError('quantile_dqn with dueling_dqn is not supported: choose one head')
        if quantile_dqn and categorical_dqn:
            raise ValueError('quantile_dqn with categorical_dqn is not supported: choose one head')
        if not isinstance(distributional_dueling, bool):
            raise ValueError(f'distributional_dueling must be a bool, got {distributional_dueling!r}')
        if distributional_dueling and dueling_dqn:
            raise ValueError('distributional_dueling with dueling_dqn is not supported: dueling_dqn is the scalar dueling head')
        if distributional_dueling and not (categorical_dqn or quantile_dqn):
            raise ValueError('distributional_dueling needs categorical_dqn or quantile_dqn')
        if quantile_dqn:
            return cls(noisy=noisy_dqn, num_quantiles=int(num_quantiles), kappa=float(quantile_kappa), dist_dueling=distributional_dueling)
        if categorical_dqn:
            return cls(False, int(num_atoms), float(v_min), float(v_max), noisy_dqn, dist_dueling=distributional_dueling)
        return cls(dueling_dqn, noisy=noisy_dqn)

    def __str__(self):
        s = f'dueling_dqn={self.dueling}, categorical_dqn={self.num_atoms > 0}, noisy_dqn={self.noisy}'
        if self.num_quantiles:
            s += f', quantile_dqn=True, (num_quantiles, quantile_kappa)={(self.num_quantiles, self.kappa)}'
        elif self.num_atoms:
            s += f', (num_atoms, v_min, v_max)={(self.num_atoms, self.v_min, self.v_max)}'
        return s + ', distributional_dueling=True' if self.dist_dueling else s

    def names(self):
        return apex_param_names(self.dueling or self.dist_dueling, self.noisy)

    def shapes(self, num_actions: int):
        return apex_param_shapes(num_actions, self.dueling, self.num_atoms, self.noisy, self.num_quantiles, self.dist_dueling)

    def layout(self, num_actions: int):
        """(total floats, offsets, counts) of the flat buffer"""
        return _lib.apex_param_layout(num_actions, self.dueling, self.num_atoms, self.noisy, self.num_quantiles, self.dist_dueling)


def flat_views(flat: torch.Tensor, off, cnt, shapes) -> 'OrderedDict[str, torch.Tensor]':
    """the named tensors of a flat buffer in srl_apex_param_layout order, as views"""
    return OrderedDict((n, flat[off[i]:off[i] + cnt[i]].view(shp)) for i, (n, shp) in enumerate(shapes.items()))


def load_views(dst: Dict[str, torch.Tensor], sd: Dict[str, torch.Tensor]) -> None:
    """copies an AtariQNet-compatible state_dict into the views ``dst`` (KeyError on a missing name, ValueError on a shape)"""
    for n, v in dst.items():
        if n not in sd:
            raise KeyError(f'missing key {n} in state_dict')
        if tuple(sd[n].shape) != tuple(v.shape):
            raise ValueError(f'{n}: shape {tuple(sd[n].shape)} != {tuple(v.shape)}')
        v.copy_(sd[n].to(v.device, torch.float32))


def default_q_state_dict(num_actions: int, seed: int = 0, dueling: bool = False, num_atoms: int = 0, noisy: bool = False,
                         noisy_std: float = 0.5, num_quantiles: int = 0, dist_dueling: bool = False) -> 'OrderedDict[str, torch.Tensor]':
    """AtariQNet's initial weights under ``torch.manual_seed(seed)``, drawn without disturbing the global RNG (num_atoms > 0: the
    categorical head's; num_quantiles > 0: the quantile head's; dist_dueling: either as dueling rows; noisy: the noisy network's with
    sigma0 = noisy_std)"""
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        net = AtariQNet(num_actions, dueling=dueling, categorical=num_atoms > 0, num_atoms=num_atoms or 51, noisy=noisy, noisy_std=noisy_std,
                        quantile=num_quantiles > 0, num_quantiles=num_quantiles or 200, distributional_dueling=dist_dueling)
    return OrderedDict((k, v.detach().clone()) for k, v in net.state_dict().items())


class B200ApexLearner(BaseAgent):
    """The Ape-X learner on one GPU.  ``learn((obs, action, reward, next_obs, done), weights, idxs, sampler)`` runs one update:
    obs / next_obs u8 [B, 4, 84, 84], action int64 [B], reward float32 [B], done bool / uint8 [B], importance weights float32 [B]
    (None = 1) and the sampled indices int64 [B] of ``sampler`` (a GpuPrioritizedSampler), all contiguous CUDA tensors.  The step
    is captured as a CUDA graph per set of input addresses (first call eager, second captures, later calls replay), so a caller that
    gathers into fixed buffers replays -- the sampled idxs and weights included: ``GpuPrioritizedSampler.sample`` returns new tensors,
    copy them into fixed ones (each new address set costs an eager step and a capture, and its graph is kept).  The target network follows DQNAgent's cadence: after update k (from 0), when
    k % target_update_frequency == 0, target <- tau * online + (1 - tau) * target.  With ``hp.noisy_dqn`` the noise of update k is
    drawn from (``seed``, k): two learners with the same seed and step count draw the same noise."""

    def __init__(self, hp: ApexHParams, device=None, init_state_dict: Optional[Dict[str, torch.Tensor]] = None, seed: int = 0,
                 use_graph: bool = True):
        if not torch.cuda.is_available():
            raise RuntimeError('B200ApexLearner needs a CUDA device: scalerl_b200 has no CPU fallback')
        super().__init__(hp)
        cfg = hp.to_c()
        cfg.noise_seed = int(seed) % 2 ** 64
        self.hp = hp
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self._L = _lib.lib()
        head = hp.head
        self.names = head.names()
        self.shapes = head.shapes(hp.num_actions)
        with torch.cuda.device(self.device):
            total, self._off, self._cnt = head.layout(hp.num_actions)
            z = lambda: torch.zeros(total, dtype=torch.float32, device=self.device)
            self.flat_params, self.flat_grads, self.exp_avg, self.exp_avg_sq, self.flat_target = z(), z(), z(), z(), z()
            self.params = self._views(self.flat_params)
            self.grads = self._views(self.flat_grads)
            self.target_params = self._views(self.flat_target)
            self._cfg = cfg
            h = C.c_void_p()
            _lib.check(self._L.srl_apex_learner_create(C.addressof(cfg), self.flat_params.data_ptr(), self.flat_grads.data_ptr(),
                                                       self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(), self.flat_target.data_ptr(),
                                                       C.byref(h)), 'srl_apex_learner_create')
            self._h = h
            self._stats = torch.zeros(4, device=self.device)      # {loss, gradient norm, clip coefficient, pad}
        sd = default_q_state_dict(hp.num_actions, seed, head.dueling, head.num_atoms, head.noisy, hp.noisy_std, head.num_quantiles,
                                  head.dist_dueling) if init_state_dict is None else init_state_dict
        self.load_state_dict(sd)
        self.load_state_dict(sd, target=True)       # actor_target starts as a copy (dqn_agent.py:66-67)
        self.use_graph = use_graph
        self._graphs = {}
        self._seen = set()
        self._from = None
        self._opt_steps = 0
        self.learner_update_step = 0
        self.target_model_update_step = 0

    # ------------------------------------------------------------------ parameters
    def _views(self, flat):
        return flat_views(flat, self._off, self._cnt, self.shapes)

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def state_dict(self, target: bool = False) -> 'OrderedDict[str, torch.Tensor]':
        """AtariQNet-compatible state_dict of the online (or, ``target``, the target) network"""
        src = self.target_params if target else self.params
        return OrderedDict((n, p.detach().clone()) for n, p in src.items())

    def load_state_dict(self, sd: Dict[str, torch.Tensor], target: bool = False) -> None:
        load_views(self.target_params if target else self.params, sd)

    def get_weights(self):
        return {k: v.cpu() for k, v in self.state_dict().items()}

    def set_weights(self, weights) -> None:
        self.load_state_dict(weights)

    # ------------------------------------------------------------------ optimizer state and checkpoints
    def _opt_tensors(self):
        return {'exp_avg': self._views(self.exp_avg), 'exp_avg_sq': self._views(self.exp_avg_sq)}

    def optimizer_state_dict(self) -> dict:
        """``torch.optim.Adam(AtariQNet(A, dueling=hp.dueling_dqn, categorical=hp.categorical_dqn, noisy=hp.noisy_dqn,
        quantile=hp.quantile_dqn, distributional_dueling=hp.distributional_dueling, ...).parameters()).state_dict()`` layout"""
        return to_torch_optimizer_state(self.hp, self._opt_tensors(), self._opt_steps, order=self.names)

    def load_optimizer_state_dict(self, sd: dict) -> None:
        step, kinds = from_torch_optimizer_state(sd, False, order=self.names)
        for kind in kinds:
            if kind not in ('exp_avg', 'exp_avg_sq'):
                raise ValueError(f"optimizer_state_dict holds '{kind}' but this learner runs Adam")
        for kind, views in self._opt_tensors().items():
            if kind not in kinds and step > 0:
                raise ValueError(f"optimizer_state_dict lacks '{kind}' for Adam")
            for n, v in views.items():
                v.copy_(kinds[kind][n]) if kind in kinds else v.zero_()
        self.set_step(step)

    def set_step(self, step: int) -> None:
        """Adam's step count (the device counter the captured step reads) and the target cadence's counters: one learn() is one
        optimizer step, so a resumed run continues all three where the checkpoint left them (updates k < step with k % freq == 0
        have refreshed the target)"""
        _lib.check(self._L.srl_apex_learner_set_step(self._h, int(step), self._stream()), 'srl_apex_learner_set_step')
        self._opt_steps = int(step)
        self.learner_update_step = int(step)
        self.target_model_update_step = -(-int(step) // self.hp.target_update_frequency)

    def save_checkpoint(self, path: str) -> None:
        """the keys of DQNAgent.save_checkpoint (dqn_agent.py:210-219)"""
        torch.save({'actor_state_dict': {k: v.cpu() for k, v in self.state_dict().items()},
                    'actor_target_state_dict': {k: v.cpu() for k, v in self.state_dict(target=True).items()},
                    'optimizer_state_dict': self.optimizer_state_dict()}, path)

    def load_checkpoint(self, path: str) -> None:
        ck = torch.load(path, map_location='cpu', weights_only=False)
        self.load_state_dict(ck['actor_state_dict'])
        self.load_state_dict(ck['actor_target_state_dict'], target=True)
        self.load_optimizer_state_dict(ck.get('optimizer_state_dict', {}))

    # ------------------------------------------------------------------ acting
    def _obs(self, obs):
        obs = torch.as_tensor(obs)
        if obs.dim() == 3:
            obs = obs.unsqueeze(0)
        if obs.dtype != torch.uint8 or tuple(obs.shape[1:]) != (4, 84, 84) or obs.shape[0] < 1:
            raise ValueError(f'obs must be uint8 [N, 4, 84, 84], got {tuple(obs.shape)} {obs.dtype}')
        return obs.to(self.device).contiguous()

    @torch.no_grad()
    def q_values(self, obs) -> torch.Tensor:
        """Q(obs) with the online network (noisy: its mean weights mu): uint8 [N, 4, 84, 84] (or one [4, 84, 84] frame stack) ->
        float32 [N, A].  Runs on its own
        encoder context and buffers, so actors may call it on another stream than learn(); it reads the parameters as they are when
        it runs."""
        obs = self._obs(obs)
        q = torch.empty(obs.shape[0], self.hp.num_actions, device=self.device)
        _lib.check(self._L.srl_apex_learner_q_values(self._h, obs.data_ptr(), obs.shape[0], q.data_ptr(), self._stream()),
                   'srl_apex_learner_q_values')
        return q

    def predict(self, obs) -> torch.Tensor:
        """greedy actions argmax_a Q(obs, a), int64 [N] on the learner's device (dqn_agent.py:114-134)"""
        return torch.argmax(self.q_values(obs), dim=-1)

    def get_action(self, obs, eps: float) -> torch.Tensor:
        """epsilon-greedy (dqn_agent.py:90-112) at the caller's epsilon: with probability eps one uniformly random action per row,
        drawn as the reference draws it, else predict(obs).  The decay schedule belongs to the agent loop."""
        obs = self._obs(obs)
        if random.random() < eps:
            a = np.argmax(np.random.uniform(0, 1, (obs.shape[0], self.hp.num_actions)), axis=1)
            return torch.from_numpy(a).to(self.device)
        return self.predict(obs)

    # ------------------------------------------------------------------ learning
    def _check(self, t, name, shape, dtypes):
        if not isinstance(t, torch.Tensor) or tuple(t.shape) != shape or t.dtype not in dtypes:
            got = (tuple(t.shape), t.dtype) if isinstance(t, torch.Tensor) else type(t)
            raise ValueError(f'{name}: expected {shape} {" or ".join(str(d) for d in dtypes)}, got {got}')
        if t.device != self.device or not t.is_contiguous():
            raise ValueError(f'{name} must be a contiguous tensor on {self.device}')

    def _inputs(self, experiences, weights, idxs, sampler):
        if len(experiences) != 5:
            raise ValueError('experiences must be (obs, action, reward, next_obs, done)')
        obs, action, reward, next_obs, done = experiences
        B = self.hp.batch_size
        self._check(obs, 'obs', (B, 4, 84, 84), (torch.uint8,))
        self._check(next_obs, 'next_obs', (B, 4, 84, 84), (torch.uint8,))
        self._check(action, 'action', (B,), (torch.int64,))
        self._check(reward, 'reward', (B,), (torch.float32,))
        self._check(done, 'done', (B,), (torch.bool, torch.uint8))
        if weights is not None:
            self._check(weights, 'weights', (B,), (torch.float32,))
        if (idxs is None) != (sampler is None):
            raise ValueError('idxs and sampler go together: pass both or neither')
        if idxs is not None:
            self._check(idxs, 'idxs', (B,), (torch.int64,))
        return obs, action, reward, next_obs, done.view(torch.uint8)

    def _enqueue(self, obs, action, reward, next_obs, done, weights, idxs, sampler):
        _lib.check(self._L.srl_apex_learner_step(
            self._h, obs.data_ptr(), action.data_ptr(), reward.data_ptr(), next_obs.data_ptr(), done.data_ptr(),
            weights.data_ptr() if weights is not None else None, idxs.data_ptr() if idxs is not None else None,
            sampler._h if sampler is not None else None, self._stats.data_ptr(), self._stream()), 'srl_apex_learner_step')

    def _graph_step(self, key, enqueue, keep=None):
        """enqueue() through the graph of `key` (`keep`: what the graph's buffers belong to, held while the graph lives)"""
        g = self._graphs.get(key)
        if g is None:
            if key not in self._seen:          # first sight: eager (warm-up of attributes and allocator state)
                self._seen.add(key)
                enqueue()
                return
            torch.cuda.current_stream(self.device).synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                enqueue()
            self._graphs[key] = (g, keep)
        else:
            g = g[0]
        g.replay()

    def _run(self, key, enqueue, use_graph, keep=None):
        if self.use_graph if use_graph is None else use_graph:
            self._graph_step(key, enqueue, keep)
        else:
            enqueue()

    @torch.no_grad()
    def learn(self, experiences, weights: Optional[torch.Tensor] = None, idxs: Optional[torch.Tensor] = None, sampler=None,
              sync_stats: bool = True, use_graph: Optional[bool] = None) -> Dict[str, float]:
        """one update (apex/worker.py:134-161; dqn_agent.py:136-190) -> {'loss': float}, or {} with nothing synchronised.  The
        categorical head's loss is mean(w * cross-entropy), the quantile head's mean(w * quantile Huber loss)."""
        obs, action, reward, next_obs, done = self._inputs(experiences, weights, idxs, sampler)
        args = (obs, action, reward, next_obs, done, weights, idxs, sampler)
        key = tuple(a.data_ptr() if isinstance(a, torch.Tensor) else (a._h.value if a is not None else None) for a in args)
        self._run(key, lambda: self._enqueue(*args), use_graph)
        return self._finish_update(sync_stats)

    @torch.no_grad()
    def learn_from(self, memory, beta: float = 0.4, sync_stats: bool = True, use_graph: Optional[bool] = None) -> Dict[str, float]:
        """one update on a batch of ``batch_size`` transitions sampled from ``memory`` (a GpuPrioritizedReplayBuffer or a
        GpuFrameReplayBuffer on this learner's device), all on the device: uniforms drawn by ``torch.rand`` (the default CUDA generator) into a fixed buffer, the
        prioritized sample and the gather into learner-owned fixed buffers, the step, and the new priorities written into
        ``memory``'s trees.  It is captured as one graph per memory (first call eager, second captures, later calls replay); the
        sampler reads the stored count and ``beta`` from the device, so a replay sees every add made since and a new ``beta`` costs
        one fill, not a recapture.  ``hp.gamma`` is used as given: for n-step memories pass ``gamma ** n_step``.  The target cadence
        and the step counters are learn()'s.  -> {'loss': float}, or {} with nothing synchronised."""
        from ...data.replay_memory import GpuFrameReplayBuffer, GpuPrioritizedReplayBuffer
        if not isinstance(memory, (GpuPrioritizedReplayBuffer, GpuFrameReplayBuffer)):
            raise ValueError(f'memory must be a GpuPrioritizedReplayBuffer or a GpuFrameReplayBuffer, got {type(memory).__name__}')
        if memory.device != self.device:
            raise ValueError(f'memory is on {memory.device}, the learner on {self.device}')
        if len(memory) < 2:
            raise ValueError(f'learn_from needs at least 2 stored transitions, the memory has {len(memory)}')
        memory._set_beta(beta)
        b = self._from_buffers()

        def enqueue():
            torch.rand(b['u'].shape, dtype=torch.float64, device=self.device, out=b['u'])
            memory._sample_into(b['u'], b['obs'], b['action'], b['reward'], b['next_obs'], b['done'], b['idxs'], b['weights'])
            self._enqueue(b['obs'], b['action'], b['reward'], b['next_obs'], b['done'], b['weights'], b['idxs'], memory.sampler)

        self._run(('learn_from', memory._h.value), enqueue, use_graph, keep=memory)
        return self._finish_update(sync_stats)

    def _from_buffers(self):
        """learn_from's fixed inputs: the uniforms and the gathered batch (the graph is keyed by the memory, not by these)"""
        if self._from is None:
            B, z = self.hp.batch_size, lambda *shape, dtype: torch.empty(*shape, dtype=dtype, device=self.device)
            self._from = {'u': z(B, dtype=torch.float64), 'obs': z(B, 4, 84, 84, dtype=torch.uint8), 'action': z(B, dtype=torch.int64),
                          'reward': z(B, dtype=torch.float32), 'next_obs': z(B, 4, 84, 84, dtype=torch.uint8), 'done': z(B, dtype=torch.uint8),
                          'idxs': z(B, dtype=torch.int64), 'weights': z(B, dtype=torch.float32)}
        return self._from

    def _finish_update(self, sync_stats):
        self._opt_steps += 1
        if self.learner_update_step % self.hp.target_update_frequency == 0:
            self.update_target(self.hp.soft_update_tau)
            self.target_model_update_step += 1
        self.learner_update_step += 1
        if not sync_stats:
            return {}
        return {'loss': float(self._stats[0].item())}

    def update_target(self, tau: float) -> None:
        """soft_target_update(online, target, tau) (utils/model_utils.py:29-32) on the current stream"""
        _lib.check(self._L.srl_apex_learner_update_target(self._h, float(tau), self._stream()), 'srl_apex_learner_update_target')

    def stats(self) -> Dict[str, float]:
        """{loss, grad_norm, clip_coef} of the last step (synchronises)"""
        s = self._stats.tolist()
        return {'loss': s[0], 'grad_norm': s[1], 'clip_coef': s[2]}

    def debug_buffer(self, name: str) -> torch.Tensor:
        """copy of one of the step's device buffers (tests only; names: srl_apex_learner_debug_buffer; the categorical head's
        logits, dlogits and m come flat, [B * A * num_atoms] and [B * num_atoms], and so do the quantile head's theta, dtheta and
        target_quantiles)"""
        p, n = C.c_void_p(), C.c_int64()
        _lib.check(self._L.srl_apex_learner_debug_buffer(self._h, name.encode(), C.byref(p), C.byref(n)), 'debug_buffer')
        dt = {'priorities': torch.float64, 'step': torch.int32, 'a1': torch.bfloat16, 'a2': torch.bfloat16, 'a3': torch.bfloat16}.get(name, torch.float32)
        out = torch.empty(n.value, dtype=dt, device=self.device)
        _lib.check(self._L.srl_memcpy_d2d(out.data_ptr(), p.value, n.value * out.element_size(), self._stream()), 'memcpy_d2d')
        torch.cuda.current_stream(self.device).synchronize()
        return out

    def release_graphs(self):
        torch.cuda.synchronize(self.device)
        self._graphs.clear()
        self._seen.clear()

    def close(self):
        if getattr(self, '_h', None) is not None:
            self._L.srl_apex_learner_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
