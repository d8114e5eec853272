"""B200ActorModel -- batched GPU actor inference behind the reference's actor calling convention (SURVEY.md §8f-4).

The reference's actors each run ``AtariNet`` on the CPU for ONE environment per call
(/root/reference scalerl/algorithms/impala/impala_atari.py:177-197).  This module evaluates the same network for N environments in
one call on the sm_90a forward kernels (``srl_learner_forward``: space-to-depth, the three wgmma convs, fc, heads) and samples the
actions on the device (``srl_sample_actions``) -- SEED-style central inference, but behind the SAME interface:

    agent_output, agent_state = actor_model(env_output, agent_state)        # env_output tensors are [1, N, ...]
    actor_model.initial_hidden_state(batch_size)   state_dict()   load_state_dict()   train() / eval()

so ``ImpalaTrainer.get_action``-style loops (and ``get_action_batched`` for N environments per actor process) use it unchanged.
Weights: its own flat fp32 buffer in the learner's layout; ``refresh(shared_flat, version)`` pulls a newer published version from
the shared-memory actor parameters with one H2D copy (the versioned publish of ImpalaTrainer.publish_weights), ``sync_from(learner)``
copies device-to-device when actor and learner share a process.

``use_lstm=True`` evaluates AtariNet(use_lstm=True): each call is one step of the 2-layer LSTM core for the N environments
(``srl_learner_forward_lstm_step``: the encoder and heads as above, one fused wgmma GEMM + cell kernel per LSTM layer).  The state
``(h, c)`` [2, N, 513 + A] is reset by ``env_output['done']`` before the step, as in the reference; it may be given on the host
or on the device, is never modified, and the new state comes back as new device tensors, so passing it back costs no copy.
The step reads a packed bf16 copy of the LSTM weights that ``load_state_dict``, ``refresh`` and ``sync_from`` re-derive."""
from collections import OrderedDict
from typing import Dict, Optional

import torch

from ... import _lib
from ...learner import B200ImpalaLearner, ImpalaHParams


class B200ActorModel:
    def __init__(self, num_envs: int, num_actions: int = 6, device=None, init_state_dict: Optional[Dict[str, torch.Tensor]] = None, seed: int = 0,
                 use_lstm: bool = False):
        # a forward-only context: T = 1 gives room for the single row an actor step evaluates (rows <= T + 1)
        self._ctx = B200ImpalaLearner(ImpalaHParams(rollout_length=1, batch_size=num_envs, num_actions=num_actions, use_lstm=use_lstm),
                                      device=device, process_group=False, init_state_dict=init_state_dict, seed=seed, use_graph=False)
        self.device = self._ctx.device
        self.num_envs, self.num_actions = num_envs, num_actions
        self.use_lstm = bool(use_lstm)
        self.core_size = 513 + num_actions
        self.training = True
        self.weights_version = 0
        self._gen = torch.Generator(device=self.device)
        self._gen.manual_seed(seed)
        B = num_envs
        self._pin = {'obs': torch.empty(1, B, 4, 84, 84, dtype=torch.uint8).pin_memory(), 'reward': torch.empty(1, B).pin_memory(),
                     'action': torch.empty(1, B, dtype=torch.int64).pin_memory()}
        if self.use_lstm:
            self._pin['done'] = torch.empty(1, B, dtype=torch.bool).pin_memory()
            self._pin_state = torch.empty(2, 2, B, self.core_size).pin_memory()           # host (h, c) in -> one H2D copy
            self._dev_state = torch.empty(2, 2, B, self.core_size, device=self.device)
            self._state_copied = torch.cuda.Event()
        self._dev = {k: torch.empty_like(v, device=self.device) for k, v in self._pin.items()}
        self._out_host = {'policy_logits': torch.empty(1, B, num_actions).pin_memory(), 'baseline': torch.empty(1, B).pin_memory(),
                          'action': torch.empty(1, B, dtype=torch.int64).pin_memory()}
        self._flat_pin = None

    # ---- module-like surface ---------------------------------------------------------------------------------------------
    def train(self, mode: bool = True):
        self.training = bool(mode)
        return self

    def eval(self):
        return self.train(False)

    def share_memory(self):
        return self

    def initial_hidden_state(self, batch_size: int):
        """atari_model.py:61-75: () without LSTM, else (h0, c0) zeros [2, batch, 513 + A] on the host"""
        if not self.use_lstm:
            return tuple()
        return tuple(torch.zeros(2, batch_size, self.core_size) for _ in range(2))

    def state_dict(self):
        return OrderedDict((k, v.cpu()) for k, v in self._ctx.state_dict().items())

    def load_state_dict(self, sd, strict=True):
        self._ctx.load_state_dict(sd)

    # ---- weights -----------------------------------------------------------------------------------------------------------
    def sync_from(self, learner: B200ImpalaLearner, version: Optional[int] = None) -> None:
        """same process: device-to-device copy of the learner's flat parameters (same layout by construction)"""
        if learner.numel != self._ctx.numel:
            raise ValueError('learner and actor were built for different num_actions')
        self._ctx.flat_params.copy_(learner.flat_params, non_blocking=True)
        self._pack()
        self.weights_version = self.weights_version + 1 if version is None else int(version)

    def refresh(self, shared_flat: torch.Tensor, version: int) -> bool:
        """pull a newer published version from the shared-memory flat actor parameters (ActorNet.flat_params): one H2D copy"""
        if int(version) == self.weights_version:
            return False
        if shared_flat.numel() != self._ctx.numel:
            raise ValueError('shared parameter buffer has another layout')
        if self._flat_pin is None:
            self._flat_pin = torch.empty(self._ctx.numel).pin_memory()
        self._flat_pin.copy_(shared_flat)                 # snapshot (the learner may be writing the next version)
        self._ctx.flat_params.copy_(self._flat_pin, non_blocking=True)
        self._pack()
        self.weights_version = int(version)
        return True

    def _pack(self):
        """the LSTM step reads a packed bf16 copy of the LSTM weights: re-derive it after the parameters changed"""
        if self.use_lstm:
            _lib.check(_lib.lib().srl_learner_pack_weights(self._ctx._h, torch.cuda.current_stream(self.device).cuda_stream), 'pack_weights')

    # ---- inference -----------------------------------------------------------------------------------------------------------
    def _state_ptrs(self, agent_state):
        """(h, c) device pointers of an input state: device fp32 [2, N, H] tensors are used in place, anything else is staged"""
        shape = (2, self.num_envs, self.core_size)
        if len(agent_state) != 2:
            raise ValueError('the LSTM actor needs agent_state = (h, c)')
        h, c = agent_state
        if all(t.device == self.device and t.dtype == torch.float32 and tuple(t.shape) == shape and t.is_contiguous() for t in (h, c)):
            return h.data_ptr(), c.data_ptr()
        self._state_copied.synchronize()            # the previous call's H2D copy has left the pinned staging buffer
        for i, t in enumerate((h, c)):
            if tuple(t.shape) != shape:
                raise ValueError(f'agent_state[{i}]: expected {shape}, got {tuple(t.shape)}')
            if t.is_cuda:
                self._dev_state[i].copy_(t)
            else:
                self._pin_state[i].copy_(t)
                self._dev_state[i].copy_(self._pin_state[i], non_blocking=True)
        self._state_copied.record(torch.cuda.current_stream(self.device))
        return self._dev_state[0].data_ptr(), self._dev_state[1].data_ptr()

    @torch.no_grad()
    def forward_device(self, obs: torch.Tensor, reward: torch.Tensor, action: torch.Tensor, done: Optional[torch.Tensor] = None,
                       agent_state=()):
        """device tensors [1, N, ...] -> (policy_logits [1,N,A], baseline [1,N], action [1,N]) on the device, nothing synchronised.
        With use_lstm also ``done`` [1, N] (bool or uint8) and ``agent_state`` = (h, c) [2, N, 513 + A] (host or device); the
        result then has a fourth element, the new state (h', c') as new device tensors.  The input state is not modified."""
        stream = torch.cuda.current_stream(self.device).cuda_stream
        if not self.use_lstm:
            out = self._ctx.forward({'obs': obs, 'reward': reward, 'action': action})
            return out['policy_logits'], out['baseline'], self._sample(out['policy_logits'], stream)
        if done is None:
            raise ValueError('the LSTM actor needs done')
        d = done.view(torch.uint8) if done.dtype == torch.bool else done
        for k, t in (('obs', obs), ('reward', reward), ('action', action), ('done', d)):
            if not t.is_cuda or not t.is_contiguous():
                raise ValueError(f'{k} must be a contiguous CUDA tensor')
        hp, cp = self._state_ptrs(agent_state)
        B, A = self.num_envs, self.num_actions
        lg = torch.empty(1, B, A, device=self.device)
        bs = torch.empty(1, B, device=self.device)
        h_new = torch.empty(2, B, self.core_size, device=self.device)
        c_new = torch.empty_like(h_new)
        _lib.check(_lib.lib().srl_learner_forward_lstm_step(
            self._ctx._h, obs.data_ptr(), reward.data_ptr(), d.data_ptr(), action.data_ptr(), hp, cp, lg.data_ptr(), bs.data_ptr(),
            h_new.data_ptr(), c_new.data_ptr(), stream), 'srl_learner_forward_lstm_step')
        return lg, bs, self._sample(lg, stream), (h_new, c_new)

    def _sample(self, lg, stream):
        """actions [1, N] on the device: softmax samples in training mode, argmax in eval mode (atari_model.py:130-134)"""
        N = lg.shape[0] * lg.shape[1]
        act = torch.empty(lg.shape[0], lg.shape[1], dtype=torch.int64, device=self.device)
        u = torch.rand(N, device=self.device, generator=self._gen) if self.training else None
        _lib.check(_lib.lib().srl_sample_actions(lg.data_ptr(), u.data_ptr() if u is not None else None, N, self.num_actions, act.data_ptr(),
                                                 stream), 'srl_sample_actions')
        return act

    @torch.no_grad()
    def __call__(self, env_output: Dict[str, torch.Tensor], agent_state=()):
        """the reference's ``actor_model(env_output, agent_state)`` for N environments: host tensors in, host tensors out.
        With use_lstm the new state comes back as (h', c') device tensors (pass them back as they are: no copy)."""
        for k in self._dev:
            t = env_output[k]
            if t.is_cuda:
                self._dev[k].copy_(t, non_blocking=True)
            else:
                self._pin[k].copy_(t)
                self._dev[k].copy_(self._pin[k], non_blocking=True)
        if self.use_lstm:
            lg, bs, act, state = self.forward_device(self._dev['obs'], self._dev['reward'], self._dev['action'], self._dev['done'], agent_state)
        else:
            (lg, bs, act), state = self.forward_device(self._dev['obs'], self._dev['reward'], self._dev['action']), tuple()
        self._out_host['policy_logits'].copy_(lg, non_blocking=True)
        self._out_host['baseline'].copy_(bs, non_blocking=True)
        self._out_host['action'].copy_(act, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        return {k: v.clone() for k, v in self._out_host.items()}, state

    def close(self):
        self._ctx.close()
