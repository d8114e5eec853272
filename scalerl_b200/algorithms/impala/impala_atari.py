"""ImpalaTrainer -- drop-in for scalerl/algorithms/impala/impala_atari.py with the learner on an H100.

Same public surface as the reference class (``ImpalaTrainer(args)``, ``create_buffers``, ``create_rnn_state_buffers``,
``get_action``, ``get_batch``, ``learn``, ``learn_process``, ``train``, ``save_checkpoint``; impala_atari.py:40-515), same
trajectory key schema (:122-151), same actor calling convention ``actor_model(env_output, agent_state) -> (outputs, state)``
(:177-197 -- the reference's own ``AtariNet`` can be passed as ``actor_model_fn``), same stats keys (:333-340) and
checkpoint keys (:506-511).  What changes behind it:

  * buffers live in ONE shared-memory block per slot (obs + the small fields), registered as pinned host memory by the
    learner process: ``get_batch`` issues one asynchronous H2D copy per slot on a copy stream + one unpack kernel instead of
    ``torch.stack`` + a pageable ``.to(device)`` (:248-265).  Nothing in it waits for the GPU: a slot returns to
    ``free_queue`` when its copy event has fired (polled; ownership rule of SURVEY.md §8b), the learner stream waits for the
    copy on the device, and two device batches alternate so the copy of batch k+1 overlaps the step on batch k;
  * ``learn`` enqueues the sm_90a step (B200ImpalaLearner.learn_async), a device-side snapshot of the new weights and
    their asynchronous D2H on a publish stream straight into the (pinned, shared-memory) actor parameters, followed by a
    version counter (:348 + SURVEY.md §8f-4); stats are read one step behind (``stats_lag``; 0 = the reference's
    synchronous behaviour);
  * CUDA is first touched inside the learner process (the reference forks after building models in the parent,
    SURVEY.md §7 hard part 8); ``global_step`` is a shared counter (the reference's plain int never reaches the parent).

Actors stay ordinary Python processes running a CPU policy.  Inside ScaleRL they use the reference's own ``AtariNet`` +
``TorchEnvWrapper``; ``env_fn`` / ``actor_model_fn`` default to the self-contained stand-ins of
``scalerl_b200.algorithms.utils`` because gymnasium / ale_py are not installed in this image.
"""
from __future__ import annotations

import collections
import ctypes
import math
import os
import time
import timeit
import traceback
from dataclasses import dataclass
from typing import Any, Callable, Dict, List, Optional, Tuple

import torch
from torch import multiprocessing as mp

from ...learner import B200ImpalaLearner, ImpalaHParams
from ...utils.profile import Timings, nvtx_range
from ..utils.atari_model import ActorNet, SyntheticAtariEnv


@dataclass
class ImpalaArguments:
    """RLArguments fields ImpalaTrainer reads (rl_args.py:71-159) plus the ones it reads but RLArguments never
    defined (impala_atari.py:56,72-77,303-308,325-327,375,412,502) with upstream torchbeast defaults."""
    env_id: str = 'PongNoFrameskip-v4'
    project: str = 'impala'
    algo_name: str = 'impala_b200'
    output_dir: str = './work_dir'
    use_cuda: bool = True
    num_actors: int = 4
    num_learners: int = 1
    num_buffers: Optional[int] = None
    batch_size: int = 8
    rollout_length: int = 20
    total_steps: int = 100000
    use_lstm: bool = False
    reward_clipping: str = 'abs_one'
    discounting: float = 0.99
    baseline_cost: float = 0.5
    entropy_cost: float = 0.0006
    max_grad_norm: float = 40.0
    learning_rate: float = 1e-4
    alpha: float = 0.99
    momentum: float = 0.0
    epsilon: float = 1e-5
    optimizer: str = 'rmsprop'
    lr_schedule: str = 'constant'  # 'linear': decay to min_learning_rate over total_steps frames (torchbeast's LambdaLR; rl_args.py:233-252)
    min_learning_rate: float = 0.0
    disable_checkpoint: bool = False
    num_actions: int = 6
    obs_shape: Tuple[int, int, int] = (4, 84, 84)
    seed: int = 0
    stats_lag: int = 1            # learn() returns the stats of step k - stats_lag (0: synchronous, as the reference)
    publish_every: int = 1        # weight publish cadence in learner steps (the reference publishes every step, :348)


def slot_layout(T: int, A: int, obs_shape=(4, 84, 84)):
    """byte layout of one trajectory slot: every key of create_buffers (impala_atari.py:135-147), 64-byte aligned"""
    n = T + 1
    specs = [('obs', (n, *obs_shape), torch.uint8), ('reward', (n,), torch.float32), ('done', (n,), torch.bool),
             ('last_action', (n,), torch.int64), ('action', (n,), torch.int64), ('episode_return', (n,), torch.float32),
             ('episode_step', (n,), torch.int32), ('policy_logits', (n, A), torch.float32), ('baseline', (n,), torch.float32)]
    off, out = 0, {}
    for k, shp, dt in specs:
        nbytes = torch.empty(0, dtype=dt).element_size()
        for d in shp:
            nbytes *= d
        out[k] = (off, shp, dt, nbytes)
        off = (off + nbytes + 63) & ~63
    return out, off


_REGISTERED: Dict[int, torch.Tensor] = {}       # data_ptr -> tensor (kept alive while pinned)


def _host_register(t: torch.Tensor) -> None:
    """pin a host tensor for DMA (srl_host_register); it must be unpinned (_host_unregister) before its memory goes away"""
    from ... import _lib
    _lib.check(_lib.lib().srl_host_register(t.data_ptr(), t.numel() * t.element_size()), 'srl_host_register')
    _REGISTERED[t.data_ptr()] = t


def _host_unregister(t: torch.Tensor) -> None:
    from ... import _lib
    if _REGISTERED.pop(t.data_ptr(), None) is not None:
        _lib.lib().srl_host_unregister(t.data_ptr())


class TrajectoryRing:
    """num_buffers slots in one shared-memory uint8 block; ``buffers[key][m]`` are typed views (the reference's
    ``buffers[key][index][t, ...] = value`` writes work unchanged).  ``pin()`` registers the block with CUDA."""

    def __init__(self, T: int, A: int, num_buffers: int, obs_shape=(4, 84, 84)):
        self.T, self.A, self.num_buffers = T, A, num_buffers
        self.layout, self.slot_bytes = slot_layout(T, A, obs_shape)
        self.block = torch.zeros(num_buffers * self.slot_bytes, dtype=torch.uint8).share_memory_()
        self.buffers: Dict[str, List[torch.Tensor]] = {k: [] for k in self.layout}
        for m in range(num_buffers):
            base = m * self.slot_bytes
            for k, (off, shp, dt, nbytes) in self.layout.items():
                self.buffers[k].append(self.block[base + off: base + off + nbytes].view(dt).view(shp))
        self._pinned = False

    def pin(self):
        if not self._pinned:
            _host_register(self.block)
            self._pinned = True

    def unpin(self):
        if self._pinned:
            _host_unregister(self.block)
            self._pinned = False


class ImpalaTrainer:
    stat_keys = ['total_loss', 'mean_episode_return', 'pg_loss', 'baseline_loss', 'entropy_loss']

    def __init__(self, args: ImpalaArguments, env_fn: Optional[Callable[[], Any]] = None,
                 actor_model_fn: Optional[Callable[[], torch.nn.Module]] = None, learner: Optional[B200ImpalaLearner] = None) -> None:
        """``learner``: adopt an existing B200ImpalaLearner (same T / B / A) instead of creating one at the first learner call"""
        self.args = args
        self._adopt = learner
        if args.num_buffers is None:                                   # impala_atari.py:72-73, applied BEFORE create_buffers
            args.num_buffers = max(2 * args.num_actors, args.batch_size)
        if args.num_actors >= args.num_buffers:                        # :74-75
            raise ValueError('num_buffers should be larger than num_actors')
        if args.num_buffers < args.batch_size:                         # :76-77
            raise ValueError('num_buffers should be larger than batch_size')
        self.env_fn = env_fn or (lambda: SyntheticAtariEnv(args.obs_shape, args.num_actions, seed=args.seed))
        # any module with the reference AtariNet's interface: __call__(env_output, agent_state) -> (dict, state),
        # initial_hidden_state(batch_size), state_dict() / load_state_dict() with AtariNet's parameter names
        self.actor_model = (actor_model_fn or (lambda: ActorNet(args.obs_shape, args.num_actions, use_lstm=args.use_lstm)))()
        self.actor_model.share_memory()                                # :58
        self.ring = self.create_buffers(args.obs_shape, args.num_actions)
        self.buffers = self.ring.buffers
        self.rnn_state_buffers = self.create_rnn_state_buffers()
        args.checkpoint_path = os.path.join(args.output_dir, args.project, args.algo_name)
        os.makedirs(args.checkpoint_path, exist_ok=True)
        self._ctx = mp.get_context('fork')
        self._global_step = self._ctx.Value('q', 0)
        # version of the weights the actors currently read: written by the GPU's copy engine (D2H on the publish stream,
        # after the parameter copies of that version), readable from every process (SURVEY.md §8f-4)
        self.weights_version = torch.zeros(1, dtype=torch.int64).share_memory_()
        self.learner: Optional[B200ImpalaLearner] = None
        self._pending_release = collections.deque()          # (copy event, slot indices, free_queue)
        self._tickets = collections.deque()

    # -------------------------------------------------------------------------------------------------
    @property
    def global_step(self) -> int:
        return int(self._global_step.value)

    def hparams(self) -> ImpalaHParams:
        a = self.args
        return ImpalaHParams(rollout_length=a.rollout_length, batch_size=a.batch_size, num_actions=a.num_actions,
                             discounting=a.discounting, baseline_cost=a.baseline_cost, entropy_cost=a.entropy_cost,
                             reward_clipping=a.reward_clipping, max_grad_norm=a.max_grad_norm, learning_rate=a.learning_rate,
                             alpha=a.alpha, momentum=a.momentum, epsilon=a.epsilon, optimizer=a.optimizer, use_lstm=a.use_lstm,
                             lr_schedule=a.lr_schedule, min_learning_rate=a.min_learning_rate,
                             total_frames=a.total_steps)     # total_steps counts frames: global_step += T * B (impala_atari.py:391)

    def create_buffers(self, obs_shape, num_actions) -> TrajectoryRing:
        """impala_atari.py:122-151 -- same keys/dtypes/shapes, slot-contiguous shared memory"""
        return TrajectoryRing(self.args.rollout_length, num_actions, self.args.num_buffers, obs_shape)

    def create_rnn_state_buffers(self) -> List[Tuple[torch.Tensor, ...]]:
        """impala_atari.py:108-120: one initial (h, c) per slot, shared memory; views of ONE block [slot][h|c][2][1][H] so a
        batch's states are gathered with a single index_select before their H2D copy.  () per slot without LSTM."""
        state0 = self.actor_model.initial_hidden_state(batch_size=1)
        if len(state0) == 0:
            self._rnn_block = None
            return [tuple() for _ in range(self.args.num_buffers)]
        shp = tuple(state0[0].shape)                                   # [num_layers, 1, hidden]
        self._rnn_block = torch.zeros(self.args.num_buffers, len(state0), *shp).share_memory_()
        return [tuple(self._rnn_block[m, i] for i in range(len(state0))) for m in range(self.args.num_buffers)]

    # ------------------------------------------------------------------------------------------------- actors
    def get_action(self, actor_index, free_queue, full_queue, actor_model, buffers, rnn_state_buffers) -> None:
        """actor process (impala_atari.py:153-220).  Key collision of the reference (env 'action' vs agent 'action',
        SURVEY.md §0.9) is kept as the reference behaves: the agent's action overwrites the env's."""
        try:
            torch.set_num_threads(1)
            timings = Timings()
            env = self.env_fn()
            env_output = env.reset()
            agent_state = actor_model.initial_hidden_state(batch_size=1)
            agent_output, unused_state = actor_model(env_output, agent_state)
            while True:
                index = free_queue.get()
                if index is None:
                    break
                for key in env_output:
                    buffers[key][index][0, ...] = env_output[key]
                for key in agent_output:
                    buffers[key][index][0, ...] = agent_output[key]
                for i, tensor in enumerate(agent_state):
                    rnn_state_buffers[index][i][...] = tensor
                for t in range(self.args.rollout_length):
                    timings.reset()
                    with torch.no_grad():
                        agent_output, agent_state = actor_model(env_output, agent_state)
                    timings.time('model')
                    env_output = env.step(agent_output['action'])
                    timings.time('step')
                    for key in env_output:
                        buffers[key][index][t + 1, ...] = env_output[key]
                    for key in agent_output:
                        buffers[key][index][t + 1, ...] = agent_output[key]
                    timings.time('write')
                full_queue.put(index)
        except KeyboardInterrupt:
            pass
        except Exception:
            traceback.print_exc()
            raise

    def get_action_batched(self, actor_index, free_queue, full_queue, actor_model, buffers, rnn_state_buffers, num_envs: int) -> None:
        """One actor process driving ``num_envs`` environments with ONE model call per step (SURVEY.md §8f-4: batched actor
        inference, e.g. ``gpu_actor.B200ActorModel`` or any model with the reference's calling convention evaluated at batch N).
        Same slot protocol as ``get_action`` (impala_atari.py:153-220): environment e fills its own trajectory slot."""
        try:
            torch.set_num_threads(1)
            envs = [self.env_fn() for _ in range(num_envs)]
            cat = lambda outs: {k: torch.cat([o[k] for o in outs], dim=1) for k in outs[0]}          # [1, N, ...]
            env_output = cat([e.reset() for e in envs])
            agent_state = actor_model.initial_hidden_state(batch_size=num_envs)
            agent_output, unused_state = actor_model(env_output, agent_state)
            T = self.args.rollout_length
            while True:
                indices = [free_queue.get() for _ in range(num_envs)]
                if any(i is None for i in indices):
                    break
                state = agent_state
                if len(state) and state[0].is_cuda:       # a device-resident state (GPU actor): one D2H per rollout, not one per environment
                    state = torch.stack(state).cpu().unbind(0)
                for e, index in enumerate(indices):
                    for key in env_output:
                        buffers[key][index][0, ...] = env_output[key][0, e]
                    for key in agent_output:
                        buffers[key][index][0, ...] = agent_output[key][0, e]
                    for i, tensor in enumerate(state):
                        rnn_state_buffers[index][i][...] = tensor[:, e:e + 1]
                for t in range(T):
                    with torch.no_grad():
                        agent_output, agent_state = actor_model(env_output, agent_state)
                    env_output = cat([env.step(agent_output['action'][0, e]) for e, env in enumerate(envs)])
                    for e, index in enumerate(indices):
                        for key in env_output:
                            buffers[key][index][t + 1, ...] = env_output[key][0, e]
                        for key in agent_output:
                            buffers[key][index][t + 1, ...] = agent_output[key][0, e]
                for index in indices:
                    full_queue.put(index)
        except KeyboardInterrupt:
            pass
        except Exception:
            traceback.print_exc()
            raise

    # ------------------------------------------------------------------------------------------------- learner
    def _ensure_learner(self):
        if self.learner is not None:
            return
        if not (self.args.use_cuda and torch.cuda.is_available()):
            raise RuntimeError('this ImpalaTrainer needs CUDA (no CPU learner path)')
        if self._adopt is not None:
            hp, want = self._adopt.hp, self.hparams()
            if (hp.rollout_length, hp.batch_size, hp.num_actions, hp.use_lstm) != (want.rollout_length, want.batch_size, want.num_actions, want.use_lstm):
                raise ValueError('the adopted learner was built for another T / B / A / use_lstm')
            self.learner = self._adopt
        else:
            sd = {k: v.detach().clone() for k, v in self.actor_model.state_dict().items()}
            self.learner = B200ImpalaLearner(self.hparams(), init_state_dict=sd, process_group=None)
        self.ring.pin()
        from ...data.feeder import batch_specs, H2D_KEYS
        hp = self.learner.hp
        specs = batch_specs(hp.rollout_length, hp.batch_size, hp.num_actions)
        dev = self.learner.device
        self._copy_stream = torch.cuda.Stream(dev)
        self._publish_stream = torch.cuda.Stream(dev)
        self._dev_batches = [{k: torch.empty(specs[k][0], dtype=specs[k][1], device=dev) for k in H2D_KEYS} for _ in range(2)]
        self._consumed = [None, None]
        self._slot = 0
        self._cur_slot = None
        # slot-level staging: one H2D copy per trajectory slot (all keys), then one unpack kernel
        self._staging = [torch.empty(hp.batch_size, self.ring.slot_bytes, dtype=torch.uint8, device=dev) for _ in range(2)]
        lay = self.ring.layout
        self._slot_off = (ctypes.c_int64 * 6)(*[lay[k][0] for k in ('obs', 'reward', 'done', 'action', 'policy_logits', 'episode_return')])
        if self._rnn_block is not None:          # initial LSTM states of a batch: host gather -> pinned -> device [h|c][2][B][H]
            n_state, (nl, _, hid) = self._rnn_block.shape[1], self._rnn_block.shape[2:]
            self._rnn_host = [torch.zeros(n_state, nl, hp.batch_size, hid).pin_memory() for _ in range(2)]
            self._rnn_dev = [torch.zeros(n_state, nl, hp.batch_size, hid, device=dev) for _ in range(2)]
            self._rnn_copied = [None, None]
        # weight publish: snapshot (device) -> D2H straight into the actors' shared-memory parameters
        self._snapshot = self.learner.flat_params.clone()        # last good weights (the device-side finite guard keeps them)
        self._pub_done = None
        self._version_dev = torch.zeros(1, dtype=torch.int64, device=dev)
        _host_register(self.weights_version)
        self._registered_actor = None
        self._steps_done = 0

    def close(self) -> None:
        """drain the GPU work, unpin the shared host memory and drop the learner (safe to call twice)"""
        if self.learner is None:
            return
        try:
            self.flush()
        finally:
            for t in getattr(self, '_actor_targets', []):
                _host_unregister(t)
            self._actor_targets = []
            self._registered_actor = None
            _host_unregister(self.weights_version)
            self.ring.unpin()
            self.learner.release_graphs()
            self.learner.close()
            self.learner = None

    def __del__(self):
        try:
            self.close()
        except Exception:       # noqa: BLE001 -- interpreter shutdown
            pass

    def _poll_releases(self) -> None:
        """hand slots whose H2D copy has finished back to the actors (never blocks)"""
        while self._pending_release and self._pending_release[0][0].query():
            _, indices, fq = self._pending_release.popleft()
            for m in indices:
                fq.put(m)

    def flush(self) -> None:
        """wait for everything in flight (copies, steps, weight publish) and release every slot"""
        if self.learner is None:
            return
        torch.cuda.synchronize(self.learner.device)
        self._poll_releases()

    def get_batch(self, free_queue, full_queue, buffers=None, rnn_state_buffers=None, timings=None, lock=None):
        """impala_atari.py:222-268: dequeue B slot indices, copy them column-wise into a time-major device batch
        (async, pinned, copy stream); the slots go back to ``free_queue`` once their copies have finished (polled here,
        in ``learn`` and while waiting for trajectories -- the host never waits for the GPU)."""
        self._ensure_learner()
        from ...data.feeder import H2D_KEYS
        from ... import _lib
        buffers = buffers or self.buffers
        timings = timings or Timings()
        self._poll_releases()
        if lock is not None:
            with lock:
                timings.time('lock')
                indices = self._dequeue_batch(full_queue)
        else:
            timings.time('lock')
            indices = self._dequeue_batch(full_queue)
        timings.time('dequeue')
        s = self._slot
        self._slot ^= 1
        dst = self._dev_batches[s]
        sb = self.ring.slot_bytes
        hp = self.learner.hp
        state: Tuple[torch.Tensor, ...] = tuple()
        unpack = False
        with nvtx_range('get_batch'), torch.cuda.stream(self._copy_stream):
            if self._consumed[s] is not None:
                self._copy_stream.wait_event(self._consumed[s])          # the step that read this device batch has finished
            if buffers is self.buffers:       # ring slots: ONE pinned H2D copy per slot, then scatter on the device
                stg = self._staging[s]
                b = 0
                while b < len(indices):                  # runs of consecutive slots travel as ONE copy
                    e = b + 1
                    while e < len(indices) and indices[e] == indices[e - 1] + 1:
                        e += 1
                    m = indices[b]
                    stg[b:e].view(-1).copy_(self.ring.block[m * sb:(m + e - b) * sb], non_blocking=True)
                    b = e
                unpack = True                 # the scatter kernel runs on the LEARNER stream (below): the copy stream stays pure DMA,
                                              # so the next batch's H2D is not queued behind a kernel launch
            else:                             # foreign buffer dict (reference-style lists of tensors): per-key column copies
                for b, m in enumerate(indices):
                    for k in H2D_KEYS:
                        dst[k][:, b].copy_(buffers[k][m], non_blocking=True)
            if self._rnn_block is not None:   # initial_rnn_state = cat over the batch on dim 1 (:252-253)
                rsb = rnn_state_buffers if rnn_state_buffers is not None else self.rnn_state_buffers
                host = self._rnn_host[s]
                if self._rnn_copied[s] is not None:
                    self._rnn_copied[s].synchronize()       # the H2D that last read this pinned buffer (two batches ago) is done
                if rsb is self.rnn_state_buffers:
                    g = self._rnn_block.index_select(0, torch.as_tensor(indices))           # [B][h|c][2][1][H]
                    host.copy_(g.squeeze(3).permute(1, 2, 0, 3))
                else:
                    for i in range(host.shape[0]):
                        host[i].copy_(torch.cat([rsb[m][i] for m in indices], dim=1))
                self._rnn_dev[s].copy_(host, non_blocking=True)
                self._rnn_copied[s] = torch.cuda.Event()
                self._rnn_copied[s].record(self._copy_stream)
                state = tuple(self._rnn_dev[s][i] for i in range(host.shape[0]))
            ev = torch.cuda.Event()
            ev.record(self._copy_stream)
        timings.time('batch')
        self._pending_release.append((ev, indices, free_queue))              # slots stay owned until their copy has finished
        self._poll_releases()
        timings.time('enqueue')
        cur = torch.cuda.current_stream(self.learner.device)
        cur.wait_event(ev)                                                   # device-side wait: the host moves on
        if unpack:
            stg = self._staging[s]
            _lib.check(_lib.lib().srl_unpack_slots(
                stg.data_ptr(), sb, self._slot_off, hp.rollout_length, hp.batch_size, hp.num_actions, dst['obs'].data_ptr(),
                dst['reward'].data_ptr(), dst['done'].data_ptr(), dst['action'].data_ptr(), dst['policy_logits'].data_ptr(),
                dst['episode_return'].data_ptr(), cur.cuda_stream), 'srl_unpack_slots')
        self._cur_slot = s
        timings.time('device')
        return dst, state

    def _dequeue_batch(self, full_queue) -> List[int]:
        """B indices from the full queue: in bulk when the queue offers ``get_many`` (SlotQueue), else one ``get`` each"""
        B = self.args.batch_size
        if not hasattr(full_queue, 'get_many'):
            return [self._dequeue(full_queue) for _ in range(B)]
        out: List[int] = []
        while len(out) < B:
            got = full_queue.get_many(B - len(out), timeout=0.0005)
            out.extend(got)
            if not got:
                self._poll_releases()
                actors = getattr(self, '_actors', None)
                if actors:
                    dead = [p.name for p in actors if not p.is_alive()]
                    if dead:
                        raise RuntimeError(f'actor process(es) exited while the learner was waiting for trajectories: {dead}')
        return out

    def _dequeue(self, full_queue):
        """full_queue.get() that (a) keeps releasing slots whose copies finish meanwhile -- the actors may be waiting for
        exactly those -- and (b) notices dead actors: the reference blocks forever when an actor process has died
        (impala_atari.py:238-241); here a crashed actor surfaces as an error in the learner instead of a hang."""
        actors = getattr(self, '_actors', None)
        if not actors and not self._pending_release:
            return full_queue.get()
        while full_queue.empty():
            self._poll_releases()
            if actors:
                dead = [p.name for p in actors if not p.is_alive()]
                if dead:
                    raise RuntimeError(f'actor process(es) exited while the learner was waiting for trajectories: {dead}')
            time.sleep(0.0002)
        return full_queue.get()

    def learn(self, actor_model, learner_model, batch, initial_rnn_state=(), lock=None) -> Dict[str, Any]:
        """impala_atari.py:270-349.  ``learner_model`` is ignored (the learner state lives in B200ImpalaLearner).
        Returns the stats of step k - ``args.stats_lag`` (the first call(s) return their own step's stats)."""
        self._ensure_learner()
        L = self.learner
        with nvtx_range('learn'):
            ticket = L.learn_async(batch, initial_rnn_state)
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(L.device))
            if self._cur_slot is not None:
                self._consumed[self._cur_slot] = ev
            self._steps_done += 1
            if self._steps_done % max(1, self.args.publish_every) == 0 and not getattr(self, '_publish_rank0_only', False):
                self.publish_weights(actor_model, wait=False)      # data-parallel learners: replicas are identical, rank 0 publishes
        self._tickets.append(ticket)
        self._poll_releases()
        lag = max(0, int(self.args.stats_lag))
        while len(self._tickets) > lag + 1:
            self._tickets.popleft()
        t_wait = time.perf_counter()
        stats = L.result(self._tickets[0])
        self.wait_seconds = getattr(self, 'wait_seconds', 0.0) + (time.perf_counter() - t_wait)     # time blocked on the GPU (diagnostics)
        self._poll_releases()
        if not math.isfinite(stats['total_loss']):          # the device-side guard already kept these weights from the actors
            raise FloatingPointError(f'non-finite learner loss: {stats}')
        if os.environ.get('SRL_CHECK_FINITE'):               # debugging aid: name the first poisoned tensors
            bad_p = [n for n, v in L.params.items() if not bool(torch.isfinite(v).all())]
            bad_g = [n for n, v in L.grads.items() if not bool(torch.isfinite(v).all())]
            if bad_p or bad_g:
                raise FloatingPointError(f'step {L.global_step}: non-finite params {bad_p} grads {bad_g} stats {stats}')
        return stats

    def _register_actor(self, actor_model):
        """pin the actor's shared-memory parameters so the publish D2H writes them directly (no host-side copy)"""
        if self._registered_actor is actor_model:
            return
        sd = actor_model.state_dict()
        missing = [n for n in self.learner.names if n not in sd]
        if missing:
            raise KeyError(f'actor_model.state_dict() lacks {missing}')
        self._actor_targets = []
        self._actor_flat = None
        flat = getattr(actor_model, 'flat_params', None)
        if (isinstance(flat, torch.Tensor) and flat.numel() == self.learner.numel and flat.is_shared() and flat.dtype == torch.float32 and
                all(sd[n].data_ptr() == flat.data_ptr() + 4 * self.learner._off[i] for i, n in enumerate(self.learner.names))):
            _host_register(flat)             # the actor keeps ONE flat buffer in the learner's layout: one D2H copy per publish
            self._actor_flat = flat
            self._actor_targets = [flat]
            self._registered_actor = actor_model
            return
        for n in self.learner.names:
            t = sd[n]
            if tuple(t.shape) != tuple(self.learner.shapes[n]) or t.dtype != torch.float32 or not t.is_contiguous():
                raise ValueError(f'actor parameter {n}: expected contiguous float32 {tuple(self.learner.shapes[n])}')
            if not t.is_shared():
                raise ValueError('actor_model must live in shared memory (actor_model.share_memory())')
            _host_register(t)
            self._actor_targets.append(t)
        self._registered_actor = actor_model

    def publish_weights(self, actor_model, wait: bool = True) -> int:
        """impala_atari.py:348 ``actor_model.load_state_dict(learner_model.state_dict())`` as an asynchronous, versioned
        pipeline: (learner stream) snapshot of the flat fp32 parameters, skipped on the device when the step's loss is not
        finite -> (publish stream) D2H of every tensor into the actors' pinned shared-memory parameters, then the version
        counter.  Actors read lock-free, as in the reference.  Returns the version being published."""
        self._ensure_learner()
        self._register_actor(actor_model)
        L = self.learner
        cur = torch.cuda.current_stream(L.device)
        if self._pub_done is not None:
            cur.wait_event(self._pub_done)                    # the previous publish has read the snapshot
        L.snapshot_params(self._snapshot)
        snap_ev = torch.cuda.Event()
        snap_ev.record(cur)
        version = int(getattr(self, '_version', 0)) + 1
        self._version = version
        with torch.cuda.stream(self._publish_stream):
            self._publish_stream.wait_event(snap_ev)
            if self._actor_flat is not None:
                self._actor_flat.copy_(self._snapshot, non_blocking=True)
            else:
                for i, t in enumerate(self._actor_targets):
                    t.copy_(L._view(self._snapshot, i), non_blocking=True)
            self._version_dev.fill_(version)
            self.weights_version.copy_(self._version_dev, non_blocking=True)
            self._pub_done = torch.cuda.Event()
            self._pub_done.record(self._publish_stream)
        if wait:
            self._pub_done.synchronize()
        return version

    def learn_process(self, threading_id, actor_model, learner_model, free_queue, full_queue, buffers, rnn_state_buffers, lock=None,
                      max_iters: Optional[int] = None):
        """impala_atari.py:351-401.  ``max_iters``: run exactly that many steps (data-parallel learners must agree on the count:
        every step contains a collective) instead of watching the shared ``global_step``."""
        try:
            timings = Timings()
            it = 0
            while (it < max_iters) if max_iters is not None else (self.global_step < self.args.total_steps):
                it += 1
                timings.reset()
                batch, state = self.get_batch(free_queue, full_queue, buffers, rnn_state_buffers, timings, lock)
                stats = self.learn(actor_model, learner_model, batch, state, lock)
                timings.time('learn')
                with self._global_step.get_lock():
                    self._global_step.value += self.args.rollout_length * self.args.batch_size   # :391
                self.last_stats = stats
            self.flush()
            self.timings = timings
        except KeyboardInterrupt:
            return
        except Exception:
            traceback.print_exc()
            raise

    def _learner_worker(self, rank, world, port, free_queue, full_queue, deq_lock, iters, result_q):
        """one data-parallel learner process (forked before any CUDA use): GPU `rank`, NCCL group over the `world` learners, its
        batch = whichever ``batch_size`` slots of the SHARED ring it dequeues (the columns of a batch are exchangeable, so any
        disjoint slot sets form a valid sharding of the global batch of batch_size * world columns; SURVEY.md §8e)"""
        try:
            import sys
            import torch.distributed as dist
            from ...utils.numa import bind_to_gpu_numa
            say = lambda msg: (sys.stderr.write(f'[learner {rank}] {msg}\n'), sys.stderr.flush())
            torch.set_num_threads(1)           # forked child: the parent's OpenMP pool does not exist here (a parallel CPU op would hang)
            torch.cuda.set_device(rank)
            bind_to_gpu_numa(rank)
            os.environ['MASTER_ADDR'], os.environ['MASTER_PORT'] = '127.0.0.1', str(port)
            say('init_process_group')
            dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
            say('process group up; building the learner')
            self._ensure_learner()
            say(f'learner ready (gradient path: {getattr(self.learner, "dp_path", "nccl")}); {iters} steps')
            self._publish_rank0_only = rank != 0
            self.learn_process(rank, self.actor_model, None, free_queue, full_queue, self.buffers, self.rnn_state_buffers, deq_lock, max_iters=iters)
            self.flush()
            chk = int(self.learner.flat_params.view(torch.int32).to(torch.int64).sum())
            result_q.put((rank, dict(getattr(self, 'last_stats', {})), chk, getattr(self.learner, 'dp_path', 'nccl')))
            if rank == 0:
                self.save_checkpoint(os.path.join(self.args.output_dir, self.args.project, 'model.tar'))
            self.learner.release_graphs()
            dist.barrier(device_ids=[rank])
            os._exit(0)                    # skip NCCL teardown at interpreter exit (seen to hang)
        except Exception:
            traceback.print_exc()
            result_q.put((rank, None, None, None))
            os._exit(1)

    def _train_multi_learner(self) -> Dict[str, Any]:
        """``num_learners`` > 1 (impala_atari.py:420-456 starts that many learner threads on one device): here one learner PROCESS per
        GPU, all dequeuing from the same trajectory ring, gradients SUM-reduced inside the step (NVLS / peer memory / NCCL)."""
        from ...data.slot_queue import SlotQueue
        import socket
        a = self.args
        world = a.num_learners
        free_queue, full_queue = SlotQueue(2 * a.num_buffers + a.num_actors + 4, self._ctx), SlotQueue(2 * a.num_buffers + 4, self._ctx)
        sock = socket.socket(); sock.bind(('127.0.0.1', 0)); port = sock.getsockname()[1]; sock.close()
        per_step = a.rollout_length * a.batch_size * world
        iters = (a.total_steps + per_step - 1) // per_step
        deq_lock, result_q = self._ctx.Lock(), self._ctx.SimpleQueue()
        actors = [self._ctx.Process(target=self.get_action, name=f'actor-process-{i}',
                                    args=(i, free_queue, full_queue, self.actor_model, self.buffers, self.rnn_state_buffers)) for i in range(a.num_actors)]
        learners = [self._ctx.Process(target=self._learner_worker, name=f'learner-process-{r}',
                                      args=(r, world, port, free_queue, full_queue, deq_lock, iters, result_q)) for r in range(world)]
        for p in actors + learners:
            p.start()
        for m in range(a.num_buffers):
            free_queue.put(m)
        t0 = timeit.default_timer()
        results = []
        limit = float(os.environ.get('SRL_LEARNER_TIMEOUT_S', '3600'))
        while len(results) < world:             # a learner that died without reporting must not hang the trainer
            if not result_q.empty():
                results.append(result_q.get())
                continue
            dead = [p.name for p in learners if not p.is_alive() and p.exitcode not in (0, None)]
            if dead or timeit.default_timer() - t0 > limit:
                for p in learners + actors:
                    if p.is_alive():
                        p.terminate()
                raise RuntimeError(f'learner processes failed or timed out after {timeit.default_timer() - t0:.0f} s (dead: {dead}, reported: {len(results)}/{world})')
            time.sleep(0.01)
        dt = timeit.default_timer() - t0
        for p in learners:
            p.join(timeout=30)
        for _ in range(a.num_actors):
            free_queue.put(None)
        for p in actors:
            p.join(timeout=2)
            if p.is_alive():
                p.terminate()
        if any(r[1] is None for r in results):
            raise RuntimeError('a learner process failed (see its traceback above)')
        results.sort(key=lambda r: r[0])
        return dict(steps=self.global_step, sps=self.global_step / max(dt, 1e-9), weights_version=int(self.weights_version[0]), learners=world,
                    replica_checksums=[r[2] for r in results], grad_path=results[0][3], **results[0][1])

    def train(self, log_every_s: float = 5.0, learner_in_process: bool = True) -> Dict[str, Any]:
        """impala_atari.py:403-494.  Actors are forked BEFORE CUDA is touched; with ``num_learners == 1`` the learner loop runs in this
        process; with ``num_learners > 1`` one learner process per GPU is forked as well (data parallel over a shared ring) --
        alternatively launch one trainer per rank with torchrun (each with its own actors and ring)."""
        if self.args.num_learners > 1:
            return self._train_multi_learner()
        from ...data.slot_queue import SlotQueue          # mp.SimpleQueue's put/get/empty over a shared-memory index ring
        free_queue, full_queue = SlotQueue(2 * self.args.num_buffers + self.args.num_actors + 4, self._ctx), SlotQueue(2 * self.args.num_buffers + 4, self._ctx)
        actors = []
        for i in range(self.args.num_actors):
            p = self._ctx.Process(target=self.get_action, name=f'actor-process-{i}',
                                  args=(i, free_queue, full_queue, self.actor_model, self.buffers, self.rnn_state_buffers))
            p.start()
            actors.append(p)
        self._actors = actors
        for m in range(self.args.num_buffers):
            free_queue.put(m)
        timer = timeit.default_timer
        t0, s0 = timer(), self.global_step
        checkpoint_path = os.path.join(self.args.output_dir, self.args.project, 'model.tar')
        try:
            self.learn_process(0, self.actor_model, None, free_queue, full_queue, self.buffers, self.rnn_state_buffers, None)
        finally:
            self._actors = None
            self.flush()
            for _ in range(self.args.num_actors):
                free_queue.put(None)
            for p in actors:
                p.join(timeout=2)
                if p.is_alive():
                    p.terminate()
        sps = (self.global_step - s0) / max(timer() - t0, 1e-9)
        self.save_checkpoint(checkpoint_path)
        return dict(steps=self.global_step, sps=sps, weights_version=int(self.weights_version[0]), **getattr(self, 'last_stats', {}))

    def save_checkpoint(self, checkpoint_path: str) -> None:
        """impala_atari.py:496-515 (same dict keys; the optimizer state is in torch.optim's own layout)"""
        if self.args.disable_checkpoint:
            return
        os.makedirs(os.path.dirname(checkpoint_path), exist_ok=True)
        if self.learner is not None:
            model = {k: v.cpu() for k, v in self.learner.state_dict().items()}
            opt = self.learner.optimizer_state_dict()
        else:
            model = {k: v.detach().clone() for k, v in self.actor_model.state_dict().items()}
            opt = {}
        torch.save({'model_state_dict': model, 'optimizer_state_dict': opt,
                    'hparam': {k: v for k, v in vars(self.args).items()}}, checkpoint_path)
