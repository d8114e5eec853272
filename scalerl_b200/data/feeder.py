"""Host -> device batch feeder: the GPU replacement of the tail of ImpalaTrainer.get_batch
(/root/reference scalerl/algorithms/impala/impala_atari.py:259-265, a synchronous pageable ``.to(device)``).

Time-major pinned host batches (the reference's ``torch.stack(..., dim=1)`` result, keys of
impala_atari.py:122-151) are copied on a dedicated copy stream into one of ``depth`` device slots while the
previous slot is being learned from; per-slot CUDA events order copy -> learn -> reuse, so the host buffer may be
refilled by actors as soon as ``copied(slot)`` fires (the ownership rule of SURVEY.md §8b).  The step result
(4 loss scalars + grad norm) is read back every step into pinned memory, one step behind the launch front.
"""
from typing import Dict, List, Optional

import torch

H2D_KEYS = ('obs', 'reward', 'done', 'action', 'policy_logits', 'episode_return')


def batch_specs(T: int, B: int, A: int):
    """shapes/dtypes of one [T+1, B] trajectory batch (create_buffers, impala_atari.py:135-147)"""
    return {
        'obs': ((T + 1, B, 4, 84, 84), torch.uint8), 'reward': ((T + 1, B), torch.float32), 'done': ((T + 1, B), torch.bool),
        'last_action': ((T + 1, B), torch.int64), 'action': ((T + 1, B), torch.int64),
        'episode_return': ((T + 1, B), torch.float32), 'episode_step': ((T + 1, B), torch.int32),
        'policy_logits': ((T + 1, B, A), torch.float32), 'baseline': ((T + 1, B), torch.float32)}


def pinned_batch(T: int, B: int, A: int, keys=H2D_KEYS) -> Dict[str, torch.Tensor]:
    specs = batch_specs(T, B, A)
    return {k: torch.empty(specs[k][0], dtype=specs[k][1]).pin_memory() for k in keys}


class HostBatchFeeder:
    def __init__(self, learner, depth: int = 2):
        self.learner = learner
        hp = learner.hp
        self.dev = learner.device
        specs = batch_specs(hp.rollout_length, hp.batch_size, hp.num_actions)
        self.depth = depth
        with torch.cuda.device(self.dev):
            self.copy_stream = torch.cuda.Stream(self.dev)
            self.slots: List[Dict[str, torch.Tensor]] = [
                {k: torch.empty(specs[k][0], dtype=specs[k][1], device=self.dev) for k in H2D_KEYS} for _ in range(depth)]
            self.ready = [torch.cuda.Event() for _ in range(depth)]      # H2D of slot finished
            self.consumed = [torch.cuda.Event() for _ in range(depth)]   # learn on slot finished
            self.result_host = [torch.zeros(8, dtype=torch.float32).pin_memory() for _ in range(depth)]
            self.result_ev = [torch.cuda.Event() for _ in range(depth)]
        self._submitted = 0
        self._learned = 0
        self._used = [False] * depth
        self.h2d_bytes = sum(self.slots[0][k].numel() * self.slots[0][k].element_size() for k in H2D_KEYS)
        self.d2h_bytes = 6 * 4

    def submit(self, host_batch: Dict[str, torch.Tensor]) -> int:
        """enqueue the async H2D of one pinned batch; returns the slot"""
        if self._submitted - self._learned >= self.depth:
            raise RuntimeError('feeder: all device slots are in flight; call learn() first')
        s = self._submitted % self.depth
        with torch.cuda.stream(self.copy_stream):
            if self._used[s]:
                self.copy_stream.wait_event(self.consumed[s])
            for k in H2D_KEYS:
                self.slots[s][k].copy_(host_batch[k], non_blocking=True)
            self.ready[s].record(self.copy_stream)
        self._used[s] = True
        self._submitted += 1
        return s

    def copied(self, slot: int) -> bool:
        """True once the H2D of `slot` finished (the host buffer may be recycled to the free queue)"""
        return self.ready[slot].query()

    def learn(self) -> int:
        """run one learner step on the oldest submitted slot (no host sync); returns the slot"""
        if self._learned >= self._submitted:
            raise RuntimeError('feeder: nothing submitted')
        s = self._learned % self.depth
        cur = torch.cuda.current_stream(self.dev)
        cur.wait_event(self.ready[s])
        L = self.learner
        L.learn(self.slots[s], sync_stats=False)
        self.consumed[s].record(cur)
        self.result_host[s][:4].copy_(L._losses, non_blocking=True)
        self.result_host[s][4:6].copy_(L._coef[:2], non_blocking=True)      # grad norm, clip coefficient
        self.result_ev[s].record(cur)
        self._learned += 1
        return s

    def result(self, slot: int) -> Dict[str, float]:
        """block until the step that used `slot` finished and return its stats (reference stat keys)"""
        self.result_ev[slot].synchronize()
        h = self.result_host[slot]
        return {'pg_loss': float(h[0]), 'baseline_loss': float(h[1]), 'entropy_loss': float(h[2]), 'total_loss': float(h[3]),
                'grad_norm': float(h[4])}
