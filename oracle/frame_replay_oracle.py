"""CPU oracle of the frame replay memory (GpuFrameReplayBuffer, csrc/frame_replay.cu).  TEST INFRASTRUCTURE ONLY.

ReplayOracle's ring and fold (oracle/replay_oracle.py, pinned to the reference's PrioritizedReplayBuffer) over frame handles instead of
frame stacks, with the memory's frame pool, its dedup rule and its retirement rule restated in numpy:
  * pool: frame_capacity (F) frames; the frame of sequence number s lives at s mod F.
  * dedup, per env, frames in the order state 0..3, next_state 0..3: a frame equal (byte for byte) to an earlier frame of the same call
    takes that frame's handle; else one equal to the env's previous next_state frames, newest first, takes its handle if
    s >= head + 8 E n_step - F (it outlives the step's stay in the window); else it is new.  New frames are numbered from head in env
    order, then in frame order.
  * retirement: before the new frames are written, every stored slot whose oldest handle is below head_after - F retires, once; a
    slot the add's fold then writes is live again.
The Atari-like stream (``atari_stream``) is shared by the CPU and GPU tests and tools/bench_frame_replay.py: per env, an episode starts
with the reset frame repeated 4 times (FrameStack.reset), each step shifts in one new frame, and a done either resets (a new episode) or
is a lost life (the stack continues).
"""
import numpy as np

from .replay_oracle import ReplayOracle

FRAME = (84, 84)


def default_frame_capacity(memory_size, num_envs, n_step):
    return memory_size + memory_size // 8 + 8 * num_envs * (n_step + 4)


class FrameReplayOracle(ReplayOracle):
    def __init__(self, memory_size, num_envs, n_step=1, gamma=0.99, frame_capacity=None):
        super().__init__(memory_size, num_envs, n_step, gamma)
        self.F = default_frame_capacity(memory_size, num_envs, n_step) if frame_capacity is None else frame_capacity
        assert self.F >= 8 * num_envs * (n_step + 1)
        self.pool = np.zeros((self.F,) + FRAME, np.uint8)
        self.head = 0                               # frames written since creation
        self.oldest = {}                            # ring slot -> its oldest handle
        self.retired_slots = set()
        self.retired = 0                            # slots retired since creation (each retirement counted)

    def _dedup(self, e, frames):
        """env e's 8 incoming frames -> handles (int: reused, ('new', k): its k-th new frame) and the new frames"""
        E, n = self.num_envs, self.n_step
        prev = self.windows[e][-1][3] if self.windows[e] else None
        keep_from = self.head + 8 * E * n - self.F
        hs, new = [], []
        for j, x in enumerate(frames):
            h = next((hs[c] for c in range(j) if np.array_equal(frames[c], x)), None)
            if h is None and prev is not None:
                h = next((s for s in reversed(prev) if s >= keep_from and np.array_equal(self.pool[s % self.F], x)), None)
            if h is None:
                h = ('new', len(new))
                new.append(x)
            hs.append(h)
        return hs, new

    def add(self, state, action, reward, next_state, done):
        """one vector step: state / next_state u8 [E, 4, 84, 84], action, reward, done [E]"""
        per_env = [self._dedup(e, list(state[e]) + list(next_state[e])) for e in range(self.num_envs)]
        handles, base = [], self.head
        for hs, new in per_env:
            handles.append(tuple(h if isinstance(h, (int, np.integer)) else base + h[1] for h in hs))
            base += len(new)
        limit = base - self.F
        for slot, lo in self.oldest.items():
            if lo < limit and slot not in self.retired_slots:
                self.retired_slots.add(slot)
                self.retired += 1
        for hs, new in per_env:
            for k, x in enumerate(new):
                self.pool[(self.head + k) % self.F] = x
            self.head += len(new)
        ptr = self.tree_ptr
        super().add([h[:4] for h in handles], action, reward, [h[4:] for h in handles], done)
        if all(len(w) == self.n_step for w in self.windows):
            for e in range(self.num_envs):
                slot = (ptr + e) % self.memory_size
                s, _, _, ns, _ = self.slots[slot]
                self.oldest[slot] = min(s + ns)
                self.retired_slots.discard(slot)

    def stack(self, handles):
        return np.stack([self.pool[h % self.F] for h in handles])

    def gather(self, slot):
        """(state, action, reward, next_state, done) of a ring slot, the stacks rebuilt from the pool"""
        s, a, r, ns, d = self.slots[slot]
        return self.stack(s), a, r, self.stack(ns), d


def atari_stream(num_envs, steps, seed, done=None, done_rate=0.05, reset_rate=0.5):
    """an Atari-like stream of frame indices -> (state_idx, next_idx int64 [steps, E, 4], done uint8 [steps, E], frames per env K): stack
    rows are indices into each env's own sequence of K frames.  ``done`` (uint8 [steps, E]) may be given; a done resets with probability
    ``reset_rate``, else it is a lost life and the stack continues."""
    rng = np.random.RandomState(seed)
    if done is None:
        done = (rng.rand(steps, num_envs) < done_rate).astype(np.uint8)
    state_idx = np.zeros((steps, num_envs, 4), np.int64)
    next_idx = np.zeros((steps, num_envs, 4), np.int64)
    K = 0
    for e in range(num_envs):
        nxt, stack = 0, None
        for t in range(steps):
            if stack is None:                       # FrameStack.reset: the reset observation 4 times
                stack, nxt = [nxt] * 4, nxt + 1
            state_idx[t, e] = stack
            stack = stack[1:] + [nxt]
            nxt += 1
            next_idx[t, e] = stack
            if done[t, e] and rng.rand() < reset_rate:
                stack = None
        K = max(K, nxt)
    return state_idx, next_idx, done.astype(np.uint8), K


def stream_frames(num_envs, K, seed):
    """K distinct random frames per env, u8 [E, K, 84, 84]"""
    return np.random.RandomState(seed).randint(0, 256, size=(num_envs, K) + FRAME).astype(np.uint8)


def stream_stacks(frames, idx):
    """the stacks of one vector step: frames [E, K, 84, 84], idx [E, 4] -> u8 [E, 4, 84, 84]"""
    return frames[np.arange(frames.shape[0])[:, None], idx]


def expected_new_frames(state_idx):
    """frames a pool that never ages a frame out stores for an Atari-like stream: one per env step, plus one per episode start"""
    starts = np.all(state_idx == state_idx[..., :1], axis=-1)
    return int(state_idx.shape[0] * state_idx.shape[1] + starts.sum())
