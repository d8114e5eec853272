"""CPU oracle of the GPU prioritized replay memory's storage (GpuPrioritizedReplayBuffer, csrc/replay.cu).  TEST INFRASTRUCTURE ONLY.

Restates, in numpy, the storage half of the reference's
  scalerl/data/replay_buffer.py:197-218 (MultiStepReplayBuffer.save_to_memory_vect_envs: one n-deep window per env; no transition
                                        until every window is full; then one n-step transition per env, in env order)
  scalerl/data/replay_buffer.py:230-273 (_get_n_step_info: state and action of the oldest step; reward r0 + r1 * gamma**1 + ...
                                        in float32, numpy's rounding; stop at the first done, whose step gives next_state and done)
  scalerl/data/replay_buffer.py:319-323 (PrioritizedReplayBuffer._add: the transition takes tree leaf tree_ptr)
The tree half (priorities, sampling, weights) is oracle/per_oracle.py.  Transitions are kept by RING SLOT = tree leaf.  Reference
defects this does not inherit:
  * once the memory is full the reference's deque index no longer equals the tree index (replay_buffer.py:41-44 append to a
    deque(maxlen) that drops its left end, vs :319-323 tree_ptr wrapping): ``sample`` reads ``self.memory[i]`` for a tree leaf i, so
    it returns a different transition than the one whose priority it sampled.  Here slot i is leaf i at every fill level; the
    reference's deque entry i is slot (tree_ptr - len + i) mod memory_size.
  * MultiStepReplayBuffer asserts the field names 'next_state' and 'done' (replay_buffer.py:160-169), which OffPolicyTrainer's own
    'obs' / 'next_obs' fields fail (trainer/off_policy.py:81).  The fields here are positional.
Pinned by tests/golden/replay_cases.npz, written by oracle/make_replay_golden.py from the reference's own PrioritizedReplayBuffer.
"""
from collections import deque

import numpy as np

# (memory_size, num_envs, n_step, done_rate, vector steps, seed): n_step in {1, 3, 5}, E in {1, 4}, done rates 0 and 0.3, memories that
# wrap (7 with E = 1; 10 with E = 4, not a multiple of E) and one that does not fill (64)
CASES = [(m, e, n, dr, steps, 100 * n + 10 * e + int(dr * 10))
         for e, sizes, steps in ((1, (7,), 15), (4, (10, 64), 9))
         for m in sizes for n in (1, 3, 5) for dr in (0.0, 0.3)]
GAMMA = 0.99


def case_inputs(num_envs, steps, done_rate, seed):
    """the raw vector steps of a case: action int64 [steps, E], reward float32 [steps, E], done uint8 [steps, E].  The state of step t for
    env e is identified by (t, e), as is its next_state."""
    rng = np.random.RandomState(seed)
    action = rng.randint(0, 18, size=(steps, num_envs)).astype(np.int64)
    reward = rng.randn(steps, num_envs).astype(np.float32)
    done = (rng.rand(steps, num_envs) < done_rate).astype(np.uint8)
    return action, reward, done


def fold(window, gamma):
    """_get_n_step_info over one env's window [(state, action, reward, next_state, done), ...], oldest first"""
    state, action, reward, next_state, done = window[0]
    reward, done = np.float32(reward), np.uint8(done)
    for k, (_, _, r, ns, d) in enumerate(list(window)[1:], start=1):
        if done:
            break
        reward = np.float32(reward + np.float32(np.float32(r) * np.float32(gamma ** k)))
        next_state, done = ns, np.uint8(d)
    return state, action, reward, next_state, done


class ReplayOracle:
    def __init__(self, memory_size, num_envs, n_step=1, gamma=0.99):
        self.memory_size, self.num_envs, self.n_step, self.gamma = memory_size, num_envs, n_step, gamma
        self.windows = [deque(maxlen=n_step) for _ in range(num_envs)]
        self.slots = [None] * memory_size          # ring slot -> (state, action, reward, next_state, done)
        self.tree_ptr, self.size = 0, 0

    def add(self, state, action, reward, next_state, done):
        """one vector step: sequences of num_envs entries each"""
        for e, w in enumerate(self.windows):
            w.append((state[e], action[e], reward[e], next_state[e], done[e]))
        if any(len(w) < self.n_step for w in self.windows):
            return
        for w in self.windows:
            self.slots[self.tree_ptr] = fold(w, self.gamma)
            self.tree_ptr = (self.tree_ptr + 1) % self.memory_size
            self.size = min(self.size + 1, self.memory_size)

    def deque_to_slot(self, i):
        """the ring slot of the reference's deque entry i"""
        return (self.tree_ptr - self.size + i) % self.memory_size


def run_case(memory_size, num_envs, n_step, done_rate, steps, seed, gamma=GAMMA):
    """the oracle over a case -> per ring slot [size]: state step, state env, action, reward bits (uint32), next_state step, done"""
    action, reward, done = case_inputs(num_envs, steps, done_rate, seed)
    o = ReplayOracle(memory_size, num_envs, n_step, gamma)
    for t in range(steps):
        ids = [(t, e) for e in range(num_envs)]
        o.add(ids, action[t], reward[t], ids, done[t])
    return slot_table(o.slots[:o.size]), o.tree_ptr


def slot_table(slots):
    return {'s_step': np.array([s[0][0] for s in slots], dtype=np.int64), 's_env': np.array([s[0][1] for s in slots], dtype=np.int64),
            'action': np.array([s[1] for s in slots], dtype=np.int64),
            'reward_bits': np.array([s[2] for s in slots], dtype=np.float32).view(np.uint32),
            'ns_step': np.array([s[3][0] for s in slots], dtype=np.int64), 'done': np.array([s[4] for s in slots], dtype=np.uint8)}
