"""Generate tests/golden/replay_cases.npz by running the REFERENCE's own PrioritizedReplayBuffer (scalerl/data/replay_buffer.py:276-381)
with field names ['state', 'action', 'reward', 'next_state', 'done'].  Run where the reference tree is present (SRL_REFERENCE_ROOT):

    python oracle/make_replay_golden.py

States are tiny int arrays [step, env], so the fixture stores, per ring slot, which raw step and env a transition's state and
next_state came from, its action, the bits of its float32 reward and its done.  The reference's deque entry i is mapped to ring slot
(tree_ptr - len + i) mod memory_size (oracle/replay_oracle.py says why the two differ once the memory is full).  Inputs are regenerated
from seeds by oracle.replay_oracle.case_inputs.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from oracle import replay_oracle as O  # noqa: E402

sys.path.insert(0, os.environ.get('SRL_REFERENCE_ROOT', '/root/reference'))
from scalerl.data.replay_buffer import PrioritizedReplayBuffer  # noqa: E402


def main():
    out = {}
    for ci, (M, E, n, dr, steps, seed) in enumerate(O.CASES):
        action, reward, done = O.case_inputs(E, steps, dr, seed)
        buf = PrioritizedReplayBuffer(M, ['state', 'action', 'reward', 'next_state', 'done'], E, alpha=0.6, n_step=n, gamma=O.GAMMA)
        for t in range(steps):
            ids = np.array([[t, e] for e in range(E)], dtype=np.int64)
            if E == 1:       # the single-env form (save_to_memory_single_env)
                buf.save_to_memory(ids[0], action[t, 0], reward[t, 0], ids[0], done[t, 0])
            else:
                buf.save_to_memory(ids, action[t], reward[t], ids, done[t], is_vectorised=True)
        size = len(buf)
        slots = [None] * size
        for i, tr in enumerate(buf.memory):
            slot = (buf.tree_ptr - size + i) % M
            slots[slot] = ((int(tr.state[0]), int(tr.state[1])), int(np.asarray(tr.action).reshape(-1)[0]),
                           np.float32(np.asarray(tr.reward).reshape(-1)[0]), (int(tr.next_state[0]), int(tr.next_state[1])),
                           int(np.asarray(tr.done).reshape(-1)[0]))
        for k, v in O.slot_table(slots).items():
            out[f'c{ci}_{k}'] = v
        out[f'c{ci}_meta'] = np.array([M, E, n, dr, steps, seed, size, buf.tree_ptr], dtype=np.float64)
    np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'replay_cases.npz'), **out)
    print('wrote replay_cases:', len(O.CASES), 'cases')


if __name__ == '__main__':
    main()
