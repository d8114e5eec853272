"""The frame replay memory (GpuFrameReplayBuffer) against the stack memory (GpuPrioritizedReplayBuffer) on an Atari-like stream
(oracle/frame_replay_oracle.py: one new frame per env step, resets that repeat the reset frame 4 times, lost lives that continue the
stack), at tools/bench_replay.py's M = 65,536, E = 64, A = 18, n_step = 3.  Prints, with the card's name and power limit:
  * bytes per transition of each memory, computed from its allocation layout (not measured);
  * save_to_memory env steps/s of each memory (CUDA inputs), filling it from empty;
  * per batch size, the gather kernel's time over CUDA events and its bandwidth (4 x 28,224 B per transition for both memories: the
    two stacks read and written) against the H100 SXM's 3.35 TB/s, and learn_from learner steps/s of each memory in alternating rounds.

    python tools/bench_frame_replay.py [--rounds 5] [--steps 50] [--batches 32,512]
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import frame_replay_oracle as FO  # noqa: E402
from scalerl_b200.algorithms.apex import ApexHParams, B200ApexLearner  # noqa: E402
from scalerl_b200.data.replay_memory import GpuFrameReplayBuffer, GpuPrioritizedReplayBuffer  # noqa: E402
from tools.bench_apex import card, timed  # noqa: E402

M, E, A, N_STEP = 65536, 64, 18, 3
HBM_BYTES_PER_S = 3.35e12
ROW = 4 * 84 * 84


def bytes_per_transition(mem):
    """the ring's bytes per slot plus, for the frame memory, its pool over memory_size (the layouts of csrc/replay.cu and
    csrc/frame_replay.cu; the staging window and the trees are left out)"""
    if isinstance(mem, GpuFrameReplayBuffer):
        slot = 8 * 8 + 8 + 8 + 4 + 1 + 1 + 8      # handles, oldest, action, reward, done, retired mask, retire list
        return slot + mem.frame_capacity * 84 * 84 / mem.memory_size
    return 2 * ROW + 8 + 4 + 1


def stream(steps, seed=0):
    """the Atari-like stream's steps as CUDA tensors"""
    si, ni, done, K = FO.atari_stream(E, steps, seed)
    g = torch.Generator(device='cuda').manual_seed(seed)
    frames = torch.randint(0, 256, (E, K, 84, 84), dtype=torch.uint8, device='cuda', generator=g)
    rows = torch.arange(E, device='cuda')[:, None]
    si, ni = torch.from_numpy(si).cuda(), torch.from_numpy(ni).cuda()
    return [(frames[rows, si[t]], torch.randint(0, A, (E,), device='cuda', generator=g), torch.randn(E, device='cuda', generator=g),
             frames[rows, ni[t]], torch.from_numpy(done[t]).cuda()) for t in range(steps)]


def gather_bandwidth(mem, B, reps=50):
    idxs = torch.randint(0, len(mem), (B,), device='cuda')
    out = mem._outputs(B)
    args = (mem._h, idxs.data_ptr(), B, *(t.data_ptr() for t in out))
    run = lambda: mem._fn('gather')(*args, mem._stream())
    run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    s = e0.elapsed_time(e1) / 1e3 / reps
    gbs = 4 * ROW * B / s
    return {'us': s * 1e6, 'GB_per_s': gbs / 1e9, 'fraction_of_3.35TB_per_s': gbs / HBM_BYTES_PER_S}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--batches', default='32,512')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_frame_replay.py measures on a CUDA device; none is present')
    name = card()
    steps = stream(M // E + N_STEP)
    mems = {'stack': GpuPrioritizedReplayBuffer(M, E, n_step=N_STEP, gamma=0.99),
            'frame': GpuFrameReplayBuffer(M, E, n_step=N_STEP, gamma=0.99)}
    fill = {}
    for k, mem in mems.items():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for s in steps:
            mem.save_to_memory(*s, is_vectorised=True)
        torch.cuda.synchronize()
        fill[k] = len(steps) / (time.perf_counter() - t0)
    fm = mems['frame']
    head = {'card': name, 'memory_size': M, 'num_envs': E, 'n_step': N_STEP, 'frame_capacity': fm.frame_capacity,
            'frames_allocated': fm.frames_allocated(), 'retired': fm.retired(),
            'bytes_per_transition_computed': {k: bytes_per_transition(m) for k, m in mems.items()},
            'save_to_memory_env_steps_per_s': fill}
    print(json.dumps(head), flush=True)
    for B in (int(x) for x in a.batches.split(',')):
        hp = lambda: ApexHParams(batch_size=B, num_actions=A, gamma=0.99 ** N_STEP, double_dqn=True)
        learners = {k: B200ApexLearner(hp()) for k in mems}
        variants = {k: (lambda L=learners[k], m=mems[k]: L.learn_from(m, beta=0.4, sync_stats=False)) for k in mems}
        for fn in variants.values():           # the first call runs eagerly, the second captures
            for _ in range(3):
                fn()
        rates = {k: [] for k in variants}
        for _ in range(a.rounds):
            for k, fn in variants.items():
                rates[k].append(timed(fn, a.steps))
        out = {'card': name, 'B': B, 'A': A, 'memory_size': M, 'rounds': a.rounds, 'steps_per_round': a.steps}
        for k, r in rates.items():
            r = sorted(r)
            out[f'learn_from_{k}'] = {'steps_per_s_median': r[len(r) // 2], 'steps_per_s_range': [r[0], r[-1]]}
        out['frame_over_stack_learn_from'] = out['learn_from_frame']['steps_per_s_median'] / out['learn_from_stack']['steps_per_s_median']
        out['gather_kernel'] = {k: gather_bandwidth(m, B) for k, m in mems.items()}
        out['frame_over_stack_gather_GB_per_s'] = out['gather_kernel']['frame']['GB_per_s'] / out['gather_kernel']['stack']['GB_per_s']
        print(json.dumps(out), flush=True)
        for L in learners.values():
            L.release_graphs()
            L.close()


if __name__ == '__main__':
    main()
