"""The GPU prioritized replay memory on the Ape-X learner: learner steps/s of three ways to feed B200ApexLearner from a prioritized
memory of M = 65,536 transitions (A = 18, captured, bf16), rounds alternating between them:
  * learn_from   -- GpuPrioritizedReplayBuffer + learn_from: sample, gather, step and priorities as one captured graph;
  * caller       -- INTEGRATION.md §2b's former caller pattern: GpuPrioritizedSampler.sample, two copy_ and five index_select gathers
                    from caller-owned device storage into fixed buffers (eager), then the captured learn(..., idxs, sampler);
  * learn_fixed  -- learn on pre-gathered fixed buffers with the same sampler (no sampling, no gather): the upper bound.
It also times save_to_memory (E = 64 envs, CUDA inputs) in env steps/s and the gather kernel alone with CUDA events, with its
achieved bandwidth (4 x 28,224 B per transition: read and write two frame stacks) against the H100 SXM's 3.35 TB/s.  Prints the
card's name and power limit, one JSON line per batch size.

    python tools/bench_replay.py [--rounds 5] [--steps 50] [--batches 32,512]
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scalerl_b200.algorithms.apex import ApexHParams, B200ApexLearner  # noqa: E402
from scalerl_b200.data.per_sampler import GpuPrioritizedSampler  # noqa: E402
from scalerl_b200.data.replay_memory import GpuPrioritizedReplayBuffer  # noqa: E402
from tools.bench_apex import card, timed  # noqa: E402

M, E, A = 65536, 64, 18
HBM_BYTES_PER_S = 3.35e12
ROW = 4 * 84 * 84


def env_step(g):
    return (torch.randint(0, 256, (E, 4, 84, 84), dtype=torch.uint8, device='cuda', generator=g), torch.randint(0, A, (E,), device='cuda', generator=g),
            torch.randn(E, device='cuda', generator=g), torch.randint(0, 256, (E, 4, 84, 84), dtype=torch.uint8, device='cuda', generator=g),
            torch.rand(E, device='cuda', generator=g) < 0.05)


class CallerPattern:
    """the sampler, hand-kept storage indexed like its leaves, and fixed input buffers for the captured learn"""

    def __init__(self, L, B, g):
        self.L, self.B = L, B
        self.S = GpuPrioritizedSampler(M)
        self.S.add(M)
        self.store = (torch.randint(0, 256, (M, 4, 84, 84), dtype=torch.uint8, device='cuda', generator=g), torch.randint(0, A, (M,), device='cuda', generator=g),
                      torch.randn(M, device='cuda', generator=g), torch.randint(0, 256, (M, 4, 84, 84), dtype=torch.uint8, device='cuda', generator=g),
                      (torch.rand(M, device='cuda', generator=g) < 0.05).to(torch.uint8))
        self.inputs = tuple(torch.empty((B,) + t.shape[1:], dtype=t.dtype, device='cuda') for t in self.store)
        self.idxs, self.weights = torch.empty(B, dtype=torch.int64, device='cuda'), torch.empty(B, device='cuda')

    def __call__(self):
        i, w = self.S.sample(self.B, beta=0.4)
        self.idxs.copy_(i)
        self.weights.copy_(w)
        for src, dst in zip(self.store, self.inputs):
            torch.index_select(src, 0, self.idxs, out=dst)
        self.L.learn(self.inputs, weights=self.weights, idxs=self.idxs, sampler=self.S, sync_stats=False)


def gather_bandwidth(mem, B, reps=50):
    idxs = torch.randint(0, M, (B,), device='cuda')
    out = mem._outputs(B)
    args = (mem._h, idxs.data_ptr(), B, *(t.data_ptr() for t in out))
    run = lambda: mem._L.srl_replay_gather(*args, mem._stream())
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
        sys.exit('bench_replay.py measures on a CUDA device; none is present')
    name = card()
    g = torch.Generator(device='cuda').manual_seed(0)
    mem = GpuPrioritizedReplayBuffer(M, E, n_step=3, gamma=0.99)
    steps = [env_step(g) for _ in range(8)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(M // E):
        mem.save_to_memory(*steps[k % len(steps)], is_vectorised=True)
    torch.cuda.synchronize()
    add_rate = (M // E) / (time.perf_counter() - t0)
    print(json.dumps({'card': name, 'memory_size': M, 'num_envs': E, 'n_step': 3, 'save_to_memory_env_steps_per_s': add_rate,
                      'transitions_per_s': add_rate * E}), flush=True)
    for B in (int(x) for x in a.batches.split(',')):
        hp = lambda: ApexHParams(batch_size=B, num_actions=A, gamma=0.99 ** 3, double_dqn=True)
        L1, L2, L3 = B200ApexLearner(hp()), B200ApexLearner(hp()), B200ApexLearner(hp())
        caller = CallerPattern(L2, B, g)
        fixed = tuple(t.clone() for t in caller.inputs)
        fidx, fw = caller.idxs.clone(), torch.rand(B, device='cuda')
        variants = {'learn_from': lambda: L1.learn_from(mem, beta=0.4, sync_stats=False),
                    'caller': caller,
                    'learn_fixed': lambda: L3.learn(fixed, weights=fw, idxs=fidx, sampler=caller.S, sync_stats=False)}
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
            out[k] = {'steps_per_s_median': r[len(r) // 2], 'steps_per_s_range': [r[0], r[-1]]}
        out['learn_from_over_caller'] = out['learn_from']['steps_per_s_median'] / out['caller']['steps_per_s_median']
        out['learn_from_over_learn_fixed'] = out['learn_from']['steps_per_s_median'] / out['learn_fixed']['steps_per_s_median']
        out['gather_kernel'] = gather_bandwidth(mem, B)
        print(json.dumps(out), flush=True)
        del variants, caller
        for L in (L1, L2, L3):
            L.release_graphs()
            L.close()


if __name__ == '__main__':
    main()
