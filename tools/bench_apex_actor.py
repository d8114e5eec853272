"""Env steps/s of the Ape-X acting side on one GPU: acting plus adding one vector step of E envs to an n-step prioritized memory,
frames resident on the device (no env is stepped: the numbers price the GPU work an env step costs).  Three legs:
  (a) actor:     B200ApexActor.act + save_to_memory(priorities_from=actor)  (per-env epsilons, actor-computed initial priorities)
  (b) plain:     B200ApexLearner.get_action(obs, eps) + plain save_to_memory  (one epsilon for the batch, max_priority on insert)
  (c) reference: the reference's statements on torch/cuDNN AtariQNet: per-env epsilon-greedy in torch, plain save_to_memory, then
                 compute_prior (apex/worker.py:59-79) on the transitions the add completed and update_priorities of their slots
Rounds alternate between the legs; the median and range over rounds are printed with the card's name and power limit, one JSON line
per workload.  With --noisy a noisy actor (B200ApexActor(..., noisy_dqn=True): a new noise draw and the composition of its weights on
every act) runs leg (a) beside the plain actor, and the act calls alone are timed for both ('act', 'noisy_act').  With --quantile a
quantile actor (B200ApexActor(..., quantile_dqn=True, num_quantiles=--quantiles): the quantile GEMM, the quantile means and the quantile
Huber priorities) runs leg (a) the same way ('quantile_actor', 'act', 'quantile_act').

    python tools/bench_apex_actor.py [--rounds 5] [--steps 100] [--configs 64x6,64x18,256x6,256x18] [--noisy | --quantile [--quantiles 200]]
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scalerl_b200.algorithms.apex import (ApexHParams, AtariQNet, B200ApexActor, B200ApexLearner, apex_epsilons,  # noqa: E402
                                          default_q_state_dict)
from scalerl_b200.data.replay_memory import GpuPrioritizedReplayBuffer  # noqa: E402
from tools.bench_apex import card  # noqa: E402

MEMORY, N_STEP, GAMMA, PRIORITY_EPS = 65536, 3, 0.99, 1e-6


def vector_step(E, A, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    obs = torch.randint(0, 256, (E, 4, 84, 84), dtype=torch.uint8, device='cuda', generator=g)
    nobs = torch.randint(0, 256, (E, 4, 84, 84), dtype=torch.uint8, device='cuda', generator=g)
    rew = torch.randn(E, device='cuda', generator=g)
    done = torch.rand(E, device='cuda', generator=g) < 0.01
    return obs, nobs, rew, done


class TorchActor:
    """the reference's acting and priority statements on torch/cuDNN; its memory takes the plain add, then the new slots' priorities"""

    def __init__(self, E, A):
        self.model = AtariQNet(A).cuda()
        self.model.load_state_dict(default_q_state_dict(A))
        self.E, self.A = E, A
        self.eps = torch.tensor(apex_epsilons(E), dtype=torch.float32, device='cuda')
        self.mem = GpuPrioritizedReplayBuffer(MEMORY, E, n_step=N_STEP, gamma=GAMMA)
        self.gamma_n = GAMMA ** N_STEP
        self.steps, self.env_ids = 0, torch.arange(E, device='cuda')

    @torch.no_grad()
    def __call__(self, obs, nobs, rew, done):
        q = self.model(obs)
        explore = torch.rand(self.E, device='cuda') < self.eps
        action = torch.where(explore, torch.randint(0, self.A, (self.E,), device='cuda'), q.argmax(1))
        self.mem.save_to_memory(obs, action, rew, nobs, done, is_vectorised=True)
        self.steps += 1
        if self.steps < N_STEP:
            return
        slots = (self.env_ids + (self.steps - N_STEP) * self.E) % MEMORY                # the slots this add filled
        s, a, r, ns, d = self.mem.gather(slots)
        pred = self.model(s)                                                          # worker.py:69-72
        pred_action = pred.gather(1, a.unsqueeze(1)).squeeze(1)
        target = r + (1 - d.float()) * self.gamma_n * self.model(ns).max(1)[0]       # :74
        prior = (pred_action - target).abs() + PRIORITY_EPS                           # :76-77
        self.mem.update_priorities(slots, prior, validate=False)


def timed(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return steps / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=100)
    ap.add_argument('--configs', default='64x6,64x18,256x6,256x18')
    ap.add_argument('--noisy', action='store_true', help='add the noisy actor and time act alone for both actors')
    ap.add_argument('--quantile', action='store_true', help='add the quantile actor and time act alone for both actors')
    ap.add_argument('--quantiles', type=int, default=200)
    a = ap.parse_args()
    if a.noisy and a.quantile:
        sys.exit('--noisy and --quantile are separate comparisons: pass one')
    if not torch.cuda.is_available():
        sys.exit('bench_apex_actor.py measures on a CUDA device; none is present')
    name = card()
    for cfg in a.configs.split(','):
        E, A = (int(x) for x in cfg.split('x'))
        obs, nobs, rew, done = vector_step(E, A, 0)
        X = B200ApexActor(E, A, priority_eps=PRIORITY_EPS)
        L = B200ApexLearner(ApexHParams(batch_size=32, num_actions=A, gamma=GAMMA ** N_STEP))
        mem_a = GpuPrioritizedReplayBuffer(MEMORY, E, n_step=N_STEP, gamma=GAMMA)
        mem_b = GpuPrioritizedReplayBuffer(MEMORY, E, n_step=N_STEP, gamma=GAMMA)
        ref = TorchActor(E, A)

        def actor():
            mem_a.save_to_memory(obs, X.act(obs), rew, nobs, done, is_vectorised=True, priorities_from=X)

        def plain():
            mem_b.save_to_memory(obs, L.get_action(obs, 0.1), rew, nobs, done, is_vectorised=True)

        legs = {'actor': actor, 'plain': plain, 'reference': lambda: ref(obs, nobs, rew, done)}
        if a.noisy:
            XN = B200ApexActor(E, A, priority_eps=PRIORITY_EPS, noisy_dqn=True)
            mem_n = GpuPrioritizedReplayBuffer(MEMORY, E, n_step=N_STEP, gamma=GAMMA)

            def noisy_actor():
                mem_n.save_to_memory(obs, XN.act(obs), rew, nobs, done, is_vectorised=True, priorities_from=XN)

            legs.update({'noisy_actor': noisy_actor, 'act': lambda: X.act(obs), 'noisy_act': lambda: XN.act(obs)})
        if a.quantile:
            XN = B200ApexActor(E, A, priority_eps=PRIORITY_EPS, quantile_dqn=True, num_quantiles=a.quantiles)
            mem_n = GpuPrioritizedReplayBuffer(MEMORY, E, n_step=N_STEP, gamma=GAMMA)

            def quantile_actor():
                mem_n.save_to_memory(obs, XN.act(obs), rew, nobs, done, is_vectorised=True, priorities_from=XN)

            legs.update({'quantile_actor': quantile_actor, 'act': lambda: X.act(obs), 'quantile_act': lambda: XN.act(obs)})
        for fn in legs.values():
            for _ in range(5):
                fn()
        rates = {k: [] for k in legs}
        for _ in range(a.rounds):
            for k, fn in legs.items():
                rates[k].append(timed(fn, a.steps) * E)
        out = {'card': name, 'E': E, 'A': A, **({'num_quantiles': a.quantiles} if a.quantile else {}), 'n_step': N_STEP, 'memory_size': MEMORY, 'precision': 'bf16', 'rounds': a.rounds,
               'vector_steps_per_round': a.steps}
        for k, r in rates.items():
            r = sorted(r)
            out[k] = {'env_steps_per_s_median': r[len(r) // 2], 'env_steps_per_s_range': [r[0], r[-1]]}
        print(json.dumps(out), flush=True)
        for m in (mem_a, mem_b, ref.mem) + ((mem_n,) if a.noisy or a.quantile else ()):
            m.close()
        X.close()
        if a.noisy or a.quantile:
            XN.close()
        L.close()
        del ref


if __name__ == '__main__':
    main()
