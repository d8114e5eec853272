"""Time the R2D2 learner step (B200R2D2Learner.learn) at the paper's shape: 64 sequences of 40 burn-in + 80 trained + 5 bootstrap rows,
A = 18, the dueling head, value rescaling, priorities written into a GpuPrioritizedSampler.

Rounds alternate between the captured step (CUDA graph replay) and the eager step; each prints the median and range over rounds of
learner steps/s and trained frames/s (B T per step), with the card's name and power limit read in the same run.  A separate
torch.profiler run of eager steps then splits the device time by kernel family: the encoder (conv / fc GEMMs, their reductions and
the weight packing), the LSTM core (its lstm_* kernels and its GEMMs, igemm_tma_kernel<LGemm*>: the sequential recurrence of both
networks), the Q head and sequence tail (the r2d2_* kernels) and the clip + Adam step.  Needs a GPU.

    python tools/bench_r2d2.py [--rounds 5 --steps 20 --B 64 --burn-in 40 --T 80 --n 5 --A 18]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scalerl_b200.algorithms.r2d2 import B200R2D2Learner, R2D2HParams  # noqa: E402
from scalerl_b200.data.per_sampler import GpuPrioritizedSampler  # noqa: E402


def card():
    """'<name>, <power limit>' as nvidia-smi reports them (the name alone when nvidia-smi is unavailable)"""
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
        if q.returncode == 0 and q.stdout.strip():
            return q.stdout.strip().splitlines()[torch.cuda.current_device()]
    except OSError:
        pass
    return torch.cuda.get_device_name()


def inputs(hp, dev='cuda'):
    g = torch.Generator(device=dev).manual_seed(0)
    L, B, A, H = hp.seq_rows, hp.batch_size, hp.num_actions, 513 + hp.num_actions
    seq = dict(frame=torch.randint(0, 256, (L, B, 4, 84, 84), generator=g, device=dev, dtype=torch.uint8),
               last_action=torch.randint(0, A, (L, B), generator=g, device=dev),
               reward=torch.randn(L, B, generator=g, device=dev),
               done=torch.rand(L, B, generator=g, device=dev) < 0.01,
               state=tuple(torch.randn(2, B, H, generator=g, device=dev) * 0.3 for _ in range(2)))
    sampler = GpuPrioritizedSampler(4 * B, alpha=0.9, device=dev)
    sampler.add(4 * B)
    idxs = torch.randperm(4 * B, device=dev)[:B].contiguous()
    weights = torch.rand(B, generator=g, device=dev) + 0.5
    return seq, weights, idxs, sampler


def timed(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return steps / (time.perf_counter() - t0)


FAMILIES = (('head_and_tail', ('r2d2_',)), ('optimizer', ('clip_optim', 'optim', 'adam', 'grad_norm')),
            ('lstm', ('lstm', 'lgemm')), ('encoder', ('',)))


def split(learner, args, steps):
    """device time per eager step by kernel family (ms), from a torch.profiler run of its own"""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(2):
        learner.learn(*args, use_graph=False, sync_stats=False)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            learner.learn(*args, use_graph=False, sync_stats=False)
        torch.cuda.synchronize()
    fam = {k: 0.0 for k, _ in FAMILIES}
    for e in prof.key_averages():
        t = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0.0)
        if not t or e.key.startswith('Memcpy') or e.key.startswith('Memset'):
            continue
        name = e.key.lower()
        for k, keys in FAMILIES:
            if any(s in name for s in keys):
                fam[k] += t / 1e3 / steps
                break
    total = sum(fam.values())
    return {'eager_device_ms_per_step': total, **{f'{k}_ms': v for k, v in fam.items()},
            **{f'{k}_share': v / total for k, v in fam.items() if total}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--B', type=int, default=64)
    ap.add_argument('--burn-in', type=int, default=40)
    ap.add_argument('--T', type=int, default=80)
    ap.add_argument('--n', type=int, default=5)
    ap.add_argument('--A', type=int, default=18)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_r2d2.py needs a GPU')
    hp = R2D2HParams(batch_size=a.B, num_actions=a.A, burn_in=a.burn_in, seq_len=a.T, n_step=a.n, target_update_frequency=10 ** 9)
    learner = B200R2D2Learner(hp)
    seq, w, idxs, sampler = inputs(hp)
    args = (seq, w, idxs, sampler)
    step = {'captured': lambda: learner.learn(*args, use_graph=True, sync_stats=False),
            'eager': lambda: learner.learn(*args, use_graph=False, sync_stats=False)}
    for fn in step.values():          # warm-up: the captured variant's eager first call and its capture
        for _ in range(3):
            fn()
    rates = {k: [] for k in step}
    for _ in range(a.rounds):
        for k, fn in step.items():
            rates[k].append(timed(fn, a.steps))
    out = {'bench': 'r2d2_learner_step', 'card': card(), 'B': a.B, 'burn_in': a.burn_in, 'T': a.T, 'n': a.n, 'A': a.A, 'dueling': True,
           'rounds': a.rounds, 'steps_per_round': a.steps}
    for k, r in rates.items():
        r = sorted(r)
        out[k] = {'steps_per_s_median': r[len(r) // 2], 'steps_per_s_range': [r[0], r[-1]],
                  'trained_frames_per_s_median': r[len(r) // 2] * a.B * a.T}
    print(json.dumps(out), flush=True)
    print(json.dumps({'bench': 'r2d2_eager_split', 'card': card(), **split(learner, args, a.steps)}), flush=True)
    learner.close()
    sampler.close()


if __name__ == '__main__':
    main()
