"""Time of the fused clip + optimizer kernel (profile slot 'optimizer' of srl_learner_set_profiling) with and without RMSprop
momentum and the linear learning-rate schedule (python tools/optimizer_profile.py [--T 20 --B 32 --rounds 10 --steps 20]).

Each configuration is its own learner on the same weights and batches; the rounds alternate between them so that drift of the
clocks affects all alike.  A step runs eagerly with CUDA events around every launch (srl_learner_profile_collect).  Per
configuration it prints the median and minimum kernel time over all profiled steps and the HBM bytes per step the update must
move, from the parameter count: 20 B per parameter without momentum (read g, p, v; write p, v), 28 B with it (+ read and write
the momentum buffer).  Prints the GPU name and power limit first, then one JSON line per configuration.  Needs a CUDA device;
writes nothing."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import impala_oracle as O                                   # noqa: E402  (input generator only)
from scalerl_b200 import _lib                                           # noqa: E402
from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams       # noqa: E402

CONFIGS = {
    'rmsprop': {},
    'rmsprop_momentum': dict(momentum=0.9),
    'rmsprop_momentum_linear': dict(momentum=0.9, lr_schedule='linear', total_frames=10 ** 9),
}


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                       capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(), 'nvidia_smi': q.stdout.strip() or q.stderr.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--T', type=int, default=20)
    ap.add_argument('--B', type=int, default=32)
    ap.add_argument('--A', type=int, default=6)
    ap.add_argument('--rounds', type=int, default=10)
    ap.add_argument('--steps', type=int, default=20)
    a = ap.parse_args()
    print(json.dumps(gpu_info()), flush=True)
    T, B, A = a.T, a.B, a.A
    lib = _lib.lib()
    slot = [lib.srl_profile_slot_name(i).decode() for i in range(lib.srl_profile_slot_count())].index('optimizer')
    buf = (C.c_float * lib.srl_profile_slot_count())()
    params = O.init_params(A, seed=0)
    batch = {k: v.cuda() for k, v in O.synthetic_batch(T, B, A, seed=1, done_p=0.02).items()}
    learners = {name: B200ImpalaLearner(ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A, **kw), init_state_dict=params,
                                        process_group=False) for name, kw in CONFIGS.items()}
    times = {name: [] for name in CONFIGS}
    for L in learners.values():
        _lib.check(lib.srl_learner_set_profiling(L._h, 1))
        for _ in range(3):                                   # warm-up: module load, occupancy query
            L.learn(batch, sync_stats=False, use_graph=False)
    torch.cuda.synchronize()
    for _ in range(a.rounds):
        for name, L in learners.items():
            for _ in range(a.steps):
                L.learn(batch, sync_stats=False, use_graph=False)
                _lib.check(lib.srl_learner_profile_collect(L._h, buf))
                times[name].append(buf[slot])
    for name, L in learners.items():
        _lib.check(lib.srl_learner_set_profiling(L._h, 0))
        n = sum(L._cnt)
        per_param = 28 if L.opt_state2 is not None else 20
        med, lo = statistics.median(times[name]), min(times[name])
        print(json.dumps({'config': name, 'T': T, 'B': B, 'params': n, 'optimizer_ms_median': round(med, 5), 'optimizer_ms_min': round(lo, 5),
                          'samples': len(times[name]), 'update_bytes': per_param * n,
                          'update_GBps_at_median': round(per_param * n / (med * 1e-3) / 1e9, 1)}), flush=True)


if __name__ == '__main__':
    main()
