"""Eager per-kernel times of the three conv kernels at the 21x21 end of the encoder -- conv1_fwd, conv2_dgrad and conv1_wgrad --
against the HBM bytes they must move (python tools/conv_chain_profile.py [--T 20 --B 32 --A 6 --steps 200 --warmup 10]).

Builds the default learner, turns per-kernel profiling on (srl_learner_set_profiling: CUDA events around every launch of an
eager step) and runs --steps eager steps on one seeded batch.  Per slot it prints the median, minimum and maximum time, the
algorithmic bytes per launch (bench.py's SLOT_BYTES formula), the achieved GB/s at the median and the time those bytes take at
the data-sheet HBM rate, then the same for the other GEMM slots of the chain, so that a change of a shared mainloop shows up
in all of them.  The GPU name, power limit and maximum SM clock are read in the same run and printed first.  Prints one JSON
line per slot.  Needs a CUDA device; writes nothing."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import SLOT_BYTES, peaks                                      # noqa: E402  (the benchmark's byte formula)
from oracle import impala_oracle as O                                   # noqa: E402  (input generator only)
from scalerl_b200 import _lib                                           # noqa: E402
from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams       # noqa: E402

FOCUS = ('conv1_fwd', 'conv2_dgrad', 'conv1_wgrad')
OTHERS = ('conv2_fwd', 'conv3_fwd', 'conv3_dgrad', 'conv3_wgrad', 'conv2_wgrad', 'obs_s2d')


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                       capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(), 'nvidia_smi': q.stdout.strip() or q.stderr.strip(),
            'sms': torch.cuda.get_device_properties(0).multi_processor_count}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--T', type=int, default=20)
    ap.add_argument('--B', type=int, default=32)
    ap.add_argument('--A', type=int, default=6)
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=10)
    a = ap.parse_args()
    print(json.dumps(gpu_info()), flush=True)
    T, B, A = a.T, a.B, a.A
    lib = _lib.lib()
    names = [lib.srl_profile_slot_name(i).decode() for i in range(lib.srl_profile_slot_count())]
    buf = (C.c_float * len(names))()
    L = B200ImpalaLearner(ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A), init_state_dict=O.init_params(A, seed=0),
                          process_group=False)
    batch = {k: v.cuda() for k, v in O.synthetic_batch(T, B, A, seed=1, done_p=0.02).items()}
    _lib.check(lib.srl_learner_set_profiling(L._h, 1))
    for _ in range(a.warmup):
        L.learn(batch, sync_stats=False, use_graph=False)
        _lib.check(lib.srl_learner_profile_collect(L._h, buf))
    times = {n: [] for n in FOCUS + OTHERS}
    for _ in range(a.steps):
        L.learn(batch, sync_stats=False, use_graph=False)
        _lib.check(lib.srl_learner_profile_collect(L._h, buf))
        for n in times:
            times[n].append(buf[names.index(n)])
    _lib.check(lib.srl_learner_set_profiling(L._h, 0))
    hbm = peaks()
    for n in FOCUS + OTHERS:
        frames = (T + 1) * B if n in ('conv1_fwd', 'conv2_fwd', 'conv3_fwd', 'obs_s2d') else T * B
        by = SLOT_BYTES[n][0] * frames + SLOT_BYTES[n][1] if n in SLOT_BYTES else None
        ms = times[n]
        med = statistics.median(ms)
        row = {'slot': n, 'T': T, 'B': B, 'steps': len(ms), 'ms_median': round(med, 5), 'ms_min': round(min(ms), 5), 'ms_max': round(max(ms), 5)}
        if by is not None:
            row.update(bytes=by, GBps_at_median=round(by / (med * 1e-3) / 1e9, 1),
                       us_at_hbm_rate=round(by / (hbm['hbm_gbs'] * 1e9) * 1e6, 1), hbm_rate_source=hbm['source'])
        print(json.dumps(row), flush=True)


if __name__ == '__main__':
    main()
