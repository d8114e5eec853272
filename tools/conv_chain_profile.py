"""Eager per-kernel times of the conv kernels of the encoder against the HBM bytes they must move and the MMAs they issue
(python tools/conv_chain_profile.py [--focus edge|mid|fc] [--T 20 --B 32 --A 6 --steps 200 --warmup 10]).

--focus edge (default): the three kernels at the 21x21 end of the encoder -- conv1_fwd, conv2_dgrad and conv1_wgrad.
--focus mid: the three resident-window kernels in the middle of it -- conv2_fwd, conv3_fwd and conv3_dgrad.
--focus fc: the fc layer's three GEMMs on the TMA mainloop -- fc_fwd, fc_dgrad and fc_wgrad.

Builds the default learner, turns per-kernel profiling on (srl_learner_set_profiling: CUDA events around every launch of an
eager step) and runs --steps eager steps on one seeded batch.  Per slot it prints the median, minimum and maximum time, the
algorithmic bytes per launch (bench.py's SLOT_BYTES formula), the achieved GB/s at the median and the time those bytes take at
the data-sheet HBM rate, then the same for the other GEMM slots of the chain, so that a change of a shared mainloop shows up
in all of them.  For conv2_fwd, conv3_fwd and conv3_dgrad it also prints the launch's tiles, CTAs and rounds, the m64n64k16
wgmma it issues (rows computed and discarded included) and an MMA-only time: 48 clocks per wgmma (the N = 64 rate of
tma_problems.cuh), spread over the SMs at the maximum SM clock -- an estimate, not a measurement.  For fc_fwd, fc_dgrad and fc_wgrad
it prints the grid, CTAs, waves, the wgmma issued (m64nNk16, N = each warpgroup's columns) and an MMA-only time: one CTA per SM
(their shared memory allows no second), a CTA's wgmma at max(N / 2, 48) clocks each -- the tensor array's rate for N = 128 and 256,
the N = 64 cost above, assumed for N = 32 -- times the waves, at the maximum SM clock: again an estimate, not a measurement.  The GPU name, power limit and maximum SM clock
are read in the same run and printed first.  Prints one JSON line per slot.  Needs a CUDA device; writes nothing."""
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

SLOTS = ('conv1_fwd', 'conv2_dgrad', 'conv1_wgrad', 'conv2_fwd', 'conv3_fwd', 'conv3_dgrad', 'conv3_wgrad', 'conv2_wgrad', 'obs_s2d',
         'fc_fwd', 'fc_dgrad', 'fc_wgrad')
FOCUS = {'edge': ('conv1_fwd', 'conv2_dgrad', 'conv1_wgrad'), 'mid': ('conv2_fwd', 'conv3_fwd', 'conv3_dgrad'),
         'fc': ('fc_fwd', 'fc_dgrad', 'fc_wgrad')}
FWD_SLOTS = ('conv1_fwd', 'conv2_fwd', 'conv3_fwd', 'obs_s2d', 'fc_fwd')
# the N = 64 res_fwd_kernel slots: (grid positions per frame, taps, frames 'fwd' = (T+1)*B or 'bwd' = T*B, CTAs 'all' SMs or 'bwd' =
# SMs - SMs/9, encoder.cu's bwd_ctas())
RES_FWD = {'conv2_fwd': (100, 8, 'fwd', 'all'), 'conv3_fwd': (81, 9, 'fwd', 'all'), 'conv3_dgrad': (81, 9, 'bwd', 'bwd')}


def mma_estimate(slot, T, B, sms, mhz):
    """tiles, CTAs, rounds, wgmma issued and the MMA-only microseconds of one res_fwd_kernel launch (not measured)"""
    grid, taps, fr, ctas = RES_FWD[slot]
    tiles = -(-(T + 1 if fr == 'fwd' else T) * B * grid // 128)
    ctas = min(tiles, sms if ctas == 'all' else sms - sms // 9)
    wgmma = tiles * 2 * taps * 4
    return {'tiles': tiles, 'ctas': ctas, 'rounds': round(tiles / ctas, 2), 'wgmma': wgmma,
            'us_mma_only': round(wgmma * 48 / sms / mhz, 2) if mhz else None}


def fc_estimate(slot, T, B, sms, mhz):
    """grid, CTAs, waves, wgmma issued and the MMA-only microseconds of one igemm_tma_kernel launch of the fc layer (bf16 mode,
    encoder.cu's grids; not measured)"""
    fr = (T + 1) * B if slot == 'fc_fwd' else T * B
    if slot == 'fc_fwd':          # TFcFwd: (frame tiles, 8 column tiles x 4 K splits), 49 k-blocks of 64 per column tile, N = 32
        grid, n, wg_tile = (-(-fr // 128), 32), 32, 49 * 4 * 2 * 2 / 4
    elif slot == 'fc_dgrad':      # TFcDgrad: (frame tiles, 49 pixels), 8 k-blocks of 64, N = 32
        grid, n, wg_tile = (-(-fr // 128), 49), 32, 8 * 4 * 2 * 2
    else:                         # TFcWgradN: (1, 4 row tiles x 14 column tiles), one k-block per 64 frames, N = 128
        grid, n, wg_tile = (1, 56), 128, -(-fr // 64) * 4 * 2 * 2
    ctas = grid[0] * grid[1]
    waves = -(-ctas // sms)
    return {'grid': list(grid), 'ctas': ctas, 'waves': waves, 'wgmma': round(ctas * wg_tile), 'wgmma_n': n,
            'us_mma_only': round(waves * wg_tile * max(n // 2, 48) / mhz, 2) if mhz else None}


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader,nounits', '-i', str(torch.cuda.current_device())],
                       capture_output=True, text=True)
    fields = q.stdout.strip().split(', ')
    try:
        mhz = float(fields[2])
    except (IndexError, ValueError):
        mhz = None
    return {'torch_name': torch.cuda.get_device_name(), 'nvidia_smi': q.stdout.strip() or q.stderr.strip(),
            'sms': torch.cuda.get_device_properties(0).multi_processor_count, 'max_sm_mhz': mhz}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--focus', choices=sorted(FOCUS), default='edge')
    ap.add_argument('--T', type=int, default=20)
    ap.add_argument('--B', type=int, default=32)
    ap.add_argument('--A', type=int, default=6)
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=10)
    a = ap.parse_args()
    info = gpu_info()
    print(json.dumps(info), flush=True)
    order = FOCUS[a.focus] + tuple(n for n in SLOTS if n not in FOCUS[a.focus])
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
    times = {n: [] for n in order}
    for _ in range(a.steps):
        L.learn(batch, sync_stats=False, use_graph=False)
        _lib.check(lib.srl_learner_profile_collect(L._h, buf))
        for n in times:
            times[n].append(buf[names.index(n)])
    _lib.check(lib.srl_learner_set_profiling(L._h, 0))
    hbm = peaks()
    for n in order:
        frames = (T + 1) * B if n in FWD_SLOTS else T * B
        by = SLOT_BYTES[n][0] * frames + SLOT_BYTES[n][1] if n in SLOT_BYTES else None
        ms = times[n]
        med = statistics.median(ms)
        row = {'slot': n, 'T': T, 'B': B, 'steps': len(ms), 'ms_median': round(med, 5), 'ms_min': round(min(ms), 5), 'ms_max': round(max(ms), 5)}
        if by is not None:
            row.update(bytes=by, GBps_at_median=round(by / (med * 1e-3) / 1e9, 1),
                       us_at_hbm_rate=round(by / (hbm['hbm_gbs'] * 1e9) * 1e6, 1), hbm_rate_source=hbm['source'])
        if n in RES_FWD:
            row.update(mma_estimate(n, T, B, info['sms'], info['max_sm_mhz']))
        if n in FOCUS['fc']:
            row.update(fc_estimate(n, T, B, info['sms'], info['max_sm_mhz']))
        print(json.dumps(row), flush=True)


if __name__ == '__main__':
    main()
