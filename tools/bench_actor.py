"""Actor inference throughput of B200ActorModel, feed-forward and LSTM (python tools/bench_actor.py [--n 16,64,256]).

Per actor kind and N environments per call:
  * calls/s and env-steps/s device-resident (forward_device on device tensors, state passed back as returned) and
    host-in / host-out (__call__ with host env tensors: pinned H2D copies, one D2H of the outputs, a synchronise per call);
  * LSTM only: the step kernel's own time per call (both layers, lstm_step_kernel) from CUDA kernel records of torch.profiler
    over many calls after warm-up, for every K split (cluster size) the library offers, and its achieved bytes/s computed
    from shapes: 2 layers x 2304 x 1152 bf16 packed weights (10.6 MB) + the operands and the fp32 state it reads and writes.
Prints the GPU name and power limit first, then one JSON line per measurement.  Needs a CUDA device; writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_PEAK = 3.35e12          # H100 SXM data sheet, bytes/s


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                       capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(), 'nvidia_smi': q.stdout.strip() or q.stderr.strip()}


def step_bytes(N, A):
    """bytes one actor call's two step launches must move, from shapes"""
    H, Hp = 513 + A, 576
    weights = 2 * (4 * Hp) * (2 * Hp) * 2
    operands = 2 * N * (2 * Hp) * 2                 # [x | m.h] bf16 read per layer
    state = 2 * N * H * 4 * 3 + N * H * 2 + 2 * 4 * H * 4 * 2     # c in, c/h out per layer; bf16 x of layer 1; biases
    return weights + operands + state


def rate(fn, calls, N):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(calls):
        fn()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return {'calls_per_sec': calls / dt, 'env_steps_per_sec': calls * N / dt, 'ms_per_call': dt / calls * 1e3}


def kernel_ms(fn, calls, name='lstm_step_kernel'):
    """mean device time per call of the kernels whose name contains `name` (torch.profiler CUDA records)"""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if name in e.key)
    launches = sum(e.count for e in prof.key_averages() if name in e.key)
    return us / 1e3 / calls, launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', default='16,64,256')
    ap.add_argument('--calls', type=int, default=300)
    ap.add_argument('--num-actions', type=int, default=6)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_actor needs a CUDA device')
    from scalerl_b200 import _lib
    from scalerl_b200.algorithms.impala.gpu_actor import B200ActorModel
    A = args.num_actions
    print(json.dumps({'gpu': gpu_info()}), flush=True)
    for N in (int(v) for v in args.n.split(',')):
        g = torch.Generator().manual_seed(N)
        host = dict(obs=torch.randint(0, 256, (1, N, 4, 84, 84), dtype=torch.uint8, generator=g), reward=torch.randn(1, N, generator=g),
                    done=torch.rand(1, N, generator=g) < 0.05, action=torch.randint(0, A, (1, N), generator=g))
        dev = {k: v.cuda() for k, v in host.items()}
        for lstm in (False, True):
            m = B200ActorModel(N, A, use_lstm=lstm).eval()
            rec = {'actor': 'lstm' if lstm else 'feed_forward', 'N': N}
            if lstm:
                st = [tuple(s.cuda() for s in m.initial_hidden_state(N))]
                hst = [m.initial_hidden_state(N)]

                def dev_call():
                    st[0] = m.forward_device(dev['obs'], dev['reward'], dev['action'], dev['done'], st[0])[3]

                def host_call():
                    hst[0] = m(host, hst[0])[1]
            else:
                def dev_call():
                    m.forward_device(dev['obs'], dev['reward'], dev['action'])

                def host_call():
                    m(host, ())
            rec['device_resident'] = rate(dev_call, args.calls, N)
            rec['host_in_host_out'] = rate(host_call, args.calls, N)
            if lstm:
                nbytes = step_bytes(N, A)
                rec['step_bytes'] = nbytes
                rec['step_kernel'] = {}
                for ks in (1, 2, 3, 6):
                    _lib.check(_lib.lib().srl_learner_set_option(m._ctx._h, b'lstm_step_ksplit', ks), 'set_option')
                    ms, launches = kernel_ms(dev_call, args.calls)
                    bw = nbytes / (ms * 1e-3)
                    rec['step_kernel'][f'ksplit{ks}'] = {'ms_per_call': ms, 'launches': launches, 'bytes_per_sec': bw,
                                                        'above_hbm_peak': bw > HBM_PEAK}
            print(json.dumps(rec), flush=True)
            m.close()


if __name__ == '__main__':
    main()
