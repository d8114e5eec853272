#!/usr/bin/env python
"""profiles/ncu_traffic.json from the summary table written by tools/ncu_summary.py:
   python tools/ncu_summary.py ncu_out/prof.ncu-rep ncu_out/prof.md
   python tools/ncu_traffic.py ncu_out/prof.md 'source text' > profiles/ncu_traffic.json
Per bench.py profile slot: mean DRAM read+write bytes per launch, ncu duration, tensor-pipe activity."""
import json
import re
import sys

SLOT = {'RConv1Fwd': 'conv1_fwd', 'RConv2Fwd': 'conv2_fwd', 'RConv3Fwd': 'conv3_fwd', 'TFcFwd': 'fc_fwd', 'TFcWgrad': 'fc_wgrad',
        'TFcDgrad': 'fc_dgrad', 'RConv3Wgrad': 'conv3_wgrad', 'RConv3Dgrad': 'conv3_dgrad', 'RConv2Wgrad': 'conv2_wgrad',
        'RConv2Dgrad': 'conv2_dgrad', 'RConv1Wgrad': 'conv1_wgrad', 'obs_s2d_kernel': 'obs_s2d', 'column_step_kernel': 'vtrace_loss_tail',
        'clip_optim_kernel': 'optimizer', 'WgradReduce1': 'conv_wgrad_finalize', 'pack_weights_kernel': 'pack_weights',
        'head_wgrad_kernel': 'head_bwd'}


def num(cell):
    m = re.match(r'\s*([0-9.eE+-]+)\s*(\w*)', cell)
    v = float(m.group(1))
    return v * {'Mbyte': 1e6, 'Kbyte': 1e3, 'Gbyte': 1e9, 'byte': 1.0}.get(m.group(2), 1.0)


def main():
    acc = {}
    for line in open(sys.argv[1]):
        c = [x.strip() for x in line.strip().strip('|').split('|')]
        if len(c) < 10 or c[0] in ('kernel', '---'):
            continue
        m = re.search(r'<(?:srl::)?(\w+)', c[0])
        key = SLOT.get(m.group(1) if m else None) or SLOT.get(c[0].split('<')[0].strip())
        if not key:
            continue
        a = acc.setdefault(key, dict(b=0.0, d=0.0, t=0.0, n=0))
        a['b'] += num(c[2]) + num(c[3]); a['d'] += num(c[1]); a['t'] += num(c[7]); a['n'] += 1
    out = {'source': sys.argv[2], 'kernels': {k: {'dram_bytes_per_launch': a['b'] / a['n'], 'ncu_duration_us': a['d'] / a['n'],
                                                   'tensor_pipe_active_pct': a['t'] / a['n'], 'launches_averaged': a['n']} for k, a in acc.items()}}
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
