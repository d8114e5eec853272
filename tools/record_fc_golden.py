"""Record tests/golden/fc_digests.json: SHA-256 digests of h (the fc layer's output: its split-K partials summed with the bias,
ReLU'd), da3 (the fc layer's data gradient on conv3's 9x9 grid) and fc.weight's and fc.bias's gradients after one default learner
step from fixed seeds, at T=20, B=32, A=6 and at the ragged T=7, B=19, A=18, whose 152 forward and 133 backward frames end in
partial 128-frame tiles and a partial 64-frame k-block (python tools/record_fc_golden.py [--out PATH]).

tests/test_gpu_fc_golden.py recomputes the same digests and requires them to match bit for bit: the fc layer's forward,
data-gradient and weight-gradient GEMMs may change how they store their tiles, not what they compute.  Each of these elements is
one warpgroup's fixed sequence of wgmma over K (plus, for h, a fixed-order sum of the partials), so the digests do not depend on
the device.  Needs a CUDA device."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.record_conv_chain_golden import SHAPES, step_digests      # noqa: E402

BUFFERS = ('h', 'da3')
GRADS = ('fc.weight', 'fc.bias')
OUT = os.path.join(ROOT, 'tests', 'golden', 'fc_digests.json')


def fc_digests(T, B, A):
    return step_digests(T, B, A, buffers=BUFFERS, grads=GRADS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=OUT)
    a = ap.parse_args()
    rec = {'device': torch.cuda.get_device_name(), 'shapes': {f'{T}x{B}x{A}': fc_digests(T, B, A) for T, B, A in SHAPES}}
    with open(a.out, 'w') as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write('\n')
    print(json.dumps(rec))


if __name__ == '__main__':
    main()
