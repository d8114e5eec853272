"""Record tests/golden/conv_mid_digests.json: SHA-256 digests of a2 (conv2's output), a3 (conv3's output) and da2g (conv3's data
gradient on conv2's 10x10 grid) after one default learner step from fixed seeds, at T=20, B=32, A=6 and at the ragged T=7, B=19,
A=18 (python tools/record_conv_mid_golden.py [--out PATH]).

tests/test_gpu_conv_mid_golden.py recomputes the same digests and requires them to match bit for bit: conv2's and conv3's forward
and conv3's data gradient may change how they tile, schedule and store their work, not what they compute.  Each of these elements
is one warpgroup's fixed sequence of wgmma over K, so the digests do not depend on the device.  Needs a CUDA device."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.record_conv_chain_golden import SHAPES, step_digests      # noqa: E402

BUFFERS = ('a2', 'a3', 'da2')
OUT = os.path.join(ROOT, 'tests', 'golden', 'conv_mid_digests.json')


def mid_digests(T, B, A):
    return step_digests(T, B, A, buffers=BUFFERS, grads=())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=OUT)
    a = ap.parse_args()
    rec = {'device': torch.cuda.get_device_name(), 'shapes': {f'{T}x{B}x{A}': mid_digests(T, B, A) for T, B, A in SHAPES}}
    with open(a.out, 'w') as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write('\n')
    print(json.dumps(rec))


if __name__ == '__main__':
    main()
