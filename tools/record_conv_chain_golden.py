"""Record tests/golden/conv_chain_digests.json: SHA-256 digests of the default learner step's a1 (both row-parity planes), da1g
and conv weight / bias gradients after one step from fixed seeds, at T=20, B=32, A=6 and at the ragged T=7, B=19, A=18
(python tools/record_conv_chain_golden.py [--out PATH]).

tests/test_gpu_conv_chain_golden.py recomputes the same digests and requires them to match bit for bit: the conv kernels at
the 21x21 end of the encoder may change how they tile and schedule their work, not what they compute.  The conv gradients are
per-CTA partial sums added in CTA order, so their bits depend on the number of CTAs and therefore on the SM count, which is
stored beside them.  Needs a CUDA device."""
import argparse
import hashlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = ((20, 32, 6), (7, 19, 18))
GRADS = ('conv1.weight', 'conv1.bias', 'conv2.weight', 'conv2.bias', 'conv3.weight', 'conv3.bias')
OUT = os.path.join(ROOT, 'tests', 'golden', 'conv_chain_digests.json')


def step_digests(T, B, A, buffers=('a1', 'da1'), grads=GRADS):
    """{array name: sha256 of its raw bytes} of the named workspace buffers and parameter gradients after one default learner
    step on seeded parameters and batch"""
    from oracle import impala_oracle as O
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    L = B200ImpalaLearner(ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A), init_state_dict=O.init_params(A, seed=0),
                          process_group=False)
    L.learn({k: v.cuda() for k, v in O.synthetic_batch(T, B, A, seed=1, done_p=0.02).items()})
    torch.cuda.synchronize()
    arrays = {n: L.debug_buffer(n) for n in buffers}
    arrays.update((n, L.grads[n]) for n in grads)
    return {n: hashlib.sha256(t.detach().contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest() for n, t in arrays.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=OUT)
    a = ap.parse_args()
    rec = {'sms': torch.cuda.get_device_properties(0).multi_processor_count, 'device': torch.cuda.get_device_name(),
           'shapes': {f'{T}x{B}x{A}': step_digests(T, B, A) for T, B, A in SHAPES}}
    with open(a.out, 'w') as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write('\n')
    print(json.dumps(rec))


if __name__ == '__main__':
    main()
