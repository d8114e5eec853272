"""The conv kernels at the 21x21 end of the encoder (conv1's forward, conv2's data gradient, conv1's weight gradient) compute,
bit for bit, what they computed before their output tiles were staged through shared memory: a1 (both row-parity planes), da1g
and the conv weight / bias gradients of one default learner step from fixed seeds, at T=20, B=32 and at a ragged T=7, B=19,
against SHA-256 digests recorded by tools/record_conv_chain_golden.py (tests/golden/conv_chain_digests.json).

a1 and da1g are per-element sums in a fixed K order, so their bits do not depend on the device.  The conv gradients are per-CTA
partial sums added in CTA order: they are compared on a device with the recorded SM count only."""
import json
import os

import pytest
import torch

from tests.conftest import GOLDEN
from tools.record_conv_chain_golden import SHAPES, step_digests

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('T,B,A', SHAPES)
def test_conv_chain_bits_match_recorded(T, B, A):
    rec = json.load(open(os.path.join(GOLDEN, 'conv_chain_digests.json')))
    want = rec['shapes'][f'{T}x{B}x{A}']
    got = step_digests(T, B, A)
    same_sms = torch.cuda.get_device_properties(0).multi_processor_count == rec['sms']
    names = [n for n in want if same_sms or not n.startswith('conv')]
    assert {n: got[n] for n in names} == {n: want[n] for n in names}
