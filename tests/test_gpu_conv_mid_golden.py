"""conv2's and conv3's forward and conv3's data gradient compute, bit for bit, what they computed before their output tiles were
staged through shared memory: a2, a3 and da2g of one default learner step from fixed seeds, at T=20, B=32 and at a ragged
T=7, B=19, against SHA-256 digests recorded by tools/record_conv_mid_golden.py (tests/golden/conv_mid_digests.json).

Every element of these tensors is a sum in a fixed K order, so the digests hold on any device."""
import json
import os

import pytest

from tests.conftest import GOLDEN
from tools.record_conv_mid_golden import SHAPES, mid_digests

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('T,B,A', SHAPES)
def test_conv_mid_bits_match_recorded(T, B, A):
    rec = json.load(open(os.path.join(GOLDEN, 'conv_mid_digests.json')))
    assert mid_digests(T, B, A) == rec['shapes'][f'{T}x{B}x{A}']
