"""The fc layer's forward, data-gradient and weight-gradient GEMMs compute, bit for bit, what they computed before their output
tiles were staged through shared memory: h, da3 and fc.weight's and fc.bias's gradients of one default learner step from fixed
seeds, at T=20, B=32 and at a ragged T=7, B=19, against SHA-256 digests recorded by tools/record_fc_golden.py
(tests/golden/fc_digests.json).

Every element of these tensors is a sum in a fixed K order, so the digests hold on any device."""
import json
import os

import pytest

from tests.conftest import GOLDEN
from tools.record_fc_golden import SHAPES, fc_digests

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('T,B,A', SHAPES)
def test_fc_bits_match_recorded(T, B, A):
    rec = json.load(open(os.path.join(GOLDEN, 'fc_digests.json')))
    assert fc_digests(T, B, A) == rec['shapes'][f'{T}x{B}x{A}']
