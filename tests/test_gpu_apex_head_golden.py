"""Every Q head of the Ape-X learner and actor (plain, dueling, categorical) computes, bit for bit, what it computed before the
heads were described by one binding: the learner's q_values, its first step's q, y, priorities, dcore and loss (and the categorical
logits, m, ce and dlogits), its parameters, target and Adam moments after three steps, and the actor's two consecutive act() calls,
q_values and prioritized tree leaves, at B=32, A=6 and a ragged B=19, A=18, with and without double DQN, on bf16 and fp32_split
operands, against SHA-256 digests recorded by tools/record_apex_head_golden.py (tests/golden/apex_head_digests.json).  The noisy
networks of each head are pinned the same way, with their noise and composed weights (tests/golden/apex_noisy_digests.json).

The state after three steps is downstream of the encoder's conv weight gradients, per-CTA partial sums added in CTA order: it is
compared on a device with the recorded SM count only."""
import json
import os

import pytest
import torch

from tests.conftest import GOLDEN
from tools.record_apex_head_golden import CASES, NOISY_CASES, PER_SM, case_digests

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('case', CASES + NOISY_CASES)
def test_apex_head_bits_match_recorded(case):
    rec = json.load(open(os.path.join(GOLDEN, 'apex_noisy_digests.json' if case in NOISY_CASES else 'apex_head_digests.json')))
    want = rec['cases'][case]
    got = case_digests(case)
    same_sms = torch.cuda.get_device_properties(0).multi_processor_count == rec['sms']
    names = [n for n in want if same_sms or not n.startswith(PER_SM)]
    assert {n: got[n] for n in names} == {n: want[n] for n in names}
