"""The Ape-X layout entry points of the C ABI (srl_apex_param_layout, _ex, _cat and _noisy) return exactly what
tools/record_apex_layouts.py recorded in tests/golden/apex_layouts.json: every offset and count, padding included, for A = 1..31 and
every head with and without noise, and the same return values and error texts for bad arguments.  Host code only."""
import json
import os

from tests.conftest import GOLDEN
from tools.record_apex_layouts import record


def test_apex_layouts_match_recorded():
    want = json.load(open(os.path.join(GOLDEN, 'apex_layouts.json')))
    got = record()
    assert got.keys() == want.keys()
    assert [k for k in want if got[k] != want[k]] == []
