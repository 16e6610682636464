"""The fused backward is deterministic: on seeded inputs it writes the hash-grid and weight gradients bit for bit as the stored digests
(tests/golden/make_bwd_digests.py) say, at the lego and fox level tables, at a full 2^18-row batch, at a row count that is not a
multiple of 256 and with a device-side live count below the launch size."""
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SCRIPT = os.path.join(HERE, "golden", "make_bwd_digests.py")

pytestmark = pytest.mark.gpu


def test_fused_backward_gradients_match_stored_digests(tmp_path):
    # a fresh process: no fixed-point scratch sized for a level table that an earlier test freed (see make_bwd_digests.run_case)
    out = tmp_path / "bwd_digests.json"
    subprocess.check_call([sys.executable, SCRIPT, str(out)])
    got = json.load(open(out))["cases"]
    want = json.load(open(os.path.join(HERE, "golden", "bwd_digests.json")))["cases"]
    assert got == want
