"""-m gpu: the affinity build's output bits are pinned. tests/golden/affinity_bits.json holds SHA-256 digests of W (every
byte, pitch padding included) and of the degree written by dss_affinity on seeded features (tools/affinity_bits.py,
which also generates the file): every width class of an image's last column tile, last row tiles with at most and
with more than 64 rows, B in {1, 2, 3}, d in {64, 384, 768}, every DSS_AFF_* flag, colour counts and row pitches
wider than N. Each digest must be reproduced exactly."""
import importlib.util
import json

import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu

GOLDEN = json.loads((ROOT / "tests" / "golden" / "affinity_bits.json").read_text())
_spec = importlib.util.spec_from_file_location("affinity_bits", ROOT / "tools" / "affinity_bits.py")
bits = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(bits)


@pytest.mark.parametrize("B,N,d,flags,lam,ldw", bits.CASES, ids=[bits.key(*c) for c in bits.CASES])
def test_affinity_bits(cuda, B, N, d, flags, lam, ldw):
    W, deg = bits.affinity(B, N, d, flags, lam, ldw)
    want = GOLDEN[bits.key(B, N, d, flags, lam, ldw)]
    assert bits.digest(W) == want["W"]
    assert bits.digest(deg) == want["degree"]
