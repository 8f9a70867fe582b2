"""-m gpu: the fp16 attention kernel's output bits are pinned. tests/golden/attention_f16_bits.json holds SHA-256 digests of
its outputs on seeded inputs (tools/attention_bits.py, which also generates the file): dss_op_attention_tc_f16 at every
width class of an image's last key tile and both kinds of last query tile (at most / more than 64 rows), and the K
features of a ragged ViT-S/16 forward over images of those token counts. Each digest must be reproduced exactly."""
import importlib.util
import json

import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu

GOLDEN = json.loads((ROOT / "tests" / "golden" / "attention_f16_bits.json").read_text())
_spec = importlib.util.spec_from_file_location("attention_bits", ROOT / "tools" / "attention_bits.py")
bits = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(bits)


@pytest.mark.parametrize("B,T,heads", bits.UNIFORM)
def test_uniform_attention_bits(cuda, B, T, heads):
    assert bits.digest(bits.attention_uniform(B, T, heads)) == GOLDEN[bits.uniform_key(B, T, heads)]


def test_ragged_forward_bits(cuda):
    assert bits.digest(bits.ragged_features()) == GOLDEN["ragged_vits16_k"]
