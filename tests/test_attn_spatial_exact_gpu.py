"""Spatial attention is bit-exact against stored digests (scripts/attn_digests.py): the kernel's schedule may change, the
arithmetic of every output row may not. The digests were taken on an H100 from the kernel that ran the softmax and both
MMAs of a key tile one after the other."""
import json

import pytest
import torch

from scripts import attn_digests as AD

pytestmark = pytest.mark.gpu

CASES = AD.cases()


@pytest.fixture(scope="module")
def stored():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device: the product path has no CPU fallback")
    return json.loads(AD.GOLDEN.read_text())["digests"]


@pytest.fixture(scope="module")
def ops():
    from mimo_b200 import ops as O
    return O


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_attn_spatial_digest(ops, stored, c):
    assert AD.run(ops, c, torch.device("cuda", 0)) == stored[c["name"]], c
