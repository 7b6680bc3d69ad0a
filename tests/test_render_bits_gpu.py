"""The forward image is pinned bit for bit: tests/golden/render_digests.json holds the SHA-256 of every image of
tests/render_digest_cases.py as the render kernel produced it before its lanes were remapped to whole tile rows
(written by scripts/gpu/render_digests.py).  A change to the render kernel's work layout must reproduce them exactly."""
import json
import os

import pytest

import render_digest_cases as rdc

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "render_digests.json")


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)["images"]


def test_golden_covers_every_case():
    want = _golden()
    names = [name for name, _, _ in rdc.cases()]
    assert sorted(names) == sorted(want)


@pytest.mark.parametrize("name", sorted(_golden()))
def test_forward_image_bits(name):
    want = _golden()[name]
    cloud, view = next((c, v) for n, c, v in rdc.cases() if n == name)
    got = rdc.render(cloud, view)
    assert got["shape"] == want["shape"] and got["R"] == want["R"], (got, want)
    assert got["sha256"] == want["sha256"], f"{name}: image differs from the pinned bits"
