"""The engineered inputs of tests/regime_cases.py land where they claim, judged by the CPU oracle's forward and the
regime classifier: this is what keeps tests/test_regimes_gpu.py and the regime assertions of the parity tests from
silently testing something else after a retune.  Also checks the classifier itself on inputs whose regime is plain."""
import numpy as np
import pytest

import regime_cases as rc
import util

CASES = {c.name: c for c in rc.engineered_cases()}


def test_constants_are_read_from_the_sources():
    k = rc.K
    assert k["DIRECT_BLOCK"] > 0 and k["FILL_STAGE_TILES"] <= k["DIRECT_MAX_TILES"]
    assert k["PLAN_CHUNK"] < k["VOX_CHUNK_CAP"] and k["PLAN_ITEMS"] > 0 and k["SUP"] > 1
    assert k["RAS_LW_MIN"] < 0 < k["RAS_LW_MAX"] and k["VOX_LW_MIN"] < 0 < k["VOX_LW_MAX"]
    assert k["CAREFUL_LO"] < 1.0 < k["CAREFUL_HI"]


def test_a_missing_constant_is_an_error():
    with pytest.raises(LookupError):
        rc._constexpr("NO_SUCH_CONSTANT", rc._source("r2x_binning.cuh"), {})


@pytest.mark.parametrize("name", list(CASES))
def test_engineered_case_lands_on_its_side(name):
    case = CASES[name]
    orc = case.oracle()
    lines = rc.check_case(case, orc)
    assert lines
    print(f"\n{name}:\n  " + "\n  ".join(lines))


def test_classifier_on_plain_inputs():
    # tile-count boundaries follow from the shape alone
    assert rc.binning_path((1024, 1024)) == "direct" and rc.binning_path((256, 4096)) == "direct"
    assert rc.binning_path((272, 3856)) == "radix"
    assert rc.binning_path((128, 128, 128)) == "direct"
    assert rc.binning_path((136, 1928, 8)) == "two_level"
    assert rc.binning_path((8, 8, 131072)) == "two_level" and rc.binning_path((8, 8, 131104)) == "radix"
    # chunk policy: the rasterizer's chunk is fixed; the voxelizer's grows past PLAN_CHUNK above PLAN_ITEMS * PLAN_CHUNK
    C, n = rc.K["PLAN_CHUNK"], rc.K["PLAN_ITEMS"]
    assert rc.plan_chunk_for(10 ** 8, C) == C
    assert rc.plan_chunk_for(n * C, rc.K["VOX_CHUNK_CAP"]) == C
    assert rc.plan_chunk_for(n * (C + 1), rc.K["VOX_CHUNK_CAP"]) == 2 * C
    assert rc.plan_chunk_for(10 ** 9, rc.K["VOX_CHUNK_CAP"]) == rc.K["VOX_CHUNK_CAP"]
    # a random cloud: per-CTA sums and the fast flags agree with a direct restatement
    cloud, view = util.case("cone_trained_small")
    orc = util.oracle_raster_forward(cloud, view)
    reg = rc.regime(orc, (view.image_height, view.image_width))
    assert reg["path"] == "direct" and int(reg["cta_total"].sum()) == orc["R"]
    assert reg["cta_total"][0] == int(orc["tiles_touched"][:rc.K["DIRECT_BLOCK"]].sum())
    assert reg["fast"].dtype == bool and reg["fast"].shape == (cloud.P,)
