"""oracle/labels.py against the reference's own __getitem__ targets (tests/golden/labels.npz, tools/gen_golden_labels.py)."""
import os

import numpy as np
import pytest

from oracle import labels as ol

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "labels.npz"))
VARIANTS = ["shipped", "all3", "clip2d", "inverse", "none", "meanshape", "val", "e2e"]


@pytest.mark.parametrize("name", VARIANTS)
def test_oracle_reproduces_the_reference_targets(name):
    offsets, recs, P2s = ol.gold_bank(GOLD)
    n = len(GOLD[f"{name}.seeds"])
    got = ol.encode_batch(offsets, recs, P2s, range(n), GOLD["sizes"][:n], GOLD[f"{name}.flip"], GOLD[f"{name}.crop_scale"],
                          GOLD[f"{name}.trans"], **ol.gold_config(GOLD, name))
    ol.assert_targets_match(got, {k: GOLD[f"{name}.{k}"] for k in ol.KEYS}, name)


def test_fixture_covers_the_cases():
    """Every filter of the encoder removes something somewhere, and the slot pattern has gaps and a cut at 50."""
    assert max(GOLD["parsed.count"]) > ol.MAX_OBJS
    cls = [str(c) for c in GOLD["parsed.cls"]]
    assert {"Pedestrian", "Car", "Cyclist", "Van", "DontCare", "Misc"} <= set(cls)
    assert "UnKnown" in set(str(v) for v in GOLD["parsed.level"])
    z = GOLD["parsed.pos"][:, 2]
    assert (z < 2).any() and (z > 65).any()
    lab = GOLD["clip2d.size_2d"][..., 0] != 0
    assert (lab & ~GOLD["clip2d.mask_2d"]).any()                  # kept with mask 0
    assert (GOLD["all3.size_2d"][..., 0] != 0).sum() > (GOLD["all3.boxes"][..., 0] != 0).sum()   # labelled, then cut by l/r/t/b
    assert (GOLD["clip2d.boxes"][..., 0] != 0).sum() > (GOLD["all3.boxes"][..., 0] != 0).sum()
    assert not np.array_equal(GOLD["meanshape.size_3d"], GOLD["meanshape.src_size_3d"])
