"""oracle/postprocess.py (restatement of voxel_postprocessor.post_process + box_utils helpers) against
tests/golden/postprocess.pt, produced by the UNMODIFIED reference VoxelPostprocessor (oracle/make_golden.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import golden

from oracle import postprocess as opp


@pytest.fixture(scope="module")
def gold(golden_dir):
    return golden.load(os.path.join(golden_dir, "postprocess.pt"))


def test_anchor_box_matches_reference(gold):
    a = opp.generate_anchor_box(gold["params"]["anchor_args"], gold["params"]["order"])
    assert a.shape == tuple(gold["anchors"].shape)
    assert np.array_equal(a, gold["anchors"].numpy())


@pytest.mark.parametrize("case", ["dense", "sparse"])
def test_post_process_matches_reference(gold, case):
    c = gold["cases"][case]
    boxes, scores = opp.post_process(c["cls"].clone(), c["reg"].clone(), c["dir"].clone(), gold["anchors"], c["T"], gold["params"])
    assert boxes.shape == c["boxes"].shape and boxes.shape[0] > 0
    assert torch.equal(boxes, c["boxes"]) and torch.equal(scores, c["scores"])


def test_quad_intersection_known_answers():
    sq = np.array([[0, 0], [2, 0], [2, 2], [0, 2]], dtype=np.float64)
    assert opp.quad_intersection_area(sq, sq) == pytest.approx(4.0)
    assert opp.quad_intersection_area(sq, sq + [1, 1]) == pytest.approx(1.0)
    assert opp.quad_intersection_area(sq, sq + [3, 0]) == 0.0
    assert opp.quad_intersection_area(sq, sq[::-1] + [1, 0]) == pytest.approx(2.0)            # clockwise input
    d = np.array([[1, -1], [3, 1], [1, 3], [-1, 1]], dtype=np.float64)                        # diamond, area 8, centred on (1,1)
    assert opp.quad_intersection_area(sq, d) == pytest.approx(4.0)
    p, q = opp.QuadPolygon(sq), opp.QuadPolygon(sq + [1, 1])
    assert p.intersection(q).area / p.union(q).area == pytest.approx(1.0 / 7.0)
