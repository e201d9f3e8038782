"""CPU: oracle/s3fd_ref.py (the fp32 restatement of the S3FD detector and its arg-max selection) against the unmodified
reference's outputs in tests/golden/s3fd_golden.npz (tests/golden/make_s3fd_golden.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import s3fd_ref as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "s3fd_golden.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def sd():
    return R.synth_state_dict(0)


def _heads(g, case):
    return [torch.from_numpy(g[f"{case}_head{k}"]) for k in range(12)]


@pytest.mark.parametrize("case", ["even", "odd"])
def test_forward_matches_reference_heads(g, sd, case):
    frames = g[f"{case}_frames"]
    with torch.no_grad():
        ol = R.forward(sd, R.prep(frames))
    for k, (a, b) in enumerate(zip(ol, _heads(g, case))):
        assert tuple(a.shape) == tuple(b.shape), (k, a.shape, b.shape)
        tol = 1e-4 * (1.0 + b.abs().max())
        assert (a - b).abs().max() <= tol, (k, float((a - b).abs().max()))
    assert [tuple(o.shape[2:]) for o in ol[::2]] == R.head_shapes(*frames.shape[1:3])


@pytest.mark.parametrize("case", ["even", "odd"])
def test_argmax_selection_equals_candidates_and_nms(g, case):
    """On the reference's own head outputs, the arg-max rule gives get_detections_for_batch's result for every image."""
    found, box, score, _ = R.select(_heads(g, case))
    np.testing.assert_array_equal(found, g[f"{case}_found"])
    np.testing.assert_array_equal(box[found], g[f"{case}_box"][found])
    # margins: winning scores clear of the 0.5 threshold, and a batch-mate below 0.5 still contributes candidates
    assert np.all(np.abs(score - 0.5) > 0.1), score
    s, _ = R.scores_and_boxes(_heads(g, case))
    s = s.numpy()
    assert any((~found[i]) and (s[i] > R.CANDIDATE).any() for i in range(len(found))), "no sub-threshold candidates"
    assert found.any() and (~found).any()


def test_gmac_table():
    assert abs(R.gmac_per_frame(720, 1280) - 290.78) < 0.01
    assert R.head_shapes(720, 1280) == [(180, 320), (90, 160), (45, 80), (26, 44), (13, 22), (7, 11)]


def test_package_flop_count_matches_oracle():
    from livetalking_b200 import s3fd
    for H, W in ((720, 1280), (477, 851), (128, 224)):
        assert abs(s3fd.gflop_per_frame(H, W) - 2 * R.gmac_per_frame(H, W)) < 1e-9
