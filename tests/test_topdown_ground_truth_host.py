"""Host side of the ground-truth top-down step: the centroid table sb_topdown_gt_submit takes, and the per-run K a
labels reader gives (its largest instance count, read from the labels without decoding a frame)."""
import numpy as np
import pytest
from numpy.testing import assert_array_equal

F = np.float32


def test_centroid_table_packing():
    from sleap_b200.nn.inference import _centroid_table
    cents = [np.array([[1.5, 2.5], [3, 4]], F), np.zeros((0, 2), F), [[np.nan, np.nan]], np.array([[-7.25, 1e6]], np.float64)]
    table, counts = _centroid_table(cents, 3)
    assert table.dtype == F and table.shape == (4, 3, 2) and table.flags.c_contiguous
    assert counts.dtype == np.int32 and counts.tolist() == [2, 0, 1, 1]
    assert_array_equal(table[0, :2], cents[0])
    assert_array_equal(table[3, 0], F([-7.25, 1e6]))
    assert np.isnan(table[2, 0]).all()                               # an all-NaN labelled instance stays one centroid
    for b, n in enumerate(counts):
        assert np.isnan(table[b, n:]).all()
    # more centroids than K: the count is kept, so the submit refuses the batch instead of dropping centroids
    table, counts = _centroid_table([np.arange(8, dtype=F).reshape(4, 2)], 2)
    assert table.shape == (1, 2, 2) and counts.tolist() == [4]
    table, counts = _centroid_table([], 1)
    assert table.shape == (0, 1, 2) and counts.shape == (0,)


class _NoDecode:
    """A video that must not be read."""

    shape = (3, 8, 8, 1)

    def get_frame(self, idx):
        raise AssertionError("frame decoded")


def _labels():
    from sleap_b200.io.labels import Instance, LabeledFrame, Labels, Skeleton
    sk = Skeleton(["a", "b"], [("a", "b")])
    pts = np.array([[1, 2], [3, 4]], F)
    user = lambda: Instance(pts, sk)                                  # noqa: E731
    pred = lambda: Instance(pts, sk, predicted=True)                  # noqa: E731
    lfs = [LabeledFrame(0, 0, [user(), pred(), pred(), pred()]),     # 1 user, 4 in all
           LabeledFrame(0, 1, [user(), user(), pred()]),             # 2 user, 3 in all
           LabeledFrame(0, 2, [])]
    lab = Labels(lfs, [{}], [sk])
    lab.set_video(0, _NoDecode())
    return lab


@pytest.mark.parametrize("user_only,indices,want", [(False, None, 4), (True, None, 2), (False, [1, 2], 3), (True, [0, 2], 1),
                                                   (False, [2], 0), (False, [], 0)])
def test_max_instance_count(user_only, indices, want):
    from sleap_b200.io.labels import LabelsReader
    r = LabelsReader(_labels(), example_indices=indices, user_instances_only=user_only, with_centroids=True)
    assert r.max_instance_count() == want


def test_max_instance_count_is_the_examples_largest_centroid_count():
    from sleap_b200.io.labels import LabelsReader
    from sleap_b200.io.video import Video
    lab = _labels()
    lab.set_video(0, Video.from_numpy(np.zeros((3, 8, 8, 1), np.uint8)))
    for user_only in (False, True):
        r = LabelsReader(lab, user_instances_only=user_only, with_centroids=True)
        assert r.max_instance_count() == max(len(e["centroids"]) for e in r)
