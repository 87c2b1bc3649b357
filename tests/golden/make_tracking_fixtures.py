"""Generates the tracking clip fixtures under tests/golden/tracks/ from the reference's own test data.

Needs a checkout of the reference project (its tests/data directory):

    python tests/golden/make_tracking_fixtures.py <reference checkout>

Sources (data files only, no reference code is imported or copied):
  tests/data/tracks/clip.mp4               1024x1024, 1500 frames, two flies, stored as 3 equal channels
  tests/data/tracks/clip.predictions.slp   predicted instances (head, thorax) of every frame

Outputs:
  tracks/clip.mp4                          the clip as is
  tracks/clip_predictions.npz              points (frame, instance, node, xy) float32 NaN padded, scores,
                                           n_instances, frame_idx, node_names
"""
import os
import shutil
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from sleap_b200.io.labels import Labels              # noqa: E402


def main():
    if len(sys.argv) != 2 or not os.path.isdir(os.path.join(sys.argv[1], "tests", "data", "tracks")):
        sys.exit("usage: python tests/golden/make_tracking_fixtures.py <reference checkout (with tests/data)>")
    src = os.path.join(sys.argv[1], "tests", "data", "tracks")
    dst = os.path.join(HERE, "tracks")
    os.makedirs(dst, exist_ok=True)
    shutil.copyfile(os.path.join(src, "clip.mp4"), os.path.join(dst, "clip.mp4"))
    labels = Labels.load_file(os.path.join(src, "clip.predictions.slp"))
    n_inst = max(len(lf.instances) for lf in labels)
    n_nodes = len(labels.skeleton.nodes)
    pts = np.full((len(labels), n_inst, n_nodes, 2), np.nan, np.float32)
    scores = np.full((len(labels), n_inst), np.nan, np.float32)
    for i, lf in enumerate(labels):
        for j, inst in enumerate(lf.instances):
            pts[i, j], scores[i, j] = inst.numpy(), inst.score
    np.savez_compressed(os.path.join(dst, "clip_predictions.npz"), points=pts, scores=scores,
                        n_instances=np.asarray([len(lf.instances) for lf in labels], np.int32),
                        frame_idx=np.asarray([lf.frame_idx for lf in labels], np.int64),
                        node_names=np.asarray(labels.skeleton.nodes))
    print("tracks clip", pts.shape)


if __name__ == "__main__":
    main()
