"""``Labels`` for the inference path's caller side: ground-truth / predicted instances from a
SLEAP ``.slp`` file, and the ``LabelsReader`` provider the predictors accept.

Restates the *data model* the path consumes, not the reference's editing API:
  sleap/io/format/hdf5.py:132-263    LabelsV1Adaptor.read (tables frames / instances / points / pred_points,
                                     videos_json, metadata attrs["json"] with skeletons + nodes)
  sleap/instance.py:51-117           point record dtypes (x, y, visible, complete[, score])
  sleap/skeleton.py:1416-1480        Skeleton.to_dict / from_dict (jsonpickle graph: nodes by index, links with EdgeType)
  sleap/nn/data/providers.py:11-305  LabelsReader (keys image, raw_image_size, example_ind, video_ind, frame_ind,
                                     scale, instances, skeleton_inds, track_inds, n_tracks)
  sleap/nn/data/instance_centroids.py:12-52, 55-200   InstanceCentroidFinder (bounding-box midpoint or anchor part)
The HDF5 container is read by the in-tree ``h5lite`` reader.
"""
import json
import os
from typing import List, Optional, Sequence

import numpy as np

from sleap_b200.io import h5lite
from sleap_b200.io.video import Video


class Skeleton:
    def __init__(self, node_names: Sequence[str], edges: Sequence[Sequence[str]], symmetries=(), name="Skeleton-0"):
        self.node_names = list(node_names)
        self.edge_names = [tuple(e) for e in edges]
        self.symmetry_names = [tuple(e) for e in symmetries]
        self.name = name

    @property
    def nodes(self):
        return self.node_names

    @property
    def edge_inds(self):
        return [(self.node_names.index(a), self.node_names.index(b)) for a, b in self.edge_names]

    def __len__(self):
        return len(self.node_names)

    @classmethod
    def from_dict(cls, sk: dict, global_nodes: List[dict]):
        """jsonpickle node-link graph: ``nodes[i]["id"]`` indexes the file-level node list; link ``type`` is
        ``EdgeType(1)`` = BODY or ``EdgeType(2)`` = SYMMETRY, later occurrences are ``{"py/id": k}`` back-references
        to the k-th distinct object met while decoding (skeleton.py:31-46 EdgeType, :88-376 SkeletonDecoder)."""
        def node_name(ref):
            if isinstance(ref, dict) and "py/object" in ref:          # inline Node object (older files)
                return ref.get("py/state", {}).get("py/tuple", [ref.get("name")])[0]
            if isinstance(ref, dict):
                ref = ref.get("id", ref.get("py/id"))
            return global_nodes[int(ref)]["name"] if global_nodes else str(ref)

        names = [node_name(n["id"]) for n in sk["nodes"]]
        seen_types = []
        edges, syms = [], []
        for link in sorted(sk.get("links", []), key=lambda l: l.get("edge_insert_idx", 0)):
            t = link.get("type", {})
            if "py/reduce" in t:
                val = int(t["py/reduce"][1]["py/tuple"][0])
                seen_types.append(val)
            elif "py/id" in t:
                val = seen_types[int(t["py/id"]) - 1] if int(t["py/id"]) - 1 < len(seen_types) else 1
            else:
                val = 1
            src = global_nodes[int(link["source"])]["name"] if global_nodes else str(link["source"])
            dst = global_nodes[int(link["target"])]["name"] if global_nodes else str(link["target"])
            (edges if val == 1 else syms).append((src, dst))
        return cls(names, edges, syms, sk.get("graph", {}).get("name", "Skeleton-0"))


class Instance:
    """Points of one animal: ``numpy()`` -> (n_nodes, 2) float32 with NaN for invisible nodes (instance.py:900-950)."""

    def __init__(self, points: np.ndarray, skeleton: Skeleton, track: int = -1, score: float = float("nan"),
                 point_scores: Optional[np.ndarray] = None, predicted: bool = False, tracking_score: float = 0.0):
        self.points = np.asarray(points, np.float32)
        self.skeleton = skeleton
        self.track = track
        self.score = score
        self.point_scores = point_scores
        self.predicted = predicted
        self.tracking_score = tracking_score

    def numpy(self):
        return self.points

    @property
    def n_visible_points(self):
        return int(np.sum(~np.isnan(self.points[:, 0])))


class LabeledFrame:
    def __init__(self, video: int, frame_idx: int, instances: List[Instance]):
        self.video, self.frame_idx, self.instances = video, frame_idx, instances

    def __len__(self):
        return len(self.instances)

    def __getitem__(self, i):
        return self.instances[i]

    @property
    def user_instances(self):
        return [i for i in self.instances if not i.predicted]

    @property
    def predicted_instances(self):
        return [i for i in self.instances if i.predicted]


class Labels:
    def __init__(self, labeled_frames: List[LabeledFrame], videos: List[dict], skeletons: List[Skeleton], tracks=()):
        self.labeled_frames = labeled_frames
        self.video_specs = videos
        self.skeletons = skeletons
        self.tracks = list(tracks)
        self._videos = {}

    def __len__(self):
        return len(self.labeled_frames)

    def __getitem__(self, i):
        return self.labeled_frames[i]

    @property
    def skeleton(self):
        return self.skeletons[0]

    @property
    def videos(self):
        return [self.video(i) for i in range(len(self.video_specs))]

    def video(self, ind: int, search: Sequence[str] = ()) -> Video:
        """Opens the video of ``videos_json[ind]`` (path as stored, then relative to each ``search`` directory by
        basename, like ``Labels.load_file(video_search=...)``, sleap/io/dataset.py:1990-2050)."""
        if ind in self._videos:
            return self._videos[ind]
        be = self.video_specs[ind].get("backend", {})
        fn = be.get("filename", "")
        cands = [fn] + [os.path.join(d, os.path.basename(fn)) for d in search]
        for c in cands:
            if c and os.path.exists(c):
                self._videos[ind] = Video.from_filename(c, grayscale=be.get("grayscale"), bgr=be.get("bgr", True))
                return self._videos[ind]
        raise FileNotFoundError(f"video {fn!r} not found (searched {list(search)})")

    def set_video(self, ind: int, video: Video):
        self._videos[ind] = video

    def save_file(self, filename: str):
        save_file(self, filename)

    save = save_file

    @classmethod
    def load_file(cls, filename: str, video_search: Sequence[str] = ()):
        if not str(filename).endswith((".slp", ".h5", ".hdf5")):
            raise ValueError("only the HDF5 .slp labels format is read here")
        f = h5lite.File(filename)
        meta = f["metadata"].attrs["json"]
        meta = json.loads(meta.decode() if isinstance(meta, (bytes, np.bytes_)) else meta)
        gnodes = meta.get("nodes", [])
        skeletons = [Skeleton.from_dict(s, gnodes) for s in meta.get("skeletons", [])]
        vj = f["videos_json"].read() if "videos_json" in f else []
        videos = [json.loads(v.decode() if isinstance(v, (bytes, np.bytes_)) else v) for v in np.atleast_1d(vj)] if len(vj) else []
        frames, inst = f["frames"].read(), f["instances"].read()
        pts, ppts = f["points"].read(), f["pred_points"].read()
        # hdf5.py:143-155: user points of files older than format 1.1 were saved on a gridline coordinate system;
        # tracking_score exists from format 1.2 on (:221-224)
        fid = f["metadata"].attrs.get("format_id") if hasattr(f["metadata"].attrs, "get") else None
        try:
            format_id = None if fid is None else float(np.asarray(fid).reshape(-1)[0])
        except (TypeError, ValueError):
            format_id = None
        if (format_id or 0) < 1.1 and len(pts):
            pts = pts.copy()
            pts["x"] = pts["x"] - 0.5
            pts["y"] = pts["y"] - 0.5
        has_ts = format_id is not None and format_id >= 1.2 and "tracking_score" in (inst.dtype.names or ())
        lfs = []
        for fr in frames:
            ins = []
            for i in range(int(fr["instance_id_start"]), int(fr["instance_id_end"])):
                row = inst[i]
                sk = skeletons[int(row["skeleton"])] if skeletons else None
                predicted = int(row["instance_type"]) == 1            # 0 = user Instance, 1 = PredictedInstance
                table = ppts if predicted else pts
                p = table[int(row["point_id_start"]):int(row["point_id_end"])]
                xy = np.stack([p["x"], p["y"]], -1).astype(np.float32)
                xy[p["visible"] == 0] = np.nan
                ins.append(Instance(xy, sk, int(row["track"]), float(row["score"]),
                                    p["score"].astype(np.float32) if predicted else None, predicted,
                                    float(row["tracking_score"]) if (predicted and has_ts) else 0.0))
            lfs.append(LabeledFrame(int(fr["video"]), int(fr["frame_idx"]), ins))
        tracks = meta.get("tracks", [])
        if "tracks_json" in f:                                   # one '[spawned_on,"name"]' string per track (hdf5.py:150-160)
            tj = f["tracks_json"].read()
            if len(tj) and getattr(tj, "dtype", np.dtype("f8")).kind == "S":
                tracks = [json.loads(t.decode()) for t in tj]
        lab = cls(lfs, videos, skeletons, tracks)
        lab._search = list(video_search)
        return lab


# Table dtypes of the .slp container (sleap/instance.py:51-58, 115-117; sleap/io/format/hdf5.py:330-420)
FRAME_DTYPE = np.dtype([("frame_id", "u8"), ("video", "u4"), ("frame_idx", "u8"), ("instance_id_start", "u8"), ("instance_id_end", "u8")])
INSTANCE_DTYPE = np.dtype([("instance_id", "i8"), ("instance_type", "u1"), ("frame_id", "u8"), ("skeleton", "u4"), ("track", "i4"),
                           ("from_predicted", "i8"), ("score", "f4"), ("point_id_start", "u8"), ("point_id_end", "u8"),
                           ("tracking_score", "f4")])
POINT_DTYPE = np.dtype([("x", "f8"), ("y", "f8"), ("visible", "?"), ("complete", "?")])
PRED_POINT_DTYPE = np.dtype([("x", "f8"), ("y", "f8"), ("visible", "?"), ("complete", "?"), ("score", "f8")])


def skeleton_to_dict(sk: Skeleton, node_index: dict) -> dict:
    """Inverse of ``Skeleton.from_dict``: the jsonpickle node-link form ``Skeleton.to_dict`` / ``SkeletonEncoder`` write (skeleton.py:378-582, 1416-1437):
    the first EdgeType of each kind is spelled out (``py/reduce``), later ones are ``py/id`` back-references."""
    seen = {}
    links = []

    def etype(val):
        if val not in seen:
            seen[val] = len(seen) + 1
            return {"py/reduce": [{"py/type": "sleap.skeleton.EdgeType"}, {"py/tuple": [val]}]}
        return {"py/id": seen[val]}

    for i, (a, b) in enumerate(sk.edge_names):
        links.append({"edge_insert_idx": i, "key": 0, "source": node_index[a], "target": node_index[b], "type": etype(1)})
    for a, b in sk.symmetry_names:
        links.append({"key": 0, "source": node_index[a], "target": node_index[b], "type": etype(2)})
    return {"directed": True, "graph": {"name": sk.name, "num_edges_inserted": len(sk.edge_names)}, "links": links, "multigraph": True,
            "nodes": [{"id": node_index[n]} for n in sk.node_names]}


def save_file(labels: "Labels", filename: str):
    """Writes the ``.slp`` (HDF5) container ``LabelsV1Adaptor.write`` produces (sleap/io/format/hdf5.py:265-575,
    format 1.2): ``metadata`` group (attrs ``format_id``, ``json``), ``videos_json`` / ``tracks_json`` /
    ``suggestions_json`` and the ``frames`` / ``instances`` / ``points`` / ``pred_points`` tables; predicted instances
    carry per-point scores and an instance score.  Written with the in-tree ``h5write`` (no h5py)."""
    from sleap_b200.io import h5write
    sk_list = labels.skeletons
    node_names = []
    for sk in sk_list:
        for n in sk.node_names:
            if n not in node_names:
                node_names.append(n)
    node_index = {n: i for i, n in enumerate(node_names)}
    meta = {"version": "2.0.0", "skeletons": [skeleton_to_dict(sk, node_index) for sk in sk_list],
            "nodes": [{"name": n, "weight": 1.0} for n in node_names], "videos": [], "tracks": [], "suggestions": [],
            "negative_anchors": {}, "provenance": {"writer": "sleap_b200"}}
    frames = np.zeros(len(labels.labeled_frames), FRAME_DTYPE)
    n_inst = sum(len(lf.instances) for lf in labels.labeled_frames)
    inst = np.zeros(n_inst, INSTANCE_DTYPE)
    pts, ppts = [], []
    ii = 0
    for fi, lf in enumerate(labels.labeled_frames):
        frames[fi] = (fi, lf.video, lf.frame_idx, ii, ii + len(lf.instances))
        for ins in lf.instances:
            xy = np.asarray(ins.numpy(), np.float64)
            vis = ~np.isnan(xy[:, 0])
            table = ppts if ins.predicted else pts
            start = sum(len(t) for t in table)
            if ins.predicted:
                sc = np.asarray(ins.point_scores if ins.point_scores is not None else np.zeros(len(xy)), np.float64)
                rec = np.zeros(len(xy), PRED_POINT_DTYPE)
                rec["score"] = np.where(vis, sc, 0.0)
            else:
                rec = np.zeros(len(xy), POINT_DTYPE)
            rec["x"], rec["y"], rec["visible"], rec["complete"] = xy[:, 0], xy[:, 1], vis, False if ins.predicted else vis
            table.append(rec)
            sk_ind = sk_list.index(ins.skeleton) if ins.skeleton in sk_list else 0
            inst[ii] = (ii, 1 if ins.predicted else 0, fi, sk_ind, ins.track, -1, ins.score if ins.predicted else np.nan, start,
                        start + len(xy), float(getattr(ins, "tracking_score", 0.0) or 0.0) if ins.predicted else 0.0)
            ii += 1
    videos = [json.dumps(v, separators=(",", ":")).encode() for v in labels.video_specs]

    def strings(rows):
        return np.asarray(rows, dtype=f"S{max(len(r) for r in rows)}") if rows else np.zeros(0, np.float64)

    with h5write.File(filename) as f:
        g = f.create_group("metadata")
        g.attrs["format_id"] = np.float64(1.2)
        g.attrs["json"] = json.dumps(meta, separators=(",", ":"))
        f.create_dataset("videos_json", strings(videos))
        f.create_dataset("tracks_json", strings([json.dumps(list(t), separators=(",", ":")).encode() for t in labels.tracks]))
        f.create_dataset("suggestions_json", np.zeros(0, np.float64))
        f.create_dataset("frames", frames)
        f.create_dataset("instances", inst)
        f.create_dataset("points", np.concatenate(pts) if pts else np.zeros(0, POINT_DTYPE))
        f.create_dataset("pred_points", np.concatenate(ppts) if ppts else np.zeros(0, PRED_POINT_DTYPE))


def labels_from_predictions(frames, skeleton: Skeleton, video_spec: Optional[dict] = None, video_filename: str = "") -> "Labels":
    """``Predictor.predict(..., make_labels=True)`` output (``LabeledFrame`` / ``PredictedInstance`` of
    sleap_b200.nn.inference) -> ``Labels`` that ``save_file`` can write (sleap/nn/inference.py:3230-3343)."""
    spec = video_spec or {"backend": {"filename": video_filename, "grayscale": True, "bgr": True, "dataset": "", "input_format": ""}}
    lfs, track_ids, tracks = [], {}, []
    for fr in frames:
        ins = []
        for i in fr.instances:
            tr = getattr(i, "track", None)
            ti = -1
            if tr is not None:                                   # sleap_b200.nn.tracking.Track objects -> [spawned_on, name] rows
                if id(tr) not in track_ids:
                    track_ids[id(tr)] = len(tracks)
                    tracks.append([int(getattr(tr, "spawned_on", 0)), str(getattr(tr, "name", f"track_{len(tracks)}"))])
                ti = track_ids[id(tr)]
            ins.append(Instance(i.numpy(), skeleton, ti, float(i.score), np.asarray(i.point_confidences, np.float32), True,
                                float(getattr(i, "tracking_score", 0.0) or 0.0)))
        lfs.append(LabeledFrame(int(fr.video) if isinstance(fr.video, (int, np.integer)) else 0, int(fr.frame_idx), ins))
    return Labels(lfs, [spec], [skeleton], tracks)


def find_points_bbox_midpoint(points: np.ndarray) -> np.ndarray:
    """instance_centroids.py:12-33: NaN-ignoring bounding-box midpoint over the node axis."""
    lo = np.min(np.where(np.isnan(points), np.inf, points), axis=-2)
    hi = np.max(np.where(np.isnan(points), -np.inf, points), axis=-2)
    return ((hi + lo) * np.float32(0.5)).astype(np.float32)


def find_instance_centroids(instances: np.ndarray, anchor_ind: Optional[int] = None) -> np.ndarray:
    """instance_centroids.py:137-200 ``InstanceCentroidFinder.transform_dataset``: the anchor node where it is visible, else the
    bounding-box midpoint of the visible nodes."""
    instances = np.asarray(instances, np.float32)
    mid = find_points_bbox_midpoint(instances)
    if anchor_ind is None:
        return mid
    anchors = instances[:, anchor_ind, :]
    ok = ~np.isnan(anchors).any(axis=-1, keepdims=True)
    return np.where(ok, anchors, mid).astype(np.float32)


class LabelsReader:
    """Provider over ``Labels`` (providers.py:23-300): examples carry the frame and its instances; with
    ``center_on_part`` set (or ``with_centroids=True``) also ``centroids`` (InstanceCentroidFinder,
    instance_centroids.py:55-200), which the ground-truth stand-in layers of the top-down model consume."""

    def __init__(self, labels: Labels, example_indices: Optional[Sequence[int]] = None, user_instances_only: bool = False,
                 with_centroids: bool = False, center_on_part: Optional[str] = None, video_search: Sequence[str] = ()):
        self.labels = labels
        self.example_indices = example_indices
        self.user_instances_only = user_instances_only
        self.with_centroids = with_centroids or center_on_part is not None
        self.center_on_part = center_on_part
        self.video_search = list(video_search) or list(getattr(labels, "_search", []))

    @classmethod
    def from_user_instances(cls, labels: Labels, **kw):
        return cls(labels, user_instances_only=True, **kw)

    @classmethod
    def from_filename(cls, filename: str, **kw):
        return cls(Labels.load_file(filename), **kw)

    @property
    def output_keys(self):
        keys = ["image", "raw_image_size", "example_ind", "video_ind", "frame_ind", "scale", "instances", "skeleton_inds",
                "track_inds", "n_tracks"]
        return keys + (["centroids"] if self.with_centroids else [])

    def indices(self):
        if self.example_indices is None:
            return list(range(len(self.labels)))
        return [int(i) for i in self.example_indices]

    def __len__(self):
        return len(self.indices())

    @property
    def videos(self):
        return self.labels.videos

    def _instances(self, lf):
        return lf.user_instances if self.user_instances_only else lf.instances

    def max_instance_count(self) -> int:
        """The most instances (= ground-truth centroids) of any frame the reader yields, read from the labels alone:
        no frame is decoded."""
        return max([len(self._instances(self.labels[i])) for i in self.indices()] + [0])

    def example(self, ind: int) -> dict:
        lf = self.labels[ind]
        video = self.labels.video(lf.video, self.video_search)
        img = video.get_frame(lf.frame_idx)
        insts = self._instances(lf)
        n_nodes = len(self.labels.skeleton) if self.labels.skeletons else (insts[0].points.shape[0] if insts else 0)
        pts = np.stack([i.numpy() for i in insts]) if insts else np.zeros((0, n_nodes, 2), np.float32)
        ex = {"image": img, "raw_image_size": np.asarray(img.shape, np.int32), "example_ind": np.int64(ind),
              "video_ind": np.int32(lf.video), "frame_ind": np.int64(lf.frame_idx), "scale": np.ones(2, np.float32),
              "instances": pts.astype(np.float32), "skeleton_inds": np.zeros(len(insts), np.int32),
              "track_inds": np.asarray([i.track for i in insts], np.int32), "n_tracks": np.int32(len(self.labels.tracks))}
        if self.with_centroids:
            anchor = None
            if self.center_on_part is not None:
                anchor = self.labels.skeleton.node_names.index(self.center_on_part)
            ex["centroids"] = find_instance_centroids(pts, anchor) if len(pts) else np.zeros((0, 2), np.float32)
        return ex

    def __iter__(self):
        for i in self.indices():
            yield self.example(i)

    make_dataset = __iter__
