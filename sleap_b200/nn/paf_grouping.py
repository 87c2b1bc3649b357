"""Drop-in for ``sleap.nn.paf_grouping`` (reference: sleap/nn/paf_grouping.py).

Same function names and argument order.  tf.RaggedTensors become Python lists of per-sample
NumPy arrays.  Scoring, matching (SciPy-compatible rectangular LSAP) and greedy grouping run as
sm_90a kernels behind the C-ABI; host code only does index bookkeeping and edge ordering.
"""
from typing import List, Tuple

import numpy as np

from sleap_b200 import _lib
from sleap_b200._lib import f32, i32, ptr


def get_connection_candidates(peak_channel_inds_sample, skeleton_edges, n_nodes):
    """sleap/nn/paf_grouping.py:82-142 (pure index bookkeeping, host side)."""
    ch = i32(peak_channel_inds_sample).reshape(-1)
    edges = i32(skeleton_edges).reshape(-1, 2)
    order = np.argsort(ch, kind="stable").astype(np.int32)
    grouped = [order[ch[order] == k] for k in range(n_nodes)]
    ei, epi = [], []
    for k in range(edges.shape[0]):
        s, d = np.meshgrid(grouped[edges[k, 0]], grouped[edges[k, 1]], indexing="ij")
        sd = np.stack([s, d], axis=2).reshape(-1, 2)
        ei.append(np.full((sd.shape[0],), k, np.int32))
        epi.append(sd.astype(np.int32))
    if not ei:
        return np.zeros((0,), np.int32), np.zeros((0, 2), np.int32)
    return np.concatenate(ei), np.concatenate(epi).reshape(-1, 2)


def _lines(pafs_sample, lines_in, peaks_sample, edge_peak_inds, edge_inds, n_line_points, pafs_stride,
           max_edge_length, dist_penalty_weight, handle=None):
    h = handle or _lib.default_handle()
    peaks = f32(peaks_sample).reshape(-1, 2)
    epi = i32(edge_peak_inds).reshape(-1, 2)
    n = epi.shape[0]
    P = int(n_line_points)
    ei = None if edge_inds is None else i32(edge_inds).reshape(-1)
    subs = np.zeros((n, P, 2), np.int32)
    lines = np.zeros((n, P, 2), np.float32)
    scores = np.zeros((n,), np.float32)
    if pafs_sample is not None:
        pafs = f32(pafs_sample)
        Hp, Wp, C2 = pafs.shape
    else:
        pafs, Hp, Wp, C2 = None, 0, 0, 0
    lin = None if lines_in is None else f32(lines_in).reshape(n, P, 2)
    if n > 0:
        h.call("sb_paf_lines", ptr(pafs), Hp, Wp, C2, ptr(lin), ptr(peaks), peaks.shape[0], ptr(epi), ptr(ei), n, P,
               int(pafs_stride), float(max_edge_length), float(dist_penalty_weight), ptr(subs), ptr(lines), ptr(scores))
    return subs, lines, scores


def make_line_subs(peaks_sample, edge_peak_inds, edge_inds, n_line_points, pafs_stride, handle=None):
    """sleap/nn/paf_grouping.py:145-222 -> (n, P, 2, 3) [row, col, channel]."""
    subs, _, _ = _lines(None, None, peaks_sample, edge_peak_inds, edge_inds, n_line_points, pafs_stride, 1.0, 1.0,
                        handle)
    ei = i32(edge_inds).reshape(-1, 1, 1)
    ch = np.broadcast_to(ei, subs.shape[:2] + (1,))
    a = np.concatenate([subs, ch * 2], axis=2)
    b = np.concatenate([subs, ch * 2 + 1], axis=2)
    return np.stack([a, b], axis=2).astype(np.int32)


def get_paf_lines(pafs_sample, peaks_sample, edge_peak_inds, edge_inds, n_line_points, pafs_stride, handle=None):
    """sleap/nn/paf_grouping.py:225-275 -> (n, P, 2).  Out-of-range samples read 0 (TF-GPU
    gather_nd semantics; the reference's TF-CPU path raises, see its TODO at :197)."""
    _, lines, _ = _lines(pafs_sample, None, peaks_sample, edge_peak_inds, edge_inds, n_line_points, pafs_stride,
                         1.0, 1.0, handle)
    return lines


def compute_distance_penalty(spatial_vec_lengths, max_edge_length, dist_penalty_weight=1.0, handle=None):
    """sleap/nn/paf_grouping.py:278-322 (evaluated by the line-scoring kernel on zero lines)."""
    l = f32(spatial_vec_lengths)
    flat = l.reshape(-1)
    n = flat.shape[0]
    peaks = np.zeros((2 * n, 2), np.float32)
    peaks[1::2, 0] = flat
    epi = np.stack([np.arange(n) * 2, np.arange(n) * 2 + 1], axis=1).astype(np.int32)
    _, _, sc = _lines(None, np.zeros((n, 1, 2), np.float32), peaks, epi, None, 1, 1, max_edge_length,
                      dist_penalty_weight, handle)
    return sc.reshape(l.shape)


def score_paf_lines(paf_lines_sample, peaks_sample, edge_peak_inds_sample, max_edge_length,
                    dist_penalty_weight=1.0, handle=None):
    """sleap/nn/paf_grouping.py:325-403."""
    lines = f32(paf_lines_sample)
    _, _, sc = _lines(None, lines, peaks_sample, edge_peak_inds_sample, None, lines.shape[1], 1, max_edge_length,
                      dist_penalty_weight, handle)
    return sc


def score_paf_lines_batch(pafs, peaks, peak_channel_inds, skeleton_edges, n_line_points, pafs_stride,
                          max_edge_length_ratio, dist_penalty_weight, n_nodes, handle=None):
    """sleap/nn/paf_grouping.py:406-550.  Returns per-sample lists (edge_inds, edge_peak_inds, line_scores)."""
    h = handle or _lib.default_handle()
    pafs = f32(pafs)
    B, Hp, Wp, C2 = pafs.shape
    edges = i32(skeleton_edges).reshape(-1, 2)
    counts = [len(np.asarray(p).reshape(-1, 2)) for p in peaks]
    offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    allp = f32(np.concatenate([np.asarray(p, np.float32).reshape(-1, 2) for p in peaks])) if offs[-1] else np.zeros((0, 2), np.float32)
    allc = i32(np.concatenate([np.asarray(c, np.int32).reshape(-1) for c in peak_channel_inds])) if offs[-1] else np.zeros((0,), np.int32)
    cap = 0
    for b in range(B):
        cb = np.bincount(allc[offs[b]:offs[b + 1]], minlength=n_nodes)
        cap += int(sum(cb[s] * cb[d] for s, d in edges))
    cap = max(cap, 1)
    ei = np.zeros((cap,), np.int32)
    epi = np.zeros((cap, 2), np.int32)
    ls = np.zeros((cap,), np.float32)
    co = np.zeros((B + 1,), np.int32)
    h.call("sb_score_paf_lines_batch", ptr(pafs), B, Hp, Wp, C2, ptr(allp), ptr(allc), ptr(offs), ptr(edges),
           edges.shape[0], int(n_nodes), int(n_line_points), int(pafs_stride), float(max_edge_length_ratio),
           float(dist_penalty_weight), cap, ptr(ei), ptr(epi), ptr(ls), ptr(co))
    sl = [slice(co[b], co[b + 1]) for b in range(B)]
    return [ei[s].copy() for s in sl], [epi[s].copy() for s in sl], [ls[s].copy() for s in sl]


def linear_sum_assignment(cost_matrix, handle=None):
    """sleap/nn/utils.py:79-98 (cost matrix in; SciPy-compatible result)."""
    cost = f32(cost_matrix)
    r, c, _ = _lsap_scores([-cost], handle)[0]
    return r, c


def _lsap_scores(score_mats, handle=None):
    h = handle or _lib.default_handle()
    n = len(score_mats)
    if n == 0:
        return []
    ns = i32([m.shape[0] for m in score_mats])
    nd = i32([m.shape[1] for m in score_mats])
    sizes = ns.astype(np.int64) * nd
    offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int32)
    flat = f32(np.concatenate([np.asarray(m, np.float32).reshape(-1) for m in score_mats] + [np.zeros((1,), np.float32)]))
    K = int(max(1, ns.max(), nd.max()))
    rows = np.zeros((n, K), np.int32)
    cols = np.zeros((n, K), np.int32)
    sc = np.zeros((n, K), np.float32)
    cnt = np.zeros((n,), np.int32)
    h.call("sb_linear_sum_assignment_batch", ptr(flat), ptr(ns), ptr(nd), ptr(offs), n, K, ptr(rows), ptr(cols),
           ptr(sc), ptr(cnt))
    return [(rows[p, :cnt[p]].copy(), cols[p, :cnt[p]].copy(), sc[p, :cnt[p]].copy()) for p in range(n)]


def _edge_problems(edge_inds_sample, edge_peak_inds_sample, line_scores_sample, n_edges):
    ei = i32(edge_inds_sample).reshape(-1)
    epi = i32(edge_peak_inds_sample).reshape(-1, 2)
    ls = f32(line_scores_sample).reshape(-1)
    mats = []
    for k in range(n_edges):
        sel = np.nonzero(ei == k)[0]
        n_src = len(np.unique(epi[sel, 0]))
        n_dst = len(np.unique(epi[sel, 1]))
        mats.append(ls[sel].reshape(n_src, n_dst))
    return mats


def match_candidates_sample(edge_inds_sample, edge_peak_inds_sample, line_scores_sample, n_edges, handle=None):
    """sleap/nn/paf_grouping.py:553-670 (edge-LOCAL indices out)."""
    res = match_candidates_batch([edge_inds_sample], [edge_peak_inds_sample], [line_scores_sample], n_edges, handle)
    return tuple(r[0] for r in res)


def match_candidates_batch(edge_inds, edge_peak_inds, line_scores, n_edges, handle=None):
    """sleap/nn/paf_grouping.py:673-796."""
    B = len(edge_inds)
    mats = []
    for b in range(B):
        mats.extend(_edge_problems(edge_inds[b], edge_peak_inds[b], line_scores[b], n_edges))
    sols = _lsap_scores(mats, handle)
    me, ms, md, msc = [], [], [], []
    for b in range(B):
        e_l, s_l, d_l, sc_l = [], [], [], []
        for k in range(n_edges):
            r, c, s = sols[b * n_edges + k]
            e_l.append(np.full((len(r),), k, np.int32))
            s_l.append(r)
            d_l.append(c)
            sc_l.append(s)
        cat = lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.zeros((0,), dt)
        me.append(cat(e_l, np.int32)); ms.append(cat(s_l, np.int32)); md.append(cat(d_l, np.int32)); msc.append(cat(sc_l, np.float32))
    return me, ms, md, msc


def group_instances_sample(peaks_sample, peak_scores_sample, peak_channel_inds_sample, match_edge_inds_sample,
                           match_src_peak_inds_sample, match_dst_peak_inds_sample, match_line_scores_sample,
                           n_nodes, sorted_edge_inds, edge_types, min_instance_peaks, min_line_scores=0.25,
                           handle=None):
    """sleap/nn/paf_grouping.py:984-1112."""
    res = group_instances_batch([peaks_sample], [peak_scores_sample], [peak_channel_inds_sample],
                                [match_edge_inds_sample], [match_src_peak_inds_sample],
                                [match_dst_peak_inds_sample], [match_line_scores_sample], n_nodes,
                                sorted_edge_inds, edge_types, min_instance_peaks, min_line_scores, handle)
    return tuple(r[0] for r in res)


def group_instances_batch(peaks, peak_vals, peak_channel_inds, match_edge_inds, match_src_peak_inds,
                          match_dst_peak_inds, match_line_scores, n_nodes, sorted_edge_inds, edge_types,
                          min_instance_peaks, min_line_scores=0.25, handle=None):
    """sleap/nn/paf_grouping.py:1115-1290."""
    h = handle or _lib.default_handle()
    B = len(peaks)
    cat = lambda xs, dt, w=None: (np.ascontiguousarray(np.concatenate([np.asarray(x, dt).reshape((-1,) + ((w,) if w else ())) for x in xs]))
                                   if len(xs) else np.zeros((0,) + ((w,) if w else ()), dt))
    pc = [len(np.asarray(p).reshape(-1, 2)) for p in peaks]
    po = np.concatenate([[0], np.cumsum(pc)]).astype(np.int32)
    mc = [len(np.asarray(m).reshape(-1)) for m in match_edge_inds]
    mo = np.concatenate([[0], np.cumsum(mc)]).astype(np.int32)
    P, PV, PC = cat(peaks, np.float32, 2), cat(peak_vals, np.float32), cat(peak_channel_inds, np.int32)
    ME, MS, MD, MSC = (cat(match_edge_inds, np.int32), cat(match_src_peak_inds, np.int32),
                       cat(match_dst_peak_inds, np.int32), cat(match_line_scores, np.float32))
    et = i32([[int(a), int(b)] for a, b in edge_types]).reshape(-1, 2)
    se = i32(list(sorted_edge_inds))
    if isinstance(min_instance_peaks, float):
        min_instance_peaks = int(min_instance_peaks * n_nodes)   # paf_grouping.py:900-901
    max_inst = max(1, max(pc) if pc else 1)
    inst = np.zeros((B, max_inst, n_nodes, 2), np.float32)
    ps = np.zeros((B, max_inst, n_nodes), np.float32)
    isc = np.zeros((B, max_inst), np.float32)
    ni = np.zeros((B,), np.int32)
    pad = lambda a: a if a.size else np.zeros((1,) + a.shape[1:], a.dtype)
    h.call("sb_group_instances_batch", B, int(n_nodes), ptr(pad(P)), ptr(pad(PV)), ptr(pad(PC)), ptr(po),
           ptr(pad(ME)), ptr(pad(MS)), ptr(pad(MD)), ptr(pad(MSC)), ptr(mo), ptr(et), et.shape[0], ptr(pad(se)),
           len(se), int(min_instance_peaks), float(min_line_scores), max_inst, ptr(inst), ptr(ps), ptr(isc), ptr(ni))
    return ([inst[b, :ni[b]].copy() for b in range(B)], [ps[b, :ni[b]].copy() for b in range(B)],
            [isc[b, :ni[b]].copy() for b in range(B)])


def toposort_edges(edge_types) -> Tuple[int, ...]:
    """sleap/nn/paf_grouping.py:1293-1315 without NetworkX: root = first node (insertion order)
    of a topological sort; edges in BFS order from it (nx.topological_sort -> nx.bfs_edges)."""
    edges = [(int(a), int(b)) for a, b in edge_types]
    nodes, adj, indeg = [], {}, {}
    for a, b in edges:
        for n in (a, b):
            if n not in adj:
                adj[n] = []
                indeg[n] = 0
                nodes.append(n)
        if b not in adj[a]:
            adj[a].append(b)
            indeg[b] += 1
    zero = [n for n in nodes if indeg[n] == 0]
    if not zero:
        raise ValueError("Graph contains a cycle.")
    root = zero[0]
    out, seen, queue = [], {root}, [root]
    while queue:
        u = queue.pop(0)
        for v in adj[u]:
            if v not in seen:
                seen.add(v)
                out.append(edges.index((u, v)))
                queue.append(v)
    return tuple(out)


class PAFScorer:
    """sleap/nn/paf_grouping.py:1318-1705."""

    def __init__(self, part_names, edges, pafs_stride, max_edge_length_ratio=0.25, dist_penalty_weight=1.0,
                 n_points=10, min_instance_peaks=0, min_line_scores=0.25):
        self.part_names = list(part_names)
        self.edges = [tuple(e) for e in edges]
        self.pafs_stride = pafs_stride
        self.max_edge_length_ratio = max_edge_length_ratio
        self.dist_penalty_weight = dist_penalty_weight
        self.n_points = n_points
        self.min_instance_peaks = min_instance_peaks
        self.min_line_scores = min_line_scores
        self.edge_inds = [(self.part_names.index(s), self.part_names.index(d)) for s, d in self.edges]
        self.edge_types = list(self.edge_inds)
        self.n_nodes = len(self.part_names)
        self.n_edges = len(self.edges)
        self.sorted_edge_inds = toposort_edges(self.edge_types)

    @classmethod
    def from_config(cls, config, max_edge_length_ratio=0.25, dist_penalty_weight=1.0, n_points=10,
                    min_instance_peaks=0, min_line_scores=0.25):
        """config: the ``multi_instance`` head dict of a training_config.json."""
        return cls(part_names=config["confmaps"]["part_names"], edges=config["pafs"]["edges"],
                   pafs_stride=config["pafs"]["output_stride"], max_edge_length_ratio=max_edge_length_ratio,
                   dist_penalty_weight=dist_penalty_weight, n_points=n_points,
                   min_instance_peaks=min_instance_peaks, min_line_scores=min_line_scores)

    def score_paf_lines(self, pafs, peaks, peak_channel_inds):
        return score_paf_lines_batch(pafs, peaks, peak_channel_inds, self.edge_inds, self.n_points,
                                     self.pafs_stride, self.max_edge_length_ratio, self.dist_penalty_weight,
                                     self.n_nodes)

    def match_candidates(self, edge_inds, edge_peak_inds, line_scores):
        return match_candidates_batch(edge_inds, edge_peak_inds, line_scores, self.n_edges)

    def group_instances(self, peaks, peak_vals, peak_channel_inds, match_edge_inds, match_src_peak_inds,
                        match_dst_peak_inds, match_line_scores):
        return group_instances_batch(peaks, peak_vals, peak_channel_inds, match_edge_inds, match_src_peak_inds,
                                     match_dst_peak_inds, match_line_scores, self.n_nodes, self.sorted_edge_inds,
                                     self.edge_types, self.min_instance_peaks, min_line_scores=self.min_line_scores)

    def predict(self, pafs, peaks, peak_vals, peak_channel_inds):
        edge_inds, edge_peak_inds, line_scores = self.score_paf_lines(pafs, peaks, peak_channel_inds)
        me, ms, md, msc = self.match_candidates(edge_inds, edge_peak_inds, line_scores)
        inst, ps, isc = self.group_instances(peaks, peak_vals, peak_channel_inds, me, ms, md, msc)
        return inst, ps, isc, edge_inds, edge_peak_inds, line_scores
