"""Frame sharding across GPUs (one process per GPU) and the single exchange step of the path:
an all-gather of fixed-size instance records (SURVEY 8e).  The reference is single-GPU
(sleap/nn/system.py:29-46 raises when more than one GPU is visible); frames are independent, so
ranks own contiguous chunks of every global batch and weights are replicated.

Backend: ``torch.distributed`` (NCCL over NVLink on GPUs; gloo in the CPU tests).
"""
from typing import Tuple

import numpy as np
import torch
import torch.distributed as dist


def frame_shard(n_frames: int, rank: int, world: int) -> slice:
    """Contiguous chunk of a global batch owned by ``rank`` (remainder spread over the first ranks)."""
    base, rem = divmod(n_frames, world)
    start = rank * base + min(rank, rem)
    return slice(start, start + base + (1 if rank < rem else 0))


def record_width(max_instances: int, n_nodes: int) -> int:
    """Floats per frame record: peaks | peak values | instance scores | n_valid | flags, padded to a multiple of 4
    (= ``sb_record_width`` of the library: the grouping kernel writes exactly this record)."""
    return (max_instances * n_nodes * 3 + max_instances + 2 + 3) // 4 * 4


def pack_records(instance_peaks, instance_peak_vals, instance_scores, n_valid, flags=None) -> torch.Tensor:
    """(B,I,C,2), (B,I,C), (B,I), (B,) [, (B,)] -> (B, record_width) float32 records (tensors, any device) -- the host-side
    twin of the record the grouping kernel writes on the device."""
    B, I, C = instance_peaks.shape[0], instance_peaks.shape[1], instance_peaks.shape[2]
    rec = torch.zeros((B, record_width(I, C)), dtype=torch.float32, device=instance_peaks.device)
    o = I * C * 3 + I
    rec[:, :o] = torch.cat([instance_peaks.reshape(B, -1), instance_peak_vals.reshape(B, -1), instance_scores.reshape(B, -1)], dim=1)
    rec[:, o] = n_valid.reshape(B).to(torch.float32)
    if flags is not None:
        rec[:, o + 1] = flags.reshape(B).to(torch.float32)
    return rec


def unpack_records(rec: torch.Tensor, max_instances: int, n_nodes: int):
    B, I, C = rec.shape[0], max_instances, n_nodes
    o = 0
    peaks = rec[:, o:o + I * C * 2].reshape(B, I, C, 2); o += I * C * 2
    vals = rec[:, o:o + I * C].reshape(B, I, C); o += I * C
    scores = rec[:, o:o + I]; o += I
    n_valid = rec[:, o].round().to(torch.int64)
    return peaks, vals, scores, n_valid


def all_gather_records(local: torch.Tensor, out: torch.Tensor = None) -> torch.Tensor:
    """Every rank ends up with the records of the whole global batch, in frame order
    (rank-major = frame order because shards are contiguous and equally sized)."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    if world == 1:
        return local
    if out is None:
        out = torch.empty((world * local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    if dist.get_backend() == "nccl":
        dist.all_gather_into_tensor(out, local)
    else:
        parts = [torch.empty_like(local) for _ in range(world)]
        dist.all_gather(parts, local)
        out.copy_(torch.cat(parts, dim=0))
    return out


def predict_sharded(predict_on_batch, frames, global_batch: int, max_instances: int, n_nodes: int, device=None):
    """Frame-sharded prediction over all ranks of the default process group (SURVEY 8e).

    Every rank calls this with the same ``frames`` (array-like, ``len`` + slicing).  Each global batch of
    ``global_batch`` frames is cut into contiguous per-rank shards (``frame_shard``); a rank runs
    ``predict_on_batch(shard)`` -- the ``predict_on_batch`` of a bottom-up / top-down / single-instance inference
    model: a dict with ``instance_peaks (b, i, C, 2)``, ``instance_peak_vals (b, i, C)``, optional
    ``instance_scores (b, i)`` and ``n_valid (b,)`` -- packs fixed-size records and joins the ONE exchange step of the
    path, an all-gather (NCCL on GPUs, gloo on CPU).  Yields, on every rank, one dict per global batch in frame order
    with the arrays NaN-padded to ``max_instances``.  Ragged tails (fewer frames than ranks) are handled by padding
    the local record block to the largest shard and dropping the padding rows after the gather."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    I, C = max_instances, n_nodes
    width = record_width(I, C)
    n = len(frames)
    for g0 in range(0, n, global_batch):
        g1 = min(n, g0 + global_batch)
        nb = g1 - g0
        sl = frame_shard(nb, rank, world)
        cap = -(-nb // world)                                     # largest shard
        rec = torch.full((cap, width), float("nan"), dtype=torch.float32)
        nv_col = I * C * 3 + I
        rec[:, nv_col] = -1.0                                     # n_valid = -1 marks a padding row
        if sl.stop > sl.start:
            out = predict_on_batch(frames[g0 + sl.start:g0 + sl.stop])
            b = sl.stop - sl.start
            ip = np.full((b, I, C, 2), np.nan, np.float32); iv = np.full((b, I, C), np.nan, np.float32)
            isc = np.full((b, I), np.nan, np.float32)
            k = min(I, out["instance_peaks"].shape[1])
            ip[:, :k] = out["instance_peaks"][:, :k]
            iv[:, :k] = out["instance_peak_vals"][:, :k]
            if "instance_scores" in out:
                isc[:, :k] = out["instance_scores"][:, :k]
            nv = np.minimum(np.asarray(out.get("n_valid", np.full(b, k)), np.int64), I)
            rec[:b] = pack_records(torch.from_numpy(ip), torch.from_numpy(iv), torch.from_numpy(isc), torch.from_numpy(nv))
        if device is not None:
            rec = rec.to(device)
        allrec = all_gather_records(rec).cpu()
        keep = allrec[:, nv_col] >= 0                             # rank-major order == frame order (contiguous shards)
        peaks, vals, scores, n_valid = unpack_records(allrec[keep], I, C)
        assert peaks.shape[0] == nb, (peaks.shape, nb)
        yield {"instance_peaks": peaks.numpy(), "instance_peak_vals": vals.numpy(), "instance_scores": scores.numpy(),
               "n_valid": n_valid.numpy(), "frame_ind": np.arange(g0, g1)}


class PeerGather:
    """The path's ONE exchange step without a collective call: every rank's grouping kernel stores its frames' records
    straight into a gather window in each peer's HBM (CUDA IPC mappings over NVLink / NVSwitch; ``sb_gather_*`` in
    include/sleap_b200.h).  This class only does the out-of-band part: it exchanges the 64-byte IPC handles of the
    windows through ``torch.distributed`` (any backend) and maps the peers.

    ``model``: a configured bottom-up ``DeviceModel`` (``sb_bottomup_configure`` done).  After construction every
    ``sb_infer_bottomup*`` / ``sb_bottomup_submit`` call of that model is one exchange *step*.  The host-facing calls
    (``sb_bottomup_submit`` / ``collect``, and ``sb_infer_bottomup``, which is a submit into slot 0 and its collect)
    consume their own step: the whole gather window rides on the result copy they do anyway (``gathered``); the
    device-resident call (``sb_infer_bottomup_dev``) leaves consumption to ``consume_next_dev``.  A producer blocks only when it is ``generations`` steps ahead of the slowest consumer."""

    def __init__(self, model, generations: int = 8, group=None):
        import ctypes
        self.model, self.handle = model, model.handle
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.generations = int(generations)
        buf = ctypes.create_string_buffer(64)
        self.handle.call("sb_gather_init", model.model_id, self.rank, self.world, self.generations, buf)
        handles = [None] * self.world
        if self.world > 1:
            dist.all_gather_object(handles, bytes(buf.raw), group=group)
        else:
            handles[0] = bytes(buf.raw)
        blob = ctypes.create_string_buffer(b"".join(handles), 64 * self.world)
        err = None
        try:
            self.handle.call("sb_gather_connect", model.model_id, blob)
        except Exception as e:                       # e.g. peer access not permitted between two of the GPUs
            err = e
        if self.world > 1:                           # all ranks agree before anybody pushes (or everybody falls back)
            dev = torch.device("cuda", self.handle.device_id) if dist.get_backend(group) == "nccl" else torch.device("cpu")
            ok = torch.tensor([0 if err else 1], dtype=torch.int32, device=dev)
            dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
            if int(ok.item()) == 0:
                try:
                    self.handle.call("sb_gather_close", model.model_id)
                finally:
                    raise RuntimeError(f"peer-memory exchange unavailable on at least one rank ({err})")
        elif err:
            raise err
        model.peer_gather = self

    def _status(self):
        import ctypes
        st, n, c = ctypes.c_int32(0), ctypes.c_int64(0), ctypes.c_int64(0)
        self.handle.call("sb_gather_status", self.model.model_id, ctypes.byref(st), ctypes.byref(n), ctypes.byref(c))
        if st.value:
            raise RuntimeError(f"record exchange reported status {st.value} (1: arrivals timed out, 2: acknowledgements timed out)")
        return int(n.value), int(c.value)

    def pushed(self) -> int:
        return self._status()[0]

    @property
    def consumed(self) -> int:
        return self._status()[1]

    def consume_next_dev(self):
        """Device consumer of the oldest unconsumed step (wait + acknowledge, queued on the post-processing stream)."""
        self.handle.call("sb_gather_consume_dev", self.model.model_id, -1)

    def window(self, step: int):
        """(device pointer, float count) of the [world][Bmax][width] window that holds ``step``."""
        from ctypes import byref, c_int64, c_void_p
        p, n = c_void_p(), c_int64()
        self.handle.call("sb_gather_window", self.model.model_id, int(step), byref(p), byref(n))
        return p.value, n.value

    def gathered(self, slot: int, B: int, max_instances: int, n_nodes: int):
        """Every rank's records of the batch last collected from ``slot`` (0 / 1; 0 after the synchronous
        sb_infer_bottomup): (world*B, width) in rank-major (= frame) order + frames pushed per rank.  Host memory only: the
        window came over with the batch's own result copy."""
        from sleap_b200._lib import ptr
        w = record_width(max_instances, n_nodes)
        out = np.zeros((self.world, B, w), np.float32)
        counts = np.zeros((self.world,), np.int32)
        self.handle.call("sb_bottomup_gathered", self.model.model_id, int(slot), int(B), ptr(out), ptr(counts))
        return out.reshape(self.world * B, w), counts

    def close(self):
        self.model.peer_gather = None
        self.handle.call("sb_gather_close", self.model.model_id)
