"""Frame source for the inference path: video -> batches of uint8 frames in (pinned) host memory.

Replaces, for inference, the reference's reader chain
  sleap/io/video.py:340-535          MediaVideo (cv2.VideoCapture backend, grayscale auto-detect, BGR flip)
  sleap/nn/data/providers.py:307-439 VideoReader provider (one py_function frame fetch per example)
  sleap/nn/data/dataset_ops.py:232-275, 76-160   Batcher / Prefetcher
  sleap/nn/inference.py:329-371      Predictor.make_pipeline
which decodes one frame at a time on a single thread.  Here decoding is chunked over worker
threads (cv2 releases the GIL while it decodes), each with its own VideoCapture, writing straight
into a ring of batch buffers that are page-locked when CUDA is present, so the device upload of
``sb_bottomup_submit`` is a true asynchronous DMA.  Frame order and pixel values are exactly what
``MediaVideo.get_frame`` returns (first channel for grayscale videos, BGR -> RGB otherwise).
"""
import os
import queue
import threading
from typing import List, Optional, Sequence, Union

import numpy as np


def _cv2():
    import cv2          # imported lazily: the C-ABI / kernels do not need it
    return cv2


class Video:
    """Minimal ``sleap.Video`` / ``MediaVideo`` (sleap/io/video.py:340-509, 1001-1330): random access to frames.

    ``Video.from_filename(path, grayscale=None)``; ``.shape == (frames, height, width, channels)``;
    ``video[i]`` / ``video.get_frame(i)`` -> (H, W, C) uint8; ``video.get_frames(idxs)`` -> (n, H, W, C).
    A (frames, H, W, C) array is accepted in place of a path (``NumpyVideo``, video.py:511-620).
    """

    def __init__(self, filename: Union[str, np.ndarray], grayscale: Optional[bool] = None, bgr: bool = True):
        self.bgr = bgr
        self._lock = threading.Lock()
        self._reader = None
        if isinstance(filename, np.ndarray):
            if filename.ndim != 4:
                raise ValueError("array videos must be (frames, height, width, channels)")
            self._data = filename
            self.filename = "Raw Video Data"
            self.grayscale = filename.shape[-1] == 1 if grayscale is None else grayscale
            self._n, self._h, self._w = filename.shape[:3]
            return
        self._data = None
        self.filename = os.fspath(filename)
        if not os.path.exists(self.filename):
            raise FileNotFoundError(f"Could not find filename video filename named {self.filename}")   # video.py:381-386
        cap = self._open()
        cv2 = _cv2()
        self._n = int(cap.get(cv2.CAP_PROP_FRAME_COUNT))
        self._w = int(cap.get(cv2.CAP_PROP_FRAME_WIDTH))
        self._h = int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))
        if grayscale is None:                      # auto-detect on the first frame (video.py:392-397)
            ok, f = cap.read()
            if not ok or f is None:
                raise KeyError(f"Unable to load frame 0 from {self}.")
            cap.set(cv2.CAP_PROP_POS_FRAMES, 0)
            grayscale = bool(np.all(f[..., 0] == f[..., -1]))
        self.grayscale = bool(grayscale)

    @classmethod
    def from_filename(cls, filename, grayscale: Optional[bool] = None, **kwargs):
        return cls(filename, grayscale=grayscale, **kwargs)

    @classmethod
    def from_numpy(cls, array, **kwargs):
        return cls(np.asarray(array), **kwargs)

    def _open(self):
        if self._reader is None:
            self._reader = _cv2().VideoCapture(self.filename)
            if not self._reader.isOpened():
                raise IOError(f"cv2 could not open {self.filename}")
        return self._reader

    def __repr__(self):
        return f"Video(filename={self.filename!r}, shape={self.shape})"

    @property
    def frames(self):
        return self._n

    num_frames = frames

    @property
    def height(self):
        return self._h

    @property
    def width(self):
        return self._w

    @property
    def channels(self):
        if self._data is not None:
            return self._data.shape[-1]
        return 1 if self.grayscale else 3

    @property
    def shape(self):
        return (self.frames, self.height, self.width, self.channels)

    def __len__(self):
        return self.frames

    def convert(self, frame):
        """cv2 BGR frame -> what ``MediaVideo.get_frame`` returns (video.py:501-507)."""
        if self.grayscale:
            frame = frame[..., 0][..., None]
        if self.bgr:
            frame = frame[..., ::-1]
        return frame

    def get_frame(self, idx: int) -> np.ndarray:
        if self._data is not None:
            if not 0 <= idx < self._n:
                raise KeyError(f"Unable to load frame {idx} from {self}.")
            return self._data[idx]
        cv2 = _cv2()
        with self._lock:
            cap = self._open()
            if cap.get(cv2.CAP_PROP_POS_FRAMES) != idx:
                cap.set(cv2.CAP_PROP_POS_FRAMES, idx)
            ok, frame = cap.read()
        if not ok or frame is None:
            raise KeyError(f"Unable to load frame {idx} from {self}.")      # video.py:495-496
        return np.ascontiguousarray(self.convert(frame))

    def get_frames(self, idxs: Sequence[int]) -> np.ndarray:
        return np.stack([self.get_frame(int(i)) for i in idxs])

    def __getitem__(self, key):
        if isinstance(key, slice):
            return self.get_frames(range(*key.indices(self._n)))
        if isinstance(key, (list, tuple, np.ndarray, range)):
            return self.get_frames(key)
        return self.get_frame(int(key))


class VideoReader:
    """Provider over a ``Video`` (sleap/nn/data/providers.py:307-439): ``video``, ``example_indices``,
    ``from_filepath``; iterating yields the reference's example dicts (``image, raw_image_size, video_ind,
    frame_ind, scale``)."""

    def __init__(self, video: Video, example_indices: Optional[Sequence[int]] = None):
        self.video = video
        self.example_indices = example_indices

    @classmethod
    def from_filepath(cls, filename, example_indices=None, **kwargs):
        return cls(Video.from_filename(filename, **kwargs), example_indices)

    @property
    def output_keys(self) -> List[str]:
        return ["image", "raw_image_size", "video_ind", "frame_ind", "scale"]

    @property
    def videos(self):
        return [self.video]

    def indices(self) -> np.ndarray:
        if self.example_indices is None:
            return np.arange(len(self.video), dtype=np.int64)
        return np.asarray(list(self.example_indices), dtype=np.int64)

    def __len__(self):
        return len(self.indices())

    def __iter__(self):
        for i in self.indices():
            img = self.video.get_frame(int(i))
            yield {"image": img, "raw_image_size": np.asarray(img.shape, np.int32), "video_ind": 0,
                   "frame_ind": np.int64(i), "scale": np.ones(2, np.float32)}

    make_dataset = __iter__


def _host_buffer(shape, pinned: bool):
    """uint8 batch buffer; page-locked through torch when a CUDA device is present."""
    if pinned:
        try:
            import torch
            if torch.cuda.is_available():
                t = torch.empty(shape, dtype=torch.uint8).pin_memory()
                return t.numpy(), t
        except Exception:
            pass
    a = np.empty(shape, np.uint8)
    return a, a


class FrameFeeder:
    """Ordered batches of frames from a video, decoded ahead of the consumer by worker threads.

    The frame list (``example_indices`` or the whole video) is cut into batches of ``batch_size``
    and the batches into chunks of ``chunk_batches``; worker ``w`` decodes chunks ``w, w + n, ...`` with
    its own ``VideoCapture`` (one seek per chunk when the indices are consecutive, sequential reads
    after it).  Every batch lands in one slot of a ring of ``depth`` host buffers; the consumer gets
    them strictly in order.  A slot is handed back to the decoders once the consumer has moved
    ``hold`` batches past it, so the last ``hold`` batches returned stay valid (the double-buffered
    device pipeline still reads batch k while it asks for k + 1).

    Sequence protocol (what ``InferenceModel.predict_batches`` needs): ``len(feeder)`` frames,
    ``feeder[a:b]`` for consecutive batch-aligned slices.  ``for inds, batch in feeder.batches()`` is
    the generator form.
    """

    def __init__(self, source, batch_size: int = 4, n_workers: int = 4, chunk_batches: int = 8, depth: Optional[int] = None,
                 pinned: bool = True, hold: int = 2):
        if isinstance(source, VideoReader):
            video, inds = source.video, source.indices()
        elif isinstance(source, Video):
            video, inds = source, np.arange(len(source), dtype=np.int64)
        else:
            video = Video.from_filename(source)
            inds = np.arange(len(video), dtype=np.int64)
        self.video, self.inds = video, inds
        self.batch_size = int(batch_size)
        self.n_batches = (len(inds) + self.batch_size - 1) // self.batch_size
        self.chunk_batches = max(1, int(chunk_batches))
        self.n_workers = max(1, min(int(n_workers), max(1, (self.n_batches + self.chunk_batches - 1) // self.chunk_batches)))
        if video._data is not None:
            self.n_workers = 1
        self.hold = int(hold)
        # every worker must be able to finish the chunk it is in while the consumer drains an earlier one
        min_depth = self.n_workers * self.chunk_batches + self.hold + 1
        self.depth = max(min_depth, depth or 0)
        H, W, C = video.height, video.width, video.channels
        self.frame_shape = (H, W, C)
        self._slots = [_host_buffer((self.batch_size, H, W, C), pinned) for _ in range(min(self.depth, max(1, self.n_batches)))]
        self.depth = len(self._slots)
        self._ready = [threading.Event() for _ in range(self.n_batches)]
        self._free = threading.Semaphore(0)         # unused; slot reuse is tracked by _released
        self._released = -1                          # highest batch index whose slot may be overwritten
        self._cv = threading.Condition()
        self._error = None
        self._stop = False
        self._next = 0                               # next batch the consumer will take
        self._threads = []
        self._started = False

    # -- sequence protocol -------------------------------------------------------------------
    def __len__(self):
        return len(self.inds)

    @property
    def shape(self):
        return (len(self.inds),) + self.frame_shape

    def __getitem__(self, key):
        if not isinstance(key, slice):
            return self.video.get_frame(int(self.inds[int(key)]))
        a, b, step = key.indices(len(self.inds))
        if step == 1 and a == self._next * self.batch_size and b == min(len(self.inds), a + self.batch_size):
            _, batch = self._take()
            return batch
        if step == 1 and a % self.batch_size == 0 and a // self.batch_size == self._next - 1 and self._started:
            k = self._next - 1                       # the batch just handed out, asked for again
            n = min(self.batch_size, len(self.inds) - k * self.batch_size)
            if b == a + n:
                return self._slots[k % self.depth][0][:n]
        return self.video.get_frames(self.inds[a:b:step])       # random access: synchronous decode

    # -- producer side -----------------------------------------------------------------------
    def _start(self):
        if self._started:
            return
        self._started = True
        for w in range(self.n_workers):
            t = threading.Thread(target=self._work, args=(w,), daemon=True, name=f"sb-decode-{w}")
            t.start()
            self._threads.append(t)

    def _wait_slot(self, k):
        """Block until batch k's ring slot is free: batch k - depth must have been released."""
        with self._cv:
            while not self._stop and k - self.depth > self._released:
                self._cv.wait(0.05)
            return not self._stop

    def _work(self, w):
        try:
            cap = None
            if self.video._data is None:
                cap = _cv2().VideoCapture(self.video.filename)
                if not cap.isOpened():
                    raise IOError(f"cv2 could not open {self.video.filename}")
            cv2 = _cv2() if cap is not None else None
            pos = -1
            n_chunks = (self.n_batches + self.chunk_batches - 1) // self.chunk_batches
            for c in range(w, n_chunks, self.n_workers):
                for k in range(c * self.chunk_batches, min(self.n_batches, (c + 1) * self.chunk_batches)):
                    if not self._wait_slot(k):
                        return
                    buf = self._slots[k % self.depth][0]
                    ids = self.inds[k * self.batch_size:(k + 1) * self.batch_size]
                    for j, fi in enumerate(ids):
                        fi = int(fi)
                        if cap is None:
                            buf[j] = self.video._data[fi]
                            continue
                        if pos != fi:
                            cap.set(cv2.CAP_PROP_POS_FRAMES, fi)
                        ok, frame = cap.read()
                        if not ok or frame is None:
                            raise KeyError(f"Unable to load frame {fi} from {self.video}.")
                        pos = fi + 1
                        buf[j] = self.video.convert(frame)
                    self._ready[k].set()
        except BaseException as e:            # surfaces in the consumer thread
            self._error = e
            for ev in self._ready:
                ev.set()

    # -- consumer side -----------------------------------------------------------------------
    def _take(self):
        self._start()
        k = self._next
        if k >= self.n_batches:
            raise IndexError("no more batches")
        self._ready[k].wait()
        if self._error is not None:
            self.close()
            raise self._error
        self._next = k + 1
        with self._cv:
            self._released = max(self._released, k - self.hold)
            self._cv.notify_all()
        ids = self.inds[k * self.batch_size:(k + 1) * self.batch_size]
        return ids, self._slots[k % self.depth][0][:len(ids)]

    def batches(self):
        """Yields ``(frame_indices, batch)``; ``batch`` is a view of a ring slot, valid until ``hold`` more
        batches have been taken."""
        while self._next < self.n_batches:
            yield self._take()

    def close(self):
        with self._cv:
            self._stop = True
            self._cv.notify_all()
        for t in self._threads:
            t.join(timeout=2.0)

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()
        return False
