"""sleap_b200: H100-native (sm_90a) batched-frame pose inference path with the
``sleap.nn.inference`` surface.  All device work goes through ``libsleapb200.so`` (C-ABI);
there is no CPU fallback: using any op without a CUDA device raises."""
__version__ = "0.1.0"

from sleap_b200 import _lib  # noqa: F401


def load_model(*args, **kwargs):
    """Mirror of ``sleap.load_model`` (sleap/nn/inference.py:4865)."""
    from sleap_b200.nn.inference import load_model as _lm

    return _lm(*args, **kwargs)


def load_video(filename, **kwargs):
    """Mirror of ``sleap.load_video`` (sleap/io/video.py:1638): a ``Video`` over a media file."""
    from sleap_b200.io.video import Video

    return Video.from_filename(filename, **kwargs)


def load_file(filename, **kwargs):
    """Mirror of ``sleap.load_file`` (sleap/io/dataset.py:2747) for the ``.slp`` (HDF5) labels format."""
    from sleap_b200.io.labels import Labels

    return Labels.load_file(filename, **kwargs)
