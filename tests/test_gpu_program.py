"""The two programs of a forward pass (sb_model.cu).  The production program elides the stores nobody reads inside the
network: a conv output read only by its fused pool or fused residual ADD, and the fused first block's tensors.  A forward
that asks for one of those tensors runs the all-stores program instead.  Switching to it and back must leave the
production forward as it was: the same heads, byte for byte, from the same launches."""
import numpy as np
import pytest

import layer_audit as la
from test_gpu_layer_audit import _c4, _fetch, _frames, _op_kinds, _resnet

pytestmark = pytest.mark.gpu


def _alternate(spec, in_ch, imgs, monkeypatch, env):
    """A production forward (heads only), a forward that fetches every buffer the layer audit's all-buffers run fetches,
    then a production forward again.  Returns [(heads, launches)] of the three and the number of fp16 buffers fetched."""
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    w = la.synthetic_weights(A.compile_model(spec, in_ch), 5)
    model = DeviceModel(spec, w, input_channels=in_ch, precision=0)
    B, H, W, C = imgs.shape
    model.configure(B, H, W, C)
    aud = la.Audit(model.cm, model.cm.pack_weights(w), 0, imgs, _op_kinds(model, B, H, W, C))
    elided = aud.internal_buffers(True) - aud.internal_buffers(False)
    assert elided, "the production program elides no store: the all-stores program would never run"
    heads = [model.cm.head_buffers[h["name"]] for h in spec["heads"]]
    ids = [b for b in aud.bufs if b not in aud.internal_buffers(False)]
    runs = []
    for all_stores in (False, True, False):
        l0 = model.handle.gpu_launches()
        outs = _fetch(model, aud, imgs, ids) if all_stores else dict(zip(heads, model.forward(imgs)))
        runs.append(([np.asarray(outs[b]) for b in heads], model.handle.gpu_launches() - l0))
    return runs, sum(1 for b in ids if not aud.bufs[b]["f32"])


def _same(a, b):
    return all(x.shape == y.shape and x.tobytes() == y.tobytes() for x, y in zip(a, b))


def test_program_switch_c4(monkeypatch):
    """C4 without the fused first block: the programs differ only in the elided stores, so all three forwards compute the
    same heads, and the all-stores forward adds one fp16-to-fp32 conversion per fp16 buffer fetched and nothing else."""
    ((p0, l0), (a, l_all), (p1, l1)), n_half = _alternate(_c4(), 1, _frames((2, 200, 232, 1), 1), monkeypatch,
                                                          {"SB_FORCE_CONV01": "0"})
    assert _same(p0, a) and _same(p0, p1)
    assert l0 == l1
    assert l_all == l0 + n_half, (l_all, l0, n_half)


@pytest.mark.parametrize("case", ["resnet50", "conv01"])
def test_program_switch_back(case, monkeypatch):
    """The residual ADD fused into the conv epilogue (ResNet50) and the fused first block (C4, forced): the all-stores
    forward runs them as separate launches, and the production forward after it is the one before it."""
    spec, in_ch, imgs, env = {"resnet50": (_resnet("interp_add"), 3, _frames((1, 150, 176, 3), 4), {}),
                              "conv01": (_c4(), 1, _frames((2, 200, 232, 1), 1), {"SB_FORCE_CONV01": "1"})}[case]
    ((p0, l0), _, (p1, l1)), _ = _alternate(spec, in_ch, imgs, monkeypatch, env)
    assert _same(p0, p1)
    assert l0 == l1
