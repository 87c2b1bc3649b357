"""The cache key DeviceModel.configure_chain compares before it configures a post-processing chain again."""
from ctypes import c_float, c_void_p

import numpy as np
import pytest

from sleap_b200._lib import BottomUpParams, CentroidParams, GlobalParams, MultiClassParams
from sleap_b200.nn.model import chain_key


def _filled(cls, edges=None, sorted_edges=None):
    p = cls()
    for i, (name, typ) in enumerate(cls._fields_):
        if typ is c_void_p:
            continue
        setattr(p, name, float(i) + 0.25 if typ is c_float else i + 1)
    if edges is not None:
        p.edges, p.sorted_edge_inds = edges.ctypes.data, sorted_edges.ctypes.data
    return p


def _arrays(cls):
    if cls is not BottomUpParams:
        return ()
    return np.array([[0, 1], [1, 2]], np.int32), np.array([0, 1], np.int32)


@pytest.mark.parametrize("cls", [GlobalParams, CentroidParams, MultiClassParams, BottomUpParams])
def test_every_field_is_in_the_key(cls):
    arrays = _arrays(cls)
    base = chain_key(_filled(cls, *arrays), *arrays)
    assert chain_key(_filled(cls, *arrays), *arrays) == base
    for name, typ in cls._fields_:
        if typ is c_void_p:
            continue
        p = _filled(cls, *arrays)
        setattr(p, name, getattr(p, name) + (0.5 if typ is c_float else 1))
        assert chain_key(p, *arrays) != base, name


def test_edges_by_value():
    e1, s1 = _arrays(BottomUpParams)
    e2, s2 = e1.copy(), s1.copy()
    key = chain_key(_filled(BottomUpParams, e1, s1), e1, s1)
    assert chain_key(_filled(BottomUpParams, e2, s2), e2, s2) == key     # other pointers, same edges
    e2[1, 1] = 0
    assert chain_key(_filled(BottomUpParams, e2, s2), e2, s2) != key
    s2[:] = s1[::-1]
    assert chain_key(_filled(BottomUpParams, e1, s2), e1, s2) != key
