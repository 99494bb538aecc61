"""The argument checks of b200mvs_depthmap_confidence_clean_device and b200mvs_depthmap_cleanup_device that come before
any device call, with their exact codes and messages, on a machine without a GPU: the pointers are never dereferenced.
An empty batch returns 0 without touching anything, NULL arrays included."""
import ctypes as C

import numpy as np
import pytest

INVALID = -1
CC = "b200mvs_depthmap_confidence_clean_device"
CU = "b200mvs_depthmap_cleanup_device"
BASE = 1 << 40                    # a fake, 4-byte aligned address; nothing at or after it is read


def _lib():
    from mve_b200 import depthmap as D
    return D._lib()


def _ptrs(addrs):
    return (C.c_void_p * max(len(addrs), 1))(*addrs)


def _i32(v):
    return np.ascontiguousarray(v, np.int32)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _conf_clean(L, n, depth, conf, ws, hs):
    return L.b200mvs_depthmap_confidence_clean_device(0, n, depth, conf, _p(ws), _p(hs), None)


def _cleanup(L, n, depth, ws, hs, thres, out):
    return L.b200mvs_depthmap_cleanup_device(0, n, depth, _p(ws), _p(hs), _p(thres), out, None)


def _expect(L, rc, msg):
    assert (rc, L.b200mvs_last_error(None).decode()) == (INVALID, msg)
    assert L.b200mvs_depthmap_last_error().decode() == msg


# two 8 x 4 maps (128 bytes each) far apart, unless a case moves them
W2, H2 = _i32([8, 8]), _i32([4, 4])
T2 = np.array([1, 1], np.int64)
A, B, X, Y = BASE, BASE + (1 << 20), BASE + (2 << 20), BASE + (3 << 20)


def test_empty_batch_touches_nothing():
    L = _lib()
    assert L.b200mvs_depthmap_confidence_clean_device(0, 0, None, None, None, None, None) == 0
    assert L.b200mvs_depthmap_cleanup_device(0, 0, None, None, None, None, None, None) == 0
    # with a device that does not exist: nothing is looked at
    assert L.b200mvs_depthmap_cleanup_device(999, 0, None, None, None, None, None, None) == 0


@pytest.mark.parametrize("fn", [CC, CU])
def test_negative_count(fn):
    L = _lib()
    rc = getattr(L, fn)(*([0, -1] + [None] * (5 if fn == CC else 6)))
    _expect(L, rc, "%s: n_maps is -1, must not be negative" % fn)


CONF_CASES = [
    ("null depth array", lambda L: _conf_clean(L, 2, None, _ptrs([X, Y]), W2, H2), "depth_dev is NULL"),
    ("null conf array", lambda L: _conf_clean(L, 2, _ptrs([A, B]), None, W2, H2), "conf_dev is NULL"),
    ("null widths", lambda L: _conf_clean(L, 2, _ptrs([A, B]), _ptrs([X, Y]), None, H2), "widths is NULL"),
    ("null heights", lambda L: _conf_clean(L, 2, _ptrs([A, B]), _ptrs([X, Y]), W2, None), "heights is NULL"),
    ("null depth map", lambda L: _conf_clean(L, 2, _ptrs([A, None]), _ptrs([X, Y]), W2, H2), "depth_dev[1] is NULL"),
    ("null conf map", lambda L: _conf_clean(L, 2, _ptrs([A, B]), _ptrs([None, Y]), W2, H2), "conf_dev[0] is NULL"),
    ("width", lambda L: _conf_clean(L, 2, _ptrs([A, B]), _ptrs([X, Y]), _i32([8, 0]), H2), "widths[1] is 0, must be at least 1"),
    ("height", lambda L: _conf_clean(L, 2, _ptrs([A, B]), _ptrs([X, Y]), W2, _i32([-3, 4])), "heights[0] is -3, must be at least 1"),
    ("too large", lambda L: _conf_clean(L, 2, _ptrs([A, B]), _ptrs([X, Y]), _i32([8, 65536]), _i32([4, 65536])),
     "map 1 has 4294967296 pixels (widths[1] x heights[1]), more than 4294967280"),
    ("depth on its conf", lambda L: _conf_clean(L, 2, _ptrs([A, B]), _ptrs([X, B]), W2, H2), "depth_dev[1] overlaps conf_dev[1]"),
    ("depth on its conf, shifted", lambda L: _conf_clean(L, 2, _ptrs([A, B]), _ptrs([A + 64, Y]), W2, H2),
     "depth_dev[0] overlaps conf_dev[0]"),
    ("depth on depth", lambda L: _conf_clean(L, 2, _ptrs([A, A + 124]), _ptrs([X, Y]), W2, H2), "depth_dev[0] overlaps depth_dev[1]"),
    ("depth on a later conf", lambda L: _conf_clean(L, 2, _ptrs([A, B]), _ptrs([X, A - 4]), W2, H2), "depth_dev[0] overlaps conf_dev[1]"),
]

CLEANUP_CASES = [
    ("null depth array", lambda L: _cleanup(L, 2, None, W2, H2, T2, _ptrs([X, Y])), "depth_dev is NULL"),
    ("null out array", lambda L: _cleanup(L, 2, _ptrs([A, B]), W2, H2, T2, None), "out_dev is NULL"),
    ("null widths", lambda L: _cleanup(L, 2, _ptrs([A, B]), None, H2, T2, _ptrs([X, Y])), "widths is NULL"),
    ("null heights", lambda L: _cleanup(L, 2, _ptrs([A, B]), W2, None, T2, _ptrs([X, Y])), "heights is NULL"),
    ("null thres", lambda L: _cleanup(L, 2, _ptrs([A, B]), W2, H2, None, _ptrs([X, Y])), "thres is NULL"),
    ("null depth map", lambda L: _cleanup(L, 2, _ptrs([None, B]), W2, H2, T2, _ptrs([X, Y])), "depth_dev[0] is NULL"),
    ("null out map", lambda L: _cleanup(L, 2, _ptrs([A, B]), W2, H2, T2, _ptrs([X, None])), "out_dev[1] is NULL"),
    ("width", lambda L: _cleanup(L, 2, _ptrs([A, B]), _i32([0, 8]), H2, T2, _ptrs([X, Y])), "widths[0] is 0, must be at least 1"),
    ("height", lambda L: _cleanup(L, 2, _ptrs([A, B]), W2, _i32([4, 0]), T2, _ptrs([X, Y])), "heights[1] is 0, must be at least 1"),
    ("too large", lambda L: _cleanup(L, 2, _ptrs([A, B]), _i32([65536, 8]), _i32([65536, 4]), T2, _ptrs([X, Y])),
     "map 0 has 4294967296 pixels (widths[0] x heights[0]), more than 4294967280"),
    ("outputs overlap", lambda L: _cleanup(L, 2, _ptrs([A, B]), W2, H2, T2, _ptrs([X, X + 64])), "out_dev[0] overlaps out_dev[1]"),
    ("same output twice", lambda L: _cleanup(L, 2, _ptrs([A, B]), W2, H2, T2, _ptrs([Y, Y])), "out_dev[0] overlaps out_dev[1]"),
    ("output on another map", lambda L: _cleanup(L, 2, _ptrs([A, B]), W2, H2, T2, _ptrs([B, Y])), "out_dev[0] overlaps depth_dev[1]"),
    ("output shifted on its map", lambda L: _cleanup(L, 2, _ptrs([A, B]), W2, H2, T2, _ptrs([X, B + 4])),
     "out_dev[1] overlaps depth_dev[1]"),
    ("in place, then overlapping", lambda L: _cleanup(L, 2, _ptrs([A, A + 64]), W2, H2, T2, _ptrs([A, Y])),
     "out_dev[0] overlaps depth_dev[1]"),
]


@pytest.mark.parametrize("name,call,msg", CONF_CASES, ids=[c[0] for c in CONF_CASES])
def test_confidence_clean_device_errors(name, call, msg):
    L = _lib()
    _expect(L, call(L), "%s: %s" % (CC, msg))


@pytest.mark.parametrize("name,call,msg", CLEANUP_CASES, ids=[c[0] for c in CLEANUP_CASES])
def test_cleanup_device_errors(name, call, msg):
    L = _lib()
    _expect(L, call(L), "%s: %s" % (CU, msg))


def test_map_checks_come_before_overlaps():
    L = _lib()
    # map 0 overlaps map 1's output, and map 1 has no width: the map's own fields are checked first
    rc = _cleanup(L, 2, _ptrs([A, B]), _i32([8, 0]), H2, T2, _ptrs([A + 4, Y]))
    _expect(L, rc, "%s: widths[1] is 0, must be at least 1" % CU)
